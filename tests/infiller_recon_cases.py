"""The seeded inputs of the cases in tests/golden/infiller_recon.npz (the motion infiller's reconstruction sweep), shared with the
script that writes it and with the tests that read it."""
import numpy as np
import torch

from glamr_b200.synthetic_nets import make_infiller_posterior_state, make_prior_states

# (tag, B, T, gaps (sequence, first frame, end), in_body_pose given).  Sequence 0 keeps every frame visible unless a gap names it.
CASES = [('b1_t40', 1, 40, [(0, 15, 30)], False),
         ('b1_t300_ibp', 1, 300, [(0, 50, 120), (0, 200, 260), (0, 285, 300)], True),
         ('b3_t41', 3, 41, [], False),
         ('b3_t71_ibp', 3, 71, [(1, 30, 60), (2, 10, 71)], True),
         ('b8_t41', 8, 41, [(3, 20, 35), (7, 30, 41)], False),
         ('b9_t41_ibp', 9, 41, [(2, 12, 40), (8, 35, 41)], True)]


def infiller_state():
    """the stand-in infiller weights with the posterior encoder's"""
    return {**make_prior_states(1234)[0], **make_infiller_posterior_state()}


def case_seed(tag):
    return 71 + [c[0] for c in CASES].index(tag)


def case_batch(tag):
    """the inputs of a case, regenerated from its seed: pose [B,T,72] (ground truth), pose_mask [B,T,72], frame_mask [B,T],
    in_motion_latent [windows,128] (the infer sweeps' latents) and, where the case says so, an in_body_pose [B,T,69] that differs
    from the default (pose * pose_mask)[..., 3:]"""
    _, B, T, gaps, ibp = next(c for c in CASES if c[0] == tag)
    g = torch.Generator().manual_seed(case_seed(tag))
    pose = torch.randn(B, T, 72, generator=g) * 0.3
    mask = torch.ones(B, T)
    for b, s, e in gaps:
        mask[b, s:e] = 0
    batch = {'pose': pose, 'pose_mask': mask[..., None].repeat(1, 1, 72), 'frame_mask': mask,
             'in_motion_latent': torch.randn(int(np.ceil((T - 10) / 30)), 128, generator=g)}
    if ibp:
        batch['in_body_pose'] = (pose[..., 3:] + 0.05 * torch.randn(B, T, 69, generator=g)) * mask[..., None]
    return batch
