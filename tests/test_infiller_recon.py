"""Reconstruction mode of the motion infiller: MotionInfillerVAE.inference(batch, sample_num, recon=True, multi_step=True).

CPU: the float32 oracle (tests/infiller_recon_oracle.py) against the executed reference (tests/golden/infiller_recon.npz), and the
stand-in prior weights pinned by a hash (the posterior's weights come from a seed of their own, so adding them moved no other weight).
GPU: the library against the golden and, element by element, against the float64 oracle under the block bound of
test_prior_float64 (C = 4, R = 8, one block per 30-frame window) at B on each side of the GEMM dispatch edges; the infer half of a
recon call against a plain infer call, the caller's tensors, graph replay, and the errors.
"""
import hashlib

import numpy as np
import pytest
import torch

from infiller_recon_cases import CASES, case_batch, infiller_state
from infiller_recon_oracle import recon_model
from test_prior_float64 import block_bound, peak_floor, window_blocks, worst
from glamr_b200.synthetic_nets import make_infiller_posterior_state, make_prior_states, infiller_posterior_param_shapes

DEV = 'cuda:0'
GOLDEN = 'infiller_recon'
TAGS = [c[0] for c in CASES]
PRIOR_STATES_SHA256 = '11d80d0d25e1ebc4d9f4be08045a3a8635f78d29236a92b7c262b42cadd377ca'


def _golden():
    from helpers import load_golden
    return load_golden(GOLDEN)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize('tag', TAGS)
def test_oracle_recon_matches_reference(tag):
    g = _golden()
    B, T = (int(x) for x in g[f'{tag}/shape'])
    batch = case_batch(tag)
    assert tuple(batch['pose'].shape) == (B, T, 72)
    before = {k: v.clone() for k, v in batch.items()}
    out = recon_model(infiller_state()).recon(batch)
    for k in ('recon_out_pose', 'recon_out_body_pose'):
        np.testing.assert_allclose(out[k].numpy(), g[f'{tag}/{k}'], atol=2e-5, err_msg=f'{tag} {k}')
    assert all(torch.equal(batch[k], before[k]) for k in batch)


def test_prior_stand_in_weights_unchanged():
    """make_prior_states(1234) is what nets.npz, trajpred_multistep.npz and the global-opt goldens were generated with"""
    h = hashlib.sha256()
    for st in make_prior_states(1234):
        for k in sorted(st):
            a = np.ascontiguousarray(st[k], dtype=np.float32)
            h.update(k.encode())
            h.update(str(a.shape).encode())
            h.update(a.tobytes())
    assert h.hexdigest() == PRIOR_STATES_SHA256


def test_posterior_weights_are_their_own():
    post = make_infiller_posterior_state()
    assert set(post) == set(infiller_posterior_param_shapes()) and all(k.startswith('data_encoder.') for k in post)
    assert not set(post) & set(make_prior_states(1234)[0])


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope='module')
def mfiller():
    from glamr_b200.motion_traj import MotionInfillerVAE
    return MotionInfillerVAE(infiller_state(), torch.device(DEV))


def _dev(batch):
    return {k: v.to(DEV) for k, v in batch.items()}


@pytest.mark.gpu
@pytest.mark.parametrize('tag', TAGS)
def test_recon_matches_reference(tag, mfiller):
    g = _golden()
    out = mfiller.inference(_dev(case_batch(tag)), sample_num=1, recon=True, multi_step=True)
    for k in ('recon_out_pose', 'recon_out_body_pose'):
        np.testing.assert_allclose(out[k].cpu().numpy(), g[f'{tag}/{k}'], atol=1e-4, err_msg=f'{tag} {k}')


def recon_inputs(B, T, seed, gaps=(), ibp=False):
    g = torch.Generator().manual_seed(seed)
    pose = torch.randn(B, T, 72, generator=g) * 0.3
    mask = (torch.rand(B, T, generator=g) > 0.3).float()
    mask[:, :10] = 1
    mask[0] = 1                                               # one sequence with every frame visible
    for b, s, e in gaps:
        mask[b, s:e] = 0
    batch = {'pose': pose, 'pose_mask': mask[..., None].repeat(1, 1, 72), 'frame_mask': mask}
    if ibp:
        batch['in_body_pose'] = (pose[..., 3:] + 0.05 * torch.randn(B, T, 69, generator=g)) * mask[..., None]
    return batch


# B <= 5: every Linear on the skinny FP32 GEMM (50 B <= 256); B = 6..8: the posterior's 32-row Linears skinny, the 50-row ones on the
# tensor cores; B >= 9: all of them on the tensor cores.  T: one window, ragged last windows, a single frame past a window edge.
F64_CASES = [(1, 40, [], False), (1, 101, [(0, 40, 80)], True), (5, 71, [(2, 30, 71)], False), (6, 41, [(1, 12, 40)], True),
             (8, 100, [(3, 45, 75)], False), (9, 71, [(4, 5, 50)], True), (16, 130, [(7, 60, 130)], False)]


@pytest.mark.gpu
@pytest.mark.parametrize('B,T,gaps,ibp', F64_CASES, ids=[f'{c[0]}x{c[1]}' for c in F64_CASES])
def test_recon_matches_float64(B, T, gaps, ibp, mfiller):
    batch = recon_inputs(B, T, 1000 + 7 * B + T, gaps, ibp)
    got = mfiller.inference(_dev(batch), sample_num=1, recon=True)['recon_out_body_pose'].transpose(0, 1)
    o32 = recon_model(infiller_state()).recon(batch)['recon_out_body_pose'].transpose(0, 1)
    o64 = recon_model(infiller_state(), torch.float64).to(DEV).recon(_dev(batch))['recon_out_body_pose'].transpose(0, 1).cpu()
    r = worst(got, o64, block_bound(o32, o64, window_blocks(T), peak_floor(o64)))
    print(f'recon {B}x{T}: {r:.3g}')
    assert r <= 1.0, f'worst |o - o64| / bound = {r}'


@pytest.mark.gpu
@pytest.mark.parametrize('B,T,S', [(1, 100, 3), (3, 71, 1)])
def test_recon_call_keeps_infer_outputs_and_inputs(B, T, S, mfiller):
    """the infer half of a recon=True call equals a recon=False call with the same latents, bit for bit; the infer root is the
    ground-truth root; no caller tensor is written"""
    batch = _dev(recon_inputs(B, T, 5 + B, [(0, 30, 60)], ibp=B > 1))
    batch['in_motion_latent'] = torch.randn(int(np.ceil((T - 10) / 30)), 128, generator=torch.Generator().manual_seed(B)).to(DEV)
    before = {k: v.clone() for k, v in batch.items()}
    rec = mfiller.inference(batch, sample_num=S, recon=True)
    assert all(torch.equal(batch[k], before[k]) for k in batch)
    inf = mfiller.inference(batch, sample_num=S, recon=False)
    assert all(torch.equal(batch[k], before[k]) for k in batch)
    for k in ('infer_out_body_pose', 'infer_out_pose'):
        assert torch.equal(rec[k], inf[k]), k
    assert rec['infer_out_pose'].shape == (B, S, T, 72)
    assert torch.equal(rec['infer_out_pose'][..., :3], batch['pose'][:, None, :, :3].expand(-1, S, -1, -1))
    assert torch.equal(rec['recon_out_pose'][..., :3], batch['pose'][..., :3])
    assert torch.equal(rec['recon_out_pose'][..., 3:], rec['recon_out_body_pose'])
    if 'in_body_pose' not in batch:
        # the default input body pose: the infer sweep without `pose` on (pose * pose_mask)[..., 3:] gives the same body
        plain = {'in_body_pose': (batch['pose'] * batch['pose_mask'])[..., 3:], 'frame_mask': batch['frame_mask'],
                 'in_motion_latent': batch['in_motion_latent']}
        assert torch.equal(mfiller.inference(plain, sample_num=S)['infer_out_body_pose'], inf['infer_out_body_pose'])


@pytest.mark.gpu
def test_recon_graph_replay_is_bit_identical_to_eager(mfiller):
    from glamr_b200.motion_traj import _GraphCache
    saved = mfiller.graphs
    try:
        for B, T in [(1, 100), (9, 71)]:
            ins = [_dev(recon_inputs(B, T, seed, [(0, 20, 45)])) for seed in (1, 2)]
            mfiller.graphs = _GraphCache(enabled=False)
            eager = [mfiller.inference(x, recon=True)['recon_out_pose'] for x in ins]
            mfiller.graphs = _GraphCache(enabled=True)
            for k, x in enumerate([ins[0], ins[0], ins[1]]):      # warm-up + capture, replay, replay with new inputs
                assert torch.equal(mfiller.inference(x, recon=True)['recon_out_pose'], eager[0 if k < 2 else 1]), (B, T, k)
            assert any(key[0] == 'recon' and e['graph'] is not None for key, e in mfiller.graphs.entries.items())
    finally:
        mfiller.graphs = saved


@pytest.mark.gpu
def test_recon_errors(mfiller, smpl_assets):
    from glamr_b200.motion_traj import MotionInfillerVAE, MotionTrajJointModel
    from glamr_b200.smpl import SMPL
    batch = _dev(recon_inputs(2, 40, 3))
    with pytest.raises(ValueError, match='pose'):
        mfiller.inference({'in_body_pose': batch['pose'][..., 3:], 'frame_mask': batch['frame_mask']}, recon=True)
    with pytest.raises(ValueError, match='pose_mask'):
        mfiller.inference({'pose': batch['pose'], 'frame_mask': batch['frame_mask']}, recon=False)
    with pytest.raises(NotImplementedError):
        mfiller.inference({**batch, 'seq_len': [40, 30]}, recon=True)
    with pytest.raises(NotImplementedError):
        mfiller.inference(batch, recon=True, multi_step=False)
    no_post = MotionInfillerVAE(make_prior_states(1234)[0], torch.device(DEV))
    with pytest.raises(ValueError, match='data_encoder'):
        no_post.inference(batch, recon=True)
    states = (infiller_state(), make_prior_states(1234)[1])
    mt = MotionTrajJointModel(None, torch.device(DEV), None, smpl=SMPL(smpl_assets, device=DEV), states=states)
    with pytest.raises(NotImplementedError):
        mt.inference({'in_body_pose': batch['pose'][..., 3:], 'frame_mask': batch['frame_mask']}, recon=True)


@pytest.mark.gpu
def test_library_refuses_a_net_without_the_full_posterior():
    """glamr_infiller_recon_forward: a net missing any data_encoder.* tensor it reads returns GLAMR_EINVAL"""
    from glamr_b200 import lib as L
    from glamr_b200.motion_traj import _Net, _declare
    lib = L.load()
    _declare(lib)
    st = infiller_state()
    del st['data_encoder.temporal_net.layers.1.norm3.bias']
    net = _Net(st, torch.device(DEV))
    B, T = 2, 40
    pose = torch.zeros(T, B, 69, device=DEV)
    gt = torch.zeros(T, B, 69, device=DEV)
    kp = torch.zeros(B, T, dtype=torch.uint8, device=DEV)
    ws = torch.empty(int(lib.glamr_infiller_recon_workspace_floats(B)), device=DEV)
    rc = lib.glamr_infiller_recon_forward(net.h, T, B, pose.data_ptr(), gt.data_ptr(), kp.data_ptr(), ws.data_ptr(), ws.numel(),
                                          torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == -1
    rc = lib.glamr_infiller_recon_forward(net.h, T, B, pose.data_ptr(), gt.data_ptr(), kp.data_ptr(), ws.data_ptr(), ws.numel() - 1,
                                          torch.cuda.current_stream().cuda_stream)
    assert rc == -2
