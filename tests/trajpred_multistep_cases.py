"""Windowed trajectory prediction (TrajPredVAE.inference_multi_step, traj_pred_vae.py:484-520) restated in plain torch on top of
oracle.nets, and the seeded inputs of the cases in tests/golden/trajpred_multistep.npz (shared with the script that writes it).

Everything runs in the dtype of the predictor module and its inputs, so the float64 route of test_prior_float64 works unchanged.
"""
import numpy as np
import torch

from oracle import nets as on
from oracle import rotations as rt
from oracle import traj_codec as tc

WINDOW = 100                   # seq_len of the reference's traj_pred_demo.yml
# (tag, B, T, gaps (sequence, first frame, end))
CASES = [('b2_t40', 2, 40, []), ('b1_t100', 1, 100, []), ('b2_t101', 2, 101, []),
         ('b3_t250_gaps', 3, 250, [(0, 60, 140), (1, 190, 250), (2, 95, 105)]), ('b1_t600', 1, 600, [])]


def case_batch(tag):
    """the inputs of a golden case, regenerated from its seed: in_body_pose [B,T,69], frame_mask [B,T], in_motion_latent
    [windows,128] and in_traj_latent [1,128] (which windowed prediction must ignore)"""
    i, (_, B, T, gaps) = next((i, c) for i, c in enumerate(CASES) if c[0] == tag)
    g = torch.Generator().manual_seed(31 + i)
    pose = torch.randn(B, T, 69, generator=g) * 0.3
    mask = torch.ones(B, T)
    for b, s, e in gaps:
        mask[b, s:e] = 0
    return {'in_body_pose': pose * mask[..., None], 'frame_mask': mask,
            'in_motion_latent': torch.randn(int(np.ceil((T - 10) / 30)), 128, generator=g), 'in_traj_latent': torch.randn(1, 128, generator=g)}


@torch.no_grad()
def traj_raw(tp, joint_pos, eps):
    """TrajPredictor's network: joint_pos [T,B,69] -> decoder output [T,B,11] before the frame-0 override (traj_pred_vae.py:72-92,
    :281-318); eps [1|B,128] or None (-> randn)"""
    ce, dd = tp.context_encoder, tp.data_decoder
    x = ce.in_mlp(joint_pos)
    for net in ce.temporal_net:
        x = net(x)
    ctx = ce.out_mlp(x)
    mu, logvar = torch.chunk(dd.p_z_net(dd.prior_mlp(ctx.mean(dim=0))), 2, dim=-1)
    z = mu + (eps if eps is not None else torch.randn_like(mu)) * torch.exp(0.5 * logvar)
    return dd.out_fc(dd.out_mlp(torch.cat([z.repeat(ctx.shape[0], 1, 1), ctx], dim=-1)))


@torch.no_grad()
def inference_multi_step(tp, joint_pos, seq_len, eps=None):
    """traj_pred_vae.py:484-520 (infer, sample_num 1) with TrajPredictor tp: windows of seq_len frames, the last one zero-padded in
    joint-position space (get_seg_data :484-498); each window draws its own z (eps [C,B,128] or None -> randn) and takes the default
    frame-0 override (no in_traj_latent / init_xy / init_heading reaches a window); window 0 contributes its overridden output,
    window c >= 1 its raw output with frame 0's heading vector taken from the stitched output's last frame (get_res_from_cur_data
    :500-506).  -> local [T,B,11], trans [T,B,3], orient axis-angle [T,B,3]"""
    T = joint_pos.shape[0]
    parts = []
    for c in range(int(np.ceil(T / seq_len))):
        s, e = c * seq_len, (c + 1) * seq_len
        eb = min(e, T)
        win = joint_pos[s:eb]
        if e > eb:
            win = torch.cat([win, torch.zeros((e - eb,) + win.shape[1:], dtype=win.dtype, device=win.device)], dim=0)
        out = traj_raw(tp, win, None if eps is None else eps[c]).clone()
        if c == 0:
            out[0, :, :2] = 0.0
            out[0, :, -2:] = torch.tensor([0.0, 1.0], dtype=out.dtype, device=out.device)
        else:
            out[0, :, 9:] = rt.heading_to_vec(rt.get_heading(rt.rot6d_to_quat(parts[-1][-1, :, 3:-2])))
        parts.append(out[:eb - s])
    local = torch.cat(parts, dim=0)
    trans, q = tc.local_to_global(local)
    return local, trans, rt.quat_to_aa(q)


class MotionTrajJointMultiStep(on.MotionTrajJoint):
    """oracle.nets.MotionTrajJoint with multi_step_trajpred: windows of traj_seq_len frames, eps from `in_traj_window_latent`
    [C,B,128] (randn when absent)"""

    def __init__(self, state_mfiller, state_traj, smpl, dtype=torch.float32, traj_seq_len=WINDOW):
        super().__init__(state_mfiller, state_traj, smpl, dtype)
        self.traj_seq_len = traj_seq_len

    @torch.no_grad()
    def inference(self, batch, sample_num=1):
        assert sample_num == 1
        data = dict(batch)
        data.update(self.mfiller.inference(batch))
        body = data['infer_out_body_pose'][:, 0]                                          # [B,T,69]
        B, T = body.shape[:2]
        flat = body.reshape(-1, 69)
        z3 = torch.zeros_like(flat[:, :3])
        joints = self.smpl.get_joints(z3, flat, root_trans=z3)[:, 1:].reshape(B, T, 69).transpose(0, 1).contiguous()
        eps = batch['in_traj_window_latent'].to(self.dtype) if 'in_traj_window_latent' in batch else None
        local, trans, orient = inference_multi_step(self.traj_predictor, joints, self.traj_seq_len, eps)
        data['infer_out_local_traj_tp'] = local.view(T, B, 1, 11)
        data['infer_out_trans'] = trans.transpose(0, 1).unsqueeze(1).contiguous()
        data['infer_out_orient'] = orient.transpose(0, 1).unsqueeze(1).contiguous()
        data['infer_out_pose'] = torch.cat([data['infer_out_orient'], data['infer_out_body_pose']], dim=-1)
        return data
