"""ORACLE for the motion infiller's reconstruction mode (test infrastructure): the posterior encoder q(z | X, C) (DataEncoder,
motion_infiller/models/motion_infiller_vae.py:126-249, pooling 'attn') and the recon sweep of inference_multi_step(..., recon=True)
(:551-557, :589-632) restated in plain torch on top of oracle.nets.MotionInfiller, in the module's dtype (float32 or float64).

The sweep is the clean one: it starts from the masked input body pose and writes no input tensor.  The reference at B = 1 with a
caller-supplied `in_body_pose` starts its recon sweep from the infilled pose instead (transpose(0, 1).contiguous() of a [1,T,69]
tensor is a view, so its infer sweep overwrites the caller's tensor); the golden generator runs those cases on a fresh copy.
"""
import numpy as np
import torch
from torch import nn

from oracle import nets as on
from oracle.nets import CUR, D, FUT, NZ, PAST


class InfillerPosterior(nn.Module):
    def __init__(self):
        super().__init__()
        self.in_fc = nn.Linear(69, D)
        self.pos_enc = on._PosEnc(D, D)
        self.temporal_net = nn.TransformerDecoder(nn.TransformerDecoderLayer(D, 8, 512, 0.1), 2)
        self.mu_token = nn.Parameter(torch.zeros(D))
        self.logvar_token = nn.Parameter(torch.zeros(D))
        self.q_z_mu_net = nn.Linear(D, NZ)
        self.q_z_logvar_net = nn.Linear(D, NZ)

    def mean(self, gt_cur, ctx, key_pad):
        """gt_cur [30,B,69]: the ground-truth body pose of a window's current frames -> the posterior mean [B,128] (:204-233, :375-376)"""
        B = gt_cur.shape[1]
        x = torch.cat([self.mu_token.repeat(1, B, 1), self.logvar_token.repeat(1, B, 1), self.in_fc(gt_cur)], dim=0)
        x = self.temporal_net(self.pos_enc(x), ctx, memory_key_padding_mask=key_pad)
        return self.q_z_mu_net(x[0])


class MotionInfillerRecon(on.MotionInfiller):
    """MotionInfiller with the posterior encoder: state dicts need the data_encoder.* names too"""

    def __init__(self):
        super().__init__()
        self.data_encoder = InfillerPosterior()
        self.eval()

    def recon_window(self, in_pose, gt_cur, key_pad):
        """one 50-frame window in mode 'recon': in_pose [50,B,69] (running input), gt_cur [30,B,69], key_pad [B,50] -> [40,B,69]"""
        ce, dd = self.context_encoder, self.data_decoder
        ctx = ce.temporal_net(ce.pos_enc(ce.in_fc(in_pose)), src_key_padding_mask=key_pad)
        z = self.data_encoder.mean(gt_cur, ctx, key_pad)
        x = dd.temporal_net(dd.pos_enc(z.repeat(CUR, 1, 1), pos_offset=PAST), ctx, memory_key_padding_mask=key_pad)
        x = dd.out_fc(dd.out_mlp(x))
        return torch.cat([in_pose[:PAST], x], dim=0)

    @torch.no_grad()
    def recon(self, batch):
        """pose [B,T,72] (ground truth), pose_mask [B,T,72], frame_mask [B,T] (1 = visible), optional in_body_pose [B,T,69]
        (default (pose * pose_mask)[..., 3:]) -> recon_out_pose [B,T,72] (root from pose), recon_out_body_pose [B,T,69]"""
        dt = self.data_decoder.out_fc.weight.dtype
        gt = batch['pose']
        body_in = batch['in_body_pose'] if batch.get('in_body_pose') is not None else (gt * batch['pose_mask'])[..., 3:]
        pose = body_in.transpose(0, 1).contiguous().to(dt).clone()                        # [T,B,69], the running input
        gt_body = gt[..., 3:].transpose(0, 1).to(dt)
        key_pad_all = ~(batch['frame_mask'] == 1)
        T, B = pose.shape[:2]
        dev = pose.device
        outs = []
        for i in range(int(np.ceil((T - PAST) / CUR))):
            s, e = i * CUR, i * CUR + PAST + CUR + FUT
            eb = min(e, T)
            win, kp = pose[s:eb], key_pad_all[:, s:eb]
            if e > eb:
                win = torch.cat([win, torch.zeros(e - eb, B, 69, dtype=dt, device=dev)], dim=0)
                kp = torch.cat([kp, torch.ones(B, e - eb, dtype=torch.bool, device=dev)], dim=1)
            gwin = gt_body[s + PAST:min(s + PAST + CUR, T)]
            if gwin.shape[0] < CUR:
                gwin = torch.cat([gwin, torch.zeros(CUR - gwin.shape[0], B, 69, dtype=dt, device=dev)], dim=0)
            kp = kp.clone()
            kp[:, :PAST] = False
            out = self.recon_window(win, gwin, kp)
            nfr = min(e - FUT, T) - s
            pose[s:s + nfr] = out[:nfr]
            outs.append(out[:nfr] if i == 0 else out[PAST:nfr])
        body = torch.cat(outs, dim=0).transpose(0, 1).contiguous()                         # [B,T,69]
        return {'recon_out_body_pose': body, 'recon_out_pose': torch.cat([gt[..., :3].to(dt), body], dim=-1)}


def recon_model(state, dtype=torch.float32):
    """MotionInfillerRecon with `state` (infiller and posterior weights) in `dtype`"""
    m = MotionInfillerRecon()
    on.load_state(m, state, dtype)
    return m
