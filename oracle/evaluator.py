"""ORACLE (test infrastructure): torch-CPU restatement of the reference's Evaluator.prepare_seq + metric functions
(global_recon/utils/evaluator.py:15-167,202-343), pinned against the executed reference by tests/golden/evaluator.npz
(generator: tests/golden/make_golden.py evaluator).  The product (glamr_b200/evaluator.py) never imports it."""
import numpy as np
import torch

from . import rotations as rt
from .smpl import OracleSMPL

H36M_TO_J17 = [6, 5, 4, 1, 2, 3, 16, 15, 14, 11, 12, 13, 8, 10, 0, 7, 9]          # lib/models/smpl.py:23
H36M_TO_J15 = [H36M_TO_J17[14]] + H36M_TO_J17[:14]                                 # lib/models/smpl.py:25
BASE = [0.5, 0.5, 0.5, 0.5]


def quat_apply(q, v):
    """lib/utils/torch_transform.py:39-45"""
    xyz = q[..., 1:]
    t = torch.cross(xyz, v, dim=-1) * 2
    return v + q[..., :1] * t + torch.cross(xyz, t, dim=-1)


def world2heading(orient_q, trans):
    """traj_pred/utils/traj_utils.py:97-107 with apply_base_orient_after=True"""
    base = torch.tensor(BASE, dtype=orient_q.dtype, device=orient_q.device)
    nobase = rt.quat_mul(orient_q, rt.quat_conj(base).expand_as(orient_q))
    inv_h = rt.quat_conj(rt.get_heading_q(nobase[0])).expand_as(nobase)
    oh = rt.quat_mul(inv_h, nobase)
    local = trans.clone()
    local[..., :2] -= trans[0, ..., :2]
    return rt.quat_mul(oh, base.expand_as(oh)), quat_apply(inv_h, local)


def similarity_align(S1, S2):
    """lib/utils/torch_transform.py:282-345 for [n, J, 3] inputs, aligned frame by frame.  The reference transposes its inputs
    only when the batch size is neither 2 nor 3 (torch_transform.py:298-302, a test of S1.shape[0]), so for n in {2, 3} it aligns
    across frames; this restatement, like the product, keeps the per-frame alignment at every n."""
    S1, S2 = S1.permute(0, 2, 1), S2.permute(0, 2, 1)
    mu1, mu2 = S1.mean(dim=-1, keepdim=True), S2.mean(dim=-1, keepdim=True)
    X1, X2 = S1 - mu1, S2 - mu2
    var1 = (X1 ** 2).sum(dim=1).sum(dim=1)
    K = X1.bmm(X2.permute(0, 2, 1))
    U, s, V = torch.svd(K)
    Z = torch.eye(3, dtype=S1.dtype, device=S1.device).unsqueeze(0).repeat(U.shape[0], 1, 1)
    Z[:, -1, -1] *= torch.sign(torch.det(U.bmm(V.permute(0, 2, 1))))
    R = V.bmm(Z.bmm(U.permute(0, 2, 1)))
    scale = torch.stack([torch.trace(x) for x in R.bmm(K)]) / var1
    t = mu2 - scale[:, None, None] * R.bmm(mu1)
    return (scale[:, None, None] * R.bmm(S1) + t).permute(0, 2, 1)


class OracleEvaluator:
    def __init__(self, smpl_assets, h36m_regressor, dataset='', align_freq=250, dtype=torch.float32, device='cpu'):
        """dtype, device: where and in what precision everything is computed; the inputs are converted to them (the float32
        constants and inputs are read as float32 first, so a float64 oracle sees the same values as the float32 one)"""
        self.dtype, self.device = dtype, torch.device(device)
        self.smpl = OracleSMPL(smpl_assets, device=self.device, dtype=dtype)
        self.J = torch.tensor(np.asarray(h36m_regressor, np.float32), device=self.device).to(dtype)
        self.dataset, self.align_freq = dataset, align_freq

    def _w(self, x):
        """an input in the working dtype on the working device"""
        return torch.as_tensor(x).to(self.device, self.dtype)

    def aligned(self, d):
        """:202-216"""
        oq, tr = rt.aa_to_quat(d['smpl_orient_world']), d['root_trans_world']
        qs, ts = [], []
        for i in range(int(np.ceil(oq.shape[0] / self.align_freq))):
            s, e = i * self.align_freq - int(i > 0), min((i + 1) * self.align_freq, oq.shape[0])
            q, t = world2heading(oq[s:e], tr[s:e])
            qs.append(q[int(i > 0):])
            ts.append(t[int(i > 0):])
        d['aligned_orient'] = rt.quat_to_aa(torch.cat(qs))
        d['aligned_trans'] = torch.cat(ts)

    def _eval(self, orient, pose, betas, trans, scale=None):
        joints, verts = self.smpl(orient, pose, betas, root_trans=trans, root_scale=scale)
        return verts, torch.matmul(self.J, verts)[:, H36M_TO_J15]

    def prepare_seq(self, data):
        """:218-327 (world coordinates only, as the reference's `for coord in ['world']`)"""
        for idx, pd in data['person_data'].items():
            if 'exist_frames' in pd:
                ex = pd['exist_frames']
                for d in (pd, data['gt'][idx]):
                    for k in ['smpl_orient_world', 'root_trans_world', 'smpl_pose', 'smpl_beta', 'pose', 'root_trans', 'scale', 'visible_orig']:
                        if k in d and d[k] is not None:        # every key containing a use_keys substring (:221-236), 'visible_orig' included
                            d[k] = d[k][ex]
        for idx, gd in data['gt'].items():
            vis = data['person_data'][idx]['visible_orig']
            gd['vis_frames'], gd['invis_frames'] = vis == 1, vis == 0
            gd['smpl_orient_world'], gd['root_trans_world'] = self._w(gd['pose'][:, :3]), self._w(gd['root_trans'])
            if self.dataset == '3DPW':
                oq = rt.aa_to_quat(gd['smpl_orient_world'])
                quat = rt.aa_to_quat(torch.tensor([[np.pi * 0.5, 0, 0]], dtype=self.dtype, device=self.device)).expand_as(oq)
                gd['smpl_orient_world'] = rt.quat_to_aa(rt.quat_mul(quat, oq))
                gd['root_trans_world'] = quat_apply(quat, gd['root_trans_world'])
            n = gd['pose'].shape[0]
            body, betas = self._w(gd['pose'][:, 3:]), self._w(gd['shape']).reshape(1, -1).repeat(n, 1)
            verts, j15 = self._eval(gd['smpl_orient_world'], body, betas, gd['root_trans_world'])
            pelvis = (j15[:, [3]] + j15[:, [4]]) * 0.5
            gd['eval_joints_world'], gd['eval_verts_world'] = j15[:, 1:] - pelvis, verts - pelvis
            self.aligned(gd)
            verts, j15 = self._eval(gd['aligned_orient'], body, betas, gd['aligned_trans'])
            gd['aligned_eval_joints_world'], gd['aligned_eval_verts_world'] = j15[:, 1:], verts
        for idx, pd in data['person_data'].items():
            vis = pd['visible_orig']
            pd['vis_frames'], pd['invis_frames'] = vis == 1, vis == 0
            for k in ('smpl_orient_world', 'smpl_pose', 'smpl_beta', 'root_trans_world', 'scale'):
                if pd.get(k) is not None:
                    pd[k] = self._w(pd[k])
            verts, j15 = self._eval(pd['smpl_orient_world'], pd['smpl_pose'], pd['smpl_beta'], pd['root_trans_world'], pd.get('scale'))
            pelvis = (j15[:, [3]] + j15[:, [4]]) * 0.5
            pd['eval_joints_world'], pd['eval_verts_world'] = j15[:, 1:] - pelvis, verts - pelvis
            self.aligned(pd)
            pd['eval_joints_world_PA'] = similarity_align(pd['eval_joints_world'], data['gt'][idx]['eval_joints_world'])
            verts, j15 = self._eval(pd['aligned_orient'], pd['smpl_pose'], pd['smpl_beta'], pd['aligned_trans'], pd.get('scale'))
            pd['aligned_eval_joints_world'], pd['aligned_eval_verts_world'] = j15[:, 1:], verts

    @staticmethod
    def _metric(data, ek, gk, mode='all'):
        num, tot = 0, 0.0
        for idx, pd in data['person_data'].items():
            e, g = pd[ek], data['gt'][idx][gk]
            if mode != 'all':
                m = pd['vis_frames'] if mode == 'vis' else pd['invis_frames']
                e, g = e[m], g[m]
            if g.shape[0] == 0:
                continue
            tot = tot + (torch.norm(e - g, dim=2).mean(dim=1) * 1000).sum()
            num += g.shape[0]
        return (float(tot / num) if num else 0.0), num

    def metrics(self, data):
        """values of evaluator.py:172-186 metrics_func (sample metric excluded)"""
        self.prepare_seq(data)
        out = {'PA-MPJPE': self._metric(data, 'eval_joints_world_PA', 'eval_joints_world'),
               'PA-MPJPE-vis': self._metric(data, 'eval_joints_world_PA', 'eval_joints_world', 'vis'),
               'PA-MPJPE-invis': self._metric(data, 'eval_joints_world_PA', 'eval_joints_world', 'invis'),
               'G-MPJPE': self._metric(data, 'aligned_eval_joints_world', 'aligned_eval_joints_world'),
               'G-MPVE': self._metric(data, 'aligned_eval_verts_world', 'aligned_eval_verts_world')}
        num, tot = 0, 0.0
        for idx, pd in data['person_data'].items():
            j, g = pd['eval_joints_world'], data['gt'][idx]['eval_joints_world']
            a, ga = j[:-2] - 2 * j[1:-1] + j[2:], g[:-2] - 2 * g[1:-1] + g[2:]
            tot = tot + (torch.norm(a - ga, dim=2).mean(dim=1) * 1000).sum()
            num += a.shape[0]
        out['ACCEL'] = (float(tot / num), num)
        return out
