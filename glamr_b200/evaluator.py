"""``Evaluator`` -- drop-in for the reference class of the same name (global_recon/utils/evaluator.py:172-397), the step
that follows the optimiser in ``run_dataset -> eval_dataset`` (SURVEY.md §8(f)-2), with the heavy parts on the CUDA
library:

* the four SMPL evaluations per person (ground truth and estimate, world and heading-aligned trajectories;
  evaluator.py:254-262,275-283,296-304,313-321) run through ``glamr_smpl_forward`` WITH vertices,
* ``J_regressor_h36m @ vertices`` (:263,:284,:306,:322) is a CSR regression kernel (``glamr_sparse_regress``),
* the per-frame similarity Procrustes of PA-MPJPE (:311, lib/utils/torch_transform.py:282-345) is
  ``glamr_procrustes_align`` (3x3 Jacobi SVD per frame in fp64),
* the trajectory alignment (:202-216, traj_pred/utils/traj_utils.py:97-107) uses the library's row-wise rotation algebra.

The metric reductions themselves (means of joint distances) are a handful of elementwise device ops.  Same metric names,
same accumulation / multi-seed logic, same log line format.  No CPU fallback.
"""
import ctypes
import logging
from collections import defaultdict

import numpy as np
import torch

from . import geometry as G
from . import lib as L
from .recon import tensor_to
from .smpl import SMPL, SMPL_MODEL_DIR

# lib/models/smpl.py:23-25
H36M_TO_J17 = [6, 5, 4, 1, 2, 3, 16, 15, 14, 11, 12, 13, 8, 10, 0, 7, 9]
H36M_TO_J15 = [H36M_TO_J17[14]] + H36M_TO_J17[:14]
JOINT_REGRESSOR_H36M = 'data/J_regressor_h36m.npy'
BASE_ORIENT = [0.5, 0.5, 0.5, 0.5]


class AverageMeter:
    """lib/utils/tools.py:9-35"""

    def __init__(self, avg=None, count=1):
        self.reset()
        if avg is not None:
            self.val, self.avg, self.count, self.sum = avg, avg, count, avg * count

    def __repr__(self):
        return f'{self.avg: .4f}'

    def reset(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        if n > 0:
            self.val = val
            self.sum += val * n
            self.count += n
            self.avg = self.sum / self.count


def quat_apply(q, v):
    """lib/utils/torch_transform.py:39-45"""
    xyz = q[..., 1:]
    t = torch.cross(xyz, v, dim=-1) * 2
    return v + q[..., :1] * t + torch.cross(xyz, t, dim=-1)


def convert_traj_world2heading(orient_q, trans, apply_base_orient_after=False):
    """traj_pred/utils/traj_utils.py:97-107: remove the first frame's heading and xy position"""
    base = torch.tensor(BASE_ORIENT, device=orient_q.device)
    nobase = G.quat_mul(orient_q, G.quat_conjugate(base).expand_as(orient_q))
    heading_q = G.get_heading_q(nobase[:1])
    inv_h = G.quat_conjugate(heading_q).expand_as(nobase)
    orient_h = G.quat_mul(inv_h, nobase)
    local = trans.clone()
    local[..., :2] -= trans[0, ..., :2]
    trans_h = quat_apply(inv_h, local)
    if apply_base_orient_after:
        orient_h = G.quat_mul(orient_h, base.expand_as(orient_h))
    return orient_h, trans_h


def _select(x, pose_dict, mode):
    if mode == 'vis':
        return x[pose_dict['vis_frames']]
    if mode == 'invis':
        return x[pose_dict['invis_frames']]
    return x


def _mean_dist_metric(data, est_key, gt_key, mode='all', per_frame=False):
    """shared body of compute_MPJPE / compute_PAMPJPE / compute_MPVE (evaluator.py:15-122): mm, mean over joints, summed over frames"""
    num, total, rows = 0, 0.0, []
    for idx, pd in data['person_data'].items():
        est = _select(pd[est_key], pd, mode)
        gt = _select(data['gt'][idx][gt_key], pd, mode)
        if gt.shape[0] == 0:
            if per_frame:
                rows.append(torch.zeros((0,), device=gt.device))
            continue
        dist = torch.norm(est - gt, dim=2).mean(dim=1) * 1000
        if per_frame:
            rows.append(dist)
        else:
            total = total + dist.sum()
        num += gt.shape[0]
    if per_frame:
        return torch.cat(rows).cpu().numpy(), {'num_data': num}
    val = (total / num).item() if num > 0 else 0
    return val, {'num_data': num}


def compute_PAMPJPE(data, mode='all'):
    return _mean_dist_metric(data, 'eval_joints_world_PA', 'eval_joints_world', mode)


def compute_PAMPJPE_seq(data, mode='all'):
    return _mean_dist_metric(data, 'eval_joints_world_PA', 'eval_joints_world', mode, per_frame=True)


def compute_Global_MPJPE(data):
    return _mean_dist_metric(data, 'aligned_eval_joints_world', 'aligned_eval_joints_world')


def compute_Global_MPVE(data):
    return _mean_dist_metric(data, 'aligned_eval_verts_world', 'aligned_eval_verts_world')


def compute_accel_error(data):
    """evaluator.py:153-167"""
    num, total = 0, 0.0
    for idx, pd in data['person_data'].items():
        j, g = pd['eval_joints_world'], data['gt'][idx]['eval_joints_world']
        acc = j[:-2] - 2 * j[1:-1] + j[2:]
        gacc = g[:-2] - 2 * g[1:-1] + g[2:]
        total = total + (torch.norm(acc - gacc, dim=2).mean(dim=1) * 1000).sum()
        num += acc.shape[0]
    return (total / num).item(), {'num_data': num}


class Evaluator:

    def __init__(self, algo='', dataset='', device=torch.device('cuda'), log_file='nofile', align_freq=250, compute_sample=True,
                 smpl=None, h36m_regressor=None, log=None):
        """Reference signature (evaluator.py:172) plus optional injection of the body model (a glamr_b200.smpl.SMPL or an assets
        dict; default: SMPL_MODEL_DIR) and of the [17, 6890] H36M joint regressor (default: data/J_regressor_h36m.npy)."""
        self.algo, self.dataset = algo, dataset
        self.device = L.require_cuda(device)
        self.align_freq, self.compute_sample = align_freq, compute_sample
        self.log = log if log is not None else _create_logger(log_file)
        self.smpl = smpl if isinstance(smpl, SMPL) else SMPL(smpl if smpl is not None else SMPL_MODEL_DIR, pose_type='body26fk', device=self.device)
        reg = np.load(JOINT_REGRESSOR_H36M) if h36m_regressor is None else np.asarray(h36m_regressor)
        self._set_regressor(reg.astype(np.float32))
        self._lib = L.load()
        self.metrics_func = {
            'PA-MPJPE': lambda d: compute_PAMPJPE(d, 'all'), 'PA-MPJPE-vis': lambda d: compute_PAMPJPE(d, 'vis'),
            'PA-MPJPE-invis': lambda d: compute_PAMPJPE(d, 'invis'), 'G-MPJPE': compute_Global_MPJPE, 'G-MPVE': compute_Global_MPVE,
            'ACCEL': compute_accel_error,
        }
        if self.compute_sample:
            self.metrics_func['sample_PA-MPJPE-invis'] = lambda d: compute_PAMPJPE_seq(d, 'invis')
        self.metrics_name = list(self.metrics_func.keys())
        self.seed_min_metrics = ['PA-MPJPE-invis']
        self.reset()

    def _set_regressor(self, reg):
        """dense [rows, V] -> CSR on the device (the H36M regressor is ~99.9 % zeros).  V must be the body model's vertex count: the
        kernel takes it as the per-frame vertex stride, so any other width would read other frames' vertices or past the end."""
        nv = self.smpl.num_verts
        if reg.ndim != 2 or reg.shape[0] <= 0 or reg.shape[1] != nv:
            raise L.GlamrError(f'h36m_regressor must be [rows, {nv}] (one column per vertex of the body model); got {list(reg.shape)}')
        rows, V = reg.shape
        ptr, ci, w = [0], [], []
        for r in range(rows):
            nz = np.nonzero(reg[r])[0]
            ci += nz.tolist()
            w += reg[r, nz].tolist()
            ptr.append(len(ci))
        dev = self.device
        self._reg = (rows, V, torch.tensor(ptr, dtype=torch.int32, device=dev), torch.tensor(ci or [0], dtype=torch.int32, device=dev),
                     torch.tensor(w or [0.0], dtype=torch.float32, device=dev))

    def reset(self):
        self.metrics_dict_collection = dict()
        self.acc_metrics_dict = {'metrics': defaultdict(AverageMeter)}

    # ------------------------------------------------------------------------------------------------ device helpers
    def regress_h36m(self, vertices):
        """torch.matmul(self.J_regressor, vertices) (:263) -> [n, 17, 3]"""
        rows, V, ptr, ci, w = self._reg
        if vertices.dim() != 3 or vertices.shape[1:] != (V, 3):
            raise L.GlamrError(f'regress_h36m: vertices must be [n, {V}, 3] to match the regressor; got {list(vertices.shape)}')
        v = vertices.contiguous().float()
        out = torch.empty((v.shape[0], rows, 3), device=self.device)
        with torch.cuda.device(self.device):
            L.check(self._lib.glamr_sparse_regress(v.shape[0], V, rows, L.ptr(ptr), L.ptr(ci), L.ptr(w), L.ptr(v), L.ptr(out), L.stream_ptr()),
                    'glamr_sparse_regress')
        return out

    def procrustes(self, S1, S2):
        """batch_compute_similarity_transform_torch (lib/utils/torch_transform.py:282-345) for [n, J, 3] point sets"""
        a, b = S1.contiguous().float(), S2.contiguous().float()
        out = torch.empty_like(a)
        with torch.cuda.device(self.device):
            L.check(self._lib.glamr_procrustes_align(a.shape[0], a.shape[1], L.ptr(a), L.ptr(b), L.ptr(out), L.stream_ptr()), 'glamr_procrustes_align')
        return out

    def get_aligned_orient_trans(self, pose_dict):
        """:202-216: heading / origin re-alignment every `align_freq` frames"""
        orient_q = G.angle_axis_to_quaternion(pose_dict['smpl_orient_world'].float())
        trans = pose_dict['root_trans_world'].float()
        qs, ts = [], []
        for i in range(int(np.ceil(orient_q.shape[0] / self.align_freq))):
            sind = i * self.align_freq - int(i > 0)
            eind = min((i + 1) * self.align_freq, orient_q.shape[0])
            q, t = convert_traj_world2heading(orient_q[sind:eind].contiguous(), trans[sind:eind].contiguous(), apply_base_orient_after=True)
            qs.append(q[int(i > 0):])
            ts.append(t[int(i > 0):])
        pose_dict['aligned_orient_q'] = torch.cat(qs)
        pose_dict['aligned_orient'] = G.quaternion_to_angle_axis(pose_dict['aligned_orient_q'])
        pose_dict['aligned_trans'] = torch.cat(ts)

    def _smpl_eval(self, orient, body_pose, betas, trans, scale=None):
        out = self.smpl(global_orient=orient.float().contiguous(), body_pose=body_pose.float().contiguous(), betas=betas.float().contiguous(),
                        root_trans=trans.float().contiguous(), root_scale=scale, return_full_pose=True)
        j15 = self.regress_h36m(out.vertices)[:, H36M_TO_J15]
        return out, j15

    # ------------------------------------------------------------------------------------------------ reference API
    def prepare_seq(self, data):
        """:218-327"""
        use_keys = ['pose', 'pose_cam', 'root_trans', 'root_trans_cam', 'smpl_orient_cam', 'smpl_orient_world', 'smpl_pose', 'smpl_beta',
                    'root_trans_cam', 'root_trans_world', 'scale', 'vis_frames', 'invis_frames', 'visible', 'j3d_h36m', 'kp']
        exclude_keys = ['smpl_pose_rotmat']
        for idx, pd in data['person_data'].items():
            if 'exist_frames' in pd:
                ex = pd['exist_frames']
                gd = data['gt'][idx]
                for d in (pd, gd):
                    for key in list(d.keys()):
                        if not any(x in key for x in use_keys) or key in exclude_keys or d[key] is None:
                            continue
                        d[key] = d[key][ex]
        # ---- ground truth
        for idx, gd in data['gt'].items():
            if 'pose' not in gd:
                continue
            visible = data['person_data'][idx]['visible_orig']
            gd['vis_frames'], gd['invis_frames'] = visible == 1, visible == 0
            gd['smpl_orient_world'] = gd['pose'][:, :3].float()
            gd['root_trans_world'] = gd['root_trans'].float()
            if self.dataset == '3DPW':
                oq = G.angle_axis_to_quaternion(gd['smpl_orient_world'].contiguous())
                quat = G.angle_axis_to_quaternion(torch.tensor([[np.pi * 0.5, 0, 0]], device=self.device)).expand_as(oq)
                gd['smpl_orient_world'] = G.quaternion_to_angle_axis(G.quat_mul(quat, oq))
                gd['root_trans_world'] = quat_apply(quat, gd['root_trans_world'])
            n = gd['pose'].shape[0]
            body, betas = gd['pose'][:, 3:].float(), gd['shape'].float().reshape(1, -1).repeat(n, 1)
            out, j15 = self._smpl_eval(gd['smpl_orient_world'], body, betas, gd['root_trans_world'])
            gd['smpl_verts_world'], gd['smpl_joints_world'] = out.vertices, out.joints
            pelvis = (j15[:, [3]] + j15[:, [4]]) * 0.5
            gd['eval_joints_world'] = j15[:, 1:] - pelvis
            gd['eval_verts_world'] = out.vertices - pelvis
            gd['smpl_pose'] = body
            self.get_aligned_orient_trans(gd)
            out, j15 = self._smpl_eval(gd['aligned_orient'], body, betas, gd['aligned_trans'])
            gd['aligned_eval_joints_world'] = j15[:, 1:]
            gd['aligned_eval_verts_world'] = out.vertices
        # ---- estimate
        for idx, pd in data['person_data'].items():
            visible = pd['visible_orig']
            pd['vis_frames'], pd['invis_frames'] = visible == 1, visible == 0
            scale = pd['scale'] if pd.get('scale') is not None else None
            out, j15 = self._smpl_eval(pd['smpl_orient_world'], pd['smpl_pose'], pd['smpl_beta'], pd['root_trans_world'], scale)
            pd['smpl_verts_world'], pd['smpl_joints_world'] = out.vertices, out.joints
            pelvis = (j15[:, [3]] + j15[:, [4]]) * 0.5
            pd['eval_joints_world'] = j15[:, 1:] - pelvis
            pd['eval_verts_world'] = out.vertices - pelvis
            self.get_aligned_orient_trans(pd)
            pd['eval_joints_world_PA'] = self.procrustes(pd['eval_joints_world'], data['gt'][idx]['eval_joints_world'])
            out, j15 = self._smpl_eval(pd['aligned_orient'], pd['smpl_pose'], pd['smpl_beta'], pd['aligned_trans'], scale)
            pd['aligned_eval_joints_world'] = j15[:, 1:]
            pd['aligned_eval_verts_world'] = out.vertices

    def compute_sequence_metrics(self, data, name=None, accumulate=True):
        """:329-343"""
        data = tensor_to(data, self.device)
        self.prepare_seq(data)
        data['log'], data['name'] = self.log, name
        metrics_dict = defaultdict(dict)
        metrics_dict['seq_len'] = data['seq_len']
        for metric, func in self.metrics_func.items():
            val, info = func(data)
            metrics_dict['metrics'][metric] = AverageMeter(val, info['num_data'])
        if accumulate:
            self.update_accumulated_metrics(metrics_dict, name)
        self.last_data = data
        return metrics_dict

    def update_accumulated_metrics(self, metrics_dict, name=None):
        """:345-350"""
        if name is not None:
            self.metrics_dict_collection[name] = metrics_dict
        for metric in self.metrics_name:
            self.acc_metrics_dict['metrics'][metric].update(metrics_dict['metrics'][metric].avg, metrics_dict['metrics'][metric].count)
        return self.acc_metrics_dict

    def metrics_from_multiple_seeds(self, metrics_dict_arr):
        """:352-378"""
        metrics_dict = defaultdict(dict)
        metrics_dict['seq_len'] = metrics_dict_arr[0]['seq_len']
        for metric in self.metrics_name:
            num = metrics_dict_arr[0]['metrics'][metric].count
            if 'sample' in metric or 'mean' in metric:
                arr = np.stack([x['metrics'][metric].avg for x in metrics_dict_arr])
                if num == 0:
                    val = 0
                else:
                    val = (arr.min(axis=0) if 'sample' in metric else arr.mean(axis=0)).mean()
            else:
                arr = np.array([x['metrics'][metric].avg for x in metrics_dict_arr])
                val = arr.min() if metric in self.seed_min_metrics else arr.mean()
            metrics_dict['metrics'][metric] = AverageMeter(val, num)
        return metrics_dict

    def print_metrics(self, metrics_dict=None, fmt='.3f', prefix='', print_accum=True):
        """:380-388 same line format"""
        if metrics_dict is None:
            metrics_dict = self.acc_metrics_dict
        fmt_str = f"%s: %{fmt} (%{fmt})" if print_accum else f"%s: %{fmt}"
        stats = f'{prefix}{self.algo} --- ' + ' '.join(fmt_str % ((x, y.avg, y.val) if print_accum else (x, y.avg))
                                                      for x, y in metrics_dict['metrics'].items() if not isinstance(y.avg, np.ndarray))
        if 'sample_PA-MPJPE-invis' not in metrics_dict['metrics']:
            stats += ' sample_PA-MPJPE-invis: None (need multiple seeds)'
        self.log.info(stats)
        return stats


def _create_logger(file_path):
    """lib/utils/log_utils.py:8-29 (console handler; file handler unless 'nofile')"""
    import os
    logger = logging.getLogger(file_path)
    logger.propagate = False
    logger.setLevel(logging.DEBUG)
    if not logger.handlers:
        ch = logging.StreamHandler()
        ch.setLevel(logging.INFO)
        ch.setFormatter(logging.Formatter('%(message)s'))
        logger.addHandler(ch)
        if file_path != 'nofile':
            os.makedirs(os.path.dirname(file_path) or '.', exist_ok=True)
            fh = logging.FileHandler(file_path, mode='a')
            fh.setLevel(logging.DEBUG)
            fh.setFormatter(logging.Formatter('[%(asctime)s] %(message)s'))
            logger.addHandler(fh)
    return logger
