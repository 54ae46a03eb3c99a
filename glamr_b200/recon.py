"""``GlobalReconOptimizer`` -- drop-in for the reference class of the same name
(global_recon/models/global_recon_model.py:23-659) with the optimisation loop running in the CUDA library.

Same constructor, ``optimize(in_dict, continue_opt=False) -> dict`` (numpy), ``init_data``, ``forward``,
``compute_loss``, ``optimize_main``; same YAML stage specs; same output keys / shapes / dtypes (SURVEY.md Appendix B).
``optimize_seeds(in_dict, seeds) -> [dict]`` runs several seeds of one sequence as one problem, and
``optimize_batch(in_dicts, seeds) -> [[dict]]`` every (sequence, seed) pair of several sequences (groups, see glamr_b200/problem.py):
every pair's result is the one ``optimize`` gives for that sequence and seed.
Every array of an ``in_dict['est']`` pose_dict (bboxes_dict.exist, smpl_pose_quat_wroot, smpl_beta, root_trans, kp_2d, cam_K) may be
a numpy array or a torch tensor on the CPU or a GPU; the data dict and the output are the same for either.  ``init_data``'s per-frame
work (rotation vectors, gap interpolation, filter_pose) runs in kernels for all persons at once, after one upload and with one
read-back; host Python keeps the dict bookkeeping and the log lines.  Every formula of the per-iteration path -- trajectory codec,
camera, SMPL, projection, residuals, analytic backward, Adam -- is a kernel of glamr_b200/csrc.  No autograd, no CPU fallback.
"""
import copy
import ctypes
import time

import numpy as np
import torch

from . import geometry as G
from . import lib as L
from . import problem as PB
from .smpl import SMPL, SMPL_MODEL_DIR
from .synthetic import SMPL_TO_BODY26FK

NUM_TERMS = L.NUM_TERMS
_TERM_NAMES = {v: k for k, v in L.TERM_INDEX.items()}


def tensor_to(x, device):
    """lib/utils/torch_utils.py:101 -- numpy / nested containers -> tensors on `device` (dtype preserved)"""
    if isinstance(x, np.ndarray):
        return torch.tensor(x, device=device)
    if isinstance(x, torch.Tensor):
        return x.to(device)
    if isinstance(x, dict):
        return {k: tensor_to(v, device) for k, v in x.items()}
    return x


_GROUP_CPU_TENSORS = False      # tests flip this to run the grouped-copy path on CPU tensors


def tensor_to_numpy(x):
    """lib/utils/torch_utils.py:118 -- nested containers of tensors -> numpy.  The output dict of `optimize` holds several
    hundred small tensors per person; instead of one synchronous device->host copy each, the tensors of one dtype are
    concatenated on the device, copied once and split into views on the host (same values, shapes and dtypes)."""
    leaves = []

    def walk(v):
        if isinstance(v, torch.Tensor):
            leaves.append(v.detach())
            return ('leaf', len(leaves) - 1)
        if isinstance(v, dict):
            return ('dict', {k: walk(u) for k, u in v.items()})
        if isinstance(v, (list, tuple)):
            return (type(v), [walk(u) for u in v])
        return ('raw', v)
    tree = walk(x)
    arrays = [None] * len(leaves)
    groups = {}
    for i, t in enumerate(leaves):
        groups.setdefault((t.dtype, t.device), []).append(i)
    for (dtype, device), idx in groups.items():
        if len(idx) == 1 or (device.type == 'cpu' and not _GROUP_CPU_TENSORS):
            for i in idx:
                arrays[i] = leaves[i].cpu().numpy()
            continue
        flat = torch.cat([leaves[i].reshape(-1) for i in idx]).cpu().numpy()
        off = 0
        for i in idx:
            n = leaves[i].numel()
            arrays[i] = flat[off:off + n].reshape(tuple(leaves[i].shape))
            off += n

    def build(node):
        kind, v = node
        if kind == 'leaf':
            return arrays[v]
        if kind == 'dict':
            return {k: build(u) for k, u in v.items()}
        if kind == 'raw':
            return v
        return kind(build(u) for u in v)
    return build(tree)


def rotmats_to_rotvec(mats):
    """``Rotation.from_matrix(mats).as_rotvec()`` (global_recon_model.py:106-107) as vectorised numpy, float64.

    SciPy projects every float32-accurate input onto SO(3) with one SVD per matrix (12 ms for a 300-frame track); the
    same polar factor U V^T is reached here by two Newton steps R <- (R + R^-T) / 2 written with cross products, then
    the usual largest-diagonal quaternion branch and the rotation-vector scaling (series below 1e-3 rad).  The nine
    entries are kept as nine contiguous arrays (structure of arrays): every step is a handful of long vector operations."""
    R0 = np.asarray(mats, dtype=np.float64).reshape(-1, 3, 3)
    n = R0.shape[0]
    r = np.ascontiguousarray(R0.reshape(n, 9).T)                      # r[3 i + j] = R[:, i, j], contiguous
    det = None
    for _ in range(2):
        a0, a1, a2, b0, b1, b2, c0, c1, c2 = r
        cof = np.empty_like(r)                                       # cofactor rows = cross products of the other two rows
        cof[0] = b1 * c2 - b2 * c1
        cof[1] = b2 * c0 - b0 * c2
        cof[2] = b0 * c1 - b1 * c0
        cof[3] = c1 * a2 - c2 * a1
        cof[4] = c2 * a0 - c0 * a2
        cof[5] = c0 * a1 - c1 * a0
        cof[6] = a1 * b2 - a2 * b1
        cof[7] = a2 * b0 - a0 * b2
        cof[8] = a0 * b1 - a1 * b0
        det = a0 * cof[0] + a1 * cof[1] + a2 * cof[2]
        with np.errstate(divide='ignore', invalid='ignore'):
            r = 0.5 * (r + cof / det)
    # two Newton steps reach the polar factor only from a near-orthogonal start (HybrIK's float32 matrices).  Rows that are
    # not there yet (or improper / singular inputs) go through SciPy's SVD projection like the reference (which also raises
    # on non-finite input).
    a0, a1, a2, b0, b1, b2, c0, c1, c2 = r
    resid = np.maximum.reduce([np.abs(a0 * a0 + a1 * a1 + a2 * a2 - 1), np.abs(b0 * b0 + b1 * b1 + b2 * b2 - 1), np.abs(c0 * c0 + c1 * c1 + c2 * c2 - 1),
                               np.abs(a0 * b0 + a1 * b1 + a2 * b2), np.abs(a0 * c0 + a1 * c1 + a2 * c2), np.abs(b0 * c0 + b1 * c1 + b2 * c2)])
    bad = ~(det > 0) | ~(resid < 1e-9)
    if bad.any():
        from scipy.spatial.transform import Rotation
        r = r.copy()
        r[:, bad] = Rotation.from_matrix(R0[bad]).as_matrix().reshape(-1, 9).T
        a0, a1, a2, b0, b1, b2, c0, c1, c2 = r
    tr = a0 + b1 + c2
    d = np.stack([a0, b1, c2, tr])
    choice = d.argmax(axis=0)
    q = np.empty((4, n))
    R = r.reshape(3, 3, n)
    for i in range(3):
        sel = np.where(choice == i)[0]
        if sel.size == 0:
            continue
        j, k = (i + 1) % 3, (i + 2) % 3
        q[i, sel] = 1 - tr[sel] + 2 * R[i, i, sel]
        q[j, sel] = R[j, i, sel] + R[i, j, sel]
        q[k, sel] = R[k, i, sel] + R[i, k, sel]
        q[3, sel] = R[k, j, sel] - R[j, k, sel]
    sel = np.where(choice == 3)[0]
    q[0, sel] = R[2, 1, sel] - R[1, 2, sel]
    q[1, sel] = R[0, 2, sel] - R[2, 0, sel]
    q[2, sel] = R[1, 0, sel] - R[0, 1, sel]
    q[3, sel] = 1 + tr[sel]
    q /= np.sqrt((q * q).sum(axis=0))
    q[:, q[3] < 0] *= -1
    angle = 2 * np.arctan2(np.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]), q[3])
    small = angle <= 1e-3
    a2_ = angle * angle
    with np.errstate(divide='ignore', invalid='ignore'):
        scale = np.where(small, 2 + a2_ / 12 + 7 * a2_ * a2_ / 2880, angle / np.sin(angle / 2))
    return np.ascontiguousarray((scale * q[:3]).T)


class _Slot:
    def __init__(self, i):
        self.i = i


def _torch_dtype(np_dtype):
    return torch.from_numpy(np.zeros(0, np_dtype)).dtype


class _Upload:
    """Host arrays packed into one pinned buffer and sent to the device with one non-blocking copy; CUDA tensors are used
    where they are.  source() returns the tensor or a slot; get() the device tensor of either once allocate() ran."""

    def __init__(self):
        self._host, self._nbytes, self._views, self._dev = [], 0, None, None

    def source(self, x, device):
        if isinstance(x, torch.Tensor):
            if x.is_cuda:
                return x.detach().to(device)
            x = x.detach().numpy()
        return self._add(np.ascontiguousarray(x))

    def _add(self, a):
        off = (self._nbytes + 15) // 16 * 16
        self._host.append((a, off))
        self._nbytes = off + a.nbytes
        return _Slot(len(self._host) - 1)

    def reserve(self, nbytes):
        return self._add(np.zeros(nbytes, np.uint8))

    def host(self, h):
        return self._host[h.i][0]

    def shape(self, h):
        return tuple(h.shape) if isinstance(h, torch.Tensor) else self._host[h.i][0].shape

    def dtype(self, h):
        return h.dtype if isinstance(h, torch.Tensor) else _torch_dtype(self._host[h.i][0].dtype)

    def numel(self, h):
        return h.numel() if isinstance(h, torch.Tensor) else self._host[h.i][0].size

    def allocate(self, device):
        self._dev = torch.empty(max(self._nbytes, 16), dtype=torch.uint8, device=device)
        self._views = [self._dev[off:off + a.nbytes].view(_torch_dtype(a.dtype)).view(a.shape) for a, off in self._host]

    def get(self, h):
        return h if isinstance(h, torch.Tensor) else self._views[h.i]

    def fill(self, h, data):
        self._host[h.i][0][:] = np.frombuffer(data, np.uint8)

    def send(self):
        buf = torch.empty(self._dev.shape, dtype=torch.uint8, pin_memory=True)
        hb = buf.numpy()
        for a, off in self._host:
            hb[off:off + a.nbytes] = a.reshape(-1).view(np.uint8)
        self._dev.copy_(buf, non_blocking=True)


def _upload_index(arrays, device):
    """int64 index arrays -> device tensors with one pinned non-blocking copy"""
    up = _Upload()
    slots = [up.source(np.asarray(a, np.int64), device) for a in arrays]
    up.allocate(device)
    up.send()
    return [up.get(h) for h in slots]


def _sec_to_time(secs):
    secs = int(secs)
    return f'{secs // 3600}:{(secs % 3600) // 60:02d}:{secs % 60:02d}'


class GlobalReconOptimizer:

    def __init__(self, cfg, device=torch.device('cuda'), log=None, smpl=None, mt_model=None, dist=None):
        """cfg/device/log as in the reference (:25).  Extra, optional:
        smpl      a glamr_b200.smpl.SMPL (or an assets dict); default loads SMPL_MODEL_DIR like the reference
        mt_model  object with .inference(batch, sample_num) (the learned prior); default: the CUDA MotionTrajJointModel
        dist      (rank, world_size) for person sharding across GPUs (torch.distributed must be initialised)"""
        self.cfg = cfg
        self.specs = specs = cfg.grecon_model_specs
        self.device = L.require_cuda(device)
        self.log = log
        self.cur_iter = 0
        if isinstance(smpl, SMPL):
            self.smpl = smpl
        else:
            self.smpl = SMPL(smpl if smpl is not None else SMPL_MODEL_DIR, pose_type='body26fk', device=self.device)
        g = specs.get
        self.use_gt = g('use_gt', False)
        self.est_type = g('est_type', 'hybrik')
        self.flag_infer_motion_traj = g('flag_infer_motion_traj', False)
        self.flag_infill_motion = g('flag_infill_motion', True)
        self.flag_pred_traj = g('flag_pred_traj', True)
        self.flag_opt_traj = g('flag_opt_traj', True)
        self.flag_opt_cam = g('flag_opt_cam', True)
        self.flag_fixed_cam = g('flag_fixed_cam', False)
        self.flag_opt_vis_local_rot = g('flag_opt_vis_local_rot', False)
        self.flag_opt_person2cam_rot = g('flag_opt_person2cam_rot', False)
        self.flag_opt_person2cam_trans = g('flag_opt_person2cam_trans', False)
        self.flag_cam_inv_trans_res_all = g('flag_cam_inv_trans_res_all', True)
        self.flag_filter_pose = g('flag_filter_pose', True)
        self.flag_make_invis_with_keypoint = g('flag_make_invis_with_keypoint', False)
        self.make_invis_keypoint_min_score = g('make_invis_keypoint_min_score', 0.6)
        self.make_invis_keypoint_min_num = g('make_invis_keypoint_min_num', 15)
        self.flag_opt_cam_from_person_pose = g('flag_opt_cam_from_person_pose', False)
        self.flag_init_cam_all_frames = g('flag_init_cam_all_frames', False)
        self.cam_fix_frames = g('cam_fix_frames', [[0, None]])
        self.flag_traj_from_cam = g('flag_traj_from_cam', False)
        self.traj_interp_method = g('traj_interp_method', 'linear_interp')
        self.opt_stage_specs = self.cfg.opt_stage_specs
        for flag in ['flag_opt_motion_latent', 'flag_opt_traj_latent', 'flag_use_pen_loss']:
            if g(flag, False):
                raise NotImplementedError(f'{flag} is not implemented in the CUDA path (SURVEY.md §8(f)-4); no CPU fallback')
        if g('absolute_heading', False):
            raise NotImplementedError('absolute_heading is not implemented in the CUDA path: without latent optimisation the reference '
                                      "reads the predictor's per-frame heading increments as absolute headings (:283,:421), which "
                                      'does not give a usable trajectory')
        self.heading_type = g('heading_type', 'scalar')
        if self.heading_type not in ('scalar', 'vec'):
            raise ValueError(f"unknown heading_type {self.heading_type!r} (expected 'scalar' or 'vec')")
        self.heading_vec = self.heading_type == 'vec'
        # world_dxy gets its own block of theta only when a stage can create it, so every other problem keeps its layout
        self.world_dxy = any('world_dxy' in st.get('opt_variables', []) for st in cfg.opt_stage_specs.values())
        if self.flag_traj_from_cam and self.traj_interp_method not in ('linear_interp', 'last_pose'):
            raise ValueError(f'unknown traj interp method: {self.traj_interp_method}!')          # :347-348
        # the learned trajectory (predictor + codec) is optimised only through the local variables, which the reference
        # creates only with flag_opt_traj (:171-199); its forward then fails on the missing traj_local_xy (:397)
        if not self.flag_opt_traj and self.flag_infer_motion_traj and self.flag_pred_traj:
            raise ValueError('flag_opt_traj=false needs flag_infer_motion_traj=false or flag_pred_traj=false: the predicted '
                             'trajectory is composed with the local trajectory variables, which exist only with flag_opt_traj')
        # which trajectory the kernels evaluate (include/glamr_b200.h, enum glamr_traj_source)
        self.traj_source = L.TRAJ_PREDICTED if (self.flag_infer_motion_traj and self.flag_pred_traj) else L.TRAJ_BASE
        self.rank, self.world = dist if dist is not None else (0, 1)
        self.log_interval = g('log_interval', 1)
        self.use_cuda_graph = g('use_cuda_graph', True)
        self.mt_cfg = None
        self.mt_model = mt_model
        if mt_model is None and 'motion_traj_cfg' in specs and self.flag_infer_motion_traj:
            self.load_model()
        self._lib = L.load()
        self._opt = None
        self._consts = {}
        self.iter_ms = []              # (stage, niters, ms per iteration) of every optimize_main call

    def load_model(self):
        from .motion_traj import MotionTrajJointModel
        self.mt_model = MotionTrajJointModel(self.specs['motion_traj_cfg'], self.device, self.log, smpl=self.smpl)
        self.mt_cfg = getattr(self.mt_model, 'cfg', None)

    @property
    def _flags(self):
        return {k: getattr(self, k) for k in ['flag_fixed_cam', 'flag_opt_cam', 'flag_opt_cam_from_person_pose',
                                              'flag_cam_inv_trans_res_all', 'flag_opt_vis_local_rot', 'cam_fix_frames',
                                              'flag_opt_traj', 'traj_source', 'heading_vec', 'world_dxy', 'flag_opt_person2cam_rot',
                                              'flag_opt_person2cam_trans']}

    # ------------------------------------------------------------------------------------------------ init_data
    def _const(self, key, values):
        """small constant tensor on the device, uploaded once per optimiser"""
        c = self._consts.get(key)
        if c is None:
            c = self._consts[key] = torch.tensor(values, device=self.device)
        return c

    def _persons_from_estimates(self, in_dict, num_fr):
        """global_recon_model.py:88-137 and filter_pose (:250-271) for every person of the sequence on the device: the host
        arrays of all persons go up in one pinned copy, the rotation vectors, gap fill and filter_pose run as one launch each
        for all persons, and one read-back brings the visibility the host needs for its index tables.  Estimates may be
        numpy arrays or torch tensors (CPU or CUDA); the person dicts equal those of the numpy path."""
        dev, T = self.device, num_fr
        keys = list(in_dict['est'].keys())
        P = len(keys)
        up = _Upload()
        srcs = []
        for idx in keys:
            est = in_dict['est'][idx]
            gt = in_dict['gt'].get(idx)
            s = {n: up.source(x, dev) for n, x in [('exist', est['bboxes_dict']['exist']), ('rot', est['smpl_pose_quat_wroot']),
                                                    ('beta', est['smpl_beta']), ('trans', est['root_trans']), ('kp', est['kp_2d']),
                                                    ('K', est['cam_K'])]}
            if gt is not None:
                s['gt'] = up.source(gt['pose'][:, 3:], dev)
            srcs.append(s)
        for idx, s in zip(keys, srcs):
            nv = up.shape(s['rot'])[0]
            if up.shape(s['exist'])[0] != T:
                raise ValueError(f'person {idx}: bboxes_dict.exist has {up.shape(s["exist"])[0]} frames, person 0 has {T}')
            if nv == 0 or (nv < T and nv < 2):
                raise ValueError(f'person {idx}: {nv} visible frames; filling the invisible frames needs at least two')
            ex = s['exist']
            if not isinstance(ex, torch.Tensor) and np.count_nonzero(up.host(ex)) != nv:
                raise ValueError(f'person {idx}: bboxes_dict.exist marks {np.count_nonzero(up.host(ex))} frames visible, the estimates have {nv} rows')
            for n in ('beta', 'trans'):
                if up.dtype(s[n]) not in (torch.float32, torch.float64):
                    raise TypeError(f'person {idx}: {n} must be float32 or float64, got {up.dtype(s[n])}')
        nvs = [up.shape(s['rot'])[0] for s in srcs]
        s0 = np.concatenate([[0], np.cumsum(nvs)]).astype(np.int64)
        J = up.numel(srcs[0]['rot']) // (nvs[0] * 9)
        jobs_slot = up.reserve(8 * P * ctypes.sizeof(L.FillJob))
        up.allocate(dev)
        get = up.get
        f32, f64 = torch.float32, torch.float64
        exists = [get(s['exist']) for s in srcs]
        rot_dt = f64 if any(get(s['rot']).dtype != f32 for s in srcs) else f32
        N = int(s0[-1]) * J
        rot_all = torch.empty((N, 9), dtype=rot_dt, device=dev)
        after_send = [lambda: [rot_all[s0[p] * J:s0[p + 1] * J].copy_(get(s['rot']).reshape(-1, 9)) for p, s in enumerate(srcs)]]
        aa_all = torch.empty((N, 3), device=dev)
        flags = torch.empty(N, dtype=torch.uint8, device=dev)
        rb = torch.zeros(1 + 3 * P + P * T, dtype=torch.int32, device=dev)
        pose_all = torch.empty((P, T, (J - 1) * 3), device=dev)
        orient_all = torch.empty((P, T, 3), device=dev)
        kp_all = torch.empty((P, T, 26, 2), dtype=f64, device=dev)
        score_all = torch.empty((P, T, 26), dtype=f64, device=dev)
        aligned_all = torch.empty((P, T, 26, 2), dtype=f64, device=dev)
        K_all = torch.empty((P, T) + tuple(up.shape(srcs[0]['K'])[1:]), device=dev)
        m0, m1 = self._const('kp_dst', SMPL_TO_BODY26FK[:, 0].tolist()), self._const('kp_src', SMPL_TO_BODY26FK[:, 1].tolist())
        keep, jobs, outs = [], [], []
        for p, s in enumerate(srcs):
            nv, gaps = nvs[p], int(nvs[p] < T)
            o = {}
            aa_p = aa_all[s0[p] * J:s0[p + 1] * J]
            jobs.append((aa_p, pose_all[p], p, (J - 1) * 3, J * 3, 3, L.FILL_F32, gaps))
            jobs.append((aa_p, orient_all[p], p, 3, J * 3, 0, L.FILL_F32, gaps))
            for n in ('beta', 'trans'):
                x = get(s[n])                       # only its pointer is read before the upload: host arrays arrive contiguous
                o[n] = torch.empty((T,) + tuple(x.shape[1:]), dtype=x.dtype, device=dev)
                C = x.numel() // nv
                jobs.append((x.contiguous(), o[n], p, C, C, 0, L.FILL_F32 if x.dtype == f32 else L.FILL_F64, gaps))
            kp2 = torch.zeros((nv, 26, 2), dtype=f64, device=dev)
            score = torch.zeros((nv, 26), dtype=f64, device=dev).index_fill_(1, m0, 1.0)
            camk = torch.empty(up.shape(s['K']), device=dev)
            after_send.append(lambda kp2=kp2, camk=camk, s=s: (kp2.index_copy_(1, m0, get(s['kp'])[:, :24].index_select(1, m1).to(f64)),
                                                              camk.copy_(get(s['K']))))
            jobs += [(kp2, kp_all[p], p, 52, 52, 0, L.FILL_F64, 0), (score, score_all[p], p, 26, 26, 0, L.FILL_F64, 0),
                     (kp2, aligned_all[p], p, 52, 52, 0, L.FILL_F64, 0), (camk, K_all[p], p, camk[0].numel(), camk[0].numel(), 0, L.FILL_F32, 0)]
            keep += [kp2, score, camk]
            outs.append(o)
        table = (L.FillJob * len(jobs))(*[L.FillJob(src.data_ptr(), dst.data_ptr(), p, C, stride, col0, kind, interp, nvs[p])
                                            for src, dst, p, C, stride, col0, kind, interp in jobs])
        up.fill(jobs_slot, bytes(table))
        up.send()
        for f in after_send:
            f()
        jobs_dev = up.get(jobs_slot)
        vis_orig = torch.stack([e.to(f32) for e in exists]).contiguous()
        before = torch.empty((P, T), dtype=torch.int32, device=dev)
        frames = torch.empty((P, T), dtype=torch.int32, device=dev)
        exist_all = torch.empty((P, T), dtype=torch.bool, device=dev)
        jump = torch.empty((P, T), dtype=torch.uint8, device=dev)
        info, visf_dev = rb[1:1 + 3 * P], rb[1 + 3 * P:]
        lib = self._lib
        with torch.cuda.device(dev):
            st = L.stream_ptr()
            L.check(lib.glamr_init_rotvec(N, L.ptr(rot_all), int(rot_dt == f64), L.ptr(aa_all), L.ptr(flags), L.ptr(rb), st), 'glamr_init_rotvec')
            L.check(lib.glamr_init_vis_tables(P, T, L.ptr(vis_orig), L.ptr(before), L.ptr(frames), L.ptr(info), L.ptr(exist_all), st),
                    'glamr_init_vis_tables')
        max_cols = max(j[3] for j in jobs)
        kp_rule = self.flag_filter_pose and self.flag_make_invis_with_keypoint

        def fill_and_filter():
            vis = vis_orig.clone()
            with torch.cuda.device(dev):
                L.check(lib.glamr_init_fill(len(jobs), L.ptr(jobs_dev), T, max_cols, L.ptr(before), L.ptr(frames), L.ptr(info), L.stream_ptr()),
                        'glamr_init_fill')
                L.check(lib.glamr_init_filter_pose(P, T, int(self.flag_filter_pose), L.ptr(orient_all), L.ptr(vis), L.ptr(jump),
                                                   L.ptr(score_all) if kp_rule else None, ctypes.c_double(self.make_invis_keypoint_min_score),
                                                   ctypes.c_double(self.make_invis_keypoint_min_num), L.ptr(visf_dev), L.stream_ptr()),
                        'glamr_init_filter_pose')
            host = torch.empty(rb.shape, dtype=torch.int32, pin_memory=True)
            host.copy_(rb, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()                 # the one read-back of init_data
            return vis, host.numpy()
        vis32, rb_h = fill_and_filter()
        if rb_h[0] > 0:
            # rows the Newton steps could not bring onto SO(3) (not HybrIK's float32 rotations): SciPy's projection, as
            # rotmats_to_rotvec does, then the fill and the filter again
            bad = torch.nonzero(flags).reshape(-1)
            aa_all[bad] = torch.from_numpy(rotmats_to_rotvec(rot_all[bad].cpu().numpy()).astype(np.float32)).to(dev)
            vis32, rb_h = fill_and_filter()
        info_h = rb_h[1:1 + 3 * P].reshape(P, 3)
        visf_h = rb_h[1 + 3 * P:].reshape(P, T).astype(bool)
        self._init_host = {}
        persons = {}
        for p, (idx, s) in enumerate(zip(keys, srcs)):
            if info_h[p, 0] != nvs[p]:
                raise ValueError(f'person {idx}: bboxes_dict.exist marks {info_h[p, 0]} frames visible, the estimates have {nvs[p]} rows')
            ex = exists[p]
            visible = vis32[p].to(ex.dtype) if self.flag_filter_pose else ex.clone()
            start, end = np.int64(info_h[p, 1]), np.int64(info_h[p, 2] + 1)
            d = {'visible': visible, 'visible_orig': ex.clone(), 'fr_start': start, 'fr_end': end, 'exist_frames': exist_all[p],
                 'exist_len': end - start, 'max_len': T, 'frames': torch.arange(T, device=dev), 'vis_frames': visible == 1,
                 'invis_frames': visible == 0, 'frame2ind': {f: i for i, f in enumerate(np.arange(T))}, 'scale': None,
                 'smpl_pose': pose_all[p]}
            if 'gt' in s:
                gt = get(s['gt'])          # a caller's CUDA tensor is copied, as the numpy path copies
                d['smpl_pose_gt'] = gt.clone(memory_format=torch.contiguous_format) if isinstance(s['gt'], torch.Tensor) else gt
            d['smpl_beta'] = outs[p]['beta']
            d['smpl_orient_cam'] = orient_all[p]
            d['root_trans_cam'] = outs[p]['trans']
            d['kp_2d'], d['kp_2d_score'], d['kp_2d_aligned'], d['cam_K'] = kp_all[p], score_all[p], aligned_all[p], K_all[p]
            persons[idx] = d
            self._init_host[idx] = {'p': p, 'vis': visf_h[p], 'start': int(start), 'end': int(end)}
        self._init_visf = (visf_h, visf_dev.view(P, T))
        self._init_tables_f = None
        return persons

    def _filtered_tables(self):
        """sample tables (glamr_init_vis_tables) of the filtered visibility: the heading interpolants' samples"""
        if self._init_tables_f is None:
            visf_h, visf_dev = self._init_visf
            P, T = visf_h.shape
            vis = visf_dev.to(torch.float32)
            t = tuple(torch.empty((P, T), dtype=torch.int32, device=self.device) for _ in range(2)) + \
                (torch.empty((P, 3), dtype=torch.int32, device=self.device),)
            with torch.cuda.device(self.device):
                L.check(self._lib.glamr_init_vis_tables(P, T, L.ptr(vis), L.ptr(t[0]), L.ptr(t[1]), L.ptr(t[2]), None, L.stream_ptr()),
                        'glamr_init_vis_tables')
            self._init_tables_f = t
        return self._init_tables_f

    def infer_motion_traj(self, d):
        """:353-392"""
        if self.mt_model is None:
            return
        ex = _exist_range(d)
        batch = {'in_body_pose': d['smpl_pose_nofill'][ex].unsqueeze(0).clone(), 'frame_mask': d['visible'][ex].unsqueeze(0).clone()}
        out = self.mt_model.inference(batch, sample_num=1)
        self._take_prior_output(d, out, 0)

    def infer_motion_traj_all(self, persons):
        """The reference runs the learned prior once per person with batch size 1 (:230-232 -> :353-392).  When every
        person exists for the same number of frames and the prior object declares `supports_person_batch`, the persons
        form one batch [P, T, 69] instead (SURVEY.md §8(f)-1): same per-person arithmetic, P times fewer launches.  Persons of
        different lengths go into one ragged call when the prior declares `supports_ragged_batch`, with each person's outputs and
        eps those of its own call."""
        if self.mt_model is None:
            return
        ds = list(persons.values())
        lens = {int(d['exist_len']) for d in ds}
        if len(ds) > 1 and len(lens) == 1 and getattr(self.mt_model, 'supports_person_batch', False):
            batch = {'in_body_pose': torch.stack([d['smpl_pose_nofill'][_exist_range(d)] for d in ds]),
                     'frame_mask': torch.stack([d['visible'][_exist_range(d)] for d in ds])}
            out = self.mt_model.inference(batch, sample_num=1)
            for b, d in enumerate(ds):
                self._take_prior_output(d, out, b)
        elif len(ds) > 1 and getattr(self.mt_model, 'supports_ragged_batch', False):
            # persons of different exist lengths: one ragged call whose row p reproduces person p's own call, eps included (the
            # prior draws them person by person in the serial calls' order and shapes)
            self._ragged_prior(ds, [1] * len(ds))
        else:
            for d in ds:
                self.infer_motion_traj(d)

    def _prior_rows(self, persons):
        """the persons and the row_batch of each in a ragged prior call that reproduces infer_motion_traj_all: one block of P for
        P persons of one exist length, else one row per person"""
        ds = list(persons.values())
        lens = {int(d['exist_len']) for d in ds}
        P = len(ds)
        block = P > 1 and len(lens) == 1 and getattr(self.mt_model, 'supports_person_batch', False)
        return ds, [P if block else 1] * P

    def _ragged_prior(self, ds, row_batch, latents=None):
        """one ragged prior call over the exist ranges of the persons `ds` (of one or several data dicts); each person's outputs
        and, without `latents`, its eps are those of its serial call"""
        seq_len = [int(d['exist_len']) for d in ds]
        Tm = max(seq_len)
        pose = torch.zeros((len(ds), Tm, 69), device=self.device)
        mask = torch.zeros((len(ds), Tm), device=self.device)
        for b, d in enumerate(ds):
            pose[b, :seq_len[b]] = d['smpl_pose_nofill'][_exist_range(d)]
            mask[b, :seq_len[b]] = d['visible'][_exist_range(d)]
        batch = {'in_body_pose': pose, 'frame_mask': mask, 'seq_len': seq_len, **(latents or {})}
        out = self.mt_model.inference(batch, sample_num=1, row_batch=row_batch)
        for b, d in enumerate(ds):
            n = seq_len[b]
            self._take_prior_output(d, {'infer_out_body_pose': out['infer_out_body_pose'][:, :, :n],
                                        'infer_out_local_traj_tp': out['infer_out_local_traj_tp'][:n],
                                        'infer_out_pose': out['infer_out_pose'][:, :, :n],
                                        'infer_out_orient': out['infer_out_orient'][:, :, :n],
                                        'infer_out_trans': out['infer_out_trans'][:, :, :n]}, b)

    def _take_prior_output(self, d, out, b):
        """:368-392 for batch row b of the prior's output"""
        ex = _exist_range(d)
        if self.flag_infill_motion:
            d['infilled'] = True
            d['smpl_pose'] = d['smpl_pose'].detach().clone()
            d['smpl_pose'][ex] = out['infer_out_body_pose'][b, 0].to(d['smpl_pose'])
        if self.flag_pred_traj:
            d['traj_predicted'] = True
            d['traj_local_pred'] = out['infer_out_local_traj_tp'][:, b, 0, :].clone().float()
            d['smpl_orient_world_base'] = d['smpl_orient_world_base'].detach().clone()
            d['root_trans_world_base'] = d['root_trans_world_base'].detach().clone()
            if 'infer_out_pose' in out:
                d['smpl_orient_world_base'][ex] = out['infer_out_pose'][b, 0, :, :3].to(d['smpl_orient_world_base'])
            if 'infer_out_orient' in out:
                d['smpl_orient_world_base'][ex] = out['infer_out_orient'][b, 0].to(d['smpl_orient_world_base'])
            d['root_trans_world_base'][ex] = out['infer_out_trans'][b, 0].to(d['root_trans_world_base'])
            d['smpl_orient_world'] = d['smpl_orient_world_base']
            d['root_trans_world'] = d['root_trans_world_base']

    def init_default_traj(self, d):
        """:319-323"""
        d['root_trans_world_base'][:] = self._const('default_trans', [0.0, 0.0, 0.8])
        d['smpl_orient_world_base'][:] = G.quaternion_to_angle_axis(self._const('default_q', [[0.0, 0.0, 0.7071, 0.7071]]))[0]
        d['root_trans_world'] = d['root_trans_world_base']
        d['smpl_orient_world'] = d['smpl_orient_world_base']

    def get_traj_from_cam(self, data):
        """:325-351 -- the world trajectory seen through the initial camera: translation as observed (the estimate is
        already interpolated over gaps), orientation interpolated with separate heading ('linear_interp') or both held at
        the last visible frame over the exist range ('last_pose', which also holds the body pose unless the prior infilled it)."""
        ds = data['person_data']
        trans, orient_q = {}, {}
        for key, d in ds.items():
            d['person_transform_world'] = torch.matmul(data['cam_pose_inv'], d['person_transform_cam'])
            trans[key] = d['person_transform_world'][:, :3, 3]
            orient_q[key] = G.rotation_matrix_to_quaternion(d['person_transform_world'][:, :3, :3].contiguous())
        if self.traj_interp_method == 'linear_interp':
            orient_q = self._interp_orient_q_sep_heading(orient_q)
        else:
            # forward fill from the last visible frame, over the exist range only (its first frame is visible); the
            # source frames are visible, so one gather reproduces the reference's frame-by-frame loop.  One upload for all persons.
            fills = {}
            for key in ds:
                h = self._init_host[key]
                vis_h = h['vis']
                src = np.maximum.accumulate(np.where(vis_h, np.arange(len(vis_h)), 0))
                fill = np.nonzero(~vis_h[h['start']:h['end']])[0] + h['start']
                if fill.size:
                    fills[key] = (fill, src[fill])
            idx = iter(_upload_index([a for f in fills.values() for a in f], self.device)) if fills else None
            for key, d in ds.items():
                if key in fills:
                    dst_t, src_t = next(idx), next(idx)
                    trans[key][dst_t] = trans[key][src_t]
                    orient_q[key][dst_t] = orient_q[key][src_t]
                    if not (self.flag_infer_motion_traj and self.flag_infill_motion):
                        d['smpl_pose'][dst_t] = d['smpl_pose'][src_t]
        for key, d in ds.items():
            d['root_trans_world'] = d['root_trans_world_base'] = trans[key]
            d['smpl_orient_world'] = d['smpl_orient_world_base'] = G.quaternion_to_angle_axis(orient_q[key])

    def init_cam_pose(self, data, all_frames=False):
        """:294-317"""
        d0 = next(iter(data['person_data'].values()))          # the reference builds every person's candidate and takes person 0's
        cand = torch.matmul(d0['person_transform_world'], d0['person2cam']) * d0['vis_frames'][:, None, None]
        has = data['fr_num_persons'] > 0
        start = int(np.nonzero(self._init_visf[0].any(axis=0))[0][0])
        inv = torch.where(has[:, None, None], cand, torch.zeros_like(data['cam_pose']))
        data['pose_infer_cam_pose_inv'] = inv
        # all_frames: the reference's forward fill over frames without persons writes into the data['cam_pose_inv'] that
        # the assignment below replaces, so the frames without persons keep zeros
        if not all_frames:
            inv[...] = inv[start].clone()
        inv[:, :3, :3] = G.rot6d_to_rotmat(G.rotmat_to_rot6d(inv[:, :3, :3]))
        data['cam_pose_inv'] = inv
        data['cam_pose'] = G.inverse_transform(inv)

    def _traj_local2global(self, locals_, local_heading=True):
        """traj_pred/utils/traj_utils.py:65-88 for a list of sequences [L_i,11] -> [(trans [L_i,3], orient_q [L_i,4])], one launch
        per distinct length (the kernel runs one CTA per sequence)"""
        out = [None] * len(locals_)
        by_len = {}
        for i, l in enumerate(locals_):
            by_len.setdefault(l.shape[0], []).append(i)
        for T, idx in by_len.items():
            B = len(idx)
            loc = torch.stack([locals_[i].float() for i in idx], dim=1).contiguous()        # time-major [T,B,11]
            trans = torch.empty((T, B, 3), device=self.device)
            oq = torch.empty((T, B, 4), device=self.device)
            scratch = torch.empty(B * T * 3, device=self.device)
            with torch.cuda.device(self.device):
                L.check(self._lib.glamr_traj_local2global(T, B, L.ptr(loc), int(local_heading), L.ptr(trans), L.ptr(oq), L.ptr(scratch),
                                                          L.stream_ptr()), 'glamr_traj_local2global')
            for b, i in enumerate(idx):
                out[i] = (trans[:, b], oq[:, b])
        return out

    def _traj_global2local(self, trans, orient_q):
        """traj_pred/utils/traj_utils.py:44-62 (init only) for [..., T, 3] / [..., T, 4]"""
        base = self._const('base_q', [0.5, 0.5, 0.5, 0.5])
        xy, z = trans[..., :2], trans[..., 2]
        q = G.quat_mul(orient_q, G.quat_conjugate(base).expand_as(orient_q))
        heading = G.get_heading(q)
        d6 = G.quat_to_rot6d(G.deheading_quat(q, G.get_heading_q(q)))
        d_heading = torch.cat([heading[..., :1], heading[..., 1:] - heading[..., :-1]], dim=-1)
        hvec = G.heading_to_vec(d_heading)
        dxy = xy[..., 1:, :] - xy[..., :-1, :]
        th = -heading[..., :-1]
        c, s = torch.cos(th), torch.sin(th)
        dxy_h = torch.stack([dxy[..., 0] * c - dxy[..., 1] * s, dxy[..., 0] * s + dxy[..., 1] * c], dim=-1)
        return torch.cat([torch.cat([xy[..., :1, :], dxy_h], dim=-2), z.unsqueeze(-1), d6, hvec], dim=-1)

    def _interp_orient_q_sep_heading(self, orient_q):
        """traj_pred/utils/traj_utils.py:120-142 for every person: orient_q {key: [T,4]} -> {key: [T,4]}.  The heading vectors
        and 6d rotations of each person's visible frames are linearly interpolated over the invisible ones (glamr_init_fill,
        SciPy's operation order), all persons in one upload and one launch."""
        before, frames, info = self._filtered_tables()
        visf_h = self._init_visf[0]
        keys = list(orient_q)
        ps = [self._init_host[k]['p'] for k in keys]
        T = visf_h.shape[1]
        ns = [int(visf_h[p].sum()) for p in ps]
        for k, n in zip(keys, ns):
            if n < T and n < 2:              # filter_pose can leave fewer samples than the estimates had
                raise ValueError(f'x and y arrays must have at least 2 entries: {n} frames of person {k} stay visible after '
                                 'filter_pose, too few to interpolate the orientation over the others')
        rows = np.concatenate([np.nonzero(visf_h[p])[0] + i * T for i, p in enumerate(ps)])
        offs = np.concatenate([[0], np.cumsum(ns)])
        packed = torch.empty((int(offs[-1]), 8), device=self.device)
        both = torch.empty((len(keys), T, 8), device=self.device)
        # a person whose every frame is a sample copies its samples, as the reference skips the interpolation
        table = (L.FillJob * len(keys))(*[L.FillJob(packed[offs[i]:].data_ptr() if ns[i] else packed.data_ptr(), both[i].data_ptr(), p, 8, 8, 0,
                                                    L.FILL_F32_W64, int(ns[i] < T), ns[i]) for i, p in enumerate(ps)])
        up = _Upload()
        rows_slot = up.source(rows.astype(np.int64), self.device)
        job_slot = up.source(np.frombuffer(bytes(table), np.uint8), self.device)
        up.allocate(self.device)
        up.send()
        q_all = torch.stack([orient_q[k] for k in keys]).reshape(-1, 4)
        q_vis = q_all.index_select(0, up.get(rows_slot))
        base = self._const('base_q', [0.5, 0.5, 0.5, 0.5])
        q = G.quat_mul(q_vis, G.quat_conjugate(base).expand_as(q_vis))
        hq = G.get_heading_q(q)
        torch.cat([G.heading_to_vec(G.get_heading(q)), G.quat_to_rot6d(G.deheading_quat(q, hq))], dim=-1, out=packed)
        with torch.cuda.device(self.device):
            L.check(self._lib.glamr_init_fill(len(keys), L.ptr(up.get(job_slot)), T, 8, L.ptr(before), L.ptr(frames), L.ptr(info),
                                              L.stream_ptr()), 'glamr_init_fill')
        hvec_i, d6_i = both[..., :2].contiguous(), both[..., 2:].contiguous()
        out = G.quat_mul(G.heading_to_quat(G.vec_to_heading(hvec_i)), G.rot6d_to_quat(d6_i))
        out = G.quat_mul(out, base.expand_as(out))
        return {k: out[i] for i, k in enumerate(keys)}

    def init_traj_heading_from_cam(self, data):
        """:273-292 for every person: the interpolation and global->local conversion over [P, T], the codec per exist length"""
        ds = data['person_data']
        world = {key: torch.matmul(data['cam_pose_inv'], d['person_transform_cam']) for key, d in ds.items()}
        q = {key: G.rotation_matrix_to_quaternion(w[:, :3, :3].contiguous()) for key, w in world.items()}
        q_interp = self._interp_orient_q_sep_heading(q)
        keys = list(ds)
        local = self._traj_global2local(torch.stack([world[k][:, :3, 3] for k in keys]), torch.stack([q_interp[k] for k in keys]))
        for i, (key, d) in enumerate(ds.items()):
            ex = _exist_range(d)
            for (s, e) in self.cam_fix_frames:
                d['traj_local_pred'][s:e, -2:] = local[i][ex][s:e, -2:]
        codec = self._traj_local2global([d['traj_local_pred'] for d in ds.values()])
        for (trans, oq), d in zip(codec, ds.values()):
            ex = _exist_range(d)
            d['smpl_orient_world_base'] = d['smpl_orient_world_base'].detach().clone()
            d['root_trans_world_base'] = d['root_trans_world_base'].detach().clone()
            d['smpl_orient_world_base'][ex] = G.quaternion_to_angle_axis(oq)
            d['root_trans_world_base'][ex] = trans
            d['smpl_orient_world'] = d['smpl_orient_world_base'].clone()
            d['root_trans_world'] = d['root_trans_world_base'].clone()
            d['person_transform_world'] = G.make_transform(d['smpl_orient_world'], d['root_trans_world'], 'axis_angle')

    def init_data(self, in_dict):
        st = self._init_data_head(in_dict)
        if self.flag_infer_motion_traj:
            self.infer_motion_traj_all(st['persons'])
        return self._init_data_tail(st)

    def _init_data_head(self, in_dict):
        """init_data up to the learned prior -> the state _init_data_tail finishes from"""
        if self.est_type != 'hybrik':
            raise ValueError(f'est_type {self.est_type} not supported')
        dev = self.device
        num_fr = len(in_dict['est'][0]['bboxes_dict']['exist'])
        cam_pose = torch.eye(4, device=dev).repeat(num_fr, 1, 1)
        cam_pose_inv = G.inverse_transform(cam_pose)
        persons = self._persons_from_estimates(in_dict, num_fr)
        for d in persons.values():
            d['root_trans_world'] = G.transform_trans(cam_pose_inv, d['root_trans_cam'].float())
            d['smpl_orient_world'] = G.transform_rot(cam_pose_inv, d['smpl_orient_cam'].float())
            d['root_trans_world_base'] = d['root_trans_world'].clone()
            d['smpl_orient_world_base'] = d['smpl_orient_world'].clone()
            d['smpl_pose_nofill'] = d['smpl_pose'].clone()
            d['smpl_pose_nofill'][:int(d['fr_start'])] = 0.0
            d['smpl_pose_nofill'][int(d['fr_end']):] = 0.0
        return {'in_dict': in_dict, 'num_fr': num_fr, 'cam_pose': cam_pose, 'cam_pose_inv': cam_pose_inv, 'persons': persons,
                'init_state': (self._init_host, self._init_visf, self._init_tables_f)}

    def _init_data_tail(self, st):
        """init_data after the learned prior"""
        dev, in_dict, num_fr, persons = self.device, st['in_dict'], st['num_fr'], st['persons']
        cam_pose, cam_pose_inv = st['cam_pose'], st['cam_pose_inv']
        self._init_host, self._init_visf, self._init_tables_f = st['init_state']
        if not (self.flag_infer_motion_traj and self.flag_pred_traj):
            for d in persons.values():
                self.init_default_traj(d)
        for d in persons.values():
            d['person_transform_world'] = G.make_transform(d['smpl_orient_world'], d['root_trans_world'], 'axis_angle')
            d['person_transform_cam'] = G.make_transform(d['smpl_orient_cam'].float(), d['root_trans_cam'].float(), 'axis_angle')
            d['person2cam'] = G.inverse_transform(d['person_transform_cam'])
        rel = None
        if self.flag_opt_traj:                                     # :171-205
            last = d
            for d in persons.values():
                if self.flag_opt_person2cam_rot or self.flag_opt_person2cam_trans:        # identity 6d, zero translation (:173-175)
                    d['person2cam_res_rot'] = self._const('p2c_rot', [1., 0., 0., 0., 1., 0.]).repeat(num_fr, 1)
                    d['person2cam_res_trans'] = torch.zeros(num_fr, 3, device=dev)
                d['smpl_orient_world_res'] = torch.zeros_like(last['smpl_orient_world'])
                d['root_trans_world_res'] = torch.zeros_like(last['root_trans_world'])
            rel = {}
            ids = list(persons.keys())
            for i in range(len(ids)):
                for j in range(len(ids)):
                    if i != j:
                        rel[(i, j)] = torch.matmul(G.inverse_transform(persons[ids[i]]['person_transform_cam']), persons[ids[j]]['person_transform_cam'])
            if self.flag_pred_traj:
                for d in persons.values():
                    Ln = int(d['exist_len'].sum())
                    d['traj_local_xy'] = torch.zeros(2, device=dev)
                    d['traj_local_dxy'] = torch.zeros(Ln - 1, 2, device=dev)
                    hd = 2 if self.heading_vec else 1                   # heading_type 'vec': heading vectors (:191-196)
                    d['traj_local_heading'] = torch.zeros(hd, device=dev)
                    d['traj_local_dheading'] = torch.zeros((Ln - 1, 2) if self.heading_vec else (Ln - 1,), device=dev)
                    d['traj_local_z'] = torch.zeros(Ln, device=dev)
                    d['traj_local_rot'] = torch.zeros(Ln, 6, device=dev)
            else:
                for d in persons.values():
                    d['root_trans_world_base'][:] = d['root_trans_world_base'][0].clone()
                    d['smpl_orient_world_base'][:] = d['smpl_orient_world_base'][0].clone()
        fr_num_persons = sum(d['vis_frames'] for d in persons.values())
        n_empty = int((~self._init_visf[0].any(axis=0)).sum())
        data = {
            'seq_name': in_dict['seq_name'], 'person_data': persons, 'seq_len': num_fr, 'fr_num_persons': fr_num_persons,
            'cam_pose': cam_pose, 'cam_pose_inv': cam_pose_inv,
            'cam_inv_rot_residual': torch.zeros(n_empty, 6, device=dev),
            'cam_inv_trans_residual': torch.zeros(num_fr if self.flag_cam_inv_trans_res_all else n_empty, 3, device=dev),
            'rel_transform_cam': rel, 'gt': in_dict['gt'], 'gt_meta': in_dict['gt_meta'],
            'meta': {'algo': 'global_recon', 'mt_cfg': getattr(self.mt_cfg, 'yml_dict', None), 'num_fr': num_fr},
        }
        self.init_cam_pose(data)
        if self.flag_traj_from_cam:
            self.get_traj_from_cam(data)
        if self.flag_infer_motion_traj and self.flag_pred_traj:
            self.init_traj_heading_from_cam(data)
        if self.flag_init_cam_all_frames:
            self.init_cam_pose(data, all_frames=True)
        self._attach(data)
        self.forward(data, [], {'stage': 'init'})
        return data

    # ------------------------------------------------------------------------------------------------ device state
    def _attach(self, data):
        """Pack the optimisation variables into theta and build the constant tables.  The CUDA handle (scratch arena,
        Adam moments, captured iteration graph) is kept across calls while (P, T, J, n_params) and the group shapes stay the same.
        `data`: one data dict, or the groups of optimize_batch (a list of per-sequence lists of seed dicts)."""
        self._fresh_attach = True
        self._data = data
        self._n_groups = len(PB._groups(data))
        self._layout = PB.make_layout(data, self._flags)
        self._theta = torch.zeros(self._layout.n_params, device=self.device)
        PB.bind_variables(data, self._layout, self._theta)
        self._comp = PB.StageCompiler(data, self._layout, self._flags, self.device, G.angle_axis_to_rot6d, num_joints=self.smpl.num_joints,
                                      aa_to_quat=G.angle_axis_to_quaternion)
        # [grad | term sums of every group], and the loss terms of every group
        self._reduce = torch.zeros(self._layout.n_params + self._n_groups * NUM_TERMS, device=self.device)
        self._terms = torch.zeros(self._n_groups * (NUM_TERMS + 1), device=self.device)
        self._stage_key = None
        # multi-GPU: contiguous shards of the frame-persons n = p*T + t (SMPL + per-frame residuals are independent per
        # frame-person, so a person may straddle two ranks; P persons on P GPUs gives one person each)
        N = self._comp.N
        self._n_range = (N * self.rank // self.world, N * (self.rank + 1) // self.world)

    def _release(self, at_exit=False):
        if getattr(self, '_opt', None):
            if not at_exit:
                self._drop_peers()
            self._lib.glamr_opt_destroy(self._opt)
        self._opt = None

    # ------------------------------------------------------------------------------------------------ multi-GPU
    def _setup_peers(self):
        """Exchange CUDA-IPC handles of one small buffer per rank so that the per-iteration gradient reduction runs over
        NVLink peer memory inside the Adam kernel (include/glamr_b200.h, glamr_opt_set_peers).  Collective: every rank
        calls it at the same point.  Opt-in (GLAMR_ALLREDUCE=peer): the NCCL all-reduce captured in the iteration graph
        is the default; any rank failing to map a peer also falls back to NCCL."""
        import os
        self._peer_ok, self._peer_own, self._peer_opened = False, None, []
        if self.world <= 1:
            return
        dist, lib = torch.distributed, self._lib
        want = os.environ.get('GLAMR_ALLREDUCE', 'nccl') == 'peer' and self.world <= 8
        own, handle = ctypes.c_void_p(), (ctypes.c_ubyte * 64)()
        ok = want
        if ok:
            lib.glamr_opt_peer_bytes.restype = ctypes.c_size_t
            ok = lib.glamr_peer_alloc(ctypes.c_size_t(lib.glamr_opt_peer_bytes(self._opt)), ctypes.byref(own), handle) == 0
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(handle) if ok else None)
        ptrs = []
        if all(h is not None for h in handles):
            for r, h in enumerate(handles):
                if r == self.rank:
                    ptrs.append(own.value)
                    continue
                p = ctypes.c_void_p()
                if lib.glamr_peer_open((ctypes.c_ubyte * 64).from_buffer_copy(h), ctypes.byref(p)) != 0:
                    ok = False
                    break
                ptrs.append(p.value)
                self._peer_opened.append(p)
        else:
            ok = False
        flag = torch.tensor([1 if ok else 0], device=self.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        self._peer_own = own if own.value else None
        if int(flag[0]) == 1:
            table = (ctypes.c_void_p * self.world)(*ptrs)
            L.check(lib.glamr_opt_set_peers(self._opt, self.rank, self.world, table), 'glamr_opt_set_peers')
            self._peer_ok = True
        else:
            self._drop_peers(collective=False)
            if self.log is not None and want:
                self.log.info('peer-memory gradient reduction unavailable; using the NCCL all-reduce')

    def _drop_peers(self, collective=True):
        lib = self._lib
        if getattr(self, '_peer_ok', False):
            torch.cuda.synchronize(self.device)
            if collective:
                torch.distributed.barrier()             # nobody may still be reading this rank's buffer
            lib.glamr_opt_set_peers(self._opt, 0, 0, None)
        for p in getattr(self, '_peer_opened', []):
            lib.glamr_peer_close(p)
        if getattr(self, '_peer_own', None) is not None:
            lib.glamr_peer_free(self._peer_own)
        self._peer_ok, self._peer_own, self._peer_opened = False, None, []

    def __del__(self):
        try:
            self._release(at_exit=True)            # no collectives in a finaliser; peer buffers die with the process
        except Exception:
            pass

    def _set_stage(self, data, opt_variables, loss_cfg, stage, reset_adam, begin=False):
        if begin:            # get_parameter side effects happen once per optimize_main, not on every forward
            PB.begin_stage_variables(data, self._layout, self._theta, self._flags, opt_variables)
        pb = self._comp.compile(self._theta, opt_variables, loss_cfg, stage, n_begin=self._n_range[0], n_end=self._n_range[1],
                                owner=(self.rank == 0))
        self._pb = pb
        dims = (pb.P, pb.T, pb.J, pb.n_params, tuple(zip(self._comp.Qs, self._comp.Ts)))
        if self._opt is not None and dims != getattr(self, '_opt_dims', None):
            self._release()
        with torch.cuda.device(self.device):
            if self._opt is None:
                self._opt = ctypes.c_void_p()
                L.check(self._lib.glamr_opt_create(ctypes.byref(self._opt), self.smpl.handle, ctypes.byref(pb)), 'glamr_opt_create')
                self._opt_dims = dims
                self._setup_peers()
            else:                                   # bit 1: a new sequence re-uses the handle -> scratch back to its initial zeros
                flags = int(bool(reset_adam)) | (2 if self._fresh_attach else 0)
                L.check(self._lib.glamr_opt_set_problem(self._opt, ctypes.byref(pb), flags, L.stream_ptr()), 'glamr_opt_set_problem')
        self._fresh_attach = False

    def _backward(self, for_apply=False):
        """for_apply: glamr_opt_apply follows on this stream (the optimisation loop); the library then joins its side stream there, so the
        exchange below overlaps the tail of the pipelined blend"""
        fn = self._lib.glamr_opt_backward_for_apply if for_apply else self._lib.glamr_opt_backward
        L.check(fn(self._opt, L.ptr(self._theta), L.ptr(self._reduce), L.stream_ptr()), 'glamr_opt_backward')
        if self.world > 1:                                     # the one collective of the path: packed gradient + term sums
            if getattr(self, '_peer_ok', False):              # one-shot NVLink all-reduce of the library (no NCCL call)
                L.check(self._lib.glamr_allreduce_inplace(self._opt, L.ptr(self._reduce), self._reduce.numel(), L.stream_ptr()), 'glamr_allreduce_inplace')
            else:
                torch.distributed.all_reduce(self._reduce)

    def launches_per_iteration(self):
        """kernels of the CUDA library launched per optimiser iteration for the current stage (excludes the NCCL kernel)"""
        return int(self._lib.glamr_opt_launch_count(self._opt))

    def _read(self, what, *shape):
        p, n = ctypes.c_void_p(), ctypes.c_size_t()
        L.check(self._lib.glamr_opt_read(self._opt, what, ctypes.byref(p), ctypes.byref(n)), 'glamr_opt_read')
        return _device_view(p.value, n.value, self.device).view(*shape).clone()

    def _scatter_outputs(self, data):
        """copy what forward() stores into the data dict (each seed group's, for a list) in the reference (:421-528)"""
        comp = self._comp
        N, J = comp.N, comp.J
        ow, tw = self._read(L.R_ORIENT_WORLD, N, 3), self._read(L.R_TRANS_WORLD, N, 3)
        ob, tb = self._read(L.R_ORIENT_BASE, N, 3), self._read(L.R_TRANS_BASE, N, 3)
        kp = self._read(L.R_KP_PRED, N, J, 2)
        ociw, tciw = self._read(L.R_ORIENT_CIW, N, 3), self._read(L.R_TRANS_CIW, N, 3)
        tl = self._read(L.R_TRAJ_LOCAL, N, 11) if self.traj_source == L.TRAJ_PREDICTED else None
        jw = self._read(L.R_JOINTS_WORLD, N, J, 3)
        if self.world > 1:
            # per-frame-person outputs exist only on the rank that evaluated that frame-person: keep the own shard, sum over ranks
            own = torch.zeros(N, device=self.device)
            own[self._n_range[0]:self._n_range[1]] = 1.0
            packed = torch.cat([(x * own.view(N, *([1] * (x.dim() - 1)))).reshape(N, -1) for x in (kp, ociw, tciw, jw)], dim=1).contiguous()
            torch.distributed.all_reduce(packed)
            o = 0
            outs = []
            for x in (kp, ociw, tciw, jw):
                w = x[0].numel()
                outs.append(packed[:, o:o + w].reshape(x.shape))
                o += w
            kp, ociw, tciw, jw = outs
        datas = PB._groups(data)
        cam, cam_inv = self._read(L.R_CAM_POSE, sum(comp.Ts), 12), self._read(L.R_CAM_POSE_INV, sum(comp.Ts), 12)
        for g, dg in enumerate(datas):
            r, T = comp.c0s[g], comp.Ts[g]
            dg['cam_pose'] = G.from34(cam[r:r + T])
            dg['cam_pose_inv'] = G.from34(cam_inv[r:r + T])
            for q, d in enumerate(dg['person_data'].values()):
                p = comp.p0s[g] + q
                rows = slice(comp.n0s[g] + q * T, comp.n0s[g] + (q + 1) * T)
                ow_p, tw_p = ow[rows], tw[rows]
                d['smpl_orient_world'], d['root_trans_world'] = ow_p, tw_p
                d['smpl_orient_world_base'], d['root_trans_world_base'] = ob[rows], tb[rows]
                d['kp_2d_pred'] = kp[rows]
                d['smpl_orient_cam_in_world'], d['root_trans_cam_in_world'] = ociw[rows], tciw[rows]
                if self.traj_source == L.TRAJ_PREDICTED:           # without the codec the reference has no traj_local
                    d['traj_local'] = tl[rows][d['exist_frames']]
                d['joints_world'] = jw[rows]
                d['person_transform_world'] = G.make_transform(ow_p, tw_p, 'axis_angle')

    # ------------------------------------------------------------------------------------------------ reference API
    def forward(self, data, opt_variables, opt_meta):
        """:428-531 -- evaluates the current variables and refreshes the derived entries of `data`."""
        with torch.cuda.device(self.device):
            self._set_stage(data, opt_variables, getattr(self, '_loss_cfg', {}) or {}, opt_meta['stage'], reset_adam=False)
            self._backward()
            self._scatter_outputs(data)

    def compute_loss(self, data, loss_cfg):
        """:533-545 -> (total, weighted dict, unweighted dict) of 0-d CUDA tensors"""
        with torch.cuda.device(self.device):
            stage = getattr(self, '_cur_stage', 'opt')
            self._set_stage(data, getattr(self, '_cur_vars', []), loss_cfg, stage, reset_adam=False)
            self._backward()
            L.check(self._lib.glamr_opt_losses(self._opt, L.ptr(self._reduce), L.ptr(self._terms), L.stream_ptr()), 'glamr_opt_losses')
            terms = self._terms.clone()
        uw = {name: terms[L.TERM_INDEX[name]] for name in loss_cfg}
        wt = {name: uw[name] * loss_cfg[name]['weight'] for name in loss_cfg}
        return terms[NUM_TERMS], wt, uw

    def optimize_main(self, data, opt_variables, opt_lr, opt_niters, loss_cfg, opt_meta):
        """:547-570 -- opt_niters fused iterations (forward + residuals + backward [+ allreduce] + Adam).  `data` may be the
        groups attached by optimize_batch."""
        stage = opt_meta['stage']
        self._cur_vars, self._cur_stage, self._loss_cfg = opt_variables, stage, loss_cfg
        lib = self._lib
        datas = PB._groups(data)
        ng = len(datas)
        seq_names = [d['seq_name'] for d in datas]
        if ng > 1:
            seq_names = [f'{n} (seed group {g})' for g, n in enumerate(seq_names)]
        stride = ng * (NUM_TERMS + 1)                            # one row of loss terms per group and iteration
        with torch.cuda.device(self.device):
            self._set_stage(data, opt_variables, loss_cfg, stage, reset_adam=True, begin=True)
            hist = torch.zeros((max(opt_niters, 1), stride), device=self.device)
            stream = torch.cuda.current_stream()

            def one_iteration():
                self._backward(for_apply=True)
                L.check(lib.glamr_opt_apply(self._opt, L.ptr(self._theta), L.ptr(self._reduce), float(opt_lr), L.ptr(hist), stride,
                                            L.stream_ptr()), 'glamr_opt_apply')
            graph = None
            done = 0
            t_stage = time.time()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            # the library owns the loop when nothing has to happen between backward and apply: one GPU, or the reduction
            # fused into the Adam kernel over peer memory
            native = self.world == 1 or getattr(self, '_peer_ok', False)
            if native and opt_niters > 0:
                L.check(lib.glamr_opt_iterate(self._opt, L.ptr(self._theta), L.ptr(self._reduce), float(opt_lr), L.ptr(hist), stride,
                                              1, int(self.use_cuda_graph), L.stream_ptr()), 'glamr_opt_iterate')
                done = 1
            elif opt_niters > 0:
                one_iteration()                                  # warm-up (also sets kernel attributes) = iteration 0
                done = 1
                if self.use_cuda_graph and opt_niters > 2:
                    try:                                         # the NCCL all-reduce is capturable too
                        graph = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(graph):
                            one_iteration()
                    except Exception as e:                       # capture is an optimisation, eager launches are equivalent
                        graph = None
                        torch.cuda.synchronize()
                        if self.log is not None:
                            self.log.info(f'CUDA-graph capture with NCCL unavailable ({e}); running eager iterations')
            ev0.record()
            chunk = max(int(self.log_interval), 1)
            logging_on = self.log is not None or self.specs.get('print_logs', False)
            if native and not logging_on:
                chunk = max(opt_niters, 1)
            logged = 0
            while done < opt_niters:
                todo = min(chunk, opt_niters - done)
                if native:
                    L.check(lib.glamr_opt_iterate(self._opt, L.ptr(self._theta), L.ptr(self._reduce), float(opt_lr), L.ptr(hist), stride,
                                                  todo, int(self.use_cuda_graph), L.stream_ptr()), 'glamr_opt_iterate')
                else:
                    for _ in range(todo):
                        if graph is not None:
                            graph.replay()
                        else:
                            one_iteration()
                done += todo
                if logging_on:
                    logged = self._write_group_logs(hist, ng, logged, done, opt_niters, opt_lr, loss_cfg, stage, seq_names, t_stage)
            ev1.record()
            ev1.synchronize()
            if opt_niters > 1:
                self.iter_ms.append((stage, opt_niters - 1, ev0.elapsed_time(ev1) / (opt_niters - 1)))
            if self.log is not None or self.specs.get('print_logs', False):
                self._write_group_logs(hist, ng, logged, done, opt_niters, opt_lr, loss_cfg, stage, seq_names, t_stage)
            # [iterations, terms + total]; seed groups: [iterations, groups, terms + total]
            self.loss_history = hist if ng == 1 else hist.view(hist.shape[0], ng, NUM_TERMS + 1)
            self.cur_iter = max(opt_niters - 1, 0)
            if opt_niters > 0:
                self._scatter_outputs(data)                      # state of the last closure, like the reference
        return data

    def _write_group_logs(self, hist, ng, start, end, opt_niters, opt_lr, loss_cfg, stage, seq_names, t_stage):
        """_write_logs for each seed group's columns of the loss history"""
        for g in range(ng):
            rows = hist if ng == 1 else hist.view(hist.shape[0], ng, NUM_TERMS + 1)[:, g]
            self._write_logs(rows, start, end, opt_niters, opt_lr, loss_cfg, stage, seq_names[g], t_stage)
        return end

    def _write_logs(self, hist, start, end, opt_niters, opt_lr, loss_cfg, stage, seq_name, t_stage):
        """:646-659 same line format; values are read back in blocks of `log_interval` iterations."""
        if end <= start:
            return end
        vals = hist[start:end].cpu().numpy()
        per_iter = (time.time() - t_stage) / max(end, 1)
        for k, it in enumerate(range(start, end)):
            loss_str = ' | '.join(f'{name}: {vals[k, L.TERM_INDEX[name]]:7.3f}' for name in loss_cfg)
            eta = _sec_to_time(per_iter * (opt_niters - it - 1))
            info = f'{self.cfg.id} - {seq_name} - {stage} | {it:4d}/{opt_niters} | TE: {_sec_to_time(per_iter)} ETA: {eta} | LR: {opt_lr:.0e} | {loss_str}'
            if self.log is None:
                print(info)
            else:
                self.log.info(info)
        return end

    def optimize(self, in_dict, continue_opt=False):
        """:572-589"""
        t0 = time.perf_counter()
        if continue_opt:
            data = tensor_to(in_dict, self.device)
            self._attach(data)
        else:
            data = self.init_data(in_dict)
        t1 = time.perf_counter()
        for stage, stage_specs in self.opt_stage_specs.items():
            opt_meta = {'stage': stage, 'opt_latent_start_iter': stage_specs.get('opt_latent_start_iter', 0)}
            self.optimize_main(data, stage_specs['opt_variables'], stage_specs['opt_lr'], stage_specs['opt_niters'],
                               stage_specs['loss_cfg'], opt_meta)
            if stage_specs.get('reinitialize_cam', False):
                data['cam_pose'][:] = data['cam_pose'][[0]]
                data['cam_pose_inv'] = G.inverse_transform(data['cam_pose'])
        t2 = time.perf_counter()
        out = tensor_to_numpy(data)
        # host wall-clock of the three phases of the last call (init_data includes the learned prior; stages include the waits)
        self.phase_seconds = {'init_data': t1 - t0, 'stages': t2 - t1, 'to_numpy': time.perf_counter() - t2}
        return out

    def optimize_seeds(self, in_dict, seeds):
        """Optimise several seeds of one sequence as one problem: ``optimize_batch([in_dict], seeds)[0]``.  Element k of the result
        is what ``np.random.seed(s); torch.manual_seed(s); optimize(copy.deepcopy(in_dict))`` returns for s = seeds[k], bit for bit.
        ``self.seed_loss_histories[k]`` is seed k's loss history of the last stage (``loss_history`` of its serial run)."""
        if self.world > 1:
            raise ValueError('optimize_seeds runs on one GPU: shard sequences over ranks and batch the seeds on each rank')
        if not list(seeds):
            return []
        outs = self.optimize_batch([in_dict], seeds)[0]
        self.seed_loss_histories = self.batch_loss_histories[0]
        return outs

    def optimize_batch(self, in_dicts, seeds):
        """Optimise every (sequence, seed) pair of `in_dicts` x `seeds` as one group of one problem.  The sequences share this
        optimiser's config and may differ in frames, persons, exist ranges and visibility.  ``outs[i][k]`` is what
        ``np.random.seed(s); torch.manual_seed(s); optimize(copy.deepcopy(in_dicts[i]))`` returns for s = seeds[k], bit for bit:
        every pair's init_data runs as in the serial path after setting the RNGs the same way, with the learned prior of all pairs
        in one ragged call when the prior supports it (_init_groups), then the data dicts are attached as the groups of one problem (glamr_b200/problem.py) and the stages run once for all of them.
        Each group's camera, terms and gradient are reduced exactly as in its own one-group problem, from its own normalisers.
        ``self.batch_loss_histories[i][k]`` is that pair's loss history of the last stage.  Scratch grows with the frame-persons of
        all groups (sum of persons x frames).  No continue_opt; one GPU only (run_dataset shards sequences over ranks)."""
        if self.world > 1:
            raise ValueError('optimize_batch runs on one GPU: shard sequences over ranks and batch them on each rank')
        seeds = [int(s) for s in seeds]
        in_dicts = list(in_dicts)
        if not seeds or not in_dicts:
            return [[] for _ in in_dicts]
        t0 = time.perf_counter()
        batch = self._init_groups(in_dicts, seeds)
        t1 = time.perf_counter()
        self._optimize_groups(batch)
        t2 = time.perf_counter()
        outs = [[tensor_to_numpy(data) for data in seq] for seq in batch]
        self.phase_seconds = {'init_data': t1 - t0, 'stages': t2 - t1, 'to_numpy': time.perf_counter() - t2}
        return outs

    def _init_groups(self, in_dicts, seeds):
        """init_data of every (sequence, seed) pair with the RNGs set as run_dataset sets them -> [[data dict]].  With a prior that
        takes ragged batches, init_data is split at the prior: each pair runs up to it, draws its eps as its serial prior call would
        and keeps its RNG states; one ragged prior call then serves every person of every pair (rows in the classes of their serial
        calls: a block of P for P equal-length persons, one row per person otherwise); and each pair finishes from its RNG states."""
        ragged = self.flag_infer_motion_traj and getattr(self.mt_model, 'supports_ragged_batch', False)
        heads = []
        for in_dict in in_dicts:
            for s in seeds:
                np.random.seed(s)
                torch.manual_seed(s)
                if not ragged:
                    heads.append(self.init_data(copy.deepcopy(in_dict)))
                    continue
                st = self._init_data_head(copy.deepcopy(in_dict))
                st['ds'], st['row_batch'] = self._prior_rows(st['persons'])
                st['latents'] = self.mt_model.draw_ragged_latents([int(d['exist_len']) for d in st['ds']], st['row_batch'])
                st['rng'] = (np.random.get_state(), torch.get_rng_state(), torch.cuda.get_rng_state(self.device))
                heads.append(st)
        if ragged:
            self._ragged_prior([d for st in heads for d in st['ds']], [r for st in heads for r in st['row_batch']],
                               _cat_latents([st['latents'] for st in heads]))
            datas = []
            for st in heads:
                np.random.set_state(st['rng'][0])
                torch.set_rng_state(st['rng'][1])
                torch.cuda.set_rng_state(st['rng'][2], self.device)
                datas.append(self._init_data_tail(st))
            heads = datas
        S = len(seeds)
        return [heads[i * S:(i + 1) * S] for i in range(len(in_dicts))]

    def _optimize_groups(self, batch):
        """the stages of optimize for the groups of `batch` ([[data dict]] from _init_groups) as one problem; each pair's loss history
        of the last stage goes to batch_loss_histories"""
        datas = [d for seq in batch for d in seq]
        groups = batch[0] if len(batch) == 1 else batch        # one sequence: its seed groups, with the layout they always had
        self._attach(groups)
        for stage, stage_specs in self.opt_stage_specs.items():
            opt_meta = {'stage': stage, 'opt_latent_start_iter': stage_specs.get('opt_latent_start_iter', 0)}
            self.optimize_main(groups, stage_specs['opt_variables'], stage_specs['opt_lr'], stage_specs['opt_niters'],
                               stage_specs['loss_cfg'], opt_meta)
            if stage_specs.get('reinitialize_cam', False):
                for data in datas:
                    data['cam_pose'][:] = data['cam_pose'][[0]]
                    data['cam_pose_inv'] = G.inverse_transform(data['cam_pose'])
        lh, S = self.loss_history, len(batch[0])
        hists = [lh] if len(datas) == 1 else [lh[:, g] for g in range(len(datas))]
        self.batch_loss_histories = [hists[i * S:(i + 1) * S] for i in range(len(batch))]


def _cat_latents(parts):
    """the latents of several ragged prior calls (MotionTrajJointModel.draw_ragged_latents) as those of one call on all their rows"""
    out = {}
    for k, dim in (('in_motion_latent', 0), ('in_traj_latent', 0), ('in_traj_window_latent', 1)):
        xs = [p[k] for p in parts if k in p]
        if not xs:
            continue
        if k != 'in_traj_latent':
            n = max(x.shape[1 - dim] for x in xs)
            xs = [torch.nn.functional.pad(x, (0, 0, 0, n - x.shape[1])) if dim == 0 else
                  torch.nn.functional.pad(x, (0, 0, 0, 0, 0, n - x.shape[0])) for x in xs]
        out[k] = torch.cat(xs, dim=dim)
    return out


def _exist_range(d):
    """the exist frames of a person dict as a slice: they run from the first to the last visible frame"""
    return slice(int(d['fr_start']), int(d['fr_end']))


def _device_view(addr, count, device):
    """float32 tensor aliasing `count` floats of device memory at `addr` (owned by a CUDA-library handle)."""
    class _Holder:
        pass
    h = _Holder()
    h.__cuda_array_interface__ = {'shape': (count,), 'typestr': '<f4', 'data': (addr, False), 'version': 2}
    return torch.as_tensor(h, device=device)
