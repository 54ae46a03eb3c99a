"""Learned motion / trajectory prior on the CUDA library -- drop-in for the inference surface of the reference's
``MotionTrajJointModel`` (motion_infiller/models/motion_traj_joint_model.py:17-145): ``inference(batch, sample_num)``,
``get_motion_latent``, ``get_traj_latent``.

The networks run in ``glamr_infiller_forward`` (the autoregressive sweep of 50-frame windows of
MotionInfillerVAE.inference_multi_step, motion_infiller_vae.py:618-632, batched over ALL sequences instead of the
reference's batch of one) and ``glamr_trajpred_forward`` / ``glamr_trajpred_windows_forward`` (single pass / every window of
multi_step_trajpred in one batch; glamr_b200/csrc/nets_kernels.cu); this module runs SMPL FK for the joint-position features and reshapes the outputs into the reference's
dict layout.  Weights come from the reference's Lightning checkpoints (state_dict names are kept) or from an explicit
state dict; there is no CPU fallback.
"""
import ctypes
import glob
import os

import numpy as np
import torch

from . import lib as L

PAST, CUR, FUT, NZ = 10, 30, 10, 128
TRAJ_WINDOW = 100        # seq_len of traj_pred/cfg/traj_pred_demo.yml: the window of multi-step trajectory prediction
PRIOR_GRAPH_DEFAULT = '0'
SKINNY_MAX_M = 256       # nets_kernels.cu kSkinnyMaxM: Linears of at most this many rows run the exact FP32 skinny GEMM
WINDOW = PAST + CUR + FUT


def _declare(lib):
    if getattr(lib, '_nets_declared', False):
        return
    lib.glamr_infiller_workspace_floats.restype = ctypes.c_size_t
    lib.glamr_infiller_sequence_workspace_floats.restype = ctypes.c_size_t
    lib.glamr_infiller_forward.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                                                                                     ctypes.c_void_p]
    lib.glamr_infiller_recon_workspace_floats.restype = ctypes.c_size_t
    lib.glamr_infiller_recon_workspace_floats.argtypes = [ctypes.c_int]
    lib.glamr_infiller_recon_forward.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 4 + [ctypes.c_size_t, ctypes.c_void_p]
    lib.glamr_trajpred_workspace_floats.restype = ctypes.c_size_t
    lib.glamr_net_set_tensor.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_size_t]
    lib.glamr_infiller_window_forward.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_void_p,
                                                                                                             ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.glamr_trajpred_forward.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + \
        [ctypes.c_void_p] * 6 + [ctypes.c_size_t, ctypes.c_void_p]
    lib.glamr_trajpred_windows_workspace_floats.restype = ctypes.c_size_t
    lib.glamr_trajpred_windows_workspace_floats.argtypes = [ctypes.c_int] * 3
    lib.glamr_trajpred_windows_forward.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 6 + [ctypes.c_size_t, ctypes.c_void_p]
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    lib.glamr_infiller_ragged_workspace_floats.restype = sz
    lib.glamr_infiller_ragged_workspace_floats.argtypes = [ctypes.c_int]
    lib.glamr_infiller_forward_ragged.argtypes = [vp, ctypes.c_int] + [vp] * 6 + [ctypes.c_int, vp, sz, vp]
    lib.glamr_trajpred_ragged_workspace_floats.restype = sz
    lib.glamr_trajpred_ragged_workspace_floats.argtypes = [ctypes.c_int, vp]
    lib.glamr_trajpred_forward_ragged.argtypes = [vp, ctypes.c_int] + [vp] * 11 + [sz, vp]
    lib.glamr_trajpred_windows_ragged_workspace_floats.restype = sz
    lib.glamr_trajpred_windows_ragged_workspace_floats.argtypes = [ctypes.c_int, vp, ctypes.c_int]
    lib.glamr_trajpred_windows_forward_ragged.argtypes = [vp, ctypes.c_int, ctypes.c_int] + [vp] * 10 + [sz, vp]
    lib._nets_declared = True


def _np_ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _infiller_class(rb):
    """which of the infiller's Linears (50, 30, 2 and 1 rows per track) a call of rb tracks runs above the skinny-GEMM limit"""
    return sum(s * rb > SKINNY_MAX_M for s in (50, 30, 2, 1))


def ragged_plan(seq_len, row_batch=None, sample_num=1, traj_window=TRAJ_WINDOW, multi_step_traj=False):
    """Host plan of a ragged prior call (MotionTrajJointModel.inference with `seq_len`).

    Input row b is a track of seq_len[b] frames; row_batch[b] is the batch size of the single-track call it reproduces: runs of
    row_batch[b] consecutive rows of equal length are one block, the persons of one equal-length call.  Each row becomes
    `sample_num` expanded rows e = b * sample_num + s, which reproduce a call of row_batch[b] * sample_num tracks.  The library
    needs the rows ordered by the kernels their Linears run (include/glamr_b200.h): `inf_order` / `pred_order` are the expanded
    rows in the infiller's and the predictor's order, `inf_off` / `pred_off` the packed frame offsets in that order and
    `pred_woff` the window offsets of the windowed predictor."""
    lens = [int(t) for t in seq_len]
    B, S = len(lens), int(sample_num)
    rb = [1] * B if row_batch is None else [int(r) for r in row_batch]
    if len(rb) != B or B == 0 or S < 1:
        raise ValueError(f'seq_len and row_batch need one entry per row, got {B} and {len(rb)}')
    blocks, b = [], 0
    while b < B:
        P = rb[b]
        if P < 1 or b + P > B or any(rb[q] != P or lens[q] != lens[b] for q in range(b, b + P)):
            raise ValueError(f'rows {b}..{b + P - 1}: row_batch {P} must name a block of {P} consecutive rows of equal length')
        blocks.append((b, P))
        b += P
    short = [t for t in lens if t <= PAST]
    if short:
        # the error type the single-track call raises for such a track (its library call refuses it)
        raise L.GlamrError(f'ragged_plan: tracks of {short} frames have no infiller window (the infiller needs more than {PAST} frames)')
    E = B * S
    lens_e = np.repeat(np.asarray(lens, dtype=np.int32), S)
    rb_e = np.repeat(np.asarray(rb, dtype=np.int32) * S, S)
    nwin_e = -(-(lens_e - PAST) // CUR)
    C_e = -(-lens_e // int(traj_window))
    inf_order = np.array(sorted(range(E), key=lambda e: (_infiller_class(int(rb_e[e])), -int(lens_e[e]), e)), dtype=np.int64)

    def pred_class(e):
        f, r = (int(C_e[e]) * int(traj_window), int(C_e[e])) if multi_step_traj else (int(lens_e[e]), 1)
        return (f * int(rb_e[e]) > SKINNY_MAX_M) + (r * int(rb_e[e]) > SKINNY_MAX_M)
    pred_order = np.array(sorted(range(E), key=lambda e: (pred_class(e), e)), dtype=np.int64)
    off = lambda order, n: np.concatenate([[0], np.cumsum(n[order])]).astype(np.int32)
    return {'B': B, 'S': S, 'E': E, 'blocks': blocks, 'lens': lens_e, 'row_batch': rb_e, 'nwin': nwin_e, 'C': C_e,
            'inf_order': inf_order, 'pred_order': pred_order, 'inf_off': off(inf_order, lens_e), 'pred_off': off(pred_order, lens_e),
            'pred_woff': off(pred_order, C_e), 'multi_step_traj': bool(multi_step_traj), 'traj_window': int(traj_window)}


def draw_ragged_eps(plan, device, infiller=True, traj=True):
    """The prior's eps for the expanded rows of `plan`, drawn as the serial calls draw them: for each block in row order, the
    infiller's randn((windows, P * S, 128)) and then the predictor's randn((P * S, 128)) (single pass) or
    randn((windows, P * S, 128)) (windowed); `infiller` / `traj` False: that network's eps are given and not drawn (None).
    -> (infiller eps [E, max windows, 128], predictor eps per expanded row: [E, 128] or a list of [C_e, 128])"""
    S = plan['S']
    inf = torch.zeros((plan['E'], int(plan['nwin'].max()), NZ), device=device) if infiller else None
    rows = [None] * plan['E']
    for b0, P in plan['blocks']:
        e0, n = b0 * S, P * S
        nwin, C = int(plan['nwin'][e0]), int(plan['C'][e0])
        if infiller:
            inf[e0:e0 + n, :nwin] = torch.randn((nwin, n, NZ), device=device).transpose(0, 1)
        if traj and plan['multi_step_traj']:
            rows[e0:e0 + n] = list(torch.randn((C, n, NZ), device=device).transpose(0, 1))
        elif traj:
            rows[e0:e0 + n] = list(torch.randn((n, NZ), device=device))
    if not traj:
        return inf, None
    return inf, (rows if plan['multi_step_traj'] else torch.stack(rows))


class _GraphCache:
    """Replays a fixed launch sequence as ONE CUDA graph.  The prior networks are launch-latency bound (about 70 small kernels
    per 50-frame window, 10 windows for a 300-frame track): `run(key, fn, inputs)` copies `inputs` into static device
    buffers, replays the graph captured for `key` (same shapes -> same launches) and returns clones of the static outputs.
    The first call for a key runs `fn` eagerly (lazy initialisation must happen outside capture) and then captures it; if
    capture is refused the key stays on the eager path."""

    def __init__(self, enabled=None, max_entries=8):
        if enabled is None:          # GLAMR_PRIOR_GRAPH=1|0
            enabled = os.environ.get('GLAMR_PRIOR_GRAPH', PRIOR_GRAPH_DEFAULT) == '1'
        self.enabled, self.max_entries, self.entries = enabled, max_entries, {}

    def run(self, key, fn, inputs):
        if not self.enabled:
            return fn(*inputs)
        ent = self.entries.get(key)
        if ent is None:
            if len(self.entries) >= self.max_entries:
                self.entries.pop(next(iter(self.entries)))
            static_in = [None if x is None else x.clone() for x in inputs]
            out = fn(*static_in)                                   # eager warm-up; also the result of this first call
            ent = {'in': static_in, 'graph': None, 'out': None}
            self.entries[key] = ent
            try:
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    ent['out'] = fn(*static_in)
                ent['graph'] = g
            except Exception:
                ent['graph'], ent['out'] = None, None
                torch.cuda.synchronize()
            return out
        if ent['graph'] is None:
            return fn(*inputs)
        for dst, src in zip(ent['in'], inputs):
            if dst is not None:
                dst.copy_(src)
        ent['graph'].replay()
        return tuple(o.clone() for o in ent['out']) if isinstance(ent['out'], tuple) else ent['out'].clone()


class _Net:
    """opaque glamr_net_t with the parameters of one network"""

    def __init__(self, state, device):
        self.device = L.require_cuda(device)
        self.lib = L.load()
        _declare(self.lib)
        self.h = ctypes.c_void_p()
        L.check(self.lib.glamr_net_create(ctypes.byref(self.h)), 'glamr_net_create')
        self.names = set()
        with torch.cuda.device(self.device):
            for name, val in state.items():
                arr = np.ascontiguousarray(val.detach().cpu().numpy() if isinstance(val, torch.Tensor) else np.asarray(val), dtype=np.float32)
                if arr.size == 0 or arr.dtype != np.float32:
                    continue
                L.check(self.lib.glamr_net_set_tensor(self.h, name.encode(), arr.ctypes.data_as(ctypes.c_void_p), arr.size), f'set_tensor {name}')
                self.names.add(name)
        self._ws = None

    def workspace(self, floats):
        if self._ws is None or self._ws.numel() < floats:
            if self._ws is not None:                 # captured graphs may hold the old address: retire, do not free
                self._retired = getattr(self, '_retired', []) + [self._ws]
            self._ws = torch.empty(int(floats), dtype=torch.float32, device=self.device)
        return self._ws

    def __del__(self):
        try:
            self.lib.glamr_net_destroy(self.h)
        except Exception:
            pass


class MotionInfillerVAE:
    """inference surface of motion_infiller/models/motion_infiller_vae.py:440-667 (pose_rep 'body', axis-angle)"""
    model_type = 'angle'

    def __init__(self, state, device):
        self.net = _Net(state, device)
        self.device = self.net.device
        self.nz, self.past_nframe, self.cur_nframe, self.fut_nframe = NZ, PAST, CUR, FUT
        self.graphs = _GraphCache()

    def get_latent(self, seq_len):
        return torch.randn((int(np.ceil((seq_len - PAST) / CUR)), NZ))

    def inference(self, batch, sample_num=1, recon=False, multi_step=True):
        """multi-step inference (:643-652): `sample_num` infer sweeps, then with `recon` one reconstruction sweep.

        `pose` [B,T,72] (with `pose_mask` [B,T,72]) is the ground truth: the infer outputs carry its root orientation, the input body
        pose defaults to (pose * pose_mask)[..., 3:] when `in_body_pose` is not given, and `recon` encodes it with the posterior
        (z = the posterior mean) into `recon_out_pose` [B,T,72] / `recon_out_body_pose` [B,T,69].  Both sweeps start from the input
        body pose; the caller's tensors are never written."""
        if not multi_step:
            raise NotImplementedError('only the multi-step path (multi_step=True) is implemented on CUDA')
        gt = batch.get('pose')
        if gt is not None and batch.get('pose_mask') is None:
            raise ValueError('`pose` needs `pose_mask` (the input body pose is (pose * pose_mask)[..., 3:])')
        if recon:
            if gt is None:
                raise ValueError('recon=True needs the ground-truth `pose` [B, T, 72] that the posterior encodes')
            if batch.get('seq_len') is not None:
                raise NotImplementedError('recon=True is not implemented for tracks of different lengths (`seq_len`)')
            if not any(k.startswith('data_encoder.') for k in self.net.names):
                raise ValueError('recon=True needs the posterior encoder weights (data_encoder.*), which this net does not have')
        dev = self.device
        if gt is not None:
            gt = gt.to(dev, torch.float32)
        if batch.get('in_body_pose') is not None:
            pose_in = batch['in_body_pose'].to(dev, torch.float32).contiguous()
        elif gt is not None:
            pose_in = (gt * batch['pose_mask'].to(dev, torch.float32))[..., 3:].contiguous()
        else:
            raise KeyError('in_body_pose')
        frame_mask = batch['frame_mask'].to(dev, torch.float32).contiguous()
        latent = batch.get('in_motion_latent')
        latent = None if latent is None else latent.to(dev, torch.float32).contiguous()
        B0, T = pose_in.shape[:2]
        self.net.workspace(self.net.lib.glamr_infiller_sequence_workspace_floats(B0 * sample_num))        # sized before any capture
        key = ('infill', B0, T, sample_num, None if latent is None else tuple(latent.shape))
        with torch.cuda.device(dev):
            body = self.graphs.run(key, lambda a, b, c: self._windows(a, b, c, sample_num), (pose_in, frame_mask, latent))
        data = dict(batch)
        data['infer_out_body_pose'] = body
        root = torch.zeros_like(body[..., :3]) if gt is None else gt[:, None, :, :3].expand(-1, sample_num, -1, -1)
        data['infer_out_pose'] = torch.cat([root, body], dim=-1)
        data['batch_size'], data['seq_len'] = B0, T
        if recon:
            gt_body = gt[..., 3:].contiguous()
            self.net.workspace(self.net.lib.glamr_infiller_recon_workspace_floats(B0))
            with torch.cuda.device(dev):
                rbody = self.graphs.run(('recon', B0, T), self._recon_windows, (pose_in, gt_body, frame_mask))
            data['recon_out_body_pose'] = rbody
            data['recon_out_pose'] = torch.cat([gt[..., :3], rbody], dim=-1)
        return data

    def _recon_windows(self, pose_in, gt_body, frame_mask):
        """the reconstruction sweep (inference_multi_step with recon=True): one library call, [B, T, 69] out"""
        B, T = pose_in.shape[:2]
        pose = pose_in.transpose(0, 1).contiguous().clone()                                       # [T,B,69], overwritten in place
        gt_tb = gt_body.transpose(0, 1).contiguous()
        key_pad_all = (~(frame_mask == 1)).to(torch.uint8).contiguous()                           # [B,T]
        lib = self.net.lib
        ws = self.net.workspace(lib.glamr_infiller_recon_workspace_floats(B))
        L.check(lib.glamr_infiller_recon_forward(self.net.h, T, B, pose.data_ptr(), gt_tb.data_ptr(), key_pad_all.data_ptr(), ws.data_ptr(),
                                                 ws.numel(), torch.cuda.current_stream().cuda_stream), 'glamr_infiller_recon_forward')
        return pose.transpose(0, 1).contiguous()

    def _windows(self, pose_in, frame_mask, latent, sample_num):
        """motion_infiller_vae.py:618-632: autoregressive 50-frame windows, stride 30 -- one library call for the whole sweep
        (device tensors in, [B0, S, T, 69] out; no host sync)"""
        dev = self.device
        B0, T = pose_in.shape[:2]
        B = B0 * sample_num
        pose = pose_in.repeat_interleave(sample_num, dim=0).transpose(0, 1).contiguous().clone()       # [T,B,69], overwritten in place
        key_pad_all = (~(frame_mask == 1)).repeat_interleave(sample_num, dim=0).to(torch.uint8).contiguous()      # [B,T]
        nwin = int(np.ceil((T - PAST) / CUR))
        if latent is not None and latent.dim() == 3:                 # [B0, windows, nz]: one latent per sequence and window
            eps, rows = latent[:, :nwin].repeat_interleave(sample_num, dim=0).transpose(0, 1).contiguous(), B
        elif latent is not None:                                     # [windows, nz]: shared by the batch
            eps, rows = latent[:nwin].contiguous(), 1
        else:
            eps, rows = torch.randn((nwin, B, NZ), device=dev), B
        if eps.shape[0] < nwin:
            raise ValueError(f'{nwin} windows need {nwin} latents, got {eps.shape[0]}')
        lib = self.net.lib
        ws = self.net.workspace(lib.glamr_infiller_sequence_workspace_floats(B))
        L.check(lib.glamr_infiller_forward(self.net.h, T, B, pose.data_ptr(), key_pad_all.data_ptr(), eps.data_ptr(), rows, ws.data_ptr(), ws.numel(),
                                           torch.cuda.current_stream().cuda_stream), 'glamr_infiller_forward')
        return pose.transpose(0, 1).reshape(B0, sample_num, T, 69).contiguous()


class TrajPredVAE:
    """inference surface of traj_pred/models/traj_pred_vae.py:341-548 (6d local orientation, joint-position input).
    seq_len: the window of multi-step inference (the predictor config's seq_len)."""
    model_type = 'joint'
    in_joint_pos_only = False

    def __init__(self, state, device, smpl, seq_len=TRAJ_WINDOW):
        self.net = _Net(state, device)
        self.device, self.smpl, self.nz = self.net.device, smpl, NZ
        self.seq_len = int(seq_len)
        self.graphs = _GraphCache()

    def get_latent(self, seq_len):
        return torch.zeros((1, NZ))

    def get_joint_pos(self, body_pose):
        """:384-394  23 FK joints (root removed), zero orientation, rest joints from v_template"""
        flat = body_pose.reshape(-1, 69).to(self.device, torch.float32).contiguous()
        z3 = torch.zeros((flat.shape[0], 3), device=self.device)
        joints = self.smpl.get_joints(global_orient=z3, body_pose=flat, root_trans=z3)
        return joints[:, 1:, :].reshape(body_pose.shape[:-1] + (69,))

    def num_windows(self, seq_len):
        return -(-int(seq_len) // self.seq_len)

    def inference(self, batch, sample_num=1, recon=False, recon_only=False, multi_step=False):
        """Single pass (multi_step False): one network pass over the whole track; `in_traj_latent` [1 or B,128], `init_xy`
        [B,2] and `init_heading` [B] are used when given.

        Multi-step (traj_pred_vae.py:484-520): the track is cut into ceil(T / seq_len) windows, the last one zero-padded, each
        window draws its own z and the windows are stitched with the heading hand-over of the reference.  As in the
        reference, `in_traj_latent`, `init_xy` and `init_heading` do not reach the windows and are ignored.  The windows' eps
        come from `in_traj_window_latent` [windows, B, 128] when given, else from torch.randn on the device."""
        if recon or recon_only or sample_num != 1:
            raise NotImplementedError('only sampling with sample_num=1 is implemented on CUDA (no reconstruction mode)')
        dev = self.device
        body = batch['in_body_pose'].to(dev, torch.float32).contiguous()           # [B,T,69]
        B, T = body.shape[:2]
        dv = lambda k: batch[k].to(dev, torch.float32).contiguous() if k in batch and batch[k] is not None else None
        self.smpl._workspace(B * T, fk_only=True)
        if multi_step:
            wlat = dv('in_traj_window_latent')
            C = self.num_windows(T)
            if wlat is not None and tuple(wlat.shape) != (C, B, NZ):
                raise ValueError(f'in_traj_window_latent: {C} windows of {B} sequences need shape {(C, B, NZ)}, got {tuple(wlat.shape)}')
            self.net.workspace(self.net.lib.glamr_trajpred_windows_workspace_floats(T, B, self.seq_len))
            key = ('traj_windows', self.seq_len, B, T, wlat is not None)
            with torch.cuda.device(dev):
                local, trans, orient = self.graphs.run(key, self._forward_windows, (body, wlat))
        else:
            latent, ixy, ih = dv('in_traj_latent'), dv('init_xy'), dv('init_heading')
            self.net.workspace(self.net.lib.glamr_trajpred_workspace_floats(T, B))
            key = ('traj', B, T, None if latent is None else tuple(latent.shape), ixy is not None, ih is not None)
            with torch.cuda.device(dev):
                local, trans, orient = self.graphs.run(key, self._forward, (body, latent, ixy, ih))
        out = {'infer_out_local_traj_tp': local.view(T, B, 1, 11), 'infer_out_trans_tp': trans.view(T, B, 1, 3),
               'infer_out_orient_tp': orient.view(T, B, 1, 3)}
        out['infer_out_orient'] = out['infer_out_orient_tp'].permute(1, 2, 0, 3).contiguous()
        out['infer_out_trans'] = out['infer_out_trans_tp'].permute(1, 2, 0, 3).contiguous()
        out['infer_out_pose'] = torch.cat([out['infer_out_orient'], body.unsqueeze(1)], dim=-1)
        return out

    def _forward(self, body, latent, ixy, ih):
        """joint-position features (SMPL FK) + the network, device tensors only"""
        dev = self.device
        B, T = body.shape[:2]
        jp = self.get_joint_pos(body).transpose(0, 1).contiguous()                # [T,B,69]
        lib = self.net.lib
        ws = self.net.workspace(lib.glamr_trajpred_workspace_floats(T, B))
        local = torch.empty((T, B, 11), dtype=torch.float32, device=dev)
        trans = torch.empty((T, B, 3), dtype=torch.float32, device=dev)
        orient = torch.empty((T, B, 3), dtype=torch.float32, device=dev)
        if latent is not None:
            eps, rows = latent, (1 if latent.shape[0] == 1 else B)
        else:
            eps, rows = torch.randn((B, NZ), device=dev), B
        L.check(lib.glamr_trajpred_forward(self.net.h, T, B, jp.data_ptr(), eps.data_ptr(), rows, None if ixy is None else ixy.data_ptr(),
                                           None if ih is None else ih.data_ptr(), local.data_ptr(), trans.data_ptr(), orient.data_ptr(),
                                           ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream), 'glamr_trajpred_forward')
        return local, trans, orient

    def _forward_windows(self, body, wlat):
        """joint-position features (SMPL FK on the whole track) + every window of every sequence in one library call"""
        dev = self.device
        B, T = body.shape[:2]
        jp = self.get_joint_pos(body).transpose(0, 1).contiguous()                # [T,B,69]
        lib = self.net.lib
        ws = self.net.workspace(lib.glamr_trajpred_windows_workspace_floats(T, B, self.seq_len))
        local = torch.empty((T, B, 11), dtype=torch.float32, device=dev)
        trans = torch.empty((T, B, 3), dtype=torch.float32, device=dev)
        orient = torch.empty((T, B, 3), dtype=torch.float32, device=dev)
        eps = wlat if wlat is not None else torch.randn((self.num_windows(T), B, NZ), device=dev)
        L.check(lib.glamr_trajpred_windows_forward(self.net.h, T, B, self.seq_len, jp.data_ptr(), eps.data_ptr(), local.data_ptr(),
                                                   trans.data_ptr(), orient.data_ptr(), ws.data_ptr(), ws.numel(),
                                                   torch.cuda.current_stream().cuda_stream), 'glamr_trajpred_windows_forward')
        return local, trans, orient


def load_lightning_state_dict(path):
    """state_dict of a PyTorch-Lightning ``.ckpt`` (lib/utils/tools.py:94-104 -> ``load_from_checkpoint``) as plain float32
    numpy arrays.  Lightning checkpoints pickle hyper-parameter objects next to the tensors; tensors-only loading
    (``weights_only=True``) is tried first so that nothing but tensors is unpickled, the permissive path is the fall-back
    for files that need it."""
    try:
        ck = torch.load(path, map_location='cpu', weights_only=True)
    except Exception:
        ck = torch.load(path, map_location='cpu', weights_only=False)
    sd = ck.get('state_dict', ck)
    return {k: (v.detach().float().numpy() if isinstance(v, torch.Tensor) else v) for k, v in sd.items()}


def _find_checkpoint(cfg_dir, cp='best', version=None):
    """lib/utils/tools.py:41-45 (find_last_version) + :94-104 (get_checkpoint_path): 'best' = the LAST of the sorted
    *best*.ckpt names, 'last' = last.ckpt, an integer = model-epoch=NNNN.ckpt"""
    if version is None:
        numbers = sorted(int(os.path.basename(p)[len('version_'):]) for p in glob.glob(os.path.join(cfg_dir, 'version_*')))
        if not numbers:
            raise FileNotFoundError(f'no checkpoint versions under {cfg_dir}')
        version = numbers[-1]
    ck_dir = os.path.join(cfg_dir, f'version_{version}', 'checkpoints')
    if cp == 'last':
        return os.path.join(ck_dir, 'last.ckpt')
    if cp == 'best':
        files = sorted(glob.glob(os.path.join(ck_dir, '*best*.ckpt')))
        if not files:
            raise FileNotFoundError(f'no *best*.ckpt under {ck_dir}')
        return files[-1]
    return os.path.join(ck_dir, f'model-epoch={int(cp):04d}.ckpt')


# motion_infiller/cfg_infer/joint_motion_traj_demo.yml (the only joint config the reference ships)
_JOINT_DEMO_YML = {
    'results_root_dir': 'results/motion_filler_infer', 'seed': 1,
    'model_specs': {'mfiller_cfg': 'motion_infiller_demo', 'mfiller_cp': 'best', 'trajpred_cfg': 'traj_pred_demo', 'trajpred_cp': 'best'},
    'amass_dir': 'datasets/amass_processed/v1', 'seq_len': 300, 'seq_sampling_method': 'length',
    'data_mask_methods': {'drop_frames': {'preserve_first_n': 10, 'min_drop_len': 5, 'max_drop_len': 200}},
    'num_motion_samp': 3, 'multi_step_mfiller': True, 'multi_step_trajpred': False,
}
_RESULTS_ROOT = {'motion_infiller': 'results/motion_filler', 'traj_pred': 'results/traj_pred'}   # results_root_dir of the two shipped network configs


class MTConfig:
    """motion_infiller/utils/config_motion_traj.py:7-45: the joint model's YAML (cwd-relative glob like the reference; the
    shipped joint_motion_traj_demo.yml is built in) and the checkpoint directories of the two networks it names
    (motion_infiller/utils/config.py:16-26, traj_pred/utils/config.py:16-26).  `trajpred_seq_len` is the window of multi-step
    trajectory prediction: the `seq_len` of the predictor's config (traj_pred/cfg/**/<trajpred_cfg>.yml), TRAJ_WINDOW when the
    file is not found or does not set it."""

    def __init__(self, cfg_id):
        import yaml
        self.id = cfg_id
        files = glob.glob(f'motion_infiller/cfg_infer/**/{cfg_id}.yml', recursive=True)
        if len(files) == 1:
            self.yml_dict = yaml.safe_load(open(files[0]))
        elif cfg_id == 'joint_motion_traj_demo':
            self.yml_dict = {k: (dict(v) if isinstance(v, dict) else v) for k, v in _JOINT_DEMO_YML.items()}
        else:
            raise FileNotFoundError(f'motion_infiller/cfg_infer/**/{cfg_id}.yml not found')
        y = self.yml_dict
        self.model_specs = y.get('model_specs', {})
        self.seed = y.get('seed', 1)
        self.multi_step_mfiller = y.get('multi_step_mfiller', True)
        self.multi_step_trajpred = y.get('multi_step_trajpred', True)
        tp_cfg = self.network_cfg('traj_pred', self.model_specs.get('trajpred_cfg', _JOINT_DEMO_YML['model_specs']['trajpred_cfg']))
        self.trajpred_seq_len = int(tp_cfg.get('seq_len', TRAJ_WINDOW))

    @staticmethod
    def network_cfg(package, net_cfg_id):
        """the YAML of a network config (`<package>/cfg/**/<id>.yml`, cwd-relative like the reference) or {} if not found"""
        import yaml
        files = glob.glob(f'{package}/cfg/**/{net_cfg_id}.yml', recursive=True)
        return (yaml.safe_load(open(files[0])) or {}) if len(files) == 1 else {}

    @staticmethod
    def network_cfg_dir(package, net_cfg_id):
        root = os.path.expanduser(MTConfig.network_cfg(package, net_cfg_id).get('results_root_dir', _RESULTS_ROOT[package]))
        return f'{root}/{net_cfg_id}'


class MotionTrajJointModel:
    supports_person_batch = True     # inference() accepts [B, T, 69] with B > 1 (GlobalReconOptimizer.infer_motion_traj_all)
    supports_ragged_batch = True     # inference() accepts seq_len [B]: tracks of different lengths in one call

    def __init__(self, cfg=None, device=torch.device('cuda'), log=None, smpl=None, states=None):
        """cfg: config id / object of the joint model (its checkpoint locations, `multi_step_trajpred` and
        `trajpred_seq_len`; None = the shipped joint config's settings).  states: optional (infiller_state_dict,
        trajpred_state_dict); otherwise the reference's checkpoint files are loaded."""
        self.device, self.log = L.require_cuda(device), log
        if isinstance(cfg, str):
            cfg = MTConfig(cfg)
        self.cfg = cfg
        self.multi_step_mfiller = getattr(cfg, 'multi_step_mfiller', True)
        self.multi_step_trajpred = getattr(cfg, 'multi_step_trajpred', False)
        if smpl is None:
            from .smpl import SMPL
            smpl = SMPL(device=self.device)
        self.smpl = smpl
        if states is None:
            specs = getattr(cfg, 'model_specs', None) or _JOINT_DEMO_YML['model_specs']
            states = []
            for package, key in [('motion_infiller', 'mfiller'), ('traj_pred', 'trajpred')]:
                path = _find_checkpoint(MTConfig.network_cfg_dir(package, specs[f'{key}_cfg']), specs.get(f'{key}_cp', 'best'),
                                        specs.get(f'{key}_version'))
                if log is not None:
                    log.info(f'loading {package} from check point {path}')
                states.append(load_lightning_state_dict(path))
        self.mfiller = MotionInfillerVAE(states[0], self.device)
        self.traj_predictor = TrajPredVAE(states[1], self.device, self.smpl, getattr(cfg, 'trajpred_seq_len', TRAJ_WINDOW))

    def get_motion_latent(self, seq_len):
        return self.mfiller.get_latent(seq_len)

    def get_traj_latent(self, seq_len):
        return self.traj_predictor.get_latent(seq_len)

    def inference(self, batch, sample_num=1, recon=False, row_batch=None):
        """motion_traj_joint_model.py:141-145 (+ pred_trajectory :73-133, 'infer' mode).  With multi_step_trajpred the
        trajectory's window latents come from `in_traj_window_latent` [windows, B * sample_num, 128] when given.

        With `batch['seq_len']` [B], row b of `in_body_pose` [B, T_max, 69] / `frame_mask` [B, T_max] is a track of seq_len[b]
        frames: all tracks run in one ragged call, and row b's outputs over its first seq_len[b] frames are bit-identical to
        `inference` on that track alone (frames past its end are zero).  Row b uses the first windows of `in_motion_latent`
        [B, windows, 128] (or of a shared [windows, 128]) and of `in_traj_window_latent` [windows, B * sample_num, 128] that its
        length needs; `in_traj_latent` is [1 or B * sample_num, 128].  Latents that are not given are drawn in the order and shapes
        of the single-track calls (draw_ragged_eps).  `row_batch` (internal: GlobalReconOptimizer) names blocks of equal-length
        rows whose outputs must equal one call on the whole block instead (ragged_plan)."""
        if recon:
            raise NotImplementedError('recon mode needs the trajectory predictor\'s posterior encoder, which is not implemented on CUDA '
                                      '(MotionInfillerVAE.inference(recon=True) reconstructs the motion)')
        if batch.get('seq_len') is not None:
            return self._inference_ragged(batch, sample_num, row_batch)
        data = self.mfiller.inference(batch, sample_num, recon=False, multi_step=True)
        motion = data['infer_out_body_pose']                                        # [B,S,T,69]
        B, S, T = motion.shape[:3]
        tb = {'in_body_pose': motion.reshape(B * S, T, 69)}
        for k in ('in_traj_latent', 'in_traj_window_latent'):
            if k in data:
                tb[k] = data[k]
        out = self.traj_predictor.inference(tb, sample_num=1, multi_step=self.multi_step_trajpred)
        data['infer_out_pose'] = out['infer_out_pose'].view(B, S, T, 72)
        data['infer_out_trans'] = out['infer_out_trans'].view(B, S, T, 3)
        data['infer_out_orient'] = out['infer_out_orient'].view(B, S, T, 3)
        data['infer_out_local_traj_tp'] = out['infer_out_local_traj_tp'].view(T, B, S, 11)
        return data

    def ragged_plan(self, seq_len, row_batch=None, sample_num=1):
        return ragged_plan(seq_len, row_batch, sample_num, self.traj_predictor.seq_len, self.multi_step_trajpred)

    def draw_ragged_latents(self, seq_len, row_batch=None):
        """eps of a sample_num 1 ragged call drawn as its serial calls draw them, as the latent keys `inference` takes"""
        plan = self.ragged_plan(seq_len, row_batch)
        inf, traj = draw_ragged_eps(plan, self.device)
        out = {'in_motion_latent': inf}
        if self.multi_step_trajpred:
            wl = torch.zeros((int(plan['C'].max()), plan['E'], NZ), device=self.device)
            for e, t in enumerate(traj):
                wl[:t.shape[0], e] = t
            out['in_traj_window_latent'] = wl
        else:
            out['in_traj_latent'] = traj
        return out

    def _ragged_eps(self, plan, batch):
        """expanded-row eps from the batch's latents, or drawn (draw_ragged_eps) when none is given"""
        dev, S, E = self.device, plan['S'], plan['E']
        keys = ('in_motion_latent', 'in_traj_latent', 'in_traj_window_latent')
        given = {k: batch[k].to(dev, torch.float32) for k in keys if batch.get(k) is not None}
        tkey = 'in_traj_window_latent' if plan['multi_step_traj'] else 'in_traj_latent'
        inf, traj = draw_ragged_eps(plan, dev, 'in_motion_latent' not in given, tkey not in given)
        nmax = int(plan['nwin'].max())
        ml = given.get('in_motion_latent')
        if ml is not None:
            ml = ml.unsqueeze(0).expand(plan['B'], -1, -1) if ml.dim() == 2 else ml
            if ml.shape[1] < nmax:
                raise ValueError(f'{nmax} windows need {nmax} latents, got {ml.shape[1]}')
            inf = ml[:, :nmax].repeat_interleave(S, dim=0).contiguous()
        if tkey not in given:
            return inf, traj
        if plan['multi_step_traj']:
            wl = given[tkey]
            if wl.shape[0] < int(plan['C'].max()) or wl.shape[1] != E:
                raise ValueError(f'in_traj_window_latent: need [>= {int(plan["C"].max())}, {E}, {NZ}], got {tuple(wl.shape)}')
            traj = [wl[:int(plan['C'][e]), e] for e in range(E)]
        else:
            tl = given[tkey]
            traj = tl.expand(E, -1) if tl.shape[0] == 1 else tl
            if traj.shape[0] != E:
                raise ValueError(f'in_traj_latent: need [1 or {E}, {NZ}], got {tuple(tl.shape)}')
        return inf, traj

    def _inference_ragged(self, batch, sample_num, row_batch):
        dev = self.device
        pose_in = batch['in_body_pose'].to(dev, torch.float32)
        frame_mask = batch['frame_mask'].to(dev, torch.float32)
        B, Tmax = pose_in.shape[:2]
        seq_len = [int(t) for t in (batch['seq_len'].tolist() if isinstance(batch['seq_len'], torch.Tensor) else batch['seq_len'])]
        if len(seq_len) != B or max(seq_len) > Tmax:
            raise ValueError(f'seq_len {seq_len} does not fit in_body_pose {tuple(pose_in.shape)}')
        plan = self.ragged_plan(seq_len, row_batch, sample_num)
        S, E = plan['S'], plan['E']
        eps_inf, eps_traj = self._ragged_eps(plan, batch)
        lens = plan['lens']
        # frame (e, t) of expanded row e = b S + s is input frame b Tmax + t; packed rows in each network's order
        src = lambda order: np.concatenate([(e // S) * Tmax + np.arange(lens[e]) for e in order])
        dst = lambda order: np.concatenate([e * Tmax + np.arange(lens[e]) for e in order])
        io, po = plan['inf_order'], plan['pred_order']
        d_io, d_po = dst(io), dst(po)
        srt = np.argsort(d_io, kind='stable')
        host = np.concatenate([src(io), srt[np.searchsorted(d_io[srt], d_po)], d_po])       # + the infiller row of each predictor row
        idx = torch.from_numpy(host).to(dev, non_blocking=False)
        M = int(lens.sum())
        ints = torch.from_numpy(np.concatenate([plan['inf_off'], plan['pred_off'], plan['pred_woff']]).astype(np.int32)).to(dev)
        eps_inf = eps_inf[torch.from_numpy(io).to(dev)].contiguous()
        if eps_traj is not None:
            eps_traj = torch.stack([eps_traj[e] for e in po]) if not plan['multi_step_traj'] else torch.cat([eps_traj[e] for e in po])
            eps_traj = eps_traj.contiguous()
        lib = self.mfiller.net.lib
        self.mfiller.net.workspace(lib.glamr_infiller_ragged_workspace_floats(E))
        lens_p = np.ascontiguousarray(lens[po], dtype=np.int32)
        tws = lib.glamr_trajpred_windows_ragged_workspace_floats(E, _np_ptr(lens_p), plan['traj_window']) if plan['multi_step_traj'] \
            else lib.glamr_trajpred_ragged_workspace_floats(E, _np_ptr(lens_p))
        self.traj_predictor.net.workspace(tws)
        self.smpl._workspace(M, fk_only=True)
        key = ('ragged', tuple(seq_len), None if row_batch is None else tuple(int(r) for r in row_batch), S,
               Tmax, eps_traj is None)
        with torch.cuda.device(dev):
            body, local, trans, orient = self.mfiller.graphs.run(
                key, lambda *a: self._ragged_forward(plan, *a), (pose_in, frame_mask, idx, ints, eps_inf, eps_traj))
        T = Tmax
        data = dict(batch)
        data['infer_out_body_pose'] = body.view(B, S, T, 69)
        data['batch_size'] = B
        data['infer_out_trans'] = trans.view(B, S, T, 3)
        data['infer_out_orient'] = orient.view(B, S, T, 3)
        data['infer_out_pose'] = torch.cat([data['infer_out_orient'], data['infer_out_body_pose']], dim=-1)
        data['infer_out_local_traj_tp'] = local.view(B, S, T, 11).permute(2, 0, 1, 3).contiguous()
        return data

    def _ragged_forward(self, plan, pose_in, frame_mask, idx, ints, eps_inf, eps_traj):
        """the ragged infiller sweep, SMPL FK and the ragged predictor, device tensors only -> [E, T_max, *] outputs"""
        dev, E = self.device, plan['E']
        B, Tmax = pose_in.shape[:2]
        M = int(plan['lens'].sum())
        g_src, g_pred, g_dst = idx[:M], idx[M:2 * M], idx[2 * M:]
        off_i, off_p, woff_p = ints[:E + 1], ints[E + 1:2 * E + 2], ints[2 * E + 2:]
        io, po = plan['inf_order'], plan['pred_order']
        lens_i = np.ascontiguousarray(plan['lens'][io], dtype=np.int32)
        rb_i = np.ascontiguousarray(plan['row_batch'][io], dtype=np.int32)
        lens_p = np.ascontiguousarray(plan['lens'][po], dtype=np.int32)
        rb_p = np.ascontiguousarray(plan['row_batch'][po], dtype=np.int32)
        pose = pose_in.reshape(B * Tmax, 69)[g_src].contiguous()                             # [M,69], infiller order
        key_pad = (~(frame_mask.reshape(B * Tmax)[g_src] == 1)).to(torch.uint8).contiguous()
        stream = torch.cuda.current_stream().cuda_stream
        net = self.mfiller.net
        ws = net.workspace(net.lib.glamr_infiller_ragged_workspace_floats(E))
        L.check(net.lib.glamr_infiller_forward_ragged(net.h, E, _np_ptr(lens_i), _np_ptr(rb_i), off_i.data_ptr(), pose.data_ptr(),
                                                      key_pad.data_ptr(), eps_inf.data_ptr(), eps_inf.shape[1], ws.data_ptr(), ws.numel(),
                                                      stream), 'glamr_infiller_forward_ragged')
        body = pose[g_pred].contiguous()                                                     # predictor order
        jp = self.traj_predictor.get_joint_pos(body).contiguous()
        local = torch.empty((M, 11), dtype=torch.float32, device=dev)
        trans = torch.empty((M, 3), dtype=torch.float32, device=dev)
        orient = torch.empty((M, 3), dtype=torch.float32, device=dev)
        tnet = self.traj_predictor.net
        eps_p = None if eps_traj is None else eps_traj.data_ptr()
        if plan['multi_step_traj']:
            ws = tnet.workspace(tnet.lib.glamr_trajpred_windows_ragged_workspace_floats(E, _np_ptr(lens_p), plan['traj_window']))
            L.check(tnet.lib.glamr_trajpred_windows_forward_ragged(
                tnet.h, E, plan['traj_window'], _np_ptr(lens_p), _np_ptr(rb_p), off_p.data_ptr(), woff_p.data_ptr(), jp.data_ptr(), eps_p,
                local.data_ptr(), trans.data_ptr(), orient.data_ptr(), ws.data_ptr(), ws.numel(), stream), 'glamr_trajpred_windows_forward_ragged')
        else:
            ws = tnet.workspace(tnet.lib.glamr_trajpred_ragged_workspace_floats(E, _np_ptr(lens_p)))
            L.check(tnet.lib.glamr_trajpred_forward_ragged(
                tnet.h, E, _np_ptr(lens_p), _np_ptr(rb_p), off_p.data_ptr(), jp.data_ptr(), eps_p, None, None, local.data_ptr(),
                trans.data_ptr(), orient.data_ptr(), ws.data_ptr(), ws.numel(), stream), 'glamr_trajpred_forward_ragged')
        outs = []
        for x, w in ((body, 69), (local, 11), (trans, 3), (orient, 3)):
            o = torch.zeros((E * Tmax, w), dtype=torch.float32, device=dev)
            o.index_copy_(0, g_dst, x)
            outs.append(o)
        return tuple(outs)
