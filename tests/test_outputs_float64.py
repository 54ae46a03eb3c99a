"""The optimiser's per-frame outputs against a float64 forward, element by element, at the variables of its check points.

What forward() leaves in the R_* buffers (world and base pose, keypoint projections, the persons' pose in the camera, the
camera and its inverse, traj_local) is what optimize() returns, run_dataset saves and the evaluator reads.  The gradient tests
do not hold it: a weighted term never sees an element of weight zero (kp_2d_pred of an invisible frame, the camera-space pose
where ctr_w is 0, the base pose outside the exist range that the next stage reads back as orient_base_init).  Here each output
element o is compared with the oracle's forward in float64 (o64) at the same variables and state, with the same forward in
float32 (o32) as the yardstick of a legitimate float32 implementation:

    |o[e] - o64[e]|  <=  C_NOISE * D(b(e))  +  C_ULP * 2^-24 * (|o64[e]| + A[e])
    D(b) = max(max_{e in b} |o32[e] - o64[e]|,  FLOOR * max |o64|)

b(e) is the element's block of BLOCK consecutive frames of one person's output (of the camera for cam_pose / cam_pose_inv);
the constants are test_grad_float64's.  The three axis-angle outputs are compared as float64 Rodrigues matrices of the
candidate and of both references, so the branch at pi (where the camera-space root orientation sits) is not read as an error;
cam_pose / cam_pose_inv as 3x4 matrices; traj_local on the exist frames.

A[e] is 0 except where a step amplifies float32 rounding beyond the element's own magnitude (conditioning): a projection from
near the camera plane (z cancels terms much larger than itself) and the camera from the persons where they disagree (Gram-Schmidt
of a mean with short columns), with everything computed from that camera.  One sample of the float32 reference's rounding
does not bound those: in the four-person person2cam case the host emulator exceeded C_NOISE D by x15 on a joint projected from
~1e-3 m depth (|kp_2d_pred| ~ 3e6 px) and by x2.4 on the camera of a frame whose Gram-Schmidt amplification is 15x.

The trajectory codec's heading and xy prefix sums: torch's float32 cumsum accumulates in float64 on the CPU, so the float32
reference runs both as sequential float32 sums (float32_scans), and their error reaches every output downstream (the camera
from the persons, the camera-space pose, the projections) through o32.  On top of that, the outputs of the scans themselves
(world / base translation x and y, the orientation of codec frames) keep test_grad_float64's scan floor, 2^-22 sqrt(n) times
the scan's largest partial sum.  With torch's cumsum as the float32 scans instead, the host emulator's worst ratio on
dynamic_p1_t1025 rises from 0.29 to 0.80 (orient_ciw), every other family unchanged.

Beyond the bound, exact rules: every element is written by every evaluation (the buffers are filled with NaN before each
check-point closure); the base pose on frames the codec does not produce (every frame without it) is orient/trans_base_init,
bit for bit; kp_2d_pred is 0 on frames whose intrinsics are 0 (the invisible ones, which no term sees); traj_local rows
outside the exist range are 0; a constant camera is the constant.  forward(), the public path,
copies the buffers into the data dict bit for bit.

On one H100 80GB HBM3 (700 W limit) the worst |cuda - o64| / bound over every case, output and check point was 0.26 (orient_ciw,
static_multi_p4_t300); per family: orient_ciw 0.26, kp_pred 0.24, orient_world / orient_base 0.17, cam_pose_inv 0.16, trans_ciw
0.15, cam_pose 0.14, traj_local 0.02, trans_world / trans_base 0.02 (their bound set by the scan floor); 0.11-0.26 per case.  The
GPU tests of this file took 196 s there.
GLAMR_OUTPUT_REPORT=<file> appends the worst |o - o64| of every case, output and check point next to its bound.

CPU: the host emulator's outputs (a second float32 implementation, sequential scans) pass the bound, and modelled bugs applied to
them do not (each prints the factor by which it fails)."""
import contextlib
import copy
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from glamr_b200 import lib as L
from test_grad_float64 import (ALL as GRAD_ALL, BLOCK, C_NOISE, C_ULP, DEV, EPS32, FLOOR, SCAN_CHUNK, SCAN_FLOOR, _closure, _emu_runner,
                               _init, _make_model, _snapshot, case, oracle_for, oracle_state, p2c_flags, param_order, view)
from test_grad_float64_modes import ALL as MODE_ALL, EMU_P2C, mode_case

ALL = GRAD_ALL + MODE_ALL
# the last: four persons, a joint projected from ~1e-3 m depth and a camera from the persons that Gram-Schmidt amplifies 15x
EMU_CASES = ['dynamic_p1_t1025', 'static_multi_p3_t1100_gaps', EMU_P2C, 'p2c_3dpw_p4_t300_gaps']
# family -> (R_* buffer, data dict key, values per frame (None: 2 J))
PERSON_OUT = {
    'orient_world': (L.R_ORIENT_WORLD, 'smpl_orient_world', 3),
    'trans_world': (L.R_TRANS_WORLD, 'root_trans_world', 3),
    'orient_base': (L.R_ORIENT_BASE, 'smpl_orient_world_base', 3),
    'trans_base': (L.R_TRANS_BASE, 'root_trans_world_base', 3),
    'kp_pred': (L.R_KP_PRED, 'kp_2d_pred', None),
    'orient_ciw': (L.R_ORIENT_CIW, 'smpl_orient_cam_in_world', 3),
    'trans_ciw': (L.R_TRANS_CIW, 'root_trans_cam_in_world', 3),
    'traj_local': (L.R_TRAJ_LOCAL, 'traj_local', 11),
}
CAMERA = {'cam_pose': L.R_CAM_POSE, 'cam_pose_inv': L.R_CAM_POSE_INV}
AXIS_ANGLE = {'orient_world', 'orient_base', 'orient_ciw'}
BUFFER_NAME = {what: name for name, what in vars(L).items() if name.startswith('R_') and isinstance(what, int)}
# Every R_* buffer checked here is rewritten by every evaluation: traj_cam_forward_kernel writes the base and world pose of every
# frame of every person (traj_post) and traj_local of every row (traj_pre on the exist range, zeros elsewhere); the camera of
# every row comes from traj_cam_forward_kernel or, from the persons, cam_forward_kernel; frame_residuals_kernel writes kp_pred
# (every joint) and the camera-space pose of every frame-person of the rank's range, which is all of them here.  So no buffer is
# carried from one evaluation to the next and none is excluded from the NaN fill.  R_JOINTS_WORLD is test_lbs_float64's.
FILLED = [what for what, _, _ in PERSON_OUT.values()] + list(CAMERA.values())


def _setup(name):
    return mode_case if name in MODE_ALL else case


# ------------------------------------------------------------------------------------------------ outputs of a run
def split_buffers(read, P, T, J):
    """the R_* buffers (read(what) -> flat float32 tensor) as {'persons': [{family: [T, k]}], 'cam_pose': [T, 12], ...}"""
    out = {'persons': [{} for _ in range(P)]}
    for fam, (what, _, k) in PERSON_OUT.items():
        a = read(what).reshape(P, T, -1).numpy()
        for p in range(P):
            out['persons'][p][fam] = a[p].copy()
    for fam, what in CAMERA.items():
        out[fam] = read(what).reshape(T, 12).numpy().copy()
    return out


def data_outputs(data):
    """the same families from a data dict (the oracle's, or the CUDA path's after forward), float64; traj_local: exist rows"""
    out = {'persons': []}
    for d in data['person_data'].values():
        out['persons'].append({fam: torch.as_tensor(d[key]).detach().cpu().double().reshape(len(d[key]), -1).numpy()
                               for fam, (_, key, _) in PERSON_OUT.items() if key in d})
    for fam in CAMERA:
        out[fam] = torch.as_tensor(data[fam]).detach().cpu().double()[:, :3, :4].reshape(-1, 12).numpy()
    return out


def base_init(comp):
    """per person (orient_base_init, trans_base_init) of a StageCompiler: the base the kernels write on frames the codec does not
    produce, trans x / y from world_dxy_base where the layout has world_dxy"""
    out = []
    for c in comp.const:
        tb = c['trans_base_init'].detach().cpu().numpy().copy()
        if c['world_dxy_base'] is not None:
            tb[:, :2] = c['world_dxy_base'].detach().cpu().numpy()
        out.append((c['orient_base_init'].detach().cpu().numpy().copy(), tb))
    return out


# ------------------------------------------------------------------------------------------------ the float64 / float32 forward
class _Float32ScanTorch:
    """torch, with cumsum of float32 tensors a sequential float32 sum (numpy accumulates in the array's dtype); counts the
    cumsum calls, so that a codec which stops calling torch.cumsum by name is noticed (oracle_outputs asserts two per person)"""

    def __init__(self):
        self.calls = 0

    def __getattr__(self, k):
        return getattr(torch, k)

    def cumsum(self, x, dim):
        self.calls += 1
        if x.dtype != torch.float32:
            return torch.cumsum(x, dim)
        return torch.from_numpy(np.cumsum(x.detach().numpy(), axis=dim, dtype=np.float32))


@contextlib.contextmanager
def float32_scans():
    """the trajectory codec's heading and xy prefix sums in float32, one rounding per addition; yields the counting stand-in"""
    from oracle import traj_codec as tc
    saved = tc.torch
    tc.torch = _Float32ScanTorch()
    try:
        yield tc.torch
    finally:
        tc.torch = saved


def camera_conditioning(ora, data):
    """per camera row: the amplification 1 / (|a1| |a2 - (b1.a2) b1|) with which Gram-Schmidt turns the rounding of the 6d it
    orthonormalises into the rotation, when the camera is the mean of the persons' camera-to-world transforms (oracle
    _camera_from_persons, restated in float64; the result is checked against the camera it made).  Persons that disagree
    shorten the mean's columns.  1 for a camera that is not from the persons."""
    from oracle import rotations as rt
    cands = []
    for d in data['person_data'].values():
        p2c = d['person2cam']
        if any(p2c_flags(ora)):
            p2c = torch.matmul(p2c, rt.make_transform(d['person2cam_res_rot'], d['person2cam_res_trans'], '6d'))
        cands.append(torch.matmul(d['person_transform_world'], p2c) * d['vis_frames'][:, None, None])
    npers = data['fr_num_persons']
    mean = sum(cands) / npers.clamp(min=1)[:, None, None].to(cands[0].dtype)
    src = np.maximum.accumulate(np.where(npers.numpy() > 0, np.arange(len(npers)), int(np.argmax(npers.numpy() > 0))))
    d6 = rt.rotmat_to_rot6d(mean[torch.as_tensor(src)][:, :3, :3])
    empty = npers == 0
    if empty.any():
        d6[empty] = d6[empty] + data['cam_inv_rot_residual']
    assert torch.allclose(rt.rot6d_to_rotmat(d6), data['cam_pose_inv'][:, :3, :3], atol=1e-9)
    a1, a2 = d6[:, :3], d6[:, 3:]
    n1 = a1.norm(dim=-1)
    b1 = a1 / n1[:, None]
    n2 = (a2 - (b1 * a2).sum(-1, keepdim=True) * b1).norm(dim=-1)
    return (1.0 / (n1 * n2)).numpy()


def oracle_outputs(Oracle, cfg, assets, state, stage, variables, lay, theta, dtype):
    """forward-only oracle_closure: the oracle's outputs in `dtype` with every variable of the stage set to its value in theta"""
    ora = Oracle(copy.deepcopy(cfg), assets)
    data = copy.deepcopy(state)
    if dtype == torch.float64:
        data = ora.to_float64(data)
    params = ora.get_parameter(data, variables)
    order = param_order(variables, len(data['person_data']), ora.flag_fixed_cam, ora.flag_opt_traj, p2c_flags(ora))
    assert len(order) == len(params)
    th = theta.detach().cpu()
    with torch.no_grad():
        for (p, name), prm in zip(order, params):
            prm.copy_(view(lay, th, p, name).reshape(prm.shape).to(prm.dtype))
        with (float32_scans() if dtype == torch.float32 else contextlib.nullcontext()) as scans:
            ora.forward(data, variables, {'stage': stage})
        codec = ora.flag_infer_motion_traj and ora.flag_pred_traj
        if scans is not None:
            assert scans.calls == (2 * len(data['person_data']) if codec else 0), f'{scans.calls} cumsum calls in the codec'
        out = data_outputs(data)
        if dtype == torch.float64:
            out['joints'] = [d['joints_world'].numpy() for d in data['person_data'].values()]
            from_persons = ora.flag_opt_cam and stage != 'init' and 'cam' not in variables and ora.flag_opt_cam_from_person_pose
            out['cam_cond'] = camera_conditioning(ora, data) if from_persons else np.ones(len(out['cam_pose']))
    return out


def add_references(r, Oracle, cfg, assets, template):
    state = oracle_state(template, r['state'], r['layout'], r['theta'])
    args = (Oracle, cfg, assets, state, r['stage'], r['specs']['opt_variables'], r['layout'], r['theta'])
    r['o64'], r['o32'] = oracle_outputs(*args, torch.float64), oracle_outputs(*args, torch.float32)


# ------------------------------------------------------------------------------------------------ the bound
def rodrigues64(aa):
    """[n, 3] axis-angle -> [n, 9] rotation matrices, float64"""
    aa = np.asarray(aa, np.float64)
    th = np.linalg.norm(aa, axis=1)
    k = aa / np.where(th > 0, th, 1.0)[:, None]
    K = np.zeros((len(aa), 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    K = K - K.transpose(0, 2, 1)
    s, c = np.sin(th)[:, None, None], (1.0 - np.cos(th))[:, None, None]
    R = np.eye(3) + s * K + c * (K @ K)
    return R.reshape(-1, 9)


def out_bound(o64, o32, extra=None, ulp_extra=None):
    """per-element bound of one person's (or the camera's) output [frames, k]; extra: per-element floor (scan floors);
    ulp_extra: per-element magnitude added to |o64| in the ULP term, for the rounding an ill-conditioned step amplifies
    (conditioning)"""
    d = np.abs(o32 - o64).max(axis=1) if o64.size else np.zeros(len(o64))
    floor = FLOOR * float(np.abs(o64).max()) if o64.size else 0.0
    nb = (len(d) + BLOCK - 1) // BLOCK
    blk = np.zeros(nb * BLOCK)
    blk[:len(d)] = d
    D = np.maximum(np.repeat(blk.reshape(nb, BLOCK).max(axis=1), BLOCK)[:len(d)], floor)[:, None] * np.ones_like(o64)
    if extra is not None:
        D = np.maximum(D, extra)
    ulp = np.abs(o64) if ulp_extra is None else np.abs(o64) + ulp_extra
    return C_NOISE * D + C_ULP * EPS32 * ulp


def conditioning(o64, T):
    """ULP-term additions (ulp_extra) of the outputs that amplify float32 rounding beyond their own magnitude, by family.
    The projection u = f x / z + c: z is a sum of terms of size sum_k |R_2k j_k| + |t_z| and carries the rounding of those,
    so u - c moves by that relative to |z|; near the camera plane this reaches 1e4 (|kp_2d_pred| ~ 3e6 px at a depth of
    ~1e-3 m in the four-person person2cam case).  The camera from the persons: its rotation carries Gram-Schmidt's
    amplification kappa (camera_conditioning), and so does everything computed with it, scaled by the magnitudes the
    rotation multiplies (unit entries, the translations)."""
    kap = o64['cam_cond']
    cam = o64['cam_pose'].reshape(T, 3, 4)
    out = {'persons': [], 'cam_pose': (kap - 1.0)[:, None] * np.abs(o64['cam_pose']).max(axis=1, keepdims=True),
           'cam_pose_inv': (kap - 1.0)[:, None] * np.abs(o64['cam_pose_inv']).max(axis=1, keepdims=True)}
    for p, jw in enumerate(o64['joints']):
        Xc = np.einsum('tik,tjk->tji', cam[:, :, :3], jw) + cam[:, None, :, 3]
        zsum = np.einsum('tk,tjk->tj', np.abs(cam[:, 2, :3]), np.abs(jw)) + np.abs(cam[:, None, 2, 3])
        with np.errstate(divide='ignore', invalid='ignore'):
            kz = np.where(np.abs(Xc[..., 2]) > 0, zsum / np.abs(Xc[..., 2]), 1.0)
        kp = o64['persons'][p]['kp_pred']
        scale = (np.maximum(kz, 1.0) * kap[:, None] - 1.0)
        tw = np.abs(o64['persons'][p]['trans_world']).max(axis=1) + np.abs(cam[:, :, 3]).max(axis=1)
        out['persons'].append({'kp_pred': np.repeat(scale, 2, axis=1) * np.abs(kp),
                               'orient_ciw': np.repeat((kap - 1.0)[:, None], 9, axis=1),
                               'trans_ciw': np.repeat(((kap - 1.0) * tw)[:, None], 3, axis=1)})
    return out


def scan_floors(o64p, start, n, T):
    """floors of the outputs of a person's heading and xy scans over its n exist frames: the heading's error (radians) bounds
    the matrix entries of the codec frames' orientation, the xy scan's the translation x / y"""
    tl = o64p['traj_local']
    heading = np.cumsum(np.arctan2(tl[:, 10], tl[:, 9]))
    rot = np.zeros((T, 9))
    rot[start:start + n] = SCAN_FLOOR * math.sqrt(n) * float(np.abs(heading).max())
    xy = np.zeros((T, 3))
    xy[start:start + n, :2] = SCAN_FLOOR * math.sqrt(n) * float(np.abs(o64p['trans_base'][start:start + n, :2]).max())
    return {'orient_world': rot, 'orient_base': rot, 'trans_world': xy, 'trans_base': xy}


def _compare(label, c, a64, a32, extra, first_frame, person, rep, msgs, ulp_extra=None):
    b = out_bound(a64, a32, extra, ulp_extra)
    err = np.abs(c - a64)
    bad = ~(err <= b)
    with np.errstate(divide='ignore', invalid='ignore'):
        ratio = np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err > 0, np.inf, 0.0))
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    i = int(np.argmax(ratio)) if ratio.size else 0
    worst = (float(ratio.flat[i]), float(err.flat[i]), float(b.flat[i])) if ratio.size else (0.0, 0.0, 0.0)
    rep.append((label, worst[1], worst[2], worst[0]))
    if bad.any():
        row = int(np.where(bad.any(axis=1))[0][0])
        who = f'frame {first_frame + row}' if person is None else f'person {person} frame {first_frame + row}'
        msgs.append(f'{label}: {int(bad.sum())} elements outside the bound, first at {who}; worst |o-o64| {worst[1]:.3e} vs bound '
                    f'{worst[2]:.3e} (x{worst[0]:.2f})')


def check_bound(what, cand, r):
    """-> (messages, report lines (label, worst |o - o64|, bound there, ratio)) of candidate outputs at record r's variables"""
    rep, msgs = [], []
    o64, o32 = r['o64'], r['o32']
    T = len(cand['cam_pose'])
    cond = conditioning(o64, T)
    for p, (s, n) in enumerate(zip(r['starts'], r['lens'])):
        floors = scan_floors(o64['persons'][p], s, n, T) if r['codec'] else {}
        for fam in PERSON_OUT:
            c = cand['persons'][p][fam].astype(np.float64)
            if fam == 'traj_local':
                if not r['codec']:
                    continue
                c, first = c[s:s + n], s
            else:
                first = 0
            a64, a32 = o64['persons'][p][fam], o32['persons'][p][fam]
            assert c.shape == a64.shape == a32.shape, (fam, c.shape, a64.shape, a32.shape)
            if fam in AXIS_ANGLE:
                c, a64, a32 = rodrigues64(c), rodrigues64(a64), rodrigues64(a32)
            _compare(f'{what} {fam}[{p}]', c, a64, a32, floors.get(fam), first, p, rep, msgs, cond['persons'][p].get(fam))
    for fam in CAMERA:
        _compare(f'{what} {fam}', cand[fam].astype(np.float64), o64[fam], o32[fam], None, 0, None, rep, msgs, cond[fam])
    return msgs, rep


def check_written(what, cand):
    """every element of every checked buffer is finite: a NaN left from the fill names the buffer and the (person, frame)"""
    msgs = []
    for fam, (what_r, _, _) in PERSON_OUT.items():
        for p, d in enumerate(cand['persons']):
            rows = np.where(np.isnan(d[fam]).any(axis=1))[0]
            if rows.size:
                msgs.append(f'{what} {BUFFER_NAME[what_r]}: person {p} frames {rows[:8].tolist()} ({rows.size} frames) not written')
    for fam, what_r in CAMERA.items():
        rows = np.where(np.isnan(cand[fam]).any(axis=1))[0]
        if rows.size:
            msgs.append(f'{what} {BUFFER_NAME[what_r]}: frames {rows[:8].tolist()} ({rows.size} frames) not written')
    return msgs


def check_exact(what, cand, r):
    """base pose on the frames the codec does not produce = orient/trans_base_init and the state the oracle copies, bit for bit;
    kp_2d_pred 0 on frames whose intrinsics are 0 (the invisible frames: no term sees them); traj_local rows outside the exist
    range 0; a constant camera is the constant"""
    msgs = []
    state = list(r['state']['person_data'].values())
    T = len(cand['cam_pose'])
    for p, (s, n) in enumerate(zip(r['starts'], r['lens'])):
        outside = np.ones(T, bool)
        if r['codec']:
            outside[s:s + n] = False
        for k, (fam, key) in enumerate((('orient_base', 'smpl_orient_world_base'), ('trans_base', 'root_trans_world_base'))):
            c = cand['persons'][p][fam]
            for ref, src in ((r['base_init'][p][k], 'orient/trans_base_init'), (torch.as_tensor(state[p][key]).cpu().numpy(), 'the state')):
                diff = np.where(outside & (c != ref).any(axis=1))[0]
                if diff.size:
                    msgs.append(f'{what} {fam}: person {p} frames {diff[:8].tolist()} ({diff.size}) differ from {src}')
        zero_K = np.where(~torch.as_tensor(state[p]['cam_K']).reshape(T, -1).cpu().numpy().any(axis=1))[0]
        nz = zero_K[cand['persons'][p]['kp_pred'][zero_K].any(axis=1)]
        if nz.size:
            msgs.append(f'{what} kp_pred: person {p} frames {nz[:8].tolist()} with zero intrinsics are not 0')
        tl = cand['persons'][p]['traj_local']
        nz = np.where(outside & (tl != 0).any(axis=1))[0]
        if nz.size:
            msgs.append(f'{what} traj_local: person {p} rows {nz[:8].tolist()} outside the exist range are not 0')
    if r['cam_mode'] == L.CAM_CONST:
        const = torch.as_tensor(r['state']['cam_pose']).cpu()[:, :3, :4].reshape(-1, 12).numpy()
        diff = np.where((cand['cam_pose'] != const).any(axis=1))[0]
        if diff.size:
            msgs.append(f'{what} cam_pose: frames {diff[:8].tolist()} ({diff.size}) differ from the constant camera')
    return msgs


REPORT = os.environ.get('GLAMR_OUTPUT_REPORT')     # file to append the per-output worst |o - o64| and bound to


def check_records(name, recs, tag=''):
    rep, msgs = [], []
    for r in recs:
        what = f'{name}{tag} {r["stage"]} {r["point"]}'
        msgs += check_written(what, r['cand'])
        m, rp = check_bound(what, r['cand'], r)
        msgs += m
        rep += rp
        msgs += check_exact(what, r['cand'], r)
    if REPORT:
        with open(REPORT, 'a') as f:
            for label, err, b, ratio in rep:
                f.write(f'{label}\t{err:.3e}\t{b:.3e}\t{ratio:.3f}\n')
    worst = max(rep, key=lambda x: x[3])
    print(f'{name}{tag}: worst |o-o64|/bound {worst[3]:.3f} at {worst[0]} ({worst[1]:.3e} vs {worst[2]:.3e})')
    assert not msgs, '\n'.join(msgs)
    return rep


def _record(stage, point, specs, cand, state, layout, theta, comp, cam_mode):
    persons = list(state['person_data'].values())
    return {'stage': stage, 'point': point, 'specs': specs, 'cand': cand, 'state': state, 'layout': layout, 'theta': theta,
            'cam_mode': cam_mode, 'codec': comp.traj_source == L.TRAJ_PREDICTED, 'base_init': base_init(comp),
            'starts': [int(d['fr_start']) for d in persons], 'lens': [int(torch.as_tensor(d['exist_len']).sum()) for d in persons]}


# ------------------------------------------------------------------------------------------------ CPU: host emulator
def emulator_outputs(name, assets):
    """the host-compiled frame functions from the oracle's float32 init: outputs at the first closure of every stage and after
    the stage's Adam steps, each with the oracle's float64 / float32 outputs at the same variables"""
    cfg, in_dict, make_prior = _setup(name)(name, assets)
    Oracle = oracle_for(cfg)
    template = Oracle(copy.deepcopy(cfg), assets, mt_model=make_prior('cpu')).init_data(copy.deepcopy(in_dict))
    ora_e = Oracle(copy.deepcopy(cfg), assets, mt_model=make_prior('cpu'))
    data_e = ora_e.init_data(copy.deepcopy(in_dict))
    run = _emu_runner(ora_e, data_e)
    run.set_stage([], {}, 'init')
    run.backward()
    P, T, J = run.comp.P, run.comp.T, run.comp.J
    recs = []
    for stage, specs in cfg.opt_stage_specs.items():
        run.set_stage(specs['opt_variables'], specs['loss_cfg'], stage)
        for point in ('first', 'stepped'):
            if point == 'stepped':
                for _ in range(specs['opt_niters']):
                    run.backward()
                    run.step(specs['opt_lr'])
            for what in FILLED:
                run.buffer(what).fill_(float('nan'))
            run.backward()
            cand = split_buffers(lambda w: run.buffer(w).clone(), P, T, J)
            r = _record(stage, point, specs, cand, _snapshot(data_e), run.layout, run.theta.clone(), run.comp, run.pb.cam_mode)
            add_references(r, Oracle, cfg, assets, template)
            recs.append(r)
        cam = run.buffer(L.R_CAM_POSE).view(T, 3, 4)
        data_e['cam_pose'] = torch.cat([cam, torch.tensor([0., 0., 0., 1.]).expand(T, 1, 4)], dim=1).clone()
    return recs


_EMU_CACHE = {}


@pytest.fixture(scope='module')
def emu(smpl_assets):
    def get(name):
        if name not in _EMU_CACHE:
            _EMU_CACHE[name] = emulator_outputs(name, smpl_assets)
        return _EMU_CACHE[name]
    return get


@pytest.mark.parametrize('name', EMU_CASES)
def test_host_emulator_outputs_within_the_bound(name, emu):
    """a second legitimate float32 implementation (sequential scans, its own rounding) passes the bound and the exact rules at
    every stage, before and after the stage's Adam steps"""
    check_records(name, emu(name))


# ------------------------------------------------------------------------------------------------ CPU: modelled bugs
def _main_first(recs):
    return [r for r in recs if r['point'] == 'first'][-1]


def _rejection(what, r, mutate, family):
    """assert that the bound or the exact rules reject the emulator's outputs changed by mutate(cand) (in place); print the
    factor by which `family` fails the bound"""
    cand = copy.deepcopy(r['cand'])
    mutate(cand)
    msgs, rep = check_bound(what, cand, r)
    exact = check_exact(what, cand, r)
    assert msgs or exact, f'{what}: not rejected'
    ratio = max(x[3] for x in rep if x[0].split(' ')[-1].startswith(family))
    print(f'{what}: rejected, worst |o-o64|/bound of {family} {ratio:.3g}' + (' (and by the exact rules)' if exact else ''))
    assert ratio > 1 or exact


def _vis(r, p):
    return np.asarray(list(r['state']['person_data'].values())[p]['vis_frames'], bool)


def _lost_carry(r):
    """world x / y of person 0's frame at its 512-frame scan edge taken from its predecessor"""
    s, n = r['starts'][0], r['lens'][0]
    assert n > SCAN_CHUNK
    t = s + SCAN_CHUNK

    def mutate(cand):
        cand['persons'][0]['trans_world'][t, :2] = cand['persons'][0]['trans_world'][t - 1, :2]
    return mutate


def _edge_orientation(r, last):
    def mutate(cand):
        for p, (s, n) in enumerate(zip(r['starts'], r['lens'])):
            ow = cand['persons'][p]['orient_world']
            if last:
                ow[s + n - 1] = ow[s + n - 2]
            else:
                ow[s] = ow[s + 1]
    return mutate


def _previous_camera(r):
    """orient_ciw / trans_ciw of one frame of person 0 (the middle of its exist range) from the camera of the frame before"""
    s, n = r['starts'][0], r['lens'][0]
    t = s + n // 2

    def mutate(cand):
        from scipy.spatial.transform import Rotation
        cam = cand['cam_pose'][t - 1].astype(np.float64).reshape(3, 4)
        d = cand['persons'][0]
        Rw = rodrigues64(d['orient_world'][t:t + 1]).reshape(3, 3)
        d['orient_ciw'][t] = Rotation.from_matrix(cam[:, :3] @ Rw).as_rotvec()
        d['trans_ciw'][t] = cam[:, :3] @ d['trans_world'][t].astype(np.float64) + cam[:, 3]
    return mutate


def _invisible_kp(r):
    """one kp_2d_pred coordinate of a frame inside a person's exist range where it is invisible, which no term sees, moved by
    1e-4 of the person's largest coordinate.  (Scaling it by 1 + 1e-4 would not move it: the projection of an invisible frame
    is exactly 0 in both references and in the emulator, its intrinsics being 0.)"""
    p, t = next((p, t) for p, (s, n) in enumerate(zip(r['starts'], r['lens'])) for t in range(s, s + n) if not _vis(r, p)[t])
    peak = float(np.abs(r['o64']['persons'][p]['kp_pred']).max())

    def mutate(cand):
        cand['persons'][p]['kp_pred'][t, 0] += 1e-4 * peak
    return mutate


def _codec_off_by_one(r):
    """the base orientation of the first frame after each exist range from the codec (the last codec frame's) instead of
    orient_base_init"""
    T = len(r['cand']['cam_pose'])

    def mutate(cand):
        for p, (s, n) in enumerate(zip(r['starts'], r['lens'])):
            if s + n < T:
                ob = cand['persons'][p]['orient_base']
                ob[s + n] = ob[s + n - 1]
    return mutate


BUGS = {
    'lost_scan_carry': ('dynamic_p1_t1025', _lost_carry, 'trans_world'),
    'first_frame_orientation': ('static_multi_p3_t1100_gaps', lambda r: _edge_orientation(r, False), 'orient_world'),
    'last_frame_orientation': ('static_multi_p3_t1100_gaps', lambda r: _edge_orientation(r, True), 'orient_world'),
    'previous_camera': ('dynamic_p1_t1025', _previous_camera, 'orient_ciw'),
    'previous_camera_from_persons': (EMU_P2C, _previous_camera, 'orient_ciw'),
    'invisible_kp_moved': ('static_multi_p3_t1100_gaps', _invisible_kp, 'kp_pred'),
    'codec_range_off_by_one': ('static_multi_p3_t1100_gaps', _codec_off_by_one, 'orient_base'),
}


@pytest.mark.parametrize('bug', list(BUGS))
def test_bound_rejects_a_modelled_bug(bug, emu):
    name, make, family = BUGS[bug]
    r = _main_first(emu(name))
    _rejection(f'{name} {bug}', r, make(r), family)


# ------------------------------------------------------------------------------------------------ GPU
def _fill_nan(model):
    """NaN into every checked R_* buffer, through the pointers glamr_opt_read returns"""
    from glamr_b200.recon import _device_view
    torch.cuda.synchronize()
    for what in FILLED:
        p, n = ctypes.c_void_p(), ctypes.c_size_t()
        L.check(model._lib.glamr_opt_read(model._opt, what, ctypes.byref(p), ctypes.byref(n)), 'glamr_opt_read')
        _device_view(p.value, n.value, torch.device(DEV)).fill_(float('nan'))
    torch.cuda.synchronize()


def gpu_outputs(name, assets):
    """the CUDA path's outputs at the first closure of every stage and after its Adam steps (the check points of
    test_grad_float64.gpu_run), each from buffers filled with NaN before the closure; then forward() at the last check point's
    variables -> (records, (data dict outputs after forward, R_* buffers after forward))"""
    cfg, in_dict, make_prior = _setup(name)(name, assets)
    model = _make_model(cfg, assets, make_prior(DEV))
    data = _init(model, in_dict)
    comp = model._comp
    P, T, J = comp.P, comp.T, comp.J
    read = lambda w: model._read(w, -1).cpu()
    recs, stages = [], list(cfg.opt_stage_specs.items())
    for stage, specs in stages:
        variables = specs['opt_variables']
        model._cur_vars, model._cur_stage, model._loss_cfg = variables, stage, specs['loss_cfg']
        model._set_stage(data, variables, specs['loss_cfg'], stage, reset_adam=True, begin=True)
        for point in ('first', 'stepped'):
            if point == 'stepped':
                model.optimize_main(data, variables, specs['opt_lr'], specs['opt_niters'], specs['loss_cfg'], {'stage': stage})
                model._set_stage(data, variables, specs['loss_cfg'], stage, reset_adam=False)
            _fill_nan(model)
            _closure(model)
            recs.append(_record(stage, point, specs, split_buffers(read, P, T, J), _snapshot(data), model._layout,
                                model._theta.detach().cpu().clone(), comp, model._pb.cam_mode))
        if stage == stages[-1][0]:
            model.forward(data, variables, {'stage': stage})
            torch.cuda.synchronize()
            public = (data_outputs(data), split_buffers(read, P, T, J))
        if specs.get('reinitialize_cam', False):
            from glamr_b200 import geometry as G
            data['cam_pose'][:] = data['cam_pose'][[0]]
            data['cam_pose_inv'] = G.inverse_transform(data['cam_pose'])
    del model
    torch.cuda.empty_cache()
    Oracle = oracle_for(cfg)
    template = Oracle(copy.deepcopy(cfg), assets, mt_model=make_prior('cpu')).init_data(copy.deepcopy(in_dict))
    for r in recs:
        add_references(r, Oracle, cfg, assets, template)
    return recs, public


def check_public(name, recs, public):
    """forward() copies the R_* buffers into the data dict bit for bit (traj_local on the exist frames), and evaluates the same
    outputs as the last check point's closure at the same variables, so they pass the same bound"""
    got, bufs = public
    r = recs[-1]
    msgs = []
    for fam in CAMERA:
        if not np.array_equal(got[fam], bufs[fam].astype(np.float64)):
            msgs.append(f'{name} forward: data[{fam!r}] differs from {BUFFER_NAME[CAMERA[fam]]}')
    for p, (s, n) in enumerate(zip(r['starts'], r['lens'])):
        for fam, (what, key, _) in PERSON_OUT.items():
            buf = bufs['persons'][p][fam]
            if fam == 'traj_local':
                if not r['codec']:                  # without the codec forward() leaves traj_local out of the data dict
                    continue
                buf = buf[s:s + n]
            if not np.array_equal(got['persons'][p][fam], buf.astype(np.float64)):
                msgs.append(f'{name} forward: {key} of person {p} differs from {BUFFER_NAME[what]}')
    for fam in CAMERA:
        if not np.array_equal(bufs[fam], r['cand'][fam]):
            msgs.append(f'{name} forward: {fam} differs from the closure at the same variables')
    for p in range(len(r['starts'])):
        for fam in PERSON_OUT:
            if not np.array_equal(bufs['persons'][p][fam], r['cand']['persons'][p][fam]):
                msgs.append(f'{name} forward: {fam} of person {p} differs from the closure at the same variables')
    assert not msgs, '\n'.join(msgs)
    m, _ = check_bound(f'{name} forward', bufs, r)
    assert not m, '\n'.join(m)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ALL)
def test_gpu_outputs_within_float64_bound(name, smpl_assets):
    """every output element at the first closure of every stage and after the stage's Adam steps: written, within the bound,
    the exact rules; and forward()'s data dict"""
    recs, public = gpu_outputs(name, smpl_assets)
    check_records(name, recs)
    check_public(name, recs, public)
