"""The optimiser's analytic gradients against float64 autograd, element by element.

Every iteration of the optimiser is a hand-written backward (frame_residuals_kernel, camera_backward / scatter,
traj_cam_backward_kernel with its three CTA-wide reverse prefix scans) followed by Adam.  Here each gradient element is
compared with torch autograd through the full-LBS oracle in float64 (g64), with the same autograd in float32 (g32) as the
yardstick of what a legitimate float32 implementation deviates by:

    |g[e] - g64[e]|  <=  C_NOISE * D_V(b(e))  +  C_ULP * 2^-24 * |g64[e]|
    D_V(b) = max(max_{e in b} |g32[e] - g64[e]|,  FLOOR * max_V |g64|)

b(e) is the element's block of BLOCK consecutive frames (rows) of its variable; per-person scalars (traj_local_xy,
traj_local_heading) and the fixed camera are one block.  Where g64 and g32 are both exactly zero the gradient must be exactly
zero, and so must every variable autograd never reaches.  Unlike a max-normalised comparison, a frame whose gradient is far
below the variable's peak (outside an exist range, in an occlusion gap, past a scan-chunk edge) is held to its own noise.

FLOOR: |g32 - g64| can vanish by coincidence in a block (e.g. a block whose float32 sums happen to round exactly); 2^-20 of
the variable's peak is 16 float32 roundings of its largest element, below any per-frame term a kernel could lose and
above the re-association noise of a float32 sum of a few dozen terms of that size.  C_NOISE = 4, C_ULP = 8: on one H100
80GB HBM3 (700 W limit) the worst |cuda - g64| over every case, variable and check point was 0.58 of this bound
(dynamic_p1_t1025, traj_local_rot), 0.37-0.58 per case.  The prefix-sum variables
and the terms sit far lower (scanned variables <= 0.29, terms <= 0.09), their bounds being set by the floors below, which
rest on the host emulator's sequential float32 scans.  GLAMR_GRAD_REPORT=<file> writes the worst |g - g64| of every case and
variable next to its bound.  The CPU tests below show that a second
legitimate float32 implementation (the host-compiled frame functions) passes and that modelled kernel bugs do not.

Cases: the golden shapes (ReplayMT replays the recorded prior) and new shapes past the 512-frame chunks of
block_scan_inplace (glamr_b200/csrc/block_scan.cuh) with a seeded SyntheticPrior on each side.  The new cases optimise every
per-frame local variable in their last stage (local_dheading, local_dxy, local_z) with cam_fix_frames [[0, 16]], so the
reverse heading scan reaches per-frame rows past its chunk edges."""
import copy
import os

import numpy as np
import pytest
import torch

from helpers import ReplayMT, case_setup
from traj_variable_cases import cfg_path

EPS32 = 2.0 ** -24
BLOCK = 32
C_NOISE, C_ULP, FLOOR = 4.0, 8.0, 2.0 ** -20
# a term whose value is ~0 (e.g. cam_traj_rot of a camera that matches the persons) is a mean of squared differences of
# float32 quantities of magnitude ~1, each difference carrying ~2^-24 of rounding: its float32 value is noise of
# (2^-24)^2 x (number of terms, up to ~1e5) ~ 4e-10
TERM_ATOL = 1e-9
# traj_local_xy / _heading / _dxy / _dheading are (reverse) prefix sums over the person's n exist frames.  torch's float32
# cumsum accumulates in float64 on the CPU, so g32 does not show the rounding of a float32 scan: one rounding per addition,
# ~sqrt(n) of the largest partial sum as a random walk.  The floor allows 4 of those: 2^-22 sqrt(n) times the largest partial
# sum, which is max_V |g64| for the per-frame rows and, for traj_local_xy (the scan's total, which can be far smaller than its
# partial sums), the largest row of traj_local_dxy's gradient (taken whether or not the stage optimises it).  A plain
# sequential float32 loop (the host emulator) was measured at up to 2.3 (1 x 1025, traj_local_xy after 4 Adam steps)
SCANNED = {'traj_local_xy', 'traj_local_heading', 'traj_local_dxy', 'traj_local_dheading'}
SCAN_FLOOR = 2.0 ** -22
# the same scans place the trajectory every term is evaluated on: a sequential float32 scan moved cam_traj_rot by 7.4e-6
# relative (host emulator, 1 x 1025 after 4 Adam steps) where float64-accumulating torch moved it by 1e-7
TERM_SCAN_REL = 2.0 ** -16
SCAN_CHUNK = 512                # kScanThreads: elements per chunk of block_scan_inplace
CAM_FIX_ROWS = 16               # cam_fix_frames [[0, 16]] of the new cases: dheading rows 0-15 (exist frames 1-16) are masked
NITERS = 4                      # Adam steps per stage before the second check point
DEV = 'cuda:0'
WHOLE = {'traj_local_xy', 'traj_local_heading', 'cam_rot_6d_fix', 'cam_trans_fix'}
PERSON_VARS = ['traj_local_xy', 'traj_local_heading', 'traj_local_dxy', 'traj_local_dheading', 'traj_local_z', 'traj_local_rot',
               'smpl_orient_world_res', 'root_trans_world_res', 'world_dheading', 'world_dxy', 'person2cam_res_rot',
               'person2cam_res_trans']
GLOBAL_ROWS = {'smpl_orient_world_res', 'root_trans_world_res', 'world_dheading', 'world_dxy'}   # rows are frames t of the sequence

GOLDEN = ['dynamic_p1_t300', 'static_multi_p4_t300', '3dpw_p1_t600_gaps']
# name -> (config, T, [(first exist frame, exist length, visibility gap relative to the start or None)])
SYNTHETIC = {
    # three scan chunks, the last holding one element
    'dynamic_p1_t1025': ('glamr_dynamic', 1025, [(0, 1025, None)]),
    # exist lengths around one chunk on strict sub-ranges; frame 512 and 1024 of the sequence fall inside the tracks
    'static_multi_p3_t1100_gaps': ('glamr_static_multi', 1100, [(300, 511, (150, 170)), (500, 512, (200, 230)), (580, 513, (300, 310))]),
    # fixed camera: reduce_tail's float64 sum over T
    'static_p1_t1024': ('glamr_static', 1024, [(0, 1024, None)]),
    # heading vectors and world_dxy past one chunk
    'vec_dxy_p2_t600_gaps': (cfg_path('glamr_static_multi_vec_world_dxy'), 600, [(0, 600, (200, 230)), (45, 530, (100, 120))]),
}
ALL = GOLDEN + list(SYNTHETIC)
EMU_CASES = ['dynamic_p1_t1025', 'static_multi_p3_t1100_gaps']


# ------------------------------------------------------------------------------------------------ cases
def _is_vec(cfg):
    return cfg.grecon_model_specs.get('heading_type', 'scalar') == 'vec'


def oracle_for(cfg):
    from oracle.global_opt import OracleGlobalRecon
    g = cfg.grecon_model_specs
    if _is_vec(cfg) or any('world_dxy' in st['opt_variables'] for st in cfg.opt_stage_specs.values()):
        from traj_variable_cases import oracle_class
        return oracle_class()
    if g.get('flag_traj_from_cam', False):
        import traj_source_cases
        return traj_source_cases.oracle_class()
    if g.get('flag_opt_person2cam_rot', False) or g.get('flag_opt_person2cam_trans', False):
        import person2cam_cases
        return person2cam_cases.oracle_class()
    return OracleGlobalRecon


def p2c_flags(model):
    """(flag_opt_person2cam_rot, flag_opt_person2cam_trans) of an oracle or GlobalReconOptimizer"""
    return (getattr(model, 'flag_opt_person2cam_rot', False), getattr(model, 'flag_opt_person2cam_trans', False))


def synthetic_in_dict(assets, name):
    from glamr_b200.synthetic import make_pose_dict
    _, T, tracks = SYNTHETIC[name]
    est = {}
    for p, (s, n, gap) in enumerate(tracks):
        vis = np.zeros(T)
        vis[s:s + n] = 1
        if gap is not None:
            vis[s + gap[0]:s + gap[1]] = 0
        est[p] = make_pose_dict(assets, p, T, seed=5, exist=vis)
    return {'est': est, 'gt': {}, 'gt_meta': {}, 'seq_name': name}


def case(name, assets):
    """-> (cfg, in_dict, prior factory(device))"""
    from glamr_b200.config import Config
    from glamr_b200.synthetic import SyntheticPrior
    if name in SYNTHETIC:
        cfg = Config(SYNTHETIC[name][0])
        cfg.grecon_model_specs['cam_fix_frames'] = [[0, CAM_FIX_ROWS]]
        last = list(cfg.opt_stage_specs.values())[-1]
        last['opt_variables'] = list(last['opt_variables']) + [v for v in ['local_dheading', 'local_dxy', 'local_z']
                                                                if v not in last['opt_variables']]
        in_dict = synthetic_in_dict(assets, name)
        make_prior = lambda dev: SyntheticPrior(seed=23, device=dev)
    else:
        gold, cfg, in_dict = case_setup(name, assets)
        make_prior = lambda dev: ReplayMT(gold, dev)
    for st in cfg.opt_stage_specs.values():
        st['opt_niters'] = NITERS
    return cfg, in_dict, make_prior


def param_order(opt_variables, P, fixed_cam, opt_traj=True, p2c=(False, False)):
    """(person or None, name) of every tensor get_parameter returns, in its order (global_recon_model.py:591-633); p2c: the
    person2cam flags (p2c_flags), a residual being returned when its flag is set and the stage lists it"""
    if 'cam' not in opt_variables:
        order = [(None, 'cam_inv_rot_residual'), (None, 'cam_inv_trans_residual')]
    elif fixed_cam:
        order = [(None, 'cam_rot_6d_fix'), (None, 'cam_trans_fix')]
    else:
        order = [(None, 'cam_rot_6d'), (None, 'cam_trans')]
    for p in range(P):
        if opt_traj:
            for key in opt_variables:
                if key == 'world_res':
                    order += [(p, 'smpl_orient_world_res'), (p, 'root_trans_world_res')]
                if 'local' in key:
                    order.append((p, f'traj_{key}'))
        for flag, key in zip(p2c, ('rot', 'trans')):
            if flag and f'person2cam_{key}' in opt_variables:
                order.append((p, f'person2cam_res_{key}'))
        if 'world_dheading' in opt_variables:
            order.append((p, 'world_dheading'))
        if 'world_dxy' in opt_variables:
            order.append((p, 'world_dxy'))
    return order


def view(lay, vec, p, name):
    return (lay.views(vec) if p is None else lay.views(vec, p))[name]


# ------------------------------------------------------------------------------------------------ oracle references
def oracle_state(template, src, lay, theta):
    """A copy of the oracle's data dict `template` holding the float32 state of `src` (the data dict of the CUDA path or of
    the host emulator): every floating tensor both hold, and every variable from the packed `theta`."""
    out = copy.deepcopy(template)
    th = theta.detach().cpu()
    for k in ['cam_pose', 'cam_pose_inv']:
        out[k] = torch.as_tensor(src[k]).detach().cpu().to(out[k].dtype).clone()
    gv = lay.views(th)
    for k in ['cam_inv_rot_residual', 'cam_inv_trans_residual']:
        out[k] = gv[k].clone()
    for p, (ds, do) in enumerate(zip(src['person_data'].values(), out['person_data'].values())):
        pv = lay.views(th, p)
        for k, v in ds.items():
            if k in PERSON_VARS or not (isinstance(v, torch.Tensor) and v.is_floating_point()):
                continue
            if isinstance(do.get(k), torch.Tensor) and tuple(do[k].shape) == tuple(v.shape):
                do[k] = v.detach().cpu().to(do[k].dtype).clone()
        for k in PERSON_VARS:
            if k in ds:
                do[k] = pv[k].clone()
    return out


def oracle_closure(Oracle, cfg, assets, state, specs, stage, lay, theta, dtype):
    """gradients (float64 numpy, None where autograd never reaches) and unweighted term values of one closure of the oracle in
    `dtype`, with every optimised variable set to its value in theta"""
    ora = Oracle(copy.deepcopy(cfg), assets)
    data = copy.deepcopy(state)
    if dtype == torch.float64:
        data = ora.to_float64(data)
    variables = specs['opt_variables']
    params = ora.get_parameter(data, variables)
    order = param_order(variables, len(data['person_data']), ora.flag_fixed_cam, ora.flag_opt_traj, p2c_flags(ora))
    assert len(order) == len(params)
    th = theta.detach().cpu()
    with torch.no_grad():
        for (p, name), prm in zip(order, params):
            prm.copy_(view(lay, th, p, name).reshape(prm.shape).to(prm.dtype))
    # traj_local_dxy's gradient rows are the partial sums of the reverse xy scan whose total is traj_local_xy's gradient: taken
    # even where the stage does not optimise it, as the scale of that scan's rounding (scan_scale)
    partial = [d['traj_local_dxy'] if 'traj_local_dxy' in d else None for d in data['person_data'].values()]
    for prm in params + [x for x in partial if x is not None]:
        prm.requires_grad_(True)
        prm.grad = None
    ora.forward(data, variables, {'stage': stage})
    total, _, uw = ora.compute_loss(data, specs['loss_cfg'])
    total.backward()
    grads = [None if prm.grad is None else prm.grad.detach().double().numpy().copy() for prm in params]
    scan_scale = [0.0 if x is None or x.grad is None or x.numel() == 0 else float(x.grad.abs().max()) for x in partial]
    return grads, {k: float(v) for k, v in uw.items()}, scan_scale


def references(Oracle, cfg, assets, state, specs, stage, lay, theta):
    g64, t64, scan_scale = oracle_closure(Oracle, cfg, assets, state, specs, stage, lay, theta, torch.float64)
    g32, t32, _ = oracle_closure(Oracle, cfg, assets, state, specs, stage, lay, theta, torch.float32)
    lens = [int(d['exist_len'].sum()) if torch.is_tensor(d['exist_len']) else int(d['exist_len']) for d in state['person_data'].values()]
    return {'g64': g64, 'g32': g32, 't64': t64, 't32': t32, 'lens': lens, 'scan_scale': scan_scale}


# ------------------------------------------------------------------------------------------------ the bound
def bound_of(name, g64, g32, n_scan=0, scan_scale=0.0):
    """per-element bound (same shape as g64) for variable `name`; n_scan: exist length of the person for the variables that
    are prefix sums over its exist frames, scan_scale: the largest partial sum of the person's xy scan"""
    g64, g32 = np.asarray(g64, np.float64), np.asarray(g32, np.float64)
    d = np.abs(g32 - g64)
    floor = FLOOR * float(np.abs(g64).max()) if g64.size else 0.0
    if name in SCANNED and g64.size:
        peak = max(float(np.abs(g64).max()), scan_scale if name == 'traj_local_xy' else 0.0)
        floor = max(floor, SCAN_FLOOR * np.sqrt(n_scan) * peak)
    if name in WHOLE or g64.ndim == 0 or g64.shape[0] <= 2:
        D = np.full(g64.shape, max(float(d.max()) if d.size else 0.0, floor))
    else:
        rows = d.reshape(d.shape[0], -1).max(axis=1)
        nb = (rows.size + BLOCK - 1) // BLOCK
        blk = np.zeros(nb * BLOCK)
        blk[:rows.size] = rows
        blk = np.maximum(blk.reshape(nb, BLOCK).max(axis=1), floor)
        D = np.repeat(blk, BLOCK)[:rows.size].reshape((-1,) + (1,) * (g64.ndim - 1)) * np.ones_like(g64)
    return C_NOISE * D + C_ULP * EPS32 * np.abs(g64)


def violations(name, g, g64, g32, n_scan=0, scan_scale=0.0):
    """-> (number of elements outside the bound, worst |g - g64| / bound, worst |g - g64|, bound there)"""
    g = np.asarray(g, np.float64).reshape(np.shape(g64))
    b = bound_of(name, g64, g32, n_scan, scan_scale)
    err = np.abs(g - np.asarray(g64))
    exact = (np.asarray(g64) == 0) & (np.asarray(g32) == 0)
    bad = (err > b) | (exact & (g != 0))
    with np.errstate(divide='ignore', invalid='ignore'):
        ratio = np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err > 0, np.inf, 0.0))
    i = int(np.argmax(ratio)) if ratio.size else 0
    return int(bad.sum()), (float(ratio.flat[i]) if ratio.size else 0.0), (float(err.flat[i]) if err.size else 0.0), \
        (float(b.flat[i]) if b.size else 0.0)


def check_grads(what, order, grads, ref, report=None):
    """every variable's gradient against the bound; grads[i] is the candidate of param i (array)"""
    msgs = []
    lens, scales = ref['lens'], ref['scan_scale']
    for i, ((p, name), g) in enumerate(zip(order, grads)):
        g = np.asarray(g, np.float64)
        g64, g32 = ref['g64'][i], ref['g32'][i]
        label = f'{what} {name}' + ('' if p is None else f'[{p}]')
        if g64 is None or g32 is None:
            assert g64 is None and g32 is None, label
            if g.size and float(np.abs(g).max()) != 0.0:
                msgs.append(f'{label}: autograd never reaches it, gradient max {np.abs(g).max():.3e}')
            continue
        n_bad, ratio, err, b = violations(name, g, g64, g32, 0 if p is None else lens[p], 0.0 if p is None else scales[p])
        if report is not None:
            report.append((label, err, b, ratio))
        if n_bad:
            msgs.append(f'{label}: {n_bad} elements outside the bound, worst |g-g64| {err:.3e} vs bound {b:.3e} (x{ratio:.2f})')
    assert not msgs, '\n'.join(msgs)


def check_terms(what, terms, ref, report=None):
    msgs = []
    for k, v64 in ref['t64'].items():
        v32, got = ref['t32'][k], terms[k]
        if not np.isfinite(v64):             # the reference's own value is undefined (kp_2d_dist without any visible joint)
            continue
        tol = C_NOISE * max(abs(v32 - v64), FLOOR * abs(v64), TERM_SCAN_REL * abs(v64)) + C_ULP * EPS32 * abs(v64) + TERM_ATOL
        err = abs(got - v64)
        if report is not None:
            report.append((f'{what} term {k}', err, tol, err / tol if tol > 0 else (0.0 if err == 0 else np.inf)))
        if not err <= tol and not (err == 0.0):
            msgs.append(f'{what} term {k}: {got!r} vs float64 {v64!r}: {err:.3e} > {tol:.3e}')
    assert not msgs, '\n'.join(msgs)


# ------------------------------------------------------------------------------------------------ CPU: host emulator
def _emu_runner(ora, data):
    if any(p2c_flags(ora)):
        from test_person2cam import _emu_runner as make
        return make(ora, data)
    if not hasattr(ora, 'heading_type'):
        from emu_runner import EmuRunner
        return EmuRunner(ora, data)
    from test_traj_variables import _emu_runner as make
    return make(ora, data)


def emulator_records(name, assets, setup=case):
    """the host-compiled frame functions (tests/emu_runner.py) from the oracle's float32 init: first closure of every stage
    and the closure after the stage's Adam steps, each with the oracle's float64 / float32 gradients at the same state (kept as
    r['state']); setup(name, assets) -> (cfg, in_dict, prior factory) of the case"""
    from glamr_b200 import lib as L
    cfg, in_dict, make_prior = setup(name, assets)
    Oracle = oracle_for(cfg)
    ora_t = Oracle(copy.deepcopy(cfg), assets, mt_model=make_prior('cpu'))
    template = ora_t.init_data(copy.deepcopy(in_dict))
    ora_e = Oracle(copy.deepcopy(cfg), assets, mt_model=make_prior('cpu'))
    data_e = ora_e.init_data(copy.deepcopy(in_dict))
    run = _emu_runner(ora_e, data_e)
    run.set_stage([], {}, 'init')
    run.backward()
    P, T = run.comp.P, run.comp.T
    recs = []
    for stage, specs in cfg.opt_stage_specs.items():
        variables = specs['opt_variables']
        order = param_order(variables, P, ora_e.flag_fixed_cam, ora_e.flag_opt_traj, p2c_flags(ora_e))
        run.set_stage(variables, specs['loss_cfg'], stage)
        for point in ('first', 'stepped'):
            if point == 'stepped':
                for _ in range(specs['opt_niters']):
                    run.backward()
                    run.step(specs['opt_lr'])
            grad, terms = run.backward()
            grad = grad.clone()
            state = oracle_state(template, data_e, run.layout, run.theta)
            ref = references(Oracle, cfg, assets, state, specs, stage, run.layout, run.theta)
            recs.append({'stage': stage, 'point': point, 'order': order,
                         'grads': [view(run.layout, grad, p, n).numpy().astype(np.float64) for p, n in order],
                         'terms': {k: float(terms[L.TERM_INDEX[k]]) for k in specs['loss_cfg']}, 'ref': ref, 'state': state,
                         'specs': specs, 'layout': run.layout, 'theta': run.theta.clone(),
                         'starts': [int(d['fr_start']) for d in data_e['person_data'].values()],
                         'lens': [int(d['exist_len']) for d in data_e['person_data'].values()]})
        cam = run.buffer(L.R_CAM_POSE).view(T, 3, 4)
        data_e['cam_pose'] = torch.cat([cam, torch.tensor([0., 0., 0., 1.]).expand(T, 1, 4)], dim=1).clone()
    return recs


_EMU_CACHE = {}


@pytest.fixture(scope='module')
def emu(smpl_assets):
    def get(name):
        if name not in _EMU_CACHE:
            _EMU_CACHE[name] = emulator_records(name, smpl_assets)
        return _EMU_CACHE[name]
    return get


@pytest.mark.parametrize('name', EMU_CASES)
def test_host_emulator_gradients_within_the_bound(name, emu):
    """a second legitimate float32 implementation (host-compiled frame functions, its own rounding) passes the bound at every
    stage, before and after the stage's Adam steps"""
    for r in emu(name):
        what = f'{name} {r["stage"]} {r["point"]}'
        check_grads(what, r['order'], r['grads'], r['ref'])
        check_terms(what, r['terms'], r['ref'])


# ------------------------------------------------------------------------------------------------ CPU: modelled bugs
def _frame_rows(name, t, start, ln):
    """row of variable `name` that holds frame t of the sequence (person with exist range [start, start + ln)), or None"""
    i = t - start
    if name in GLOBAL_ROWS:
        return t
    if name in ('traj_local_z', 'traj_local_rot'):
        return i if 0 <= i < ln else None
    if name in ('traj_local_dxy', 'traj_local_dheading'):
        return i - 1 if 1 <= i < ln else None
    return None


def _rejected(r, mutate):
    """True when the bound rejects the float32 autograd gradient changed by mutate(person, name, array) (in place)"""
    grads = []
    for (p, name), g32 in zip(r['order'], r['ref']['g32']):
        g = None if g32 is None else np.array(g32, np.float64)
        if g is not None and p is not None:
            mutate(p, name, g)
        grads.append(np.zeros(0) if g is None else g)
    try:
        check_grads('modelled bug', r['order'], grads, r['ref'])
    except AssertionError:
        return True
    return False


def _main_first(records):
    return [r for r in records if r['point'] == 'first'][-1]


def _edges(ln):
    """exist-local frames at a chunk edge of the forward (i = 512 k) and reverse (i = ln - 1 - 512 k) scans"""
    e = set()
    for k in range(1, (ln - 1) // SCAN_CHUNK + 1):
        e.update({SCAN_CHUNK * k, ln - 1 - SCAN_CHUNK * k, SCAN_CHUNK * k - 1, ln - SCAN_CHUNK * k})
    return sorted(i for i in e if 0 <= i < ln)


def _drop_frame(t, person, start, ln, only):
    """frame t of `person` dropped from every per-frame variable (only=None) or from variable `only` alone"""
    def mutate(p, name, g):
        if p == person and name not in WHOLE and only in (None, name):
            row = _frame_rows(name, t, start, ln)
            if row is not None:
                g[row] = 0.0
    return mutate


def _swap_frames(t, person, start, ln, only):
    """frames t - 1 and t of `person` swapped in every per-frame variable (only=None) or in variable `only` alone"""
    def mutate(p, name, g):
        if p == person and name not in WHOLE and only in (None, name):
            a, b = _frame_rows(name, t - 1, start, ln), _frame_rows(name, t, start, ln)
            if a is not None and b is not None:
                g[[a, b]] = g[[b, a]]
    return mutate


def _unmasked(only, i):
    """does exist frame i have a row in variable `only` (every per-frame variable: None) that the loss reaches?"""
    if only is None:
        return True
    return i >= 1 and not (only == 'traj_local_dheading' and i <= CAM_FIX_ROWS)


# every per-frame variable at once, then each output of the reverse scans on its own (their bound carries SCAN_FLOOR)
ONLY = [None, 'traj_local_dxy', 'traj_local_dheading']


@pytest.mark.parametrize('only', ONLY, ids=['all', 'dxy', 'dheading'])
@pytest.mark.parametrize('name', EMU_CASES)
def test_bound_rejects_a_frame_dropped_at_every_chunk_edge(name, only, emu):
    r = _main_first(emu(name))
    for p, (s, ln) in enumerate(zip(r['starts'], r['lens'])):
        for i in _edges(ln) + [SCAN_CHUNK]:
            if i < ln and _unmasked(only, i):
                assert _rejected(r, _drop_frame(s + i, p, s, ln, only)), \
                    f'person {p}: frame {s + i} (exist frame {i}) dropped from {only or "every variable"} is not rejected'


@pytest.mark.parametrize('only', ONLY, ids=['all', 'dxy', 'dheading'])
@pytest.mark.parametrize('name', EMU_CASES)
def test_bound_rejects_the_first_or_last_exist_frame_dropped(name, only, emu):
    r = _main_first(emu(name))
    for p, (s, ln) in enumerate(zip(r['starts'], r['lens'])):
        # the scanned variables have no row for exist frame 0; cam_fix_frames masks the first dheading rows
        i0 = min(i for i in range(ln) if _unmasked(only, i))
        for t in (s + i0, s + ln - 1):
            assert _rejected(r, _drop_frame(t, p, s, ln, only)), f'person {p}: frame {t} dropped from {only or "every variable"} is not rejected'


@pytest.mark.parametrize('only', ONLY, ids=['all', 'dxy', 'dheading'])
@pytest.mark.parametrize('name', EMU_CASES)
def test_bound_rejects_two_frames_swapped_across_a_chunk_edge(name, only, emu):
    r = _main_first(emu(name))
    checked = 0
    for p, (s, ln) in enumerate(zip(r['starts'], r['lens'])):
        # exist-local scan chunk edges, and frames 512 / 1024 of the sequence (the camera blocks of traj_cam_backward_kernel)
        for i in [SCAN_CHUNK, ln - SCAN_CHUNK, SCAN_CHUNK - s, 2 * SCAN_CHUNK - s]:
            if not (1 < i < ln - 1 and _unmasked(only, i - 1)):
                continue
            assert _rejected(r, _swap_frames(s + i, p, s, ln, only)), \
                f'person {p}: exist frames {i - 1} and {i} swapped in {only or "every variable"} is not rejected'
            checked += 1
    assert checked


@pytest.mark.parametrize('sign', [-1.0, 1.0], ids=['lost', 'duplicated'])
def test_bound_rejects_a_lost_or_duplicated_scan_carry(sign, emu):
    """traj_local_dheading (scalar heading) is a reverse prefix sum over the exist frames: the total of the chunk of the 512
    last frames missing from (lost carry) or added twice to (duplicated carry) every frame before it"""
    r = _main_first(emu('dynamic_p1_t1025'))
    ln = r['lens'][0]
    first = ln - SCAN_CHUNK                       # exist frame where the reverse scan's first chunk begins
    k = [n for _, n in r['order']].index('traj_local_dheading')
    total = float(r['ref']['g32'][k][first - 1])  # row first - 1 holds exist frame `first`: the chunk's inclusive sum

    def mutate(p, name, g):
        if name == 'traj_local_dheading':
            g[:first - 1] += sign * total
    assert abs(total) > 0
    assert _rejected(r, mutate)


@pytest.mark.parametrize('name', EMU_CASES)
def test_bound_rejects_one_element_scaled_by_1e_4(name, emu):
    """the element of median magnitude of the per-frame variable with the largest median |g64|, scaled by 1 + 1e-4"""
    r = _main_first(emu(name))
    meds = [(float(np.median(np.abs(g))) if g is not None and g.shape[0] > 2 else -1.0, i) for i, g in enumerate(r['ref']['g64'])]
    _, k = max(meds)
    g64 = np.abs(r['ref']['g64'][k]).ravel()
    nz = np.where(g64 > 0)[0]
    e = int(nz[np.argsort(g64[nz])[nz.size // 2]])
    target = r['order'][k]

    def mutate(p, name, g):
        if (p, name) == target:
            g.flat[e] *= 1.0 + 1e-4
    assert _rejected(r, mutate), f'{target} element {e} (|g64| {g64[e]:.3e}) scaled by 1 + 1e-4 is not rejected'


def test_bound_accepts_the_float32_reference_itself(emu):
    """sanity of the construction: g32 itself is inside its own bound"""
    r = _main_first(emu('dynamic_p1_t1025'))
    assert not _rejected(r, lambda p, name, g: None)


# ------------------------------------------------------------------------------------------------ GPU
def _make_model(cfg, assets, mt, rank_range=None):
    """GlobalReconOptimizer on cuda:0; rank_range (rank, (n_begin, n_end)): this instance evaluates only that frame-person range,
    as rank `rank` of a sharded run (world stays 1: no collective)"""
    from glamr_b200.recon import GlobalReconOptimizer
    model = GlobalReconOptimizer(copy.deepcopy(cfg), torch.device(DEV), None, smpl=assets, mt_model=mt)
    if rank_range is not None:
        orig = model._attach

        def attach(data):
            orig(data)
            model.rank, model._n_range = rank_range[0], tuple(rank_range[1])
        model._attach = attach
    return model


def _init(model, in_dict):
    return model.init_data(copy.deepcopy(in_dict))


def _closure(model):
    """-> (packed gradient, term sums (un-normalised, float32), unweighted term values) of one evaluation at the current theta"""
    from glamr_b200 import lib as L
    model._backward()
    with torch.cuda.device(DEV):
        L.check(model._lib.glamr_opt_losses(model._opt, L.ptr(model._reduce), L.ptr(model._terms), L.stream_ptr()), 'glamr_opt_losses')
    torch.cuda.synchronize()
    return model._reduce.clone(), model._terms.cpu().clone()


def _snapshot(data):
    """float32 host copy of the data dict entries oracle_state reads"""
    out = {'cam_pose': data['cam_pose'].detach().cpu().clone(), 'cam_pose_inv': data['cam_pose_inv'].detach().cpu().clone(), 'person_data': {}}
    for pid, d in data['person_data'].items():
        out['person_data'][pid] = {k: (v.detach().cpu().clone() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}
    return out


def gpu_run(name, assets, setup=case):
    """first closure of every stage and the closure after its Adam steps on the CUDA path: packed gradients, term values,
    theta and the state the oracle needs"""
    from glamr_b200 import lib as L
    cfg, in_dict, make_prior = setup(name, assets)
    model = _make_model(cfg, assets, make_prior(DEV))
    data = _init(model, in_dict)
    P = len(data['person_data'])
    recs = []
    for stage, specs in cfg.opt_stage_specs.items():
        variables = specs['opt_variables']
        model._cur_vars, model._cur_stage, model._loss_cfg = variables, stage, specs['loss_cfg']
        model._set_stage(data, variables, specs['loss_cfg'], stage, reset_adam=True, begin=True)
        for point in ('first', 'stepped'):
            if point == 'stepped':
                model.optimize_main(data, variables, specs['opt_lr'], specs['opt_niters'], specs['loss_cfg'], {'stage': stage})
                model._set_stage(data, variables, specs['loss_cfg'], stage, reset_adam=False)
            grad, terms = _closure(model)
            recs.append({'stage': stage, 'point': point, 'specs': specs,
                         'order': param_order(variables, P, model.flag_fixed_cam, model.flag_opt_traj, p2c_flags(model)),
                         'grad': grad[:model._layout.n_params].cpu(), 'sums': grad[model._layout.n_params:].cpu(),
                         'terms': {k: float(terms[L.TERM_INDEX[k]]) for k in specs['loss_cfg']},
                         'theta': model._theta.detach().cpu().clone(), 'state': _snapshot(data)})
        if specs.get('reinitialize_cam', False):
            from glamr_b200 import geometry as G
            data['cam_pose'][:] = data['cam_pose'][[0]]
            data['cam_pose_inv'] = G.inverse_transform(data['cam_pose'])
    return model, cfg, recs


def _references_of(name, cfg, assets, lay, recs, template=None, setup=case):
    """the oracle's float64 / float32 references at the theta and state of each record (r['ref']), and the record's gradient
    split into its variables (r['grads']); -> the oracle's init data, re-usable as `template`"""
    _, in_dict, make_prior = setup(name, assets)
    Oracle = oracle_for(cfg)
    if template is None:
        template = Oracle(copy.deepcopy(cfg), assets, mt_model=make_prior('cpu')).init_data(copy.deepcopy(in_dict))
    for r in recs:
        if 'ref' not in r:
            state = oracle_state(template, r['state'], lay, r['theta'])
            r['ref'] = references(Oracle, cfg, assets, state, r['specs'], r['stage'], lay, r['theta'])
        r['grads'] = [view(lay, r['grad'], p, n).numpy().astype(np.float64) for p, n in r['order']]
    return template


_GPU_CACHE = {}


@pytest.fixture(scope='module')
def gpu_refs(smpl_assets):
    """per case: the default-path run with the oracle's float64 / float32 references at each of its check points"""
    def get(name):
        if name not in _GPU_CACHE:
            model, cfg, recs = gpu_run(name, smpl_assets)
            lay = model._layout
            template = _references_of(name, cfg, smpl_assets, lay, recs)
            _GPU_CACHE[name] = (lay, cfg, recs, template)
            del model
            torch.cuda.empty_cache()
        return _GPU_CACHE[name]
    return get


REPORT = os.environ.get('GLAMR_GRAD_REPORT')      # file to append the per-variable worst |g - g64| and bound to


def _report(lines):
    if REPORT:
        with open(REPORT, 'a') as f:
            for label, err, b, ratio in lines:
                f.write(f'{label}\t{err:.3e}\t{b:.3e}\t{ratio:.3f}\n')


def _check_records(name, recs, tag=''):
    rep, msgs = [], []
    for r in recs:
        what = f'{name}{tag} {r["stage"]} {r["point"]}'
        for fn, args in ((check_grads, (what, r['order'], r['grads'], r['ref'], rep)), (check_terms, (what, r['terms'], r['ref'], rep))):
            try:
                fn(*args)
            except AssertionError as e:
                msgs.append(str(e))
    _report(rep)
    worst = max(rep, key=lambda x: x[3])
    print(f'{name}{tag}: worst |g-g64|/bound {worst[3]:.3f} at {worst[0]} ({worst[1]:.3e} vs {worst[2]:.3e})')
    assert not msgs, '\n'.join(msgs)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ALL)
def test_gpu_gradients_within_float64_bound(name, gpu_refs):
    """default iteration path: every variable's gradient and every term value at the first closure of every stage and after
    the stage's Adam steps"""
    _check_records(name, gpu_refs(name)[2])


SPLITS = {'dynamic_p1_t1025': [512],                    # inside the person, at its exist frame 512
          'static_multi_p3_t1100_gaps': [1100, 2200]}   # at person boundaries


def _sharded_closure(models):
    red = []
    for m in models:
        m._backward()
        red.append(m._reduce.clone())
    torch.cuda.synchronize()
    return red


def _centred_on(center, ref):
    """a reference whose float64 gradient is `center` and whose float32 noise |g32 - g64| is that of `ref`: bounds a candidate
    against another evaluation at the same theta (variables autograd never reaches stay None)"""
    g64 = [None if b is None else a for a, b in zip(center, ref['g64'])]
    g32 = [None if b is None else a + (np.asarray(c) - np.asarray(b)) for a, b, c in zip(center, ref['g64'], ref['g32'])]
    return {'g64': g64, 'g32': g32, 'lens': ref['lens'], 'scan_scale': ref['scan_scale']}


@pytest.mark.gpu
@pytest.mark.parametrize('name,split', [(n, s) for n, ss in SPLITS.items() for s in ss])
def test_gpu_two_ranks_on_one_gpu(name, split, gpu_refs, smpl_assets):
    """two GlobalReconOptimizers own the frame-persons [0, split) and [split, P T) as ranks 0 and 1 (pointer offsets of the
    per-frame kernels, the blend and skinning on [n_begin, n_end), `owner`): the host sum of their reduce buffers passes the
    float64 bound at the first closure of the first stage.  Then Adam steps driven by that sum (apply on both with the summed
    buffer, as the NCCL all-reduce would); the summed gradient after them matches a single-range evaluation at the same
    theta, within the bound with the float32 noise of the default run's own stepped closure."""
    from glamr_b200 import lib as L
    lay, cfg, recs, _ = gpu_refs(name)
    _, in_dict, make_prior = case(name, smpl_assets)
    N = recs[0]['state']['cam_pose'].shape[0] * len(recs[0]['state']['person_data'])
    models = [_make_model(cfg, smpl_assets, make_prior(DEV), rank_range=(r, rng)) for r, rng in enumerate([(0, split), (split, N)])]
    datas = [_init(m, in_dict) for m in models]
    stage, specs = list(cfg.opt_stage_specs.items())[0]
    variables = specs['opt_variables']
    for m, d in zip(models, datas):
        assert m._n_range in ((0, split), (split, N))
        m._cur_vars, m._cur_stage, m._loss_cfg = variables, stage, specs['loss_cfg']
        m._set_stage(d, variables, specs['loss_cfg'], stage, reset_adam=True, begin=True)
    red = _sharded_closure(models)
    n = lay.n_params
    first, stepped = recs[0], recs[1]
    order = first['order']
    split_grads = lambda red: [view(lay, (red[0].double() + red[1].double()).cpu()[:n], p, k).numpy() for p, k in order]
    assert torch.equal(models[0]._theta.cpu(), first['theta'])
    check_grads(f'{name} split {split} first', order, split_grads(red), first['ref'])
    hist = torch.zeros(L.NUM_TERMS + 1, device=DEV)
    for _ in range(specs['opt_niters']):
        summed = red[0] + red[1]
        for m in models:
            with torch.cuda.device(DEV):
                L.check(m._lib.glamr_opt_apply(m._opt, L.ptr(m._theta), L.ptr(summed), float(specs['opt_lr']), L.ptr(hist), 0,
                                               L.stream_ptr()), 'glamr_opt_apply')
        red = _sharded_closure(models)
    assert torch.equal(models[0]._theta, models[1]._theta)
    single = _make_model(cfg, smpl_assets, make_prior(DEV))
    d1 = _init(single, in_dict)
    single._cur_vars, single._cur_stage, single._loss_cfg = variables, stage, specs['loss_cfg']
    single._set_stage(d1, variables, specs['loss_cfg'], stage, reset_adam=True, begin=True)
    single._theta.copy_(models[0]._theta)
    g1, _ = _closure(single)
    center = [view(lay, g1[:n].double().cpu(), p, k).numpy() for p, k in order]
    check_grads(f'{name} split {split} stepped vs single range', order, split_grads(red), _centred_on(center, stepped['ref']))


@pytest.mark.gpu
def test_gpu_changed_rank_range_re_primes_the_blend(smpl_assets):
    """glamr_opt_set_problem with a new [n_begin, n_end) and without the new-sequence bit: the next evaluation skins v_posed of
    the NEW range (re-primed blend), bit-identical to a handle that evaluated that range from the start"""
    name = 'dynamic_p1_t1025'
    cfg, in_dict, make_prior = case(name, smpl_assets)
    stage, specs = list(cfg.opt_stage_specs.items())[0]
    variables = specs['opt_variables']
    N = 1025
    fresh = _make_model(cfg, smpl_assets, make_prior(DEV), rank_range=(1, (512, N)))
    moved = _make_model(cfg, smpl_assets, make_prior(DEV))
    outs = []
    for m in (fresh, moved):
        d = _init(m, in_dict)
        m._cur_vars, m._cur_stage, m._loss_cfg = variables, stage, specs['loss_cfg']
        m._set_stage(d, variables, specs['loss_cfg'], stage, reset_adam=True, begin=True)
        if m is moved:
            _closure(m)                                  # primes the pipelined blend for [0, N)
            m.rank, m._n_range = 1, (512, N)
            m._set_stage(d, variables, specs['loss_cfg'], stage, reset_adam=False)
        outs.append(_closure(m)[0].cpu())
    assert torch.equal(outs[0], outs[1]), f'max |d| {float((outs[0] - outs[1]).abs().max()):.3e}'


def _dev_u8(addr, count):
    class _H:
        pass
    h = _H()
    h.__cuda_array_interface__ = {'shape': (count,), 'typestr': '|u1', 'data': (addr, False), 'version': 2}
    return torch.as_tensor(h, device=DEV)


HIST_ROWS = 64


class AdamProbe:
    """the optimiser state around one Adam step of a model: theta, moments, the gradient the step consumed and the device's
    step count, read from the loss-history row the step wrote (row = steps taken since the last reset)"""

    def __init__(self, model):
        from glamr_b200 import lib as L
        self.model, self.n = model, model._layout.n_params
        self.hist = torch.full((HIST_ROWS, L.NUM_TERMS + 1), float('nan'), device=DEV)

    def state(self):
        from glamr_b200 import lib as L
        m = self.model
        torch.cuda.synchronize()
        return (m._theta.cpu().clone(), m._read(L.R_ADAM_M, self.n).cpu(), m._read(L.R_ADAM_V, self.n).cpu())

    def step(self, lr, via_iterate):
        """one Adam step: via_iterate, one eager glamr_opt_iterate iteration (evaluation + apply_kernel); else glamr_opt_apply
        (apply_kernel) on the gradient already in the model's reduce buffer -> (before, after, g, device step)"""
        from glamr_b200 import lib as L
        m = self.model
        before = self.state()
        self.hist.fill_(float('nan'))
        with torch.cuda.device(DEV):
            if via_iterate:
                L.check(m._lib.glamr_opt_iterate(m._opt, L.ptr(m._theta), L.ptr(m._reduce), float(lr), L.ptr(self.hist), L.NUM_TERMS + 1,
                                                 1, 0, L.stream_ptr()), 'glamr_opt_iterate')
            else:
                L.check(m._lib.glamr_opt_apply(m._opt, L.ptr(m._theta), L.ptr(m._reduce), float(lr), L.ptr(self.hist), L.NUM_TERMS + 1,
                                               L.stream_ptr()), 'glamr_opt_apply')
        after = self.state()
        rows = (~torch.isnan(self.hist[:, 0])).nonzero().flatten().tolist()
        assert len(rows) == 1
        return before, after, m._reduce[:self.n].cpu().clone(), rows[0] + 1


def _ulp(x):
    return torch.from_numpy(np.spacing(np.abs(x.numpy()).astype(np.float32)).astype(np.float64))


def _check_adam_step(what, model, lr, before, after, g, step):
    """theta, m and v after one step vs torch.optim.Adam (betas 0.9 / 0.999, eps 1e-8) in float64 from the same gradient,
    moments and device step count: theta within 2 float32 ulp of |theta| + 2 of the step, m within 2 ulp of |m| + 2 of
    0.1 |g - m|, v within 2 ulp of |v| + 2 of 0.001 g^2; inactive entries of all three bitwise unchanged"""
    (th0, m0, v0), (th1, m1, v1) = before, after
    g, m0, v0 = g.double(), m0.double(), v0.double()
    m = 0.9 * m0 + 0.1 * g
    v = 0.999 * v0 + 0.001 * g * g
    stepv = (lr / (1 - 0.9 ** step)) * m / (v.sqrt() / np.sqrt(1 - 0.999 ** step) + 1e-8)
    th = th0.double() - stepv
    a = _dev_u8(model._pb.active, th0.numel()).cpu().bool()
    assert int(a.sum()) > 0 and float(stepv[a].abs().max()) > 0
    for label, got, ref, tol in (('theta', th1, th, 2 * _ulp(th) + 2 * _ulp(stepv)), ('m', m1, m, 2 * _ulp(m) + 2 * _ulp(0.1 * (g - m0))),
                                 ('v', v1, v, 2 * _ulp(v) + 2 * _ulp(0.001 * g * g))):
        err = (got.double() - ref).abs()
        assert bool((err[a] <= tol[a]).all()), f'{what} {label}: {int((err[a] > tol[a]).sum())} entries, worst ' \
                                                f'{float((err[a] / tol[a]).max()):.2f} x tol'
    for label, x0, x1 in (('theta', th0, th1), ('m', m0, m1), ('v', v0, v1)):
        assert torch.equal(x1[~a].double(), x0[~a].double()), f'{what}: inactive entries of {label} changed'


ADAM_CASE, ADAM_K = 'static_multi_p4_t300', 5


@pytest.mark.gpu
def test_gpu_adam_step_matches_float64_adam(smpl_assets):
    """apply_kernel at step 1, at step k and at the first step after a stage change with reset_adam (the device's own step
    count), each fed the model's own gradient"""
    cfg, in_dict, make_prior = case(ADAM_CASE, smpl_assets)
    model = _make_model(cfg, smpl_assets, make_prior(DEV))
    data = _init(model, in_dict)
    probe = AdamProbe(model)
    for stage, specs in list(cfg.opt_stage_specs.items())[:2]:
        model._cur_vars, model._cur_stage, model._loss_cfg = specs['opt_variables'], stage, specs['loss_cfg']
        model._set_stage(data, specs['opt_variables'], specs['loss_cfg'], stage, reset_adam=True, begin=True)
        for k in range(1, ADAM_K + 1):
            model._backward()
            before, after, g, step = probe.step(specs['opt_lr'], via_iterate=False)
            assert step == k, f'{stage}: device step {step}, expected {k}'
            if k in (1, ADAM_K):
                _check_adam_step(f'{stage} step {k}', model, specs['opt_lr'], before, after, g, step)


@pytest.mark.gpu
def test_gpu_iterate_matches_backward_for_apply_and_apply(smpl_assets):
    """glamr_opt_iterate (one eager iteration per call) at step 1, step k and after a stage change matches float64 Adam, and a
    twin handle driven by glamr_opt_backward_for_apply + glamr_opt_apply from the same theta ends every step with the same
    gradient, bit-identical theta, m and v and the same device step count"""
    cfg, in_dict, make_prior = case(ADAM_CASE, smpl_assets)
    model, twin = _make_model(cfg, smpl_assets, make_prior(DEV)), _make_model(cfg, smpl_assets, make_prior(DEV))
    dm, dt = _init(model, in_dict), _init(twin, in_dict)
    pm, pt = AdamProbe(model), AdamProbe(twin)
    for stage, specs in list(cfg.opt_stage_specs.items())[:2]:
        for m, d in ((model, dm), (twin, dt)):
            m._cur_vars, m._cur_stage, m._loss_cfg = specs['opt_variables'], stage, specs['loss_cfg']
            m._set_stage(d, specs['opt_variables'], specs['loss_cfg'], stage, reset_adam=True, begin=True)
        assert torch.equal(model._theta, twin._theta), f'{stage}: the two handles start the stage from different theta'
        for k in range(1, ADAM_K + 1):
            before, after, g, step = pm.step(specs['opt_lr'], via_iterate=True)
            assert step == k, f'{stage}: device step {step}, expected {k}'
            if k in (1, ADAM_K):
                _check_adam_step(f'iterate {stage} step {k}', model, specs['opt_lr'], before, after, g, step)
            twin._backward(for_apply=True)
            _, after_t, g_t, step_t = pt.step(specs['opt_lr'], via_iterate=False)
            assert step_t == step
            for label, x, y in zip(('gradient', 'theta', 'm', 'v'), (g, *after), (g_t, *after_t)):
                assert torch.equal(x, y), f'{stage} step {k}: {label} of glamr_opt_iterate and backward_for_apply + apply differ, ' \
                                          f'max {float((x - y).abs().max()):.3e}'
