"""Trajectory sources without the learned trajectory predictor (include/glamr_b200.h, GLAMR_TRAJ_BASE): the default
trajectory (flag_infer_motion_traj / flag_pred_traj false), the camera-derived one (flag_traj_from_cam with
'linear_interp' or 'last_pose') and fixed trajectories (flag_opt_traj false, camera only).

CPU: the oracle against the executed reference (tests/golden/globalopt_ts_*.npz), the host-compiled frame functions and
Adam against oracle autograd, person sharding over two gloo ranks.  GPU (-m gpu): the CUDA path against the fixtures'
float64 noise floor, iteration-0 gradients against oracle autograd, CUDA graph vs eager, and a run_dataset sweep without
any learned prior."""
import copy
import ctypes
import os
import socket
import sys

import numpy as np
import pytest
import torch

from helpers import ReplayMT, load_golden
from traj_source_cases import CASES, TRAJ_SOURCE_CASES, case_config, case_in_dict, cfg_path, oracle_class

HERE = os.path.dirname(os.path.abspath(__file__))
ALL = [c[0] for c in TRAJ_SOURCE_CASES]
SMALL = [c[0] for c in TRAJ_SOURCE_CASES if c[3] <= 80]
EPS32 = 2.0 ** -24


def _setup(name, smpl_assets):
    return load_golden('globalopt_' + name), case_config(name), case_in_dict(name, smpl_assets)


def _noise_tol(r32, r64, rp, ulps=32):
    """c x the larger of the reference's own float32-vs-float64 deviation and its one-rounding perturbation response
    (tests/golden/make_traj_source_golden.py), plus a few float32 roundings of the magnitude"""
    noise = max(float(np.abs(r32 - r64).max()), float(np.abs(rp - r32).max()))
    return 4.0 * noise + ulps * EPS32 * max(float(np.abs(r64).max()), 1.0)


def _oracle_grads(model, data, specs, stage):
    params = model.get_parameter(data, specs['opt_variables'])
    for p in params:
        p.requires_grad_(True)
        p.grad = None
    model.forward(data, specs['opt_variables'], {'stage': stage})
    total, _, uw = model.compute_loss(data, specs['loss_cfg'])
    total.backward()
    grads = [None if p.grad is None else p.grad.detach().clone() for p in params]
    for p in params:
        p.requires_grad_(False)
        p.grad = None
    return params, grads, {k: float(v) for k, v in uw.items()}, float(total)


def _grad_views(lay, grad, P, opt_variables, fixed_cam, opt_traj):
    """views of a packed gradient in the order of get_parameter (global_recon_model.py:591-633)"""
    gv = lay.views(grad)
    if 'cam' not in opt_variables:
        order = [gv['cam_inv_rot_residual'], gv['cam_inv_trans_residual']]
    elif fixed_cam:
        order = [gv['cam_rot_6d_fix'], gv['cam_trans_fix']]
    else:
        order = [gv['cam_rot_6d'], gv['cam_trans']]
    for p in range(P):
        pv = lay.views(grad, p)
        if opt_traj:
            for key in opt_variables:
                if key == 'world_res':
                    order += [pv['smpl_orient_world_res'], pv['root_trans_world_res']]
                if 'local' in key:
                    order.append(pv[f'traj_{key}'])
        if 'world_dheading' in opt_variables:
            order.append(pv['world_dheading'])
    return order


def _compare_grads(views, params, grads, what, tol):
    assert len(views) == len(params), what
    for i, (g_, gr) in enumerate(zip(views, grads)):
        if gr is None:                       # autograd never reached it (Adam skips it): ours must be exactly zero
            assert g_.numel() == 0 or float(g_.abs().max()) == 0.0, f'{what} param {i}'
            continue
        scale = max(float(gr.abs().max()), 1e-9)
        err = float((g_.reshape(gr.shape) - gr).abs().max()) / scale
        assert err < tol, f'{what} grad of param {i} shape {tuple(gr.shape)}: rel err {err:.2e} (scale {scale:.2e})'


# ------------------------------------------------------------------------------------------------ CPU: oracle vs reference
def test_cases_cover_the_new_modes():
    specs = {c[1]: case_config(c[0]).grecon_model_specs for c in TRAJ_SOURCE_CASES}
    assert {s.get('traj_interp_method') for s in specs.values()} == {'linear_interp', 'last_pose'}
    assert any(not s.get('flag_opt_traj', True) for s in specs.values())
    assert any(not s['flag_infer_motion_traj'] for s in specs.values())
    assert any(s['flag_infer_motion_traj'] and not s['flag_pred_traj'] for s in specs.values())
    assert any(s.get('flag_opt_cam_from_person_pose') for s in specs.values())
    assert ('ts_static_multi_cam_p4_t300_gaps' in CASES) and CASES['ts_static_multi_cam_p4_t300_gaps'][2:4] == (4, 300)


@pytest.mark.parametrize('name', ALL)
def test_oracle_init_matches_reference_golden(name, smpl_assets):
    """get_traj_from_cam (both interpolation methods), the default trajectory and the base reset of init_data: the world pose,
    the (forward-filled) body pose, the camera and the projected keypoints right after init"""
    Oracle = oracle_class()
    gold, cfg, in_dict = _setup(name, smpl_assets)
    ora = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data = ora.init_data(in_dict)
    P = len(data['person_data'])
    if P > 1:                                          # the last person exists on a strict sub-range of the sequence
        last = data['person_data'][P - 1]
        assert 0 < int(last['fr_start']) and int(last['fr_end']) < data['seq_len']
    for pid, pd in data['person_data'].items():
        assert 'traj_local_pred' not in pd
        for k in ['smpl_orient_world', 'root_trans_world', 'smpl_pose', 'kp_2d_pred']:
            if f'init/{pid}/{k}' not in gold:              # left out of the large fixture (traj_source_cases.COMPACT)
                continue
            np.testing.assert_allclose(pd[k].detach().numpy(), gold[f'init/{pid}/{k}'], atol=1e-3 if k == 'kp_2d_pred' else 1e-5,
                                       err_msg=f'init {pid} {k}')
    np.testing.assert_allclose(data['cam_pose'].numpy(), gold['init/cam_pose'], atol=1e-5)


@pytest.mark.parametrize('name', ALL)
def test_oracle_trajectory_matches_reference_golden(name, smpl_assets):
    """iteration-0 gradients of every stage, per-iteration residuals and the final state: first-stage values tightly, the
    whole trajectory within the reference's own float32 noise"""
    Oracle = oracle_class()
    gold, cfg, in_dict = _setup(name, smpl_assets)
    ora = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data = ora.init_data(in_dict)
    first = list(cfg.opt_stage_specs)[0]
    for stage, specs in cfg.opt_stage_specs.items():
        logs, grads0 = [], {}
        params = ora.get_parameter(data, specs['opt_variables'])

        def on_iter(it, last, dt):
            logs.append({k: float(v) for k, v in last['uw'].items()})
            if it == 0:
                for i, p in enumerate(params):
                    grads0[i] = None if p.grad is None else p.grad.detach().clone().numpy()
        orig = ora.get_parameter
        ora.get_parameter = lambda d, v: params
        ora.optimize_main(data, specs['opt_variables'], specs['opt_lr'], specs['opt_niters'], specs['loss_cfg'], {'stage': stage}, on_iter)
        ora.get_parameter = orig
        for i in range(len(params)):
            ref = gold[f'grad0/{stage}/{i}']
            if ref.size == 0:
                assert grads0[i] is None or not np.any(grads0[i])
                continue
            scale = max(np.abs(ref).max(), 1e-12)
            assert np.abs(grads0[i] - ref).max() / scale < (2e-4 if stage == first else 1e-3), f'grad {stage} param {i}'
        for k in logs[0]:
            r32, r64, rp = gold[f'loss/{stage}/{k}'], gold[f'loss64/{stage}/{k}'], gold[f'loss_pert/{stage}/{k}']
            got = np.array([l[k] for l in logs])
            if stage == first:
                np.testing.assert_allclose(got[:1], r32[:1], rtol=2e-4, atol=1e-6, err_msg=f'{stage} {k} iteration 0')
            tol = 4.0 * max(np.abs(r32 - r64).max(), np.abs(rp - r32).max()) + 2e-4 * np.abs(r64).max() + 1e-6
            assert np.abs(got - r64).max() <= tol, f'{stage} {k}'
    for pid, pd in data['person_data'].items():
        for k in ['smpl_orient_world', 'root_trans_world', 'world_dheading', 'smpl_orient_world_res', 'root_trans_world_res']:
            if f'final64/{pid}/{k}' in gold:
                r32, r64, rp = gold[f'final/{pid}/{k}'], gold[f'final64/{pid}/{k}'], gold[f'final_pert/{pid}/{k}']
                assert np.abs(pd[k].detach().numpy() - r64).max() <= _noise_tol(r32, r64, rp), f'final {pid} {k}'
        assert 'traj_local' not in pd and f'final/{pid}/traj_local' not in gold
    r32, r64, rp = gold['final/cam_pose'], gold['final64/cam_pose'], gold['final_pert/cam_pose']
    assert np.abs(data['cam_pose'].numpy() - r64).max() <= _noise_tol(r32, r64, rp)


# ------------------------------------------------------------------------------------------------ CPU: host-compiled kernels
@pytest.mark.parametrize('name', SMALL)
def test_frame_functions_and_adam_match_oracle_autograd(name, smpl_assets):
    """the frame functions of globalopt_frames.cuh (g++) with traj_source = GLAMR_TRAJ_BASE: every variable's gradient and
    every residual of every stage against autograd through the oracle, then the stage's Adam steps in both"""
    from emu_runner import EmuRunner
    from glamr_b200 import lib as L
    Oracle = oracle_class()
    gold, cfg, in_dict = _setup(name, smpl_assets)
    ora = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data_o = ora.init_data(copy.deepcopy(in_dict))
    ora2 = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data_e = ora2.init_data(copy.deepcopy(in_dict))
    run = EmuRunner(ora2, data_e)
    assert run.comp.traj_source == L.TRAJ_BASE and run.comp.opt_traj == ora.flag_opt_traj
    run.set_stage([], {}, 'init')
    run.backward()
    P, T = run.comp.P, run.comp.T
    kp = run.buffer(L.R_KP_PRED).view(P, T, 26, 2)
    for p, d in enumerate(data_o['person_data'].values()):
        np.testing.assert_allclose(kp[p].numpy(), d['kp_2d_pred'].numpy(), atol=2e-3, err_msg='init kp_2d_pred')
        np.testing.assert_allclose(run.buffer(L.R_ORIENT_WORLD).view(P, T, 3)[p].numpy(), d['smpl_orient_world'].detach().numpy(), atol=1e-6)
    for stage, specs in cfg.opt_stage_specs.items():
        variables = specs['opt_variables']
        params = ora.get_parameter(data_o, variables)
        run.set_stage(variables, specs['loss_cfg'], stage)
        thetas = _grad_views(run.layout, run.theta, P, variables, ora.flag_fixed_cam, ora.flag_opt_traj)
        assert len(thetas) == len(params)
        # Independent Adam runs drift apart wherever the loss amplifies rounding (cam_up_reg x 1e6, ill-conditioned world
        # residuals), so every step is checked on IDENTICAL variables: the oracle evaluates the emulator's theta, and the host
        # Adam is checked against torch.optim.Adam fed the same gradient.
        with torch.no_grad():
            for v, p_ in zip(thetas, params):
                p_.copy_(v.reshape(p_.shape))
        adam = torch.optim.Adam(params, lr=specs['opt_lr'], betas=(0.9, 0.999)) if params else None
        for it in range(specs['opt_niters']):
            for p_ in params:
                p_.requires_grad_(True)
                p_.grad = None
            ora.forward(data_o, variables, {'stage': stage})
            total, _, uw = ora.compute_loss(data_o, specs['loss_cfg'])
            total.backward()
            grads = [None if p_.grad is None else p_.grad.detach().clone() for p_ in params]
            uw, total = {k: float(v) for k, v in uw.items()}, float(total)
            _, terms = run.backward()
            for k, v in uw.items():
                got = float(terms[L.TERM_INDEX[k]])
                assert abs(got - v) <= 2e-4 * max(abs(v), 1e-3) + 1e-7, f'{stage} it {it} term {k}: {got} vs {v}'
            assert abs(float(terms[-1]) - total) <= 2e-4 * abs(total) + 1e-6
            views = _grad_views(run.layout, run.reduce[:run.layout.n_params], P, variables, ora.flag_fixed_cam, ora.flag_opt_traj)
            _compare_grads(views, params, grads, f'{stage} it {it}', 3e-4)
            for g_, p_ in zip(views, params):
                p_.grad = g_.reshape(p_.shape).clone()
            adam.step()
            run.step(specs['opt_lr'])
            with torch.no_grad():
                for i, (v, p_) in enumerate(zip(thetas, params)):
                    err = float((v.reshape(p_.shape) - p_).abs().max()) if p_.numel() else 0.0
                    assert err <= 1e-6 * max(float(p_.abs().max()), 1.0), f'{stage} it {it} Adam step of param {i}: {err:.2e}'
                    p_.copy_(v.reshape(p_.shape))
                    p_.grad = None
        for p_ in params:
            p_.requires_grad_(False)
        cam = run.buffer(L.R_CAM_POSE).view(T, 3, 4)
        np.testing.assert_allclose(cam.numpy(), data_o['cam_pose'][:, :3, :].detach().numpy(), atol=2e-5, err_msg=f'{stage} cam_pose')
        data_e['cam_pose'] = torch.cat([cam, torch.tensor([0., 0., 0., 1.]).expand(T, 1, 4)], dim=1).clone()
        data_o['cam_pose'], data_o['cam_pose_inv'] = data_o['cam_pose'].detach(), data_o['cam_pose_inv'].detach()


def test_problem_struct_carries_the_trajectory_source():
    """the ctypes mirror and the C struct agree (host build of the header), and zero means the predicted trajectory"""
    import host_harness as hh
    from glamr_b200 import lib as L
    assert hh.lib().glamr_host_sizeof_problem() == ctypes.sizeof(L.Problem)
    assert L.Problem().traj_source == L.TRAJ_PREDICTED == 0 and L.TRAJ_BASE == 1


@pytest.mark.parametrize('name,what', [('ts_static_multi_last_p3_t30_gaps', 'local_var'), ('ts_static_multi_last_p3_t30_gaps', 'local_reg'),
                                       ('ts_cam_only_p2_t32_gaps', 'rel'), ('ts_cam_only_p2_t32_gaps', 'res')])
def test_combinations_the_reference_fails_on_raise(name, what, smpl_assets):
    """variables / residuals the reference has not created in these modes (its get_parameter or loss_func.py fails on them)"""
    from glamr_b200 import problem as PB
    from oracle import rotations as rt
    Oracle = oracle_class()
    gold, cfg, in_dict = _setup(name, smpl_assets)
    ora = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data = ora.init_data(in_dict)
    flags = {k: getattr(ora, k) for k in ['flag_fixed_cam', 'flag_opt_cam', 'flag_opt_cam_from_person_pose', 'flag_cam_inv_trans_res_all',
                                          'flag_opt_vis_local_rot', 'cam_fix_frames']}
    lay = PB.make_layout(data, flags)
    theta = torch.zeros(lay.n_params)
    PB.bind_variables(data, lay, theta)
    comp = PB.StageCompiler(data, lay, flags, 'cpu', rt.aa_to_rot6d, aa_to_quat=rt.aa_to_quat)
    variables, loss = ['cam'], {'kp_2d': {'weight': 1.0}}
    if what == 'local_var':
        variables = ['world_res', 'local_xy']
    elif what == 'local_reg':
        loss['local_traj_rot_reg'] = {'weight': 1.0}
    elif what == 'rel':
        loss['rel_transform'] = {'weight': 1.0}
    else:
        loss['traj_rot_res'] = {'weight': 1.0}
    with pytest.raises(ValueError):
        comp.compile(theta, variables, loss, 'opt')


# ------------------------------------------------------------------------------------------------ CPU: two ranks
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, name, ret):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    torch.set_num_threads(1)
    from emu_runner import EmuRunner
    from glamr_b200.synthetic import make_smpl_assets
    Oracle = oracle_class()
    assets = make_smpl_assets(0)
    gold, cfg, in_dict = _setup(name, assets)
    results = {}
    for mode in ['single', 'sharded']:
        ora = Oracle(copy.deepcopy(cfg), assets, mt_model=ReplayMT(gold))
        run = EmuRunner(ora, ora.init_data(copy.deepcopy(in_dict)))
        stage, specs = list(cfg.opt_stage_specs.items())[-1]
        N = run.comp.P * run.comp.T
        kw = {} if mode == 'single' else dict(n_begin=N * rank // world, n_end=N * (rank + 1) // world, owner=(rank == 0))
        run.set_stage(specs['opt_variables'], specs['loss_cfg'], stage, **kw)
        for it in range(3):
            run.backward()
            if mode == 'sharded':
                dist.all_reduce(run.reduce)
            run.step(specs['opt_lr'])
        results[mode] = (run.reduce.clone(), run.theta.clone())
    g_err = float((results['single'][0] - results['sharded'][0]).abs().max() / results['single'][0].abs().max())
    t_err = float((results['single'][1] - results['sharded'][1]).abs().max())
    ret[rank] = (g_err, t_err)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('name', ['ts_static_multi_last_p3_t30_gaps', 'ts_3dpw_cam_p2_t80_gaps'])
def test_person_sharding_allreduce_equals_single_rank(name):
    """frame-persons split over two gloo ranks (with 3 persons, person 1 straddles them): the summed world-variable
    gradients and the parameters after 3 Adam steps equal the single-rank run"""
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ret = mp.get_context('spawn').Manager().dict()
    mp.spawn(_gloo_worker, args=(world, port, name, ret), nprocs=world, join=True)
    for rank in range(world):
        g_err, t_err = ret[rank]
        assert g_err < 1e-5, f'rank {rank}: reduced gradient differs from single-rank by {g_err:.2e} (relative)'
        assert t_err < 1e-5, f'rank {rank}: parameters after 3 steps differ by {t_err:.2e}'


# ------------------------------------------------------------------------------------------------ GPU
DEV = 'cuda:0'


def _make(name, smpl_assets, **spec_over):
    from glamr_b200.recon import GlobalReconOptimizer
    gold, cfg, in_dict = _setup(name, smpl_assets)
    cfg.grecon_model_specs.update(spec_over)
    model = GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=smpl_assets, mt_model=ReplayMT(gold, DEV))
    return gold, cfg, in_dict, model


def _align_half_turns(model, data, gold):
    """The default trajectory's orientation (quaternion (0, 0, 0.7071, 0.7071)) is a rotation by exactly pi, and person 0's first
    frame keeps it when the camera is derived from that person.  There the sign of the axis-angle vector is decided by the last
    bit of the quaternion's scalar part, so the reference and the CUDA row-ops may pick opposite vectors for the SAME rotation.
    world_res is added to that vector, so the two representations optimise differently: the CUDA path is restarted from the
    reference's representation of exactly those frames (same rotation, antipodal vector), and from nothing else."""
    changed = False
    for pid, pd in data['person_data'].items():
        ref = torch.tensor(gold[f'init/{pid}/smpl_orient_world'], device=DEV, dtype=torch.float32)
        base = pd['smpl_orient_world_base']
        flip = ((base + ref).abs().amax(-1) < 1e-5) & ((base - ref).abs().amax(-1) > 1.0) & ((ref.norm(dim=-1) - np.pi).abs() < 1e-5)
        if flip.any():
            base = base.clone()
            base[flip] = ref[flip]
            pd['smpl_orient_world_base'], pd['smpl_orient_world'] = base, base.clone()
            changed = True
    if changed:
        model._attach(data)
        model.forward(data, [], {'stage': 'init'})
    return changed


def _check_init(data, gold):
    for pid, pd in data['person_data'].items():
        if f'init/{pid}/kp_2d_pred' in gold:              # left out of the large fixture (traj_source_cases.COMPACT)
            np.testing.assert_allclose(pd['kp_2d_pred'].cpu().numpy(), gold[f'init/{pid}/kp_2d_pred'], atol=5e-3, err_msg='init kp')
        for k in ['smpl_orient_world', 'root_trans_world', 'smpl_pose']:
            if f'init/{pid}/{k}' in gold:
                np.testing.assert_allclose(pd[k].cpu().numpy(), gold[f'init/{pid}/{k}'], atol=1e-4, err_msg=f'init {pid} {k}')
    np.testing.assert_allclose(data['cam_pose'].cpu().numpy(), gold['init/cam_pose'], atol=1e-5)


def _check_trajectory(model, data, cfg, gold):
    from glamr_b200 import lib as L
    first = list(cfg.opt_stage_specs)[0]
    for stage, specs in cfg.opt_stage_specs.items():
        n = specs['opt_niters']
        model.optimize_main(data, specs['opt_variables'], specs['opt_lr'], n, specs['loss_cfg'], {'stage': stage})
        hist = model.loss_history.cpu().numpy()
        for k in specs['loss_cfg']:
            r32, r64, rp = gold[f'loss/{stage}/{k}'], gold[f'loss64/{stage}/{k}'], gold[f'loss_pert/{stage}/{k}']
            got = hist[:n, L.TERM_INDEX[k]]
            if stage == first:       # a pure forward on identical variables; later stages start where Adam's amplified noise left them
                np.testing.assert_allclose(got[:1], r64[:1], rtol=2e-4, atol=1e-6, err_msg=f'{stage} {k} (iteration 0)')
            tol = 4.0 * max(np.abs(r32 - r64).max(), np.abs(rp - r32).max()) + 2e-4 * np.abs(r64).max() + 1e-6
            err = np.abs(got - r64).max()
            assert err <= tol, f'{stage} {k}: |cuda-ref64| {err:.3e} > {tol:.3e}'
    checks = [('cam_pose', data['cam_pose'].cpu().numpy())]
    for pid, pd in data['person_data'].items():
        assert 'traj_local' not in pd
        for k in ['smpl_orient_world', 'root_trans_world', 'smpl_orient_world_res', 'root_trans_world_res', 'world_dheading', 'kp_2d_pred']:
            if k in pd and f'final64/{pid}/{k}' in gold:
                checks.append((f'{pid}/{k}', pd[k].cpu().numpy()))
    for key, got in checks:
        r32, r64, rp = gold[f'final/{key}'], gold[f'final64/{key}'], gold[f'final_pert/{key}']
        tol = _noise_tol(r32, r64, rp, ulps=256 if 'kp_2d_pred' in key else 32)
        name_ = key.split('/')[-1]
        if name_ in ('cam_pose', 'smpl_orient_world', 'root_trans_world'):
            tol = max(tol, 1e-4)                         # the north-star bound on output poses (m, rad)
        elif name_ == 'kp_2d_pred':
            tol = max(tol, 2e-2)                         # pixels: 1e-4 m at f / z = 1000 / 5
        err = float(np.abs(got.reshape(r64.shape) - r64).max())
        assert err <= tol, f'final {key}: |cuda-ref64| {err:.3e} > {tol:.3e}'


@pytest.mark.gpu
@pytest.mark.parametrize('name', ALL)
def test_gpu_trajectory_matches_reference_golden(name, smpl_assets):
    """init state (camera-derived / default trajectories, forward-filled body pose), per-iteration residual values and the
    final state of every frame vs the executed reference, at its float64 noise floor"""
    from glamr_b200 import lib as L
    gold, cfg, in_dict, model = _make(name, smpl_assets)
    assert model.traj_source == L.TRAJ_BASE
    data = model.init_data(copy.deepcopy(in_dict))
    _align_half_turns(model, data, gold)
    _check_init(data, gold)
    _check_trajectory(model, data, cfg, gold)


@pytest.mark.gpu
@pytest.mark.parametrize('name', SMALL)
def test_gpu_gradients_match_oracle_autograd(name, smpl_assets):
    """first closure of every stage: every variable's gradient and every residual vs autograd through the full-LBS oracle"""
    from glamr_b200 import lib as L
    Oracle = oracle_class()
    gold, cfg, in_dict, model = _make(name, smpl_assets)
    data = model.init_data(copy.deepcopy(in_dict))
    _align_half_turns(model, data, gold)
    ora = Oracle(copy.deepcopy(cfg), smpl_assets, mt_model=ReplayMT(gold))
    data_o = ora.init_data(copy.deepcopy(in_dict))
    P = len(data['person_data'])
    for stage, specs in cfg.opt_stage_specs.items():
        params, grads, uw, _ = _oracle_grads(ora, data_o, specs, stage)
        model._cur_vars, model._cur_stage = specs['opt_variables'], stage
        model._set_stage(data, specs['opt_variables'], specs['loss_cfg'], stage, reset_adam=True, begin=True)
        model._backward()
        with torch.cuda.device(DEV):
            L.check(model._lib.glamr_opt_losses(model._opt, L.ptr(model._reduce), L.ptr(model._terms), L.stream_ptr()), 'glamr_opt_losses')
        terms = model._terms.cpu().numpy()
        for k, v in uw.items():
            assert abs(float(terms[L.TERM_INDEX[k]]) - v) <= 3e-4 * max(abs(v), 1e-3) + 1e-7, f'{stage} term {k}'
        grad = model._reduce[:model._layout.n_params].cpu()
        views = _grad_views(model._layout, grad, P, specs['opt_variables'], model.flag_fixed_cam, model.flag_opt_traj)
        _compare_grads(views, params, grads, stage, 5e-4)
        # advance the stage on the GPU and hand its variables to the oracle: the next stage starts from identical state
        model.optimize_main(data, specs['opt_variables'], specs['opt_lr'], specs['opt_niters'], specs['loss_cfg'], {'stage': stage})
        for pd, po in zip(data['person_data'].values(), data_o['person_data'].values()):
            for k in ['traj_local_xy', 'traj_local_dxy', 'traj_local_heading', 'traj_local_dheading', 'traj_local_z', 'traj_local_rot',
                      'smpl_orient_world_res', 'root_trans_world_res', 'world_dheading']:
                if k in pd and k in po:
                    po[k] = pd[k].detach().cpu().clone()
        for k in ['cam_pose', 'cam_pose_inv', 'cam_inv_rot_residual', 'cam_inv_trans_residual']:
            data_o[k] = data[k].detach().cpu().clone()


@pytest.mark.gpu
def test_gpu_cuda_graph_and_eager_agree(smpl_assets):
    outs = []
    for graph in (True, False):
        _, _, in_dict, model = _make('ts_static_multi_last_p3_t30_gaps', smpl_assets, use_cuda_graph=graph)
        outs.append(model.optimize(copy.deepcopy(in_dict)))
    for pid in outs[0]['person_data']:
        for k in ['smpl_orient_world', 'root_trans_world', 'smpl_orient_world_res', 'kp_2d_pred']:
            np.testing.assert_array_equal(outs[0]['person_data'][pid][k], outs[1]['person_data'][pid][k])
    np.testing.assert_array_equal(outs[0]['cam_pose'], outs[1]['cam_pose'])


@pytest.mark.gpu
def test_gpu_run_dataset_without_learned_prior(tmp_path):
    """run_dataset --synthetic with flag_infer_motion_traj false: no prior, no checkpoint; the output pickle is written"""
    import pickle
    from glamr_b200.global_recon import run_dataset as rd
    args = rd.parse(['--cfg', cfg_path('glamr_dynamic_traj_from_cam'), '--out_dir', str(tmp_path), '--synthetic', '1', '--frames', '48',
                     '--gaps', '--quiet'])
    done = rd.run(args)
    assert len(done) == 1 and os.path.exists(done[0][2])
    out = pickle.load(open(done[0][2], 'rb'))
    pd = out['person_data'][0]
    assert 'traj_local_pred' not in pd and 'traj_local' not in pd
    assert pd['smpl_orient_world'].shape == (48, 3) and np.isfinite(pd['smpl_orient_world']).all()
    assert out['cam_pose'].shape == (48, 4, 4) and np.isfinite(out['cam_pose']).all()
    assert out['meta']['mt_cfg'] is None


@pytest.mark.gpu
def test_gpu_predictor_with_fixed_trajectory_is_refused(smpl_assets):
    """flag_opt_traj false with the trajectory predictor: the reference fails on the missing local variables"""
    from glamr_b200.config import Config
    from glamr_b200.recon import GlobalReconOptimizer
    cfg = Config('glamr_dynamic')
    cfg.grecon_model_specs['flag_opt_traj'] = False
    with pytest.raises(ValueError):
        GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=smpl_assets, mt_model=ReplayMT({}, DEV))
