"""heading_type 'vec' (traj_local_heading / traj_local_dheading move the predicted heading vector) and world_dxy (a world-plane
offset added in place to root_trans_world, include/glamr_b200.h: heading_vec, has_world_dxy, world_dxy_alias, world_dxy_base).

CPU: the oracle against the executed reference (tests/golden/globalopt_tv_*.npz), the host-compiled frame functions and Adam
against oracle autograd, person sharding over two gloo ranks with world_dxy accumulating in the base, and the combinations that
are refused.  GPU (-m gpu): the CUDA path against the fixtures' float64 noise floor, iteration-0 gradients against oracle
autograd, CUDA graph vs eager, and a run_dataset sweep with a vec config."""
import copy
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from helpers import ReplayMT, load_golden
from test_traj_sources import _align_half_turns, _compare_grads, _free_port, _noise_tol, _oracle_grads
from traj_variable_cases import CASES, FAILING_CASES, FINAL_VARS, TRAJ_VARIABLE_CASES, case_config, case_in_dict, cfg_path, oracle_class

HERE = os.path.dirname(os.path.abspath(__file__))
ALL = [c[0] for c in TRAJ_VARIABLE_CASES]
SMALL = [c[0] for c in TRAJ_VARIABLE_CASES if c[3] <= 80]
ALIAS_CASE = 'tv_static_multi_dxy_p3_t30_gaps'          # world_dxy next to world_dheading on the predicted trajectory
FAILING = FAILING_CASES[0][0]


def _setup(name, smpl_assets):
    return load_golden('globalopt_' + name), case_config(name), case_in_dict(name, smpl_assets)


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
        if 'world_dxy' in opt_variables:
            order.append(pv['world_dxy'])
    return order


def _emu_runner(ora, data):
    """tests/emu_runner.EmuRunner with the variable layout sized for heading vectors and world_dxy"""
    import host_harness as hh
    from emu_runner import EmuRunner
    from glamr_b200 import lib as L
    from glamr_b200 import problem as PB
    from oracle import rotations as rt
    run = EmuRunner.__new__(EmuRunner)
    run.model, run.data = ora, data
    run.flags = {k: getattr(ora, k) for k in ['flag_fixed_cam', 'flag_opt_cam', 'flag_opt_cam_from_person_pose', 'flag_cam_inv_trans_res_all',
                                              'flag_opt_vis_local_rot', 'cam_fix_frames']}
    run.flags['heading_vec'] = ora.heading_type == 'vec'
    run.flags['world_dxy'] = any('world_dxy' in st['opt_variables'] for st in ora.opt_stage_specs.values())
    run.layout = PB.make_layout(data, run.flags)
    run.theta = torch.zeros(run.layout.n_params)
    PB.bind_variables(data, run.layout, run.theta)
    run.comp = PB.StageCompiler(data, run.layout, run.flags, 'cpu', rt.aa_to_rot6d, aa_to_quat=rt.aa_to_quat)
    run.lib, run.h = hh.lib(), None
    run.reduce = torch.zeros(run.layout.n_params + L.NUM_TERMS)
    return run


# ------------------------------------------------------------------------------------------------ CPU: oracle vs reference
def test_cases_cover_the_new_options():
    specs = {c[0]: case_config(c[0]) for c in TRAJ_VARIABLE_CASES}
    vec = [n for n, c in specs.items() if c.grecon_model_specs.get('heading_type') == 'vec']
    dxy = [n for n, c in specs.items() if any('world_dxy' in st['opt_variables'] for st in c.opt_stage_specs.values())]
    assert len(vec) >= 3 and len(dxy) >= 3
    assert 'tv_static_multi_vec_dxy_p4_t300_gaps' in vec and 'tv_static_multi_vec_dxy_p4_t300_gaps' in dxy
    assert CASES['tv_static_multi_vec_dxy_p4_t300_gaps'][2:4] == (4, 300)
    # glamr_3dpw optimises local_dheading under local_traj_dheading_reg_new
    main = specs['tv_3dpw_vec_p2_t80_gaps'].opt_stage_specs['main_opt']
    assert 'local_dheading' in main['opt_variables'] and 'local_traj_dheading_reg_new' in main['loss_cfg']
    # world_dxy with world_dheading (aliased base) and with world_res alone (fresh tensor)
    st = specs['tv_dynamic_cam_dxy_p1_t40_gaps'].opt_stage_specs['init_opt']['opt_variables']
    assert 'world_res' in st and 'world_dheading' not in st
    assert 'world_dheading' in specs[ALIAS_CASE].opt_stage_specs['main_opt']['opt_variables']


@pytest.mark.parametrize('name', ALL)
def test_oracle_matches_reference_golden(name, smpl_assets):
    """init state, iteration-0 gradients of every stage, per-iteration residuals and the final state (world pose, base, heading
    vectors, world_dxy) of the oracle against the executed reference"""
    Oracle = oracle_class()
    gold, cfg, in_dict = _setup(name, smpl_assets)
    ora = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data = ora.init_data(in_dict)
    for pid, pd in data['person_data'].items():
        for k in ['smpl_orient_world', 'root_trans_world', 'kp_2d_pred', 'traj_local_heading', 'traj_local_dheading']:
            if f'init/{pid}/{k}' in gold:
                np.testing.assert_allclose(pd[k].detach().numpy(), gold[f'init/{pid}/{k}'], atol=1e-3 if k == 'kp_2d_pred' else 1e-5,
                                           err_msg=f'init {pid} {k}')
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
            assert tuple(gold[f'param_shape/{stage}/{i}']) == tuple(params[i].shape), f'{stage} param {i} shape'
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
        for k in ['smpl_orient_world', 'root_trans_world'] + FINAL_VARS:
            if f'final64/{pid}/{k}' in gold:
                r32, r64, rp = gold[f'final/{pid}/{k}'], gold[f'final64/{pid}/{k}'], gold[f'final_pert/{pid}/{k}']
                assert np.abs(pd[k].detach().numpy() - r64).max() <= _noise_tol(r32, r64, rp), f'final {pid} {k}'
    r32, r64, rp = gold['final/cam_pose'], gold['final64/cam_pose'], gold['final_pert/cam_pose']
    assert np.abs(data['cam_pose'].numpy() - r64).max() <= _noise_tol(r32, r64, rp)


def test_world_dxy_accumulates_in_the_base_outside_the_exist_range():
    """the aliased case of the reference (world_dxy with world_dheading): outside the last person's exist range the base kept the
    world_dxy of every forward, inside it the codec re-created it; the fixture shows both"""
    gold = load_golden('globalopt_' + ALIAS_CASE)
    P = int(gold['meta'][0])
    tb, tw, dxy = (gold[f'final/{P - 1}/{k}'] for k in ['root_trans_world_base', 'root_trans_world', 'world_dxy'])
    assert np.abs(dxy).max() > 0
    np.testing.assert_array_equal(tb, tw)                  # root_trans_world IS the base
    out = np.where(~np.asarray(gold[f'init/{P - 1}/vis_frames'], bool))[0]
    assert out.size and np.abs(tb[out[0], :2] - gold[f'init/{P - 1}/root_trans_world'][out[0], :2] - dxy[out[0]]).max() > 1e-7


# ------------------------------------------------------------------------------------------------ CPU: host-compiled kernels
@pytest.mark.parametrize('name', SMALL)
def test_frame_functions_and_adam_match_oracle_autograd(name, smpl_assets):
    """the frame functions of globalopt_frames.cuh (g++) with heading vectors / world_dxy: every variable's gradient and every
    residual of every stage against autograd through the oracle, then the stage's Adam steps in both.  The oracle and the
    host harness each advance their own world_dxy base once per evaluation."""
    from glamr_b200 import lib as L
    Oracle = oracle_class()
    gold, cfg, in_dict = _setup(name, smpl_assets)
    ora = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data_o = ora.init_data(copy.deepcopy(in_dict))
    ora2 = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data_e = ora2.init_data(copy.deepcopy(in_dict))
    run = _emu_runner(ora2, data_e)
    assert run.comp.heading_vec == (ora.heading_type == 'vec')
    run.set_stage([], {}, 'init')
    run.backward()
    P, T = run.comp.P, run.comp.T
    for stage, specs in cfg.opt_stage_specs.items():
        variables = specs['opt_variables']
        params = ora.get_parameter(data_o, variables)
        run.set_stage(variables, specs['loss_cfg'], stage)
        thetas = _grad_views(run.layout, run.theta, P, variables, ora.flag_fixed_cam, ora.flag_opt_traj)
        assert len(thetas) == len(params)
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
            # world pose and base (world_dxy's in-place add included) of this evaluation
            tw = run.buffer(L.R_TRANS_WORLD).view(P, T, 3)
            tb = run.buffer(L.R_TRANS_BASE).view(P, T, 3)
            for p, d in enumerate(data_o['person_data'].values()):
                np.testing.assert_allclose(tw[p].numpy(), d['root_trans_world'].detach().numpy(), atol=2e-5, err_msg=f'{stage} it {it} trans')
                np.testing.assert_allclose(tb[p].numpy(), d['root_trans_world_base'].detach().numpy(), atol=2e-5, err_msg=f'{stage} it {it} base')
                if ora.heading_type == 'vec' and 'traj_local' in d:
                    tl = run.buffer(L.R_TRAJ_LOCAL).view(P, T, 11)[p][d['exist_frames']]
                    np.testing.assert_allclose(tl.numpy(), d['traj_local'].detach().numpy(), atol=2e-5, err_msg='traj_local rows')
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
        data_e['cam_pose'] = torch.cat([cam, torch.tensor([0., 0., 0., 1.]).expand(T, 1, 4)], dim=1).clone()
        data_o['cam_pose'], data_o['cam_pose_inv'] = data_o['cam_pose'].detach(), data_o['cam_pose_inv'].detach()


def test_problem_struct_carries_the_new_fields():
    """the ctypes mirror and the C structs agree (host build of the header), and zero keeps the scalar heading without world_dxy"""
    import host_harness as hh
    from glamr_b200 import lib as L
    assert hh.lib().glamr_host_sizeof_problem() == ctypes.sizeof(L.Problem)
    assert hh.lib().glamr_host_sizeof_person() == ctypes.sizeof(L.Person)
    pb, ps = L.Problem(), L.Person()
    assert pb.heading_vec == pb.has_world_dxy == pb.world_dxy_alias == 0 and not ps.world_dxy_base


def test_reference_fails_on_world_dxy_aliasing_a_fixed_base(smpl_assets):
    """world_dxy next to world_dheading on a camera-derived trajectory: the reference fails in its second backward (the fixture
    records it); StageCompiler refuses the stage with a clear ValueError"""
    from glamr_b200 import problem as PB
    from oracle import rotations as rt
    gold = load_golden('globalopt_' + FAILING)
    assert 'backward through the graph a second time' in str(gold['ref_error']) and int(gold['ref_error_at'][0]) == 1
    Oracle = oracle_class()
    cfg, in_dict = case_config(FAILING), case_in_dict(FAILING, smpl_assets)
    ora = Oracle(cfg, smpl_assets)
    data = ora.init_data(in_dict)
    flags = {k: getattr(ora, k) for k in ['flag_fixed_cam', 'flag_opt_cam', 'flag_opt_cam_from_person_pose', 'flag_cam_inv_trans_res_all',
                                          'flag_opt_vis_local_rot', 'cam_fix_frames']}
    flags['world_dxy'] = True
    lay = PB.make_layout(data, flags)
    theta = torch.zeros(lay.n_params)
    PB.bind_variables(data, lay, theta)
    comp = PB.StageCompiler(data, lay, flags, 'cpu', rt.aa_to_rot6d, aa_to_quat=rt.aa_to_quat)
    specs = cfg.opt_stage_specs['init_opt']
    PB.begin_stage_variables(data, lay, theta, flags, specs['opt_variables'])
    with pytest.raises(ValueError, match='world_dxy'):
        comp.compile(theta, specs['opt_variables'], specs['loss_cfg'], 'init_opt')


# ------------------------------------------------------------------------------------------------ CPU: two ranks
def _gloo_worker(rank, world, port, name, ret):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    torch.set_num_threads(1)
    from glamr_b200 import lib as L
    from glamr_b200.synthetic import make_smpl_assets
    Oracle = oracle_class()
    assets = make_smpl_assets(0)
    gold, cfg, in_dict = _setup(name, assets)
    results = {}
    for mode in ['single', 'sharded']:
        ora = Oracle(copy.deepcopy(cfg), assets, mt_model=ReplayMT(gold))
        run = _emu_runner(ora, ora.init_data(copy.deepcopy(in_dict)))
        stage, specs = list(cfg.opt_stage_specs.items())[-1]
        assert 'world_dxy' in specs['opt_variables']
        N = run.comp.P * run.comp.T
        kw = {} if mode == 'single' else dict(n_begin=N * rank // world, n_end=N * (rank + 1) // world, owner=(rank == 0))
        run.set_stage(specs['opt_variables'], specs['loss_cfg'], stage, **kw)
        assert run.pb.world_dxy_alias == 1
        for it in range(3):
            run.backward()
            if mode == 'sharded':
                dist.all_reduce(run.reduce)
            run.step(specs['opt_lr'])
        results[mode] = (run.reduce.clone(), run.theta.clone(), run.buffer(L.R_TRANS_BASE).clone())
    g_err = float((results['single'][0] - results['sharded'][0]).abs().max() / results['single'][0].abs().max())
    t_err = float((results['single'][1] - results['sharded'][1]).abs().max())
    b_err = float((results['single'][2] - results['sharded'][2]).abs().max())
    ret[rank] = (g_err, t_err, b_err)
    dist.barrier()
    dist.destroy_process_group()


def test_person_sharding_with_world_dxy_equals_single_rank():
    """frame-persons split over two gloo ranks (person 1 straddles them) with world_dxy accumulating in the base on every rank:
    the summed gradients, the parameters and the base after 3 Adam steps equal the single-rank run"""
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ret = mp.get_context('spawn').Manager().dict()
    mp.spawn(_gloo_worker, args=(world, port, ALIAS_CASE, ret), nprocs=world, join=True)
    for rank in range(world):
        g_err, t_err, b_err = ret[rank]
        assert g_err < 1e-5, f'rank {rank}: reduced gradient differs from single-rank by {g_err:.2e} (relative)'
        assert t_err < 1e-5, f'rank {rank}: parameters after 3 steps differ by {t_err:.2e}'
        assert b_err < 1e-5, f'rank {rank}: base after 3 steps differs by {b_err:.2e}'


# ------------------------------------------------------------------------------------------------ GPU
DEV = 'cuda:0'


def _make(name, smpl_assets, **spec_over):
    from glamr_b200.recon import GlobalReconOptimizer
    gold, cfg, in_dict = _setup(name, smpl_assets)
    cfg.grecon_model_specs.update(spec_over)
    model = GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=smpl_assets, mt_model=ReplayMT(gold, DEV))
    return gold, cfg, in_dict, model


def _check_init(data, gold):
    for pid, pd in data['person_data'].items():
        if f'init/{pid}/kp_2d_pred' in gold:
            np.testing.assert_allclose(pd['kp_2d_pred'].cpu().numpy(), gold[f'init/{pid}/kp_2d_pred'], atol=5e-3, err_msg='init kp')
        for k in ['smpl_orient_world', 'root_trans_world', 'traj_local_heading', 'traj_local_dheading']:
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
            if stage == first:
                np.testing.assert_allclose(got[:1], r64[:1], rtol=2e-4, atol=1e-6, err_msg=f'{stage} {k} (iteration 0)')
            tol = 4.0 * max(np.abs(r32 - r64).max(), np.abs(rp - r32).max()) + 2e-4 * np.abs(r64).max() + 1e-6
            err = np.abs(got - r64).max()
            assert err <= tol, f'{stage} {k}: |cuda-ref64| {err:.3e} > {tol:.3e}'
    last_lr, last_n = float(specs['opt_lr']), int(specs['opt_niters'])
    checks = [('cam_pose', data['cam_pose'].cpu().numpy())]
    for pid, pd in data['person_data'].items():
        for k in ['smpl_orient_world', 'root_trans_world', 'kp_2d_pred'] + FINAL_VARS:
            if k in pd and f'final64/{pid}/{k}' in gold:
                checks.append((f'{pid}/{k}', pd[k].cpu().numpy()))
    assert any(k.endswith('world_dxy') for k, _ in checks) or not any(k.endswith('world_dxy') for k in gold.keys())
    for key, got in checks:
        r32, r64, rp = gold[f'final/{key}'], gold[f'final64/{key}'], gold[f'final_pert/{key}']
        tol = _noise_tol(r32, r64, rp, ulps=256 if 'kp_2d_pred' in key else 32)
        name_ = key.split('/')[-1]
        if name_ in ('cam_pose', 'smpl_orient_world', 'root_trans_world', 'root_trans_world_base'):
            tol = max(tol, 1e-4)                         # the north-star bound on output poses (m, rad)
        if name_ in ('smpl_orient_world', 'root_trans_world', 'root_trans_world_base', 'world_dheading', 'world_dxy'):
            # Adam normalises each entry's step: an entry whose gradient is only rounding noise (world_dheading / world_dxy on frames
            # that few residuals reach) moves by up to lr per iteration in whichever direction the noise points
            tol = max(tol, last_lr * last_n)
        elif name_ == 'kp_2d_pred':
            tol = max(tol, 2e-2)                         # pixels: 1e-4 m at f / z = 1000 / 5
        err = float(np.abs(got.reshape(r64.shape) - r64).max())
        assert err <= tol, f'final {key}: |cuda-ref64| {err:.3e} > {tol:.3e}'


@pytest.mark.gpu
@pytest.mark.parametrize('name', ALL)
def test_gpu_trajectory_matches_reference_golden(name, smpl_assets):
    """init state, per-iteration residual values and the final state of every frame (world pose, base, heading vectors, world_dxy)
    vs the executed reference, at its float64 noise floor"""
    gold, cfg, in_dict, model = _make(name, smpl_assets)
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
                      'smpl_orient_world_res', 'root_trans_world_res', 'world_dheading', 'world_dxy']:
                if k in pd and k in po:
                    po[k] = pd[k].detach().cpu().clone()
        for k in ['cam_pose', 'cam_pose_inv', 'cam_inv_rot_residual', 'cam_inv_trans_residual']:
            data_o[k] = data[k].detach().cpu().clone()


@pytest.mark.gpu
@pytest.mark.parametrize('name', [ALIAS_CASE, 'tv_static_multi_vec_dxy_p4_t300_gaps'])
def test_gpu_cuda_graph_and_eager_agree(name, smpl_assets):
    """the world_dxy base is device state that every replayed iteration advances exactly once: graph and eager agree bit for bit"""
    outs = []
    for graph in (True, False):
        _, _, in_dict, model = _make(name, smpl_assets, use_cuda_graph=graph)
        outs.append(model.optimize(copy.deepcopy(in_dict)))
    for pid in outs[0]['person_data']:
        for k in ['smpl_orient_world', 'root_trans_world', 'root_trans_world_base', 'world_dxy', 'traj_local_dheading', 'kp_2d_pred']:
            np.testing.assert_array_equal(outs[0]['person_data'][pid][k], outs[1]['person_data'][pid][k])
    np.testing.assert_array_equal(outs[0]['cam_pose'], outs[1]['cam_pose'])


@pytest.mark.gpu
def test_gpu_run_dataset_with_heading_vectors(tmp_path):
    """run_dataset --synthetic with heading_type vec and world_dxy: the output pickle holds the vector-shaped heading variables"""
    import pickle
    from glamr_b200.global_recon import run_dataset as rd
    args = rd.parse(['--cfg', cfg_path('glamr_static_multi_vec_world_dxy'), '--out_dir', str(tmp_path), '--synthetic', '1', '--frames', '48',
                     '--gaps', '--quiet'])
    done = rd.run(args)
    assert len(done) == 1 and os.path.exists(done[0][2])
    out = pickle.load(open(done[0][2], 'rb'))
    for pd in out['person_data'].values():
        Ln = int(pd['exist_len'])
        assert pd['traj_local_heading'].shape == (2,) and pd['traj_local_dheading'].shape == (Ln - 1, 2)
        assert pd['world_dxy'].shape == (48, 2) and np.isfinite(pd['world_dxy']).all()
        assert np.isfinite(pd['smpl_orient_world']).all() and np.isfinite(pd['root_trans_world']).all()


@pytest.mark.gpu
def test_gpu_absolute_heading_is_refused(smpl_assets):
    """absolute_heading stays refused, with the reason"""
    from glamr_b200.recon import GlobalReconOptimizer
    cfg = case_config('tv_static_multi_vec_p3_t30_gaps')
    cfg.grecon_model_specs['absolute_heading'] = True
    with pytest.raises(NotImplementedError, match='heading increments'):
        GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=smpl_assets, mt_model=ReplayMT({}, DEV))
