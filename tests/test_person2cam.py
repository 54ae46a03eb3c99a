"""The person2cam residuals (flag_opt_person2cam_rot / _trans, include/glamr_b200.h: has_person2cam, off_p2c_rot, off_p2c_trans): in
the camera-from-persons mode every person's person2cam is composed with [rot6d(person2cam_res_rot) | person2cam_res_trans] before
the camera mean, and Adam optimises the residuals in the stages that list them.

CPU: the oracle against the executed reference (tests/golden/globalopt_p2c_*.npz), the host-compiled frame functions and Adam
against oracle autograd, the residuals' gradients element by element against float64 autograd (a forward-filled frame and a person
invisible on a source frame included), person sharding over two gloo ranks, and the combinations that are refused.  GPU (-m gpu):
the CUDA path against the fixtures' float64 noise floor, iteration-0 gradients against oracle autograd, CUDA graph vs eager, the
launch count, flags without listed variables against flags off, and a run_dataset sweep."""
import copy
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from helpers import ReplayMT, load_golden
from person2cam_cases import (CASES, FAILING_CASES, FINAL_VARS, PERSON2CAM_CASES, case_config, case_in_dict, cfg_path,
                              oracle_class)
from test_traj_sources import _align_half_turns, _compare_grads, _free_port, _noise_tol, _oracle_grads

HERE = os.path.dirname(os.path.abspath(__file__))
ALL = [c[0] for c in PERSON2CAM_CASES]
SMALL = [c[0] for c in PERSON2CAM_CASES if c[3] <= 80]
BOTH = 'p2c_3dpw_p2_t80_gaps'                  # both residuals, listed in both stages
TRANS_REG, NO_OPT_TRAJ = (c[0] for c in FAILING_CASES)
P2C_VARS = ['person2cam_res_rot', 'person2cam_res_trans']
FLAG_KEYS = ['flag_fixed_cam', 'flag_opt_cam', 'flag_opt_cam_from_person_pose', 'flag_cam_inv_trans_res_all', 'flag_opt_vis_local_rot',
             'cam_fix_frames', 'flag_opt_traj', 'flag_opt_person2cam_rot', 'flag_opt_person2cam_trans']


def _setup(name, smpl_assets):
    return load_golden('globalopt_' + name), case_config(name), case_in_dict(name, smpl_assets)


def _p2c_listed(key, opt_variables, flags):
    """get_parameter's rule (:616-619): the flag of that residual is set and the stage lists it"""
    return bool(flags.get(f'flag_opt_{key}', False)) and key in opt_variables


def _grad_views(lay, grad, P, opt_variables, fixed_cam, opt_traj, flags):
    """views of a packed gradient in the order of get_parameter (global_recon_model.py:591-633), person2cam residuals included"""
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
        if _p2c_listed('person2cam_rot', opt_variables, flags):
            order.append(pv['person2cam_res_rot'])
        if _p2c_listed('person2cam_trans', opt_variables, flags):
            order.append(pv['person2cam_res_trans'])
        if 'world_dheading' in opt_variables:
            order.append(pv['world_dheading'])
    return order


def _flags(ora):
    return {k: getattr(ora, k) for k in FLAG_KEYS}


def _emu_runner(ora, data):
    """tests/emu_runner.EmuRunner with the variable layout and the stage compiler told about the person2cam flags"""
    import host_harness as hh
    from emu_runner import EmuRunner
    from glamr_b200 import lib as L
    from glamr_b200 import problem as PB
    from oracle import rotations as rt
    run = EmuRunner.__new__(EmuRunner)
    run.model, run.data = ora, data
    run.flags = _flags(ora)
    run.layout = PB.make_layout(data, run.flags)
    run.theta = torch.zeros(run.layout.n_params)
    PB.bind_variables(data, run.layout, run.theta)
    run.comp = PB.StageCompiler(data, run.layout, run.flags, 'cpu', rt.aa_to_rot6d, aa_to_quat=rt.aa_to_quat)
    run.lib, run.h = hh.lib(), None
    run.reduce = torch.zeros(run.layout.n_params + L.NUM_TERMS)
    return run


def _compiler(cfg, smpl_assets, in_dict, mt_model=None):
    """(oracle data dict, layout, theta, StageCompiler) of a case, as GlobalReconOptimizer builds them"""
    from glamr_b200 import problem as PB
    from oracle import rotations as rt
    ora = oracle_class()(cfg, smpl_assets, mt_model=mt_model)
    data = ora.init_data(copy.deepcopy(in_dict))
    flags = _flags(ora)
    lay = PB.make_layout(data, flags)
    theta = torch.zeros(lay.n_params)
    PB.bind_variables(data, lay, theta)
    return data, lay, theta, PB.StageCompiler(data, lay, flags, 'cpu', rt.aa_to_rot6d, aa_to_quat=rt.aa_to_quat)


# ------------------------------------------------------------------------------------------------ CPU: cases and layout
def test_cases_cover_the_new_variables():
    specs = {c[0]: case_config(c[0]) for c in PERSON2CAM_CASES}
    for name, cfg in specs.items():
        g = cfg.grecon_model_specs
        assert g['flag_opt_cam_from_person_pose'] and g.get('flag_opt_traj', True), name
    both = specs[BOTH]
    for st in both.opt_stage_specs.values():
        assert {'person2cam_rot', 'person2cam_trans'} <= set(st['opt_variables'])
    rot = specs['p2c_3dpw_rot_p3_t30_gaps']
    assert rot.grecon_model_specs['flag_opt_person2cam_rot'] and not rot.grecon_model_specs.get('flag_opt_person2cam_trans', False)
    assert ['person2cam_rot' in st['opt_variables'] for st in rot.opt_stage_specs.values()] == [False, True]
    assert CASES['p2c_3dpw_p4_t300_gaps'][2:4] == (4, 300)
    # every case has frames no person sees (forward-filled camera) and, with several persons, the last one on a strict sub-range
    for name in ALL:
        _, _, P, T, _, _ = CASES[name]
        gold = load_golden('globalopt_' + name)
        if 'init/0/vis_frames' not in gold:
            continue
        vis = np.stack([np.asarray(gold[f'init/{p}/vis_frames'], bool) for p in range(P)])
        assert (~vis.any(0)).sum() >= 5, name
        if P > 1:
            assert not vis[P - 1, :T // 8].any() and not vis[P - 1, T - T // 10:].any(), name


def test_layout_unchanged_without_the_flags(smpl_assets):
    """without either flag (or without flag_opt_traj, which is then a no-op) no block is added: every other problem keeps its
    layout; with a flag each person gets person2cam_res_rot [T,6] and person2cam_res_trans [T,3] at identity / zero"""
    name = 'p2c_3dpw_rot_p3_t30_gaps'
    gold, cfg, in_dict = _setup(name, smpl_assets)
    _, lay_on, theta, _ = _compiler(cfg, smpl_assets, in_dict, ReplayMT(gold))
    off = copy.deepcopy(cfg)
    off.grecon_model_specs['flag_opt_person2cam_rot'] = False
    _, lay_off, _, _ = _compiler(off, smpl_assets, in_dict, ReplayMT(gold))
    T, P = CASES[name][3], CASES[name][2]
    assert not lay_off.person2cam and lay_on.person2cam
    assert lay_on.n_params == lay_off.n_params + 9 * T * P
    for p in range(P):
        pv = lay_on.views(theta, p)
        assert torch.equal(pv['person2cam_res_rot'], torch.tensor([1., 0., 0., 0., 1., 0.]).repeat(T, 1))
        assert torch.equal(pv['person2cam_res_trans'], torch.zeros(T, 3))
        assert 'person2cam_res_rot' not in lay_off.views(torch.zeros(lay_off.n_params), p)


def test_problem_struct_carries_the_new_fields():
    """the ctypes mirror and the C structs agree (host build of the header), and zero leaves person2cam as it is"""
    import host_harness as hh
    from glamr_b200 import lib as L
    assert hh.lib().glamr_host_sizeof_problem() == ctypes.sizeof(L.Problem)
    assert hh.lib().glamr_host_sizeof_person() == ctypes.sizeof(L.Person)
    pb, ps = L.Problem(), L.Person()
    assert pb.has_person2cam == 0 and ps.off_p2c_rot == ps.off_p2c_trans == 0


# ------------------------------------------------------------------------------------------------ CPU: oracle vs reference
@pytest.mark.parametrize('name', ALL)
def test_oracle_matches_reference_golden(name, smpl_assets):
    """init state, iteration-0 gradients of every stage (the residuals' included), per-iteration residuals and the final state
    (world pose, camera, person2cam residuals) of the oracle against the executed reference"""
    Oracle = oracle_class()
    gold, cfg, in_dict = _setup(name, smpl_assets)
    ora = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data = ora.init_data(in_dict)
    for pid, pd in data['person_data'].items():
        for k in ['smpl_orient_world', 'root_trans_world', 'kp_2d_pred']:
            if f'init/{pid}/{k}' in gold:
                np.testing.assert_allclose(pd[k].detach().numpy(), gold[f'init/{pid}/{k}'], atol=1e-3 if k == 'kp_2d_pred' else 1e-5,
                                           err_msg=f'init {pid} {k}')
    first = list(cfg.opt_stage_specs)[0]
    n_p2c = 0
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
            n_p2c += int(tuple(params[i].shape[1:]) in ((6,), (3,)) and params[i].shape[0] == CASES[name][3])
            if stage != first and name not in SMALL:
                # after init_opt's 10 steps at lr 1e-2 over 300 frames the float32 states of two implementations differ by the
                # reference's own amplified rounding (~1e-3 of a local_rot gradient); the losses and the final state below hold
                # them to that noise floor
                continue
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
    assert n_p2c > 0                                     # the residuals were optimised in some stage
    for pid, pd in data['person_data'].items():
        for k in ['smpl_orient_world', 'root_trans_world'] + P2C_VARS:
            if f'final64/{pid}/{k}' in gold:
                r32, r64, rp = gold[f'final/{pid}/{k}'], gold[f'final64/{pid}/{k}'], gold[f'final_pert/{pid}/{k}']
                assert np.abs(pd[k].detach().numpy() - r64).max() <= _noise_tol(r32, r64, rp), f'final {pid} {k}'
    # the residuals moved away from their initial values
    assert any(np.abs(gold[f'final/{pid}/person2cam_res_rot'] - np.array([1., 0., 0., 0., 1., 0.])).max() > 0 for pid in data['person_data'])
    r32, r64, rp = gold['final/cam_pose'], gold['final64/cam_pose'], gold['final_pert/cam_pose']
    assert np.abs(data['cam_pose'].numpy() - r64).max() <= _noise_tol(r32, r64, rp)


# ------------------------------------------------------------------------------------------------ CPU: host-compiled kernels
@pytest.mark.parametrize('name', SMALL)
def test_frame_functions_and_adam_match_oracle_autograd(name, smpl_assets):
    """the frame functions of globalopt_frames.cuh (g++) with the person2cam residuals: every variable's gradient and every
    residual of every stage against autograd through the oracle, then the stage's Adam steps in both"""
    from glamr_b200 import lib as L
    Oracle = oracle_class()
    gold, cfg, in_dict = _setup(name, smpl_assets)
    ora = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data_o = ora.init_data(copy.deepcopy(in_dict))
    ora2 = Oracle(cfg, smpl_assets, mt_model=ReplayMT(gold))
    data_e = ora2.init_data(copy.deepcopy(in_dict))
    run = _emu_runner(ora2, data_e)
    assert run.layout.person2cam
    run.set_stage([], {}, 'init')
    run.backward()
    P, T = run.comp.P, run.comp.T
    flags = _flags(ora)
    for stage, specs in cfg.opt_stage_specs.items():
        variables = specs['opt_variables']
        params = ora.get_parameter(data_o, variables)
        run.set_stage(variables, specs['loss_cfg'], stage)
        assert run.pb.has_person2cam == 1 and run.pb.cam_mode == L.CAM_FROM_PERSONS
        thetas = _grad_views(run.layout, run.theta, P, variables, ora.flag_fixed_cam, ora.flag_opt_traj, flags)
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
            views = _grad_views(run.layout, run.reduce[:run.layout.n_params], P, variables, ora.flag_fixed_cam, ora.flag_opt_traj, flags)
            _compare_grads(views, params, grads, f'{stage} it {it}', 3e-4)
            cam = run.buffer(L.R_CAM_POSE).view(T, 3, 4)
            np.testing.assert_allclose(cam.numpy(), data_o['cam_pose'][:, :3].detach().numpy(), atol=2e-5, err_msg=f'{stage} it {it} camera')
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


def _float64_records(name, assets):
    """host emulator from the oracle's float32 init: the gradient of every variable at the first closure of the stages that list
    the residuals and after their Adam steps, with float64 / float32 oracle autograd at the same state"""
    from test_grad_float64 import oracle_state
    Oracle = oracle_class()
    gold, cfg, in_dict = _setup(name, assets)
    template = Oracle(copy.deepcopy(cfg), assets, mt_model=ReplayMT(gold)).init_data(copy.deepcopy(in_dict))
    ora_e = Oracle(copy.deepcopy(cfg), assets, mt_model=ReplayMT(gold))
    data_e = ora_e.init_data(copy.deepcopy(in_dict))
    run = _emu_runner(ora_e, data_e)
    run.set_stage([], {}, 'init')
    run.backward()
    flags = _flags(ora_e)
    P = run.comp.P
    recs = []
    for stage, specs in cfg.opt_stage_specs.items():
        variables = specs['opt_variables']
        run.set_stage(variables, specs['loss_cfg'], stage)
        for point in ('first', 'stepped'):
            if point == 'stepped':
                for _ in range(specs['opt_niters']):
                    run.backward()
                    run.step(specs['opt_lr'])
            grad, _ = run.backward()
            grad = grad.clone()
            state = oracle_state(template, data_e, run.layout, run.theta)
            refs = {}
            for dtype in (torch.float64, torch.float32):
                ora = Oracle(copy.deepcopy(cfg), assets)
                data = copy.deepcopy(state)
                for pd, pv in zip(data['person_data'].values(), range(P)):
                    for k in P2C_VARS + ['traj_local_xy', 'traj_local_heading', 'traj_local_dxy', 'traj_local_dheading', 'traj_local_z',
                                         'traj_local_rot', 'smpl_orient_world_res', 'root_trans_world_res']:
                        if k in pd:
                            pd[k] = run.layout.views(run.theta, pv)[k].clone()
                gv = run.layout.views(run.theta)
                for k in ['cam_inv_rot_residual', 'cam_inv_trans_residual']:
                    data[k] = gv[k].clone()
                if dtype == torch.float64:
                    data = ora.to_float64(data)
                params = ora.get_parameter(data, variables)
                for prm in params:
                    prm.requires_grad_(True)
                ora.forward(data, variables, {'stage': stage})
                total, _, _ = ora.compute_loss(data, specs['loss_cfg'])
                total.backward()
                refs[dtype] = [None if prm.grad is None else prm.grad.detach().double().numpy() for prm in params]
            views = _grad_views(run.layout, grad, P, variables, ora_e.flag_fixed_cam, ora_e.flag_opt_traj, flags)
            recs.append({'stage': stage, 'point': point, 'grads': [v.numpy().astype(np.float64) for v in views],
                         'g64': refs[torch.float64], 'g32': refs[torch.float32],
                         'p2c_listed': [k for k in ('person2cam_rot', 'person2cam_trans') if _p2c_listed(k, variables, flags)]})
    return recs, data_e


@pytest.mark.parametrize('name', SMALL)
def test_residual_gradients_within_float64_bound(name, smpl_assets):
    """the residuals' gradients element by element against float64 autograd (test_grad_float64's bound): on a frame the camera
    is forward-filled from, a frame filled from another gets nothing of its own, and a person invisible on a source frame gets
    exactly zero there"""
    from test_grad_float64 import violations
    recs, data = _float64_records(name, smpl_assets)
    P, T = CASES[name][2], CASES[name][3]
    npers = sum(np.asarray(d['vis_frames'], np.float64) for d in data['person_data'].values())
    vis = np.stack([np.asarray(d['vis_frames'], bool) for d in data['person_data'].values()])
    filled = np.where(npers == 0)[0]
    assert filled.size, 'the case has no forward-filled frame'
    hidden = [(p, s) for p in range(P) for s in range(T) if npers[s] > 0 and not vis[p, s]]
    assert hidden, 'no person is invisible on a source frame'
    checked = 0
    for r in recs:
        if not r['p2c_listed']:
            continue
        # residual blocks follow each person's trajectory variables (get_parameter order)
        per_person = (len(r['grads']) - 2) // P
        for p in range(P):
            for j, key in enumerate(r['p2c_listed']):
                i = 2 + p * per_person + (per_person - len(r['p2c_listed'])) + j
                g, g64, g32 = r['grads'][i], r['g64'][i], r['g32'][i]
                what = f"{name} {r['stage']} {r['point']} {key}[{p}]"
                assert g64 is not None and g.shape == g64.shape, what
                n_bad, ratio, err, b = violations('person2cam_res', g, g64, g32)
                assert n_bad == 0, f'{what}: {n_bad} elements outside the bound, worst {err:.3e} vs {b:.3e} (x{ratio:.2f})'
                assert not g[filled].any(), f'{what}: forward-filled frames have a gradient of their own'
                for (q, s) in hidden:
                    if q == p:
                        assert not g[s].any(), f'{what}: person {p} invisible on frame {s} has a gradient there'
                assert np.abs(g[vis[p]]).max() > 0, what
                checked += 1
    assert checked >= P


# ------------------------------------------------------------------------------------------------ CPU: refusals
def test_refused_combinations_raise_value_error(smpl_assets):
    """the combinations the reference fails on (its fixtures record the KeyError) raise a ValueError that names the reason"""
    from glamr_b200 import lib as L
    from glamr_b200.synthetic import SyntheticPrior
    gold = load_golden('globalopt_' + TRANS_REG)
    assert 'KeyError' in str(gold['ref_error']) and 'person2cam_res_trans' in str(gold['ref_error'])
    cfg, in_dict = case_config(TRANS_REG), case_in_dict(TRANS_REG, smpl_assets)
    data, lay, theta, comp = _compiler(cfg, smpl_assets, in_dict, SyntheticPrior(seed=23, device='cpu'))
    specs = cfg.opt_stage_specs['init_opt']
    with pytest.raises(ValueError, match='person2cam_res_trans_reg'):
        comp.compile(theta, specs['opt_variables'], specs['loss_cfg'], 'init_opt')
    # flag_opt_traj false: the residuals are never created; the camera-from-persons forward or a listed variable fails
    gold = load_golden('globalopt_' + NO_OPT_TRAJ)
    assert 'KeyError' in str(gold['ref_error']) and 'person2cam_res_rot' in str(gold['ref_error'])
    cfg, in_dict = case_config(NO_OPT_TRAJ), case_in_dict(NO_OPT_TRAJ, smpl_assets)
    data, lay, theta, comp = _compiler(cfg, smpl_assets, in_dict)
    assert not lay.person2cam
    specs = cfg.opt_stage_specs['init_opt']
    loss = {k: v for k, v in specs['loss_cfg'].items() if not k.startswith(('local_traj_', 'traj_rot_res', 'traj_trans_res', 'rel_'))}
    with pytest.raises(ValueError, match='flag_opt_traj'):
        comp.compile(theta, specs['opt_variables'], loss, 'init_opt')
    with pytest.raises(ValueError, match="'person2cam_rot' needs flag_opt_traj"):
        comp.compile(theta, ['cam', 'person2cam_rot'], loss, 'init_opt')
    # otherwise the flag is a no-op, as in the reference: the camera is a variable, the init forward, or only the other residual
    # (whose flag is off) is listed
    assert comp.compile(theta, ['cam'], loss, 'init_opt').cam_mode == L.CAM_PER_FRAME
    assert comp.compile(theta, [], {}, 'init').cam_mode == L.CAM_CONST
    assert comp.compile(theta, ['cam', 'person2cam_trans'], loss, 'init_opt').has_person2cam == 0


def test_listed_variables_without_a_reader_stay_inactive_only_without_flag(smpl_assets):
    """Adam's active ranges: on only with the flag, the stage listing the variable and flag_opt_traj; a stage listing it without
    its flag is ignored"""
    name = 'p2c_3dpw_rot_p3_t30_gaps'
    gold, cfg, in_dict = _setup(name, smpl_assets)
    data, lay, theta, comp = _compiler(cfg, smpl_assets, in_dict, ReplayMT(gold))
    T = CASES[name][3]

    def active(variables):
        pb = comp.compile(theta, variables, {}, 'main_opt')
        a = torch.frombuffer(bytearray(ctypes.string_at(pb.active, lay.n_params)), dtype=torch.uint8)
        o = lay.persons[0]
        return int(a[o['p2c_rot']:o['p2c_rot'] + 6 * T].sum()), int(a[o['p2c_trans']:o['p2c_trans'] + 3 * T].sum())
    assert active(['local_xy']) == (0, 0)
    assert active(['person2cam_rot']) == (6 * T, 0)
    assert active(['person2cam_trans']) == (0, 0)               # its flag is off: ignored, as in get_parameter
    assert active(['cam', 'person2cam_rot']) == (6 * T, 0)      # listed but unread: zero gradient, unchanged by Adam


# ------------------------------------------------------------------------------------------------ CPU: two ranks
def _gloo_worker(rank, world, port, name, ret):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import torch.distributed as dist
    os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    torch.set_num_threads(1)
    from glamr_b200.synthetic import make_smpl_assets
    Oracle = oracle_class()
    assets = make_smpl_assets(0)
    gold, cfg, in_dict = _setup(name, assets)
    results = {}
    for mode in ['single', 'sharded']:
        ora = Oracle(copy.deepcopy(cfg), assets, mt_model=ReplayMT(gold))
        run = _emu_runner(ora, ora.init_data(copy.deepcopy(in_dict)))
        stage, specs = list(cfg.opt_stage_specs.items())[-1]
        assert 'person2cam_rot' in specs['opt_variables']
        N = run.comp.P * run.comp.T
        kw = {} if mode == 'single' else dict(n_begin=N * rank // world, n_end=N * (rank + 1) // world, owner=(rank == 0))
        run.set_stage(specs['opt_variables'], specs['loss_cfg'], stage, **kw)
        for it in range(3):
            run.backward()
            if mode == 'sharded':
                dist.all_reduce(run.reduce)
            run.step(specs['opt_lr'])
        g = torch.cat([torch.cat([run.layout.views(run.reduce, p)[k].reshape(-1) for k in P2C_VARS]) for p in range(run.comp.P)])
        results[mode] = (run.reduce.clone(), run.theta.clone(), g)
    g_err = float((results['single'][0] - results['sharded'][0]).abs().max() / results['single'][0].abs().max())
    t_err = float((results['single'][1] - results['sharded'][1]).abs().max())
    r_err = float((results['single'][2] - results['sharded'][2]).abs().max() / results['single'][2].abs().max())
    ret[rank] = (g_err, t_err, r_err, float(results['single'][2].abs().max()))
    dist.barrier()
    dist.destroy_process_group()


def test_person_sharding_with_person2cam_equals_single_rank():
    """frame-persons split over two gloo ranks (person 1 straddles them): each rank pushes its share of dL/d(camera mean) into the
    residuals, and the summed gradients and the parameters after 3 Adam steps equal the single-rank run"""
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ret = mp.get_context('spawn').Manager().dict()
    mp.spawn(_gloo_worker, args=(world, port, 'p2c_3dpw_rot_p3_t30_gaps', ret), nprocs=world, join=True)
    for rank in range(world):
        g_err, t_err, r_err, r_max = ret[rank]
        assert r_max > 0, 'the residuals have no gradient'
        assert g_err < 1e-5, f'rank {rank}: reduced gradient differs from single-rank by {g_err:.2e} (relative)'
        assert r_err < 1e-5, f'rank {rank}: reduced residual gradient differs from single-rank by {r_err:.2e} (relative)'
        assert t_err < 1e-5, f'rank {rank}: parameters after 3 steps differ by {t_err:.2e}'


# ------------------------------------------------------------------------------------------------ GPU
DEV = 'cuda:0'


def _make(name, smpl_assets, cfg=None, **spec_over):
    from glamr_b200.recon import GlobalReconOptimizer
    gold, cfg0, in_dict = _setup(name, smpl_assets)
    cfg = cfg0 if cfg is None else cfg
    cfg.grecon_model_specs.update(spec_over)
    model = GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=smpl_assets, mt_model=ReplayMT(gold, DEV))
    return gold, cfg, in_dict, model


@pytest.mark.gpu
@pytest.mark.parametrize('name', ALL)
def test_gpu_trajectory_matches_reference_golden(name, smpl_assets):
    """per-iteration residual values and the final state (world pose, camera, keypoints, person2cam residuals) vs the executed
    reference, at its float64 noise floor"""
    from glamr_b200 import lib as L
    gold, cfg, in_dict, model = _make(name, smpl_assets)
    data = model.init_data(copy.deepcopy(in_dict))
    _align_half_turns(model, data, gold)
    np.testing.assert_allclose(data['cam_pose'].cpu().numpy(), gold['init/cam_pose'], atol=1e-5)
    first = list(cfg.opt_stage_specs)[0]
    for stage, specs in cfg.opt_stage_specs.items():
        n = specs['opt_niters']
        model.optimize_main(data, specs['opt_variables'], specs['opt_lr'], n, specs['loss_cfg'], {'stage': stage})
        hist = model.loss_history.cpu().numpy()
        for k in specs['loss_cfg']:
            r32, r64, rp = gold[f'loss/{stage}/{k}'], gold[f'loss64/{stage}/{k}'], gold[f'loss_pert/{stage}/{k}']
            got = hist[:n, L.TERM_INDEX[k]]
            if specs['loss_cfg'][k].get('monitor_only', False):
                # kp_2d_dist: un-robust pixel distances that feed nothing.  Once the camera moves with the persons' residuals a
                # keypoint can come close to the image plane, where a distance amplifies any rounding without bound: checked where
                # the states still agree, at the first iteration of the first stage
                if stage == first:
                    np.testing.assert_allclose(got[:1], r64[:1], rtol=5e-4, atol=1e-6, err_msg=f'{stage} {k} (iteration 0)')
                continue
            if stage == first:
                np.testing.assert_allclose(got[:1], r64[:1], rtol=2e-4, atol=1e-6, err_msg=f'{stage} {k} (iteration 0)')
            tol = 4.0 * max(np.abs(r32 - r64).max(), np.abs(rp - r32).max()) + 2e-4 * np.abs(r64).max() + 1e-6
            err = np.abs(got - r64).max()
            assert err <= tol, f'{stage} {k}: |cuda-ref64| {err:.3e} > {tol:.3e}'
    checks = [('cam_pose', data['cam_pose'].cpu().numpy())]
    for pid, pd in data['person_data'].items():
        for k in ['smpl_orient_world', 'root_trans_world', 'kp_2d_pred'] + P2C_VARS:
            if k in pd and f'final64/{pid}/{k}' in gold:
                checks.append((f'{pid}/{k}', pd[k].cpu().numpy()))
    assert sum(k.endswith('person2cam_res_rot') for k, _ in checks) == len(data['person_data'])
    # the camera is the mean over the persons, so one person's rounding moves every other person through it: a person's own
    # noise can be far below what a rounding anywhere does to it.  The reference's response to one rounding of its init state,
    # taken over all persons, is that yardstick (the float64 run is left out: it can wrap an axis-angle vector by 2 pi)
    pids = list(data['person_data'])
    shared = {k: max(float(np.abs(gold[f'final_pert/{pid}/{k}'] - gold[f'final/{pid}/{k}']).max()) for pid in pids)
              for k in ['smpl_orient_world', 'root_trans_world', 'kp_2d_pred'] + P2C_VARS if f'final_pert/{pids[0]}/{k}' in gold}
    for key, got in checks:
        r32, r64, rp = gold[f'final/{key}'], gold[f'final64/{key}'], gold[f'final_pert/{key}']
        tol = _noise_tol(r32, r64, rp, ulps=256 if 'kp_2d_pred' in key else 32)
        name_ = key.split('/')[-1]
        tol = max(tol, 4.0 * shared.get(name_, 0.0))
        if name_ in ('cam_pose', 'smpl_orient_world', 'root_trans_world'):
            tol = max(tol, 1e-4)                         # the north-star bound on output poses (m, rad)
        elif name_ == 'kp_2d_pred':
            tol = max(tol, 2e-2)                         # pixels: 1e-4 m at f / z = 1000 / 5
        err = float(np.abs(got.reshape(r64.shape) - r64).max())
        assert err <= tol, f'final {key}: |cuda-ref64| {err:.3e} > {tol:.3e}'


@pytest.mark.gpu
@pytest.mark.parametrize('name', SMALL)
def test_gpu_gradients_match_oracle_autograd(name, smpl_assets):
    """first closure of every stage: every variable's gradient (the residuals' included) and every residual vs autograd through the
    full-LBS oracle"""
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
        views = _grad_views(model._layout, grad, P, specs['opt_variables'], model.flag_fixed_cam, model.flag_opt_traj, model._flags)
        _compare_grads(views, params, grads, stage, 5e-4)
        # advance the stage on the GPU and hand its variables to the oracle: the next stage starts from identical state
        model.optimize_main(data, specs['opt_variables'], specs['opt_lr'], specs['opt_niters'], specs['loss_cfg'], {'stage': stage})
        for pd, po in zip(data['person_data'].values(), data_o['person_data'].values()):
            for k in ['traj_local_xy', 'traj_local_dxy', 'traj_local_heading', 'traj_local_dheading', 'traj_local_z', 'traj_local_rot',
                      'smpl_orient_world_res', 'root_trans_world_res'] + P2C_VARS:
                if k in pd and k in po:
                    po[k] = pd[k].detach().cpu().clone()
        for k in ['cam_pose', 'cam_pose_inv', 'cam_inv_rot_residual', 'cam_inv_trans_residual']:
            data_o[k] = data[k].detach().cpu().clone()


@pytest.mark.gpu
def test_gpu_cuda_graph_and_eager_agree(smpl_assets):
    """a replayed iteration graph and eager iterations give the same bits, residuals included"""
    outs = []
    for graph in (True, False):
        _, _, in_dict, model = _make('p2c_3dpw_p4_t300_gaps', smpl_assets, use_cuda_graph=graph)
        outs.append(model.optimize(copy.deepcopy(in_dict)))
    for pid in outs[0]['person_data']:
        for k in ['smpl_orient_world', 'root_trans_world', 'kp_2d_pred'] + P2C_VARS:
            np.testing.assert_array_equal(outs[0]['person_data'][pid][k], outs[1]['person_data'][pid][k])
    np.testing.assert_array_equal(outs[0]['cam_pose'], outs[1]['cam_pose'])


def _flags_off(cfg):
    off = copy.deepcopy(cfg)
    off.grecon_model_specs['flag_opt_person2cam_rot'] = off.grecon_model_specs['flag_opt_person2cam_trans'] = False
    return off


def _unlisted(cfg):
    out = copy.deepcopy(cfg)
    for st in out.opt_stage_specs.values():
        st['opt_variables'] = [v for v in st['opt_variables'] if not v.startswith('person2cam_')]
    return out


@pytest.mark.gpu
def test_gpu_launch_count_is_unchanged(smpl_assets):
    """the residuals add arithmetic to the camera kernels, not a launch"""
    counts = []
    for over in (lambda c: c, _flags_off):
        gold, cfg, in_dict = _setup(BOTH, smpl_assets)
        _, cfg, in_dict, model = _make(BOTH, smpl_assets, cfg=over(cfg))
        data = model.init_data(copy.deepcopy(in_dict))
        specs = cfg.opt_stage_specs['main_opt']
        model.optimize_main(data, specs['opt_variables'], specs['opt_lr'], 1, specs['loss_cfg'], {'stage': 'main_opt'})
        counts.append(model.launches_per_iteration())
    assert counts[0] == counts[1]


def _walk(a, b, path=''):
    """every array of two output dicts bit-identical (NaN equal to NaN)"""
    if isinstance(a, dict):
        assert set(a) == set(b), path
        for k in a:
            _walk(a[k], b[k], f'{path}/{k}')
    elif isinstance(a, np.ndarray):
        np.testing.assert_array_equal(a, b, err_msg=path)


@pytest.mark.gpu
def test_gpu_flags_without_listed_variables_equal_flags_off(smpl_assets):
    """glamr_3dpw with both flags set but neither residual listed: the residuals stay at identity / zero, every product with them
    is exact, and every output array equals the run with the flags off bit for bit (the residuals' own keys aside)"""
    outs = []
    for over in (_unlisted, lambda c: _flags_off(_unlisted(c))):
        gold, cfg, in_dict = _setup('p2c_3dpw_p4_t300_gaps', smpl_assets)
        _, cfg, in_dict, model = _make('p2c_3dpw_p4_t300_gaps', smpl_assets, cfg=over(cfg))
        outs.append(model.optimize(copy.deepcopy(in_dict)))
    for pid, pd in outs[0]['person_data'].items():
        np.testing.assert_array_equal(pd.pop('person2cam_res_rot'), np.tile([1., 0., 0., 0., 1., 0.], (300, 1)).astype(np.float32))
        np.testing.assert_array_equal(pd.pop('person2cam_res_trans'), np.zeros((300, 3), np.float32))
        assert 'person2cam_res_rot' not in outs[1]['person_data'][pid]
    out = {k: v for k, v in outs[0].items() if k != 'meta'}
    _walk(out, {k: v for k, v in outs[1].items() if k != 'meta'})


@pytest.mark.gpu
def test_gpu_run_dataset_with_person2cam(tmp_path):
    """run_dataset --synthetic with a person2cam config: the output pickle holds every person's residuals"""
    import pickle
    from glamr_b200.global_recon import run_dataset as rd
    args = rd.parse(['--cfg', cfg_path('glamr_3dpw_person2cam'), '--out_dir', str(tmp_path), '--synthetic', '1', '--frames', '48',
                     '--gaps', '--quiet'])
    done = rd.run(args)
    assert len(done) == 1 and os.path.exists(done[0][2])
    out = pickle.load(open(done[0][2], 'rb'))
    for pd in out['person_data'].values():
        assert pd['person2cam_res_rot'].shape == (48, 6) and pd['person2cam_res_trans'].shape == (48, 3)
        assert np.isfinite(pd['person2cam_res_rot']).all() and np.isfinite(pd['person2cam_res_trans']).all()
        assert np.abs(pd['person2cam_res_rot'] - np.array([1., 0., 0., 0., 1., 0.])).max() > 0
