"""Parity of the CUDA path (through the C-ABI library) against the oracle and the reference-generated golden
fixtures.  Runs on an H100:  python -m pytest tests -m gpu"""
import copy
import ctypes

import numpy as np
import pytest
import torch

from helpers import BENCH_SHAPE_CASES, GLOBALOPT_CASES, ReplayMT, case_setup, load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _cuda(x):
    return torch.tensor(x, device=DEV)


# ------------------------------------------------------------------------------------------------ rotation algebra
def test_rowops_match_reference_golden():
    from glamr_b200 import geometry as G
    g = load_golden('rotations')
    aa, d6, R, q, qn, q2, y, x = [_cuda(g[k]) for k in ['in_aa', 'in_d6', 'in_R', 'in_q', 'in_qn', 'in_q2', 'in_y', 'in_x']]
    M = G.make_transform(aa, d6[:, :3].contiguous(), 'axis_angle')
    got = {
        'aa_to_rotmat': G.angle_axis_to_rotation_matrix(aa), 'rotmat_to_quat': G.rotation_matrix_to_quaternion(R),
        'quat_to_aa': G.quaternion_to_angle_axis(qn), 'quat_to_aa_raw': G.quaternion_to_angle_axis(q),
        'aa_to_quat': G.angle_axis_to_quaternion(aa), 'quat_to_rotmat': G.quaternion_to_rotation_matrix(q),
        'rotmat_to_aa': G.rotation_matrix_to_angle_axis(R), 'quat_mul': G.quat_mul(qn, q2), 'quat_angle_diff': G.quat_angle_diff(qn, q2),
        'safe_atan2': G.safe_atan2(y, x), 'rot6d_to_rotmat': G.rot6d_to_rotmat(d6), 'aa_to_rot6d': G.angle_axis_to_rot6d(aa),
        'rot6d_to_quat': G.rot6d_to_quat(d6), 'get_heading': G.get_heading(qn), 'get_heading_q': G.get_heading_q(qn),
        'heading_to_quat': G.heading_to_quat(y), 'deheading_quat': G.deheading_quat(qn), 'make_transform_aa': M,
        'inverse_transform': G.inverse_transform(M), 'transform_rot': G.transform_rot(M, aa.flip(0).contiguous()),
        'transform_trans': G.transform_trans(M, d6[:, 3:].contiguous()),
    }
    for k, v in got.items():
        np.testing.assert_allclose(v.cpu().numpy(), g[k], rtol=0, atol=5e-6, err_msg=k)


def test_rowop_vjps_match_autograd():
    from glamr_b200 import lib as L
    from oracle import rotations as rt
    from oracle.smpl import rodrigues_smplx
    gen = torch.Generator().manual_seed(1)
    aa = torch.randn(512, 3, generator=gen)
    aa[:16] *= 1e-4
    aa[16:20] = 0.0
    cases = [(L.ROP_AA_TO_ROTMAT, aa, lambda a: rt.aa_to_rotmat(a).reshape(-1, 9)),
             (L.ROP_AA_TO_QUAT, aa, rt.aa_to_quat),
             (L.ROP_RODRIGUES_SMPLX, aa[20:], lambda a: rodrigues_smplx(a).reshape(-1, 9)),
             (L.ROP_ROT6D_TO_ROTMAT, torch.randn(512, 6, generator=gen), lambda a: rt.rot6d_to_rotmat(a).reshape(-1, 9)),
             (L.ROP_QUAT_TO_AA, torch.nn.functional.normalize(torch.randn(512, 4, generator=gen), dim=-1), rt.quat_to_aa),
             (L.ROP_ROTMAT_TO_AA, (rt.aa_to_rotmat(torch.randn(512, 3, generator=gen)) + 1e-3 * torch.randn(512, 3, 3, generator=gen)).reshape(-1, 9),
              lambda a: rt.rotmat_to_aa(a.reshape(-1, 3, 3)))]
    for op, a, fn in cases:
        a = a.clone().requires_grad_(True)
        ref = fn(a)
        go = torch.randn(ref.shape, generator=gen)
        (gref,) = torch.autograd.grad(ref, a, go)
        out = L.rowop(op, a.detach().to(DEV))
        np.testing.assert_allclose(out.cpu().numpy(), ref.detach().numpy(), atol=5e-6, err_msg=f'op {op} fwd')
        ga, _ = L.rowop_vjp(op, a.detach().to(DEV), None, go.to(DEV))
        scale = np.maximum(np.abs(gref.numpy()).max(axis=1, keepdims=True), 1.0)
        assert (np.abs(ga.cpu().numpy() - gref.numpy()) / scale).max() < 3e-4, f'op {op} vjp'


# ------------------------------------------------------------------------------------------------ SMPL
def _default_lbs_path():
    return -1        # library default: GLAMR_LBS_PATH, else GLAMR_DEFAULT_LBS_TC in csrc/common.cuh


LBS_PATHS = {'tensor_core': 2, 'tensor_core_blend_simt_skin': 1, 'simt': 0}


@pytest.fixture(params=list(LBS_PATHS))
def lbs_path(request):
    """the implementations of the blend + skinning: wgmma 3xTF32 blend GEMM + wgmma skinning, the same blend with the SIMT
    skinning kernel, and the single FP32 SIMT kernel"""
    from glamr_b200 import lib as L
    L.check(L.load().glamr_smpl_set_lbs_path(LBS_PATHS[request.param]), 'set_lbs_path')
    yield request.param
    L.check(L.load().glamr_smpl_set_lbs_path(_default_lbs_path()), 'set_lbs_path')


def test_smpl_forward_matches_reference_golden(smpl_assets, lbs_path):
    from glamr_b200.smpl import SMPL
    g = load_golden('smpl')
    smpl = SMPL(smpl_assets, pose_type='body26fk', device=DEV)
    o, p, b, t, s = [_cuda(g[k]) for k in ['in_orient', 'in_pose', 'in_betas', 'in_trans', 'in_scale']]
    vsel = g['vsel']
    out = smpl(global_orient=o, body_pose=p, betas=b, root_trans=t)
    np.testing.assert_allclose(out.joints.cpu().numpy(), g['joints'], atol=1e-4)       # north-star bound; expect ~1e-6
    assert np.abs(out.joints.cpu().numpy() - g['joints']).max() < 2e-5
    np.testing.assert_allclose(out.vertices[:, vsel].cpu().numpy(), g['verts_sel'], atol=2e-5)
    np.testing.assert_allclose(out.vertices.double().sum(1).cpu().numpy(), g['verts_sum'], atol=5e-3)
    np.testing.assert_allclose(out.vertices.double().abs().sum(1).cpu().numpy(), g['verts_abs_sum'], rtol=2e-6)
    out = smpl(global_orient=o, body_pose=p, betas=b, root_trans=t, root_scale=s)
    np.testing.assert_allclose(out.joints.cpu().numpy(), g['joints_scaled'], atol=2e-5)
    np.testing.assert_allclose(out.vertices[:, vsel].cpu().numpy(), g['verts_scaled_sel'], atol=2e-5)
    out = smpl(global_orient=o, body_pose=p, betas=b)
    np.testing.assert_allclose(out.joints.cpu().numpy(), g['joints_raw'], atol=2e-5)
    np.testing.assert_allclose(out.vertices[:, vsel].cpu().numpy(), g['verts_raw_sel'], atol=2e-5)
    out = smpl(global_orient=o, body_pose=p, betas=b, root_trans=t, orig_joints=True)
    np.testing.assert_allclose(out.joints.cpu().numpy(), g['joints24'], atol=2e-5)
    np.testing.assert_allclose(out.vertices[:, vsel].cpu().numpy(), g['verts24_sel'], atol=2e-5)
    np.testing.assert_allclose(smpl.get_joints(body_pose=p, global_orient=o, root_trans=t).cpu().numpy(), g['fk_joints'], atol=2e-5)


@pytest.mark.parametrize('n', [1, 31, 32, 33, 300, 1000])
def test_smpl_forward_matches_oracle_ragged_sizes(n, smpl_assets, lbs_path):
    """frame counts around the 32-frame CTA tile, all 6890 vertices compared"""
    from glamr_b200.smpl import SMPL
    from oracle.smpl import OracleSMPL
    smpl = SMPL(smpl_assets, pose_type='body26fk', device=DEV)
    ora = OracleSMPL(smpl_assets)
    gen = torch.Generator().manual_seed(n)
    o, p = torch.randn(n, 3, generator=gen), torch.randn(n, 69, generator=gen) * 0.4
    b, t = torch.randn(n, 10, generator=gen), torch.randn(n, 3, generator=gen)
    out = smpl(global_orient=o.to(DEV), body_pose=p.to(DEV), betas=b.to(DEV), root_trans=t.to(DEV))
    m = min(n, 64)
    j, v = ora(o[:m], p[:m], b[:m], root_trans=t[:m])
    assert (out.joints[:m].cpu() - j).abs().max() < 2e-5
    assert (out.vertices[:m].cpu() - v).abs().max() < 2e-5
    if n > 64:
        j, v = ora(o[-8:], p[-8:], b[-8:], root_trans=t[-8:])
        assert (out.joints[-8:].cpu() - j).abs().max() < 2e-5
        assert (out.vertices[-8:].cpu() - v).abs().max() < 2e-5


def test_smpl_tensor_core_and_simt_paths_agree(smpl_assets):
    """all 6890 vertices of 300 frame-persons: 3xTF32 tensor-core blend vs the FP32 FMA kernel"""
    from glamr_b200 import lib as L
    from glamr_b200.smpl import SMPL
    smpl = SMPL(smpl_assets, pose_type='body26fk', device=DEV)
    gen = torch.Generator().manual_seed(11)
    n = 300
    o, p = torch.randn(n, 3, generator=gen).to(DEV), (torch.randn(n, 69, generator=gen) * 0.4).to(DEV)
    b, t = torch.randn(n, 10, generator=gen).to(DEV), torch.randn(n, 3, generator=gen).to(DEV)
    outs = []
    for path in (2, 1, 0):
        L.check(L.load().glamr_smpl_set_lbs_path(path), 'set_lbs_path')
        r = smpl(global_orient=o, body_pose=p, betas=b, root_trans=t)
        outs.append((r.joints.clone(), r.vertices.clone()))
    L.check(L.load().glamr_smpl_set_lbs_path(_default_lbs_path()), 'set_lbs_path')
    for name, k in (('tensor-core blend + skinning', 0), ('tensor-core blend + SIMT skinning', 1)):
        dj, dv = (outs[k][0] - outs[2][0]).abs().max().item(), (outs[k][1] - outs[2][1]).abs().max().item()
        print(f'{name} vs SIMT: joints {dj:.2e}, vertices {dv:.2e}')
        assert dj < 5e-6 and dv < 5e-6


def test_smpl_dense_skinning_model(smpl_assets, lbs_path):
    """a model whose skinning weights are dense (24 per vertex) takes the generic-K kernel"""
    from glamr_b200.smpl import SMPL
    from oracle.smpl import OracleSMPL
    a = dict(smpl_assets)
    rng = np.random.default_rng(5)
    w = rng.random((6890, 24)).astype(np.float32)
    a['lbs_weights'] = w / w.sum(1, keepdims=True)
    smpl, ora = SMPL(a, device=DEV), OracleSMPL(a)
    gen = torch.Generator().manual_seed(0)
    o, p, b, t = torch.randn(5, 3, generator=gen), torch.randn(5, 69, generator=gen) * 0.3, torch.randn(5, 10, generator=gen), torch.randn(5, 3, generator=gen)
    out = smpl(global_orient=o.to(DEV), body_pose=p.to(DEV), betas=b.to(DEV), root_trans=t.to(DEV))
    j, v = ora(o, p, b, root_trans=t)
    assert (out.joints.cpu() - j).abs().max() < 2e-5 and (out.vertices.cpu() - v).abs().max() < 2e-5


# ------------------------------------------------------------------------------------------------ global optimisation
def _make(name, smpl_assets, **spec_over):
    from glamr_b200.recon import GlobalReconOptimizer
    gold, cfg, in_dict = case_setup(name, smpl_assets)
    cfg.grecon_model_specs.update(spec_over)
    model = GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=smpl_assets, mt_model=ReplayMT(gold, DEV))
    return gold, cfg, in_dict, model


EPS32 = 2.0 ** -24


def noise_floor_tol(ref32, ref64, ref_pert=None, c=4.0, ulps=32):
    """Tolerance of a k-step comparison against the float64 continuation stored in the fixture: `c` times the larger of the two
    noise yardsticks the fixture carries, plus `ulps` float32 roundings of the tensor's magnitude (prefix sums over T frames):
      |ref32 - ref64|    what the executed float32 reference itself deviates from its float64 continuation (rounding INSIDE the loop)
      |ref_pert - ref32| what ONE float32 rounding of the init state does to the float32 reference (any re-implementation enters
                         the loop with such differences; Adam's m / sqrt(v) turns a relative gradient change eps into ~lr * k * eps)
    Where the optimisation is well conditioned this is ~1e-6..1e-5, far below the 1e-4 north-star bound; where Adam amplifies
    rounding noise (frames without observations) it is as loose as the reference's own float32 arithmetic is -- and no looser."""
    noise = float(np.abs(ref32 - ref64).max())
    if ref_pert is not None:
        noise = max(noise, float(np.abs(ref_pert - ref32).max()))
    return c * noise + ulps * EPS32 * max(float(np.abs(ref64).max()), 1.0)


def _check_init_state(data, gold):
    for p, (pid, pd) in enumerate(data['person_data'].items()):
        np.testing.assert_allclose(pd['kp_2d_pred'].cpu().numpy(), gold[f'init/{pid}/kp_2d_pred'], atol=5e-3, err_msg='init kp')
        np.testing.assert_allclose(pd['smpl_orient_world'].cpu().numpy(), gold[f'init/{pid}/smpl_orient_world'], atol=1e-4)
        np.testing.assert_allclose(pd['root_trans_world'].cpu().numpy(), gold[f'init/{pid}/root_trans_world'], atol=1e-4)
        np.testing.assert_allclose(pd['traj_local_pred'].cpu().numpy(), gold[f'init/{pid}/traj_local_pred'], atol=1e-5)
    np.testing.assert_allclose(data['cam_pose'].cpu().numpy(), gold['init/cam_pose'], atol=1e-5)


def _check_trajectory_against_noise_floor(model, data, cfg, gold):
    """every stage: per-iteration residual values; after the last stage: final variables and poses of ALL frames
    (observed or not), each against the float64 continuation with the reference's own float32 deviation as yardstick"""
    from glamr_b200 import lib as L
    report = {}
    for stage, specs in cfg.opt_stage_specs.items():
        n = specs['opt_niters']
        model.optimize_main(data, specs['opt_variables'], specs['opt_lr'], n, specs['loss_cfg'], {'stage': stage})
        if specs.get('reinitialize_cam', False):
            from glamr_b200 import geometry as G
            data['cam_pose'][:] = data['cam_pose'][[0]]
            data['cam_pose_inv'] = G.inverse_transform(data['cam_pose'])
        hist = model.loss_history.cpu().numpy()
        for k in specs['loss_cfg']:
            r32, r64, rp = gold[f'loss/{stage}/{k}'], gold[f'loss64/{stage}/{k}'], gold[f'loss_pert/{stage}/{k}']
            got = hist[:n, L.TERM_INDEX[k]]
            # iteration 0 is a pure forward on identical variables
            np.testing.assert_allclose(got[:1], r64[:1], rtol=2e-4, atol=1e-6, err_msg=f'{stage} {k} (iteration 0)')
            tol = 4.0 * max(np.abs(r32 - r64).max(), np.abs(rp - r32).max()) + 2e-4 * np.abs(r64).max() + 1e-6
            err = np.abs(got - r64).max()
            assert err <= tol, f'{stage} {k}: |cuda-ref64| {err:.3e} > {tol:.3e} (|ref32-ref64| {np.abs(r32 - r64).max():.3e})'
    checks = [('cam_pose', data['cam_pose'].cpu().numpy())]
    for pid, pd in data['person_data'].items():
        for k in ['smpl_orient_world', 'root_trans_world', 'traj_local_xy', 'traj_local_dxy', 'traj_local_z', 'traj_local_rot',
                  'traj_local_heading', 'world_dheading', 'kp_2d_pred']:
            if k in pd and f'final64/{pid}/{k}' in gold:
                checks.append((f'{pid}/{k}', pd[k].cpu().numpy()))
    for key, got in checks:
        r32, r64, rp = gold[f'final/{key}'], gold[f'final64/{key}'], gold[f'final_pert/{key}']
        tol = noise_floor_tol(r32, r64, rp, ulps=32 if 'kp_2d_pred' not in key else 256)
        # The north star asks for joints / vertices / camera within 1e-4 (metres, radians): the derived bar is never tighter than
        # that for the OUTPUT poses (a person 5 m from the camera turns 1e-5 rad of its orientation into 5e-5 m of the camera
        # derived from it, glamr_3dpw), while the optimisation variables themselves keep the derived bar.
        name_ = key.split('/')[-1]
        if name_ in ('cam_pose', 'smpl_orient_world', 'root_trans_world'):
            tol = max(tol, 1e-4)
        elif name_ == 'kp_2d_pred':
            tol = max(tol, 2e-2)          # pixels: 1e-4 m at f / z = 1000 / 5
        err = float(np.abs(got.reshape(r64.shape) - r64).max())
        report[key] = (err, max(float(np.abs(r32 - r64).max()), float(np.abs(rp - r32).max())))
        assert err <= tol, f'final {key}: |cuda-ref64| {err:.3e} > {tol:.3e} (|ref32-ref64| {np.abs(r32 - r64).max():.3e})'
    return report


@pytest.mark.parametrize('name', GLOBALOPT_CASES + BENCH_SHAPE_CASES)
def test_globalopt_matches_reference_golden(name, smpl_assets):
    """init state, per-iteration residual values and the final state of every frame vs the executed reference.  The small
    cases cover every camera mode / config family; the BENCH_SHAPE cases are the shapes bench.py times (1 x 300
    glamr_dynamic with 50 iterations, the 4 x 300 glamr_static_multi north-star video, T = 500, and a T = 600 track with
    gaps that needs two chunks of the CTA-wide prefix scans)."""
    gold, cfg, in_dict, model = _make(name, smpl_assets)
    data = model.init_data(copy.deepcopy(in_dict))
    _check_init_state(data, gold)
    report = _check_trajectory_against_noise_floor(model, data, cfg, gold)
    worst = max(report.items(), key=lambda kv: kv[1][0] / max(kv[1][1], 1e-9))
    print(f'{name}: worst ratio |cuda-ref64| / |ref32-ref64| at {worst[0]}: {worst[1][0]:.2e} / {worst[1][1]:.2e}')


@pytest.mark.parametrize('name', ['dynamic_p1_t40', 'static_multi_p3_t30', '3dpw_p2_t80_gaps'])
def test_globalopt_gradients_match_oracle_autograd(name, smpl_assets):
    """first closure of every stage: every variable's gradient vs torch autograd through the full-LBS oracle"""
    _check_gradients(name, smpl_assets)


def _extra_terms_dynamic(cfg):
    """residuals the registry offers but no shipped config enables (loss_func.py:60-73,94-103,135-144,175-186,216-218),
    switched on next to the shipped ones: per-frame camera variables"""
    for st in cfg.opt_stage_specs.values():
        st['opt_variables'] = list(st['opt_variables']) + ['local_dheading', 'local_dxy', 'local_z']
        st['loss_cfg'].update({'cam_rot_smoothness': {'weight': 2.0}, 'cam_trans_smoothness': {'weight': 3.0}, 'cam_depth_smoothness': {'weight': 1.5},
                               'cam_traj_trans': {'weight': 4.0, 'first_frame_weight': 2.0}, 'traj_trans_smoothness': {'weight': 0.7},
                               'local_traj_dheading_reg': {'weight': 5.0}})


def _extra_terms_world_res(cfg):
    """traj_rot_res / traj_trans_res (loss_func.py:204-209) need the 'world_res' variables (global_recon_model.py:452-454,
    :609-611); world_dheading would override them (:459-465), so it is dropped from the variable list"""
    for st in cfg.opt_stage_specs.values():
        st['opt_variables'] = [v for v in st['opt_variables'] if v != 'world_dheading'] + ['world_res']
        st['loss_cfg'].update({'traj_rot_res': {'weight': 3.0}, 'traj_trans_res': {'weight': 2.0}, 'cam_traj_trans': {'weight': 1.0},
                               'traj_trans_smoothness': {'weight': 0.5}, 'cam_depth_smoothness': {'weight': 1.0}})


@pytest.mark.parametrize('name,mutate', [('dynamic_p1_t40', _extra_terms_dynamic), ('static_multi_p3_t30', _extra_terms_world_res),
                                         ('3dpw_p2_t80_gaps', _extra_terms_world_res)])
def test_unshipped_residual_terms_match_oracle_autograd(name, mutate, smpl_assets):
    """the 8 registered-but-unshipped residuals on the GPU: values and every variable's gradient vs the oracle's autograd,
    then the stage's Adam steps in both (so the second stage starts from a moved state)"""
    _check_gradients(name, smpl_assets, mutate=mutate)


def _check_gradients(name, smpl_assets, mutate=None):
    from glamr_b200 import lib as L
    from glamr_b200.recon import GlobalReconOptimizer
    from oracle.global_opt import OracleGlobalRecon
    gold, cfg, in_dict = case_setup(name, smpl_assets)
    if mutate is not None:
        mutate(cfg)
    model = GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=smpl_assets, mt_model=ReplayMT(gold, DEV))
    data = model.init_data(copy.deepcopy(in_dict))
    ora = OracleGlobalRecon(copy.deepcopy(cfg), smpl_assets, mt_model=ReplayMT(gold))
    data_o = ora.init_data(copy.deepcopy(in_dict))
    for stage, specs in cfg.opt_stage_specs.items():
        params = ora.get_parameter(data_o, specs['opt_variables'])
        for p_ in params:
            p_.requires_grad_(True)
            p_.grad = None
        ora.forward(data_o, specs['opt_variables'], {'stage': stage})
        total, _, uw = ora.compute_loss(data_o, specs['loss_cfg'])
        total.backward()
        model._cur_vars, model._cur_stage = specs['opt_variables'], stage
        model._set_stage(data, specs['opt_variables'], specs['loss_cfg'], stage, reset_adam=True, begin=True)
        model._backward()
        # un-normalised term sums ride behind the gradient in the reduce buffer: compare every enabled term's value
        with torch.cuda.device(DEV):
            L.check(model._lib.glamr_opt_losses(model._opt, L.ptr(model._reduce), L.ptr(model._terms), L.stream_ptr()), 'glamr_opt_losses')
        terms = model._terms.cpu().numpy()
        for k, v in uw.items():
            got, ref = float(terms[L.TERM_INDEX[k]]), float(v)
            assert abs(got - ref) <= 3e-4 * max(abs(ref), 1e-3) + 1e-7, f'{stage} term {k}: {got} vs {ref}'
        grad = model._reduce[:model._layout.n_params].cpu()
        lay = model._layout
        gv = lay.views(grad)
        order = []
        if 'cam' not in specs['opt_variables']:
            order += [gv['cam_inv_rot_residual'], gv['cam_inv_trans_residual']]
        elif model.flag_fixed_cam:
            order += [gv['cam_rot_6d_fix'], gv['cam_trans_fix']]
        else:
            order += [gv['cam_rot_6d'], gv['cam_trans']]
        for p in range(len(data['person_data'])):
            pv = lay.views(grad, p)
            for key in specs['opt_variables']:
                if key == 'world_res':
                    order += [pv['smpl_orient_world_res'], pv['root_trans_world_res']]
                if 'local' in key:
                    order.append(pv[f'traj_{key}'])
            if 'world_dheading' in specs['opt_variables']:
                order.append(pv['world_dheading'])
        assert len(order) == len(params)
        for i, (g_, p_) in enumerate(zip(order, params)):
            if p_.grad is None:
                continue
            scale = max(float(p_.grad.abs().max()), 1e-9)
            err = float((g_.reshape(p_.grad.shape) - p_.grad).abs().max()) / scale
            assert err < 5e-4, f'{stage} param {i}: rel err {err:.2e}'
        for p_ in params:
            p_.requires_grad_(False)
        # advance by the stage on the GPU and hand the resulting variables to the oracle: the next stage's closure is then
        # evaluated on IDENTICAL variables in both (two independent Adam runs drift apart on the ill-conditioned cases)
        model.optimize_main(data, specs['opt_variables'], specs['opt_lr'], specs['opt_niters'], specs['loss_cfg'], {'stage': stage})
        for pd, po in zip(data['person_data'].values(), data_o['person_data'].values()):
            for k in ['traj_local_xy', 'traj_local_dxy', 'traj_local_heading', 'traj_local_dheading', 'traj_local_z', 'traj_local_rot',
                      'smpl_orient_world_res', 'root_trans_world_res', 'world_dheading']:
                if k in pd:
                    po[k] = pd[k].detach().cpu().clone()
        for k in ['cam_pose', 'cam_pose_inv', 'cam_inv_rot_residual', 'cam_inv_trans_residual']:
            data_o[k] = data[k].detach().cpu().clone()


def test_optimize_output_layout_and_oracle_parity(smpl_assets):
    """optimize() end to end: output keys/dtypes of the reference (SURVEY Appendix B.2) and joints/vertices/camera
    within 1e-4 of the oracle recomputed from the returned SMPL parameters (north-star parity statement)."""
    from glamr_b200.smpl import SMPL
    from oracle.global_opt import OracleGlobalRecon
    from oracle.smpl import OracleSMPL
    gold, cfg, in_dict, model = _make('dynamic_p1_t40', smpl_assets)
    out = model.optimize(copy.deepcopy(in_dict))
    ora = OracleGlobalRecon(copy.deepcopy(cfg), smpl_assets, mt_model=ReplayMT(gold))
    ref = ora.optimize(copy.deepcopy(in_dict))
    pd, pr = out['person_data'][0], ref['person_data'][0]
    for k in ['smpl_pose', 'smpl_beta', 'smpl_orient_world', 'root_trans_world', 'scale', 'cam_K', 'exist_frames', 'vis_frames',
              'invis_frames', 'visible_orig', 'frames', 'frame2ind', 'max_len', 'kp_2d_pred', 'traj_local_rot', 'world_dheading']:
        assert k in pd, k
    for k in ['cam_pose', 'cam_pose_inv', 'seq_len', 'meta', 'gt', 'gt_meta', 'cam_rot_6d', 'cam_trans', 'rel_transform_cam']:
        assert k in out, k
    assert pd['kp_2d'].dtype == np.float64 and pd['kp_2d_pred'].dtype == np.float32 and pd['vis_frames'].dtype == np.bool_
    assert out['cam_pose'].shape == (40, 4, 4) and pd['smpl_orient_world'].shape == (40, 3)
    np.testing.assert_allclose(out['cam_pose'], ref['cam_pose'], atol=1e-4)
    np.testing.assert_allclose(out['cam_pose_inv'], ref['cam_pose_inv'], atol=1e-4)
    # joints / vertices from the returned SMPL parameters, CUDA vs oracle SMPL on the ORACLE's parameters
    smpl = SMPL(smpl_assets, device=DEV)
    o = smpl(global_orient=_cuda(pd['smpl_orient_world']), body_pose=_cuda(pd['smpl_pose']), betas=_cuda(pd['smpl_beta']),
             root_trans=_cuda(pd['root_trans_world']), orig_joints=True)
    jr, vr = OracleSMPL(smpl_assets)(torch.tensor(pr['smpl_orient_world']), torch.tensor(pr['smpl_pose']), torch.tensor(pr['smpl_beta']),
                                     root_trans=torch.tensor(pr['root_trans_world']), orig_joints=True)
    assert (o.joints.cpu() - jr).abs().max() < 2e-3      # after 6 Adam steps; per-step parity is covered above
    assert (o.vertices.cpu() - vr).abs().max() < 2e-3


def test_cuda_graph_and_eager_iterations_agree(smpl_assets):
    outs = []
    for graph in (True, False):
        gold, cfg, in_dict, model = _make('static_multi_p3_t30', smpl_assets, use_cuda_graph=graph)
        outs.append(model.optimize(copy.deepcopy(in_dict)))
    for pid in outs[0]['person_data']:
        np.testing.assert_array_equal(outs[0]['person_data'][pid]['smpl_orient_world'], outs[1]['person_data'][pid]['smpl_orient_world'])
    np.testing.assert_array_equal(outs[0]['cam_pose'], outs[1]['cam_pose'])


def test_product_fails_loudly_on_cpu_device(smpl_assets):
    from glamr_b200.lib import GlamrError
    from glamr_b200.recon import GlobalReconOptimizer
    gold, cfg, in_dict = case_setup('static_p1_t24', smpl_assets)
    with pytest.raises(GlamrError):
        GlobalReconOptimizer(cfg, torch.device('cpu'), None, smpl=smpl_assets, mt_model=ReplayMT(gold))


# ------------------------------------------------------------------------------------------------ learned prior
@pytest.mark.parametrize('M,N,K,relu', [(1, 512, 256, 1), (2, 256, 512, 0), (50, 256, 69, 0), (50, 768, 256, 0), (30, 69, 256, 0), (64, 11, 256, 0),
                                        (7, 5, 3, 1), (200, 512, 384, 1), (256, 256, 512, 0), (257, 256, 256, 0), (1500, 512, 384, 1),
                                        (3200, 768, 256, 0)])
def test_linear_layer_kernels_match_float64(M, N, K, relu):
    """Y = act(X W^T + b) of the prior networks: the skinny FP32 kernel (M <= 256), the wgmma 3xTF32 tile kernel and the
    FP32 tile kernel (mode 0) against a float64 product; ragged M / N / K, unaligned K (69) included"""
    import ctypes
    from glamr_b200 import lib as L
    lib = L.load()
    lib.glamr_linear_forward.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    g = torch.Generator().manual_seed(M * 1000 + N)
    X, W, b = torch.randn(M, K, generator=g).to(DEV), (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV), torch.randn(N, generator=g).to(DEV)
    ref = X.double() @ W.double().T + b.double()
    if relu:
        ref = ref.clamp_min(0)
    for mode in (1, 0):
        Y = torch.full((M, N), float('nan'), device=DEV)
        L.check(lib.glamr_linear_forward(M, N, K, X.data_ptr(), W.data_ptr(), b.data_ptr(), relu, Y.data_ptr(), mode, torch.cuda.current_stream().cuda_stream), 'linear')
        err = float((Y.double() - ref).abs().max())
        assert err < 2e-5, f'mode {mode}: {err}'       # |x w| ~ 1 per output: 3xTF32 keeps ~2e-6, FP32 FMA ~1e-6


@pytest.fixture(scope='module')
def cuda_prior(smpl_assets):
    from glamr_b200.motion_traj import MotionTrajJointModel
    from glamr_b200.smpl import SMPL
    from glamr_b200.synthetic_nets import make_prior_states
    return MotionTrajJointModel(None, torch.device(DEV), None, smpl=SMPL(smpl_assets, device=DEV), states=make_prior_states(1234))


@pytest.mark.parametrize('tag', ['b3_t75', 'b1_t300', 'b2_t40'])
def test_prior_inference_matches_reference_golden(tag, cuda_prior):
    """infiller (transformer, 50-frame autoregressive windows, key-padding masks, ragged last window) + trajectory
    predictor (MLP + bi-LSTM) vs the executed reference networks with identical weights and injected latents"""
    g = load_golden('nets')
    batch = {k: _cuda(g[f'{tag}/in/{k}']) for k in ['in_body_pose', 'frame_mask', 'in_motion_latent', 'in_traj_latent']}
    out = cuda_prior.inference(batch, sample_num=1)
    from oracle import rotations as rt
    T = batch['in_body_pose'].shape[1]
    acc_tol = 5e-4 + 2e-5 * T        # orientation / translation are prefix sums over T frames of the per-frame outputs
    for k, tol in [('infer_out_body_pose', 1e-4), ('infer_out_local_traj_tp', 1e-4), ('infer_out_trans', acc_tol)]:
        got = out[k].cpu().numpy()
        assert got.shape == g[f'{tag}/{k}'].shape, (k, got.shape, g[f'{tag}/{k}'].shape)
        np.testing.assert_allclose(got, g[f'{tag}/{k}'], atol=tol, err_msg=f'{tag} {k}')
    # orientations as rotation matrices (axis-angle coordinates are ill-conditioned near pi)
    for k in ['infer_out_orient', 'infer_out_pose']:
        got, ref = out[k].cpu(), torch.tensor(g[f'{tag}/{k}'])
        assert got.shape == ref.shape
        np.testing.assert_allclose(rt.aa_to_rotmat(got[..., :3]).numpy(), rt.aa_to_rotmat(ref[..., :3]).numpy(), atol=acc_tol, err_msg=f'{tag} {k}')
        np.testing.assert_allclose(got[..., 3:].numpy(), ref[..., 3:].numpy(), atol=1e-4, err_msg=f'{tag} {k} body')


def test_prior_c3_shape_matches_reference_golden(cuda_prior):
    """BASELINE.json configs[2] (64 sequences x 120 frames, frames 40-69 masked) vs the executed reference networks: four whole
    sequences element-wise, all 64 through per-sequence sums"""
    from helpers import C3_ROWS, c3_prior_inputs
    g = load_golden('nets')
    out = cuda_prior.inference({k: v.to(DEV) for k, v in c3_prior_inputs().items()}, sample_num=1)
    sel = torch.tensor(C3_ROWS, device=DEV)
    for k, bdim, tol in [('infer_out_body_pose', 0, 1e-4), ('infer_out_local_traj_tp', 1, 1e-4), ('infer_out_trans', 0, 5e-4 + 2e-5 * 120)]:
        v = out[k]
        np.testing.assert_allclose(v.index_select(bdim, sel).cpu().numpy(), g[f'c3_b64_t120/{k}'], atol=tol, err_msg=k)
        red = [d for d in range(v.dim()) if d != bdim]
        n_el = v.numel() // v.shape[bdim]
        np.testing.assert_allclose(v.double().sum(dim=red).cpu().numpy(), g[f'c3_b64_t120/{k}/sum'], atol=tol * n_el ** 0.5 * 4, err_msg=k + ' sum')
        np.testing.assert_allclose(v.double().abs().sum(dim=red).cpu().numpy(), g[f'c3_b64_t120/{k}/abs_sum'], rtol=1e-4, err_msg=k + ' abs sum')


def test_prior_batch_consistency(cuda_prior):
    """a sequence gives the same result alone and inside a batch of 64 (BASELINE config 3 shape: 64 x 120)"""
    gen = torch.Generator().manual_seed(3)
    pose = (torch.randn(64, 120, 69, generator=gen) * 0.3).to(DEV)
    mask = torch.ones(64, 120, device=DEV)
    mask[:, 40:70] = 0
    lat = {'in_motion_latent': torch.randn(4, 128, generator=gen).to(DEV), 'in_traj_latent': torch.randn(1, 128, generator=gen).to(DEV)}
    full = cuda_prior.inference({'in_body_pose': pose * mask[..., None], 'frame_mask': mask, **lat})
    one = cuda_prior.inference({'in_body_pose': (pose * mask[..., None])[5:6], 'frame_mask': mask[5:6], **lat})
    assert (full['infer_out_body_pose'][5] - one['infer_out_body_pose'][0]).abs().max() < 1e-5
    assert (full['infer_out_local_traj_tp'][:, 5] - one['infer_out_local_traj_tp'][:, 0]).abs().max() < 1e-5
    assert full['infer_out_body_pose'].shape == (64, 1, 120, 69) and full['infer_out_local_traj_tp'].shape == (120, 64, 1, 11)


def test_full_pipeline_with_cuda_prior_matches_oracle(smpl_assets, cuda_prior):
    """init_data (infill -> trajectory) + optimisation, CUDA end to end vs the oracle end to end, same weights/latents"""
    from glamr_b200.config import Config
    from glamr_b200.recon import GlobalReconOptimizer
    from glamr_b200.synthetic import make_in_dict
    from glamr_b200.synthetic_nets import make_prior_states
    from helpers import LatentInjector
    from oracle.global_opt import OracleGlobalRecon
    from oracle.nets import MotionTrajJoint
    from oracle.smpl import OracleSMPL
    cfg = Config('glamr_dynamic')
    for st in cfg.opt_stage_specs.values():
        st['opt_niters'] = 5
    in_dict = make_in_dict(smpl_assets, 1, 70, seed=3, gaps=True)
    model = GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=cuda_prior.smpl, mt_model=LatentInjector(cuda_prior, 9))
    out = model.optimize(copy.deepcopy(in_dict))
    st_m, st_t = make_prior_states(1234)
    ora = OracleGlobalRecon(copy.deepcopy(cfg), smpl_assets, mt_model=LatentInjector(MotionTrajJoint(st_m, st_t, OracleSMPL(smpl_assets)), 9))
    ref = ora.optimize(copy.deepcopy(in_dict))
    pd, pr = out['person_data'][0], ref['person_data'][0]
    np.testing.assert_allclose(pd['smpl_pose'], pr['smpl_pose'], atol=2e-4, err_msg='infilled body pose')
    np.testing.assert_allclose(pd['traj_local_pred'], pr['traj_local_pred'], atol=2e-4)
    vis = pr['vis_frames']
    np.testing.assert_allclose(pd['smpl_orient_world'][vis], pr['smpl_orient_world'][vis], atol=3e-3)
    np.testing.assert_allclose(pd['root_trans_world'][vis], pr['root_trans_world'][vis], atol=3e-3)
    np.testing.assert_allclose(out['cam_pose'], ref['cam_pose'], atol=3e-3)
