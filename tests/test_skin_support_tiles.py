"""The support vertices as vertex tiles of their own in the tensor-core LBS.

The optimiser reads only the S "support" vertices (the picked vertices and those of the extra joint regressor).  The library skins
them as extra 128-vertex tiles after the 54 mesh tiles, from copies of their blend-basis columns and skinning weights, so that the
optimiser's critical path skins one vertex tile instead of the whole mesh.  These tests pin that design down:

  * the blend GEMM's support columns of v_posed equal the mesh columns they copy, bit for bit (a wgmma output element does not
    depend on its column position);
  * the support tiles' skinned vertices (vcompact) equal the same vertices of the mesh that glamr_smpl_forward returns, bit for bit;
  * a model with more than 128 support vertices (two support tiles) runs through the optimiser and matches float64 within the bound
    of test_lbs_float64, as the tensor-core blend with the SIMT skinning (which skins the support vertices inside the mesh) does;
  * an optimiser iteration is 9 launches.

The workspace offsets below restate smpl_carve_workspace (glamr_b200/csrc/smpl_model.cuh).
"""
import copy
import ctypes
import functools

import numpy as np
import pytest
import torch

from helpers import ReplayMT, case_setup
from test_gpu_parity import LBS_PATHS, _default_lbs_path
from test_lbs_float64 import ATOL_OPT, REL, _check_optimiser_joints, _dev, _nan, make_inputs, oracle64

DEV = 'cuda:0'
NV, NJ = 6890, 24
V_TILE, V_TILES, TC_N, TC_COLS, SK_F = 128, 54, 256, 20736, 20


def support_vertices(a):
    """the support list of glamr_smpl_create: picked vertices, then the non-zeros of each extra regressor row, first occurrence wins"""
    from glamr_b200.synthetic import EXTRA_VERTEX_IDS
    sup, seen = [], set()
    for v in list(EXTRA_VERTEX_IDS) + [int(v) for r in a['J_regressor_extra'] for v in np.flatnonzero(r)]:
        if int(v) not in seen:
            seen.add(int(v))
            sup.append(int(v))
    return np.array(sup, np.int64)


@functools.lru_cache(maxsize=None)
def wide_support_assets():
    """the suite constants with a denser extra regressor: 21 picks + 9 rows x 20 vertices, more than 128 support vertices"""
    from glamr_b200.synthetic import make_smpl_assets
    a = dict(make_smpl_assets(0))
    rng = np.random.default_rng(7)
    r = np.zeros_like(a['J_regressor_extra'])
    for i in range(r.shape[0]):
        vs = rng.choice(NV, 20, replace=False)
        r[i, vs] = rng.dirichlet(np.ones(20)).astype(np.float32)
    a['J_regressor_extra'] = r
    return a


@pytest.fixture(scope='module')
def assets(smpl_assets):
    return {'suite': smpl_assets, 'wide': wide_support_assets()}


@pytest.fixture
def tensor_core_path():
    from glamr_b200 import lib as L
    L.check(L.load().glamr_smpl_set_lbs_path(LBS_PATHS['tensor_core']), 'set_lbs_path')
    yield
    L.check(L.load().glamr_smpl_set_lbs_path(_default_lbs_path()), 'set_lbs_path')


@pytest.fixture(scope='module')
def models(assets):
    from glamr_b200.smpl import SMPL
    return {k: SMPL(a, device=DEV) for k, a in assets.items()}


def workspace_views(ws, n, S):
    """vcompact [n, S, 3] and the frame-tiled v_posed [ceil(mpad / 20), vp_cols, 20] inside a glamr_smpl_forward workspace"""
    n32 = (n + 31) // 32 * 32
    o = n32 * NJ * 12 + n32 * 208 + n * NJ * 3
    vcompact = ws[o:o + n * S * 3].view(n, S, 3)
    o += n * S * 3 + n * 3
    o = (o + 63) // 64 * 64                                        # 256-byte alignment (the workspace itself is)
    mpad = (n + 127) // 128 * 128
    o += (mpad // 128) * 14 * 4096 // 2 + mpad
    nft = (mpad + SK_F - 1) // SK_F
    o += nft * 11520
    sup_tiles = (S + V_TILE - 1) // V_TILE
    vp_cols = (TC_COLS + sup_tiles * 3 * V_TILE + TC_N - 1) // TC_N * TC_N
    v_posed = ws[o:o + nft * vp_cols * SK_F].view(nft, vp_cols, SK_F)
    return vcompact, v_posed


def forward_keep_workspace(smpl, inp_dev, n):
    """glamr_smpl_forward with the mesh, no re-rooting, on a NaN-filled workspace -> (vertices [n, 6890, 3], workspace)"""
    from glamr_b200 import lib as L
    lib = L.load()
    ws = _nan((int(lib.glamr_smpl_workspace_bytes(smpl.handle, n)) + 3) // 4)
    joints, verts = _nan(n, smpl.num_joints, 3), _nan(n, NV, 3)
    L.check(lib.glamr_smpl_forward(smpl.handle, n, L.ptr(inp_dev['orient']), L.ptr(inp_dev['pose']), L.ptr(inp_dev['betas']), None, None, 0,
                                   L.ptr(joints), L.ptr(verts), L.ptr(ws), ctypes.c_size_t(ws.numel() * 4), L.stream_ptr()),
            'glamr_smpl_forward')
    torch.cuda.synchronize()
    return verts, ws


SIZES = [1, 19, 20, 21, 127, 128, 129, 300, 1000]


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['suite', 'wide'])
@pytest.mark.parametrize('n', SIZES)
def test_support_columns_and_vertices_match_the_mesh_bitwise(n, name, assets, models, tensor_core_path):
    """v_posed's support columns (20736 + 3 s + c) equal mesh column 3 sup[s] + c, and vcompact equals the mesh's support rows, bit
    for bit, on every frame"""
    from glamr_b200 import lib as L
    smpl, a = models[name], assets[name]
    sup = support_vertices(a)
    S = int(L.load().glamr_smpl_info(smpl.handle, 1))
    assert S == len(sup)
    if name == 'wide':
        assert S > V_TILE, S
    verts, ws = forward_keep_workspace(smpl, _dev(make_inputs(n, 5000 + n)), n)
    vcompact, v_posed = workspace_views(ws, n, S)
    vp = v_posed.permute(0, 2, 1).reshape(-1, v_posed.shape[1])[:n]        # [frame, column]
    mesh_cols = torch.as_tensor((sup[:, None] * 3 + np.arange(3)[None]).reshape(-1), device=DEV)
    copies = vp[:, TC_COLS:TC_COLS + 3 * S]
    assert not torch.isnan(copies).any()
    assert torch.equal(copies, vp[:, mesh_cols]), f'n={n}: a support column of v_posed differs from its mesh column'
    assert not torch.isnan(vcompact).any()
    assert torch.equal(vcompact, verts[:, torch.as_tensor(sup, device=DEV)]), f'n={n}: a support vertex differs from its mesh vertex'


def _optimiser(case, a, path):
    from glamr_b200 import lib as L
    from glamr_b200.recon import GlobalReconOptimizer
    L.check(L.load().glamr_smpl_set_lbs_path(LBS_PATHS[path]), 'set_lbs_path')
    gold, cfg, in_dict = case_setup(case, a)
    model = GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=a, mt_model=ReplayMT(gold, DEV))
    data = model.init_data(copy.deepcopy(in_dict))
    stage, specs = next(iter(cfg.opt_stage_specs.items()))
    model._cur_vars, model._cur_stage = specs['opt_variables'], stage
    model._set_stage(data, specs['opt_variables'], specs['loss_cfg'], stage, reset_adam=True, begin=True)
    return model, data, stage, specs


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['dynamic_p1_t300', 'static_multi_p4_t300'])
def test_two_support_tiles_through_the_optimiser(case, assets):
    """More than 128 support vertices: the optimiser's joints after the first closure and after 5 Adam iterations match float64 within
    ATOL_OPT, as those of the tensor-core blend with the SIMT skinning (the support vertices skinned inside the mesh) do, and after the
    first closure (same variables) the two agree with each other within twice that bound"""
    from glamr_b200 import lib as L
    a = assets['wide']
    ora = oracle64(a)
    joints = {}
    try:
        for path in ('tensor_core', 'tensor_core_blend_simt_skin'):
            model, data, stage, specs = _optimiser(case, a, path)
            model._backward()
            _check_optimiser_joints(model, ora, ATOL_OPT['suite'], f'{case} wide {path} first closure')
            comp = model._comp
            joints[path] = model._read(L.R_JOINTS_WORLD, comp.P, comp.T, comp.J, 3)
            model.optimize_main(data, specs['opt_variables'], specs['opt_lr'], 5, specs['loss_cfg'], {'stage': stage})
            _check_optimiser_joints(model, ora, ATOL_OPT['suite'], f'{case} wide {path} after 5 iterations')
    finally:
        L.check(L.load().glamr_smpl_set_lbs_path(_default_lbs_path()), 'set_lbs_path')
    got, other = joints['tensor_core'].double(), joints['tensor_core_blend_simt_skin'].double()
    excess = (got - other).abs() - 2 * REL * other.abs()
    assert float(excess.max()) <= 2 * ATOL_OPT['suite'], float(excess.max())


@pytest.mark.gpu
def test_iteration_is_nine_launches(assets, tensor_core_path):
    """traj/cam forward, pose prep, support skinning, mesh skinning, blend features, blend GEMM, residuals, traj/cam backward, apply"""
    model, _, _, _ = _optimiser('dynamic_p1_t300', assets['suite'], 'tensor_core')
    assert model.launches_per_iteration() == 9
