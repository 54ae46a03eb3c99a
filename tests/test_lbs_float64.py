"""The LBS kernels against a float64 body model: every frame, vertex and joint, at the tile edges of the tensor-core kernels, and
with model constants large enough that a blend or skinning computed with less than FP32 accuracy (3xTF32) shows.

The reference is oracle.smpl.OracleSMPL in float64 on the GPU (pure torch, never the library), fed the same float32 inputs.
Every output is compared as |got - ref64| <= a + 8 * 2^-24 * |ref64|: `a` absorbs the float32 arithmetic of the kinematic chain,
the relative term the float32 rounding of outputs that sit 20 m from the origin.  `a` was set from measurements on an H100 80GB
HBM3 (400 W power limit): at least 5x the largest measured excess |got - ref64| - 8 * 2^-24 * |ref64| of its tests, and on the
stress constants at most 1/10 of what a kernel that drops one low tf32 half costs.  The forward tests feed edge poses (3 pi
about an axis, root scales up to 2), whose float32 Rodrigues and chain cost up to 3.4e-6; the optimiser's inputs are the bench
poses, which cost 5e-7, so its bound is tighter.

Two sets of model constants:
  suite   make_smpl_assets(0) as the rest of the suite uses it (posedirs sigma 0.001, shapedirs sigma 0.01)
  stress  the same weights and regressors with posedirs sigma 0.02, shapedirs sigma 0.03 and v_template sigma 0.25 + (0, 0.3, 0).
          This is a deliberate stress choice, not a copy of SMPL: with these magnitudes a blend or skinning that loses the
          low-order tf32 half of an operand misses by far more than `a` (test_tolerances_discriminate_weakened_tf32_splits).
On the suite constants the same loss of precision stays within a few 1e-6, below what the float32 chain itself costs, so the
suite-asset tests check that every output is written and the indexing is right, and the stress-asset tests check precision.

Outputs and workspace are filled with NaN before each call and one canary frame past n is allocated, so an output that a kernel
skips, or one that it writes past n, fails the test instead of reading whatever the caching allocator handed out.
"""
import copy
import ctypes
import functools
import math

import numpy as np
import pytest
import torch

from helpers import ReplayMT, case_setup
from test_gpu_parity import LBS_PATHS, _default_lbs_path

DEV = 'cuda:0'
REL = 8 * 2.0 ** -24
# absolute part of the bound per set of constants: glamr_smpl_forward / glamr_smpl_fk24 on the edge-pose inputs, and the optimiser's
# evaluation; the measured maxima are in the docstrings of the tests
ATOL = {'suite': 1.2e-5, 'stress': 1.8e-5}
ATOL_OPT = {'suite': 3e-6, 'stress': 3e-6}
NV = 6890
CHUNK = 64                  # frames per float64 oracle call: its [B, 6890, 16] transforms stay small
SK_F, V_TILES = 20, 54      # frames per tensor-core skinning item, 128-vertex tiles (glamr_b200/csrc/common.cuh)


# ------------------------------------------------------------------------------------------------ assets and inputs
@functools.lru_cache(maxsize=None)
def stress_assets():
    from glamr_b200.synthetic import make_smpl_assets
    a = dict(make_smpl_assets(0))
    rng = np.random.default_rng(1)
    a['v_template'] = (a['v_template'] / 0.3 * 0.25 + np.array([0.0, 0.3, 0.0], np.float32)).astype(np.float32)
    a['shapedirs'] = rng.normal(0.0, 0.03, a['shapedirs'].shape).astype(np.float32)
    a['posedirs'] = rng.normal(0.0, 0.02, a['posedirs'].shape).astype(np.float32)
    return a


def dense_weights(a):
    """the same model with dense skinning weights (24 per vertex): the generic-K kernels"""
    a = dict(a)
    w = np.random.default_rng(5).random((NV, 24)).astype(np.float32)
    a['lbs_weights'] = w / w.sum(1, keepdims=True)
    return a


@pytest.fixture(scope='module')
def assets(smpl_assets):
    return {'suite': smpl_assets, 'stress': stress_assets(), 'stress_dense': dense_weights(stress_assets())}


# axis-angle magnitudes where Rodrigues goes wrong: exact zero (the 1e-8 guard), tiny, pi, just below pi, and past 2 pi
EDGE_ANGLES = (0.0, 1e-7, math.pi, math.pi - 1e-4, 3 * math.pi)


def make_inputs(n, seed):
    """float32 CPU inputs of n frame-persons.  Half of the 24 joints of every frame (root included) take an edge angle of
    EDGE_ANGLES about a random axis; betas up to +-5, root translations up to +-20 m, root scales 0.5..2."""
    g = torch.Generator().manual_seed(seed)
    aa = torch.randn(n, 24, 3, generator=g) * 0.6
    aa[:, 0] = torch.randn(n, 3, generator=g)
    axis = torch.nn.functional.normalize(torch.randn(n, 24, 3, generator=g, dtype=torch.float64), dim=-1)
    pick = (torch.arange(n)[:, None] + torch.arange(24)[None]) % 10
    for k, ang in enumerate(EDGE_ANGLES):
        m = pick == k
        aa[m] = (axis[m] * ang).float()
    aa[pick == 0] = 0.0
    return {'orient': aa[:, 0].contiguous(), 'pose': aa[:, 1:].reshape(n, 69).contiguous(),
            'betas': (torch.rand(n, 10, generator=g) * 2 - 1) * 5, 'trans': (torch.rand(n, 3, generator=g) * 2 - 1) * 20,
            'scale': 0.5 + 1.5 * torch.rand(n, generator=g)}


# ------------------------------------------------------------------------------------------------ float64 reference
def oracle64(a):
    from oracle.smpl import OracleSMPL
    return OracleSMPL(a, device=DEV, dtype=torch.float64)


def ref_forward(ora, inp, orig_joints, root):
    """float64 joints, vertices of OracleSMPL.__call__ in chunks of CHUNK frames.  root: 'trans_scale', 'trans' or None"""
    n = inp['pose'].shape[0]
    d = {k: v.to(DEV, torch.float64) for k, v in inp.items()}
    js, vs = [], []
    for s in range(0, n, CHUNK):
        sl = slice(s, min(n, s + CHUNK))
        j, v = ora(d['orient'][sl], d['pose'][sl], d['betas'][sl], root_trans=d['trans'][sl] if root else None,
                   root_scale=d['scale'][sl] if root == 'trans_scale' else None, orig_joints=orig_joints)
        js.append(j)
        vs.append(v)
    return torch.cat(js), torch.cat(vs)


def ref_fk24(ora, inp, root):
    n = inp['pose'].shape[0]
    d = {k: v.to(DEV, torch.float64) for k, v in inp.items()}
    out = []
    for s in range(0, n, CHUNK):
        sl = slice(s, min(n, s + CHUNK))
        out.append(ora.get_joints(d['orient'][sl], d['pose'][sl], root_trans=d['trans'][sl] if root else None,
                                  root_scale=d['scale'][sl] if root == 'trans_scale' else None))
    return torch.cat(out)


def check_close(what, got, ref, atol):
    """|got - ref| <= atol + REL |ref| everywhere; returns the largest excess |got - ref| - REL |ref|, the number atol bounds"""
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert not torch.isnan(got).any(), f'{what}: NaN in the output (an output was not written)'
    diff = (got.double() - ref).abs()
    excess = diff - REL * ref.abs()
    worst = int(excess.argmax())
    err = float(diff.max())
    assert float(excess.max()) <= atol, (f'{what}: |got - ref64| {float(diff.flatten()[worst]):.3e} at flat index {worst} '
                                         f'(|ref| {float(ref.abs().flatten()[worst]):.3e}) exceeds {atol:.1e} + {REL:.1e} |ref|; max {err:.3e}')
    return float(excess.max())


# ------------------------------------------------------------------------------------------------ the C ABI, poisoned
def _nan(*shape):
    return torch.full(shape, float('nan'), dtype=torch.float32, device=DEV)


def call_forward(smpl, inp_dev, n, orig_joints, root, with_vertices=True):
    """glamr_smpl_forward on NaN-filled workspace / outputs with one canary frame past n; -> joints [n], vertices [n] or None"""
    from glamr_b200 import lib as L
    lib = L.load()
    nj = 24 if orig_joints else smpl.num_joints
    ws_bytes = int(lib.glamr_smpl_workspace_bytes(smpl.handle, n))
    ws = _nan((ws_bytes + 3) // 4)
    joints = _nan(n + 1, nj, 3)
    verts = _nan(n + 1, NV, 3) if with_vertices else None
    rt = inp_dev['trans'] if root else None
    rs = inp_dev['scale'] if root == 'trans_scale' else None
    L.check(lib.glamr_smpl_forward(smpl.handle, n, L.ptr(inp_dev['orient']), L.ptr(inp_dev['pose']), L.ptr(inp_dev['betas']), L.ptr(rt),
                                   L.ptr(rs), int(orig_joints), L.ptr(joints), L.ptr(verts), L.ptr(ws), ctypes.c_size_t(ws.numel() * 4),
                                   L.stream_ptr()), 'glamr_smpl_forward')
    torch.cuda.synchronize()
    assert torch.isnan(joints[n]).all(), 'joints written past frame n'
    if verts is not None:
        assert torch.isnan(verts[n]).all(), 'vertices written past frame n'
        return joints[:n], verts[:n]
    return joints[:n], None


def _dev(inp):
    return {k: v.to(DEV).contiguous() for k, v in inp.items()}


@pytest.fixture
def lbs_path(request):
    """tensor-core blend + tensor-core skinning, tensor-core blend + SIMT skinning, the FP32 SIMT kernel"""
    from glamr_b200 import lib as L
    L.check(L.load().glamr_smpl_set_lbs_path(LBS_PATHS[request.param]), 'set_lbs_path')
    yield request.param
    L.check(L.load().glamr_smpl_set_lbs_path(_default_lbs_path()), 'set_lbs_path')


# the outermost decorator of a test: the path varies fastest, so consecutive tests share one float64 reference
each_lbs_path = pytest.mark.parametrize('lbs_path', list(LBS_PATHS), indirect=True)


@pytest.fixture(scope='module')
def models(assets):
    from glamr_b200.smpl import SMPL
    out = {k: SMPL(a, device=DEV) for k, a in assets.items()}
    yield out
    _REF_CACHE.clear()


_REF_CACHE = {}


def cached_ref(case, mode, fn):
    """the float64 reference of one case (constants, n, inputs) is shared by the three LBS paths, which run one after the other
    (the lbs_path parameter varies fastest); only the latest case is kept"""
    if any(c != case for c, _ in _REF_CACHE):
        _REF_CACHE.clear()
    if (case, mode) not in _REF_CACHE:
        _REF_CACHE[(case, mode)] = fn()
    return _REF_CACHE[(case, mode)]


# (orig_joints, root) combinations every size runs
MODES = [(0, 'trans_scale'), (1, 'trans'), (0, None), (1, None)]


def resolve_n(n):
    """sizes named after the skinning grid: the largest n whose 54 * ceil(n / 20) items fit one per SM, and the next one"""
    if isinstance(n, int):
        return n
    from glamr_b200 import lib as L
    sms = L.load().glamr_device_sm_count()
    assert sms > 0
    last = SK_F * (sms // V_TILES)
    assert last > 0
    return {'skin_one_item_per_cta': last, 'skin_two_items_per_cta': last + 1}[n]


# 20-frame skinning tiles (19/20/21, ragged last tile at 63/127/129/193/1200+...), the 64-row half blend tile (63/64/65, 192/193),
# one vs several items per CTA (skinning at 40/41 on 132 SMs, blend at 128/129), several frame tiles (300, 1200) and C4 (8 x 500)
SIZES = [1, 19, 20, 21, 'skin_one_item_per_cta', 'skin_two_items_per_cta', 63, 64, 65, 127, 128, 129, 192, 193, 300, 1200, 4000]


def _check_forward(models, assets, name, n, seed, what):
    smpl = models[name]
    inp = make_inputs(n, seed)
    inp_dev = _dev(inp)
    atol = ATOL['suite' if name == 'suite' else 'stress']
    errs = {}
    for orig, root in MODES:
        jr, vr = cached_ref((name, n, seed), (orig, root), lambda: ref_forward(oracle64(assets[name]), inp, orig, root))
        j, v = call_forward(smpl, inp_dev, n, orig, root)
        tag = f'{what} {name} n={n} orig_joints={orig} root={root}'
        errs[(orig, root)] = (check_close(tag + ' joints', j, jr, atol), check_close(tag + ' vertices', v, vr, atol))
        if (orig, root) == MODES[0]:
            j2, _ = call_forward(smpl, inp_dev, n, orig, root, with_vertices=False)
            assert torch.equal(j2, j), f'{tag}: joints without vertices differ from joints with vertices'
    worst = max(max(e) for e in errs.values())
    print(f'LBS64 {what} {name} n={n}: max excess {worst:.3e}')
    return worst


@each_lbs_path
@pytest.mark.gpu
@pytest.mark.parametrize('name', ['stress', 'suite'])
@pytest.mark.parametrize('n', SIZES)
def test_smpl_forward_matches_float64_every_output(n, name, assets, models, lbs_path):
    """glamr_smpl_forward through the C ABI: all frames, vertices and joints vs OracleSMPL in float64, for the four combinations
    of orig_joints and root translation / scale given or NULL, and joints with vertices == NULL bit-identical to joints with
    vertices.  Largest excess over 8 * 2^-24 |ref64| measured (H100 80GB HBM3), all sizes and modes:
      stress  tensor_core 3.39e-6, tensor_core_blend_simt_skin 2.87e-6, simt 2.54e-6   (bound 1.8e-5)
      suite   tensor_core 1.56e-6, tensor_core_blend_simt_skin 1.51e-6, simt 2.29e-6   (bound 1.2e-5)"""
    n = resolve_n(n)
    _check_forward(models, assets, name, n, 1000 + n, lbs_path)


@each_lbs_path
@pytest.mark.gpu
@pytest.mark.parametrize('n', [21, 129, 300])
def test_smpl_dense_weights_match_float64(n, assets, models, lbs_path):
    """a model with 24 skinning weights per vertex (the generic-K SIMT kernels; dense W image on the tensor cores), stress constants.
    Largest excess measured: tensor_core 1.76e-6, tensor_core_blend_simt_skin 1.19e-6, simt 1.07e-6"""
    _check_forward(models, assets, 'stress_dense', n, 2000 + n, lbs_path)


@each_lbs_path
@pytest.mark.gpu
def test_smpl_forward_same_handle_changing_n(assets, models, lbs_path):
    """one handle called with n = 300, 21, 300, freshly poisoned buffers each time: nothing of a larger call may stand in for an
    output of a smaller one (measured maxima are within those of test_smpl_forward_matches_float64_every_output)"""
    for n in (300, 21, 300):
        _check_forward(models, assets, 'stress', n, 3000 + n, lbs_path)


@each_lbs_path
@pytest.mark.gpu
def test_smpl_forward_n0_leaves_buffers_untouched(models, lbs_path):
    from glamr_b200 import lib as L
    lib = L.load()
    smpl = models['stress']
    inp = _dev(make_inputs(1, 7))
    g = torch.Generator(device=DEV).manual_seed(0)
    bufs = [torch.rand(1, smpl.num_joints, 3, device=DEV, generator=g), torch.rand(1, NV, 3, device=DEV, generator=g),
            torch.rand(max(int(lib.glamr_smpl_workspace_bytes(smpl.handle, 1)) // 4, 1), device=DEV, generator=g)]
    before = [b.clone() for b in bufs]
    L.check(lib.glamr_smpl_forward(smpl.handle, 0, L.ptr(inp['orient']), L.ptr(inp['pose']), L.ptr(inp['betas']), L.ptr(inp['trans']),
                                   L.ptr(inp['scale']), 0, L.ptr(bufs[0]), L.ptr(bufs[1]), L.ptr(bufs[2]),
                                   ctypes.c_size_t(bufs[2].numel() * 4), L.stream_ptr()), 'glamr_smpl_forward')
    torch.cuda.synchronize()
    for b, b0 in zip(bufs, before):
        assert torch.equal(b, b0)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['stress', 'suite'])
@pytest.mark.parametrize('n', [1, 21, 129, 300])
def test_smpl_fk24_matches_float64(n, name, assets, models):
    """glamr_smpl_fk24 (SMPL.get_joints: rest joints from v_template) vs OracleSMPL.get_joints in float64, root translation / scale
    given and NULL.  Largest excess measured: stress 1.10e-6, suite 7.2e-7"""
    from glamr_b200 import lib as L
    lib = L.load()
    smpl = models[name]
    inp = make_inputs(n, 4000 + n)
    inp_dev = _dev(inp)
    ora = oracle64(assets[name])
    for root in ('trans_scale', None):
        ws_bytes = int(lib.glamr_smpl_fk_workspace_bytes(smpl.handle, n))
        ws, joints = _nan((ws_bytes + 3) // 4), _nan(n + 1, 24, 3)
        L.check(lib.glamr_smpl_fk24(smpl.handle, n, L.ptr(inp_dev['orient']), L.ptr(inp_dev['pose']), L.ptr(inp_dev['trans'] if root else None),
                                    L.ptr(inp_dev['scale'] if root else None), L.ptr(joints), L.ptr(ws), ctypes.c_size_t(ws.numel() * 4),
                                    L.stream_ptr()), 'glamr_smpl_fk24')
        torch.cuda.synchronize()
        assert torch.isnan(joints[n]).all(), 'fk24 joints written past frame n'
        err = check_close(f'fk24 {name} n={n} root={root}', joints[:n], ref_fk24(ora, inp, root), ATOL['suite' if name == 'suite' else 'stress'])
        print(f'LBS64 fk24 {name} n={n} root={root}: max excess {err:.3e}')


# ------------------------------------------------------------------------------------------------ the optimiser's SMPL evaluation
def _check_optimiser_joints(model, ora, atol, tag):
    """R_JOINTS_WORLD of the last evaluation vs OracleSMPL on the world orientation / translation the same evaluation used"""
    from glamr_b200 import lib as L
    comp = model._comp
    P, T, J = comp.P, comp.T, comp.J
    torch.cuda.synchronize()
    jw = model._read(L.R_JOINTS_WORLD, P, T, J, 3).reshape(P * T, J, 3)
    ow = model._read(L.R_ORIENT_WORLD, P, T, 3).reshape(P * T, 3)
    tw = model._read(L.R_TRANS_WORLD, P, T, 3).reshape(P * T, 3)
    inp = {'orient': ow, 'pose': comp.pose_all.reshape(P * T, 69), 'betas': comp.beta_all.reshape(P * T, 10), 'trans': tw}
    root = 'trans'
    if comp.scale_all is not None:
        inp['scale'], root = comp.scale_all.reshape(P * T), 'trans_scale'
    jr, _ = ref_forward(ora, inp, 0, root)
    err = check_close(tag + ' joints_world', jw, jr, atol)
    print(f'LBS64 optimiser {tag}: max excess {err:.3e}')


@pytest.mark.gpu
@pytest.mark.parametrize('case,name', [('dynamic_p1_t300', 'suite'), ('static_multi_p4_t300', 'suite'), ('3dpw_p1_t600_gaps', 'suite'),
                                       ('dynamic_p1_t300', 'stress'), ('static_multi_p4_t300', 'stress')])
def test_optimiser_smpl_matches_float64(case, name, assets):
    """The optimiser's own LBS (features kernel, side-stream blend, tensor-core skinning of the support vertices only) on every
    frame-person: the joints it projects (GLAMR_R_JOINTS_WORLD) vs OracleSMPL in float64 on the body pose / betas it holds and the
    world orientation / translation it evaluated, after the first closure of the first stage and again after a few Adam
    iterations (the pipelined blend has then run several times).  The stress cases are the bench shapes built on the stress
    constants, with the learned prior replayed from the fixture of the same shape.
    Largest excess measured: stress 4.4e-7, suite 4.9e-7 (bound 3e-6 for both).  A features kernel that drops the low tf32 half of
    the pose features costs 3.8e-5 on the stress constants (and 2.2e-6 on the suite constants, which cannot show it)."""
    from glamr_b200.recon import GlobalReconOptimizer
    gold, cfg, in_dict = case_setup(case, assets[name])
    model = GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=assets[name], mt_model=ReplayMT(gold, DEV))
    data = model.init_data(copy.deepcopy(in_dict))
    ora = oracle64(assets[name])
    atol = ATOL_OPT[name]
    stage, specs = next(iter(cfg.opt_stage_specs.items()))
    model._cur_vars, model._cur_stage = specs['opt_variables'], stage
    model._set_stage(data, specs['opt_variables'], specs['loss_cfg'], stage, reset_adam=True, begin=True)
    model._backward()
    _check_optimiser_joints(model, ora, atol, f'{case} {name} first closure')
    model.optimize_main(data, specs['opt_variables'], specs['opt_lr'], 5, specs['loss_cfg'], {'stage': stage})
    _check_optimiser_joints(model, ora, atol, f'{case} {name} after 5 iterations')


# ------------------------------------------------------------------------------------------------ the bound discriminates (CPU)
def _tf32(x):
    """cvt.rna.tf32.f32 on float32 values: round to nearest, ties away from zero, 10-bit mantissa"""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _split(x):
    x = np.asarray(x, np.float32)
    hi = _tf32(x)
    return hi.astype(np.float64), _tf32(x - hi).astype(np.float64)


def emulate_lbs_errors(a, n=128, seed=11):
    """max |result - float64| of the blend GEMM (v_posed) and of the skinning GEMM (vertices) computed with the kernels' tf32
    hi / lo operand split, as shipped (3xTF32: hi hi + lo hi + hi lo) and with one low half dropped.  Products accumulate in
    float64, so only the operand split differs from the reference."""
    from oracle.smpl import rigid_chain, rodrigues_smplx
    inp = make_inputs(n, seed)
    pose = torch.cat([inp['orient'], inp['pose']], 1).double()
    R = rodrigues_smplx(pose.reshape(-1, 3)).view(n, 24, 3, 3)
    feat = torch.cat([(R[:, 1:] - torch.eye(3, dtype=torch.float64)).reshape(n, -1), inp['betas'].double(),
                      torch.ones(n, 1, dtype=torch.float64)], 1).float().numpy()                  # float32, as the kernels build them
    basis = np.concatenate([a['posedirs'], a['shapedirs'].reshape(NV * 3, 10).T, a['v_template'].reshape(1, -1)], 0).astype(np.float32)
    ref = feat.astype(np.float64) @ basis.astype(np.float64)
    fh, fl = _split(feat)
    bh, bl = _split(basis)
    pose_k, shape_k = slice(0, 207), slice(207, 217)

    def blend(drop_f=(), drop_b=()):
        fl2, bl2 = fl.copy(), bl.copy()
        for k in drop_f:
            fl2[:, k] = 0.0
        for k in drop_b:
            bl2[k] = 0.0
        return float(np.abs(fh @ bh + fl2 @ bh + fh @ bl2 - ref).max())

    out = {'blend 3xTF32': blend(), 'pose features lo dropped': blend(drop_f=[pose_k]),
           'pose blend 1xTF32': blend(drop_f=[pose_k], drop_b=[pose_k]), 'shape blend 1xTF32': blend(drop_f=[shape_k], drop_b=[shape_k])}
    # skinning: T[v] = sum_j W[v, j] A_j (3 x 4 per frame), vertex = T [v_posed; 1]
    J = torch.einsum('bik,ji->bjk', torch.tensor(a['v_template'], dtype=torch.float64)[None] +
                     torch.einsum('bl,mkl->bmk', inp['betas'].double(), torch.tensor(a['shapedirs'], dtype=torch.float64)),
                     torch.tensor(a['J_regressor'], dtype=torch.float64))
    _, A = rigid_chain(R, J, torch.tensor(a['parents']))
    A = A[..., :3, :].float().numpy()                                                  # [n, 24, 3, 4] float32, as pose prep stores it
    Am = A.transpose(1, 0, 2, 3).reshape(24, n * 12)
    W = np.asarray(a['lbs_weights'], np.float32)
    vp = ref.reshape(n, NV, 3).astype(np.float32).astype(np.float64)
    vh = np.concatenate([vp, np.ones((n, NV, 1))], -1)                                  # [n, V, 4]

    def skin(T):
        T = T.reshape(NV, n, 3, 4).transpose(1, 0, 2, 3)
        return np.einsum('nvrc,nvc->nvr', T, vh)
    vref = skin(W.astype(np.float64) @ Am.astype(np.float64))
    wh, wl = _split(W)
    ah, al = _split(Am)
    out['skinning 3xTF32'] = float(np.abs(skin(wh @ ah + wl @ ah + wh @ al) - vref).max())
    out['skinning W 1xTF32'] = float(np.abs(skin(wh @ ah + wh @ al) - vref).max())
    out['skinning A image 1xTF32'] = float(np.abs(skin(wh @ ah + wl @ ah) - vref).max())
    return out


def test_tolerances_discriminate_weakened_tf32_splits():
    """On the stress constants and the inputs of the GPU tests, both stress bounds (ATOL, ATOL_OPT) sit >= 5x above what 3xTF32
    costs and >= 5x below what each weakened operand split costs, so the GPU tests catch a kernel that drops a low half.  (On the
    suite constants the weakened blends cost only a few 1e-6: those constants cannot tell the splits apart.)
    Emulated, n = 128: blend 3xTF32 2.3e-7, skinning 3xTF32 5.5e-7; pose features lo dropped 1.9e-4, pose blend 1xTF32 3.2e-4,
    shape blend 1xTF32 6.6e-4, skinning W 1xTF32 1.1e-3, skinning A image 1xTF32 9.9e-4."""
    errs = emulate_lbs_errors(stress_assets())
    print({k: f'{v:.2e}' for k, v in errs.items()})
    for a in (ATOL['stress'], ATOL_OPT['stress']):
        for k in ('blend 3xTF32', 'skinning 3xTF32'):
            assert errs[k] <= a / 5, (a, k, errs[k])
        for k in ('pose features lo dropped', 'pose blend 1xTF32', 'shape blend 1xTF32', 'skinning W 1xTF32', 'skinning A image 1xTF32'):
            assert errs[k] >= 5 * a, (a, k, errs[k])
