"""The evaluator against a float64 restatement, element by element: the CSR joint regression, the per-frame Procrustes at its
block edges and on degenerate frames, and the whole Evaluator (every tensor it builds, every per-frame metric row and the six
scalars) at the edges of the heading re-alignment windows.

1. glamr_sparse_regress vs a dense float64 `reg @ vertices` of the same float32 inputs, per output
       |cuda - r64| <= nnz_r * 2^-24 * sum_e |w_e v_e|
   the error bound of the kernel's sequential fmaf chain over the nnz_r entries of row r.
2. glamr_procrustes_align vs oracle.evaluator.similarity_align in float64 of the same float32 inputs.  The kernel computes in
   fp64 and rounds once, so per frame |cuda - o64| <= 2^-22 * max_j |o64[f, j]| (2 ulp of the frame's peak), and the output is
   NaN exactly where the float64 result is.  The same frame set runs host-compiled (tests/host_harness) on the CPU.  Every frame
   aligned alone, in batches of 2 and 3, and inside a batch of 4097 gives the same bits: the reference aligns across frames when
   the batch holds exactly 2 or 3 frames (torch_transform.py:298-302 tests the batch size, not the point dimension); the project
   keeps the per-frame alignment at every batch size.
3. The whole Evaluator vs OracleEvaluator in float64 on every element of
       eval_joints_world, eval_verts_world (estimate and ground truth), eval_joints_world_PA, aligned_trans, aligned_orient (as
       rotation matrices), aligned_eval_joints_world, aligned_eval_verts_world, the per-frame rows of every metric, the six scalars
   held to |cuda - o64| <= C * D(b) + R * 2^-24 * |o64|, where D(b) is the float32 oracle's largest |o32 - o64| in the
   element's 32-frame block of that tensor (floor: 2^-24 of the tensor's peak).  A scalar, the mean of its metric's rows, is
   held to C * D + R * 2^-24 * |o64| with D = |s32 - s64|, or, if larger, to the mean of its rows' bounds plus the same rounding
   term: its error is at most the mean of its rows' errors plus its own rounding.  A NaN anywhere fails the check.  Counts
   must match exactly.  eval_joints_world_PA
   is also held to the bound of 2 against similarity_align in float64 of the CUDA's own eval_joints_world pair, since the float32
   oracle's torch.svd is loose on near-degenerate frames.
4. (CPU) each modelled bug, applied to the float32 oracle, breaks the bound of 3 or of 2; the factor is printed.
5. An Evaluator given a regressor whose width is not the mesh's vertex count raises GlamrError.

C = 4 and R = 8 as in the other float64 checks.  Worst measured ratio to the bound over all cases, on an H100 80GB HBM3 at a
700 W power limit:
    sparse regression            0.67 (rows = 24)
    Procrustes                   0.25 on the GPU, 0.25 host-compiled (J = 2: 6e-8)
    Evaluator, tensors           eval_joints_world 0.41, eval_verts_world 0.44, eval_joints_world_PA 0.34, aligned_trans 0.28,
                                 aligned_orient 0.43, aligned_eval_joints_world 0.38, aligned_eval_verts_world 0.41
    Evaluator, metric rows       0.79 (tracks of 2 and 3 frames; 0.58 elsewhere);  scalars 0.13
    PA stage check               0.25
Before the fix in glamr_b200/csrc/eval_math.cuh, collinear frames whose rank-1 covariance left rounding noise in the second
column of U (a 2-joint cube frame: two points along an axis) missed the Procrustes bound by 2e6x, host-compiled and on the GPU.
"""
import copy
import ctypes
import logging
import math

import numpy as np
import pytest
import torch

from helpers import load_golden

DEV = 'cuda:0'
U = 2.0 ** -24
C, R, FLOOR = 4.0, 8.0, 2.0 ** -24          # block bound; FLOOR is relative to the tensor's peak
PA_ULP = 2.0 ** -22                         # Procrustes: 2 ulp of the frame's peak
BLOCK = 32                                  # frames per block of D
NV = 6890
EINVAL = -1


# ------------------------------------------------------------------------------------------------ the bounds
def block_bound(o32, o64):
    """per-element bound C * D(b) + R * U * |o64| of tensors [n, ...] (frame-major), float64 on o64's device"""
    o32, o64 = o32.to(o64.device, torch.float64), o64.double()
    n = o64.shape[0]
    if n == 0:
        return torch.zeros_like(o64)
    d = (o32 - o64).abs().reshape(n, -1).amax(1)
    bid = torch.arange(n, device=o64.device) // BLOCK
    Db = torch.zeros(int(bid.max()) + 1, dtype=torch.float64, device=o64.device).index_reduce_(0, bid, d, 'amax')
    D = Db[bid].clamp_min(FLOOR * float(o64.abs().max()))
    return C * D.reshape((n,) + (1,) * (o64.dim() - 1)) + R * U * o64.abs()


def ratio(got, o64, bnd):
    """largest |got - o64| / bound (inf if any element is not finite; an exact element scores 0 against a zero bound)"""
    assert got.shape == o64.shape, (got.shape, o64.shape)
    if got.numel() == 0:
        return 0.0
    err = (got.to(o64.device, torch.float64) - o64.double()).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bnd)
    return float(torch.where(torch.isfinite(r), r, torch.full_like(r, math.inf)).max())


def worse(a, b):
    """the larger of two ratios, a NaN counting as infinitely bad (Python's max would drop it)"""
    return math.inf if math.isnan(a) or math.isnan(b) else max(a, b)


def procrustes_ratio(got, o64):
    """per-frame bound of test 2 on [n, J, 3]: NaN exactly where o64 is NaN, elsewhere |got - o64| <= 2^-22 * frame peak"""
    got, o64 = torch.as_tensor(got).double().cpu(), torch.as_tensor(o64).double().cpu()
    assert got.shape == o64.shape
    nan64 = torch.isnan(o64)
    if not torch.equal(torch.isnan(got), nan64):
        return math.inf
    fin = torch.where(nan64, torch.zeros_like(o64), o64)
    peak = fin.abs().reshape(fin.shape[0], -1).amax(1)[:, None, None]
    err = (torch.where(nan64, torch.zeros_like(got), got) - fin).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / (PA_ULP * peak))
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------------ C ABI helpers
def _lib():
    from glamr_b200 import lib as L
    return L.load()


def _vp(t, off=0):
    return ctypes.c_void_p(t.data_ptr() + off)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------ 1. sparse regression
def make_regressor(rows, seed):
    """[rows, 6890] float32 with 4-9 signed weights per row; from 17 rows on, row 3 is empty and row 5 holds all 6890 vertices"""
    rng = np.random.default_rng(seed)
    reg = np.zeros((rows, NV), np.float32)
    for r in range(rows):
        nz = rng.choice(NV, int(rng.integers(4, 10)), replace=False)
        reg[r, nz] = rng.uniform(-1.0, 1.0, nz.size).astype(np.float32)
    if rows >= 17:
        reg[3] = 0.0
        reg[5] = rng.uniform(-1.0, 1.0, NV).astype(np.float32) / 100
    return reg


def to_csr(reg):
    ptr, ci, w = [0], [], []
    for r in range(reg.shape[0]):
        nz = np.nonzero(reg[r])[0]
        ci += nz.tolist()
        w += reg[r, nz].tolist()
        ptr.append(len(ci))
    return (torch.tensor(ptr, dtype=torch.int32, device=DEV), torch.tensor(ci or [0], dtype=torch.int32, device=DEV),
            torch.tensor(w or [0.0], dtype=torch.float32, device=DEV))


@pytest.mark.gpu
@pytest.mark.parametrize('rows', [1, 17, 24])
def test_sparse_regress_matches_float64(rows):
    """every output of glamr_sparse_regress (n * rows * 3 threads of 256: n = 1, 5, 6, 300, 20000 land on both sides of a
    multiple of 256) vs float64, vertices up to +-20 m, output NaN-filled with one canary frame past n"""
    lib = _lib()
    reg = make_regressor(rows, 100 + rows)
    ptr, ci, w = to_csr(reg)
    reg64 = torch.tensor(reg, dtype=torch.float64, device=DEV)
    nnz = torch.tensor((reg != 0).sum(1), dtype=torch.float64, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(rows)
    worst = 0.0
    for n in (1, 5, 6, 300, 20000):
        v = (torch.rand(n, NV, 3, device=DEV, generator=g) * 2 - 1) * 20
        out = torch.full((n + 1, rows, 3), float('nan'), device=DEV)
        assert lib.glamr_sparse_regress(n, NV, rows, _vp(ptr), _vp(ci), _vp(w), _vp(v), _vp(out), _stream()) == 0
        torch.cuda.synchronize()
        assert torch.isnan(out[n]).all(), f'rows={rows} n={n}: written past frame n'
        v64 = v.double()
        r64 = torch.einsum('rv,nvc->nrc', reg64, v64)
        bnd = nnz[None, :, None] * U * torch.einsum('rv,nvc->nrc', reg64.abs(), v64.abs())
        r = ratio(out[:n], r64, bnd)
        assert r <= 1.0, f'rows={rows} n={n}: |cuda - r64| / bound = {r:.3g}'
        if rows >= 17:
            assert torch.equal(out[:n, 3], torch.zeros_like(out[:n, 3])), 'the empty row must regress to exact zeros'
        worst = max(worst, r)
        del v, v64, out
    print(f'EVAL64 sparse_regress rows={rows}: worst ratio {worst:.3g}')


@pytest.mark.gpu
def test_sparse_regress_argument_checks():
    """n == 0 returns OK and writes nothing; n < 0, rows <= 0, V <= 0 or a NULL pointer returns GLAMR_EINVAL"""
    lib = _lib()
    ptr, ci, w = to_csr(make_regressor(17, 1))
    v = torch.rand(2, NV, 3, device=DEV)
    out = torch.rand(2, 17, 3, device=DEV)
    before = out.clone()
    assert lib.glamr_sparse_regress(0, NV, 17, _vp(ptr), _vp(ci), _vp(w), _vp(v), _vp(out), _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(out, before)
    P = [_vp(ptr), _vp(ci), _vp(w), _vp(v), _vp(out)]
    for n, V, rows in ((-1, NV, 17), (2, NV, 0), (2, NV, -1), (2, 0, 17), (2, -5, 17)):
        assert lib.glamr_sparse_regress(n, V, rows, *P, _stream()) == EINVAL, (n, V, rows)
    for k in range(5):
        args = list(P)
        args[k] = None
        assert lib.glamr_sparse_regress(2, NV, 17, *args, _stream()) == EINVAL, k
    torch.cuda.synchronize()
    assert torch.equal(out, before)


# ------------------------------------------------------------------------------------------------ 2. Procrustes
KINDS = ['generic', 'identical', 'rot180', 'reflected', 'planar', 'planar_reflected', 'near_planar', 'collinear', 'collinear_axis',
         'two_points', 'cube', 'tiny', 'far', 's2_point', 's1_point']


def _rotation(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def frame_pair(kind, J, rng):
    """one (S1, S2) pair [J, 3] of the named kind"""
    S1 = rng.normal(0.0, 0.3, (J, 3))
    Rm = _rotation(rng)
    noise = rng.normal(0.0, 0.02, (J, 3))
    if kind == 'generic':
        S2 = 1.3 * S1 @ Rm.T + 0.5 + noise
    elif kind == 'identical':
        S2 = S1.copy()
    elif kind == 'rot180':
        a = rng.normal(size=3)
        a /= np.linalg.norm(a)
        S2 = S1 @ (2 * np.outer(a, a) - np.eye(3)).T
    elif kind == 'reflected':
        S2 = S1 * np.array([1.0, 1.0, -1.0]) + noise
    elif kind in ('planar', 'planar_reflected'):
        S1[:, 2] = 0.0
        c, s = math.cos(0.7), math.sin(0.7)
        S2 = S1 @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T if kind == 'planar' else S1 * np.array([-1.0, 1.0, 1.0])
        S2 = S2 + noise * np.array([1.0, 1.0, 0.0])
    elif kind == 'near_planar':
        S1[:, 2] = 1e-7 * rng.normal(size=J)
        S2 = S1 @ Rm.T + noise
    elif kind == 'collinear':
        d = rng.normal(size=3)
        S1 = rng.normal(size=3) + rng.normal(0.0, 0.3, (J, 1)) * d / np.linalg.norm(d)
        S2 = 1.1 * S1 @ Rm.T + noise
    elif kind == 'collinear_axis':
        t = rng.normal(0.0, 0.3, J)
        S1 = np.stack([t, np.zeros(J), np.zeros(J)], 1)
        S2 = np.stack([np.zeros(J), 2 * t, np.zeros(J)], 1) + np.array([0.1, 0.2, 0.3])
    elif kind == 'two_points':
        P, Q = rng.normal(size=(2, 3)), rng.normal(size=(2, 3))
        S1, S2 = P[np.arange(J) % 2], Q[np.arange(J) % 2]
    elif kind == 'cube':
        corners = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)])
        S1 = corners[np.arange(J) % 8]
        S2 = S1 @ Rm.T
    elif kind == 'tiny':
        S1 = S1 * 1e-5 / 0.3
        S2 = 1.1 * S1 @ Rm.T + noise * 1e-5
    elif kind == 'far':
        S2 = S1 @ Rm.T + noise + 1000.0
        S1 = S1 + 1000.0
    elif kind == 's2_point':
        S2 = np.tile(rng.normal(size=3), (J, 1))
    elif kind == 's1_point':
        S1, S2 = np.tile(rng.normal(size=3), (J, 1)), S1 @ Rm.T + noise
    else:
        raise ValueError(kind)
    return S1.astype(np.float32), S2.astype(np.float32)


def procrustes_frames(n, J, seed):
    """[n, J, 3] float32 S1, S2; frame f is of kind KINDS[(f + J) % len(KINDS)]"""
    rng = np.random.default_rng(seed)
    pairs = [frame_pair(KINDS[(f + J) % len(KINDS)], J, rng) for f in range(n)]
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])


def ref_procrustes(S1, S2):
    from oracle.evaluator import similarity_align
    return similarity_align(torch.as_tensor(S1).double().cpu(), torch.as_tensor(S2).double().cpu())


def host_procrustes(S1, S2):
    import host_harness as hh
    out = np.full(S1.shape, np.nan, np.float32)
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    assert hh.lib().glamr_host_procrustes(S1.shape[0], S1.shape[1], fp(S1), fp(S2), fp(out)) == 0
    return out


PA_SIZES = [1, 2, 3, 127, 128, 129, 4097]
PA_JOINTS = [2, 3, 14, 17, 24]


@pytest.mark.parametrize('J', PA_JOINTS)
def test_host_procrustes_matches_float64(J):
    """the frame function of glamr_procrustes_align, host-compiled without FMA contraction, on every size and frame kind, and
    the same bits whether a frame is aligned alone, in a batch of 2 or 3, or in the batch of 4097"""
    worst = 0.0
    for n in PA_SIZES:
        S1, S2 = procrustes_frames(n, J, 7 * n + J)
        got = host_procrustes(S1, S2)
        r = procrustes_ratio(got, ref_procrustes(S1, S2))
        assert r <= 1.0, f'n={n} J={J}: ratio {r:.3g}'
        worst = max(worst, r)
    for k in (1, 2, 3):
        parts = [host_procrustes(S1[s:s + k], S2[s:s + k]) for s in range(0, S1.shape[0], k)]
        assert np.array_equal(np.concatenate(parts).view(np.int32), got.view(np.int32)), f'J={J}: batches of {k} differ'
    print(f'EVAL64 host procrustes J={J}: worst ratio {worst:.3g}')


def test_oracle_similarity_align_is_per_frame():
    """the oracle aligns every frame on its own at n = 2 and 3 too (the reference's batch-size test is not mirrored)"""
    from oracle.evaluator import similarity_align
    S1, S2 = procrustes_frames(3, 17, 5)
    S1, S2 = torch.tensor(S1).double(), torch.tensor(S2).double()
    alone = torch.cat([similarity_align(S1[f:f + 1], S2[f:f + 1]) for f in range(3)])
    for n in (2, 3):
        torch.testing.assert_close(similarity_align(S1[:n], S2[:n]), alone[:n], rtol=0, atol=1e-12, equal_nan=True)


def cuda_procrustes(S1, S2):
    """glamr_procrustes_align on NaN-filled output with one canary frame past n"""
    n, J = S1.shape[:2]
    a, b = torch.as_tensor(S1).to(DEV).contiguous(), torch.as_tensor(S2).to(DEV).contiguous()
    out = torch.full((n + 1, J, 3), float('nan'), device=DEV)
    assert _lib().glamr_procrustes_align(n, J, _vp(a), _vp(b), _vp(out), _stream()) == 0
    torch.cuda.synchronize()
    assert torch.isnan(out[n]).all(), 'written past frame n'
    return out[:n]


@pytest.mark.gpu
@pytest.mark.parametrize('J', PA_JOINTS)
def test_cuda_procrustes_matches_float64(J):
    """glamr_procrustes_align (128-thread blocks: n = 127, 128, 129 and 4097) on every frame kind vs float64, and batch invariance:
    each frame of the 4097 gives the same bits aligned alone and in consecutive batches of 2 and 3"""
    lib = _lib()
    worst = 0.0
    for n in PA_SIZES:
        S1, S2 = procrustes_frames(n, J, 7 * n + J)
        got = cuda_procrustes(S1, S2)
        r = procrustes_ratio(got.cpu(), ref_procrustes(S1, S2))
        assert r <= 1.0, f'n={n} J={J}: ratio {r:.3g}'
        worst = max(worst, r)
    a, b = torch.tensor(S1, device=DEV), torch.tensor(S2, device=DEV)
    n, fb = a.shape[0], J * 3 * 4
    for k in (1, 2, 3):
        out = torch.full_like(a, float('nan'))
        for s in range(0, n, k):
            assert lib.glamr_procrustes_align(min(k, n - s), J, _vp(a, s * fb), _vp(b, s * fb), _vp(out, s * fb), _stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), got.view(torch.int32)), f'J={J}: batches of {k} differ from the batch of {n}'
    print(f'EVAL64 cuda procrustes J={J}: worst ratio {worst:.3g}')


@pytest.mark.gpu
def test_procrustes_argument_checks():
    lib = _lib()
    a = torch.rand(2, 14, 3, device=DEV)
    out = torch.rand(2, 14, 3, device=DEV)
    before = out.clone()
    assert lib.glamr_procrustes_align(0, 14, _vp(a), _vp(a), _vp(out), _stream()) == 0
    for n, J in ((-1, 14), (2, 0), (2, -3)):
        assert lib.glamr_procrustes_align(n, J, _vp(a), _vp(a), _vp(out), _stream()) == EINVAL, (n, J)
    for k in range(3):
        args = [_vp(a), _vp(a), _vp(out)]
        args[k] = None
        assert lib.glamr_procrustes_align(2, 14, *args, _stream()) == EINVAL, k
    torch.cuda.synchronize()
    assert torch.equal(out, before)


# ------------------------------------------------------------------------------------------------ 3. the whole Evaluator
PD_TENSORS = ['eval_joints_world', 'eval_verts_world', 'eval_joints_world_PA', 'aligned_trans', 'aligned_orient',
              'aligned_eval_joints_world', 'aligned_eval_verts_world']
GT_TENSORS = ['eval_joints_world', 'eval_verts_world', 'aligned_trans', 'aligned_orient', 'aligned_eval_joints_world',
              'aligned_eval_verts_world']
SCALARS = ['PA-MPJPE', 'PA-MPJPE-vis', 'PA-MPJPE-invis', 'G-MPJPE', 'G-MPVE', 'ACCEL']
ROW_METRICS = [('PA-MPJPE', 'eval_joints_world_PA', 'eval_joints_world', 'all'),
               ('PA-MPJPE-vis', 'eval_joints_world_PA', 'eval_joints_world', 'vis'),
               ('PA-MPJPE-invis', 'eval_joints_world_PA', 'eval_joints_world', 'invis'),
               ('G-MPJPE', 'aligned_eval_joints_world', 'aligned_eval_joints_world', 'all'),
               ('G-MPVE', 'aligned_eval_verts_world', 'aligned_eval_verts_world', 'all')]


def rotmat(aa):
    """exact axis-angle -> rotation matrix in float64 [n, 9]"""
    aa = aa.double()
    th = aa.norm(dim=-1, keepdim=True)
    k = aa / th.clamp_min(1e-300)
    K = torch.zeros(aa.shape[:-1] + (3, 3), dtype=torch.float64, device=aa.device)
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 2] = -k[..., 2], k[..., 1], -k[..., 0]
    K = K - K.transpose(-1, -2)
    s, c = torch.sin(th)[..., None], torch.cos(th)[..., None]
    return (torch.eye(3, dtype=torch.float64, device=aa.device) + s * K + (1 - c) * K @ K).reshape(aa.shape[:-1] + (9,))


def metric_rows(data, accel_shift=0):
    """the per-frame rows of every metric (mm), persons concatenated, in the data's dtype"""
    rows = {}
    for name, ek, gk, mode in ROW_METRICS:
        parts = []
        for idx, pd in data['person_data'].items():
            e, g = pd[ek], data['gt'][idx][gk]
            if mode != 'all':
                m = pd['vis_frames' if mode == 'vis' else 'invis_frames']
                e, g = e[m], g[m]
            parts.append(torch.norm(e - g, dim=2).mean(dim=1) * 1000)
        rows[name] = torch.cat(parts)
    parts = []
    for idx, pd in data['person_data'].items():
        j, g = pd['eval_joints_world'], data['gt'][idx]['eval_joints_world']
        a, ga = j[:-2] - 2 * j[1:-1] + j[2:], g[:-2] - 2 * g[1:-1] + g[2:]
        if accel_shift and a.shape[0] > 1:               # modelled bug: the estimate's acceleration one frame late
            a = a[torch.clamp(torch.arange(a.shape[0], device=a.device) + accel_shift, max=a.shape[0] - 1)]
        parts.append(torch.norm(a - ga, dim=2).mean(dim=1) * 1000)
    rows['ACCEL'] = torch.cat(parts)
    return rows


def evaluator_ratios(got, got_scalars, o32, s32, o64, s64, got_rows=None):
    """{what: worst ratio to the block bound} over every tensor, every per-frame metric row and the six scalars of one case.
    got / o32 / o64: data dicts after prepare_seq; *_scalars: {metric: (value, count)}.  Counts must match exactly."""
    out = {}

    def put(what, r):
        out[what] = worse(out.get(what, 0.0), r)

    for side, keys in (('person_data', PD_TENSORS), ('gt', GT_TENSORS)):
        for idx in o64[side]:
            for k in keys:
                g, a, b = got[side][idx][k], o32[side][idx][k], o64[side][idx][k]
                if k == 'aligned_orient':
                    g, a, b = rotmat(g.to(b.device)), rotmat(a.to(b.device)), rotmat(b)
                assert g.shape == b.shape, (side, idx, k, g.shape, b.shape)
                put(k, ratio(g, b, block_bound(a, b)))
    rows64, rows32 = metric_rows(o64), metric_rows(o32)
    got_rows = metric_rows(got) if got_rows is None else got_rows
    for k in rows64:
        if got_rows[k].shape != rows64[k].shape:
            put('rows ' + k, math.inf)
            continue
        put('rows', ratio(got_rows[k], rows64[k], block_bound(rows32[k], rows64[k])))
    for k in SCALARS:
        (g, ng), (a, na), (b, nb) = got_scalars[k], s32[k], s64[k]
        assert na == nb
        if ng != nb:
            put('count ' + k, math.inf)
            continue
        # a scalar is the mean of its rows, so its error is at most the mean of the rows' bounds plus its own rounding; it is
        # held to the larger of that and the block construction with D = |s32 - s64|
        D = max(abs(a - b), FLOOR * abs(b))
        mean_row_bound = float(block_bound(rows32[k], rows64[k]).mean()) if rows64[k].numel() else 0.0
        bound = max(C * D, mean_row_bound) + R * U * abs(b)
        put('scalars', abs(g - b) / bound if g != b else 0.0)
    return out


def _torchify(d):
    if isinstance(d, np.ndarray):
        return torch.tensor(d)
    if isinstance(d, dict):
        return {k: _torchify(v) for k, v in d.items()}
    return d


def run_oracle(assets, reg, case, dataset, freq, dtype, device, cls=None):
    from oracle.evaluator import OracleEvaluator
    ev = (cls or OracleEvaluator)(assets, reg, dataset=dataset, align_freq=freq, dtype=dtype, device=device)
    data = _torchify(copy.deepcopy(case))
    return data, ev.metrics(data)


def _all_exist(case):
    for pd in case['person_data'].values():
        pd['exist_frames'][:] = True
    return case


def eval_case(name):
    """(case, dataset, align_freq) built from make_eval_case plus edits"""
    from glamr_b200.synthetic import make_eval_case
    gold_cases = {'p2_t60': ('3DPW', 2, 60, 250), 'p1_t300_h36m': ('h36m', 1, 300, 250), 'p1_t90_realign': ('3DPW', 1, 90, 40)}
    if name in gold_cases:
        dataset, P, T, freq = gold_cases[name]
        return make_eval_case(P, T, seed=int(load_golden('evaluator')[f'{name}/seed'])), dataset, freq
    if name == 'p2_t1000':                      # 3 full windows and a ragged fourth (person 0 exists on 997 frames)
        return make_eval_case(2, 1000, seed=11), '3DPW', 250
    if name == 'p1_t1001_h36m':                 # every frame exists: the last window is the overlap frame plus one
        return _all_exist(make_eval_case(1, 1001, seed=12)), 'h36m', 250
    if name == 'p1_t751':                       # 748 frames exist: a ragged last window of 249
        return make_eval_case(1, 751, seed=13), '3DPW', 250
    if name == 'p1_t40_freq1':                  # every window holds two frames
        return make_eval_case(1, 40, seed=14), '3DPW', 1
    if name == 'p2_exist2_exist3':              # tracks of exactly 2 and 3 frames: the per-frame Procrustes at n = 2 and 3
        case = make_eval_case(2, 60, seed=15)
        for p, frames in ((0, [10, 31]), (1, [5, 6, 40])):
            ex = np.zeros(60, bool)
            ex[frames] = True
            case['person_data'][p]['exist_frames'] = ex
            case['person_data'][p]['visible_orig'][frames] = [1, 0, 1][:len(frames)]
        return case, '3DPW', 250
    if name == 'p1_all_visible':                # no invisible frame anywhere: the invis counts are 0
        case = make_eval_case(1, 60, seed=16)
        case['person_data'][0]['visible_orig'][:] = 1
        return case, '3DPW', 25
    if name == 'p2_vis_split':                  # one person always visible, the other never
        case = make_eval_case(2, 60, seed=17)
        case['person_data'][0]['visible_orig'][:] = 1
        case['person_data'][1]['visible_orig'][:] = 0
        return case, 'h36m', 25
    if name == 'p2_scale_partial':              # a per-frame scale on a partial track: filtered by exist_frames too
        case = make_eval_case(2, 80, seed=18)
        for pd in case['person_data'].values():
            pd['scale'] = (0.9 + 0.2 * np.random.default_rng(19).random(80)).astype(np.float32)
        return case, '3DPW', 30
    raise KeyError(name)


EVAL_CASES = ['p2_t60', 'p1_t300_h36m', 'p1_t90_realign', 'p2_t1000', 'p1_t1001_h36m', 'p1_t751', 'p1_t40_freq1', 'p2_exist2_exist3',
              'p1_all_visible', 'p2_vis_split', 'p2_scale_partial']


@pytest.fixture(scope='module')
def cuda_smpl(smpl_assets):
    from glamr_b200.smpl import SMPL
    return SMPL(smpl_assets, device=DEV)


@pytest.fixture
def no_tf32():
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.gpu
@pytest.mark.parametrize('name', EVAL_CASES)
def test_evaluator_matches_float64(name, smpl_assets, cuda_smpl, no_tf32):
    """compute_sequence_metrics vs OracleEvaluator in float64 (both oracles on the GPU, TF32 off) on every element of every
    tensor the evaluator builds, every per-frame metric row and the six scalars; eval_joints_world_PA also against float64
    similarity_align of the CUDA's own eval_joints_world pair"""
    from glamr_b200.evaluator import Evaluator
    from glamr_b200.synthetic import make_h36m_regressor
    from oracle.evaluator import similarity_align
    case, dataset, freq = eval_case(name)
    reg = make_h36m_regressor(0)
    ev = Evaluator('glamr', dataset, device=torch.device(DEV), align_freq=freq, compute_sample=True, smpl=cuda_smpl, h36m_regressor=reg,
                   log=logging.getLogger('test_evaluator_float64'))
    md = ev.compute_sequence_metrics(copy.deepcopy(case), 'case', accumulate=False)
    got = ev.last_data
    got_scalars = {k: (md['metrics'][k].avg, md['metrics'][k].count) for k in SCALARS}
    o64, s64 = run_oracle(smpl_assets, reg, case, dataset, freq, torch.float64, DEV)
    o32, s32 = run_oracle(smpl_assets, reg, case, dataset, freq, torch.float32, DEV)
    ratios = evaluator_ratios(got, got_scalars, o32, s32, o64, s64)
    # the product's own per-frame rows (the sample metric) against the oracle's invisible-frame rows
    rows64, rows32 = metric_rows(o64)['PA-MPJPE-invis'], metric_rows(o32)['PA-MPJPE-invis']
    sample = torch.as_tensor(np.asarray(md['metrics']['sample_PA-MPJPE-invis'].avg, np.float32), device=DEV)
    assert md['metrics']['sample_PA-MPJPE-invis'].count == s64['PA-MPJPE-invis'][1]
    ratios['rows'] = worse(ratios['rows'], ratio(sample, rows64, block_bound(rows32, rows64)))
    stage = 0.0
    for idx, pd in got['person_data'].items():
        o = similarity_align(pd['eval_joints_world'].double().cpu(), got['gt'][idx]['eval_joints_world'].double().cpu())
        stage = worse(stage, procrustes_ratio(pd['eval_joints_world_PA'].cpu(), o))
    ratios['PA stage'] = stage
    print(f'EVAL64 evaluator {name}: ' + ', '.join(f'{k} {v:.3g}' for k, v in ratios.items()))
    bad = {k: v for k, v in ratios.items() if not v <= 1.0}
    assert not bad, f'{name}: over the bound {bad}'


# ------------------------------------------------------------------------------------------------ 4. the bounds reject modelled bugs
def procrustes_variant(S1, S2, bug):
    """similarity_align in float64 with one modelled bug, rounded to float32 like the kernel's output"""
    S1, S2 = torch.as_tensor(S1).double().permute(0, 2, 1), torch.as_tensor(S2).double().permute(0, 2, 1)
    X1, X2 = S1 - S1.mean(-1, keepdim=True), S2 - S2.mean(-1, keepdim=True)
    var1 = (X1 ** 2).sum((1, 2))
    if bug == 'K float32':
        K32 = X1.float().bmm(X2.float().permute(0, 2, 1))
        U_, s_, V_ = torch.svd(K32)
        K, Uk, Vk = K32.double(), U_.double(), V_.double()
    else:
        K = X2.bmm(X1.permute(0, 2, 1)) if bug == 'K transposed' else X1.bmm(X2.permute(0, 2, 1))
        Uk, _, Vk = torch.svd(K)
    Z = torch.eye(3, dtype=torch.float64).repeat(K.shape[0], 1, 1)
    if bug != 'Z = I':
        Z[:, -1, -1] *= torch.sign(torch.det(Uk.bmm(Vk.permute(0, 2, 1))))
    Rm = Vk.bmm(Z.bmm(Uk.permute(0, 2, 1)))
    tr = torch.diagonal(K if bug == 'scale from trace(K)' else Rm.bmm(K), dim1=1, dim2=2).sum(-1)
    scale = tr / var1
    t = S2.mean(-1, keepdim=True) - scale[:, None, None] * Rm.bmm(S1.mean(-1, keepdim=True))
    return (scale[:, None, None] * Rm.bmm(S1) + t).permute(0, 2, 1).float()


@pytest.mark.parametrize('bug', ['Z = I', 'scale from trace(K)', 'K transposed', 'K float32'])
def test_procrustes_bound_rejects_modelled_bug(bug):
    """each modelled Procrustes bug breaks the bound of test 2 on its frame set (J = 17, 600 frames of every kind).  Measured:
    Z = I 9.7e6x, scale from trace(K) 8.2e6x, K transposed 1.0e7x; K accumulated and decomposed in float32 only 4.6x (rot180 and
    reflected frames; 1.9-2.8x on generic, planar, collinear, cube and tiny frames, within the bound on far and axis-collinear
    frames)"""
    S1, S2 = procrustes_frames(600, 17, 3)
    ref = ref_procrustes(S1, S2)
    assert procrustes_ratio(procrustes_variant(S1, S2, None), ref) <= 1.0
    r = procrustes_ratio(procrustes_variant(S1, S2, bug), ref)
    print(f'EVAL64 modelled Procrustes bug {bug!r}: {r:.3g} x the bound')
    assert r > 1.0, (bug, r)


BUG_ROW = 6                                 # an H36M row that reaches the evaluated joints (H36M_TO_J15[1])


def _bug_regressor(reg, bug):
    reg = reg.copy()
    nz = np.nonzero(reg[BUG_ROW])[0]
    if bug == 'CSR row without its last non-zero':
        reg[BUG_ROW, nz[-1]] = 0.0
    else:
        col = nz[0]
        assert reg[BUG_ROW, col + 1] == 0
        reg[BUG_ROW, col + 1], reg[BUG_ROW, col] = reg[BUG_ROW, col], 0.0
    return reg


def _no_overlap_oracle():
    from oracle import rotations as rt
    from oracle.evaluator import OracleEvaluator, world2heading

    class NoOverlap(OracleEvaluator):
        def aligned(self, d):
            oq, tr = rt.aa_to_quat(d['smpl_orient_world']), d['root_trans_world']
            qs, ts = [], []
            for i in range(int(np.ceil(oq.shape[0] / self.align_freq))):
                q, t = world2heading(oq[i * self.align_freq:(i + 1) * self.align_freq], tr[i * self.align_freq:(i + 1) * self.align_freq])
                qs.append(q)
                ts.append(t)
            d['aligned_orient'] = rt.quat_to_aa(torch.cat(qs))
            d['aligned_trans'] = torch.cat(ts)
    return NoOverlap


def _wrong_pelvis(data):
    """pelvis from J15 joints 2 and 3 instead of 3 and 4: shift eval_joints / eval_verts, redo PA"""
    from oracle.evaluator import similarity_align
    for d in list(data['person_data'].values()) + list(data['gt'].values()):
        shift = (d['eval_joints_world'][:, [1]] + d['eval_joints_world'][:, [2]]) * 0.5
        d['eval_joints_world'] = d['eval_joints_world'] - shift
        d['eval_verts_world'] = d['eval_verts_world'] - shift
    for idx, pd in data['person_data'].items():
        pd['eval_joints_world_PA'] = similarity_align(pd['eval_joints_world'], data['gt'][idx]['eval_joints_world'])


def _scalars_from(data, rows, s):
    """recompute the scalars after a post-hoc bug"""
    out = dict(s)
    for k in SCALARS:
        r = rows[k]
        out[k] = (float(r.sum() / r.shape[0]) if r.shape[0] else 0.0, int(r.shape[0]))
    return out


TEST3_BUGS = ['CSR row without its last non-zero', 'CSR column off by one', 'windows without the one-frame overlap',
              'pelvis from the wrong J15 pair', 'visible_orig not filtered by exist frames', 'ACCEL one frame late']


@pytest.fixture(scope='module')
def cpu_case(smpl_assets):
    """a 2-person, 60-frame 3DPW case at align_freq 20 with its float64 and float32 oracles on the CPU"""
    from glamr_b200.synthetic import make_eval_case, make_h36m_regressor
    case, dataset, freq = make_eval_case(2, 60, seed=21), '3DPW', 20
    reg = make_h36m_regressor(0)
    o64, s64 = run_oracle(smpl_assets, reg, case, dataset, freq, torch.float64, 'cpu')
    o32, s32 = run_oracle(smpl_assets, reg, case, dataset, freq, torch.float32, 'cpu')
    return case, dataset, freq, reg, o64, s64, o32, s32


@pytest.mark.parametrize('bug', TEST3_BUGS)
def test_evaluator_bound_rejects_modelled_bug(bug, smpl_assets, cpu_case):
    """each modelled evaluator bug, applied to the float32 oracle (CPU), breaks the bound of test 3 on a 2-person, 60-frame case
    at align_freq 20 (a count that differs counts as an infinite ratio)"""
    case, dataset, freq, reg, o64, s64, o32, s32 = cpu_case
    base = evaluator_ratios(o32, s32, o32, s32, o64, s64)
    assert max(base.values()) <= 1.0 / C + 1e-12, base              # the float32 oracle sits at D: ratio <= 1 / C
    bug_case, cls, bug_reg, rows = copy.deepcopy(case), None, reg, None
    if bug.startswith('CSR'):
        bug_reg = _bug_regressor(reg, bug)
    elif bug.startswith('windows'):
        cls = _no_overlap_oracle()
    elif bug.startswith('visible_orig'):
        for pd in bug_case['person_data'].values():
            ex, vis = pd['exist_frames'], pd['visible_orig']
            vis[ex] = vis[:int(ex.sum())].copy()                       # frame t of the track reads the unfiltered mask's frame t
    got, sg = run_oracle(smpl_assets, bug_reg, bug_case, dataset, freq, torch.float32, 'cpu', cls)
    if bug.startswith('pelvis'):
        _wrong_pelvis(got)
        rows = metric_rows(got)
        sg = _scalars_from(got, rows, sg)
    elif bug.startswith('ACCEL'):
        rows = metric_rows(got, accel_shift=1)
        sg = _scalars_from(got, rows, sg)
    r = evaluator_ratios(got, sg, o32, s32, o64, s64, got_rows=rows)
    worst = max(r.values())
    print(f'EVAL64 modelled evaluator bug {bug!r}: {worst:.3g} x the bound ({max(r, key=r.get)})')
    assert worst > 1.0, (bug, r)


@pytest.mark.parametrize('where', ['eval_verts_world', 'aligned_trans', 'aligned_orient', 'eval_joints_world_PA', 'G-MPVE', 'rows'])
def test_evaluator_ratios_reject_nan(where, cpu_case):
    """a single NaN in a tensor, a scalar or a per-frame row of the checked result fails the bound of test 3"""
    _, _, _, _, o64, s64, o32, s32 = cpu_case
    got, sg, rows = copy.deepcopy(o32), dict(s32), None
    if where == 'G-MPVE':
        sg[where] = (math.nan, sg[where][1])
    elif where == 'rows':
        rows = metric_rows(got)
        rows['ACCEL'][7] = math.nan
    else:
        t = got['person_data'][1][where]
        t[(5,) + (0,) * (t.dim() - 2) + (1,)] = math.nan
    r = evaluator_ratios(got, sg, o32, s32, o64, s64, got_rows=rows)
    assert max(r.values()) == math.inf, (where, r)


# ------------------------------------------------------------------------------------------------ 5. regressor validation
@pytest.mark.gpu
def test_evaluator_rejects_regressor_of_wrong_width(smpl_assets, cuda_smpl):
    """a [17, 6000] regressor (narrower than the mesh) is refused at construction, before any kernel reads with its stride"""
    from glamr_b200.evaluator import Evaluator
    from glamr_b200.lib import GlamrError
    from glamr_b200.synthetic import make_h36m_regressor
    reg = make_h36m_regressor(0)[:, :6000]
    with pytest.raises(GlamrError):
        ev = Evaluator('glamr', '3DPW', device=torch.device(DEV), smpl=cuda_smpl, h36m_regressor=reg, log=logging.getLogger('t'))
        ev.compute_sequence_metrics(eval_case('p2_t60')[0], 'case', accumulate=False)
    ev = Evaluator('glamr', '3DPW', device=torch.device(DEV), smpl=cuda_smpl, h36m_regressor=make_h36m_regressor(0),
                   log=logging.getLogger('t'))
    with pytest.raises(GlamrError):
        ev.regress_h36m(torch.zeros(2, 7000, 3, device=DEV))        # wider than the regressor: unchecked reads stay in bounds
