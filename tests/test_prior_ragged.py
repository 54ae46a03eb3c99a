"""Tracks of different lengths in one learned-prior call (MotionTrajJointModel.inference with `seq_len`).

GPU: every row of a ragged call is bit-identical to the single-track call it reproduces, across the infiller's window edges
(T = 10 + 30 k, + 1), the trajectory predictor's GEMM classes (T * row_batch around 256) and its window edges, in both predictor
modes, with drawn and explicit latents and sample_num 1 and 3; blocks of equal-length rows (row_batch) reproduce the block's own
call; GLAMR_PRIOR_GRAPH=1 keeps the equalities; `optimize` on persons of different exist ranges makes one prior call and returns
what the person-by-person path returns.  CPU: the host plan and the eps draws."""
import copy
import types

import numpy as np
import pytest
import torch

from glamr_b200 import motion_traj as MT

DEV = 'cuda:0'
LENS = [11, 40, 41, 70, 71, 100, 101, 256, 257, 300, 601, 1100]
KEYS_BS = ('infer_out_body_pose', 'infer_out_trans', 'infer_out_orient', 'infer_out_pose')


# ------------------------------------------------------------------------------------------------ CPU: host plan and eps draws
def test_plan_orders_rows_by_kernel_class():
    p = MT.ragged_plan([300, 40, 70, 70, 70, 70, 70, 70, 101], [1, 1, 6, 6, 6, 6, 6, 6, 1], 1, 100, False)
    assert p['blocks'] == [(0, 1), (1, 1), (2, 6), (8, 1)]
    assert list(p['nwin']) == [10, 1, 2, 2, 2, 2, 2, 2, 4]
    # infiller: class of row_batch (6 -> the 50-row Linears go large), then decreasing length
    assert list(p['inf_order']) == [0, 8, 1, 2, 3, 4, 5, 6, 7]
    # predictor: T * row_batch > 256 (300, 70 * 6) after the skinny rows (40, 101)
    assert list(p['pred_order']) == [1, 8, 0, 2, 3, 4, 5, 6, 7]
    assert list(p['inf_off']) == [0, 300, 401, 441, 511, 581, 651, 721, 791, 861]
    assert list(p['pred_off']) == [0, 40, 141, 441, 511, 581, 651, 721, 791, 861]


def test_plan_windowed_and_samples():
    p = MT.ragged_plan([257, 60], None, 3, 100, True)
    assert p['E'] == 6 and list(p['row_batch']) == [3] * 6 and list(p['lens']) == [257] * 3 + [60] * 3
    assert list(p['C']) == [3, 3, 3, 1, 1, 1]
    # windowed class: (C W rb > 256) + (C rb > 256); 60 frames x 3 samples = 300 window frames > 256 too
    assert list(p['pred_order']) == [0, 1, 2, 3, 4, 5]
    assert list(p['pred_woff']) == [0, 3, 6, 9, 10, 11, 12]
    assert list(p['inf_order']) == [0, 1, 2, 3, 4, 5]


def test_plan_rejects_bad_blocks_and_short_tracks():
    from glamr_b200.lib import GlamrError
    with pytest.raises(ValueError):
        MT.ragged_plan([40, 41], [2, 2])
    with pytest.raises(ValueError):
        MT.ragged_plan([40, 40, 40], [2, 2, 2])
    with pytest.raises(GlamrError):
        MT.ragged_plan([40, 10])


@pytest.mark.parametrize('multi_step', [False, True])
def test_eps_draws_equal_serial_draws(multi_step):
    """the eps of one ragged call, drawn on the CPU generator, equal what the single-track calls draw in turn"""
    lens, rb, S = [71, 40, 40, 300, 41], [1, 2, 2, 1, 1], 2
    p = MT.ragged_plan(lens, rb, S, 100, multi_step)
    torch.manual_seed(7)
    inf, traj = MT.draw_ragged_eps(p, 'cpu')
    torch.manual_seed(7)
    for b0, P in p['blocks']:
        T, n = lens[b0], P * S
        nwin, C = -(-(T - 10) // 30), -(-T // 100)
        ei = torch.randn((nwin, n, 128))                       # MotionInfillerVAE._windows
        et = torch.randn((C, n, 128)) if multi_step else torch.randn((n, 128))   # TrajPredVAE._forward_windows / _forward
        for j in range(n):
            e = b0 * S + j
            assert torch.equal(inf[e, :nwin], ei[:, j]) and not inf[e, nwin:].any()
            assert torch.equal(traj[e], et[:, j] if multi_step else et[j])


# ------------------------------------------------------------------------------------------------ GPU
def _model(multi_step, graph=False, monkeypatch=None):
    from glamr_b200.smpl import SMPL
    from glamr_b200.synthetic import make_smpl_assets
    from glamr_b200.synthetic_nets import make_prior_states
    if monkeypatch is not None:
        monkeypatch.setenv('GLAMR_PRIOR_GRAPH', '1' if graph else '0')
    cfg = types.SimpleNamespace(multi_step_mfiller=True, multi_step_trajpred=multi_step, trajpred_seq_len=100)
    return MT.MotionTrajJointModel(cfg, torch.device(DEV), None, smpl=SMPL(make_smpl_assets(0), device=DEV),
                                   states=make_prior_states(1234))


def _inputs(lens, seed=0):
    g = torch.Generator().manual_seed(seed)
    B, Tm = len(lens), max(lens)
    pose = torch.zeros(B, Tm, 69)
    mask = torch.zeros(B, Tm)
    for b, T in enumerate(lens):
        pose[b, :T] = torch.cumsum(torch.randn(T, 69, generator=g) * 0.02, 0) + torch.randn(1, 69, generator=g) * 0.2
        m = (torch.rand(T, generator=g) > 0.25).float()
        m[:10] = 1
        mask[b, :T] = m
        pose[b, :T] *= m[:, None]
    return pose.to(DEV), mask.to(DEV)


def _latents(lens, S, multi_step, seed=3):
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    nwin = max(-(-(T - 10) // 30) for T in lens)
    lat = {'in_motion_latent': torch.randn(B, nwin, 128, generator=g).to(DEV)}
    if multi_step:
        lat['in_traj_window_latent'] = torch.randn(max(-(-T // 100) for T in lens), B * S, 128, generator=g).to(DEV)
    else:
        lat['in_traj_latent'] = torch.randn(B * S, 128, generator=g).to(DEV)
    return lat


def _serial_latents(lat, rows, lens, S, multi_step):
    """the latents of the single call on rows [rows] (one block of equal length)"""
    T = lens[rows[0]]
    nwin, C = -(-(T - 10) // 30), -(-T // 100)
    out = {'in_motion_latent': lat['in_motion_latent'][rows][:, :nwin].contiguous()}
    cols = [b * S + s for b in rows for s in range(S)]
    if multi_step:
        out['in_traj_window_latent'] = lat['in_traj_window_latent'][:C, cols].contiguous()
    else:
        out['in_traj_latent'] = lat['in_traj_latent'][cols].contiguous()
    return out


def _check_rows(out, ref, rows, lens):
    """rows of the ragged output against the serial output of the block `rows`, bit for bit; zeros past each row's end"""
    for j, b in enumerate(rows):
        T = lens[b]
        for k in KEYS_BS:
            a, r = out[k][b], ref[k][j]
            assert torch.equal(a[:, :T], r), (k, b, T)
            assert not a[:, T:].any(), (k, b)
        a, r = out['infer_out_local_traj_tp'][:, b], ref['infer_out_local_traj_tp'][:, j]
        assert torch.equal(a[:T], r), ('infer_out_local_traj_tp', b, T)
        assert not a[T:].any()


def _serial_block(model, pose, mask, rows, lens, S, lat, multi_step):
    T = lens[rows[0]]
    batch = {'in_body_pose': pose[rows][:, :T].contiguous(), 'frame_mask': mask[rows][:, :T].contiguous()}
    if lat is not None:
        batch.update(_serial_latents(lat, rows, lens, S, multi_step))
    return model.inference(batch, sample_num=S)


@pytest.mark.gpu
@pytest.mark.parametrize('multi_step', [False, True])
@pytest.mark.parametrize('explicit', [False, True])
@pytest.mark.parametrize('S', [1, 3])
def test_ragged_rows_equal_single_track_calls(multi_step, explicit, S):
    model = _model(multi_step)
    lens = LENS
    pose, mask = _inputs(lens)
    lat = _latents(lens, S, multi_step) if explicit else None
    batch = {'in_body_pose': pose, 'frame_mask': mask, 'seq_len': lens, **(lat or {})}
    torch.manual_seed(11)
    out = model.inference(batch, sample_num=S)
    torch.manual_seed(11)
    for b in range(len(lens)):
        ref = _serial_block(model, pose, mask, [b], lens, S, lat, multi_step)
        _check_rows(out, ref, [b], lens)


@pytest.mark.gpu
@pytest.mark.parametrize('multi_step', [False, True])
@pytest.mark.parametrize('S', [1, 3])
def test_row_batch_block_equals_block_call(multi_step, S):
    """a block of 6 equal-length persons (its infiller encoder on the tensor cores) and a block of 2 next to lone tracks; with
    sample_num 3 the block's rows are expanded person by person, as the block call's repeat_interleave does"""
    model = _model(multi_step)
    lens = [300, 40] + [70] * 6 + [101, 257, 45, 45]
    rb = [1, 1] + [6] * 6 + [1, 1, 2, 2]
    pose, mask = _inputs(lens, seed=1)
    torch.manual_seed(5)
    out = model.inference({'in_body_pose': pose, 'frame_mask': mask, 'seq_len': lens}, sample_num=S, row_batch=rb)
    torch.manual_seed(5)
    for rows in ([0], [1], list(range(2, 8)), [8], [9], [10, 11]):
        _check_rows(out, _serial_block(model, pose, mask, rows, lens, S, None, multi_step), rows, lens)


@pytest.mark.gpu
@pytest.mark.parametrize('multi_step', [False, True])
def test_ragged_under_prior_graph(multi_step, monkeypatch):
    model = _model(multi_step, graph=True, monkeypatch=monkeypatch)
    lens = [41, 300, 101, 70]
    pose, mask = _inputs(lens, seed=2)
    lat = _latents(lens, 1, multi_step)
    for _ in range(3):                           # eager + capture, then replays
        out = model.inference({'in_body_pose': pose, 'frame_mask': mask, 'seq_len': lens, **lat}, sample_num=1)
        for b in range(len(lens)):
            _check_rows(out, _serial_block(model, pose, mask, [b], lens, 1, lat, multi_step), [b], lens)


@pytest.mark.gpu
@pytest.mark.parametrize('multi_step', [False, True])
def test_ragged_under_prior_graph_drawn_eps(multi_step, monkeypatch):
    """The ragged call draws its eps before the graph runs, in the serial calls' order: under GLAMR_PRIOR_GRAPH=1 every call,
    eager, capturing or replaying, gives what the single-track calls give eagerly from the same seed."""
    lens = [41, 300, 101, 70]
    pose, mask = _inputs(lens, seed=4)
    model = _model(multi_step, graph=True, monkeypatch=monkeypatch)
    outs = []
    for _ in range(3):
        torch.manual_seed(9)
        outs.append(model.inference({'in_body_pose': pose, 'frame_mask': mask, 'seq_len': lens}, sample_num=1))
    monkeypatch.setenv('GLAMR_PRIOR_GRAPH', '0')
    model.mfiller.graphs.enabled = model.traj_predictor.graphs.enabled = False
    torch.manual_seed(9)
    refs = [_serial_block(model, pose, mask, [b], lens, 1, None, multi_step) for b in range(len(lens))]
    for out in outs:
        for b in range(len(lens)):
            _check_rows(out, refs[b], [b], lens)


@pytest.mark.gpu
def test_short_track_raises():
    from glamr_b200.lib import GlamrError
    model = _model(False)
    pose, mask = _inputs([40, 10])
    with pytest.raises(GlamrError):
        model.inference({'in_body_pose': pose, 'frame_mask': mask, 'seq_len': [40, 10]}, sample_num=1)


@pytest.mark.gpu
def test_c_entries_reject_short_tracks_and_unordered_rows():
    """the library's own checks, called directly: GLAMR_EINVAL (-1) for a track of <= 10 frames and for rows out of class order"""
    model = _model(True)
    lib = model.mfiller.net.lib
    st = torch.cuda.current_stream().cuda_stream
    i32 = lambda v: np.ascontiguousarray(v, dtype=np.int32)
    ptr = MT._np_ptr

    def infill(lens, rb):
        lens, rb = i32(lens), i32(rb)
        off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
        pose = torch.zeros(int(lens.sum()), 69, device=DEV)
        kp = torch.zeros(int(lens.sum()), dtype=torch.uint8, device=DEV)
        eps = torch.zeros(len(lens), 40, 128, device=DEV)
        ws = torch.empty(int(lib.glamr_infiller_ragged_workspace_floats(len(lens))), device=DEV)
        return lib.glamr_infiller_forward_ragged(model.mfiller.net.h, len(lens), ptr(lens), ptr(rb), off.data_ptr(), pose.data_ptr(),
                                                 kp.data_ptr(), eps.data_ptr(), 40, ws.data_ptr(), ws.numel(), st)

    def traj(lens, rb, windows):
        lens, rb = i32(lens), i32(rb)
        tlib, h = model.traj_predictor.net.lib, model.traj_predictor.net.h
        M = int(lens.sum())
        off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
        woff = torch.tensor(np.concatenate([[0], np.cumsum(-(-lens // 100))]), dtype=torch.int32, device=DEV)
        bufs = [torch.zeros(M, n, device=DEV) for n in (69, 11, 3, 3)]
        if windows:
            ws = torch.empty(int(tlib.glamr_trajpred_windows_ragged_workspace_floats(len(lens), ptr(lens), 100)), device=DEV)
            return tlib.glamr_trajpred_windows_forward_ragged(h, len(lens), 100, ptr(lens), ptr(rb), off.data_ptr(), woff.data_ptr(),
                                                              bufs[0].data_ptr(), None, *[b.data_ptr() for b in bufs[1:]],
                                                              ws.data_ptr(), ws.numel(), st)
        ws = torch.empty(int(tlib.glamr_trajpred_ragged_workspace_floats(len(lens), ptr(lens))), device=DEV)
        return tlib.glamr_trajpred_forward_ragged(h, len(lens), ptr(lens), ptr(rb), off.data_ptr(), bufs[0].data_ptr(), None, None, None,
                                                  *[b.data_ptr() for b in bufs[1:]], ws.data_ptr(), ws.numel(), st)

    assert infill([40, 41], [1, 1]) == -1             # longer track after a shorter one of the same class
    assert infill([40, 10], [1, 1]) == -1             # no infiller window
    assert infill([41, 40], [1, 1]) == 0
    assert infill([41, 40], [6, 1]) == -1             # class 1 (row_batch 6) before class 0
    assert traj([300, 40], [1, 1], False) == -1       # 300 frames are above the skinny limit, 40 are not
    assert traj([40, 300], [1, 1], False) == 0
    assert traj([300, 40], [1, 1], True) == -1        # 3 windows x 100 frames against 1 x 100
    assert traj([40, 300], [1, 1], True) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ GPU: the optimiser
class _Counting:
    """forwards to the prior and counts calls; `ragged` False hides supports_ragged_batch, so persons of different lengths go
    through one call each"""

    def __init__(self, model, ragged):
        self.model, self.calls = model, 0
        self.supports_person_batch = True
        if ragged:
            self.supports_ragged_batch = True

    def inference(self, batch, sample_num=1, row_batch=None):
        self.calls += 1
        return self.model.inference(batch, sample_num=sample_num, row_batch=row_batch)

    def draw_ragged_latents(self, seq_len, row_batch=None):
        return self.model.draw_ragged_latents(seq_len, row_batch)


def _ranged_in_dict(P, T, seed):
    """persons entering late, leaving early, with gaps"""
    from glamr_b200.synthetic import make_exist_with_gaps, make_pose_dict, make_smpl_assets
    assets = make_smpl_assets(0)
    rng = np.random.default_rng(seed)
    est = {}
    for p in range(P):
        ex = make_exist_with_gaps(T, seed=seed * 31 + p)
        a = int(rng.integers(0, T // 4)) if p else 0
        e = T - int(rng.integers(0, T // 4)) if p else T
        ex[:a] = 0
        ex[e:] = 0
        ex[a] = ex[e - 1] = 1
        est[p] = make_pose_dict(assets, p, T, seed=seed, exist=ex)
    return {'est': est, 'gt': {}, 'gt_meta': {}, 'seq_name': f'ranged_p{P}_t{T}'}


def _optimizer(cfg_name, prior):
    from glamr_b200.config import Config
    from glamr_b200.recon import GlobalReconOptimizer
    from glamr_b200.smpl import SMPL
    from glamr_b200.synthetic import make_smpl_assets
    cfg = Config(cfg_name)
    for st in cfg.opt_stage_specs.values():
        st['opt_niters'] = 6
    return GlobalReconOptimizer(cfg, torch.device(DEV), None, smpl=SMPL(make_smpl_assets(0), device=DEV), mt_model=prior)


def _assert_same(a, b, path='out'):
    if isinstance(a, dict):
        assert list(a.keys()) == list(b.keys()), path
        for k in a:
            _assert_same(a[k], b[k], f'{path}/{k}')
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, f'{path}/{i}')
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape, path
        np.testing.assert_array_equal(a, b, err_msg=path)
    elif isinstance(a, torch.Tensor):
        assert torch.equal(a, b), path
    else:
        assert type(a) is type(b) and (a == b if not isinstance(a, float) or a == a else b != b), path


@pytest.mark.gpu
@pytest.mark.parametrize('cfg_name,P,T,seed,multi_step', [('glamr_3dpw', 3, 120, 1, False), ('glamr_static_multi', 4, 90, 2, False),
                                                          ('glamr_3dpw', 2, 301, 3, False), ('glamr_3dpw', 3, 230, 4, True)])
def test_optimize_one_ragged_prior_call(cfg_name, P, T, seed, multi_step):
    prior = _model(multi_step)
    in_dict = _ranged_in_dict(P, T, seed)
    outs, counts = [], []
    for ragged in (True, False):
        wrap = _Counting(prior, ragged)
        np.random.seed(seed)
        torch.manual_seed(seed)
        outs.append(_optimizer(cfg_name, wrap).optimize(copy.deepcopy(in_dict)))
        counts.append(wrap.calls)
    lens = set()
    for est in in_dict['est'].values():
        vis = np.flatnonzero(est['bboxes_dict']['exist'])
        lens.add(int(vis[-1] - vis[0] + 1))
    assert len(lens) > 1, 'the case must hold persons of different exist lengths'
    assert counts == [1, P]
    _assert_same(outs[0], outs[1])


@pytest.mark.gpu
@pytest.mark.parametrize('multi_step', [False, True])
def test_optimize_batch_one_prior_call(multi_step):
    """optimize_batch with the learned prior over mixed sequences (41 frames x 2 persons of one length, 23 x 1, 137 x 3 of different
    exist ranges) and two seeds: one prior call for all pairs, and every pair bit-identical to its serial optimize"""
    from glamr_b200.synthetic import make_in_dict, make_smpl_assets
    prior = _model(multi_step)
    assets = make_smpl_assets(0)
    in_dicts = [make_in_dict(assets, 2, 41, seed=5, gaps=True, seq_name='s41'), make_in_dict(assets, 1, 23, seed=6, seq_name='s23'),
                _ranged_in_dict(3, 137, 7)]
    seeds = [3, 8]
    wrap = _Counting(prior, True)
    model = _optimizer('glamr_3dpw', wrap)
    outs = model.optimize_batch(in_dicts, seeds)
    assert wrap.calls == 1
    hists = [[h.clone() for h in seq] for seq in model.batch_loss_histories]
    for i, in_dict in enumerate(in_dicts):
        for k, s in enumerate(seeds):
            np.random.seed(s)
            torch.manual_seed(s)
            ref = model.optimize(copy.deepcopy(in_dict))
            _assert_same(outs[i][k], ref, f'sequence {i} seed {s}')
            assert torch.equal(hists[i][k], model.loss_history), f'loss history of sequence {i} seed {s}'
    assert wrap.calls == 1 + len(in_dicts) * len(seeds)          # the serial runs: one call each (block, lone track, ragged)
