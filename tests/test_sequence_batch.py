"""Batches of sequences: every (sequence, seed) pair of several sequences that share one config optimised as one group of one problem
(GlobalReconOptimizer.optimize_batch, include/glamr_b200.h glamr_group_t).  Groups differ in frames, persons, exist ranges, frames
without persons and visibility; each is compiled from its own data, normalisers included, and reduced in the order of its own
one-group problem, so each pair's result is its serial run's bit for bit.

CPU: the layout of differing groups (disjoint blocks, each group's views its one-group layout shifted by its base), the group table
of equal seed groups against the arithmetic of equal groups, the config check, the host-compiled frame functions on three differing
groups (one longer than a 512-frame scan chunk) against three one-group problems term by term and gradient by gradient, and
run_dataset --batch_sequences with a stub optimiser.
GPU (-m gpu): optimize_batch against serial optimize calls on every camera mode, rel_transform, heading vectors + world_dxy, the
person2cam residuals and trajectories without the predictor, at mixed lengths that cross the blend, skinning, residual and scan-chunk
edges; a sequences x seeds batch; optimize_seeds; two problems of one shape on one CUDA handle; and a run_dataset
--batch_sequences sweep against the serial sweep."""
import copy
import ctypes
import os
import pickle
import subprocess

import numpy as np
import pytest
import torch

from glamr_b200 import lib as L
from glamr_b200 import problem as PB
from glamr_b200.global_recon import run_dataset as rd
from glamr_b200.recon import tensor_to_numpy

HERE = os.path.dirname(os.path.abspath(__file__))
FLAG_KEYS = ['flag_fixed_cam', 'flag_opt_cam', 'flag_opt_cam_from_person_pose', 'flag_cam_inv_trans_res_all', 'flag_opt_vis_local_rot',
             'cam_fix_frames']
# configs without the learned prior (the oracle's init_data runs at any size): camera from the persons + rel_transform, fixed camera
HOST_CFGS = ['glamr_3dpw_traj_from_cam', 'glamr_static_multi_last_pose']
# (persons, frames, gaps) of the three groups: 530 frames take two scan chunks of 512
HOST_SHAPES = [(2, 64, True), (1, 530, True), (3, 37, False)]


def _oracle_datas(cfg_name, smpl_assets, shapes=HOST_SHAPES, niters=2):
    from glamr_b200.config import Config
    from traj_source_cases import cfg_path, make_case_in_dict, oracle_class
    cfg = Config(cfg_path(cfg_name))
    for st in cfg.opt_stage_specs.values():
        st['opt_niters'] = niters
    ora = oracle_class()(cfg, smpl_assets)
    datas = [ora.init_data(make_case_in_dict(smpl_assets, P, T, gaps, f'seq{i}')) for i, (P, T, gaps) in enumerate(shapes)]
    return ora, cfg, datas


def _flags(ora):
    return {k: getattr(ora, k) for k in FLAG_KEYS}


# ------------------------------------------------------------------------------------------------ CPU: layout and tables
def test_batch_layout_blocks_are_disjoint(smpl_assets):
    ora, _, datas = _oracle_datas(HOST_CFGS[0], smpl_assets)
    flags = _flags(ora)
    ones = [PB.make_layout(d, flags) for d in datas]
    assert len({(l.T, l.Q, l.n_empty) for l in ones}) == 3                    # the groups really differ
    lay = PB.make_layout([[d] for d in datas], flags)
    assert isinstance(lay, PB.BatchLayout) and lay.G == 3
    assert lay.n_params == sum(l.n_params for l in ones)
    idx = torch.arange(lay.n_params)
    seen = []
    for g, (one, base) in enumerate(zip(ones, lay.bases)):
        assert lay.group_layout(g) == (lay.layouts[g], base) and vars(lay.layouts[g]) == vars(one)
        for k, v in lay.views(idx, group=g).items():
            assert torch.equal(v, one.views(torch.arange(one.n_params))[k] + base), k
            seen.append(v.reshape(-1))
        for q, p in enumerate(lay.group_persons(g)):
            assert lay.persons[p] == {k: o + base for k, o in one.persons[q].items()}
            for k, v in lay.views(idx, p).items():
                assert torch.equal(v, one.views(torch.arange(one.n_params), q)[k] + base), k
                seen.append(v.reshape(-1))
    seen = torch.cat(seen)
    assert seen.numel() == seen.unique().numel() == lay.n_params               # the blocks tile theta without overlap
    # one sequence in a batch is the one-dict layout; its seeds are the seed-group layout
    assert vars(PB.make_layout([[datas[0]]], flags)) == vars(ones[0])
    assert vars(PB.make_layout([[datas[0], copy.deepcopy(datas[0])]], flags)) == vars(PB.make_layout([datas[0], copy.deepcopy(datas[0])], flags))


def test_equal_groups_table_is_the_equal_group_arithmetic(smpl_assets):
    """the group table StageCompiler uploads for equal seed groups holds what the arithmetic of equal groups computes"""
    from oracle import rotations as rt
    ora, cfg, datas = _oracle_datas(HOST_CFGS[0], smpl_assets)
    flags = _flags(ora)
    seeds = [datas[0], copy.deepcopy(datas[0]), copy.deepcopy(datas[0])]
    lay = PB.make_layout(seeds, flags)
    theta = torch.zeros(lay.n_params)
    PB.bind_variables(seeds, lay, theta)
    comp = PB.StageCompiler(seeds, lay, flags, 'cpu', rt.aa_to_rot6d, aa_to_quat=rt.aa_to_quat)
    one_comp = PB.StageCompiler(datas[0], PB.make_layout(datas[0], flags), flags, 'cpu', rt.aa_to_rot6d, aa_to_quat=rt.aa_to_quat)
    Q, T, gp = comp.Q, comp.T, lay.group_params
    for stage, specs in cfg.opt_stage_specs.items():
        pb = comp.compile(theta, specs['opt_variables'], specs['loss_cfg'], stage)
        one = one_comp.compile(torch.zeros(gp), specs['opt_variables'], specs['loss_cfg'], stage)
        assert (pb.G, pb.P, pb.T, pb.group_params, pb.n_end) == (3, 3 * Q, T, gp, 3 * Q * T)
        for g, gr in enumerate(comp.table):
            assert (gr.p0, gr.Q, gr.n0, gr.c0, gr.T, gr.theta0, gr.rel0) == (g * Q, Q, g * Q * T, g * T, T, g * gp, g * Q * Q * T)
            assert (gr.off_cam_rot, gr.off_cam_trans) == (g * gp + pb.off_cam_rot, g * gp + pb.off_cam_trans)
            assert (pb.off_cam_rot, pb.off_cam_trans) == (one.off_cam_rot, one.off_cam_trans)
            for k in range(L.NUM_TERMS):
                if pb.term_enabled[k]:
                    assert gr.term_norm[k] == pb.term_norm[k] == one.term_norm[k]
                gs = np.float32(pb.term_weight[k]) / np.float32(pb.term_norm[k]) if pb.term_enabled[k] and not pb.term_monitor[k] else 0.0
                assert gr.gs[k] == gs


def test_groups_must_share_variable_kinds(smpl_assets):
    ora, _, datas = _oracle_datas(HOST_CFGS[0], smpl_assets)
    flags = _flags(ora)
    other = copy.deepcopy(datas[2])
    for d in other['person_data'].values():           # a heading-vector group next to scalar-heading groups
        d['traj_local_heading'] = torch.zeros(2)
    with pytest.raises(ValueError, match='heading'):
        PB.make_layout([[datas[0]], [other]], flags)
    with_dxy = copy.deepcopy(datas[1])                 # a group with world_dxy variables next to one without
    for d in with_dxy['person_data'].values():
        d['world_dxy'] = torch.zeros(with_dxy['seq_len'], 2)
    with pytest.raises(ValueError, match='world_dxy'):
        PB.make_layout([[datas[0]], [with_dxy]], flags)
    # seeds of one sequence keep their checks inside a batch
    shorter = copy.deepcopy(datas[0])
    del shorter['person_data'][list(shorter['person_data'])[-1]]
    with pytest.raises(ValueError):
        PB.make_layout([[datas[0], shorter], [datas[1]]], flags)


# ------------------------------------------------------------------------------------------------ CPU: host frame functions
def _harness(tmp_path_factory, name):
    so = str(tmp_path_factory.mktemp(name) / f'lib{name}.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-shared', '-fPIC', '-x', 'c++',
                           os.path.join(HERE, 'host_harness', f'{name}.cpp'), '-o', so])
    return ctypes.CDLL(so)


@pytest.fixture(scope='module')
def batch_emu(tmp_path_factory):
    """g++ build of tests/host_harness/emu_batch.cpp (same flags as the host harness)"""
    return _harness(tmp_path_factory, 'emu_batch')


class _HostBatch:
    """layout, theta and stage compiler of one data dict or a batch, driven through emu_batch.cpp"""

    def __init__(self, lib, data, flags, ora):
        from oracle import rotations as rt
        self.lib, self.data, self.flags, self.ora = lib, data, flags, ora
        self.layout = PB.make_layout(data, flags)
        self.theta = torch.zeros(self.layout.n_params)
        PB.bind_variables(data, self.layout, self.theta)
        self.comp = PB.StageCompiler(data, self.layout, flags, 'cpu', rt.aa_to_rot6d, aa_to_quat=rt.aa_to_quat)
        self.G = self.comp.G
        self.reduce = torch.zeros(self.layout.n_params + self.G * L.NUM_TERMS)

    def _buf(self, h, what):
        p, n = ctypes.POINTER(ctypes.c_float)(), ctypes.c_size_t()
        assert self.lib.glamr_batch_emu_buffer(h, what, ctypes.byref(p), ctypes.byref(n)) == 0
        return torch.from_numpy(np.ctypeslib.as_array(p, shape=(n.value,)))

    def evaluate(self, opt_variables, loss_cfg, stage):
        PB.begin_stage_variables(self.data, self.layout, self.theta, self.flags, opt_variables)
        pb = self.comp.compile(self.theta, opt_variables, loss_cfg, stage)
        h = ctypes.c_void_p()
        assert self.lib.glamr_batch_emu_create(ctypes.byref(h), ctypes.byref(pb)) == 0
        fp = lambda t: ctypes.c_void_p(t.data_ptr())
        comp = self.comp
        try:
            assert self.lib.glamr_batch_emu_forward_pose(h, fp(self.theta)) == 0
            N = comp.N
            ow, tw = self._buf(h, 0).view(N, 3), self._buf(h, 1).view(N, 3)
            jbuf = self._buf(h, 2).view(N, -1)
            pose, beta = comp.pose_all.reshape(N, 69), comp.beta_all.reshape(N, 10)
            for g in range(self.G):                       # the oracle's SMPL on each group's rows, as for a one-group problem
                r = slice(comp.n0s[g], comp.n0s[g] + comp.Qs[g] * comp.Ts[g])
                sc = None if comp.scale_all is None else comp.scale_all.reshape(-1)[r]
                joints, _ = self.ora.smpl(ow[r].clone(), pose[r], beta[r], root_trans=tw[r].clone(), root_scale=sc)
                jbuf[r] = joints.reshape(r.stop - r.start, -1)
            assert self.lib.glamr_batch_emu_backward(h, fp(self.theta), fp(self.reduce)) == 0
            cam = self._buf(h, 3).view(-1, 12).clone()
        finally:
            self.lib.glamr_batch_emu_destroy(h)
        n, lay = self.layout.n_params, self.layout
        bases = lay.bases if isinstance(lay, PB.BatchLayout) else [0]
        sizes = [l.n_params for l in lay.layouts] if isinstance(lay, PB.BatchLayout) else [n]
        grads = [self.reduce[b:b + s].clone() for b, s in zip(bases, sizes)]
        terms = [self.reduce[n + g * L.NUM_TERMS:n + (g + 1) * L.NUM_TERMS].clone() for g in range(self.G)]
        cams = [cam[r:r + T] for r, T in zip(comp.c0s, comp.Ts)]
        return grads, terms, cams


@pytest.mark.parametrize('cfg_name', HOST_CFGS)
def test_host_batch_equals_one_group_problems(cfg_name, smpl_assets, batch_emu):
    ora, cfg, datas = _oracle_datas(cfg_name, smpl_assets)
    flags = _flags(ora)
    singles = [_HostBatch(batch_emu, copy.deepcopy(d), flags, ora) for d in datas]
    both = _HostBatch(batch_emu, [[copy.deepcopy(d)] for d in datas], flags, ora)
    assert both.G == 3 and both.comp.Ts == [d['seq_len'] for d in datas]
    for g, single in enumerate(singles):                 # every group moved away from its initial state, by its own step
        delta = 1e-2 * torch.randn(single.layout.n_params, generator=torch.Generator().manual_seed(7 + g))
        single.theta += delta
        base = both.layout.bases[g]
        both.theta[base:base + single.layout.n_params] += delta
    norms_differ = False
    for stage, specs in cfg.opt_stage_specs.items():
        args = (specs['opt_variables'], specs['loss_cfg'], stage)
        gb, tb, cb = both.evaluate(*args)
        norms = [tuple(gr.term_norm) for gr in both.comp.table]
        norms_differ |= len(set(norms)) == 3
        for g, single in enumerate(singles):
            g1, t1, c1 = single.evaluate(*args)
            assert torch.equal(tb[g], t1[0]), (stage, g, tb[g], t1[0])                    # term by term
            assert torch.equal(gb[g], g1[0]), (stage, g, (gb[g] - g1[0]).abs().max())     # gradient by gradient
            assert torch.equal(cb[g], c1[0]), (stage, g)
    assert norms_differ                                   # the groups really have their own normalisers


# ------------------------------------------------------------------------------------------------ CPU: run_dataset --batch_sequences
class _BatchStub:
    def __init__(self):
        self.calls = []

    def optimize(self, in_dict):
        raise AssertionError('--batch_sequences must not call optimize')

    def optimize_seeds(self, in_dict, seeds):
        raise AssertionError('--batch_sequences must not call optimize_seeds')

    def optimize_batch(self, in_dicts, seeds):
        self.calls.append(([d['seq_name'] for d in in_dicts], list(seeds)))
        return [[{'seq_name': d['seq_name'], 'seed': s} for s in seeds] for d in in_dicts]


def _sweep(tmp_path, monkeypatch, extra, rank=0, world=1):
    pose_root = tmp_path / 'poses'
    pose_root.mkdir(exist_ok=True)
    for name in ['seqA', 'seqB', 'seqC', 'seqD', 'seqE']:
        with open(pose_root / f'{name}.pkl', 'wb') as fh:
            pickle.dump({0: {'tag': name}}, fh)
    monkeypatch.setenv('RANK', str(rank))
    monkeypatch.setenv('WORLD_SIZE', str(world))
    argv = ['--out_dir', str(tmp_path / 'out'), '--pose_root', str(pose_root), '--seeds', '1,7', '--quiet'] + extra
    stub = _BatchStub()
    done = rd.run(rd.parse(argv), make_model=lambda cfg, local: stub)
    return stub, done


def test_run_dataset_batch_sequences_calls_optimize_batch(tmp_path, monkeypatch):
    # one seed per call, two sequences at a time
    stub, done = _sweep(tmp_path, monkeypatch, ['--batch_sequences', '2'])
    assert stub.calls == [(['seqA', 'seqB'], [1]), (['seqA', 'seqB'], [7]), (['seqC', 'seqD'], [1]), (['seqC', 'seqD'], [7]),
                          (['seqE'], [1]), (['seqE'], [7])]
    assert sorted((d[0], d[1]) for d in done) == sorted((s, k) for s in ['seqA', 'seqB', 'seqC', 'seqD', 'seqE'] for k in [1, 7])
    for seq, seed, path, dt in done:
        assert path == rd.out_file_of(str(tmp_path / 'out'), seq, seed) and dt > 0.0
        assert pickle.load(open(path, 'rb')) == {'seq_name': seq, 'seed': seed}
    # --cached skips the finished pairs and batches the rest; with --batch_seeds, sequences with the same remaining seeds go together
    os.remove(rd.out_file_of(str(tmp_path / 'out'), 'seqB', 7))
    os.remove(rd.out_file_of(str(tmp_path / 'out'), 'seqC', 1))
    os.remove(rd.out_file_of(str(tmp_path / 'out'), 'seqC', 7))
    os.remove(rd.out_file_of(str(tmp_path / 'out'), 'seqD', 1))
    os.remove(rd.out_file_of(str(tmp_path / 'out'), 'seqD', 7))
    stub, done = _sweep(tmp_path, monkeypatch, ['--batch_sequences', '3', '--batch_seeds', '--cached', '1'])
    assert stub.calls == [(['seqB'], [7]), (['seqC'], [1, 7]), (['seqD'], [1, 7])]
    assert len(done) == 10 and sum(1 for d in done if d[3] == 0.0) == 5
    stub, _ = _sweep(tmp_path, monkeypatch, ['--batch_sequences', '3', '--batch_seeds', '--cached', '1'])
    assert stub.calls == []


def test_run_dataset_batch_sequences_with_seeds_and_ranks(tmp_path, monkeypatch):
    # rank 1 of 2 takes seqB and seqD, then batches them with all seeds in one call
    stub, done = _sweep(tmp_path, monkeypatch, ['--batch_sequences', '4', '--batch_seeds'], rank=1, world=2)
    assert stub.calls == [(['seqB', 'seqD'], [1, 7])]
    assert sorted((d[0], d[1]) for d in done) == [('seqB', 1), ('seqB', 7), ('seqD', 1), ('seqD', 7)]
    assert len({d[3] for d in done}) == 1                 # the call's time split evenly over its four pairs


# ------------------------------------------------------------------------------------------------ GPU
# (id, config, [(persons, frames, gaps) per sequence], in_dict maker, seeds).  The lengths cross the 128-frame blend tiles, the
# 20-frame skinning tiles, the 4-frame residual CTAs (odd Q*T puts a group edge inside a CTA of a concatenated grid) and, at 600
# frames, the 512-frame scan chunks.
MIXED = [(1, 41, True), (2, 137, True), (3, 300, False), (1, 600, True)]
GPU_CASES = [
    ('3dpw_from_persons', 'glamr_3dpw', MIXED, 'synthetic', [3]),
    ('static_multi_fixed', 'glamr_static_multi', [(3, 41, False), (2, 137, False), (1, 300, False)], 'synthetic', [3]),
    ('dynamic_per_frame', 'glamr_dynamic', [(1, 137, False), (1, 41, False), (1, 600, False)], 'synthetic', [3]),
    ('vec_world_dxy', 'glamr_static_multi_vec_world_dxy', [(2, 41, True), (1, 137, True)], 'case', [3]),
    ('person2cam', 'glamr_3dpw_person2cam', [(2, 50, True), (3, 41, True), (1, 137, True)], 'p2c', [3]),
    ('traj_from_cam', 'glamr_3dpw_traj_from_cam', [(2, 64, True), (1, 137, True), (3, 41, False)], 'traj_source', [3]),
    ('seqs_x_seeds', 'glamr_3dpw', [(2, 41, True), (1, 137, True)], 'synthetic', [1, 7]),
]


def _gpu_in_dict(kind, P, T, gaps, name):
    if kind == 'traj_source':
        from glamr_b200.synthetic import make_smpl_assets
        from traj_source_cases import make_case_in_dict
        return make_case_in_dict(make_smpl_assets(0), P, T, gaps, name)
    from test_seed_batch import _in_dict
    return _in_dict(kind, P, T, gaps, name)


@pytest.mark.gpu
@pytest.mark.parametrize('case', GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_optimize_batch_matches_serial_runs(case):
    from test_seed_batch import _assert_same, _gpu_model, _serial
    name, cfg_name, shapes, kind, seeds = case
    model = _gpu_model(cfg_name, 6)
    in_dicts = [_gpu_in_dict(kind, P, T, gaps, f'{name}_{i}') for i, (P, T, gaps) in enumerate(shapes)]
    refs = [[_serial(model, d, s) for s in seeds] for d in in_dicts]
    outs = model.optimize_batch(in_dicts, seeds)
    assert len(outs) == len(in_dicts) and all(len(row) == len(seeds) for row in outs)
    for i, (row, ref_row) in enumerate(zip(outs, refs)):
        for k, (out, (ref, hist)) in enumerate(zip(row, ref_row)):
            _assert_same(out, ref, f'sequence {i} seed {seeds[k]}')
            assert torch.equal(model.batch_loss_histories[i][k], hist), f'loss history of sequence {i} seed {seeds[k]}'
    # the serial path still gives the same after a batched call on the same object
    again, _ = _serial(model, in_dicts[0], seeds[0])
    _assert_same(again, refs[0][0][0], 'serial after batch')


@pytest.mark.gpu
def test_optimize_seeds_still_matches_serial_runs():
    from test_seed_batch import _assert_same, _gpu_model, _in_dict, _serial
    model = _gpu_model('glamr_3dpw', 6)
    in_dict = _in_dict('synthetic', 2, 67, True, 'seeds')
    refs = [_serial(model, in_dict, s) for s in [1, 7, 3]]
    outs = model.optimize_seeds(in_dict, [1, 7, 3])
    for k, (out, (ref, hist)) in enumerate(zip(outs, refs)):
        _assert_same(out, ref, f'seed {k}')
        assert torch.equal(model.seed_loss_histories[k], hist)


@pytest.mark.gpu
def test_run_dataset_batch_sequences_matches_serial_sweep(tmp_path):
    from test_seed_batch import _assert_same
    common = ['--cfg', 'glamr_3dpw', '--synthetic', '3', '--frames', '64', '--persons', '2', '--gaps', '--seeds', '1,7', '--quiet']
    serial = rd.run(rd.parse(common + ['--out_dir', str(tmp_path / 'serial')]))
    batched = rd.run(rd.parse(common + ['--out_dir', str(tmp_path / 'batched'), '--batch_sequences', '2', '--batch_seeds']))
    assert sorted((d[0], d[1]) for d in batched) == sorted((d[0], d[1]) for d in serial)
    paths = {(d[0], d[1]): d[2] for d in batched}
    for seq, seed, p_serial, _ in serial:
        _assert_same(pickle.load(open(paths[(seq, seed)], 'rb')), pickle.load(open(p_serial, 'rb')), f'{seq} seed {seed}')


@pytest.mark.gpu
def test_equal_shape_problems_reuse_the_handle():
    """A handle whose (P, T, J, n_params) and group shapes fit the next problem is re-used, and glamr_opt_set_problem clears its
    scratch for it: the groups must still find their CTAs and slots.  init_data attaches a one-group problem, so the pairs of two
    batches of one shape are initialised first and their stages then run back to back on one handle -- for a batch of sequences and
    for the seeds of one sequence -- each pair against its serial run.  Then a group table of another shape is refused."""
    from test_seed_batch import _assert_same, _gpu_model, _serial
    model = _gpu_model('glamr_3dpw', 6)
    in_dicts = [_gpu_in_dict('synthetic', P, T, gaps, f'reuse_{i}') for i, (P, T, gaps) in enumerate([(2, 41, True), (1, 137, True)])]
    for first, second in [((in_dicts, [3]), (in_dicts, [5])), (([in_dicts[0]], [1, 7]), ([in_dicts[0]], [3, 5]))]:
        refs = [[[_serial(model, d, s) for s in seeds] for d in dicts] for dicts, seeds in (first, second)]
        batches = [model._init_groups(dicts, seeds) for dicts, seeds in (first, second)]
        handles = []
        for c, (batch, ref, (_, seeds)) in enumerate(zip(batches, refs, (first, second))):
            model._optimize_groups(batch)
            handles.append(model._opt.value)
            for i, (seq, ref_row) in enumerate(zip(batch, ref)):
                for k, (data, (r, hist)) in enumerate(zip(seq, ref_row)):
                    _assert_same(tensor_to_numpy(data), r, f'problem {c} sequence {i} seed {seeds[k]}')
                    assert torch.equal(model.batch_loss_histories[i][k], hist), f'loss history of problem {c} sequence {i} seed {seeds[k]}'
        assert handles[0] == handles[1]                  # the second problem ran on the first one's handle
    # the handle's CTAs and slots are laid out for the shapes it was created with: another shape is an argument error
    lib = L.load()
    table = (L.Group * model._pb.G).from_buffer_copy(bytes(model._comp.table))
    pb = L.Problem.from_buffer_copy(bytes(model._pb))
    for T in (table[0].T, table[0].T - 1):
        table[0].T = T
        dev = torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8).to(model.device)
        pb.groups = dev.data_ptr()
        rc = lib.glamr_opt_set_problem(model._opt, ctypes.byref(pb), 0, L.stream_ptr())
        assert rc == (0 if T == model._comp.table[0].T else -1), (T, rc)
