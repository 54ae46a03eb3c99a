"""Seed groups: several seeds of one sequence optimised as one problem (GlobalReconOptimizer.optimize_seeds, include/glamr_b200.h
glamr_problem_t.G).  Every group's camera, term sums and gradient are reduced over the same elements in the same order as its own
one-group problem, so each seed's result is its serial run's bit for bit.

CPU: the variable layout of G groups (disjoint blocks; one group = the one-dict layout), the host-compiled frame functions on two
groups against two one-group problems (term by term, gradient by gradient), and run_dataset --batch_seeds with a stub optimiser.
GPU (-m gpu): optimize_seeds against serial optimize calls on every camera mode, heading vectors + world_dxy and the person2cam
residuals, at sizes whose S*P*T crosses the blend / skinning / residual tile edges, one seed against optimize, and a run_dataset
sweep with --batch_seeds against the serial sweep."""
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
from helpers import ReplayMT, case_setup

HERE = os.path.dirname(os.path.abspath(__file__))
FLAG_KEYS = ['flag_fixed_cam', 'flag_opt_cam', 'flag_opt_cam_from_person_pose', 'flag_cam_inv_trans_res_all', 'flag_opt_vis_local_rot',
             'cam_fix_frames']
# fixed camera + rel_transform, camera from the persons with gaps, per-frame camera
HOST_CASES = ['static_multi_p3_t30', '3dpw_p2_t80_gaps', 'dynamic_p1_t40']


def _oracle_data(name, smpl_assets):
    from oracle.global_opt import OracleGlobalRecon
    gold, cfg, in_dict = case_setup(name, smpl_assets)
    ora = OracleGlobalRecon(cfg, smpl_assets, mt_model=ReplayMT(gold))
    return ora, cfg, ora.init_data(copy.deepcopy(in_dict))


# ------------------------------------------------------------------------------------------------ CPU: layout
def _view_indices(lay):
    """every theta index that some view of the layout covers, with its multiplicity"""
    idx = torch.arange(lay.n_params, dtype=torch.float64)
    seen = []
    for g in range(lay.G):
        seen += [v.reshape(-1) for v in lay.views(idx, group=g).values()]
    for p in range(len(lay.persons)):
        seen += [v.reshape(-1) for v in lay.views(idx, p).values()]
    return torch.cat(seen).long()


@pytest.mark.parametrize('name', HOST_CASES)
def test_group_layout_blocks_are_disjoint(name, smpl_assets):
    ora, _, data = _oracle_data(name, smpl_assets)
    flags = {k: getattr(ora, k) for k in FLAG_KEYS}
    one = PB.make_layout(data, flags)
    listed = PB.make_layout([data], flags)
    assert vars(one) == vars(listed)                                       # one group: today's offsets exactly
    assert one.G == 1 and one.group_params == one.n_params
    three = PB.make_layout([data, copy.deepcopy(data), copy.deepcopy(data)], flags)
    Q, gp = len(data['person_data']), one.n_params
    assert three.G == 3 and three.Q == Q and three.group_params == gp and three.n_params == 3 * gp
    assert three.lens == one.lens * 3
    for g in range(3):
        for q in range(Q):
            assert three.persons[g * Q + q] == {k: o + g * gp for k, o in one.persons[q].items()}
        for k, v in three.views(torch.arange(three.n_params), group=g).items():
            assert torch.equal(v, one.views(torch.arange(one.n_params))[k] + g * gp), k
    for lay in (one, three):
        idx = _view_indices(lay)                        # the camera views of every group and the views of every person
        assert idx.numel() == idx.unique().numel(), 'overlapping blocks'
        assert idx.numel() == lay.n_params and int(idx.max()) == lay.n_params - 1        # the blocks tile theta


def test_groups_must_agree(smpl_assets):
    ora, _, data = _oracle_data('3dpw_p2_t80_gaps', smpl_assets)
    flags = {k: getattr(ora, k) for k in FLAG_KEYS}
    other = copy.deepcopy(data)
    del other['person_data'][list(other['person_data'])[-1]]
    with pytest.raises(ValueError):
        PB.make_layout([data, other], flags)


# ------------------------------------------------------------------------------------------------ CPU: host frame functions
@pytest.fixture(scope='module')
def group_emu(tmp_path_factory):
    """g++ build of tests/host_harness/emu_groups.cpp (same flags as the host harness)"""
    so = str(tmp_path_factory.mktemp('group_emu') / 'libglamr_group_emu.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-shared', '-fPIC', '-x', 'c++',
                           os.path.join(HERE, 'host_harness', 'emu_groups.cpp'), '-o', so])
    lib = ctypes.CDLL(so)
    return lib


class _HostProblem:
    """layout, theta and stage compiler of one data dict or a list of seed groups, driven through emu_groups.cpp"""

    def __init__(self, lib, data, flags, ora):
        from oracle import rotations as rt
        self.lib, self.data, self.flags, self.ora = lib, data, flags, ora
        self.layout = PB.make_layout(data, flags)
        self.theta = torch.zeros(self.layout.n_params)
        PB.bind_variables(data, self.layout, self.theta)
        self.comp = PB.StageCompiler(data, self.layout, flags, 'cpu', rt.aa_to_rot6d, aa_to_quat=rt.aa_to_quat)
        self.G = self.layout.G
        self.reduce = torch.zeros(self.layout.n_params + self.G * L.NUM_TERMS)

    def _buf(self, h, what):
        p, n = ctypes.POINTER(ctypes.c_float)(), ctypes.c_size_t()
        assert self.lib.glamr_group_emu_buffer(h, what, ctypes.byref(p), ctypes.byref(n)) == 0
        return torch.from_numpy(np.ctypeslib.as_array(p, shape=(n.value,)))

    def evaluate(self, opt_variables, loss_cfg, stage):
        PB.begin_stage_variables(self.data, self.layout, self.theta, self.flags, opt_variables)
        pb = self.comp.compile(self.theta, opt_variables, loss_cfg, stage)
        h = ctypes.c_void_p()
        assert self.lib.glamr_group_emu_create(ctypes.byref(h), ctypes.byref(pb)) == 0
        fp = lambda t: ctypes.c_void_p(t.data_ptr())
        try:
            assert self.lib.glamr_group_emu_forward_pose(h, fp(self.theta)) == 0
            P, T, Q = self.comp.P, self.comp.T, self.comp.Q
            ow, tw = self._buf(h, 0).view(P * T, 3), self._buf(h, 1).view(P * T, 3)
            jbuf = self._buf(h, 2).view(P * T, -1)
            for g in range(self.G):                       # the oracle's SMPL on each group's rows, as for a one-group problem
                r = slice(g * Q * T, (g + 1) * Q * T)
                sc = None if self.comp.scale_all is None else self.comp.scale_all.reshape(-1)[r]
                joints, _ = self.ora.smpl(ow[r].clone(), self.comp.pose_all.reshape(P * T, 69)[r], self.comp.beta_all.reshape(P * T, 10)[r],
                                          root_trans=tw[r].clone(), root_scale=sc)
                jbuf[r] = joints.reshape(Q * T, -1)
            assert self.lib.glamr_group_emu_backward(h, fp(self.theta), fp(self.reduce)) == 0
            cam = self._buf(h, 3).view(self.G, T, 12).clone()
        finally:
            self.lib.glamr_group_emu_destroy(h)
        gp = self.layout.group_params
        n = self.layout.n_params
        grads = [self.reduce[g * gp:(g + 1) * gp].clone() for g in range(self.G)]
        terms = [self.reduce[n + g * L.NUM_TERMS:n + (g + 1) * L.NUM_TERMS].clone() for g in range(self.G)]
        return grads, terms, cam


@pytest.mark.parametrize('name', HOST_CASES)
def test_host_two_groups_equal_two_one_group_problems(name, smpl_assets, group_emu):
    ora, cfg, data = _oracle_data(name, smpl_assets)
    flags = {k: getattr(ora, k) for k in FLAG_KEYS}
    # seed 1's state: the camera translation and every variable moved; the same move in its one-group problem and in group 1
    singles_data = [copy.deepcopy(data), copy.deepcopy(data)]
    group_data = [copy.deepcopy(data), copy.deepcopy(data)]
    dcam = torch.randn(data['cam_pose'].shape[0], 3, generator=torch.Generator().manual_seed(5)) * 1e-2
    for d in (singles_data[1], group_data[1]):
        d['cam_pose'] = d['cam_pose'].clone()
        d['cam_pose'][:, :3, 3] += dcam
    singles = [_HostProblem(group_emu, d, flags, ora) for d in singles_data]
    both = _HostProblem(group_emu, group_data, flags, ora)
    gp = both.layout.group_params
    assert gp == singles[0].layout.n_params and both.G == 2
    delta = 1e-2 * torch.randn(gp, generator=torch.Generator().manual_seed(7))
    singles[1].theta += delta
    both.theta[gp:] += delta
    for stage, specs in cfg.opt_stage_specs.items():
        args = (specs['opt_variables'], specs['loss_cfg'], stage)
        g2, t2, cam2 = both.evaluate(*args)
        for g, single in enumerate(singles):
            g1, t1, cam1 = single.evaluate(*args)
            assert torch.equal(t2[g], t1[0]), (stage, g, t2[g], t1[0])                    # term by term
            assert torch.equal(g2[g], g1[0]), (stage, g, (g2[g] - g1[0]).abs().max())     # gradient by gradient
            assert torch.equal(cam2[g], cam1[0]), (stage, g)
        assert not torch.equal(g2[0], g2[1]) and not torch.equal(t2[0], t2[1])            # the two seeds really differ


# ------------------------------------------------------------------------------------------------ CPU: run_dataset --batch_seeds
class _SeedStub:
    def __init__(self):
        self.calls = []

    def optimize(self, in_dict):
        raise AssertionError('--batch_seeds must not call optimize')

    def optimize_seeds(self, in_dict, seeds):
        self.calls.append((in_dict['seq_name'], list(seeds)))
        return [{'seq_name': in_dict['seq_name'], 'seed': s} for s in seeds]


def test_run_dataset_batch_seeds_calls_optimize_seeds(tmp_path, monkeypatch):
    pose_root = tmp_path / 'poses'
    pose_root.mkdir()
    for name in ['seqA', 'seqB']:
        with open(pose_root / f'{name}.pkl', 'wb') as fh:
            pickle.dump({0: {'tag': name}}, fh)
    out_dir = tmp_path / 'out'
    monkeypatch.setenv('RANK', '0')
    monkeypatch.setenv('WORLD_SIZE', '1')
    argv = ['--out_dir', str(out_dir), '--pose_root', str(pose_root), '--seeds', '1,7,3', '--batch_seeds', '--quiet']
    stub = _SeedStub()
    done = rd.run(rd.parse(argv), make_model=lambda cfg, local: stub)
    assert stub.calls == [('seqA', [1, 7, 3]), ('seqB', [1, 7, 3])]                # one call per sequence with the seed list
    assert sorted((d[0], d[1]) for d in done) == sorted((s, k) for s in ['seqA', 'seqB'] for k in [1, 7, 3])
    for seq, seed, path, _ in done:
        assert path == rd.out_file_of(str(out_dir), seq, seed)
        assert pickle.load(open(path, 'rb')) == {'seq_name': seq, 'seed': seed}
    # --cached 1 skips the seeds whose file exists and batches the rest
    os.remove(rd.out_file_of(str(out_dir), 'seqB', 7))
    stub = _SeedStub()
    done = rd.run(rd.parse(argv + ['--cached', '1']), make_model=lambda cfg, local: stub)
    assert stub.calls == [('seqB', [7])]
    assert len(done) == 6 and sum(1 for d in done if d[3] == 0.0) == 5
    stub = _SeedStub()
    rd.run(rd.parse(argv + ['--cached', '1']), make_model=lambda cfg, local: stub)
    assert stub.calls == []


# ------------------------------------------------------------------------------------------------ GPU
SEEDS = [1, 7, 3]
# (id, config, persons, frames, gaps, iterations per stage, in_dict maker).  S*P*T with S = 3: 402 (crosses the 128-frame blend
# tiles and the 20-frame skinning tiles, a multiple of neither nor of the 4-frame residual CTAs; P*T = 134 puts a group edge inside
# a residual CTA of the concatenated grid), 270, 192, 240, 300.
GPU_CASES = [
    ('3dpw_p2_t67_gaps', 'glamr_3dpw', 2, 67, True, 8, 'synthetic'),
    ('static_multi_p3_t30', 'glamr_static_multi', 3, 30, False, 8, 'synthetic'),
    ('dynamic_p1_t64', 'glamr_dynamic', 1, 64, False, 8, 'synthetic'),
    ('vec_dxy_p2_t40_gaps', 'glamr_static_multi_vec_world_dxy', 2, 40, True, 8, 'case'),
    ('p2c_p2_t50_gaps', 'glamr_3dpw_person2cam', 2, 50, True, 8, 'p2c'),
]


def _gpu_model(cfg_name, niters):
    from glamr_b200.config import BUILTIN_IDS, Config
    from glamr_b200.motion_traj import MotionTrajJointModel
    from glamr_b200.recon import GlobalReconOptimizer
    from glamr_b200.smpl import SMPL
    from glamr_b200.synthetic import make_smpl_assets
    from glamr_b200.synthetic_nets import make_prior_states
    from traj_source_cases import cfg_path
    cfg = Config(cfg_name if cfg_name in BUILTIN_IDS else cfg_path(cfg_name))
    for st in cfg.opt_stage_specs.values():
        st['opt_niters'] = niters
    dev = torch.device('cuda', 0)
    smpl = SMPL(make_smpl_assets(0), device=dev)
    mt = None
    if cfg.grecon_model_specs.get('flag_infer_motion_traj', False):             # the seeded prior: each seed draws its own latents
        mt = MotionTrajJointModel(None, dev, None, smpl=smpl, states=make_prior_states(1234))
    return GlobalReconOptimizer(cfg, dev, None, smpl=smpl, mt_model=mt)


def _in_dict(kind, P, T, gaps, name):
    from glamr_b200.synthetic import make_in_dict, make_smpl_assets
    assets = make_smpl_assets(0)
    if kind == 'synthetic':
        return make_in_dict(assets, P, T, seed=0, gaps=gaps, seq_name=name)
    if kind == 'p2c':
        from person2cam_cases import make_case_in_dict
        return make_case_in_dict(assets, P, T, gaps, name)
    from traj_variable_cases import make_case_in_dict
    return make_case_in_dict(assets, P, T, gaps, name)


def _assert_same(a, b, path='out'):
    """every array / value of two optimize outputs, bit for bit"""
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a.keys()) == list(b.keys()), path
        for k in a:
            _assert_same(a[k], b[k], f'{path}/{k}')
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, f'{path}/{i}')
    elif isinstance(a, np.ndarray):
        assert isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape, path
        np.testing.assert_array_equal(a, b, err_msg=path)
    else:
        assert type(a) is type(b) and (a == b if not isinstance(a, float) or a == a else b != b), path


def _serial(model, in_dict, seed):
    np.random.seed(seed)
    torch.manual_seed(seed)
    out = model.optimize(copy.deepcopy(in_dict))
    return out, model.loss_history.clone()


@pytest.mark.gpu
@pytest.mark.parametrize('case', GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_optimize_seeds_matches_serial_runs(case):
    name, cfg_name, P, T, gaps, niters, kind = case
    model = _gpu_model(cfg_name, niters)
    in_dict = _in_dict(kind, P, T, gaps, name)
    refs = [_serial(model, in_dict, s) for s in SEEDS]
    outs = model.optimize_seeds(in_dict, SEEDS)
    assert len(outs) == len(SEEDS)
    for k, (out, (ref, hist)) in enumerate(zip(outs, refs)):
        _assert_same(out, ref, f'seed {SEEDS[k]}')
        assert torch.equal(model.seed_loss_histories[k], hist), f'loss history of seed {SEEDS[k]}'
    # the seeds start from different prior draws, so the groups are not copies of one problem
    assert not np.array_equal(outs[0]['person_data'][0]['root_trans_world'], outs[1]['person_data'][0]['root_trans_world'])
    # the serial path still gives the same after a batched call on the same object
    again, hist = _serial(model, in_dict, SEEDS[1])
    _assert_same(again, refs[1][0], 'serial after batch')


@pytest.mark.gpu
def test_optimize_one_seed_equals_optimize():
    model = _gpu_model('glamr_3dpw', 10)
    in_dict = _in_dict('synthetic', 1, 41, True, 'one_seed')
    ref, hist = _serial(model, in_dict, 5)
    (out,) = model.optimize_seeds(in_dict, [5])
    _assert_same(out, ref)
    assert torch.equal(model.seed_loss_histories[0], hist)


@pytest.mark.gpu
def test_run_dataset_batch_seeds_matches_serial_sweep(tmp_path):
    common = ['--cfg', 'glamr_3dpw', '--synthetic', '2', '--frames', '64', '--persons', '2', '--gaps', '--seeds', '1,7,3', '--quiet']
    serial = rd.run(rd.parse(common + ['--out_dir', str(tmp_path / 'serial')]))
    batched = rd.run(rd.parse(common + ['--out_dir', str(tmp_path / 'batched'), '--batch_seeds']))
    assert [(d[0], d[1]) for d in batched] == [(d[0], d[1]) for d in serial]
    for (seq, seed, p_serial, _), (_, _, p_batched, _) in zip(serial, batched):
        _assert_same(pickle.load(open(p_batched, 'rb')), pickle.load(open(p_serial, 'rb')), f'{seq} seed {seed}')
