"""The optimiser's gradients against float64 autograd, element by element, in the modes test_grad_float64.py does not reach:
trajectories without the learned predictor (GLAMR_TRAJ_BASE: world_res, traj_rot_res / traj_trans_res, last_pose forward fill,
first_frame_only terms, camera-only flag_opt_traj false, flag_init_cam_all_frames) and the person2cam residuals
(flag_opt_person2cam_rot / _trans).  The bound, the references and the state hand-over are test_grad_float64's, unchanged.

The camera of a frame no person sees is forward-filled from the last frame someone sees.  camera_scatter_to_persons
(glamr_b200/csrc/globalopt_frames.cuh) gathers dL/d(camera) of every frame filled from a source frame, scales it by that frame's
inv_num_persons and pushes it into the world pose, and the person2cam residual rows, of each person visible there.  The camera
kernels run 128 frames per CTA (camera_backward / camera_scatter) and 512 per CTA (traj_cam_forward / backward), so besides the
golden shapes the cases below have seeded tracks whose filled runs, exist ranges and source frames sit on those edges; each case
asserts that it has what it is meant to cover.

Beyond the bound, exact zeros: a person2cam residual row of a forward-filled frame or of a frame its person is invisible on, and a
root_trans_world_res row outside its person's exist range.  smpl_orient_world_res has no such rule: traj_rot_smoothness runs over
every frame of the sequence (as in the reference), and traj_rot_res over rows the steps before moved, so its rows outside the exist
range carry real gradient and are held to the bound.  A residual row of a fill source with its person visible must be non-zero.

On one H100 80GB HBM3 (700 W limit) the worst |cuda - g64| / bound over every case, variable, term and check point was 0.89
(ts_3dpw_cam_p2_t80_gaps, cam_inv_rot_residual), 0.08-0.89 per case; the seeded cases reached 0.08-0.55.  GLAMR_GRAD_REPORT=<file>
writes every case's lines.  The GPU tests of this file took 158 s there, those of test_grad_float64.py 159 s.

CPU: the host emulator passes the bound on two seeded cases and the golden first_frame_only case, and modelled bugs of these
modes, applied to its gradient, do not (each prints the factor by which it fails)."""
import copy

import numpy as np
import pytest
import torch

import person2cam_cases
import traj_source_cases
from helpers import ReplayMT, load_golden
from test_grad_float64 import (NITERS, _check_records, _references_of, check_grads, check_terms, emulator_records, gpu_run,
                               oracle_closure, oracle_for)

EDGES = (128, 512)            # kFrameThreads (camera_backward / scatter CTAs) and kScanThreads (traj_cam_forward / backward CTAs)
GOLDEN = ['ts_3dpw_cam_p2_t80_gaps', 'ts_static_multi_last_p3_t30_gaps', 'ts_cam_only_p2_t32_gaps', 'ts_static_multi_cam_p4_t300_gaps',
          'p2c_3dpw_p2_t80_gaps', 'p2c_3dpw_rot_p3_t30_gaps', 'p2c_3dpw_p4_t300_gaps']
# name -> (config under tests/golden/reference_cfg, T, [(first exist frame, exist length, [absolute [a, b) ranges invisible])])
SEEDED = {
    # frames 360-519 seen by nobody (across 384 and 512), filled from 359; person 1 exists from frame 129 for 513 frames and is
    # invisible on 200-229 where person 0 is visible
    'ts_3dpw_cam_p3_t700_fill': ('glamr_3dpw_traj_from_cam', 700, [(0, 700, [(360, 520)]), (129, 513, [(200, 230), (360, 520)]),
                                                                  (300, 400, [(360, 520)])]),
    # last_pose forward fill over occlusions across 512, 256 and 384
    'ts_static_multi_last_p3_t600_gaps': ('glamr_static_multi_last_pose', 600, [(0, 600, [(500, 530)]), (40, 500, [(240, 270)]),
                                                                                (129, 471, [(380, 390), (505, 520)])]),
    # camera rows past one 512-frame CTA; init_cam_all_frames fills 120-135 (across 128) and 505-514 (across 512)
    'ts_cam_only_p2_t520_gaps': ('glamr_dynamic_cam_only', 520, [(0, 520, [(120, 136), (505, 515)]), (60, 400, [(120, 136)])]),
    # cameras of 128-139 filled from 127 and of 512-529 from 511; person 2 is invisible on both source frames
    'p2c_3dpw_p3_t640_gaps': ('glamr_3dpw_person2cam_main', 640, [(0, 640, [(128, 140), (512, 530)]), (50, 560, [(128, 140), (512, 530)]),
                                                                  (20, 600, [(100, 140), (480, 530)])]),
}
ALL = GOLDEN + list(SEEDED)
EMU_TS, EMU_P2C, EMU_FIRST_ONLY = 'ts_3dpw_cam_p3_t700_fill', 'p2c_3dpw_p3_t640_gaps', 'ts_static_multi_last_p3_t30_gaps'
WORLD_RES = ('smpl_orient_world_res', 'root_trans_world_res')


# ------------------------------------------------------------------------------------------------ cases
def mode_case(name, assets):
    """-> (cfg, in_dict, prior factory(device)): a golden case with its recorded prior replayed, or a seeded one"""
    from glamr_b200.config import Config
    from glamr_b200.synthetic import SyntheticPrior, make_pose_dict
    if name in SEEDED:
        cfg_name, T, tracks = SEEDED[name]
        cfg = Config(traj_source_cases.cfg_path(cfg_name))
        est = {}
        for p, (s, n, hidden) in enumerate(tracks):
            vis = np.zeros(T)
            vis[s:s + n] = 1
            for a, b in hidden:
                vis[a:b] = 0
            est[p] = make_pose_dict(assets, p, T, seed=5, exist=vis)
        in_dict = {'est': est, 'gt': {}, 'gt_meta': {}, 'seq_name': name}
        make_prior = lambda dev: SyntheticPrior(seed=23, device=dev)
    else:
        cases = person2cam_cases if name.startswith('p2c_') else traj_source_cases
        gold = load_golden('globalopt_' + name)
        cfg, in_dict = cases.case_config(name), cases.case_in_dict(name, assets)
        make_prior = lambda dev: ReplayMT(gold, dev)
    for st in cfg.opt_stage_specs.values():
        st['opt_niters'] = NITERS
    return cfg, in_dict, make_prior


def _visibility(state):
    """-> (vis [P, T] bool, exist ranges [(start, length)], camera fill source of every frame) of an oracle / CUDA data dict"""
    pd = list(state['person_data'].values())
    vis = np.stack([np.asarray(d['vis_frames'], bool) for d in pd])
    exist = [(int(d['fr_start']), int(d['exist_len'])) for d in pd]
    seen = np.where(vis.any(0))[0]
    src = np.maximum.accumulate(np.where(vis.any(0), np.arange(vis.shape[1]), seen[0]))
    return vis, exist, src


def _crosses(src, e):
    """a frame at or past edge e filled from a source frame before it"""
    return bool(((src < e) & (np.arange(src.size) >= e)).any())


def _runs(mask):
    """[a, b) runs of True"""
    d = np.diff(np.concatenate([[0], mask.astype(int), [0]]))
    return list(zip(np.where(d == 1)[0], np.where(d == -1)[0]))


def assert_contents(name, state):
    """the seeded case has what its SEEDED comment says (after init, filter_pose included)"""
    vis, exist, src = _visibility(state)
    P, T = vis.shape
    n = vis.sum(0)
    hidden_while_seen = any(not vis[p, t] and n[t] > 0 for p, (s, ln) in enumerate(exist) for t in range(s, s + ln))
    if name == 'ts_3dpw_cam_p3_t700_fill':
        assert any(b - a >= 150 and a < 512 <= b - 1 and any(a < e <= b - 1 and e != 512 for e in range(128, T, 128))
                   for a, b in _runs(n == 0)), 'no unseen run of >= 150 frames across 512 and a 128-frame edge'
        assert any(s in (128, 129) for s, _ in exist) and any(ln == 513 for _, ln in exist), exist
        assert hidden_while_seen
    elif name == 'ts_static_multi_last_p3_t600_gaps':
        filled = [(a, b) for p, (s, ln) in enumerate(exist) for a, b in _runs(~vis[p, s:s + ln]) for a, b in [(a + s, b + s)]]
        assert any(a < 512 < b for a, b in filled), filled
        assert any(a < e < b for a, b in filled for e in range(128, T, 128) if e != 512), filled
    elif name == 'ts_cam_only_p2_t520_gaps':
        assert T > 512 and _crosses(src, 128) and _crosses(src, 512)
    elif name == 'p2c_3dpw_p3_t640_gaps':
        for s in (127, 511):
            assert src[s + 1] == s and n[s] > 0 and not vis.all(0)[s], f'frame {s}: not a fill source with a person invisible'
    return vis, exist, src


def assert_exact_zeros(what, r):
    """person2cam residual rows of frames their person is invisible on (forward-filled frames included) and world_res rows outside
    the exist range are exactly 0; a residual row of a fill source with its person visible is not"""
    vis, exist, src = _visibility(r['state'])
    sources = [s for s in np.unique(src) if (src == s).sum() > 1]
    for (p, name), g in zip(r['order'], r['grads']):
        label = f'{what} {name}[{p}]'
        if name.startswith('person2cam_res'):
            assert not g[~vis[p]].any(), f'{label}: rows of frames the person is invisible on are not 0'
            for s in sources:
                if vis[p, s]:
                    assert g[s].any(), f'{label}: row of fill source {s} is 0'
        elif name == 'root_trans_world_res':
            s, ln = exist[p]
            assert not g[:s].any() and not g[s + ln:].any(), f'{label}: rows outside the exist range [{s}, {s + ln}) are not 0'


# ------------------------------------------------------------------------------------------------ CPU: cases, host emulator
@pytest.mark.parametrize('name', list(SEEDED))
def test_seeded_cases_contain_their_edges(name, smpl_assets):
    cfg, in_dict, make_prior = mode_case(name, smpl_assets)
    data = oracle_for(cfg)(copy.deepcopy(cfg), smpl_assets, mt_model=make_prior('cpu')).init_data(copy.deepcopy(in_dict))
    assert_contents(name, data)


_EMU_CACHE = {}


@pytest.fixture(scope='module')
def emu(smpl_assets):
    def get(name):
        if name not in _EMU_CACHE:
            _EMU_CACHE[name] = emulator_records(name, smpl_assets, setup=mode_case)
        return _EMU_CACHE[name]
    return get


@pytest.mark.parametrize('name', [EMU_TS, EMU_P2C, EMU_FIRST_ONLY])
def test_host_emulator_gradients_within_the_bound(name, emu):
    """a second float32 implementation (host-compiled frame functions) passes the bound and the exact zeros at every stage, before
    and after the stage's Adam steps"""
    for r in emu(name):
        what = f'{name} {r["stage"]} {r["point"]}'
        check_grads(what, r['order'], r['grads'], r['ref'])
        check_terms(what, r['terms'], r['ref'])
        assert_exact_zeros(what, r)


# ------------------------------------------------------------------------------------------------ CPU: modelled bugs
def _stage_first(records, stage):
    return next(r for r in records if r['stage'] == stage and r['point'] == 'first')


def _rejection(what, r, grads):
    """assert the bound rejects `grads` in place of the emulator's gradient; print and return the worst |g - g64| / bound"""
    rep = []
    with pytest.raises(AssertionError):
        check_grads(what, r['order'], grads, r['ref'], rep)
    label, _, _, ratio = max(rep, key=lambda x: x[3])
    print(f'{what}: rejected, worst |g-g64|/bound {ratio:.3g} at {label}')
    return ratio


def _detached_camera(Oracle, frames):
    """the oracle with the camera of `frames` cut from the persons: those frames' camera-from-persons mean is computed from detached
    world poses and person2cam residuals (the camera residuals keep their gradient)"""
    from oracle import rotations as rt

    class DetachedCamera(Oracle):
        def _camera_from_persons(self, data):
            persons = {pid: {k: (v.detach() if k in ('person_transform_world', 'person2cam_res_rot', 'person2cam_res_trans') else v)
                             for k, v in d.items()} for pid, d in data['person_data'].items()}
            cut = dict(data, person_data=persons)
            super()._camera_from_persons(cut)
            super()._camera_from_persons(data)
            mask = torch.zeros(data['cam_pose_inv'].shape[0], dtype=torch.bool)
            mask[list(frames)] = True
            data['cam_pose_inv'] = torch.where(mask[:, None, None], cut['cam_pose_inv'], data['cam_pose_inv'])
            data['cam_pose'] = rt.inverse_transform(data['cam_pose_inv'])
    return DetachedCamera


def _without_camera_path(name, r, assets, frames):
    """the emulator's gradient minus what reaches the persons' variables through the camera of `frames` (float64 oracle with and
    without that path): what camera_scatter_to_persons pushes when it leaves those frames out"""
    cfg = mode_case(name, assets)[0]
    cut = oracle_closure(_detached_camera(oracle_for(cfg), frames), cfg, assets, r['state'], r['specs'], r['stage'], r['layout'],
                         r['theta'], torch.float64)[0]
    out, moved = [], 0.0
    for (p, _), g, full, part in zip(r['order'], r['grads'], r['ref']['g64'], cut):
        if p is None or full is None:
            out.append(g)
            continue
        out.append(g - (full - part))
        moved = max(moved, float(np.abs(full - part).max()))
    assert moved > 0, f'the camera of frames {sorted(frames)[:4]}... reaches no person variable'
    return out


@pytest.mark.parametrize('name', [EMU_TS, EMU_P2C])
def test_bound_rejects_a_gather_stopping_at_the_cta_edge(name, emu, smpl_assets):
    """the frames of a forward-filled run past a 128-frame edge (the source frame in the CTA before) left out of the source frame's
    gather"""
    records = emu(name)
    r = _stage_first(records, list(mode_case(name, smpl_assets)[0].opt_stage_specs)[-1])
    _, _, src = _visibility(r['state'])
    past = [t for t in range(src.size) if src[t] != t and t // 128 != src[t] // 128]
    assert past
    _rejection(f'{name} gather stops at the edge', r, _without_camera_path(name, r, smpl_assets, past))


@pytest.mark.parametrize('name', [EMU_TS, EMU_P2C])
def test_bound_rejects_inv_num_persons_counting_an_invisible_person(name, emu, smpl_assets):
    """on source frames with one person invisible, the scatter scaled by 1 / (n_vis + 1) instead of 1 / n_vis: what it pushes from
    those frames times n_vis / n_all"""
    records = emu(name)
    r = _stage_first(records, list(mode_case(name, smpl_assets)[0].opt_stage_specs)[-1])
    vis, _, src = _visibility(r['state'])
    P, n = vis.shape[0], vis.sum(0)
    frames = [t for t in range(src.size) if n[src[t]] == P - 1]
    assert frames
    scale = (P - 1) / P
    dropped = _without_camera_path(name, r, smpl_assets, frames)
    grads = [g - (1.0 - scale) * (g - d) for g, d in zip(r['grads'], dropped)]
    _rejection(f'{name} inv_num_persons counts an invisible person', r, grads)


def test_bound_rejects_the_person2cam_rotation_columns_swapped(emu):
    """the 6d rotation residual's gradient at a fill-source row with its two 3-vectors (the 6d's columns) swapped"""
    r = _stage_first(emu(EMU_P2C), 'main_opt')
    vis, _, src = _visibility(r['state'])
    s = 127
    assert src[s + 1] == s
    k = next(i for i, (p, name) in enumerate(r['order']) if name == 'person2cam_res_rot' and vis[p, s])
    grads = [g.copy() for g in r['grads']]
    grads[k][s] = np.concatenate([grads[k][s, 3:], grads[k][s, :3]])
    _rejection(f'{EMU_P2C} person2cam_res_rot[{r["order"][k][0]}] row {s} columns swapped', r, grads)


def test_bound_rejects_one_world_res_row_scaled_by_1e_4(emu):
    """the world_res row with the largest gradient, scaled by 1 + 1e-4"""
    r = _stage_first(emu(EMU_TS), 'main_opt')
    k, row = max(((i, int(np.abs(g).max(axis=1).argmax())) for i, ((_, name), g) in enumerate(zip(r['order'], r['ref']['g64']))
                  if name in WORLD_RES), key=lambda x: float(np.abs(r['ref']['g64'][x[0]][x[1]]).max()))
    grads = [g.copy() for g in r['grads']]
    grads[k][row] *= 1.0 + 1e-4
    _rejection(f'{EMU_TS} {r["order"][k][1]}[{r["order"][k][0]}] row {row} x (1 + 1e-4)', r, grads)


def test_bound_rejects_a_first_frame_only_term_spread_to_the_second_frame(emu, smpl_assets):
    """half of kp_2d's first_frame_only gradient on each person's first exist frame moved to its second frame.  The stage's other
    first_frame_only terms are no test of the bound there: at its first closure rel_transform's first-frame gradient is ~1e-4 and
    cam_traj_rot's (a camera derived from the same persons) ~0.03, both within that row's float32 noise"""
    name, term = EMU_FIRST_ONLY, 'kp_2d'
    r = _stage_first(emu(name), 'init_opt')
    assert r['specs']['loss_cfg'][term].get('first_frame_only', False)
    cfg = mode_case(name, smpl_assets)[0]
    specs = dict(r['specs'], loss_cfg={term: r['specs']['loss_cfg'][term]})
    only = oracle_closure(oracle_for(cfg), cfg, smpl_assets, r['state'], specs, r['stage'], r['layout'], r['theta'], torch.float64)[0]
    _, exist, _ = _visibility(r['state'])
    grads, moved = [g.copy() for g in r['grads']], 0
    for i, ((p, name_), g) in enumerate(zip(r['order'], only)):
        if name_ in WORLD_RES and g is not None and g[exist[p][0]].any():
            f = exist[p][0]
            grads[i][f] -= 0.5 * g[f]
            grads[i][f + 1] += 0.5 * g[f]
            moved += 1
    assert moved
    _rejection(f'{name} {term} spread to the second frame', r, grads)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize('name', ALL)
def test_gpu_gradients_within_float64_bound(name, smpl_assets):
    """every variable's gradient and every term value at the first closure of every stage and after the stage's Adam steps, and
    the exact zeros"""
    model, cfg, recs = gpu_run(name, smpl_assets, setup=mode_case)
    lay = model._layout
    del model
    torch.cuda.empty_cache()
    if name in SEEDED:
        assert_contents(name, recs[0]['state'])
    _references_of(name, cfg, smpl_assets, lay, recs, setup=mode_case)
    for r in recs:
        assert_exact_zeros(f'{name} {r["stage"]} {r["point"]}', r)
    _check_records(name, recs)
