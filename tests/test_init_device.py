"""init_data on the device (glamr_b200/csrc/init_kernels.cu, init_math.cuh).

CPU: the per-row math compiled for the host against recon.rotmats_to_rotvec, SciPy interp1d and recon.filter_pose's
Python loop, bit for bit.  GPU: the kernels' rotation vectors against rotmats_to_rotvec, and init_data with numpy
estimates against init_data with the same estimates as CUDA tensors."""
import copy
import ctypes
import os
import subprocess
import warnings

import numpy as np
import pytest
import torch
from scipy.interpolate import interp1d

import host_harness as hh
from glamr_b200.recon import rotmats_to_rotvec

SRC = os.path.join(os.path.dirname(hh.__file__), 'init_host.cpp')
FILL_F32, FILL_F64, FILL_F32_W64 = 0, 1, 2


@pytest.fixture(scope='module')
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp('init_host') / 'libinit_host.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-shared', '-fPIC', '-x', 'c++', SRC, '-o', so])
    return ctypes.CDLL(so)


def _p(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


def _near_rotations(n, rng, noise=1e-7):
    aa = rng.standard_normal((n, 3))
    aa /= np.linalg.norm(aa, axis=1, keepdims=True)
    aa *= rng.uniform(0, np.pi, (n, 1))
    from scipy.spatial.transform import Rotation
    R = Rotation.from_rotvec(aa).as_matrix()
    return (R + noise * rng.standard_normal(R.shape)).astype(np.float32)


def _rotation_cases():
    rng = np.random.default_rng(3)
    from scipy.spatial.transform import Rotation
    parts = [_near_rotations(2000, rng)]
    ax = rng.standard_normal((200, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    for ang in (np.pi - 1e-6, np.pi - 1e-3, 5e-4, 1e-3, 9.99e-4, 1e-6, 0.0):
        parts.append(Rotation.from_rotvec(ax * ang).as_matrix().astype(np.float32))
    ties = np.array([[[0, 1, 0], [1, 0, 0], [0, 0, -1]],            # a0 == b1 at the maximum: argmax takes the first
                     [[1, 0, 0], [0, 0, -1], [0, 1, 0]],            # a0 == trace
                     [[-1, 0, 0], [0, 0, 1], [0, 1, 0]],            # b1 == c2 == 0 > a0, trace
                     np.eye(3), np.diag([1.0, -1.0, -1.0]), np.diag([-1.0, -1.0, 1.0])], np.float64)
    parts.append(ties.astype(np.float32))
    bad = np.stack([np.diag([1.0, 1.0, -1.0]), np.eye(3) * 1.5, np.ones((3, 3)), np.zeros((3, 3)),
                    Rotation.from_rotvec([0.3, 0.2, 0.1]).as_matrix() + 0.2 * rng.standard_normal((3, 3))]).astype(np.float32)
    parts.append(bad)
    return np.concatenate(parts).reshape(-1, 9), len(bad)


def test_rotvec_host_matches_numpy(host):
    mats, n_bad = _rotation_cases()
    n = mats.shape[0]
    m64 = np.ascontiguousarray(mats, np.float64)
    out = np.zeros((n, 3), np.float32)
    flags = np.zeros(n, np.uint8)
    assert host.glamr_host_init_rotvec(n, _p(m64), _p(out), _p(flags)) == 0
    assert flags[-n_bad:].all(), 'improper / far-off rows must be flagged'
    assert not flags[:-n_bad].any()
    ok = flags == 0
    ref = rotmats_to_rotvec(mats[ok]).astype(np.float32)
    diff = np.nonzero((out[ok].view(np.uint32) != ref.view(np.uint32)).any(axis=1))[0]
    assert diff.size == 0, ('rotation vectors differ', m64[ok][diff[:4]], out[ok][diff[:4]].astype(np.float64), ref[diff[:4]].astype(np.float64))


def _interp_ref(frames, y, T, x_dtype):
    f = interp1d(frames.astype(x_dtype), y, axis=0, assume_sorted=True, fill_value='extrapolate')
    return f(np.arange(T, dtype=np.float32))


@pytest.mark.parametrize('case', ['end_gap', 'one_frame_gap', 'two_samples', 'start_gap', 'many_gaps'])
@pytest.mark.parametrize('kind', [FILL_F32, FILL_F64, FILL_F32_W64])
def test_gap_fill_host_matches_scipy(host, case, kind):
    rng = np.random.default_rng(11)
    T = 40
    vis = np.ones(T, bool)
    if case == 'end_gap':
        vis[31:] = False
    elif case == 'one_frame_gap':
        vis[17] = False
    elif case == 'two_samples':
        vis[:] = False
        vis[[5, 23]] = True
    elif case == 'start_gap':
        vis[:6] = False
    else:
        vis[rng.random(T) < 0.4] = False
        vis[[3, 30]] = True
    frames = np.nonzero(vis)[0].astype(np.int32)
    C = 7
    ydt = np.float64 if kind == FILL_F64 else np.float32
    y = (rng.standard_normal((frames.size, C)) * 3).astype(ydt)
    y[0, 0] = -0.0
    out = np.zeros((T, C), ydt)
    assert host.glamr_host_init_interp(frames.size, _p(frames), T, C, kind, _p(y), _p(out)) == 0
    # the estimates interpolate at float32 sample frames; the heading interpolants at the int64 frame indices of np.where
    ref = _interp_ref(frames, y, T, np.int64 if kind == FILL_F32_W64 else np.float32)
    assert ref.dtype == (np.float64 if kind != FILL_F32 else np.float32)
    ref = ref.astype(ydt)
    assert out.tobytes() == ref.tobytes()


def _filter_ref(aa, vis, score, min_score, min_num, rowop):
    """recon.filter_pose's loop (host copies of the row-ops; float32 torch arithmetic as on the device)"""
    visible = torch.tensor(vis)
    q = torch.from_numpy(rowop(5, aa))
    qc = torch.cat([q[:-1, :1], -q[:-1, 1:]], dim=-1)
    qq = torch.from_numpy(rowop(6, q[1:].numpy(), qc.numpy()))
    jump = torch.acos((2 * qq[..., 0] ** 2 - 1).clamp(-1 + 1e-6, 1 - 1e-6))
    ind = (torch.where((jump > np.pi / 3) & visible[1:].bool())[0] + 1).tolist()
    for i in ind:
        if visible[i - 1]:
            if i + 1 < q.shape[0] and visible[i + 1] and (i + 1) not in ind:
                visible[i - 1] = 0
            else:
                visible[i] = 0
    if score is not None:
        vis_ind = torch.where(visible == 1.0)[0]
        nvalid = (torch.from_numpy(score)[vis_ind] > min_score).sum(dim=1)
        visible[vis_ind[nvalid < min_num]] = 0.0
    return visible.numpy()


@pytest.mark.parametrize('case', ['consecutive', 'last_frame', 'next_to_gap', 'both_in_ind', 'keypoints', 'random'])
def test_filter_pose_host_matches_loop(host, case):
    rng = np.random.default_rng(7)
    T = 30
    aa = (0.05 * rng.standard_normal((T, 3))).astype(np.float32)
    vis = np.ones(T, np.float32)
    flip = np.array([2.5, 0.0, 0.0], np.float32)
    score, min_score, min_num = None, 0.6, 15
    if case == 'consecutive':
        aa[10] += flip; aa[11] -= flip; aa[12] += flip
    elif case == 'last_frame':
        aa[T - 1] += flip
    elif case == 'next_to_gap':
        vis[14] = 0.0; aa[13] += flip; aa[15] += flip
    elif case == 'both_in_ind':
        aa[5] += flip; aa[6] += 2 * flip; aa[20] += flip; aa[21] += flip
    elif case == 'keypoints':
        aa[8] += flip
        score = (rng.random((T, 26)) < 0.6).astype(np.float64)
        min_num = 14
    else:
        aa[rng.random(T) < 0.3] += flip
        vis[rng.random(T) < 0.2] = 0.0
        score = rng.random((T, 26))
    ref = _filter_ref(aa, vis, score, min_score, min_num, hh.rowop_fwd)
    out = vis.copy()
    sc = None if score is None else np.ascontiguousarray(score)
    assert host.glamr_host_init_filter_pose(T, _p(np.ascontiguousarray(aa)), _p(out), _p(sc), ctypes.c_double(min_score), ctypes.c_double(min_num)) == 0
    assert np.array_equal(out, ref), (case, np.nonzero(out != ref))
    if case != 'keypoints':
        assert (ref != vis).any(), 'the case must make frames invisible'


# ------------------------------------------------------------------------------------------------ GPU
def _lib_rotvec(mats):
    from glamr_b200 import lib as L
    dev = torch.device('cuda:0')
    m = torch.from_numpy(np.ascontiguousarray(mats, np.float32)).to(dev)
    n = m.shape[0]
    out = torch.empty((n, 3), device=dev)
    flags = torch.empty(n, dtype=torch.uint8, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    L.check(L.load().glamr_init_rotvec(n, L.ptr(m), 0, L.ptr(out), L.ptr(flags), L.ptr(cnt), L.stream_ptr()), 'glamr_init_rotvec')
    return out.cpu().numpy(), flags.cpu().numpy().astype(bool), int(cnt.item())


@pytest.mark.gpu
def test_rotvec_kernel_matches_numpy():
    rng = np.random.default_rng(12)
    mats, n_bad = _rotation_cases()
    mats = np.concatenate([_near_rotations(100000, rng, noise=3e-8).reshape(-1, 9), mats])
    out, flags, cnt = _lib_rotvec(mats)
    assert flags[-n_bad:].all() and not flags[:-n_bad].any() and cnt == n_bad
    ref = rotmats_to_rotvec(mats[:-n_bad]).astype(np.float32)
    diff = np.nonzero((out[:-n_bad].view(np.uint32) != ref.view(np.uint32)).any(axis=1))[0]
    assert diff.size == 0, ('rotation vectors differ', diff.size, mats[diff[:4]].astype(np.float64),
                            out[diff[:4]].astype(np.float64), ref[diff[:4]].astype(np.float64))


def _to_cuda(x):
    if isinstance(x, np.ndarray):
        return torch.from_numpy(x.copy()).cuda()
    if isinstance(x, dict):
        return {k: _to_cuda(v) for k, v in x.items()}
    return x


def _flat(x, pre=''):
    from glamr_b200.recon import tensor_to_numpy
    out = {}
    if isinstance(x, dict):
        for k, v in x.items():
            if k in ('gt', 'gt_meta'):
                continue
            out.update(_flat(v, f'{pre}/{k}'))
    elif isinstance(x, torch.Tensor):
        out[pre] = tensor_to_numpy(x)
    elif isinstance(x, np.ndarray) or np.isscalar(x):
        out[pre] = np.asarray(x)
    return out


def _assert_same(a, b):
    fa, fb = _flat(a), _flat(b)
    assert fa.keys() == fb.keys()
    for k in fa:
        assert fa[k].dtype == fb[k].dtype and fa[k].shape == fb[k].shape, k
        assert fa[k].tobytes() == fb[k].tobytes(), k


CONFIGS = [('glamr_3dpw', {}), ('glamr_3dpw', {'flag_make_invis_with_keypoint': True, 'make_invis_keypoint_min_num': 14}),
           ('glamr_3dpw', {'flag_init_cam_all_frames': True}), ('glamr_dynamic', {'flag_traj_from_cam': True, 'traj_interp_method': 'last_pose'}),
           ('glamr_static_multi', {'flag_traj_from_cam': True, 'traj_interp_method': 'linear_interp'}),
           ('glamr_static_multi', {'flag_infer_motion_traj': False})]


def _in_dict_with_jumps(assets, P, T):
    from glamr_b200 import synthetic as syn
    in_dict = syn.make_in_dict(assets, P, T, seed=2, gaps=True)
    e = in_dict['est'][P - 1]
    vis = np.nonzero(e['bboxes_dict']['exist'])[0]
    e['bboxes_dict']['exist'][:9] = 0.0                     # first visible frame > 0
    keep = vis >= 9
    for k in ('smpl_pose_quat_wroot', 'smpl_beta', 'root_trans', 'kp_2d', 'cam_K'):
        e[k] = e[k][keep]
    flip = np.diag([1.0, -1.0, -1.0]).astype(np.float32)     # a half turn of the root: an orientation jump
    R = e['smpl_pose_quat_wroot'].reshape(-1, 24, 3, 3)
    for i in (20, 21, R.shape[0] // 2, R.shape[0] - 1):
        R[i, 0] = R[i, 0] @ flip
    e['smpl_pose_quat_wroot'] = R.reshape(-1, 54, 4)
    e0 = in_dict['est'][0]
    e0['kp_2d'][5:9] = 0.0
    return in_dict


@pytest.mark.gpu
@pytest.mark.parametrize('cfg_name,flags', CONFIGS)
def test_init_data_cuda_inputs_match_numpy(smpl_assets, cfg_name, flags):
    from glamr_b200.config import Config
    from glamr_b200.recon import GlobalReconOptimizer
    from glamr_b200.smpl import SMPL
    from glamr_b200.motion_traj import MotionTrajJointModel
    from glamr_b200.synthetic_nets import make_prior_states
    dev = torch.device('cuda:0')
    cfg = Config(cfg_name, out_dir='/tmp/glamr_test_init')
    cfg.grecon_model_specs.update(flags)
    smpl = SMPL(smpl_assets, device=dev)
    mt = MotionTrajJointModel(None, dev, None, smpl, make_prior_states())
    model = GlobalReconOptimizer(cfg, dev, None, smpl=smpl, mt_model=mt)
    in_dict = _in_dict_with_jumps(smpl_assets, 3, 120)
    outs = []
    for inp in (copy.deepcopy(in_dict), {**in_dict, 'est': _to_cuda(in_dict['est'])}):
        np.random.seed(0)
        torch.manual_seed(0)
        outs.append(model.init_data(inp))
    _assert_same(outs[0], outs[1])
    assert any(bool((d['visible'] != d['visible_orig']).any()) for d in outs[0]['person_data'].values()) == model.flag_filter_pose


@pytest.mark.gpu
def test_init_data_flagged_rotation_goes_through_scipy(smpl_assets):
    from glamr_b200 import synthetic as syn
    from glamr_b200.config import Config
    from glamr_b200.recon import GlobalReconOptimizer
    dev = torch.device('cuda:0')
    cfg = Config('glamr_static_multi', out_dir='/tmp/glamr_test_init')
    cfg.grecon_model_specs['flag_infer_motion_traj'] = False
    model = GlobalReconOptimizer(cfg, dev, None, smpl=smpl_assets)
    in_dict = syn.make_in_dict(smpl_assets, 1, 30, seed=4)
    R = in_dict['est'][0]['smpl_pose_quat_wroot'].reshape(-1, 24, 3, 3)
    R[7, 5] = R[7, 5] * 1.02 + 0.01                           # far from SO(3): the Newton steps do not converge
    data = model.init_data(copy.deepcopy(in_dict))
    ref = rotmats_to_rotvec(R).reshape(30, 24, 3).astype(np.float32)
    assert data['person_data'][0]['smpl_pose'].cpu().numpy().tobytes() == ref[:, 1:].reshape(30, 69).tobytes()


def _count_syncs(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return [str(x.message).splitlines()[0] + f' ({os.path.basename(x.filename)}:{x.lineno})' for x in w
            if 'synchroniz' in str(x.message)]


@pytest.mark.gpu
@pytest.mark.parametrize('cfg_name,P,gaps', [('glamr_dynamic', 1, False), ('glamr_3dpw', 4, True), ('glamr_static_multi', 4, True)])
def test_init_data_reads_back_once(smpl_assets, cfg_name, P, gaps):
    """with warm caches, init_data synchronises with the device once between its entry and _attach"""
    from glamr_b200 import synthetic as syn
    from glamr_b200.config import Config
    from glamr_b200.recon import GlobalReconOptimizer
    from glamr_b200.smpl import SMPL
    from glamr_b200.motion_traj import MotionTrajJointModel
    from glamr_b200.synthetic_nets import make_prior_states
    dev = torch.device('cuda:0')
    assert len(_count_syncs(lambda: torch.tensor(np.ones(4), device=dev))) >= 1      # the mode sees a pageable upload
    assert len(_count_syncs(lambda: torch.ones(4, device=dev).nonzero())) >= 1        # and a nonzero
    smpl = SMPL(smpl_assets, device=dev)
    model = GlobalReconOptimizer(Config(cfg_name, out_dir='/tmp/glamr_test_init'), dev, None, smpl=smpl,
                                 mt_model=MotionTrajJointModel(None, dev, None, smpl, make_prior_states()))
    in_dict = syn.make_in_dict(smpl_assets, P, 300, seed=0, gaps=gaps)
    model.init_data(copy.deepcopy(in_dict))
    attach = model._attach

    def stop(data):
        torch.cuda.set_sync_debug_mode(0)
        return attach(data)
    model._attach = stop
    d = copy.deepcopy(in_dict)
    torch.cuda.synchronize()
    syncs = _count_syncs(lambda: model.init_data(d))
    assert len(syncs) == 1, syncs


def _parent_person(est, filter_pose, make_invis_kp, min_score, min_num):
    """init_data's per-person estimate handling as the host code computed it (numpy, SciPy interp1d, the filter_pose loop
    over the row-ops): the reference the device path must equal bit for bit"""
    from glamr_b200 import geometry as G
    from glamr_b200.synthetic import SMPL_TO_BODY26FK
    dev = torch.device('cuda:0')
    visible = est['bboxes_dict']['exist'].copy()
    where = np.where(visible)[0]
    start, end = where[0], where[-1] + 1
    exist = visible == 1
    exist[start:end] = True
    n = visible.shape[0]
    vis = visible == 1
    rotmats = est['smpl_pose_quat_wroot']
    nv = rotmats.shape[0]
    aa = rotmats_to_rotvec(rotmats).reshape(nv, -1, 3).astype(np.float32)
    d = {'smpl_pose': aa[:, 1:].reshape(-1, 69), 'smpl_beta': est['smpl_beta'], 'smpl_orient_cam': aa[:, 0], 'root_trans_cam': est['root_trans']}
    j2d = est['kp_2d'][:, :24]
    j2d = np.concatenate([j2d, np.ones_like(j2d[:, :, :1])], axis=-1)
    kp = np.zeros((int(vis.sum()), 26, 3))
    kp[:, SMPL_TO_BODY26FK[:, 0]] = j2d[:, SMPL_TO_BODY26FK[:, 1]]
    d['kp_2d'], d['kp_2d_score'] = kp[:, :, :2], kp[:, :, 2]
    d['kp_2d_aligned'] = d['kp_2d'].copy()
    d['cam_K'] = est['cam_K'].astype(np.float32)
    if not np.all(visible):
        for key in ['kp_2d', 'kp_2d_score', 'kp_2d_aligned', 'cam_K']:
            full = np.zeros((n,) + d[key].shape[1:], dtype=d[key].dtype)
            full[vis] = d[key]
            d[key] = full
        vis_ind = np.where(visible)[0].astype(np.float32)
        for key in ['smpl_pose', 'smpl_beta', 'root_trans_cam', 'smpl_orient_cam']:
            d[key] = interp1d(vis_ind, d[key], axis=0, assume_sorted=True, fill_value='extrapolate')(np.arange(n, dtype=np.float32))
    visible = torch.tensor(visible, device=dev)
    if filter_pose:
        q = G.angle_axis_to_quaternion(torch.tensor(d['smpl_orient_cam'], device=dev).float())
        jump = G.quat_angle_diff(q[1:], q[:-1])
        ind = (torch.where((jump > np.pi / 3) & visible[1:].bool())[0] + 1).tolist()
        for i in ind:
            if visible[i - 1]:
                if i + 1 < q.shape[0] and visible[i + 1] and (i + 1) not in ind:
                    visible[i - 1] = 0
                else:
                    visible[i] = 0
        if make_invis_kp:
            vis_ind = torch.where(visible == 1.0)[0]
            nvalid = (torch.tensor(d['kp_2d_score'], device=dev)[vis_ind] > min_score).sum(dim=1)
            visible[vis_ind[nvalid < min_num]] = 0.0
    d['visible'] = visible.cpu().numpy()
    d['exist_frames'] = exist
    d['fr_start'], d['fr_end'] = start, end
    return d


@pytest.mark.gpu
@pytest.mark.parametrize('make_invis_kp,min_num', [(False, 15), (True, 14)])
def test_init_data_matches_host_restatement(smpl_assets, make_invis_kp, min_num):
    from glamr_b200.config import Config
    from glamr_b200.recon import GlobalReconOptimizer
    dev = torch.device('cuda:0')
    cfg = Config('glamr_static_multi', out_dir='/tmp/glamr_test_init')
    cfg.grecon_model_specs.update({'flag_infer_motion_traj': False, 'flag_make_invis_with_keypoint': make_invis_kp,
                                   'make_invis_keypoint_min_num': min_num})
    model = GlobalReconOptimizer(cfg, dev, None, smpl=smpl_assets)
    in_dict = _in_dict_with_jumps(smpl_assets, 3, 120)
    data = model.init_data(copy.deepcopy(in_dict))
    for idx, est in in_dict['est'].items():
        ref = _parent_person(est, model.flag_filter_pose, make_invis_kp, model.make_invis_keypoint_min_score, min_num)
        got = data['person_data'][idx]
        assert int(got['fr_start']) == ref['fr_start'] and int(got['fr_end']) == ref['fr_end']
        for k, v in ref.items():
            if k in ('fr_start', 'fr_end'):
                continue
            g = got[k].cpu().numpy()
            v = np.asarray(v)
            assert g.dtype == v.dtype and g.shape == v.shape and g.tobytes() == v.tobytes(), (idx, k)
    assert any((data['person_data'][i]['visible'] != data['person_data'][i]['visible_orig']).any() for i in in_dict['est'])


@pytest.mark.gpu
def test_heading_fill_rejects_a_single_filtered_sample(smpl_assets):
    """a person with two visible frames and a root jump between them keeps one: interp1d's error, not a fill from one sample"""
    from glamr_b200 import synthetic as syn
    from glamr_b200.config import Config
    from glamr_b200.recon import GlobalReconOptimizer
    dev = torch.device('cuda:0')
    cfg = Config('glamr_static_multi', out_dir='/tmp/glamr_test_init')
    cfg.grecon_model_specs.update({'flag_infer_motion_traj': False, 'flag_traj_from_cam': True, 'traj_interp_method': 'linear_interp'})
    model = GlobalReconOptimizer(cfg, dev, None, smpl=smpl_assets)
    in_dict = syn.make_in_dict(smpl_assets, 2, 30, seed=5)
    e = in_dict['est'][1]
    e['bboxes_dict']['exist'][2:] = 0.0
    for k in ('smpl_pose_quat_wroot', 'smpl_beta', 'root_trans', 'kp_2d', 'cam_K'):
        e[k] = e[k][:2].copy()
    R = e['smpl_pose_quat_wroot'].reshape(2, 24, 3, 3)
    R[1, 0] = R[1, 0] @ np.diag([1.0, -1.0, -1.0]).astype(np.float32)
    e['smpl_pose_quat_wroot'] = R.reshape(2, 54, 4)
    with pytest.raises(ValueError, match='at least 2 entries'):
        model.init_data(copy.deepcopy(in_dict))
