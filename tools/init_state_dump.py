"""Write every tensor of the init_data dict and of the optimize output for seeded synthetic inputs, so that two builds can be
compared bit for bit.

    python tools/init_state_dump.py OUT_DIR            one .npz per case under OUT_DIR
    python tools/init_state_dump.py --compare A B      report every array that differs (with float64 values)
"""
import copy, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

CASES = [(cfg, P, gaps, flags) for cfg in ('glamr_dynamic', 'glamr_static_multi', 'glamr_3dpw') for P in (1, 4) for gaps in (False, True)
         for flags in ({},)] + \
        [('glamr_3dpw', 4, True, {'flag_init_cam_all_frames': True}),
         ('glamr_dynamic', 4, True, {'flag_traj_from_cam': True, 'traj_interp_method': 'last_pose'}),
         ('glamr_static_multi', 4, True, {'flag_traj_from_cam': True, 'traj_interp_method': 'linear_interp'}),
         ('glamr_static_multi', 4, True, {'flag_infer_motion_traj': False})]


def flatten(x, pre, out):
    import torch
    if isinstance(x, dict):
        for k, v in x.items():
            if k not in ('gt', 'gt_meta', 'meta'):
                flatten(v, f'{pre}/{k}', out)
    elif isinstance(x, (list, tuple)):
        for i, v in enumerate(x):
            flatten(v, f'{pre}/{i}', out)
    elif isinstance(x, torch.Tensor):
        out[pre] = x.detach().cpu().numpy()
    elif isinstance(x, np.ndarray) or isinstance(x, (int, float, np.number)):
        out[pre] = np.asarray(x)
    return out


def dump(out_dir):
    import torch
    from glamr_b200 import synthetic as syn
    from glamr_b200.config import Config
    from glamr_b200.recon import GlobalReconOptimizer
    from glamr_b200.smpl import SMPL
    from glamr_b200.motion_traj import MotionTrajJointModel
    from glamr_b200.synthetic_nets import make_prior_states
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device('cuda:0')
    assets = syn.make_smpl_assets(0)
    smpl = SMPL(assets, device=dev)
    for k, (cfg_name, P, gaps, flags) in enumerate(CASES):
        cfg = Config(cfg_name, out_dir='/tmp/init_state_dump')
        cfg.grecon_model_specs.update(flags)
        mt = MotionTrajJointModel(None, dev, None, smpl, make_prior_states())
        model = GlobalReconOptimizer(cfg, dev, None, smpl=smpl, mt_model=mt)
        in_dict = syn.make_in_dict(assets, P, 300, seed=k, gaps=gaps)
        arrays = {}
        np.random.seed(k)
        torch.manual_seed(k)
        flatten(model.init_data(copy.deepcopy(in_dict)), 'init', arrays)
        np.random.seed(k)
        torch.manual_seed(k)
        flatten(model.optimize(copy.deepcopy(in_dict)), 'out', arrays)
        name = f'{k:02d}_{cfg_name}_p{P}_t300' + ('_gaps' if gaps else '') + ''.join(f'_{a}' for a in flags)
        np.savez(os.path.join(out_dir, name + '.npz'), **{a.replace('/', '|'): v for a, v in arrays.items()})
        print('wrote', name, len(arrays), 'arrays', flush=True)


def compare(a_dir, b_dir):
    bad = 0
    names = sorted(os.listdir(a_dir))
    assert names == sorted(os.listdir(b_dir)), 'different case lists'
    for n in names:
        A, B = np.load(os.path.join(a_dir, n)), np.load(os.path.join(b_dir, n))
        if sorted(A.files) != sorted(B.files):
            print(n, 'keys differ:', sorted(set(A.files) ^ set(B.files)))
            bad += 1
            continue
        for k in A.files:
            x, y = A[k], B[k]
            if x.dtype != y.dtype or x.shape != y.shape or x.tobytes() != y.tobytes():
                bad += 1
                if x.dtype == y.dtype and x.shape == y.shape and x.dtype.kind == 'f':
                    i = np.nonzero((x != y) & ~(np.isnan(x) & np.isnan(y)))
                    print(n, k, f'{len(i[0])} elements differ, first: {x[i][:3].astype(np.float64)} vs {y[i][:3].astype(np.float64)}')
                else:
                    print(n, k, 'differs', x.dtype, y.dtype, x.shape, y.shape)
        print(n, len(A.files), 'arrays compared')
    print('IDENTICAL' if bad == 0 else f'{bad} ARRAYS DIFFER')
    return bad


if __name__ == '__main__':
    if sys.argv[1] == '--compare':
        sys.exit(1 if compare(sys.argv[2], sys.argv[3]) else 0)
    dump(sys.argv[1])
