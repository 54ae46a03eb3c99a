"""Learned-prior inference on tracks of different lengths.

    python tools/prior_ragged_time.py [--lens 300,240,150,60] [--reps 20] [--multi-step]
    python tools/prior_ragged_time.py --batch 8,32 [--tree DIR] [--frames 300]

Default: times MotionTrajJointModel.inference (synthetic weights, sample_num 1, SMPL FK included) on the tracks with a device
synchronise around each call, one call per track against one ragged call, alternated; prints the median ms per call of each.

--batch: GlobalReconOptimizer.optimize_batch, glamr_3dpw with the synthetic-weight prior, K synthetic sequences of 1-3 persons with
gaps and different exist ranges, one seed, 1 iteration per stage; prints phase_seconds['init_data'] / K (ms per sequence) for each K.
--tree runs the glamr_b200 package of another source tree (a parent commit), so two trees can be alternated call by call.
Both modes print the GPU name and its power limit (read-only nvidia-smi query)."""
import argparse
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

TOOLS = os.path.dirname(os.path.abspath(__file__))


def gpu_line(dev):
    try:
        lim = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(dev.index or 0)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001  the number is reported, never guessed
        lim = f'unknown ({e})'
    return f'{torch.cuda.get_device_properties(dev).name}, power limit {lim}'


def ranged_in_dict(assets, P, T, seed):
    """persons entering late, leaving early, with gaps"""
    from glamr_b200.synthetic import make_exist_with_gaps, make_pose_dict
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
    return {'est': est, 'gt': {}, 'gt_meta': {}, 'seq_name': f'ranged_{seed}'}


def batch_main(a, dev):
    from glamr_b200.config import Config
    from glamr_b200.motion_traj import MotionTrajJointModel
    from glamr_b200.recon import GlobalReconOptimizer
    from glamr_b200.smpl import SMPL
    from glamr_b200.synthetic import make_smpl_assets
    from glamr_b200.synthetic_nets import make_prior_states
    import glamr_b200
    assets = make_smpl_assets(0)
    smpl = SMPL(assets, device=dev)
    cfg = Config('glamr_3dpw')
    for st in cfg.opt_stage_specs.values():
        st['opt_niters'] = 1
    mt = MotionTrajJointModel(None, dev, None, smpl=smpl, states=make_prior_states(1234))
    model = GlobalReconOptimizer(cfg, dev, None, smpl=smpl, mt_model=mt)
    print(gpu_line(dev), '| package', os.path.dirname(glamr_b200.__file__))
    for K in [int(k) for k in a.batch.split(',')]:
        ins = [ranged_in_dict(assets, 1 + i % 3, a.frames, 100 + i) for i in range(K)]
        model.optimize_batch(ins[:2], [0])                                     # warm-up
        ms = []
        for _ in range(a.reps):
            model.optimize_batch(ins, [0])
            ms.append(model.phase_seconds['init_data'] * 1e3 / K)
        print(f'K = {K}: init_data {np.median(ms):.2f} ms per sequence (min {min(ms):.2f}, max {max(ms):.2f}, {a.reps} calls)')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lens', default='300,240,150,60')
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--multi-step', action='store_true')
    ap.add_argument('--batch', default=None, help='comma list of K: time optimize_batch init_data instead')
    ap.add_argument('--frames', type=int, default=300)
    ap.add_argument('--tree', default=os.path.dirname(TOOLS), help='source tree whose glamr_b200 runs')
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.tree))
    dev = torch.device('cuda', 0)
    if a.batch:
        return batch_main(a, dev)
    from glamr_b200.motion_traj import MotionTrajJointModel
    from glamr_b200.smpl import SMPL
    from glamr_b200.synthetic import make_smpl_assets
    from glamr_b200.synthetic_nets import make_prior_states
    lens = [int(x) for x in a.lens.split(',')]
    cfg = types.SimpleNamespace(multi_step_mfiller=True, multi_step_trajpred=a.multi_step, trajpred_seq_len=100)
    m = MotionTrajJointModel(cfg, dev, None, smpl=SMPL(make_smpl_assets(0), device=dev), states=make_prior_states(1234))
    g = torch.Generator().manual_seed(0)
    pose = torch.zeros(len(lens), max(lens), 69)
    for b, T in enumerate(lens):
        pose[b, :T] = torch.randn(T, 69, generator=g) * 0.2
    pose, mask = pose.to(dev), (pose.abs().sum(-1) > 0).float().to(dev)

    def serial():
        for b, T in enumerate(lens):
            m.inference({'in_body_pose': pose[b:b + 1, :T], 'frame_mask': mask[b:b + 1, :T]})

    def ragged():
        m.inference({'in_body_pose': pose, 'frame_mask': mask, 'seq_len': lens})

    times = {'serial': [], 'ragged': []}
    for fn in (serial, ragged):
        fn()
    for _ in range(a.reps):
        for name, fn in (('serial', serial), ('ragged', ragged)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3)
    print(f'{gpu_line(dev)}; tracks {lens}; multi_step_trajpred {a.multi_step}; reps {a.reps}')
    for k, v in times.items():
        print(f'{k}: median {np.median(v):.2f} ms per call (min {min(v):.2f}, max {max(v):.2f})')


if __name__ == '__main__':
    main()
