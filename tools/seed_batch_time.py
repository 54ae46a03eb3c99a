"""Seeds of one sequence optimised together (GlobalReconOptimizer.optimize_seeds) against one optimize call per seed.

glamr_3dpw (200 + 500 iterations, camera from the persons) at 1 x 300 and 2 x 300 frames with gaps, for S = 1, 2, 4 and 8 seeds.  In
every round each (shape, S) runs the S serial optimize calls and the one batched call, alternately, on the same model object (the
seeded learned prior draws each seed's latents, as run_dataset does).  Reported per seed:
  * iter_ms_per_seed: device time of one optimiser iteration (CUDA events around the stages' replayed iteration graphs, the library's
    own iter_ms) divided by the seeds that iteration advances -- 1 for a serial call, S for the batched one;
  * wall_ms_per_seed: host wall-clock of the whole call(s) (init_data with the prior, stages, copy-out) over S.
Values are medians over rounds.  The batched results are checked bit for bit against the serial ones in the first round.

    python tools/seed_batch_time.py [--rounds 3] [--seeds 1,2,4,8] [--out result.json]
"""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from glamr_b200.config import Config  # noqa: E402
from glamr_b200.motion_traj import MotionTrajJointModel  # noqa: E402
from glamr_b200.recon import GlobalReconOptimizer  # noqa: E402
from glamr_b200.smpl import SMPL  # noqa: E402
from glamr_b200.synthetic import make_in_dict, make_smpl_assets  # noqa: E402
from glamr_b200.synthetic_nets import make_prior_states  # noqa: E402
from traj_variables_time import card  # noqa: E402

SHAPES = [(1, 300), (2, 300)]


def _iter_ms(model, start):
    """mean device ms per iteration of the stages run since iter_ms[start] (weighted by their timed iterations)"""
    rows = model.iter_ms[start:]
    return sum(ms * n for _, n, ms in rows) / max(sum(n for _, n, _ in rows), 1)


def _same(a, b):
    if isinstance(a, dict):
        return list(a) == list(b) and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=True)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b or (a != a and b != b)


def serial(model, in_dict, seeds):
    iters, outs, t0 = [], [], time.perf_counter()
    for s in seeds:
        np.random.seed(s)
        torch.manual_seed(s)
        k = len(model.iter_ms)
        outs.append(model.optimize(copy.deepcopy(in_dict)))
        iters.append(_iter_ms(model, k))
    torch.cuda.synchronize()
    return float(np.mean(iters)), (time.perf_counter() - t0) * 1e3 / len(seeds), outs


def batched(model, in_dict, seeds):
    t0 = time.perf_counter()
    k = len(model.iter_ms)
    outs = model.optimize_seeds(in_dict, seeds)
    torch.cuda.synchronize()
    return _iter_ms(model, k) / len(seeds), (time.perf_counter() - t0) * 1e3 / len(seeds), outs


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--seeds', default='1,2,4,8', help='seed counts S to time')
    ap.add_argument('--out', default=None, help='also write the JSON result to this file')
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this tool times the GPU and has nothing to measure without one')
    dev = torch.device('cuda:0')
    assets = make_smpl_assets(0)
    smpl = SMPL(assets, device=dev)
    model = GlobalReconOptimizer(Config('glamr_3dpw'), dev, None, smpl=smpl,
                                 mt_model=MotionTrajJointModel(None, dev, None, smpl=smpl, states=make_prior_states(1234)))
    counts = [int(x) for x in args.seeds.split(',')]
    inputs = {(P, T): make_in_dict(assets, P, T, seed=0, gaps=True, seq_name=f'seeds_p{P}_t{T}') for P, T in SHAPES}
    for (P, T), d in inputs.items():                      # warm-up of every shape: module loading, first graph captures
        serial(model, d, [100])
        batched(model, d, [100, 101])
    samples = {(P, T, S, arm): [] for P, T in SHAPES for S in counts for arm in ('serial', 'batched')}
    identical = {}
    for r in range(args.rounds):
        for P, T in SHAPES:
            for S in counts:
                seeds = list(range(1, S + 1))
                arms = [('serial', serial), ('batched', batched)] if r % 2 == 0 else [('batched', batched), ('serial', serial)]
                outs = {}
                for arm, fn in arms:
                    it, wall, outs[arm] = fn(model, inputs[(P, T)], seeds)
                    samples[(P, T, S, arm)].append((it, wall))
                if r == 0:
                    identical[f'{P}x{T}_S{S}'] = all(_same(a, b) for a, b in zip(outs['batched'], outs['serial']))
    res = {'card': card(), 'config': 'glamr_3dpw (200 + 500 iterations), synthetic sequence with gaps, seeded prior',
           'rounds': args.rounds, 'unit': 'ms per seed (median over rounds)', 'bit_identical_to_serial': identical, 'shapes': {}}
    for P, T in SHAPES:
        rows = {}
        for S in counts:
            med = {arm: np.median(np.array(samples[(P, T, S, arm)]), axis=0) for arm in ('serial', 'batched')}
            rows[f'S{S}'] = {'serial_iter_ms_per_seed': round(float(med['serial'][0]), 4),
                             'batched_iter_ms_per_seed': round(float(med['batched'][0]), 4),
                             'iter_speedup': round(float(med['serial'][0] / med['batched'][0]), 3),
                             'serial_wall_ms_per_seed': round(float(med['serial'][1]), 2),
                             'batched_wall_ms_per_seed': round(float(med['batched'][1]), 2),
                             'wall_speedup': round(float(med['serial'][1] / med['batched'][1]), 3)}
        res['shapes'][f'{P}x{T}'] = rows
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
