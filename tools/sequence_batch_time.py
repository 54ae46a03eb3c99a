"""Sequences optimised together (GlobalReconOptimizer.optimize_batch, one seed each) against one optimize call per sequence.

glamr_3dpw (200 + 500 iterations, camera from the persons), synthetic sequences with gaps:
  * 1 x 300 frames, K = 1, 4, 8, 16 and 32 sequences (32 x 300 is BASELINE config 5);
  * a mixed set: 60 to 900 frames, one or two persons.
In every round each set runs its serial optimize calls and the one batched call, alternately, on the same model object (the seeded
learned prior draws each sequence's latents after np.random.seed / torch.manual_seed, as run_dataset does).  Reported per sequence:
  * iter_ms_per_seq: device time of one optimiser iteration (CUDA events around the stages' replayed iteration graphs, the library's
    own iter_ms) divided by the sequences that iteration advances -- 1 for a serial call, K for the batched one;
  * wall_ms_per_seq: host wall-clock of the whole call(s) (init_data with the prior, stages, copy-out) over K.
Values are medians over rounds.  Every batched output is checked bit for bit against its serial one in the first round.

    python tools/sequence_batch_time.py [--rounds 3] [--counts 1,4,8,16,32] [--out result.json]
"""
import argparse
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
from seed_batch_time import _iter_ms, _same  # noqa: E402
from traj_variables_time import card  # noqa: E402

SEED = 1
MIXED = [(1, 60), (2, 60), (1, 150), (2, 300), (1, 450), (2, 600), (1, 900), (2, 900)]      # (persons, frames)


def serial(model, in_dicts):
    import copy
    iters, outs, t0 = [], [], time.perf_counter()
    for d in in_dicts:
        np.random.seed(SEED)
        torch.manual_seed(SEED)
        k = len(model.iter_ms)
        outs.append(model.optimize(copy.deepcopy(d)))
        iters.append(_iter_ms(model, k))
    torch.cuda.synchronize()
    return float(np.mean(iters)), (time.perf_counter() - t0) * 1e3 / len(in_dicts), outs


def batched(model, in_dicts):
    t0 = time.perf_counter()
    k = len(model.iter_ms)
    outs = [row[0] for row in model.optimize_batch(in_dicts, [SEED])]
    torch.cuda.synchronize()
    return _iter_ms(model, k) / len(in_dicts), (time.perf_counter() - t0) * 1e3 / len(in_dicts), outs


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--counts', default='1,4,8,16,32', help='sequence counts K of the 1 x 300 set')
    ap.add_argument('--no-mixed', action='store_true', help='skip the mixed set')
    ap.add_argument('--out', default=None, help='also write the JSON result to this file')
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this tool times the GPU and has nothing to measure without one')
    dev = torch.device('cuda:0')
    assets = make_smpl_assets(0)
    smpl = SMPL(assets, device=dev)
    model = GlobalReconOptimizer(Config('glamr_3dpw'), dev, None, smpl=smpl,
                                 mt_model=MotionTrajJointModel(None, dev, None, smpl=smpl, states=make_prior_states(1234)))
    sets = {f'1x300_K{K}': [make_in_dict(assets, 1, 300, seed=i, gaps=True, seq_name=f'seq{i:02d}') for i in range(K)]
            for K in (int(x) for x in args.counts.split(','))}
    if not args.no_mixed:
        sets['mixed'] = [make_in_dict(assets, P, T, seed=i, gaps=True, seq_name=f'mixed{i}') for i, (P, T) in enumerate(MIXED)]
    warm = [make_in_dict(assets, 1, 300, seed=99, gaps=True, seq_name='warm')]
    serial(model, warm)                                 # warm-up: module loading, first graph captures
    batched(model, warm * 2)
    samples = {(name, arm): [] for name in sets for arm in ('serial', 'batched')}
    identical = {}
    for r in range(args.rounds):
        for name, in_dicts in sets.items():
            arms = [('serial', serial), ('batched', batched)] if r % 2 == 0 else [('batched', batched), ('serial', serial)]
            outs = {}
            for arm, fn in arms:
                it, wall, outs[arm] = fn(model, in_dicts)
                samples[(name, arm)].append((it, wall))
            if r == 0:
                identical[name] = all(_same(a, b) for a, b in zip(outs['batched'], outs['serial']))
    res = {'card': card(), 'config': 'glamr_3dpw (200 + 500 iterations), synthetic sequences with gaps, seeded prior, one seed each',
           'mixed_set': [f'{P}x{T}' for P, T in MIXED], 'rounds': args.rounds, 'unit': 'ms per sequence (median over rounds)',
           'bit_identical_to_serial': identical, 'sets': {}}
    for name in sets:
        med = {arm: np.median(np.array(samples[(name, arm)]), axis=0) for arm in ('serial', 'batched')}
        res['sets'][name] = {'serial_iter_ms_per_seq': round(float(med['serial'][0]), 4),
                             'batched_iter_ms_per_seq': round(float(med['batched'][0]), 4),
                             'iter_speedup': round(float(med['serial'][0] / med['batched'][0]), 3),
                             'serial_wall_ms_per_seq': round(float(med['serial'][1]), 2),
                             'batched_wall_ms_per_seq': round(float(med['batched'][1]), 2),
                             'wall_speedup': round(float(med['serial'][1] / med['batched'][1]), 3)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
