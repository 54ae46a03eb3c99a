"""ms per call of the trajectory predictor: single pass over the whole track against windowed prediction (multi_step_trajpred,
windows of 100 frames, every window of every sequence in one batched launch sequence), at B in {1, 4} and T in {100, 300, 600,
1100}.  Both run TrajPredVAE.inference (SMPL FK included) with the seeded stand-in weights, eagerly and as a replayed CUDA graph;
the two modes are timed alternately in rounds with CUDA events after warm-up.  The graph-replayed outputs are compared with the
eager ones (they must be equal bit for bit).

    python tools/trajpred_windows_time.py [--calls 20] [--rounds 3] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from glamr_b200.motion_traj import TrajPredVAE, _GraphCache  # noqa: E402
from glamr_b200.smpl import SMPL  # noqa: E402
from glamr_b200.synthetic import make_smpl_assets  # noqa: E402
from glamr_b200.synthetic_nets import make_prior_states  # noqa: E402

SHAPES = [(B, T) for B in (1, 4) for T in (100, 300, 600, 1100)]
KEYS = ('infer_out_local_traj_tp', 'infer_out_trans', 'infer_out_orient')


def card():
    q = {'name': torch.cuda.get_device_name(0), 'power_limit_w': None, 'sm_max_mhz': None}
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(',')
        q['power_limit_w'], q['sm_max_mhz'] = float(out[0]), float(out[1])
    except Exception as e:                        # the numbers stay usable; the card's limits are then reported missing
        q['query_error'] = str(e)
    return q


def time_calls(tp, batch, multi, calls):
    for _ in range(3):                            # warm-up (and, with graphs on, capture)
        tp.inference(batch, multi_step=multi)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        tp.inference(batch, multi_step=multi)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    dev = torch.device('cuda:0')
    tp = TrajPredVAE(make_prior_states(1234)[1], dev, SMPL(make_smpl_assets(0), device=dev), seq_len=100)
    res = {'card': card(), 'window': tp.seq_len, 'calls': a.calls, 'rounds': a.rounds, 'shapes': []}
    print(json.dumps(res['card']))
    for B, T in SHAPES:
        g = torch.Generator().manual_seed(B * 10000 + T)
        body = (torch.randn(B, T, 69, generator=g) * 0.3).to(dev)
        batch = {'in_body_pose': body, 'in_traj_latent': torch.randn(B, 128, generator=g).to(dev),
                 'in_traj_window_latent': torch.randn(tp.num_windows(T), B, 128, generator=g).to(dev)}
        row = {'B': B, 'T': T}
        for graphs in (False, True):
            tp.graphs = _GraphCache(enabled=graphs)
            ms = {'single': [], 'windows': []}
            for _ in range(a.rounds):
                for name, multi in (('single', False), ('windows', True)):
                    ms[name].append(time_calls(tp, batch, multi, a.calls))
            tag = 'graph' if graphs else 'eager'
            for name, v in ms.items():
                row[f'{name}_{tag}_ms'] = [round(x, 4) for x in v]
        same = {}
        for multi in (False, True):
            tp.graphs = _GraphCache(enabled=False)
            eager = tp.inference(batch, multi_step=multi)
            tp.graphs = _GraphCache(enabled=True)
            outs = [tp.inference(batch, multi_step=multi) for _ in range(2)]     # eager warm-up, then a replay
            same['windows' if multi else 'single'] = all(torch.equal(outs[1][k], eager[k]) for k in KEYS)
        row['graph_equals_eager'] = same
        res['shapes'].append(row)
        med = lambda k: float(np.median(row[k]))
        print(f'B {B} T {T:5d}: single {med("single_eager_ms"):8.3f} / {med("single_graph_ms"):8.3f} ms   windows '
              f'{med("windows_eager_ms"):8.3f} / {med("windows_graph_ms"):8.3f} ms   (eager / graph, median)   graph == eager: {same}')
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
