"""ms per MotionInfillerVAE.inference call with recon=True (the infer sweeps, then the reconstruction sweep through the posterior)
and with recon=False (the infer sweeps alone), at 1 x 300 with sample_num 3 (the workload of the reference's
motion_infiller/vis_motion_infiller.py), 4 x 300 and 64 x 120.  Seeded stand-in weights; both modes run as replayed CUDA graphs and
are timed alternately in rounds with CUDA events after warm-up.  The card's name and power limit are read in the same run.

    python tools/infiller_recon_time.py [--calls 20] [--rounds 3] [--out result.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))
from glamr_b200.motion_traj import MotionInfillerVAE, _GraphCache  # noqa: E402
from glamr_b200.synthetic_nets import make_infiller_posterior_state, make_prior_states  # noqa: E402
from trajpred_windows_time import card  # noqa: E402

SHAPES = [(1, 300, 3), (4, 300, 1), (64, 120, 1)]     # B, T, sample_num


def time_calls(mf, batch, S, recon, calls):
    for _ in range(3):                            # warm-up and capture
        mf.inference(batch, sample_num=S, recon=recon)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        mf.inference(batch, sample_num=S, recon=recon)
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
    mf = MotionInfillerVAE({**make_prior_states(1234)[0], **make_infiller_posterior_state()}, dev)
    mf.graphs = _GraphCache(enabled=True, max_entries=16)
    res = {'card': card(), 'calls': a.calls, 'rounds': a.rounds, 'shapes': []}
    print(json.dumps(res['card']))
    for B, T, S in SHAPES:
        g = torch.Generator().manual_seed(B * 10000 + T)
        pose = torch.randn(B, T, 72, generator=g) * 0.3
        mask = torch.ones(B, T)
        mask[:, T // 3:T // 3 + 40] = 0
        batch = {'pose': pose.to(dev), 'pose_mask': mask[..., None].repeat(1, 1, 72).to(dev), 'frame_mask': mask.to(dev),
                 'in_motion_latent': torch.randn(int(np.ceil((T - 10) / 30)), 128, generator=g).to(dev)}
        ms = {'recon': [], 'infer': []}
        for _ in range(a.rounds):
            for name in ('recon', 'infer'):
                ms[name].append(time_calls(mf, batch, S, name == 'recon', a.calls))
        row = {'B': B, 'T': T, 'sample_num': S, **{f'{k}_ms': [round(x, 4) for x in v] for k, v in ms.items()}}
        res['shapes'].append(row)
        med = {k: float(np.median(v)) for k, v in ms.items()}
        print(f'B {B:3d} T {T:4d} S {S}: recon=True {med["recon"]:8.3f} ms   recon=False {med["infer"]:8.3f} ms   '
              f'(median of {a.rounds} rounds of {a.calls} calls, replayed graphs)')
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
