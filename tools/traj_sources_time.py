"""ms per L2-flushed optimiser iteration: the trajectory without the learned predictor (GLAMR_TRAJ_BASE: base pose composed with
the world variables, no codec, no prefix scans) against the predicted trajectory (GLAMR_TRAJ_PREDICTED), on the same problem.

Each shape runs the last stage of its shipped config (1 x 300 glamr_dynamic, 4 x 300 glamr_static_multi) twice: as shipped, and with
flag_infer_motion_traj false + flag_traj_from_cam true -- same variables, same residuals, only the trajectory source differs.
The two are timed alternately in rounds (CUDA events around each replayed iteration graph, L2 flushed before each).

    python tools/traj_sources_time.py [--steps 200] [--rounds 5] [--out result.json]
"""
import argparse
import copy
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from glamr_b200 import lib as L  # noqa: E402
from glamr_b200.config import Config  # noqa: E402
from glamr_b200.recon import GlobalReconOptimizer  # noqa: E402
from glamr_b200.smpl import SMPL  # noqa: E402
from glamr_b200.synthetic import SyntheticPrior, make_in_dict, make_smpl_assets  # noqa: E402

SHAPES = [(1, 300, 'glamr_dynamic'), (4, 300, 'glamr_static_multi')]


def card():
    q = {'name': torch.cuda.get_device_name(0), 'power_limit_w': None, 'sm_max_mhz': None}
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(',')
        q['power_limit_w'], q['sm_max_mhz'] = float(out[0]), float(out[1])
    except Exception as e:                        # the numbers stay usable; the card's limits are then reported missing
        q['query_error'] = str(e)
    return q


class Case:
    def __init__(self, P, T, cfg_id, base, smpl, assets, dev):
        cfg = Config(cfg_id)
        if base:
            cfg.grecon_model_specs.update(flag_infer_motion_traj=False, flag_traj_from_cam=True)
        self.m = m = GlobalReconOptimizer(cfg, dev, None, smpl=smpl, mt_model=SyntheticPrior(0, dev))
        assert m.traj_source == (L.TRAJ_BASE if base else L.TRAJ_PREDICTED)
        data = m.init_data(copy.deepcopy(make_in_dict(assets, P, T)))
        stage, specs = list(cfg.opt_stage_specs.items())[-1]
        m._cur_vars, m._cur_stage, m._loss_cfg = specs['opt_variables'], stage, specs['loss_cfg']
        m._set_stage(data, specs['opt_variables'], specs['loss_cfg'], stage, reset_adam=True, begin=True)
        self.lr = float(specs['opt_lr'])
        self.hist = torch.zeros((1, L.NUM_TERMS + 1), device=dev)
        for _ in range(5):
            self.step()
        torch.cuda.synchronize()

    def step(self):
        """one iteration through the library's captured graph (hist_stride 0: the row is overwritten)"""
        m = self.m
        L.check(m._lib.glamr_opt_iterate(m._opt, L.ptr(m._theta), L.ptr(m._reduce), self.lr, L.ptr(self.hist), 0, 1, 1,
                                         L.stream_ptr()), 'glamr_opt_iterate')


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None, help='also write the JSON result to this file')
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this tool times the GPU and has nothing to measure without one')
    dev = torch.device('cuda:0')
    assets = make_smpl_assets(0)
    smpl = SMPL(assets, device=dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)       # > 50 MB L2
    cases = {(P, T, src): Case(P, T, cfg_id, src == 'base', smpl, assets, dev) for P, T, cfg_id in SHAPES for src in ('predicted', 'base')}
    samples = {k: [] for k in cases}
    for _ in range(args.rounds):
        for key, c in cases.items():                                          # alternate the two sources shape by shape
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            for a, b in evs:
                flush.fill_(1)
                a.record()
                c.step()
                b.record()
            torch.cuda.synchronize()
            samples[key].append(float(np.mean([a.elapsed_time(b) for a, b in evs])))
    res = {'card': card(), 'steps_per_round': args.steps, 'rounds': args.rounds, 'l2': 'flushed before every timed iteration',
           'unit': 'ms per iteration (median over rounds of the round mean)', 'shapes': {}}
    for P, T, cfg_id in SHAPES:
        pred, base = np.median(samples[(P, T, 'predicted')]), np.median(samples[(P, T, 'base')])
        res['shapes'][f'{P}x{T}'] = {'config': cfg_id, 'predicted_ms': round(float(pred), 4), 'base_ms': round(float(base), 4),
                                     'base_over_predicted': round(float(base / pred), 4),
                                     'rounds_predicted_ms': [round(x, 4) for x in samples[(P, T, 'predicted')]],
                                     'rounds_base_ms': [round(x, 4) for x in samples[(P, T, 'base')]],
                                     'launches_per_iteration': {s: cases[(P, T, s)].m.launches_per_iteration() for s in ('predicted', 'base')}}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
