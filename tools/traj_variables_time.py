"""ms per L2-flushed optimiser iteration: heading_type 'vec' with world_dxy (added next to world_dheading, so the base of the frames
outside each exist range is advanced in place every iteration) against the shipped scalar heading, on the same problem.

Each shape runs the last stage of its shipped config (1 x 300 glamr_dynamic, 4 x 300 glamr_static_multi) twice: as shipped, and with
heading_type vec + world_dxy in opt_variables -- same residuals, same launches.  The two are timed alternately in rounds (CUDA
events around each replayed iteration graph, L2 flushed before each).

    python tools/traj_variables_time.py [--steps 200] [--rounds 5] [--out result.json]
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
    def __init__(self, P, T, cfg_id, variables, smpl, assets, dev):
        cfg = Config(cfg_id)
        stage, specs = list(cfg.opt_stage_specs.items())[-1]
        if variables:
            cfg.grecon_model_specs['heading_type'] = 'vec'
            specs['opt_variables'] = list(specs['opt_variables']) + ['world_dxy']
        self.m = m = GlobalReconOptimizer(cfg, dev, None, smpl=smpl, mt_model=SyntheticPrior(0, dev))
        data = m.init_data(copy.deepcopy(make_in_dict(assets, P, T)))
        m._cur_vars, m._cur_stage, m._loss_cfg = specs['opt_variables'], stage, specs['loss_cfg']
        m._set_stage(data, specs['opt_variables'], specs['loss_cfg'], stage, reset_adam=True, begin=True)
        assert m._pb.heading_vec == m._pb.has_world_dxy == m._pb.world_dxy_alias == int(variables)
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
    cases = {(P, T, v): Case(P, T, cfg_id, v == 'vec_dxy', smpl, assets, dev) for P, T, cfg_id in SHAPES for v in ('scalar', 'vec_dxy')}
    samples = {k: [] for k in cases}
    for _ in range(args.rounds):
        for key, c in cases.items():                                          # alternate the two variants shape by shape
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
        sc, vd = np.median(samples[(P, T, 'scalar')]), np.median(samples[(P, T, 'vec_dxy')])
        res['shapes'][f'{P}x{T}'] = {'config': cfg_id, 'scalar_ms': round(float(sc), 4), 'vec_dxy_ms': round(float(vd), 4),
                                     'vec_dxy_over_scalar': round(float(vd / sc), 4),
                                     'rounds_scalar_ms': [round(x, 4) for x in samples[(P, T, 'scalar')]],
                                     'rounds_vec_dxy_ms': [round(x, 4) for x in samples[(P, T, 'vec_dxy')]],
                                     'launches_per_iteration': {s: cases[(P, T, s)].m.launches_per_iteration() for s in ('scalar', 'vec_dxy')}}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
