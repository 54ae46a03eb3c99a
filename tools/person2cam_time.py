"""ms per L2-flushed optimiser iteration: glamr_3dpw (camera from the persons) with both person2cam residuals optimised against the
shipped glamr_3dpw, on the same problem.

Each shape (1 x 300 and 4 x 300, 300 frames with gaps as in 3DPW) runs the last stage of glamr_3dpw twice: as shipped, and with
flag_opt_person2cam_rot / _trans set and person2cam_rot / person2cam_trans in opt_variables -- same residuals, same launches.  The two
are timed alternately in rounds (CUDA events around each replayed iteration graph, L2 flushed before each).

    python tools/person2cam_time.py [--steps 200] [--rounds 5] [--out result.json]
"""
import argparse
import copy
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from glamr_b200 import lib as L  # noqa: E402
from glamr_b200.config import Config  # noqa: E402
from glamr_b200.recon import GlobalReconOptimizer  # noqa: E402
from glamr_b200.smpl import SMPL  # noqa: E402
from glamr_b200.synthetic import SyntheticPrior, make_in_dict, make_smpl_assets  # noqa: E402
from traj_variables_time import card  # noqa: E402

SHAPES = [(1, 300), (4, 300)]


class Case:
    def __init__(self, P, T, residuals, smpl, assets, dev):
        cfg = Config('glamr_3dpw')
        stage, specs = list(cfg.opt_stage_specs.items())[-1]
        if residuals:
            cfg.grecon_model_specs['flag_opt_person2cam_rot'] = cfg.grecon_model_specs['flag_opt_person2cam_trans'] = True
            specs['opt_variables'] = list(specs['opt_variables']) + ['person2cam_rot', 'person2cam_trans']
        self.m = m = GlobalReconOptimizer(cfg, dev, None, smpl=smpl, mt_model=SyntheticPrior(0, dev))
        data = m.init_data(copy.deepcopy(make_in_dict(assets, P, T, gaps=True)))
        m._cur_vars, m._cur_stage, m._loss_cfg = specs['opt_variables'], stage, specs['loss_cfg']
        m._set_stage(data, specs['opt_variables'], specs['loss_cfg'], stage, reset_adam=True, begin=True)
        assert m._pb.has_person2cam == int(residuals) and m._pb.cam_mode == L.CAM_FROM_PERSONS
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
    cases = {(P, T, v): Case(P, T, v == 'person2cam', smpl, assets, dev) for P, T in SHAPES for v in ('shipped', 'person2cam')}
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
    res = {'card': card(), 'config': 'glamr_3dpw, last stage', 'steps_per_round': args.steps, 'rounds': args.rounds,
           'l2': 'flushed before every timed iteration', 'unit': 'ms per iteration (median over rounds of the round mean)', 'shapes': {}}
    for P, T in SHAPES:
        sh, pc = np.median(samples[(P, T, 'shipped')]), np.median(samples[(P, T, 'person2cam')])
        res['shapes'][f'{P}x{T}'] = {'shipped_ms': round(float(sh), 4), 'person2cam_ms': round(float(pc), 4),
                                     'person2cam_over_shipped': round(float(pc / sh), 4),
                                     'rounds_shipped_ms': [round(x, 4) for x in samples[(P, T, 'shipped')]],
                                     'rounds_person2cam_ms': [round(x, 4) for x in samples[(P, T, 'person2cam')]],
                                     'launches_per_iteration': {s: cases[(P, T, s)].m.launches_per_iteration() for s in ('shipped', 'person2cam')}}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
