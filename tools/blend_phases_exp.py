"""Where a tile of lbs_blend_tc_kernel spends its time (clock64 phase sums of its consumer warpgroups; -DGLAMR_EXPERIMENT build only).
Runs the last stage of the 1 x 300 glamr_dynamic and the 4 x 300 glamr_static_multi problems, flushes L2 before every iteration and
prints the mean cycles per tile of each phase, over all CTAs and both warpgroups, and the cycles of the busiest CTA per launch.

    python -c "from glamr_b200 import lib; lib.build_experiment()"          # cross-compiles, no GPU needed
    GLAMR_B200_SO=glamr_b200/libglamr_b200_exp.so python tools/blend_phases_exp.py      # on an H100
"""
import copy, ctypes, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from glamr_b200 import lib as L
from glamr_b200.config import Config
from glamr_b200.recon import GlobalReconOptimizer
from glamr_b200.smpl import SMPL
from glamr_b200.synthetic import make_in_dict, make_smpl_assets, SyntheticPrior
NAMES = ['wait full (operand stage)', 'wgmma issue + retire wait', 'epilogue', 'other']
CTAS, PHASES = 1024, 5
dev = torch.device('cuda:0')
a = make_smpl_assets(0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
clock_mhz = 1980.0             # H100 SXM maximum SM clock: the us figures are lower bounds if the card runs slower
for P, T, cfgid in [(1, 300, 'glamr_dynamic'), (4, 300, 'glamr_static_multi')]:
    cfg = Config(cfgid); in_dict = make_in_dict(a, P, T)
    m = GlobalReconOptimizer(cfg, dev, None, smpl=SMPL(a, device=dev), mt_model=SyntheticPrior(0, dev))
    data = m.init_data(copy.deepcopy(in_dict))
    stage, specs = list(cfg.opt_stage_specs.items())[-1]
    m._cur_vars, m._cur_stage, m._loss_cfg = specs['opt_variables'], stage, specs['loss_cfg']
    m._set_stage(data, specs['opt_variables'], specs['loss_cfg'], stage, reset_adam=True, begin=True)
    hist = torch.zeros((400, L.NUM_TERMS + 1), device=dev)
    lib = m._lib
    out = (ctypes.c_longlong * (CTAS * 2 * PHASES))()
    acc, tiles, busiest, R = np.zeros(PHASES - 1), 0, 0.0, 20
    for r in range(R + 3):
        flush.fill_(1)
        L.check(lib.glamr_opt_iterate(m._opt, L.ptr(m._theta), L.ptr(m._reduce), float(specs['opt_lr']), L.ptr(hist), L.NUM_TERMS + 1, 1, 1, L.stream_ptr()), 'iterate')
        L.check(lib.glamr_exp_blend_phases(out), 'blend phases')
        ph = np.array(out[:], dtype=np.float64).reshape(CTAS, 2, PHASES)
        if r >= 3:
            acc += ph[:, :, :PHASES - 1].sum(axis=(0, 1))
            tiles += int(ph[:, :, PHASES - 1].sum())
            busiest += ph[:, :, :PHASES - 1].sum(axis=2).max() / R
    per = acc / tiles
    print(f'P={P} T={T} {cfgid}:{stage}   cycles per tile and warpgroup ({tiles // (2 * R)} tiles per iteration), L2 flushed before every iteration')
    for k, nme in enumerate(NAMES):
        print(f'  {nme:32s} {per[k]:8.0f}')
    print(f'  {"total":32s} {per.sum():8.0f}   ({per.sum() / clock_mhz:.2f} us at {clock_mhz:.0f} MHz)')
    print(f'  busiest warpgroup per iteration  {busiest:8.0f}   ({busiest / clock_mhz:.2f} us)')
    del m
    torch.cuda.synchronize()
