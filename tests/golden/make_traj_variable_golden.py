"""Generate the fixtures of heading_type 'vec' and world_dxy (tests/traj_variable_cases.py) by EXECUTING THE UNMODIFIED
REFERENCE through the import shims of oracle/refshim, like make_traj_source_golden.py does for the trajectory sources:

    python tests/golden/make_traj_variable_golden.py [case name]     # writes tests/golden/globalopt_tv_*.npz

Same content as make_traj_source_golden.py's fixtures (init state, learned-prior outputs, per-iteration residuals, iteration-0
gradients, final state, the float64 continuation and the one-rounding perturbation run by the oracle), plus the final world_dxy,
root_trans_world_base and heading variables.  For a case of traj_variable_cases.FAILING_CASES the fixture records the error the
reference raises (and the iteration it raised in) instead of a trajectory.
"""
import copy
import os
import sys
import traceback

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(REPO, 'tests'))

from make_golden import FINAL_GLOBAL_KEYS, FINAL_KEYS  # noqa: E402  (activates the reference tree)
from make_traj_source_golden import reference_optimizer_from_file  # noqa: E402
import torch  # noqa: E402

from glamr_b200.synthetic import make_smpl_assets  # noqa: E402
from traj_variable_cases import (COMPACT, FAILING_CASES, TRAJ_VARIABLE_CASES, FINAL_VARS, cfg_path, make_case_in_dict,  # noqa: E402
                                 oracle_class)

PERSON_KEYS = FINAL_KEYS + [k for k in FINAL_VARS if k not in FINAL_KEYS]


def _final(data, tag, out):
    for k in FINAL_GLOBAL_KEYS:
        if k in data:
            v = data[k]
            out[f'final{tag}/{k}'] = v.detach().numpy() if isinstance(v, torch.Tensor) else v
    for pid, pd in data['person_data'].items():
        for k in PERSON_KEYS:
            if k in pd and pd[k] is not None:
                v = pd[k]
                out[f'final{tag}/{pid}/{k}'] = v.detach().numpy() if isinstance(v, torch.Tensor) else v


def oracle_run(assets, cfg_file, niters, in_dict, rec, tag, float64=False, perturb=False):
    """the oracle from the reference's init state: float64 continuation, or float32 from a once-rounded init state"""
    from glamr_b200.config import Config
    from helpers import ReplayMT
    from oracle import rotations as rt
    cfg = Config(cfg_file)
    for st in cfg.opt_stage_specs.values():
        st['opt_niters'] = niters
    ora = oracle_class()(cfg, assets, mt_model=ReplayMT(rec))
    data = ora.init_data(copy.deepcopy(in_dict))
    if float64:
        data = ora.to_float64(data)
    if perturb:
        g = torch.Generator().manual_seed(12345)

        def pert(x):
            if isinstance(x, torch.Tensor) and x.dtype == torch.float32:
                return x * (1 + (torch.randint(0, 2, x.shape, generator=g).float() * 2 - 1) * 2.0 ** -23)
            if isinstance(x, dict):
                return {k: pert(v) for k, v in x.items()}
            return x
        data = pert(data)
    out = {}
    for stage, specs in cfg.opt_stage_specs.items():
        logs = []
        ora.optimize_main(data, specs['opt_variables'], specs['opt_lr'], specs['opt_niters'], specs['loss_cfg'], {'stage': stage},
                          on_iter=lambda it, last, dt: logs.append({k: float(v) for k, v in last['uw'].items()}))
        if specs.get('reinitialize_cam', False):
            data['cam_pose'][:] = data['cam_pose'][[0]]
            data['cam_pose_inv'] = rt.inverse_transform(data['cam_pose'])
        for k in logs[0]:
            out[f'loss{tag}/{stage}/{k}'] = np.asarray([l[k] for l in logs], np.float64)
    _final(data, tag, out)
    return out


def traj_variable_case(assets, name, cfg_name, P, T, gaps, niters, failing=False):
    cfg_file = cfg_path(cfg_name)
    in_dict = make_case_in_dict(assets, P, T, gaps, name)
    model, cfg = reference_optimizer_from_file(cfg_file, niters)
    rec = {}
    mt_calls = []
    if model.mt_model is not None:
        orig_inf = model.mt_model.inference

        def rec_inference(batch, sample_num=1):
            out = orig_inf(batch, sample_num=sample_num)
            mt_calls.append({k: out[k].detach().clone() for k in
                             ['infer_out_body_pose', 'infer_out_local_traj_tp', 'infer_out_orient', 'infer_out_trans']})
            return out
        model.mt_model.inference = rec_inference
    state = {'params': None}
    orig_init_opt = model.init_opt

    def rec_init_opt(data, opt_variables, opt_lr):
        opt, params = orig_init_opt(data, opt_variables, opt_lr)
        state['params'] = params
        return opt, params
    model.init_opt = rec_init_opt
    losses = {}
    progress = {'stage': None, 'iter': -1}

    def rec_logs(loss_dict, meta):
        st, it = meta['stage'], meta['cur_iter']
        progress['stage'], progress['iter'] = st, it
        for k, v in loss_dict.items():
            losses.setdefault(f'{st}/{k}', []).append(float(v))
        if it == 0:
            for i, p in enumerate(state['params']):
                rec[f'grad0/{st}/{i}'] = (p.grad.detach().clone().numpy() if p.grad is not None else np.zeros((0,), np.float32))
                rec[f'param_shape/{st}/{i}'] = np.asarray(p.shape)
    model.write_logs = rec_logs
    orig_init = model.init_data

    def rec_init(d):
        data = orig_init(d)
        for pid, pd in data['person_data'].items():
            for k in ['kp_2d_pred', 'smpl_orient_world', 'root_trans_world', 'smpl_pose', 'vis_frames', 'smpl_orient_cam',
                      'root_trans_cam', 'person2cam', 'traj_local_heading', 'traj_local_dheading']:
                if k in pd:
                    rec[f'init/{pid}/{k}'] = pd[k].detach().clone().numpy()
        rec['init/cam_pose'] = data['cam_pose'].detach().clone().numpy()
        return data
    model.init_data = rec_init
    torch.manual_seed(0)
    rec['meta'] = np.array([P, T, int(gaps), niters])
    rec['cfg_id'] = np.array(cfg_name)
    if failing:
        try:
            model.optimize(copy.deepcopy(in_dict))
        except Exception as e:                       # what the reference does on this combination is the fixture
            rec['ref_error'] = np.array(f'{type(e).__name__}: {e}')
            rec['ref_error_at'] = np.array([progress['iter'] + 1])      # iteration of the stage whose backward raised
            traceback.print_exc()
        else:
            raise SystemExit(f'{name}: the reference did not fail')
        return rec
    out = model.optimize(copy.deepcopy(in_dict))
    for i, c in enumerate(mt_calls):
        for k, v in c.items():
            rec[f'mt/{i}/{k}'] = v.numpy()
    for k, v in losses.items():
        rec[f'loss/{k}'] = np.asarray(v, np.float64)
    _final(out, '', rec)
    rec.update(oracle_run(assets, cfg_file, niters, in_dict, rec, '64', float64=True))
    rec.update(oracle_run(assets, cfg_file, niters, in_dict, rec, '_pert', perturb=True))
    drop = COMPACT.get(name, [])
    return {k: v for k, v in rec.items() if k.split('/')[-1] not in drop}


def main(only=None):
    assets = make_smpl_assets(0)
    for case, failing in [(c, False) for c in TRAJ_VARIABLE_CASES] + [(c, True) for c in FAILING_CASES]:
        if only is None or case[0] == only:
            rec = traj_variable_case(assets, *case, failing=failing)
            np.savez_compressed(os.path.join(HERE, f'globalopt_{case[0]}.npz'), **rec)
            print('wrote', case[0], len(rec), 'arrays')


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else None)
