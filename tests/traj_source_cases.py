"""Cases of the trajectory sources without the learned trajectory predictor (default / camera-derived trajectories,
fixed trajectories).  Shared by tests/golden/make_traj_source_golden.py (which runs the reference on them) and the tests,
so both regenerate the same inputs."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

# (name, config file under golden/reference_cfg, persons, frames, gaps, iterations per stage)
TRAJ_SOURCE_CASES = [
    ('ts_dynamic_cam_p1_t40_gaps', 'glamr_dynamic_traj_from_cam', 1, 40, True, 6),
    ('ts_static_multi_last_p3_t30_gaps', 'glamr_static_multi_last_pose', 3, 30, True, 5),
    ('ts_cam_only_p2_t32_gaps', 'glamr_dynamic_cam_only', 2, 32, True, 5),
    ('ts_3dpw_cam_p2_t80_gaps', 'glamr_3dpw_traj_from_cam', 2, 80, True, 4),
    # the 4 x 300 shape bench.py measures
    ('ts_static_multi_cam_p4_t300_gaps', 'glamr_static_multi_traj_from_cam', 4, 300, True, 10),
]
CASES = {c[0]: c for c in TRAJ_SOURCE_CASES}
# arrays a fixture leaves out to stay small (by the last component of the key): in the 4 x 300 case the per-joint keypoints,
# the derived transforms and the body pose (interpolated there, not held); its world poses, variables, residual histories
# and gradients are all kept
COMPACT = {'ts_static_multi_cam_p4_t300_gaps': ['kp_2d_pred', 'smpl_pose', 'person_transform_world', 'person2cam', 'smpl_orient_cam',
                                                'root_trans_cam', 'smpl_orient_cam_in_world', 'root_trans_cam_in_world']}


def cfg_path(cfg_name):
    return os.path.join(GOLDEN, 'reference_cfg', cfg_name + '.yml')


def make_case_in_dict(assets, P, T, gaps, seq_name):
    """make_in_dict's seeded persons; with several persons the last one is absent from the first T/8 and the last T/10
    frames, so its exist range is a strict sub-range of the sequence"""
    from glamr_b200.synthetic import make_exist_with_gaps, make_pose_dict
    est = {}
    for p in range(P):
        exist = make_exist_with_gaps(T, seed=p) if gaps else np.ones(T)
        if P > 1 and p == P - 1:
            exist[:T // 8] = 0
            exist[T - T // 10:] = 0
            exist[T // 8] = 1
            exist[T - T // 10 - 1] = 1
        est[p] = make_pose_dict(assets, p, T, seed=0, exist=exist)
    return {'est': est, 'gt': {}, 'gt_meta': {}, 'seq_name': seq_name}


def oracle_class():
    """The oracle (oracle/global_opt.py) with the camera-derived trajectory of the reference's init_data added: it already
    restates the default trajectory and flag_opt_traj false, and refuses flag_traj_from_cam."""
    import torch
    from oracle import rotations as rt
    from oracle import traj_codec as tc
    from oracle.global_opt import OracleGlobalRecon

    class OracleTrajSources(OracleGlobalRecon):
        def __init__(self, cfg, smpl_assets, mt_model=None, log=None):
            specs = cfg.grecon_model_specs
            flag = specs.get('flag_traj_from_cam', False)
            specs['flag_traj_from_cam'] = False              # the base class refuses the flag it does not restate
            try:
                super().__init__(cfg, smpl_assets, mt_model=mt_model, log=log)
            finally:
                specs['flag_traj_from_cam'] = flag
            self.flag_traj_from_cam = flag
            self.traj_interp_method = specs.get('traj_interp_method', 'linear_interp')

        def init_cam_pose(self, data, all_frames=False):
            """init_data calls init_cam_pose(data) once, then init_traj_heading_from_cam; the reference runs
            get_traj_from_cam in between (global_recon_model.py:235-241)"""
            super().init_cam_pose(data, all_frames)
            if not all_frames and self.flag_traj_from_cam:
                self.get_traj_from_cam(data)

        def get_traj_from_cam(self, data):
            """:325-351 world trajectory through the initial camera; orientation interpolated over invisible frames with
            separate heading ('linear_interp'), or translation / orientation (and, unless infilled, body pose) held at the
            last visible frame over the exist range ('last_pose')"""
            for d in data['person_data'].values():
                d['person_transform_world'] = torch.matmul(data['cam_pose_inv'], d['person_transform_cam'])
                trans = d['person_transform_world'][:, :3, 3]
                orient_q = rt.rotmat_to_quat(d['person_transform_world'][:, :3, :3].contiguous())
                if self.traj_interp_method == 'linear_interp':
                    orient_q = tc.interp_orient_q_sep_heading(orient_q[d['vis_frames']], d['vis_frames'])
                elif self.traj_interp_method == 'last_pose':
                    last_trans = last_q = last_pose = None
                    for fr in torch.where(d['exist_frames'])[0]:
                        if d['vis_frames'][fr]:
                            last_trans, last_q, last_pose = trans[fr], orient_q[fr], d['smpl_pose'][fr]
                        else:
                            trans[fr] = last_trans
                            orient_q[fr] = last_q
                            if not (self.flag_infer_motion_traj and self.flag_infill_motion):
                                d['smpl_pose'][fr] = last_pose
                else:
                    raise ValueError(f'unknown traj interp method: {self.traj_interp_method}!')
                d['root_trans_world'] = d['root_trans_world_base'] = trans
                d['smpl_orient_world'] = d['smpl_orient_world_base'] = rt.quat_to_aa(orient_q)

    return OracleTrajSources


def case_config(name):
    """-> glamr_b200 Config of the case with the fixture's iteration count"""
    from glamr_b200.config import Config
    _, cfg_name, _, _, _, niters = CASES[name]
    cfg = Config(cfg_path(cfg_name))
    for st in cfg.opt_stage_specs.values():
        st['opt_niters'] = niters
    return cfg


def case_in_dict(name, assets):
    _, _, P, T, gaps, _ = CASES[name]
    return make_case_in_dict(assets, P, T, gaps, name)
