"""Cases of the person2cam residuals (flag_opt_person2cam_rot / _trans: each person's person2cam is composed with a 6d rotation
and a translation residual before the camera-from-persons mean).  Shared by tests/golden/make_person2cam_golden.py (which runs the
reference on them) and tests/test_person2cam.py, so both regenerate the same inputs."""
import numpy as np

from traj_source_cases import GOLDEN, cfg_path, oracle_class  # noqa: F401  (re-exported)

# (name, config file under golden/reference_cfg, persons, frames, gaps, iterations per stage)
PERSON2CAM_CASES = [
    ('p2c_3dpw_p2_t80_gaps', 'glamr_3dpw_person2cam', 2, 80, True, 4),
    ('p2c_3dpw_rot_p3_t30_gaps', 'glamr_3dpw_person2cam_rot', 3, 30, True, 5),
    # the C5 shape (glamr_3dpw, 300 frames with gaps) with several persons
    ('p2c_3dpw_p4_t300_gaps', 'glamr_3dpw_person2cam_main', 4, 300, True, 10),
]
# combinations the reference fails on: its fixture records the error instead of a trajectory
FAILING_CASES = [
    ('p2c_3dpw_trans_reg_p2_t40_gaps', 'glamr_3dpw_person2cam_trans_reg', 2, 40, True, 2),
    ('p2c_3dpw_no_opt_traj_p2_t40_gaps', 'glamr_3dpw_person2cam_no_opt_traj', 2, 40, True, 2),
]
CASES = {c[0]: c for c in PERSON2CAM_CASES + FAILING_CASES}
# arrays a fixture leaves out to stay small (by the last component of the key), as in traj_source_cases.COMPACT; the 4 x 300 case also
# leaves out the final local-trajectory variables and the camera residuals (the tests hold it to the per-iteration residuals, the world
# pose, the camera and the person2cam residuals)
COMPACT = {'p2c_3dpw_p4_t300_gaps': ['kp_2d_pred', 'smpl_pose', 'person_transform_world', 'person2cam', 'smpl_orient_cam',
                                     'root_trans_cam', 'smpl_orient_cam_in_world', 'root_trans_cam_in_world', 'traj_local',
                                     'traj_local_xy', 'traj_local_heading', 'traj_local_dxy', 'traj_local_dheading', 'traj_local_z',
                                     'traj_local_rot', 'cam_pose_inv', 'cam_inv_rot_residual', 'cam_inv_trans_residual']}
# variables of the final state compared by the tests (next to the world pose and the camera)
FINAL_VARS = ['person2cam_res_rot', 'person2cam_res_trans', 'traj_local_xy', 'traj_local_heading', 'traj_local_dheading',
              'cam_inv_trans_residual']


def make_case_in_dict(assets, P, T, gaps, seq_name):
    """traj_source_cases.make_case_in_dict's persons (the last one of several on a strict sub-range), with gaps also a run of 5
    frames around T/2 that no person sees, so the camera is forward-filled there"""
    from glamr_b200.synthetic import make_exist_with_gaps, make_pose_dict
    est = {}
    for p in range(P):
        exist = make_exist_with_gaps(T, seed=p) if gaps else np.ones(T)
        if P > 1 and p == P - 1:
            exist[:T // 8] = 0
            exist[T - T // 10:] = 0
            exist[T // 8] = 1
            exist[T - T // 10 - 1] = 1
        if gaps:
            exist[T // 2 - 3:T // 2 + 2] = 0
        est[p] = make_pose_dict(assets, p, T, seed=0, exist=exist)
    return {'est': est, 'gt': {}, 'gt_meta': {}, 'seq_name': seq_name}


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
