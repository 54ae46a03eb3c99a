"""Cases of the heading-vector local trajectory (heading_type 'vec') and the world-plane offset world_dxy.  Shared by
tests/golden/make_traj_variable_golden.py (which runs the reference on them) and tests/test_traj_variables.py, so both
regenerate the same inputs.  The inputs are traj_source_cases.make_case_in_dict's: with several persons the last one exists on
a strict sub-range of the sequence, so world_dxy's in-place add has frames outside the codec's range to accumulate on."""
from traj_source_cases import GOLDEN, cfg_path, make_case_in_dict  # noqa: F401  (re-exported)

# (name, config file under golden/reference_cfg, persons, frames, gaps, iterations per stage)
TRAJ_VARIABLE_CASES = [
    ('tv_3dpw_vec_p2_t80_gaps', 'glamr_3dpw_vec', 2, 80, True, 4),
    ('tv_static_multi_vec_p3_t30_gaps', 'glamr_static_multi_vec', 3, 30, True, 5),
    ('tv_static_multi_dxy_p3_t30_gaps', 'glamr_static_multi_world_dxy', 3, 30, True, 5),
    ('tv_dynamic_cam_dxy_p1_t40_gaps', 'glamr_dynamic_traj_from_cam_world_dxy', 1, 40, True, 6),
    # the 4 x 300 shape bench.py measures
    ('tv_static_multi_vec_dxy_p4_t300_gaps', 'glamr_static_multi_vec_world_dxy', 4, 300, True, 10),
]
# world_dxy next to world_dheading on a trajectory that does not come from the predictor: the reference fails (its fixture
# records the error instead of a trajectory)
FAILING_CASES = [
    ('tv_dynamic_cam_dxy_alias_p1_t40_gaps', 'glamr_dynamic_traj_from_cam_world_dxy_alias', 1, 40, True, 3),
]
CASES = {c[0]: c for c in TRAJ_VARIABLE_CASES + FAILING_CASES}
# arrays a fixture leaves out to stay small (by the last component of the key), as in traj_source_cases.COMPACT
COMPACT = {'tv_static_multi_vec_dxy_p4_t300_gaps': ['kp_2d_pred', 'smpl_pose', 'person_transform_world', 'person2cam', 'smpl_orient_cam',
                                                    'root_trans_cam', 'smpl_orient_cam_in_world', 'root_trans_cam_in_world']}
# world variables of the final state compared by the tests (next to the world pose and the camera)
FINAL_VARS = ['world_dheading', 'world_dxy', 'smpl_orient_world_res', 'root_trans_world_res', 'traj_local_heading', 'traj_local_dheading',
              'root_trans_world_base']


def oracle_class():
    """The oracle of traj_source_cases.oracle_class with the reference's heading_type 'vec' (:191-196,403-405) and world_dxy
    (:467-468,628-631) added.  world_dxy is added IN PLACE to root_trans_world exactly like the reference, so the oracle
    reproduces its aliasing: whenever root_trans_world is the base, the add lands in the base, which pred_trajectory_base
    clones (detached) at the next forward."""
    import torch
    from oracle import rotations as rt
    from oracle import traj_codec as tc
    from traj_source_cases import oracle_class as traj_source_oracle

    Base = traj_source_oracle()

    class OracleTrajVariables(Base):
        def __init__(self, cfg, smpl_assets, mt_model=None, log=None):
            specs = cfg.grecon_model_specs
            heading_type = specs.get('heading_type', 'scalar')
            specs['heading_type'] = 'scalar'                 # the base class refuses the type it does not restate
            try:
                super().__init__(cfg, smpl_assets, mt_model=mt_model, log=log)
            finally:
                specs['heading_type'] = heading_type
            self.heading_type = heading_type

        def init_data(self, in_dict):
            data = super().init_data(in_dict)
            if self.heading_type == 'vec' and self.flag_opt_traj and self.flag_pred_traj:
                # :191-193 creates the heading variables as vectors; all are zeros, so init's forward saw the same trajectory
                for d in data['person_data'].values():
                    Ln = int(d['exist_len'].sum())
                    d['traj_local_heading'] = torch.zeros(2)
                    d['traj_local_dheading'] = torch.zeros(Ln - 1, 2)
            return data

        def pred_trajectory_base(self, d):
            if self.heading_type != 'vec':
                return super().pred_trajectory_base(d)
            h, dh = d['traj_local_heading'], d['traj_local_dheading']
            if h.shape != (2,):                              # init's forward runs before init_data has made them vectors (zeros)
                h, dh = torch.zeros(2, dtype=h.dtype), torch.zeros(dh.shape[0], 2, dtype=dh.dtype)
            tl = d['traj_local_pred'].detach().clone()
            xy = torch.cat([(tl[0, :2] + d['traj_local_xy'])[None], tl[1:, :2] + d['traj_local_dxy']], dim=0)
            mask = torch.ones_like(tl[1:, 0])
            for (s, e) in self.cam_fix_frames:
                mask[s:e] = 0.0
            hvec = torch.cat([(tl[0, -2:] + h)[None], tl[1:, -2:] + dh * mask.unsqueeze(1)], dim=0)
            z = tl[:, 2] + d['traj_local_z']
            if self.flag_opt_vis_local_rot:
                d6 = tl[:, 3:-2] + d['traj_local_rot'] * d['vis_frames'].to(tl.dtype)[:, None]
            else:
                d6 = tl[:, 3:-2] + d['traj_local_rot']
            d['traj_local'] = torch.cat([xy, z[:, None], d6, hvec], dim=-1)
            trans, oq = tc.local_to_global(d['traj_local'])
            ex = d['exist_frames']
            ob = d['smpl_orient_world_base'].detach().clone()
            tb = d['root_trans_world_base'].detach().clone()
            ob[ex] = rt.quat_to_aa(oq)
            tb[ex] = trans
            d['smpl_orient_world_base'], d['root_trans_world_base'] = ob, tb

        def forward(self, data, opt_variables, opt_meta):
            """the base forward (:428-531) with world_dxy added in place after the world_res / world_dheading composition
            (:467-468)"""
            persons = data['person_data']
            for d in persons.values():
                if self.flag_infer_motion_traj and self.flag_pred_traj:
                    self.pred_trajectory_base(d)
                if self.flag_opt_traj:
                    if 'world_res' in opt_variables:
                        d['smpl_orient_world'] = d['smpl_orient_world_base'] + d['smpl_orient_world_res']
                        d['root_trans_world'] = d['root_trans_world_base'] + d['root_trans_world_res']
                    else:
                        d['smpl_orient_world'] = d['smpl_orient_world_base']
                        d['root_trans_world'] = d['root_trans_world_base']
                    if 'world_dheading' in d:
                        dh = d['world_dheading']
                        dq = rt.aa_to_quat(torch.cat([torch.zeros(dh.shape[0], 2, dtype=dh.dtype), dh], dim=-1))
                        d['smpl_orient_world'] = rt.quat_to_aa(rt.quat_mul(dq, rt.aa_to_quat(d['smpl_orient_world_base'])))
                        d['root_trans_world'] = d['root_trans_world_base']
                    if 'world_dxy' in d:
                        d['root_trans_world'][:, :2] += d['world_dxy']
                d['person_transform_world'] = rt.make_transform(d['smpl_orient_world'], d['root_trans_world'], 'axis_angle')
            if self.flag_opt_cam and opt_meta['stage'] != 'init':
                if 'cam' in opt_variables:
                    T = data['cam_pose'].shape[0]
                    if self.flag_fixed_cam:
                        data['cam_rot_6d'] = data['cam_rot_6d_fix'].expand(T, -1)
                        data['cam_trans'] = data['cam_trans_fix'].expand(T, -1)
                    if 'cam_rot_6d' in data:
                        data['cam_pose'] = rt.make_transform(data['cam_rot_6d'], data['cam_trans'], '6d')
                        data['cam_pose_inv'] = rt.inverse_transform(data['cam_pose'])
                elif self.flag_opt_cam_from_person_pose:
                    self._camera_from_persons(data)
            for d in persons.values():
                d['smpl_orient_cam_in_world'] = rt.transform_rot(data['cam_pose'], d['smpl_orient_world'])
                d['root_trans_cam_in_world'] = rt.transform_trans(data['cam_pose'], d['root_trans_world'])
                if 'smpl_pose' in d and 'cam_K' in d:
                    dt = d['smpl_orient_world'].dtype
                    joints, _ = self.smpl(d['smpl_orient_world'], d['smpl_pose'].to(dt), d['smpl_beta'].to(dt),
                                          root_trans=d['root_trans_world'], root_scale=d['scale'])
                    d['joints_world'] = joints
                    d['kp_2d_pred'] = rt.perspective_projection(rt.transform_trans(data['cam_pose'], joints), d['cam_K'])

        def get_parameter(self, data, opt_variables):
            """:591-633 with world_dxy: created (zeros) the first time a stage lists it, appended after world_dheading"""
            variables = [v for v in opt_variables if v != 'world_dxy']
            params = []
            if 'cam' not in variables:
                params += [data['cam_inv_rot_residual'], data['cam_inv_trans_residual']]
            else:
                if self.flag_fixed_cam:
                    data['cam_rot_6d_fix'] = rt.rotmat_to_rot6d(data['cam_pose'][[0], :3, :3]).detach()
                    data['cam_trans_fix'] = data['cam_pose'][[0], :3, 3].clone().detach()
                    params += [data['cam_rot_6d_fix'], data['cam_trans_fix']]
                else:
                    data['cam_rot_6d'] = rt.rotmat_to_rot6d(data['cam_pose'][:, :3, :3]).detach()
                    data['cam_trans'] = data['cam_pose'][:, :3, 3].clone().detach()
                    params += [data['cam_rot_6d'], data['cam_trans']]
            for d in data['person_data'].values():
                if self.flag_opt_traj:
                    for key in variables:
                        if key == 'world_res':
                            params += [d['smpl_orient_world_res'], d['root_trans_world_res']]
                        if 'local' in key:
                            params.append(d[f'traj_{key}'])
                if 'world_dheading' in variables:
                    if 'world_dheading' not in d:
                        d['world_dheading'] = torch.zeros_like(d['smpl_orient_world'][..., [0]])
                    params.append(d['world_dheading'])
                if 'world_dxy' in opt_variables:
                    if 'world_dxy' not in d:
                        d['world_dxy'] = torch.zeros_like(d['smpl_orient_world'][..., :2])
                    params.append(d['world_dxy'])
            return params

    return OracleTrajVariables


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
