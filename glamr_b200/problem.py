"""Translate GLAMR's ``data`` dict + one stage's YAML specs into the flat description the CUDA library consumes
(``glamr_problem_t`` / ``glamr_person_t`` of include/glamr_b200.h).

* ``VariableLayout`` packs every optimisation variable of ``GlobalReconOptimizer.get_parameter``
  (global_recon/models/global_recon_model.py:591-633) into one vector ``theta``; the tensors stored in the data dict
  (``cam_rot_6d``, ``traj_local_xy`` ...) are views into it, so the dict always shows current values.
* ``StageCompiler`` turns ``loss_cfg`` (global_recon/models/loss_func.py semantics: min_conf, first_frame_only,
  first_frame_weight, visibility masks, normalisers) into per-frame weight arrays and scalar term tables.

Groups: ``make_layout`` / ``bind_variables`` / ``begin_stage_variables`` / ``StageCompiler`` also take
* a list of G data dicts, the seeds of one sequence (same persons, frames, visibility and loss normalisers, each with its own
  initial state), or
* a list of such lists, ``[[seq0 seed dicts], [seq1 seed dicts], ...]``: a batch of sequences that share one config and may differ
  in frames, persons, exist ranges, frames without persons and visibility.  Each group is compiled from its own data alone,
  normalisers included.
theta then holds group 0's blocks, group 1's, and so on; the persons of all groups are simply more persons, each with its group
index, and StageCompiler uploads one row per group of include/glamr_b200.h's glamr_group_t.  One dict is one group, with exactly the
layout it always had.

Pure tensor bookkeeping, device agnostic (tests build it on the CPU for the host harness); nothing here computes
on the optimisation path.
"""
import ctypes

import numpy as np
import torch

from . import lib as L


class VariableLayout:
    def __init__(self, T, n_empty, trans_res_rows, lens, heading_dim=1, world_dxy=False, person2cam=False, groups=1):
        """heading_dim 2: heading_type 'vec' (traj_local_heading [2], traj_local_dheading [L-1,2]); world_dxy: every person also
        gets a world_dxy [T,2] block (only when a stage can create it, so other problems keep their layout); person2cam: every
        person also gets person2cam_res_rot [T,6] and person2cam_res_trans [T,3] (only when init_data creates them).
        groups G: `lens` are the Q persons of one group; theta holds G copies of the one-group layout, group g's at
        g * group_params, and `persons` / `lens` list the G*Q persons group by group."""
        self.T, self.n_empty, self.trans_res_rows, self.lens = T, n_empty, trans_res_rows, list(lens)
        self.heading_dim, self.world_dxy, self.person2cam = heading_dim, bool(world_dxy), bool(person2cam)
        hd = heading_dim
        off = 0

        def take(n):
            nonlocal off
            o = off
            off += n
            return o
        self.cam_rot, self.cam_trans = take(6 * T), take(3 * T)
        self.cam_rot_fix, self.cam_trans_fix = take(6), take(3)
        self.cam_inv_rot_res, self.cam_inv_trans_res = take(6 * n_empty), take(3 * trans_res_rows)
        self.persons = []
        for Ln in self.lens:
            self.persons.append(dict(xy=take(2), heading=take(hd), dxy=take(2 * (Ln - 1)), dheading=take(hd * (Ln - 1)), z=take(Ln),
                                     rot=take(6 * Ln), world_dheading=take(T), orient_res=take(3 * T), trans_res=take(3 * T),
                                     world_dxy=take(2 * T if self.world_dxy else 0),
                                     p2c_rot=take(6 * T if self.person2cam else 0), p2c_trans=take(3 * T if self.person2cam else 0)))
        self.G, self.Q, self.group_params = int(groups), len(self.lens), off
        one = list(self.persons)
        for g in range(1, self.G):
            self.persons += [{k: o + g * off for k, o in d.items()} for d in one]
        self.lens = self.lens * self.G
        self.n_params = self.G * off

    def group_layout(self, g):
        """(one-group layout, first float of its block in theta) of group g"""
        if self.G == 1:
            return self, 0
        return (VariableLayout(self.T, self.n_empty, self.trans_res_rows, self.lens[:self.Q], heading_dim=self.heading_dim,
                               world_dxy=self.world_dxy, person2cam=self.person2cam), g * self.group_params)

    def group_persons(self, g):
        return range(g * self.Q, (g + 1) * self.Q)

    def views(self, theta, p=None, group=0):
        """name -> view of theta with the reference's tensor shape: the camera variables of `group` (p None), else those of
        person p (counted over all groups)"""
        T = self.T
        if p is None:
            g0 = group * self.group_params
            v = lambda o, n, *shape: theta[g0 + o:g0 + o + n].view(*shape)
            return {'cam_rot_6d': v(self.cam_rot, 6 * T, T, 6), 'cam_trans': v(self.cam_trans, 3 * T, T, 3),
                    'cam_rot_6d_fix': v(self.cam_rot_fix, 6, 1, 6), 'cam_trans_fix': v(self.cam_trans_fix, 3, 1, 3),
                    'cam_inv_rot_residual': v(self.cam_inv_rot_res, 6 * self.n_empty, self.n_empty, 6),
                    'cam_inv_trans_residual': v(self.cam_inv_trans_res, 3 * self.trans_res_rows, self.trans_res_rows, 3)}
        o, Ln, hd = self.persons[p], self.lens[p], self.heading_dim
        v = lambda k, n, *shape: theta[o[k]:o[k] + n].view(*shape)
        out = {'traj_local_xy': v('xy', 2, 2), 'traj_local_heading': v('heading', hd, hd),
               'traj_local_dxy': v('dxy', 2 * (Ln - 1), Ln - 1, 2),
               'traj_local_dheading': v('dheading', Ln - 1, Ln - 1) if hd == 1 else v('dheading', 2 * (Ln - 1), Ln - 1, 2),
               'traj_local_z': v('z', Ln, Ln), 'traj_local_rot': v('rot', 6 * Ln, Ln, 6),
               'world_dheading': v('world_dheading', T, T, 1), 'smpl_orient_world_res': v('orient_res', 3 * T, T, 3),
               'root_trans_world_res': v('trans_res', 3 * T, T, 3)}
        if self.world_dxy:
            out['world_dxy'] = v('world_dxy', 2 * T, T, 2)
        if self.person2cam:
            out['person2cam_res_rot'] = v('p2c_rot', 6 * T, T, 6)
            out['person2cam_res_trans'] = v('p2c_trans', 3 * T, T, 3)
        return out


class BatchLayout:
    """Groups of a batch of sequences: theta is the concatenation of one one-group VariableLayout per group, each at its own base
    (``bases``).  ``persons`` / ``lens`` list the persons of all groups, group by group, with offsets into the whole theta."""

    def __init__(self, lays):
        self.layouts = list(lays)
        self.G = len(self.layouts)
        self.bases, self.p0s, off, p = [], [], 0, 0
        for lay in self.layouts:
            self.bases.append(off)
            self.p0s.append(p)
            off += lay.n_params
            p += lay.Q
        self.n_params = off
        self.persons = [{k: o + b for k, o in d.items()} for lay, b in zip(self.layouts, self.bases) for d in lay.persons]
        self.lens = [n for lay in self.layouts for n in lay.lens]
        self.person_group = [g for g, lay in enumerate(self.layouts) for _ in range(lay.Q)]
        l0 = self.layouts[0]
        self.heading_dim, self.world_dxy, self.person2cam = l0.heading_dim, l0.world_dxy, l0.person2cam
        self.T = max(lay.T for lay in self.layouts)              # the longest group's frames (glamr_problem_t.T)

    def group_layout(self, g):
        return self.layouts[g], self.bases[g]

    def group_persons(self, g):
        return range(self.p0s[g], self.p0s[g] + self.layouts[g].Q)

    def views(self, theta, p=None, group=0):
        """as VariableLayout.views: the camera variables of `group` (p None), else those of person p (counted over all groups)"""
        if p is not None:
            group = self.person_group[p]
        lay, b = self.group_layout(group)
        sub = theta[b:b + lay.n_params]
        return lay.views(sub) if p is None else lay.views(sub, p - self.p0s[group])


def _f32(x, device):
    return torch.as_tensor(x).to(device=device, dtype=torch.float32).contiguous()


def _is_batch(data):
    """a list of per-sequence lists of seed dicts (a batch of sequences)"""
    return isinstance(data, (list, tuple)) and len(data) > 0 and isinstance(data[0], (list, tuple))


def _groups(data):
    """one data dict, the list of the seed groups' data dicts, or a batch's list of such lists -> flat list of group dicts"""
    if _is_batch(data):
        return [d for seq in data for d in seq]
    return list(data) if isinstance(data, (list, tuple)) else [data]


class StageCompiler:
    """Holds the per-person constant tensors and builds a ``Problem`` for every stage."""

    def __init__(self, data, layout, flags, device, aa_to_rot6d, num_joints=26, aa_to_quat=None):
        """data: one data dict, the list of the seed groups' data dicts, or a batch of sequences (see the module docstring).
        flags: dict with flag_fixed_cam, flag_opt_cam, flag_opt_cam_from_person_pose, flag_cam_inv_trans_res_all,
        flag_opt_vis_local_rot, cam_fix_frames and optionally flag_opt_traj / traj_source (when absent they are read off
        `data`: a predicted trajectory leaves traj_local_pred, flag_opt_traj leaves the world_res variables), heading_vec
        (heading_type 'vec'; default: the layout's heading size) and flag_opt_person2cam_rot / _trans (default false).
        aa_to_rot6d: callable (device math lives in the CUDA library)."""
        self.batch = _is_batch(data) and len(data) > 1       # one sequence in a batch: its seed groups
        self.datas = _groups(data)
        data = self.datas[0]
        self.data, self.layout, self.flags, self.device, self.J = data, layout, flags, device, num_joints
        self.pids = list(data['person_data'].keys())
        self.Qs = [len(dd['person_data']) for dd in self.datas]
        self.Ts = [int(dd['seq_len']) for dd in self.datas]
        if not self.batch and any(q != self.Qs[0] or t != self.Ts[0] for q, t in zip(self.Qs, self.Ts)):
            raise ValueError('seed groups need the same persons and frame count')
        self.G, self.P, self.T = len(self.datas), sum(self.Qs), max(self.Ts)   # T: every group's frames when they agree
        self.Q = self.Qs[0] if len(set(self.Qs)) == 1 else None                 # persons per group when they agree
        # first person / frame-person / camera row of each group, and the group and frames of each person
        self.p0s, self.n0s, self.c0s, p, n, r = [], [], [], 0, 0, 0
        for q, t in zip(self.Qs, self.Ts):
            self.p0s.append(p)
            self.n0s.append(n)
            self.c0s.append(r)
            p, n, r = p + q, n + q * t, r + t
        self.N = n                                   # frame-persons of all groups
        self.person_group = [g for g, q in enumerate(self.Qs) for _ in range(q)]
        self.person_T = [self.Ts[g] for g in self.person_group]
        dev = device
        persons = [d for dd in self.datas for d in dd['person_data'].values()]
        self.persons = persons
        self.traj_source = flags.get('traj_source', L.TRAJ_PREDICTED if all('traj_local_pred' in d for d in persons) else L.TRAJ_BASE)
        self.opt_traj = flags.get('flag_opt_traj', all('smpl_orient_world_res' in d for d in persons))
        self.has_local = all('traj_local_xy' in d for d in persons)        # created with flag_opt_traj and flag_pred_traj (:185-199)
        self.heading_vec = bool(flags.get('heading_vec', layout.heading_dim == 2))
        self.keep = []                               # tensors whose storage the structs point into
        self.const = []
        pose_all, beta_all, scale_all = [], [], []
        for d in persons:
            start, Ln = int(d['fr_start']), int(d['exist_len'])
            mask = torch.ones(max(Ln - 1, 0))
            for (s, e) in flags['cam_fix_frames']:
                mask[s:e] = 0.0
            c = {
                'start': start, 'len': Ln,
                # without a predicted trajectory no kernel reads it; zeros keep the pointer valid
                'traj_local_pred': _f32(d['traj_local_pred'] if 'traj_local_pred' in d else torch.zeros(Ln, 11), dev),
                'orient_base_init': _f32(d['smpl_orient_world_base'], dev).clone(),
                'trans_base_init': _f32(d['root_trans_world_base'], dev).clone(),
                'cam_K': _f32(d['cam_K'], dev).reshape(-1, 9),
                'kp_target': _f32(d['kp_2d_aligned'], dev),
                'orient_cam_6d': _f32(aa_to_rot6d(_f32(d['smpl_orient_cam'], dev)), dev),
                'orient_cam_q': None if aa_to_quat is None else _f32(aa_to_quat(_f32(d['smpl_orient_cam'], dev)), dev),
                'trans_cam': _f32(d['root_trans_cam'], dev),
                'person2cam': _f32(d['person2cam'], dev)[:, :3, :].reshape(-1, 12).contiguous(),
                'dheading_mask': _f32(mask, dev),
                'rot_mask': _f32(d['vis_frames'][start:start + Ln], dev) if flags.get('flag_opt_vis_local_rot', False) else None,
                'vis': _f32(d['vis_frames'], dev),
                # x / y of the base that world_dxy's in-place add advances (include/glamr_b200.h, world_dxy_base)
                'world_dxy_base': _f32(d['root_trans_world_base'], dev)[:, :2].contiguous().clone() if layout.world_dxy else None,
            }
            self.const.append(c)
            pose_all.append(_f32(d['smpl_pose'], dev))
            beta_all.append(_f32(d['smpl_beta'], dev))
            scale_all.append(None if d['scale'] is None else _f32(d['scale'], dev))
        # [P,T,...] when every group has T frames, else the [N,...] rows of all persons (the same memory order)
        cat = torch.stack if len(set(self.Ts)) == 1 else torch.cat
        self.pose_all = cat(pose_all).contiguous()
        self.beta_all = cat(beta_all).contiguous()
        self.scale_all = None if scale_all[0] is None else cat(scale_all).contiguous()
        # host copies of what the per-stage weight tables are built from (visibility, keypoint scores, persons per frame):
        # ONE device->host copy here instead of several per person and stage
        J_, N_ = self.J, self.N
        packed = torch.cat([torch.cat([torch.as_tensor(d['vis_frames']).to(dev).double().reshape(-1) for d in persons]),
                            torch.cat([torch.as_tensor(d['kp_2d_score']).to(dev).double().reshape(-1) for d in persons]),
                            torch.cat([torch.as_tensor(dd['fr_num_persons']).to(dev).double().reshape(-1) for dd in self.datas])]).cpu()
        self.host_vis = [v > 0.5 for v in packed[:N_].split(self.person_T)]                       # per person [T]
        self.host_score = [v.reshape(-1, J_) for v in packed[N_:N_ + N_ * J_].split([t * J_ for t in self.person_T])]   # [T, J]
        # camera-from-persons bookkeeping (global_recon_model.py:489-506), one [T] block per group
        src, empty_idx, inv_num = [], [], []
        for npers, T in zip(packed[N_ + N_ * J_:].to(torch.int64).split(self.Ts), self.Ts):
            has = npers > 0
            last, ne = int(torch.where(has)[0][0]), 0
            for t in range(T):
                if npers[t] > 0:
                    last = t
                    empty_idx.append(-1)
                else:
                    empty_idx.append(ne)
                    ne += 1
                src.append(last)
            inv_num.append(torch.where(has, 1.0 / npers.clamp(min=1).float(), torch.zeros(T)))
        self.fill_src = torch.tensor(src, dtype=torch.int32, device=dev)
        self.empty_index = torch.tensor(empty_idx, dtype=torch.int32, device=dev)
        self.inv_num = _f32(torch.cat(inv_num), dev)
        # rel_transform targets: pairs (i, j) inside each group, one [Q*Q, T] block per group starting at (pair, frame) entry rel0
        self.rel0, n_rel = [], 0
        for q, t in zip(self.Qs, self.Ts):
            self.rel0.append(n_rel)
            n_rel += q * q * t
        if any(dd.get('rel_transform_cam') for dd in self.datas):
            tgt = torch.zeros(n_rel, 12, device=dev)
            for g, dd in enumerate(self.datas):
                Q_, T = self.Qs[g], self.Ts[g]
                for (i, j), C in (dd.get('rel_transform_cam') or {}).items():
                    r = self.rel0[g] + (i * Q_ + j) * T
                    tgt[r:r + T] = torch.as_tensor(C).detach().to(dev).float()[:, :3, :].reshape(T, 12)
            self.rel_target = tgt.contiguous()
        else:
            self.rel_target = None

    # ------------------------------------------------------------------------------------------------ per stage
    def _person_weights(self, p, loss_cfg):
        T, J = self.person_T[p], self.J
        vis, score = self.host_vis[p], self.host_score[p]
        vis_idx = torch.where(vis)[0]
        nvis = int(vis.sum())
        kp_w, kp_dm = torch.zeros(T, J, dtype=torch.float64), torch.zeros(T, J, dtype=torch.float64)
        ctr_w, ctt_w = torch.zeros(T, dtype=torch.float64), torch.zeros(T, dtype=torch.float64)
        norms = {}
        if 'kp_2d' in loss_cfg:                                              # loss_func.py:15-36
            sp = loss_cfg['kp_2d']
            conf = score.clone()
            conf[conf < sp.get('min_conf', 0.05)] = 0
            ffw = sp.get('first_frame_weight', 1.0)
            if sp.get('first_frame_only', False):
                kp_w[vis_idx[0]] = ffw * (conf[vis] ** 2).sum(0)           # rho of frame 0 broadcast over all frames' scores
            else:
                fw = torch.ones(nvis, dtype=torch.float64)
                fw[:10] = ffw
                kp_w[vis] = conf[vis] ** 2 * fw[:, None]
            norms['kp_2d'] = nvis
        if 'kp_2d_dist' in loss_cfg:                                         # loss_func.py:39-57
            sp = loss_cfg['kp_2d_dist']
            m = (score > sp.get('min_conf', 0.05)).double()
            if sp.get('first_frame_only', False):
                m[1:] = 0
            kp_dm = m
            norms['kp_2d_dist'] = float(m.sum())
        if 'cam_traj_rot' in loss_cfg:                                       # loss_func.py:147-172
            sp = loss_cfg['cam_traj_rot']
            if sp.get('rot_type', '6d') not in ('6d', 'quat'):
                raise ValueError(f"cam_traj_rot: unknown rot_type {sp.get('rot_type')}")
            if sp.get('first_frame_only', False):
                ctr_w[vis_idx[0]] = 1.0
                norms['cam_traj_rot'] = 1
            else:
                ctr_w[vis] = 1.0
                ctr_w[vis_idx[0]] = sp.get('first_frame_weight', 1.0) ** 2
                norms['cam_traj_rot'] = nvis
        if 'cam_traj_trans' in loss_cfg:                                     # loss_func.py:175-186
            sp = loss_cfg['cam_traj_trans']
            ctt_w[vis] = 1.0
            ctt_w[vis_idx[0]] = sp.get('first_frame_weight', 1.0) ** 2
            norms['cam_traj_trans'] = nvis
        return kp_w, kp_dm, ctr_w, ctt_w, norms

    def compile(self, theta, opt_variables, loss_cfg, stage, n_begin=0, n_end=None, owner=True):
        data, lay, fl, dev, P, T, J = self.data, self.layout, self.flags, self.device, self.P, self.T, self.J
        G, persons_all = self.G, self.persons
        n_end = self.N if n_end is None else n_end
        if 'person2cam_res_trans_reg' in loss_cfg:           # loss_func.py:244-245
            raise ValueError("residual 'person2cam_res_trans_reg' reads data['person2cam_res_trans'], a key the reference never creates "
                             "(the residuals live per person), so the reference fails with KeyError; it has no defined meaning to implement")
        for name in loss_cfg:
            if name not in L.TERM_INDEX:
                raise NotImplementedError(f"residual '{name}' has no CUDA implementation (no CPU fallback)")
        pb = L.Problem()
        pb.P, pb.T, pb.J, pb.n_params = P, T, J, lay.n_params
        pb.G, pb.group_params = G, getattr(lay, 'group_params', 0)          # a batch describes its groups in the table below
        pb.n_begin, pb.n_end, pb.owner = n_begin, n_end, int(owner)
        keep = []
        # ---- camera mode (global_recon_model.py:473-508)
        mode = L.CAM_CONST
        if fl['flag_opt_cam'] and stage != 'init':
            if 'cam' in opt_variables:
                mode = L.CAM_FIXED if fl['flag_fixed_cam'] else L.CAM_PER_FRAME
            elif fl['flag_opt_cam_from_person_pose']:
                mode = L.CAM_FROM_PERSONS
        pb.cam_mode = mode

        def cam_offsets(lg):
            if mode == L.CAM_FIXED:
                return lg.cam_rot_fix, lg.cam_trans_fix
            if mode == L.CAM_PER_FRAME:
                return lg.cam_rot, lg.cam_trans
            return lg.cam_inv_rot_res, lg.cam_inv_trans_res
        pb.off_cam_rot, pb.off_cam_trans = cam_offsets(lay.group_layout(0)[0])
        cam_const = torch.cat([_f32(dd['cam_pose'], dev)[:, :3, :].reshape(-1, 12) for dd in self.datas]).contiguous().clone()
        keep.append(cam_const)
        pb.cam_pose_const = cam_const.data_ptr()
        pb.trans_res_all = int(fl['flag_cam_inv_trans_res_all'])
        # ---- trajectory source; the world variables enter the forward only with flag_opt_traj (:451-468)
        pb.traj_source = self.traj_source
        pb.use_world_res = int(self.opt_traj and 'world_res' in opt_variables)
        pb.has_world_dheading = int(self.opt_traj and any('world_dheading' in d for d in persons_all))
        pb.heading_vec = int(self.heading_vec)
        # world_dxy, once created, is added in place to root_trans_world (:467-468); that tensor IS the base unless world_res
        # alone composes the pose, and then the add lands in the base too
        has_dxy = self.opt_traj and any('world_dxy' in d for d in persons_all)
        alias = has_dxy and (pb.has_world_dheading or not pb.use_world_res)
        if alias and self.traj_source == L.TRAJ_BASE:
            raise ValueError("world_dxy with a trajectory that does not come from the predictor needs world_res in opt_variables and "
                             "no world_dheading: otherwise the reference adds world_dxy in place to a base it never re-creates, and "
                             "its second backward fails (autograd graph already freed)")
        pb.has_world_dxy, pb.world_dxy_alias = int(has_dxy), int(alias)
        # person2cam residuals (:173-175,484-488,616-619): created by init_data with flag_opt_traj, then composed into every
        # camera-from-persons forward; Adam moves them only in stages that list them
        p2c_flags = {'person2cam_rot': fl.get('flag_opt_person2cam_rot', False), 'person2cam_trans': fl.get('flag_opt_person2cam_trans', False)}
        if any(p2c_flags.values()) and not self.opt_traj:
            listed = [k for k, f in p2c_flags.items() if f and k in opt_variables]
            if listed:
                raise ValueError(f"optimisation variable '{listed[0]}' needs flag_opt_traj: the person2cam residuals are created only with "
                                 "it, so the reference's get_parameter fails with KeyError")
            if mode == L.CAM_FROM_PERSONS:
                raise ValueError('flag_opt_person2cam_rot / _trans need flag_opt_traj when the camera comes from the persons: the '
                                 "residuals are created only with flag_opt_traj, so the reference's forward fails with KeyError")
        pb.has_person2cam = int(lay.person2cam)
        # combinations the reference fails on (KeyError / None.items() in get_parameter or loss_func.py): fail clearly here
        if not self.has_local:
            for key in opt_variables:
                if 'local' in key and self.opt_traj:
                    raise ValueError(f"optimisation variable '{key}' needs the local trajectory variables, which exist only with "
                                     "flag_pred_traj and flag_opt_traj")
            for name in loss_cfg:
                if name.startswith('local_traj_'):
                    raise ValueError(f"residual '{name}' needs the local trajectory variables, which exist only with "
                                     "flag_pred_traj and flag_opt_traj")
        if not self.opt_traj:
            for name in ('traj_rot_res', 'traj_trans_res', 'rel_transform'):
                if name in loss_cfg:
                    raise ValueError(f"residual '{name}' needs flag_opt_traj (world_res / rel_transform_cam are not created without it)")
        pb.empty_index, pb.fill_src, pb.inv_num_persons = self.empty_index.data_ptr(), self.fill_src.data_ptr(), self.inv_num.data_ptr()
        pb.smpl_pose_all, pb.smpl_beta_all = self.pose_all.data_ptr(), self.beta_all.data_ptr()
        pb.scale_all = None if self.scale_all is None else self.scale_all.data_ptr()
        # ---- persons
        persons = (L.Person * P)()
        # normalisers of each group's persons: seed groups of one sequence must agree, the groups of a batch have their own
        group_norms = [{} for _ in range(G)]
        host_w, w_off, o = [], [], 0            # [kp_w | kp_dist_mask | ctr_w | ctt_w] per person, persons one after another
        for p in range(P):
            kp_w, kp_dm, ctr_w, ctt_w, nrm = self._person_weights(p, loss_cfg)
            host_w.append(torch.cat([kp_w.reshape(-1), kp_dm.reshape(-1), ctr_w, ctt_w]).float())
            w_off.append(o)
            o += host_w[-1].numel()
            gn = group_norms[self.person_group[p]]
            for k, v in nrm.items():
                gn[k] = gn.get(k, 0) + v
        if not self.batch and any(n != group_norms[0] for n in group_norms[1:]):
            raise ValueError('seed groups need the same loss normalisers (visibility and keypoint scores of one sequence)')
        dev_w = torch.cat(host_w).to(dev)                                        # one upload for all persons
        keep.append(dev_w)
        for p in range(P):
            c, o = self.const[p], lay.persons[p]
            ps = persons[p]
            ps.start, ps.len, ps.group = c['start'], c['len'], self.person_group[p]
            ps.off_xy, ps.off_heading, ps.off_dxy, ps.off_dheading = o['xy'], o['heading'], o['dxy'], o['dheading']
            ps.off_z, ps.off_rot, ps.off_world_dheading = o['z'], o['rot'], o['world_dheading']
            ps.off_orient_res, ps.off_trans_res, ps.off_world_dxy = o['orient_res'], o['trans_res'], o['world_dxy']
            ps.off_p2c_rot, ps.off_p2c_trans = o['p2c_rot'], o['p2c_trans']
            for name in ['traj_local_pred', 'orient_base_init', 'trans_base_init', 'cam_K', 'kp_target', 'orient_cam_6d',
                         'orient_cam_q', 'trans_cam', 'person2cam', 'dheading_mask', 'rot_mask', 'vis', 'world_dxy_base']:
                setattr(ps, name, None if c[name] is None else c[name].data_ptr())
            base, Tp = dev_w.data_ptr() + w_off[p] * 4, self.person_T[p]
            ps.kp_w, ps.kp_dist_mask = base, base + Tp * J * 4
            ps.ctr_w, ps.ctt_w = base + 2 * Tp * J * 4, base + (2 * Tp * J + Tp) * 4
        persons_dev = torch.frombuffer(bytearray(bytes(persons)), dtype=torch.uint8).to(dev)
        keep.append(persons_dev)
        pb.persons = persons_dev.data_ptr()
        # ---- rel_transform (loss_func.py:248-271)
        if self.rel_target is not None and 'rel_transform' in loss_cfg:
            sp = loss_cfg['rel_transform']
            ffw = sp.get('first_frame_weight', 10)
            rw, rwt = torch.zeros(self.rel_target.shape[0]), torch.zeros(self.rel_target.shape[0])
            for g, dd in enumerate(self.datas):
                Q, Tg, p0 = self.Qs[g], self.Ts[g], self.p0s[g]
                pairs = dd.get('rel_transform_cam') or {}
                for (i, j) in pairs.keys():
                    both = self.host_vis[p0 + i] & self.host_vis[p0 + j]
                    if both.sum() == 0:
                        continue
                    f0 = int(torch.where(both)[0][0])
                    wv = both.float()
                    wv[f0] = float(ffw) ** 2
                    r = self.rel0[g] + (i * Q + j) * Tg
                    rw[r:r + Tg] = wv
                    wt = wv.clone()
                    if sp.get('first_frame_trans_only', False):
                        wt[:] = 0
                        wt[f0] = float(ffw) ** 2
                    rwt[r:r + Tg] = wt
                group_norms[g]['rel_transform'] = Tg * len(pairs)
            rw, rwt = rw.to(dev).contiguous(), rwt.to(dev).contiguous()
            keep += [rw, rwt]
            pb.rel_target, pb.rel_w, pb.rel_wt = self.rel_target.data_ptr(), rw.data_ptr(), rwt.data_ptr()
            pb.rel_trans_weight = sp.get('trans_weight', 1.0)
        elif 'rel_transform' in loss_cfg:
            for gn in group_norms:
                gn['rel_transform'] = 0
        # ---- scalar term tables, each group's from its own persons and frames
        for g, norms in enumerate(group_norms):
            lg = lay.group_layout(g)[0]
            Q, Tg, lens = self.Qs[g], self.Ts[g], lg.lens
            norms.update({
                'traj_rot_smoothness': Q * (Tg - 1), 'traj_trans_smoothness': Q * (Tg - 1),
                'local_traj_dxy_reg': sum(n - 1 for n in lens), 'local_traj_dheading_reg': sum(n - 1 for n in lens),
                'local_traj_dheading_reg_new': sum(n - 1 for n in lens), 'local_traj_rot_reg': sum(lens), 'local_traj_z_reg': sum(lens),
                'traj_rot_res': Q * Tg, 'traj_trans_res': Q * Tg, 'cam_inv_trans_residual_reg': lg.trans_res_rows,
                'cam_inv_rot_smoothness': Tg - 1, 'cam_origin_smoothness': Tg - 1, 'cam_rot_smoothness': Tg - 1,
                'cam_trans_smoothness': Tg - 1,
                'cam_depth_smoothness': 1,          # loss_func.py:102 sums over the T-1 frame pairs (the .mean() sees a 0-d tensor)
            })
        pb.cam_traj_rot_quat = int(loss_cfg.get('cam_traj_rot', {}).get('rot_type', '6d') == 'quat')
        pb.traj_rot_smooth_quat = int(loss_cfg.get('traj_rot_smoothness', {}).get('rot_type', '6d') == 'quat')
        if (pb.cam_traj_rot_quat or pb.traj_rot_smooth_quat) and self.const[0]['orient_cam_q'] is None:
            raise ValueError("rot_type 'quat' needs the aa_to_quat callable (StageCompiler(..., aa_to_quat=...))")
        if 'cam_up_reg' in loss_cfg:
            sp = loss_cfg['cam_up_reg']
            pb.cam_up_first_weight = sp.get('first_frame_weight', 1.0)
            pb.cam_up_first_only = int(sp.get('first_frame_only', False))
            for norms, Tg in zip(group_norms, self.Ts):
                norms['cam_up_reg'] = 1 if pb.cam_up_first_only else Tg
        if ('cam_rot_smoothness' in loss_cfg or 'cam_trans_smoothness' in loss_cfg) and mode != L.CAM_PER_FRAME:
            raise NotImplementedError('cam_rot/trans_smoothness need per-frame camera variables')
        for name, sp in loss_cfg.items():
            k = L.TERM_INDEX[name]
            pb.term_enabled[k] = 1
            pb.term_monitor[k] = int(sp.get('monitor_only', False))
            pb.term_weight[k] = float(sp['weight'])
            n = float(group_norms[0].get(name, 1))
            pb.term_norm[k] = n if n > 0 else 1.0
        if G > 1:                                            # the group table (include/glamr_b200.h, glamr_group_t)
            table = (L.Group * G)()
            for g, gr in enumerate(table):
                lg, base = lay.group_layout(g)
                gr.p0, gr.Q, gr.n0, gr.c0, gr.T = self.p0s[g], self.Qs[g], self.n0s[g], self.c0s[g], self.Ts[g]
                gr.theta0, gr.rel0 = base, self.rel0[g]
                gr.off_cam_rot, gr.off_cam_trans = (base + o for o in cam_offsets(lg))
                for name in loss_cfg:
                    k, n = L.TERM_INDEX[name], float(group_norms[g].get(name, 1))
                    gr.term_norm[k] = n if n > 0 else 1.0
                for k in range(L.NUM_TERMS):                 # the handle's weight / normaliser (float32 division)
                    if pb.term_enabled[k] and not pb.term_monitor[k] and gr.term_norm[k] != 0.0:
                        gr.gs[k] = float(np.float32(pb.term_weight[k]) / np.float32(gr.term_norm[k]))
            table_dev = torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8).to(dev)
            keep.append(table_dev)
            pb.groups = table_dev.data_ptr()
            self.table = table
        # ---- which entries of theta Adam updates (get_parameter, :591-633)
        active = torch.zeros(lay.n_params, dtype=torch.uint8)

        def on(o, n):
            active[o:o + n] = 1
        for g in range(G):                                    # each group's camera variables
            lg, g0 = lay.group_layout(g)
            if 'cam' not in opt_variables:
                on(g0 + lg.cam_inv_rot_res, 6 * lg.n_empty)
                on(g0 + lg.cam_inv_trans_res, 3 * lg.trans_res_rows)
            elif fl['flag_fixed_cam']:
                on(g0 + lg.cam_rot_fix, 6)
                on(g0 + lg.cam_trans_fix, 3)
            else:
                on(g0 + lg.cam_rot, 6 * lg.T)
                on(g0 + lg.cam_trans, 3 * lg.T)
        hd = lay.heading_dim
        sizes = lambda Ln: {'xy': 2, 'heading': hd, 'dxy': 2 * (Ln - 1), 'dheading': hd * (Ln - 1), 'z': Ln, 'rot': 6 * Ln}
        for p in range(P):
            o, sz, T = lay.persons[p], sizes(lay.lens[p]), self.person_T[p]
            for key in opt_variables:
                if key == 'world_res' and self.opt_traj:
                    on(o['orient_res'], 3 * T)
                    on(o['trans_res'], 3 * T)
                if 'local' in key and self.opt_traj:
                    name = key[len('local_'):]
                    if name not in sz:
                        raise KeyError(f'unknown optimisation variable {key}')
                    on(o[name], sz[name])
                if key == 'world_dheading':
                    on(o['world_dheading'], T)
                if key == 'world_dxy' and self.opt_traj:          # without flag_opt_traj the forward never reads it (:451)
                    on(o['world_dxy'], 2 * T)
                # with the flag and flag_opt_traj (get_parameter, :616-619); a stage whose forward never reads them ('cam' listed, or
                # 'init') gives them a zero gradient, which leaves them unchanged like torch's Adam skipping a grad of None
                if key == 'person2cam_rot' and p2c_flags[key] and lay.person2cam:
                    on(o['p2c_rot'], 6 * T)
                if key == 'person2cam_trans' and p2c_flags[key] and lay.person2cam:
                    on(o['p2c_trans'], 3 * T)
        active = active.to(dev)
        keep.append(active)
        pb.active = active.data_ptr()
        self.keep = keep
        return pb


# ---------------------------------------------------------------------------------------------------- variables
_KINDS = [('heading_dim', 'heading variables (heading_type)'), ('world_dxy', 'world_dxy variables'),
          ('person2cam', 'person2cam residuals')]


def make_layout(data, flags):
    """layout of one data dict, of the seed groups in a list of data dicts (which must agree on every block), or of a batch of
    sequences (a list of such lists): a BatchLayout of one one-group layout per group, which must agree on the variable kinds"""
    if _is_batch(data) and len(data) == 1:                 # one sequence: its seed groups
        return make_layout(list(data[0]), flags)
    if _is_batch(data):
        lays = []
        for seq in data:
            one = make_layout(list(seq), flags)                # the seeds of one sequence agree on every block
            lays += [one.group_layout(g)[0] for g in range(one.G)]
        for attr, what in _KINDS:
            vals = sorted({getattr(l, attr) for l in lays})
            if len(vals) > 1:
                raise ValueError(f'the groups of one problem share one config, but their {what} differ ({attr}: {vals})')
        return lays[0] if len(lays) == 1 else BatchLayout(lays)
    datas = _groups(data)
    lays = [_one_group_layout(d, flags) for d in datas]
    key = lambda l: (l.T, l.n_empty, l.trans_res_rows, l.lens, l.heading_dim, l.world_dxy, l.person2cam)
    if any(key(l) != key(lays[0]) for l in lays[1:]):
        raise ValueError('seed groups need the same variable layout (persons, exist ranges, frames without persons, variables)')
    if len(datas) == 1:
        return lays[0]
    l0 = lays[0]
    return VariableLayout(l0.T, l0.n_empty, l0.trans_res_rows, l0.lens, heading_dim=l0.heading_dim, world_dxy=l0.world_dxy,
                          person2cam=l0.person2cam, groups=len(datas))


def _one_group_layout(data, flags):
    persons = data['person_data']
    T = data['seq_len']
    n_empty = int((torch.as_tensor(data['fr_num_persons']) == 0).sum())
    rows = T if flags['flag_cam_inv_trans_res_all'] else n_empty
    world_dxy = flags.get('world_dxy', False) or any('world_dxy' in d for d in persons.values())
    heading_vec = flags.get('heading_vec')
    if heading_vec is None:              # read off the variables init_data created (:191-196)
        heading_vec = any('traj_local_heading' in d and torch.as_tensor(d['traj_local_heading']).numel() == 2 for d in persons.values())
    # init_data created them (:173-175); with both flags off the reference neither reads nor optimises them
    person2cam = ((flags.get('flag_opt_person2cam_rot', False) or flags.get('flag_opt_person2cam_trans', False))
                  and any('person2cam_res_rot' in d for d in persons.values()))
    return VariableLayout(T, n_empty, rows, [int(d['exist_len']) for d in persons.values()],
                          heading_dim=2 if heading_vec else 1, world_dxy=world_dxy, person2cam=person2cam)


def bind_variables(data, layout, theta):
    """Move every optimisation variable that already exists in `data` into the packed vector `theta` and replace the
    dict entry by the view, so later reads (and the final tensor_to_numpy) see what the kernels update.  `data`: one dict or
    the seed groups' list."""
    for g, dd in enumerate(_groups(data)):
        gv = layout.views(theta, group=g)
        for name in ['cam_inv_rot_residual', 'cam_inv_trans_residual']:
            gv[name].copy_(torch.as_tensor(dd[name]).to(theta))
            dd[name] = gv[name]
        for p, d in zip(layout.group_persons(g), dd['person_data'].values()):
            pv = layout.views(theta, p)
            for name in ['traj_local_xy', 'traj_local_heading', 'traj_local_dxy', 'traj_local_dheading', 'traj_local_z',
                         'traj_local_rot', 'smpl_orient_world_res', 'root_trans_world_res', 'world_dheading', 'world_dxy',
                         'person2cam_res_rot', 'person2cam_res_trans']:
                # world_dheading exists once a stage has requested it (global_recon_model.py:624-627); with continue_opt it
                # arrives already optimised and forward() keeps composing with it (:459-465)
                if name in d:
                    pv[name].copy_(torch.as_tensor(d[name]).to(theta))
                    d[name] = pv[name]


def begin_stage_variables(data, layout, theta, flags, opt_variables):
    """Side effects of GlobalReconOptimizer.get_parameter (global_recon_model.py:596-631): camera variables are
    re-initialised from the current cam_pose, world_dheading / world_dxy are created (zeros) the first time they are requested.
    `data`: one dict or the seed groups' list."""
    if 'world_dxy' in opt_variables and not layout.world_dxy:
        raise ValueError("opt_variables lists 'world_dxy' but the variable layout has no world_dxy block "
                         "(make_layout(..., flags={'world_dxy': True, ...}))")
    for g, data in enumerate(_groups(data)):
        gv = layout.views(theta, group=g)
        T = layout.group_layout(g)[0].T
        if 'cam' in opt_variables:
            cam = torch.as_tensor(data['cam_pose']).to(theta)
            d6 = torch.cat([cam[:, :3, 0], cam[:, :3, 1]], dim=-1)           # rotmat_to_rot6d: first two columns
            if flags['flag_fixed_cam']:
                gv['cam_rot_6d_fix'].copy_(d6[:1])
                gv['cam_trans_fix'].copy_(cam[:1, :3, 3])
                data['cam_rot_6d_fix'], data['cam_trans_fix'] = gv['cam_rot_6d_fix'], gv['cam_trans_fix']
                data['cam_rot_6d'] = gv['cam_rot_6d_fix'].expand(T, -1)
                data['cam_trans'] = gv['cam_trans_fix'].expand(T, -1)
            else:
                gv['cam_rot_6d'].copy_(d6)
                gv['cam_trans'].copy_(cam[:, :3, 3])
                data['cam_rot_6d'], data['cam_trans'] = gv['cam_rot_6d'], gv['cam_trans']
        for p, d in zip(layout.group_persons(g), data['person_data'].values()):
            if 'world_dheading' in opt_variables and 'world_dheading' not in d:
                d['world_dheading'] = layout.views(theta, p)['world_dheading']
            if 'world_dxy' in opt_variables and 'world_dxy' not in d:
                d['world_dxy'] = layout.views(theta, p)['world_dxy']
