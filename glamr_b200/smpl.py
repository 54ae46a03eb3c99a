"""SMPL body model on the CUDA library -- drop-in for the reference's ``lib/models/smpl.py`` ``SMPL`` class
(``forward`` :289-316 and ``get_joints`` :318-343) for ``pose_type='body26fk'`` and friends.

The arithmetic (Rodrigues, kinematic chain, blend shapes, linear blend skinning, extra joint regression, remap,
re-rooting) runs in ``glamr_smpl_forward`` / ``glamr_smpl_fk24`` (glamr_b200/csrc/smpl_kernels.cu).  Inputs/outputs
are torch CUDA tensors used as plain device buffers; there is no autograd through this class (the optimiser has its
own analytic backward) and no CPU fallback.
"""
import ctypes
import os
from collections import namedtuple

import numpy as np
import torch

from . import lib as L
from .synthetic import BODY26FK_JOINT_MAP, EXTRA_VERTEX_IDS

ModelOutput = namedtuple('ModelOutput', ['vertices', 'joints', 'full_pose', 'betas', 'global_orient', 'body_pose',
                                         'expression', 'left_hand_pose', 'right_hand_pose', 'jaw_pose', 'global_trans', 'scale'])
ModelOutput.__new__.__defaults__ = (None,) * len(ModelOutput._fields)

SMPL_MODEL_DIR = 'data/body_models/smpl'
JOINT_REGRESSOR_TRAIN_EXTRA = 'data/J_regressor_extra.npy'


def load_smpl_assets(model_dir=SMPL_MODEL_DIR, extra_path=JOINT_REGRESSOR_TRAIN_EXTRA):
    """Read an SMPL model file (npz with the standard keys, or the official pickle) + J_regressor_extra.npy."""
    npz = [f for f in os.listdir(model_dir) if f.endswith('.npz')]
    if npz:
        d = dict(np.load(os.path.join(model_dir, npz[0]), allow_pickle=True))
    else:
        import pickle
        pk = [f for f in os.listdir(model_dir) if f.endswith('.pkl')]
        if not pk:
            raise FileNotFoundError(f'no SMPL model file in {model_dir}')
        with open(os.path.join(model_dir, pk[0]), 'rb') as f:
            d = pickle.load(f, encoding='latin1')
    a = {}
    for k in ['v_template', 'shapedirs', 'posedirs', 'J_regressor', 'weights', 'lbs_weights', 'kintree_table', 'parents', 'f', 'faces']:
        if k in d:
            v = d[k]
            a[k] = np.asarray(v.todense() if hasattr(v, 'todense') else v)
    if 'lbs_weights' not in a:
        a['lbs_weights'] = a.pop('weights')
    if 'parents' not in a:
        a['parents'] = a['kintree_table'][0].astype(np.int64)
        a['parents'][0] = -1
    if 'faces' not in a and 'f' in a:
        a['faces'] = a.pop('f')
    a['shapedirs'] = np.asarray(a['shapedirs'])[:, :, :10]
    pd = np.asarray(a['posedirs'])
    if pd.shape[0] == 6890:                       # official layout [6890,3,207] -> [207, 20670]
        pd = pd.reshape(-1, pd.shape[-1]).T
    a['posedirs'] = pd
    a['J_regressor_extra'] = np.load(extra_path)
    return a


class SMPL:
    """``SMPL(model_path_or_assets, pose_type='body26fk', device=...)``"""

    num_verts = 6890                              # the SMPL mesh: forward returns vertices [n, num_verts, 3]

    def __init__(self, model_path=SMPL_MODEL_DIR, *args, pose_type='body26fk', device='cuda', joint_map=None, **kwargs):
        self.device = L.require_cuda(device)
        assets = model_path if isinstance(model_path, dict) else load_smpl_assets(model_path)
        if joint_map is None:
            if pose_type != 'body26fk':
                raise NotImplementedError(f"pose_type '{pose_type}': pass joint_map explicitly")
            joint_map = BODY26FK_JOINT_MAP
        self.joint_map = np.asarray(joint_map, np.int32)
        self.faces = assets.get('faces')
        self.parents = np.asarray(assets['parents'], np.int32).copy()
        f32 = lambda k: np.ascontiguousarray(np.asarray(assets[k], np.float32))
        arrs = {k: f32(k) for k in ['v_template', 'shapedirs', 'posedirs', 'J_regressor', 'lbs_weights', 'J_regressor_extra']}
        picks = np.asarray(EXTRA_VERTEX_IDS, np.int32)
        self._lib = L.load()
        self._h = ctypes.c_void_p()
        fp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        with torch.cuda.device(self.device):
            L.check(self._lib.glamr_smpl_create(ctypes.byref(self._h), fp(arrs['v_template']), fp(arrs['shapedirs']), fp(arrs['posedirs']),
                                                fp(arrs['J_regressor']), fp(arrs['lbs_weights']), fp(self.parents),
                                                fp(arrs['J_regressor_extra']), int(arrs['J_regressor_extra'].shape[0]),
                                                fp(picks), len(picks), fp(self.joint_map), len(self.joint_map)), 'glamr_smpl_create')
        self.num_joints = len(self.joint_map)
        self._ws = None

    @property
    def handle(self):
        return self._h

    def __del__(self):
        try:
            if getattr(self, '_h', None):
                self._lib.glamr_smpl_destroy(self._h)
        except Exception:
            pass

    def to(self, device):
        if torch.device(device) != self.device and torch.device(device).index not in (None, self.device.index):
            raise L.GlamrError('an SMPL handle is bound to the device it was created on')
        return self

    def _workspace(self, n, fk_only=False):
        """scratch for n frame-persons.  A buffer that is outgrown is RETIRED, not freed: captured CUDA graphs (the prior
        networks replay their launch sequence) may still hold its address."""
        need = (self._lib.glamr_smpl_fk_workspace_bytes if fk_only else self._lib.glamr_smpl_workspace_bytes)(self._h, n)
        if self._ws is None or self._ws.numel() < need:
            if self._ws is not None:
                self._ws_retired = getattr(self, '_ws_retired', []) + [self._ws]
            self._ws = torch.empty(int(need), dtype=torch.uint8, device=self.device)
        return self._ws

    def _prep(self, t, n, d):
        if t is None:
            return None
        t = torch.as_tensor(t, device=self.device).to(torch.float32)
        if t.shape[0] != n:
            t = t.expand(n, *t.shape[1:])
        return t.reshape(n, d).contiguous() if d else t.reshape(n).contiguous()

    def forward(self, betas=None, body_pose=None, global_orient=None, root_trans=None, root_scale=None, orig_joints=False,
                return_verts=True, **kwargs):
        n = body_pose.shape[0]
        bp, be = self._prep(body_pose, n, 69), self._prep(betas, n, 10)
        go, rt, rs = self._prep(global_orient, n, 3), self._prep(root_trans, n, 3), self._prep(root_scale, n, 0)
        nj = 24 if orig_joints else self.num_joints
        joints = torch.empty((n, nj, 3), dtype=torch.float32, device=self.device)
        verts = torch.empty((n, self.num_verts, 3), dtype=torch.float32, device=self.device) if return_verts else None
        ws = self._workspace(n)
        with torch.cuda.device(self.device):
            L.check(self._lib.glamr_smpl_forward(self._h, n, L.ptr(go), L.ptr(bp), L.ptr(be), L.ptr(rt), L.ptr(rs), int(orig_joints),
                                                 L.ptr(joints), L.ptr(verts), L.ptr(ws), ctypes.c_size_t(ws.numel()), L.stream_ptr()),
                    'glamr_smpl_forward')
        if go is None:
            go = torch.zeros((n, 3), dtype=torch.float32, device=self.device)
        return ModelOutput(vertices=verts, joints=joints, full_pose=torch.cat([go, bp], dim=1), betas=be, global_orient=go, body_pose=bp)

    __call__ = forward

    def get_joints(self, betas=None, body_pose=None, global_orient=None, transl=None, pose2rot=True, root_trans=None,
                   root_scale=None, dtype=torch.float32):
        if not pose2rot or transl is not None:
            raise NotImplementedError('get_joints: rotation-matrix input / transl are not implemented')
        n = body_pose.shape[0]
        bp, go = self._prep(body_pose, n, 69), self._prep(global_orient, n, 3)
        rt, rs = self._prep(root_trans, n, 3), self._prep(root_scale, n, 0)
        joints = torch.empty((n, 24, 3), dtype=torch.float32, device=self.device)
        ws = self._workspace(n, fk_only=True)
        with torch.cuda.device(self.device):
            L.check(self._lib.glamr_smpl_fk24(self._h, n, L.ptr(go), L.ptr(bp), L.ptr(rt), L.ptr(rs), L.ptr(joints), L.ptr(ws),
                                              ctypes.c_size_t(ws.numel()), L.stream_ptr()), 'glamr_smpl_fk24')
        return joints
