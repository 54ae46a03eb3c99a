"""Generate tests/golden/trajpred_multistep.npz by EXECUTING THE UNMODIFIED REFERENCE through the import shims of oracle/refshim,
like make_golden.py's nets_vectors, with multi_step_trajpred set on the reference's MotionTrajJointModel:

    python tests/golden/make_trajpred_multistep_golden.py       # writes tests/golden/trajpred_multistep.npz

The networks carry the seeded stand-in weights of glamr_b200.synthetic_nets.  The inputs are regenerated from seeds by
tests/trajpred_multistep_cases.case_batch; the infiller's latents are injected as in nets_vectors.  The trajectory predictor's
windows cannot be given latents (TrajPredVAE.get_seg_data copies only the `tp` keys into a window), so each window's eps is drawn
from a seeded generator by a wrapper around lib.utils.dist.Normal.rsample and stored as `in_traj_window_latent` [windows, B, 128].
`in_traj_latent` is passed too and must have no effect.  Stored per case: the window eps and the trajectory outputs (the
infilled body pose is pinned by nets.npz already).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), 'tests'))

from make_golden import ref_env  # noqa: E402,F401  (activates the reference tree)
import torch  # noqa: E402

from trajpred_multistep_cases import CASES, WINDOW, case_batch  # noqa: E402

OUT_KEYS = ['infer_out_local_traj_tp', 'infer_out_orient', 'infer_out_trans']


def vectors():
    from motion_infiller.models.motion_traj_joint_model import MotionTrajJointModel
    from motion_infiller.utils.config_motion_traj import Config as MTConfig
    import lib.utils.dist as dist
    from glamr_b200.synthetic_nets import make_prior_states
    mt = MotionTrajJointModel(MTConfig('joint_motion_traj_demo'), torch.device('cpu'), None)
    mt.multi_step_trajpred = True
    assert mt.traj_predictor.seq_len == WINDOW
    st_m, st_t = make_prior_states(1234)
    for mod, st in [(mt.mfiller, st_m), (mt.traj_predictor, st_t)]:
        res = mod.load_state_dict({k: torch.tensor(v) for k, v in st.items()}, strict=False)
        assert not res.unexpected_keys
    drawn, gen = [], torch.Generator()
    orig = dist.Normal.rsample

    def rsample(self, eps=None):
        if eps is None:
            eps = torch.randn(self.sigma.shape, generator=gen, dtype=self.sigma.dtype)
            drawn.append(eps.clone())
        return orig(self, eps)

    dist.Normal.rsample = rsample
    out = {}
    try:
        for tag, B, T, _ in CASES:
            gen.manual_seed(1000 + T + B)
            drawn.clear()
            batch = case_batch(tag)
            with torch.no_grad():
                res = mt.inference({k: v.clone() for k, v in batch.items()}, sample_num=1)
            C = int(np.ceil(T / WINDOW))
            assert len(drawn) == C and all(tuple(e.shape) == (B, 128) for e in drawn), (tag, [tuple(e.shape) for e in drawn])
            out[f'{tag}/in/in_traj_window_latent'] = torch.stack(drawn).numpy()
            for k in OUT_KEYS:
                out[f'{tag}/{k}'] = res[k].detach().numpy()
            print(tag, 'windows', C)
    finally:
        dist.Normal.rsample = orig
    return out


if __name__ == '__main__':
    np.savez_compressed(os.path.join(HERE, 'trajpred_multistep.npz'), **vectors())
