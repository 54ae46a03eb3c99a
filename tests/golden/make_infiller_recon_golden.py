"""Generate tests/golden/infiller_recon.npz by EXECUTING THE UNMODIFIED REFERENCE through the import shims of oracle/refshim, like
make_trajpred_multistep_golden.py:

    python tests/golden/make_infiller_recon_golden.py       # writes tests/golden/infiller_recon.npz

The reference's MotionInfillerVAE carries the seeded stand-in weights of glamr_b200.synthetic_nets, its posterior encoder those of
make_infiller_posterior_state.  The inputs are regenerated from seeds by tests/infiller_recon_cases.case_batch; stored per case are
their seed and shape and recon_out_pose / recon_out_body_pose (the infer half of the call is pinned by nets.npz).

The recon outputs come from inference_multi_step(copy, 1, recon=True) on a fresh copy of the inputs: at B = 1 with an
in_body_pose, inference(..., recon=True) runs its recon sweep from the infilled pose, because its infer sweep writes the caller's
in_body_pose through a view.  Every other case checks that the full inference call gives the same outputs.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), 'tests'))

from make_golden import ref_env  # noqa: E402,F401  (activates the reference tree)
import torch  # noqa: E402

from infiller_recon_cases import CASES, case_batch, case_seed, infiller_state  # noqa: E402

OUT_KEYS = ['recon_out_pose', 'recon_out_body_pose']


def vectors():
    from motion_infiller.models.motion_traj_joint_model import MotionTrajJointModel
    from motion_infiller.utils.config_motion_traj import Config as MTConfig
    mt = MotionTrajJointModel(MTConfig('joint_motion_traj_demo'), torch.device('cpu'), None)
    mf = mt.mfiller
    st = infiller_state()
    own = mf.state_dict()
    assert all(k in own and tuple(own[k].shape) == v.shape for k, v in st.items()), 'state-dict names/shapes differ from the reference'
    missing = [k for k in own if k.startswith(('context_encoder.', 'data_encoder.', 'data_decoder.')) and k not in st]
    assert not missing, missing
    res = mf.load_state_dict({k: torch.tensor(v) for k, v in st.items()}, strict=False)
    assert not res.unexpected_keys
    out = {}
    for tag, B, T, _, ibp in CASES:
        batch = case_batch(tag)
        with torch.no_grad():
            rec = mf.inference_multi_step({k: v.clone() for k, v in batch.items()}, 1, recon=True)
            if not (B == 1 and ibp):
                full = mf.inference({k: v.clone() for k, v in batch.items()}, sample_num=1, recon=True, multi_step=True)
                for k in OUT_KEYS:
                    assert torch.equal(full[k], rec[k]), (tag, k)
        out[f'{tag}/seed'] = np.array(case_seed(tag), dtype=np.int64)
        out[f'{tag}/shape'] = np.array([B, T], dtype=np.int64)
        for k in OUT_KEYS:
            assert tuple(rec[k].shape) == (B, T, 72 if k == 'recon_out_pose' else 69), (tag, k, tuple(rec[k].shape))
            out[f'{tag}/{k}'] = rec[k].detach().numpy()
        print(tag, 'windows', int(np.ceil((T - 10) / 30)))
    return out


if __name__ == '__main__':
    np.savez_compressed(os.path.join(HERE, 'infiller_recon.npz'), **vectors())
