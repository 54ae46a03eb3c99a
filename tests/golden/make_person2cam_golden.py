"""Generate the fixtures of the person2cam residuals (tests/person2cam_cases.py) by EXECUTING THE UNMODIFIED REFERENCE through
the import shims of oracle/refshim, like make_traj_variable_golden.py does for heading vectors and world_dxy:

    python tests/golden/make_person2cam_golden.py [case name]     # writes tests/golden/globalopt_p2c_*.npz

Same content as make_traj_variable_golden.py's fixtures (init state, learned-prior outputs, per-iteration residuals, iteration-0
gradients, final state, the float64 continuation and the one-rounding perturbation run by the oracle), with the final
person2cam_res_rot / person2cam_res_trans.  The oracle (oracle/global_opt.py) already restates the residuals' creation, forward
and get_parameter, so the continuations pin it too.  For a case of person2cam_cases.FAILING_CASES the fixture records the error
the reference raises (and the iteration it raised in) instead of a trajectory.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(REPO, 'tests'))

import make_traj_variable_golden as mtv  # noqa: E402  (activates the reference tree)
import person2cam_cases as pc  # noqa: E402

from glamr_b200.synthetic import make_smpl_assets  # noqa: E402


def main(only=None):
    # the traj-variable generator's recording run, on this file's cases, inputs, oracle and final variables
    mtv.make_case_in_dict, mtv.oracle_class, mtv.COMPACT = pc.make_case_in_dict, pc.oracle_class, pc.COMPACT
    mtv.PERSON_KEYS = mtv.FINAL_KEYS + [k for k in pc.FINAL_VARS if k not in mtv.FINAL_KEYS]
    assets = make_smpl_assets(0)
    for case, failing in [(c, False) for c in pc.PERSON2CAM_CASES] + [(c, True) for c in pc.FAILING_CASES]:
        if only is None or case[0] == only:
            rec = mtv.traj_variable_case(assets, *case, failing=failing)
            np.savez_compressed(os.path.join(HERE, f'globalopt_{case[0]}.npz'), **rec)
            print('wrote', case[0], len(rec), 'arrays')


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else None)
