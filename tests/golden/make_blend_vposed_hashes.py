"""Rewrite blend_vposed_sha256.json (tests/test_blend_vposed_bitwise.py) from the library that is loaded, on an H100:

    python tests/golden/make_blend_vposed_hashes.py [OUT.json]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

if __name__ == '__main__':
    from glamr_b200.smpl import SMPL
    from glamr_b200.synthetic import make_smpl_assets
    from test_blend_vposed_bitwise import DEV, GOLDEN, digests
    out = sys.argv[1] if len(sys.argv) > 1 else GOLDEN
    with open(out, 'w') as f:
        json.dump(digests(SMPL(make_smpl_assets(0), device=DEV)), f, indent=1, sort_keys=True)
        f.write('\n')
    print('wrote', out)
