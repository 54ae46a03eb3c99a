"""v_posed of the tensor-core blend GEMM, bit for bit, at the edges of its staged epilogue.

lbs_blend_tc_kernel stages each warpgroup's 64 frames x 32 columns of the accumulator in shared memory and stores them as 16-byte
pieces of 4 consecutive frames, ordered by where they land in v_posed: frame-tiled [frame / 20][column][20] for the tensor-core
skinning, [column][mpad] for the SIMT skinning ("tcblend").  Every element is still the accumulator times its row's unscale factor.

The digests in golden/blend_vposed_sha256.json were recorded on an H100 with the epilogue that stored every element straight from its
accumulator register (scalar stores, no staging); make_blend_vposed_hashes.py rewrites them.  The sizes put a frame-tile edge, a half
last tile (at most 64 frames in the last 128-frame tile) or a 20-frame group across a 64- or 128-frame boundary in every place the
piece order changes.  The same n must also give the same bits in both layouts: only the store order differs between them.
"""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from test_gpu_parity import LBS_PATHS, _default_lbs_path
from test_lbs_float64 import _dev, make_inputs
from test_skin_support_tiles import TC_COLS, forward_keep_workspace, workspace_views

DEV = 'cuda:0'
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'blend_vposed_sha256.json')
SIZES = [1, 4, 5, 60, 63, 64, 65, 124, 127, 128, 129, 192, 200, 300, 1200]
LAYOUTS = {'tiled': 'tensor_core', 'tcblend': 'tensor_core_blend_simt_skin'}


def v_posed(smpl, n, layout):
    """v_posed [n, columns] (frame-major) of one glamr_smpl_forward on a NaN-filled workspace; tcblend writes the mesh columns only"""
    from glamr_b200 import lib as L
    lib = L.load()
    L.check(lib.glamr_smpl_set_lbs_path(LBS_PATHS[LAYOUTS[layout]]), 'set_lbs_path')
    try:
        _, ws = forward_keep_workspace(smpl, _dev(make_inputs(n, 7000 + n)), n)
    finally:
        L.check(lib.glamr_smpl_set_lbs_path(_default_lbs_path()), 'set_lbs_path')
    S = int(lib.glamr_smpl_info(smpl.handle, 1))
    _, tiled = workspace_views(ws, n, S)
    if layout == 'tiled':
        return tiled.permute(0, 2, 1).reshape(-1, tiled.shape[1])[:n]
    vp_cols, mpad, o = tiled.shape[1], (n + 127) // 128 * 128, tiled.storage_offset()
    return ws[o:o + vp_cols * mpad].view(vp_cols, mpad)[:TC_COLS, :n].t()


def digest(vp):
    return hashlib.sha256(np.ascontiguousarray(vp.cpu().numpy()).tobytes()).hexdigest()


def digests(smpl):
    """{layout: {n: sha256 of v_posed [n, columns]}} over SIZES"""
    return {layout: {str(n): digest(v_posed(smpl, n, layout)) for n in SIZES} for layout in LAYOUTS}


@pytest.fixture(scope='module')
def smpl(smpl_assets):
    from glamr_b200.smpl import SMPL
    return SMPL(smpl_assets, device=DEV)


@pytest.mark.gpu
@pytest.mark.parametrize('n', SIZES)
def test_v_posed_matches_the_unstaged_store_bitwise(n, smpl):
    with open(GOLDEN) as f:
        gold = json.load(f)
    vp = {layout: v_posed(smpl, n, layout) for layout in LAYOUTS}
    for layout, x in vp.items():
        assert not torch.isnan(x).any(), f'n={n} {layout}: an element of v_posed was not written'
        assert digest(x) == gold[layout][str(n)], f'n={n} {layout}: v_posed differs from the unstaged store'
    assert torch.equal(vp['tiled'][:, :TC_COLS], vp['tcblend']), f'n={n}: the two layouts hold different values'
