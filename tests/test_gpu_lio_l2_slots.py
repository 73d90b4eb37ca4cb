"""GPU: the LIO update with the lanes whose slots live in the L2-resident global block (warps 22 and 23 of every CTA,
lanes 704-767: csrc/esikf_lio.cu, LIO_L2_WARPS). Slice sizes at the boundaries of the 768-lane geometry, and the hand-built
association cases of tests/lio_assoc.py laid out so that every designed warp (extras of sub-divided voxels, neighbour
fallback, zero-probability passes, ties) runs in an L2-slot warp of some CTA. Every run is bit for bit against the
oracle's association and bit-identical across the persistent and the per-iteration launch forms and both record
stagings (cp.async.bulk for shared slots, __ldg copies)."""
import numpy as np
import pytest

import lio_assoc as A
from lio_assoc import LANES, SMEM_LANES
from fast_livo2_b200 import api
from harness import LIO_KEYS, bits_equal, compare_lio, lio_gpu, lio_oracle, sm_count, sweep

pytestmark = pytest.mark.gpu

VARIANTS = [dict(loop_mode=2), dict(loop_mode=0), dict(loop_mode=2, tuning=api.TUNE_STAGE_LDG), dict(loop_mode=0, tuning=api.TUNE_STAGE_LDG)]


def grid():
    return min(sm_count(), 160)  # one CTA per SM, at most 160 partial columns


def check_all_variants(ctx, fr):
    o = lio_oracle(fr)
    runs = sweep(ctx, lambda: lio_gpu(ctx, fr), VARIANTS)
    compare_lio(runs[0], o)
    for r in runs[1:]:
        bits_equal(runs[0], r, LIO_KEYS)
    return runs[0], o


@pytest.mark.parametrize("name", A.CASES)
def test_slices_at_the_768_lane_boundaries(gpu_ctx, name):
    """Both sides of the launch's choice of CTA geometry: G x 704 - 1 points (704-lane kernel, resident), G x 704 + 1 (one
    CTA gets a 23rd chunk: 768-lane kernel), every CTA one point short of 768, exactly 768, one point over (one CTA gets a
    25th chunk: 704-lane kernel, tiled), and 2.5 x G x 768 points (every CTA tiles)."""
    G = grid()
    fr = A.case(name)
    for n in (G * SMEM_LANES - 1, G * SMEM_LANES + 1, G * LANES - 1, G * LANES, G * LANES + 1, int(2.5 * G * LANES)):
        check_all_variants(gpu_ctx, A.tiled(fr, n))


@pytest.mark.parametrize("name", A.CASES)
def test_designed_warps_in_l2_slot_lanes(gpu_ctx, name):
    """Every designed warp of the case, in turn, in lanes 704-767 of some CTA: the association of those lanes against the
    oracle's, bit for bit, in every launch form and staging."""
    G = grid()
    fr = A.case(name)
    W = len(fr["pts"]) // 32
    matched_l2 = 0
    for start in range(0, W, 2 * G):
        f = A.l2_lane_layout(fr, G, start)
        g, o = check_all_variants(gpu_ctx, f)
        in_l2 = (np.arange(len(f["pts"])) % LANES) >= SMEM_LANES
        assert np.array_equal(g["match_plane"][in_l2], o["match_plane"][in_l2])
        matched_l2 += int((g["match_plane"][in_l2] >= 0).sum())
    assert matched_l2 > 0
