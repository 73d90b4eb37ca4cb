"""GPU: the persistent kernels (loop_mode 2, the default: the whole iteration loop in one cooperative launch, state and
per-point / per-patch invariants resident on chip, gain solve replicated in every CTA) must reproduce the per-iteration
launch path (loop_mode 0: nothing cached, every launch starts cold) bit for bit — states, associations and per-iteration
diagnostics — in both solve modes, across repeated launches (barrier counters and partial buffers alternate), for both
ways of staging the plane records (cp.async.bulk per lane / coalesced __ldg copies)."""
import numpy as np
import pytest

from conftest import get_frame
from fast_livo2_b200 import api
from harness import LIO_KEYS, VIO_KEYS, bits_equal, sweep, vio_prior, vio_setup, vio_warp

pytestmark = pytest.mark.gpu

@pytest.mark.parametrize("solve_mode", [0, 1])
def test_lio_persistent_kernel_is_bit_identical_to_per_iteration_launches(gpu_ctx, solve_mode):
    fr = get_frame(seed=4, n_pts=20000, n_map=150_000, scene_scale=0.5)
    gpu_ctx.set_extrinsics(fr["ext"])
    gpu_ctx.map_upload(fr["map"], fr["lio_cfg"].voxel_size)
    runs = sweep(gpu_ctx, lambda: gpu_ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], fr["lio_cfg"]),
                 [dict(loop_mode=m, solve_mode=solve_mode) for m in (0, 2, 2, 0, 2)])
    ref = runs[0]
    assert ref["iters"] >= 3
    for r in runs[1:]:
        assert r["iters"] == ref["iters"]
        bits_equal(ref, r, LIO_KEYS)


@pytest.mark.parametrize("n_pts,n_map,kw", [(100_000, 1_000_000, {}), (260_000, 1_000_000, dict(beam_err=0.01))])
def test_lio_full_size_frames_resident_and_several_tiles_per_cta(gpu_ctx, n_pts, n_map, kw):
    """100 k points: one tile per CTA, everything resident. 260 k points: every CTA walks several tiles, nothing stays
    resident in the lanes' slots. Both against the cold per-iteration path and for both staging variants."""
    from fast_livo2_b200 import synthetic as S

    fr = get_frame(seed=12 if n_pts > 100_000 else 0, n_pts=n_pts, n_map=n_map, **(dict(lio=S.LioCfg(**kw)) if kw else dict(n_patches=2000)))
    gpu_ctx.set_extrinsics(fr["ext"])
    gpu_ctx.map_upload(fr["map"], fr["lio_cfg"].voxel_size)
    a, b, c = sweep(gpu_ctx, lambda: gpu_ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], fr["lio_cfg"]),
                    [dict(loop_mode=0), dict(loop_mode=2), dict(loop_mode=2, tuning=api.TUNE_STAGE_LDG)])
    assert a["iters"] == b["iters"] == c["iters"]
    bits_equal(a, b, LIO_KEYS)
    bits_equal(a, c, LIO_KEYS)


@pytest.mark.parametrize("solve_mode", [0, 1])
def test_vio_persistent_kernel_is_bit_identical_to_per_iteration_launches(gpu_ctx, small_vio_frame, solve_mode):
    fr = small_vio_frame
    vio_setup(gpu_ctx, fr)
    prior = vio_prior(fr)
    w = vio_warp(gpu_ctx, fr, prior)
    args = (fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    runs = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), [dict(loop_mode=m, solve_mode=solve_mode) for m in (0, 2, 2, 0, 2)])
    ref = runs[0]
    assert ref["total_iters"] >= 4
    for r in runs[1:]:
        assert r["total_iters"] == ref["total_iters"]
        bits_equal(ref, r, VIO_KEYS)


def test_vio_tap_footprints_through_tma_are_bit_identical(gpu_ctx):
    """ESIKF_TUNE_VIO_TMA: the 11 x 11 tap footprint arrives by one tiled TMA load (cp.async.bulk.tensor.2d, elementStrides
    {1, s}) instead of per-lane byte loads. BASELINE config-2 image (640 x 512, pitch a multiple of 16) with search levels
    0 / 1 / 2 so that every tap stride up to 8 goes through the tensor maps and strides 16 / 32 fall back."""
    fr = get_frame(seed=0, n_pts=100_000, n_map=1_000_000, n_patches=2000)
    vio_setup(gpu_ctx, fr)
    prior = vio_prior(fr)
    w = vio_warp(gpu_ctx, fr, prior)
    n = len(fr["vis_pos"])
    out = []
    for sl in (w["search_levels"], (np.arange(n) % 3).astype(np.int32)):
        args = (fr["img"], fr["vis_pos"], w["warp_patch"], sl, fr["inv_ref_expo"], prior, prior)
        out.append(sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), [dict(), dict(tuning=api.TUNE_VIO_TMA), dict(tuning=api.TUNE_VIO_TMA)]))
    for a, b, b2 in out:
        assert a["total_iters"] == b["total_iters"] == b2["total_iters"] and a["total_iters"] >= 4
        bits_equal(a, b, VIO_KEYS)
        bits_equal(a, b2, VIO_KEYS)
