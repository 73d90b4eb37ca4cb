"""GPU: the VIO update on visual sub-maps drawn from many keyframes (tests/keyframe_cases.py) against the oracle, whose
outputs on these inputs are pinned to the reference source (tests/test_oracle_ref_pin_keyframes.py). Every patch has its own
inverse reference exposure, reference image and reference pose: the forward update reads inv_expo_list[i] (through the
per-warp patch cache when a CTA holds at most 32 patches, refilled every time above that), the warp producer and the
inverse-compositional precompute read reference image ref_idx[i] and the reference pose of patch i."""
import contextlib
import dataclasses

import numpy as np
import pytest

import keyframe_cases as KC
import select_cases as SC
from fast_livo2_b200 import api
from harness import VIO_KEYS, bits_equal, compare_vio, sm_count, sweep, variant

pytestmark = pytest.mark.gpu

FORWARD = ["pinhole", "pinhole_gain", "pinhole_expo_off", "pinhole_gain_expo_off", "pinhole_sorted", "pinhole_shuffled", "distorted_gain", "three_levels_mixed"]
LOOPS = [dict(loop_mode=0), dict(loop_mode=2)]


@contextlib.contextmanager
def keyframe_setup(ctx, c, inverse=False):
    """The case's camera, current image and all K reference images; the forward variant is back afterwards."""
    ctx.set_extrinsics(c["ext"])
    try:
        ctx.vio_set_camera(c["cam_cfg"], dataclasses.replace(c["vio_cfg"], inverse_composition_en=inverse))
        ctx.vio_set_image(c["img"])
        ctx.vio_set_ref_images(c["ref_imgs"])
        if inverse:
            r = c["refs"]
            ctx.vio_set_inverse_refs(r["ref_img_index"], r["ref_px"], r["ref_f"], r["ref_R"], r["ref_pos"])
        yield ctx
    finally:
        ctx.vio_set_camera(c["cam_cfg"], dataclasses.replace(c["vio_cfg"], inverse_composition_en=False))


def set_patches_run(ctx, c):
    ctx.vio_set_patches(c["vis_pos"], c["warp_patch"], c["search_levels"], c["inv_ref_expo"])
    ctx.vio_run(c["prior"], c["prior"])
    return ctx.vio_fetch()


@pytest.mark.parametrize("name", FORWARD)
def test_forward_update_matches_oracle(gpu_ctx, name):
    """vio_update, per-iteration launches and the persistent kernel: bit-identical to each other, both against the oracle."""
    c = KC.build(name)
    args = KC.update_args(c)
    with keyframe_setup(gpu_ctx, c):
        per_iter, persistent = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), LOOPS)
    bits_equal(per_iter, persistent, VIO_KEYS)
    o = KC.oracle(c).update(*args)
    assert o["total_iters"] >= 4
    for g in (per_iter, persistent):
        compare_vio(g, o, c["vio_cfg"].levels)


def test_forward_update_literal_solve_mode(gpu_ctx):
    c = KC.build("pinhole_gain")
    args = KC.update_args(c)
    with keyframe_setup(gpu_ctx, c), variant(gpu_ctx, solve_mode=1):
        g = gpu_ctx.vio_update(*args)
    compare_vio(g, KC.oracle(c).update(*args), c["vio_cfg"].levels)


@pytest.mark.parametrize("name", ["config5_4k", "config5_6k"])
def test_patch_cache(gpu_ctx, name):
    """Config 5's camera, 5 levels, mixed search levels: two patches per warp held in the per-warp cache (4 k), and more
    patches than 2 x 16 warps x SMs (6 k by replication), where slot 0 is refilled for every patch. Per-iteration launches,
    the persistent kernel and its TMA tap staging bit for bit, and against the oracle."""
    c = KC.build(name)
    n, resident = len(c["vis_pos"]), 2 * 16 * min(sm_count(), 160)
    assert (resident // 2 < n <= resident) if name == "config5_4k" else (n > resident), (n, resident)
    assert len(np.unique(c["search_levels"])) >= 2
    args = KC.update_args(c)
    with keyframe_setup(gpu_ctx, c):
        runs = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), LOOPS + [dict(loop_mode=2, tuning=api.TUNE_VIO_TMA)])
    for r in runs[1:]:
        bits_equal(runs[0], r, VIO_KEYS)
    compare_vio(runs[0], KC.oracle(c).update(*args), c["vio_cfg"].levels)


@pytest.mark.parametrize("loop_mode", [0, 2])
def test_set_patches_run_equals_update(gpu_ctx, loop_mode):
    c = KC.build("pinhole_shuffled")
    args = KC.update_args(c)
    with keyframe_setup(gpu_ctx, c), variant(gpu_ctx, loop_mode=loop_mode):
        a = set_patches_run(gpu_ctx, c)
        b = gpu_ctx.vio_update(*args)
    bits_equal(a, b, VIO_KEYS)
    compare_vio(a, KC.oracle(c).update(*args), c["vio_cfg"].levels)


@pytest.mark.parametrize("normal_en", [True, False])
def test_select_then_run_matches_oracle(gpu_ctx, normal_en):
    """vio_select_patches on the keyframe candidates, then vio_run, against the oracle's selection (on the device's warp
    matrices, see test_gpu_select_patches.py) followed by the oracle's update on the patches it kept."""
    c = KC.build("pinhole_gain")
    s, L = c["select"], c["vio_cfg"].levels
    sel = lambda **kw: gpu_ctx.vio_select_patches(s["ref_idx"], s["px_ref"], s["pos_w"], s["T_ref"], s["ref_inv_expo"], s["pc"], s["T_cur"], s["inv_expo"],
                                                  normal_w=s["normal_w"], ref_level=s["ref_level"], ref_f=s["ref_f"], ref_pos=s["ref_pos"], ref_key=s["ref_key"],
                                                  normal_en=normal_en, **kw)
    with keyframe_setup(gpu_ctx, c):
        every = sel(outlier_threshold=1e30)
        thr = float(np.quantile(every["errors"], 0.8)) / 64
        want = SC.OracleSelect(c["cam_cfg"], levels=L).select(s, normal_en=normal_en, outlier_threshold=thr, A_in=every["A_cur_ref"], sl_in=every["search_levels"])
        got = sel(outlier_threshold=thr, want_patches=True)
        gpu_ctx.vio_run(c["prior"], c["prior"])
        g = gpu_ctx.vio_fetch()
    k = want["kept"]
    assert np.array_equal(got["kept"], k) and 0.6 * len(s["pc"]) < len(k) < len(s["pc"])
    assert np.array_equal(got["warp_patch"], want["warp_patch"][k])
    assert len(np.unique(c["ref_idx"][k])) == c["K"]
    o = KC.oracle(c).update(c["img"], c["vis_pos"][k], want["warp_patch"][k], want["search_levels"][k], c["inv_ref_expo"][k], c["prior"], c["prior"])
    assert o["total_iters"] >= 4
    compare_vio(g, o, L)


@pytest.mark.parametrize("name", ["pinhole_gain", "distorted_gain", "pinhole_5k", "fisheye_gain"])
def test_warp_producer_with_many_reference_images(gpu_ctx, name):
    """vio_warp_patches with a reference image and pose per patch against the oracle's warps: the same search levels, A
    within 1e-10, patches at the bar of test_vio_matches_reference_source_golden, and bit for bit given the device's A."""
    c = KC.build(name)
    with keyframe_setup(gpu_ctx, c):
        w = gpu_ctx.vio_warp_patches(c["ref_idx"], c["px_ref"], c["vis_pos"], c["vis_normal"], c["T_ref"], KC.pack_T(*c["T_cur"]))
    assert np.array_equal(w["search_levels"], c["search_levels"])
    np.testing.assert_allclose(w["A_cur_ref"], c["A_cur_ref"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(w["warp_patch"], c["warp_patch"], atol=2e-3)
    assert np.mean(w["warp_patch"] == c["warp_patch"]) > 0.98
    orc = KC.oracle(c)
    for i in range(0, len(c["vis_pos"]), 7):
        assert np.array_equal(w["warp_patch"][i], orc.warp_affine(c["ref_imgs"][c["ref_idx"][i]], w["A_cur_ref"][i], c["px_ref"][i], w["search_levels"][i])), i


@pytest.mark.parametrize("name", ["pinhole_gain", "distorted_gain", "pinhole_5k"])
def test_inverse_variant_matches_oracle(gpu_ctx, name):
    """Inverse-compositional update with 12 reference images and per-patch ref_R / ref_pos / ref_f (pinhole_5k: more than 32
    patches per CTA): vio_update under both loop modes and set_patches + vio_run, bit for bit, against the oracle."""
    c = KC.build(name)
    args = KC.update_args(c)
    with keyframe_setup(gpu_ctx, c, inverse=True):
        per_iter, persistent = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), LOOPS)
        run = set_patches_run(gpu_ctx, c)
    bits_equal(per_iter, persistent, VIO_KEYS)
    bits_equal(persistent, run, VIO_KEYS)
    o = KC.oracle(c, inverse=True).update(*args)
    assert o["total_iters"] >= 4
    for g in (per_iter, persistent):
        compare_vio(g, o, c["vio_cfg"].levels)


def test_fisheye_forward_update(gpu_ctx):
    """Config 3's camera and extrinsics with per-patch exposures, reference images and poses (no reference pin for fisheye:
    against the oracle only, as test_vio_fisheye_camera)."""
    c = KC.build("fisheye_gain")
    args = KC.update_args(c)
    with keyframe_setup(gpu_ctx, c):
        per_iter, persistent = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), LOOPS)
    bits_equal(per_iter, persistent, VIO_KEYS)
    compare_vio(persistent, KC.oracle(c).update(*args), c["vio_cfg"].levels)


def test_reference_index_out_of_range_is_an_argument_error(gpu_ctx):
    """vio_warp_patches and vio_set_inverse_refs with a reference index outside the registered images fail with
    ESIKF_ERR_ARG and leave the installed sub-map (and the inverse refs) as they were."""
    c = KC.build("pinhole_gain")
    r, n, K = c["refs"], len(c["vis_pos"]), c["K"]
    with keyframe_setup(gpu_ctx, c, inverse=True):
        before = set_patches_run(gpu_ctx, c)
        for bad in (K, K + 7, -1):
            idx = c["ref_idx"].copy()
            idx[n // 2] = bad
            with pytest.raises(api.EsikfError, match="status -3"):
                gpu_ctx.vio_warp_patches(idx, c["px_ref"], c["vis_pos"], c["vis_normal"], c["T_ref"], KC.pack_T(*c["T_cur"]), keep_on_device=True)
            with pytest.raises(api.EsikfError, match="status -3"):
                gpu_ctx.vio_set_inverse_refs(idx, r["ref_px"], r["ref_f"], r["ref_R"], r["ref_pos"])
        gpu_ctx.vio_run(c["prior"], c["prior"])
        after = gpu_ctx.vio_fetch()
    bits_equal(before, after, VIO_KEYS)


def test_fewer_reference_images_invalidate_the_inverse_refs(gpu_ctx):
    """Registering fewer reference images drops the inverse refs (their indices may point past the new images): vio_run then
    fails with ESIKF_ERR_STATE instead of reading them; registering the images and refs again restores the result."""
    c = KC.build("pinhole_gain")
    r = c["refs"]
    with keyframe_setup(gpu_ctx, c, inverse=True):
        ok = set_patches_run(gpu_ctx, c)
        gpu_ctx.vio_set_ref_images(c["ref_imgs"][:2])
        with pytest.raises(api.EsikfError, match="status -4"):
            gpu_ctx.vio_run(c["prior"], c["prior"])
        gpu_ctx.vio_set_ref_images(c["ref_imgs"])
        with pytest.raises(api.EsikfError, match="status -4"):  # the same images again: the refs still have to be set again
            gpu_ctx.vio_run(c["prior"], c["prior"])
        gpu_ctx.vio_set_inverse_refs(r["ref_img_index"], r["ref_px"], r["ref_f"], r["ref_R"], r["ref_pos"])
        gpu_ctx.vio_run(c["prior"], c["prior"])
        again = gpu_ctx.vio_fetch()
    bits_equal(ok, again, VIO_KEYS)
