"""GPU parity of the inverse-compositional VIO variant (vio/inverse_composition_en, src/vio.cpp:792-795, 1327-1518) against
the oracle and the golden vectors."""
import dataclasses
import os

import numpy as np
import pytest

import oracle_bind as O
from harness import VIO_KEYS, bits_equal, compare_vio, sweep, vio_prior, vio_setup, vio_warp

pytestmark = pytest.mark.gpu


def test_inverse_variant_matches_oracle(gpu_ctx, small_vio_frame):
    fr = small_vio_frame
    inv_cfg = dataclasses.replace(fr["vio_cfg"], inverse_composition_en=True)
    refs = O.inverse_refs_from_frame(fr)
    prior = vio_prior(fr)
    try:
        vio_setup(gpu_ctx, fr)
        w = vio_warp(gpu_ctx, fr, prior)
        gpu_ctx.vio_set_camera(fr["cam_cfg"], inv_cfg)
        gpu_ctx.vio_set_inverse_refs(refs["ref_img_index"], refs["ref_px"], refs["ref_f"], refs["ref_R"], refs["ref_pos"])
        n = len(fr["vis_pos"])
        args = (fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], np.ones(n), prior, prior)
        g = gpu_ctx.vio_update(*args)
        g2 = gpu_ctx.vio_update(*args)
    finally:
        gpu_ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    vio.set_inverse_refs(**refs)
    vio.set_inverse(True)
    o = vio.update(*args)
    assert np.array_equal(g["state"], g2["state"])  # deterministic
    compare_vio(g, o, fr["vio_cfg"].levels)
    # the forward variant is back after restoring the configuration
    f = gpu_ctx.vio_update(*args)
    vio.set_inverse(False)
    compare_vio(f, vio.update(*args), fr["vio_cfg"].levels)


def test_inverse_variant_needs_its_reference_data(gpu_ctx, small_vio_frame):
    from fast_livo2_b200 import api

    fr = small_vio_frame
    inv_cfg = dataclasses.replace(fr["vio_cfg"], inverse_composition_en=True)
    prior = vio_prior(fr)
    try:
        vio_setup(gpu_ctx, fr)
        w = vio_warp(gpu_ctx, fr, prior)
        gpu_ctx.vio_set_camera(fr["cam_cfg"], inv_cfg)
        gpu_ctx.vio_set_inverse_refs(np.zeros(3, np.int32), np.zeros((3, 2)), np.zeros((3, 3)), np.zeros((3, 9)), np.zeros((3, 3)))
        with pytest.raises(api.EsikfError):
            gpu_ctx.vio_update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], np.ones(len(fr["vis_pos"])), prior, prior)
    finally:
        gpu_ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])


def test_inverse_variant_matches_golden_vectors(gpu_ctx):
    """tests/golden/esikf_golden_inverse.npz: the CUDA path without the oracle in the loop."""
    from parity_util import GOLDEN_DIR, assert_state_close, load_golden

    g, lio_cfg, vio_cfg, cam, ext, vmap = load_golden()
    gi = np.load(os.path.join(GOLDEN_DIR, "esikf_golden_inverse.npz"))
    n = len(g["vis_pos"])
    try:
        gpu_ctx.set_extrinsics(ext)
        gpu_ctx.vio_set_camera(cam, dataclasses.replace(vio_cfg, inverse_composition_en=True))
        gpu_ctx.vio_set_ref_images([g["img_ref"]])
        gpu_ctx.vio_set_inverse_refs(gi["ref_img_index"], gi["ref_px"], gi["ref_f"], gi["ref_R"], gi["ref_pos"])
        v = gpu_ctx.vio_update(g["img"], g["vis_pos"], g["warp_patch"], g["search_levels"], np.ones(n), g["lio_state"], g["lio_state"])
    finally:
        gpu_ctx.vio_set_camera(cam, vio_cfg)
    assert v["total_iters"] == int(gi["vio_total_iters"]) and np.array_equal(v["iters_per_level"], gi["vio_iters_per_level"])
    assert np.array_equal(v["accepted_per_level"], gi["vio_accepted_per_level"])
    assert_state_close(v["state"], gi["vio_state"], rot_tol=1e-8, pos_tol=1e-8, cov_tol=1e-6, rest_tol=1e-8)
    np.testing.assert_allclose(v["errors"], gi["vio_errors"], rtol=2e-6, atol=1e-3)


def test_inverse_variant_persistent_kernel_is_bit_identical_to_per_iteration_launches(gpu_ctx, small_vio_frame):
    """loop_mode 2 runs the inverse-compositional loop inside the same persistent kernel as the forward variant
    (vio_update_kernel<.., INVERSE>: H_sub_inv of a level precomputed by the warp that later reads it); it must reproduce
    the per-iteration launches (loop_mode 0: precompute kernel + patch kernel + solve kernel) bit for bit."""
    fr = small_vio_frame
    inv_cfg = dataclasses.replace(fr["vio_cfg"], inverse_composition_en=True)
    refs = O.inverse_refs_from_frame(fr)
    prior = vio_prior(fr)
    try:
        vio_setup(gpu_ctx, fr)
        w = vio_warp(gpu_ctx, fr, prior)
        gpu_ctx.vio_set_camera(fr["cam_cfg"], inv_cfg)
        gpu_ctx.vio_set_inverse_refs(refs["ref_img_index"], refs["ref_px"], refs["ref_f"], refs["ref_R"], refs["ref_pos"])
        n = len(fr["vis_pos"])
        args = (fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], np.ones(n), prior, prior)
        runs = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), [dict(loop_mode=m) for m in (0, 2, 2, 0)])
    finally:
        gpu_ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])
    ref = runs[0]
    assert ref["total_iters"] >= 3
    for r in runs[1:]:
        assert r["total_iters"] == ref["total_iters"]
        bits_equal(ref, r, VIO_KEYS)
