"""GPU: the VIO kernels where patch footprints reach the image border.

Four device paths decide what a footprint at the border reads: tap() (linear addressing, 0 outside [0, w·h)), the guard that
lets a footprint go through the TMA unit (TMA zero-fills outside the image, the per-lane loads wrap to the neighbouring
row), the per-warp footprint cache of the persistent kernel (keyed on the linear index of the footprint's first tap) and
warp_affine_kernel's in-frame test. Every test below places patches there (tests/vio_border.py) and asserts how many
footprints actually leave the image, so the border cases cannot silently disappear."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import oracle_bind as O
import shim_bind as SB
import vio_border as VB
from conftest import get_frame
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from harness import VIO_KEYS, bits_equal, compare_vio, sm_count, sweep, vio_prior, vio_setup
from ref_pin_cases import BORDER_FRAME, warp_affine_border_cases

pytestmark = pytest.mark.gpu
FISHEYE = dict(seed=9, n_pts=1000, n_map=100_000, n_patches=100, scene_scale=0.5, vio=S.VioCfg(img_point_cov=1000.0), ext=S.hilti_extrinsics(),
               cam=S.CamCfg(model=1, width=720, height=540, fx=351.31400364193297, fy=351.4911744656785, cx=367.8522793375995, cy=253.8402144980996,
                            d=(-0.03696737352869157, -0.008917880497032812, 0.008912969593422046, -0.0037685977496087313, 0.0)))


@pytest.fixture(scope="module")
def border():
    fr = get_frame(**BORDER_FRAME)
    prior = vio_prior(fr)
    return fr, prior, VB.border_patch_set(fr, prior)


def _args(fr, bs, prior, idx=None):
    idx = np.arange(len(bs["vis_pos"])) if idx is None else idx
    return (fr["img"], bs["vis_pos"][idx], bs["warp_patch"][idx], bs["search_levels"][idx], bs["inv_ref_expo"][idx], prior, prior)


# --------------------------------------------------------------------------------------------------------- a. getImagePatch
def test_image_patch_at_the_border_is_bit_exact(gpu_ctx, border):
    """image_patch_kernel at edge, corner and just-outside pixels, levels 0..3: reads that wrap to the neighbouring row and
    reads outside the buffer (0)."""
    fr, _, _ = border
    vio_setup(gpu_ctx, fr)
    cam, L = fr["cam_cfg"], fr["vio_cfg"].levels
    ins, outs = VB.edge_pixels(cam.width, cam.height, L, np.random.default_rng(4))
    pcs = np.concatenate([ins, outs])
    vio = O.OracleVIO(cam, fr["ext"], fr["vio_cfg"])
    wrap = beyond = 0
    for level in range(L):
        s = 1 << level
        g = gpu_ctx.vio_get_image_patch(pcs, level)
        want = np.array([vio.get_image_patch(fr["img"], pc, level) for pc in pcs])
        assert np.array_equal(g, want), level
        x0, x1, y0, y1 = VB.footprint_box(pcs, s)  # getImagePatch reads x0 + s .. x1 - s, y0 + s .. y1 - s
        wrap += int(((x0 + s < 0) | (x1 - s > cam.width - 1)).sum())
        beyond += int(((y0 + s < 0) | (y1 - s > cam.height - 1)).sum())
    assert wrap >= 60 and beyond >= 60, (wrap, beyond)


def test_shim_image_patch_and_warp_at_a_border_pixel(border):
    """VIOManager::getImagePatch / warpAffine mirrors of the shim at a corner pixel / an edge reference pixel."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    fr, _, _ = border
    shim = SB.load()
    cc, L = fr["cam_cfg"], fr["vio_cfg"].levels
    cam = api.CameraC(cc.model, cc.width, cc.height, 0, cc.fx, cc.fy, cc.cx, cc.cy)
    cam.d[:] = list(cc.d)
    vcfg = api.VioCfgC(fr["vio_cfg"].img_point_cov, L, fr["vio_cfg"].max_iterations, int(fr["vio_cfg"].exposure_estimate_en), 0)
    img, img_ref = np.ascontiguousarray(fr["img"]), np.ascontiguousarray(fr["img_ref"])
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    vio = O.OracleVIO(cc, fr["ext"], fr["vio_cfg"])
    pc = np.array([cc.width - 1.3, cc.height - 1.8])  # bottom-right corner: most reads beyond the buffer at level 3
    A = np.eye(2)
    px_ref = np.array([cc.width - 1.5, 250.0])  # samples at cols - 1.5 (inside) and cols - 0.5 (outside)
    level, search_level = 3, 0
    patch, warp = np.full(64 * L, -7.0, np.float32), np.full(64 * L, -7.0, np.float32)
    rc = shim.fl2_shim_patch_helpers(C.byref(cam), C.byref(vcfg), vp(img), img.shape[1], img.shape[0], vp(pc), level, vp(patch), vp(A), vp(img_ref), vp(px_ref),
                                     search_level, 0, vp(warp))
    assert rc == 0
    assert np.array_equal(patch[64 * level:64 * level + 64], vio.get_image_patch(img, pc, level))
    w = warp[:64]
    assert np.array_equal(w, vio.warp_affine(img_ref, A, px_ref, search_level)[:64])
    assert (w == 0).any() and (w != 0).any()


# --------------------------------------------------------------------------------------------------------- b. warp producers
def test_warp_affine_across_and_on_the_in_frame_limits(gpu_ctx, border):
    """warp_affine_kernel with caller matrices whose samples fall across and exactly on 0 / cols-1 / rows-1, search levels
    0..2, plus singular matrices (zero: NaN inverse, patch untouched; non-zero: inf entries, NaN and inf sample positions
    count as outside): bit for bit against the oracle."""
    fr, _, _ = border
    vio_setup(gpu_ctx, fr)
    cam = fr["cam_cfg"]
    cases = warp_affine_border_cases(cam.width, cam.height)
    for sl in range(3):
        cases.append((np.array([[1.0, 2.0], [2.0, 4.0]]), np.array([cam.width - 4.0, 200.0]), sl))
        cases.append((np.array([[2.0, 1.0], [4.0, 2.0]]), np.array([300.0, 250.0]), sl))
    A = np.array([c[0] for c in cases])
    px = np.array([c[1] for c in cases])
    sl = np.array([c[2] for c in cases], np.int32)
    out = gpu_ctx.vio_warp_affine(np.zeros(len(cases), np.int32), px, A, sl)
    vio = O.OracleVIO(cam, fr["ext"], fr["vio_cfg"])
    for i, (a, p, s) in enumerate(cases):
        assert np.array_equal(out[i], vio.warp_affine(fr["img_ref"], a, p, s)), i
    mixed = sum(bool((o == 0).any() and (o != 0).any()) for o in out)
    assert mixed >= len(cases) // 3, mixed


def test_warp_patches_with_px_ref_near_the_border(gpu_ctx, border):
    """warp_matrix_kernel + warp_affine_kernel on the border set (reference pixels near and beyond the reference image's
    edges): A to 1e-10, identical search levels, warp samples as in test_gpu_vio."""
    fr, prior, bs = border
    vio_setup(gpu_ctx, fr)
    n = len(bs["vis_pos"])
    st = S.unpack_state(prior)
    T_cur = S.camera_pose(fr["ext"], st["R"], st["p"])
    g = gpu_ctx.vio_warp_patches(np.zeros(n, np.int32), bs["px_ref"], bs["vis_pos"], bs["vis_normal"], np.tile(api.pack_T(*fr["T_ref"]), (n, 1)), api.pack_T(*T_cur))
    o = O.oracle_warp_patches(dict(fr, vis_pos=bs["vis_pos"], vis_normal=bs["vis_normal"], px_ref=bs["px_ref"]), prior)
    np.testing.assert_allclose(g["A_cur_ref"], o["A_cur_ref"], rtol=1e-10, atol=1e-12)
    assert np.array_equal(g["search_levels"], o["search_levels"])
    np.testing.assert_allclose(g["warp_patch"], o["warp_patch"], atol=2e-3)
    assert np.mean(g["warp_patch"] == o["warp_patch"]) > 0.98
    cam = fr["cam_cfg"]
    pr = bs["px_ref"][bs["border"]]
    near = (pr[:, 0] < 40) | (pr[:, 0] > cam.width - 41) | (pr[:, 1] < 40) | (pr[:, 1] > cam.height - 41)
    assert near.sum() >= 30, near.sum()
    assert (g["warp_patch"][bs["border"]] == 0).any()  # samples rejected by the in-frame test


# --------------------------------------------------------------------------------------------------------- c. the update
def test_vio_update_on_the_border_set_matches_oracle(gpu_ctx, border):
    fr, prior, bs = border
    assert bs["n_leave"] >= 60 and 0.2 <= bs["border"].mean() <= 0.3, (bs["n_leave"], bs["border"].mean())
    vio_setup(gpu_ctx, fr)
    args = _args(fr, bs, prior)
    g = gpu_ctx.vio_update(*args)
    o = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args)
    assert o["total_iters"] >= 4 and (o["accepted_per_level"] < o["iters_per_level"]).any()  # real accept / rollback decisions
    compare_vio(g, o, fr["vio_cfg"].levels)


@pytest.mark.parametrize("solve_mode", [0, 1])
def test_vio_update_on_the_border_set_loop_modes_are_bit_identical(gpu_ctx, border, solve_mode):
    fr, prior, bs = border
    vio_setup(gpu_ctx, fr)
    args = _args(fr, bs, prior)
    a, b, b2 = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), [dict(loop_mode=m, solve_mode=solve_mode) for m in (0, 2, 2)])
    assert a["total_iters"] >= 4
    bits_equal(a, b, VIO_KEYS)
    bits_equal(a, b2, VIO_KEYS)
    if solve_mode == 1:
        compare_vio(b, O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args), fr["vio_cfg"].levels)


@pytest.mark.parametrize("regime", ["all_cached", "at_limit", "over_limit"])
def test_vio_patch_cache_regimes_with_border_footprints(gpu_ctx, border, regime):
    """The persistent kernel caches a CTA's patches when it owns at most VIO_WARPS x VIO_KMAX = 32 of them. With
    grid = min(ceil(n / 16), min(SMs, 160)) CTAs of per = ceil(n / grid) patches: per <= 32 (every CTA cached), = 32 (the
    limit) and = 33 (slot 0 refilled for every patch). Against the cold per-iteration launches, bit for bit."""
    fr, prior, bs = border
    vio_setup(gpu_ctx, fr)
    G = min(sm_count(), 160)
    n = {"all_cached": len(bs["vis_pos"]), "at_limit": 32 * G, "over_limit": 32 * G + 1}[regime]
    grid = min(-(-n // 16), G)
    per = -(-n // grid)
    assert (per <= 32) if regime == "all_cached" else per == (32 if regime == "at_limit" else 33), (n, grid, per)
    # the border patches first so that every CTA holds some
    order = np.concatenate([np.nonzero(bs["border"])[0], np.nonzero(~bs["border"])[0]])
    idx = order[np.arange(n) % len(order)]
    args = _args(fr, bs, prior, idx)
    a, b = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), [dict(loop_mode=0), dict(loop_mode=2)])
    assert a["total_iters"] >= 4
    bits_equal(a, b, VIO_KEYS)


# --------------------------------------------------------------------------------------------------------- d. TMA guard
def _tma_targets(width, height, s, rng):
    """Prior projections whose stride-s footprint (first tap x0 = floor(u/s)*s - 5s, likewise y0) starts at x0 in {0, the
    largest multiple of s <= 15, 16}, ends exactly at the guard (x0 + 10s = the last in-image multiple of s) and one stride
    beyond each; the same for rows."""
    mid_v, mid_u = lambda: rng.uniform(0.3 * height, 0.7 * height), lambda: rng.uniform(0.3 * width, 0.7 * width)
    xs = [0, s * (15 // s), 16, -s, width - s - 10 * s, width - 10 * s]
    ys = [0, -s, height - s - 10 * s, height - 10 * s]
    at = lambda x0: x0 + 5 * s + 0.41 * s  # a pixel whose anchor floor(u/s)*s is x0 + 5s
    return np.array([(at(x0), mid_v()) for x0 in xs] + [(mid_u(), at(y0)) for y0 in ys]), np.array(xs + [None] * len(ys), object), np.array([None] * len(xs) + ys, object)


@pytest.mark.parametrize("stride", [1, 2, 4, 8])
def test_tma_footprints_at_the_guard_are_bit_identical_to_per_lane_loads(gpu_ctx, border, stride):
    """ESIKF_TUNE_VIO_TMA against the per-lane loads on the 640-wide image. The coarsest level's first iteration runs at the
    prior, so with levels = log2(stride) + 1 and search level 0 its footprints are exactly where they were placed: at the
    TMA guard and one stride beyond it (x0 + 10s = W would be zero-filled by TMA but wraps to the next row per lane)."""
    fr, prior, _ = border
    cam = fr["cam_cfg"]
    assert cam.width % 16 == 0
    L = stride.bit_length()
    vcfg = dataclasses.replace(fr["vio_cfg"], levels=L)
    px, xs, ys = _tma_targets(cam.width, cam.height, stride, np.random.default_rng(stride))
    extra = VB.patches_at(fr, prior, px, np.zeros(len(px), np.int32))
    bs = VB.with_interior(fr, prior, extra)
    bs["warp_patch"] = np.ascontiguousarray(bs["warp_patch"][:, :64 * L])
    # the first tap of each placed footprint, from the prior projection (what the kernel computes in its first iteration)
    x0, _, y0, _ = VB.footprint_box(px, stride)
    for i in range(len(px)):
        assert xs[i] is None or x0[i] == xs[i], (i, x0[i], xs[i])
        assert ys[i] is None or y0[i] == ys[i], (i, y0[i], ys[i])
    assert (x0 + 10 * stride == cam.width).sum() == 1 and (x0 + 10 * stride == cam.width - stride).sum() == 1
    try:
        vio_setup(gpu_ctx, fr)
        gpu_ctx.vio_set_camera(cam, vcfg)
        args = _args(fr, bs, prior)
        a, b, b2 = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), [dict(), dict(tuning=api.TUNE_VIO_TMA), dict(tuning=api.TUNE_VIO_TMA)])
    finally:
        gpu_ctx.vio_set_camera(cam, fr["vio_cfg"])
    assert a["total_iters"] >= 2
    bits_equal(a, b, VIO_KEYS)
    bits_equal(a, b2, VIO_KEYS)


# --------------------------------------------------------------------------------------------------------- e. drift across the edge
def test_footprint_restaged_across_the_edge_between_iterations(gpu_ctx, border):
    """Patches whose footprint is inside the image at the prior and crosses an edge as the estimate moves (a prior rotated
    by 0.5 degrees, one level of stride 1): the cached footprint is restaged across the border. Persistent against
    per-iteration launches (with and without TMA) bit for bit, and against the oracle."""
    fr, _, _ = border
    cam = fr["cam_cfg"]
    prior = vio_prior(fr, seed=11, rot_deg=0.5, pos=0.02)
    vcfg = dataclasses.replace(fr["vio_cfg"], levels=1, max_iterations=8)
    v, u = 0.5 * cam.height + 17.3, 0.5 * cam.width - 23.7
    # anchor exactly 5 px (stride 1) from each edge at the prior: the footprint touches column / row 0 or the last one
    px = np.array([(5.3, v), (cam.width - 5.7, v), (u, 5.3), (u, cam.height - 5.7)])
    extra = VB.patches_at(fr, prior, px, np.zeros(len(px), np.int32))
    bs = VB.with_interior(fr, prior, extra)
    bs["warp_patch"] = np.ascontiguousarray(bs["warp_patch"][:, :64])
    assert not VB.leaves_image(px, np.zeros(4, np.int32), 1, cam.width, cam.height).any()
    fr1 = dict(fr, vio_cfg=vcfg)
    try:
        vio_setup(gpu_ctx, fr)
        gpu_ctx.vio_set_camera(cam, vcfg)
        args = _args(fr, bs, prior)
        a, b, c = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), [dict(loop_mode=0), dict(loop_mode=2), dict(loop_mode=2, tuning=api.TUNE_VIO_TMA)])
    finally:
        gpu_ctx.vio_set_camera(cam, fr["vio_cfg"])
    assert a["total_iters"] >= 2
    bits_equal(a, b, VIO_KEYS)
    bits_equal(a, c, VIO_KEYS)
    compare_vio(b, O.OracleVIO(cam, fr["ext"], vcfg).update(*args), 1)
    # where the posterior projects them: at least one footprint now leaves the image
    st = S.unpack_state(b["state"])
    Rcw, Pcw = S.camera_pose(fr1["ext"], st["R"], st["p"])
    post = S.cam_project(cam, extra["vis_pos"] @ Rcw.T + Pcw)
    crossed = VB.leaves_image(post, np.zeros(4, np.int32), 1, cam.width, cam.height)
    assert crossed.sum() >= 1, post


# --------------------------------------------------------------------------------------------------------- f. inverse variant
def test_inverse_variant_with_reference_pixels_near_the_border(gpu_ctx, border):
    """updateStateInverse with reference pixels (Feature::px_) near and beyond the reference image's edges: the reference
    gradients of precomputeReferencePatches read across the border. Against the oracle; persistent against per-iteration."""
    fr, prior, bs = border
    fb = dict(fr, vis_pos=bs["vis_pos"], vis_normal=bs["vis_normal"], px_ref=bs["px_ref"])
    refs = O.inverse_refs_from_frame(fb)
    cam, L = fr["cam_cfg"], fr["vio_cfg"].levels
    # reference footprints (levels 0..L-1, stride 2^level) that leave the reference image
    n_ref_leave = int(VB.leaves_image(refs["ref_px"][bs["border"]], np.zeros(bs["border"].sum(), np.int32), L, cam.width, cam.height).sum())
    assert n_ref_leave >= 30, n_ref_leave
    inv_cfg = dataclasses.replace(fr["vio_cfg"], inverse_composition_en=True)
    n = len(bs["vis_pos"])
    args = (fr["img"], bs["vis_pos"], bs["warp_patch"], bs["search_levels"], np.ones(n), prior, prior)
    try:
        vio_setup(gpu_ctx, fr)
        gpu_ctx.vio_set_camera(cam, inv_cfg)
        gpu_ctx.vio_set_inverse_refs(refs["ref_img_index"], refs["ref_px"], refs["ref_f"], refs["ref_R"], refs["ref_pos"])
        a, b = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), [dict(loop_mode=0), dict(loop_mode=2)])
    finally:
        gpu_ctx.vio_set_camera(cam, fr["vio_cfg"])
    assert a["total_iters"] >= 3
    bits_equal(a, b, VIO_KEYS)
    vio = O.OracleVIO(cam, fr["ext"], fr["vio_cfg"])
    vio.set_inverse_refs(**refs)
    vio.set_inverse(True)
    compare_vio(b, vio.update(*args), L)


# --------------------------------------------------------------------------------------------------------- g. fisheye
def test_fisheye_camera_with_border_patches(gpu_ctx):
    """Config 3's equidistant camera, where distortion is largest at the edge: a few border patches among the interior ones."""
    fr = get_frame(**FISHEYE)
    prior = vio_prior(fr, 9)
    bs = VB.border_patch_set(fr, prior, every=4)
    assert bs["n_leave"] >= 10, bs["n_leave"]
    vio_setup(gpu_ctx, fr)
    args = _args(fr, bs, prior)
    a, b = sweep(gpu_ctx, lambda: gpu_ctx.vio_update(*args), [dict(loop_mode=0), dict(loop_mode=2)])
    bits_equal(a, b, VIO_KEYS)
    compare_vio(b, O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args), fr["vio_cfg"].levels)
