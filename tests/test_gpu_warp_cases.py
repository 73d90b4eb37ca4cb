"""GPU: the VIO warp producers (warp_matrix_kernel, warp_affine_kernel) on the hand-built sets of tests/warp_cases.py, and the
VIO update over 6 to 8 pyramid levels with 8 iterations each."""
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest

import oracle_bind as O
import warp_cases as W
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from test_gpu_loop_modes import VIO_KEYS, _bits_equal
from test_gpu_vio import _compare_vio, _setup
from test_gpu_vio_border import _modes
from test_warp_cases import EXT, oracle_warp_matrix

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ref_image(cam, seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:cam.height, 0:cam.width]
    return (127.5 + 60 * np.sin(xx / 9.7) * np.cos(yy / 6.3) + rng.normal(0, 25, (cam.height, cam.width))).clip(0, 255).astype(np.uint8)


def _device_warp(ctx, camera, case, levels=4, keep_on_device=False):
    cam = W.CAMERAS[camera]
    img = _ref_image(cam)
    ctx.set_extrinsics(EXT)
    ctx.vio_set_camera(cam, S.VioCfg(levels=levels))
    ctx.vio_set_ref_images([img])
    n = len(case["px_ref"])
    g = ctx.vio_warp_patches(np.zeros(n, np.int32), case["px_ref"], case["pos_w"], case["normal_w"], W.T_ref_packed(case), api.pack_T(*W.T_CUR),
                             keep_on_device=keep_on_device)
    return g, img


def _assert_warp_is_oracle_warp_affine(camera, g, img, px_ref, levels=4):
    """warp_patch = the oracle's warpAffine given the device's own A and level, bit for bit, for every patch."""
    vio = O.OracleVIO(W.CAMERAS[camera], EXT, S.VioCfg(levels=levels))
    want = np.array([vio.warp_affine(img, g["A_cur_ref"][i], px_ref[i], int(g["search_levels"][i])) for i in range(len(px_ref))])
    bad = np.nonzero((want != g["warp_patch"]).any(1))[0]
    assert len(bad) == 0, (len(bad), bad[:10])


# --------------------------------------------------------------------------------------------------------- a. thresholds
@pytest.mark.parametrize("thr", W.THRESHOLDS)
@pytest.mark.parametrize("camera", list(W.CAMERAS))
def test_search_level_at_the_thresholds(gpu_ctx, camera, thr):
    """getBestSearchLevel on the device, on geometries bisected onto D = 3 / 12: the rounded-products rule applied to the
    device's own A, on every case; both reach flags occur on the device's A; A within 1e-10 of the oracle's; a level differs
    from the oracle's only where the oracle's determinant lies within what 1e-10 on A allows; the warp is the oracle's
    warpAffine given the device's A and level, bit for bit."""
    case = W.threshold_set(camera, thr)
    g, img = _device_warp(gpu_ctx, camera, case)
    Ag = g["A_cur_ref"]
    assert np.array_equal(g["search_levels"], W.search_level(W.det_rounded(Ag)))
    near, split = W.reach(Ag, thr)
    assert near.sum() >= 50 and split.sum() >= 5, (near.sum(), split.sum())
    Ao, slo = oracle_warp_matrix(camera, case)
    np.testing.assert_allclose(Ag, Ao, rtol=0, atol=1e-10)
    # |dD| <= |a00| |da11| + |a11| |da00| + |a01| |da10| + |a10| |da01| + rounding, with |da| <= 1e-10
    bound = 1e-10 * np.abs(Ao).reshape(-1, 4).sum(1) * 2 + 8 * np.spacing(thr)
    differ = g["search_levels"] != slo
    assert (np.abs(W.det_rounded(Ao)[differ] - thr) <= bound[differ]).all()
    _assert_warp_is_oracle_warp_affine(camera, g, img, case["px_ref"])


# --------------------------------------------------------------------------------------------------------- b. edge geometries
@pytest.mark.parametrize("camera", list(W.CAMERAS))
def test_edge_geometries(gpu_ctx, camera):
    """Grazing planes (D tiny, both signs), a mirrored warp, D >> 48 (level capped at 2), H = 0 (NaN A, level 0, the patch left
    untouched: zeros, also in the patches keep_on_device installs for the update) and the fisheye principal point."""
    e = W.edge_set(camera)
    g, img = _device_warp(gpu_ctx, camera, e, keep_on_device=True)
    Ag, sl = g["A_cur_ref"], g["search_levels"]
    assert np.array_equal(sl, W.search_level(W.det_rounded(Ag)))
    for i, want in enumerate(e["want_level"]):
        assert want is None or sl[i] == want, (e["name"][i], sl[i], W.det_rounded(Ag)[i])
    h0 = np.array([nm.startswith("h_zero") for nm in e["name"]])
    assert np.isnan(Ag[h0]).all() and not np.isnan(Ag[~h0]).any()
    assert not g["warp_patch"][h0].any() and g["warp_patch"][~h0].any(1).all()
    Ao, slo = oracle_warp_matrix(camera, e)
    np.testing.assert_allclose(Ag[~h0], Ao[~h0], rtol=0, atol=1e-10)
    assert np.array_equal(sl, slo)
    _assert_warp_is_oracle_warp_affine(camera, g, img, e["px_ref"])
    # the installed patches (a zero patch among them) drive an update exactly as the same patches passed in by the caller
    n = len(e["px_ref"])
    prior = S.pack_state(np.eye(3), np.zeros(3), 1.0, cov=S.random_prior_cov(np.random.default_rng(0), scale=0.2))
    cur = _ref_image(W.CAMERAS[camera], 1)
    gpu_ctx.vio_set_image(cur)
    gpu_ctx.vio_run(prior, prior)
    a = gpu_ctx.vio_fetch()
    b = gpu_ctx.vio_update(cur, e["pos_w"], g["warp_patch"], sl, np.ones(n), prior, prior)
    _bits_equal(a, b, VIO_KEYS)


# --------------------------------------------------------------------------------------------------------- c. caller matrices
def test_warp_affine_on_cancelling_matrices(gpu_ctx):
    """esikf_vio_warp_affine and the shim's warpAffine on matrices whose determinant cancels (the contracted determinant gives
    another float inverse), pyramid depths 1..8, search levels 0, 1, 2 and 8: bit for bit against the oracle."""
    A, px, sl, img = W.caller_matrices()
    n = len(A)
    cam = dataclasses.replace(W.CAMERAS["pinhole"], width=img.shape[1], height=img.shape[0])
    shim = C.CDLL(os.path.join(ROOT, "fast_livo2_b200", "libfl2_shim.so"))
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    cc = api.CameraC(cam.model, cam.width, cam.height, 0, cam.fx, cam.fy, cam.cx, cam.cy)
    cc.d[:] = list(cam.d)
    inside = 0
    for L in range(1, 9):
        vcfg = S.VioCfg(levels=L)
        gpu_ctx.set_extrinsics(EXT)
        gpu_ctx.vio_set_camera(cam, vcfg)
        gpu_ctx.vio_set_ref_images([img])
        out = gpu_ctx.vio_warp_affine(np.zeros(n, np.int32), px, A, sl)
        vio = O.OracleVIO(cam, EXT, vcfg)
        want = np.array([vio.warp_affine(img, A[i], px[i], int(sl[i])) for i in range(n)])
        assert np.array_equal(out, want), L
        inside += int((want != 0).sum())
    assert inside > 0
    # VIOManager::warpAffine of the shim, one pyramid level per call, at the deepest pyramid
    vc = api.VioCfgC(vcfg.img_point_cov, 8, vcfg.max_iterations, int(vcfg.exposure_estimate_en), 0)
    pc = np.array([cam.cx, cam.cy])
    for i in range(0, n, 6):
        for lvl in range(8):
            patch, warp = np.zeros(64 * 8, np.float32), np.full(64 * 8, -7.0, np.float32)
            a, p = np.ascontiguousarray(A[i]), np.ascontiguousarray(px[i])
            rc = shim.fl2_shim_patch_helpers(C.byref(cc), C.byref(vc), vp(img), img.shape[1], img.shape[0], vp(pc), 0, vp(patch), vp(a), vp(img), vp(p),
                                             int(sl[i]), lvl, vp(warp))
            assert rc == 0
            assert np.array_equal(warp[64 * lvl:64 * lvl + 64], want[i][64 * lvl:64 * lvl + 64]), (i, lvl)


# --------------------------------------------------------------------------------------------------------- d. deep frames
@pytest.fixture(scope="module", params=W.DEEP_LEVELS)
def deep(request):
    return W.deep_frame(request.param)


def _deep_args(fr, prior, pt):
    return (fr["img"], pt["vis_pos"], pt["warp_patch"], pt["search_levels"], pt["inv_ref_expo"], prior, prior)


@pytest.mark.parametrize("solve_mode", [0, 1])
def test_deep_update_matches_oracle(gpu_ctx, deep, solve_mode):
    fr, prior, pt = deep
    L = fr["vio_cfg"].levels
    assert set(pt["search_levels"].tolist()) == {0, 1, 2} and (L < 7 or (~pt["in_buffer"]).any())  # taps beyond the buffer read 0
    _setup(gpu_ctx, fr)
    args = _deep_args(fr, prior, pt)
    gpu_ctx.set_solve_mode(solve_mode)
    try:
        g = gpu_ctx.vio_update(*args)
    finally:
        gpu_ctx.set_solve_mode(0)
    o = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args)
    assert (o["iters_per_level"][:L] > 0).all() and o["total_iters"] > L
    _compare_vio(g, o, L)


def test_deep_update_loop_modes_and_tma_are_bit_identical(gpu_ctx, deep):
    fr, prior, pt = deep
    _setup(gpu_ctx, fr)
    args = _deep_args(fr, prior, pt)
    a, b = _modes(gpu_ctx, args, (2, 0))
    c, = _modes(gpu_ctx, args, (2,), tuning=api.TUNE_VIO_TMA)
    assert a["total_iters"] > fr["vio_cfg"].levels
    _bits_equal(a, b, VIO_KEYS)
    _bits_equal(a, c, VIO_KEYS)


def test_timing_and_phase_stamps_at_eight_levels_and_eight_iterations(gpu_ctx):
    """At 8 levels x 8 iterations the 64 VIO timing slots and the 64 VIO phase-stamp slots are all addressed: the per-iteration
    launches time every (level, iteration) slot; the persistent kernel stamps exactly the iterations it executed (slot
    (levels - 1 - level) * max_iterations + it, as iters_per_level reports them) and leaves the others zero."""
    fr, prior, pt = W.deep_frame(8)
    _setup(gpu_ctx, fr)
    args = _deep_args(fr, prior, pt)
    try:
        gpu_ctx.set_kernel_timing(True)
        gpu_ctx.set_loop_mode(0)
        t = gpu_ctx.vio_update(*args)
        ms = gpu_ctx.get_kernel_timing()
        gpu_ctx.set_kernel_timing(False)
        gpu_ctx.set_loop_mode(2)
        gpu_ctx.set_phase_stamps(True)
        s = gpu_ctx.vio_update(*args)
        stamps = gpu_ctx.get_phase_stamps()
    finally:
        gpu_ctx.set_kernel_timing(False)
        gpu_ctx.set_phase_stamps(False)
        gpu_ctx.set_loop_mode(api.DEFAULT_LOOP_MODE)
    _bits_equal(t, s, VIO_KEYS)
    assert (ms["vio_patch_ms"] > 0).all() and (ms["vio_solve_ms"] > 0).all()
    ipl = s["iters_per_level"]
    executed = np.zeros(64, bool)
    for level in range(8):
        executed[8 * (7 - level): 8 * (7 - level) + ipl[level]] = True
    assert executed.any() and not executed.all(), ipl
    vio_rows = stamps[8:72]  # 8 LIO slots, then 64 VIO slots of 8 stamps
    assert (vio_rows[executed][:, :6] > 0).all()
    assert not vio_rows[~executed].any()
