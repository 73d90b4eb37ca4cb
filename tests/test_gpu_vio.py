"""GPU parity: the CUDA VIO update, patch extraction and affine warp (through the C ABI) against the CPU oracle."""
import numpy as np
import pytest

import oracle_bind as O
from conftest import get_frame
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from parity_util import assert_state_close, rel

pytestmark = pytest.mark.gpu


def _vio_prior(fr, seed=3, rot_deg=0.15, pos=0.01, cov_scale=0.2):
    rng = np.random.default_rng(seed)
    t = S.unpack_state(fr["state_true"])
    cov = S.random_prior_cov(rng, scale=cov_scale)
    return S.pack_state(t["R"] @ S.so3_exp(rng.normal(0, np.deg2rad(rot_deg), 3)), t["p"] + rng.normal(0, pos, 3), 1.0 + rng.normal(0, 0.01), t["v"],
                        g=t["g"], cov=cov)


def _setup(ctx, fr):
    ctx.set_extrinsics(fr["ext"])
    ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])
    ctx.vio_set_image(fr["img"])
    ctx.vio_set_ref_images([fr["img_ref"]])


def _gpu_warp(ctx, fr, state):
    st = S.unpack_state(state)
    T_cur = api.pack_T(*S.camera_pose(fr["ext"], st["R"], st["p"]))
    n = len(fr["vis_pos"])
    T_ref = np.tile(api.pack_T(*fr["T_ref"]), (n, 1))
    return ctx.vio_warp_patches(np.zeros(n, np.int32), fr["px_ref"], fr["vis_pos"], fr["vis_normal"], T_ref, T_cur)


def _compare_vio(g, o, L):
    assert g["total_iters"] == o["total_iters"]
    assert np.array_equal(g["iters_per_level"], o["iters_per_level"])
    assert np.array_equal(g["accepted_per_level"], o["accepted_per_level"])
    for lvl in range(L):
        for it in range(o["iters_per_level"][lvl]):
            # error: a sequential FLOAT accumulation over n_meas terms in the reference (rounding error ~ sqrt(n) * 6e-8, and an
            # unspecified OpenMP order); an fp64 fixed-order sum here -> compare at 1e-5 relative
            assert abs(g["error_trace"][lvl][it] - o["error_trace"][lvl][it]) <= 1e-5 * o["error_trace"][lvl][it]
        for it in range(o["accepted_per_level"][lvl]):
            assert rel(g["HTH"][lvl][it], o["HTH"][lvl][it]) < 1e-9
            assert rel(g["HTz"][lvl][it], o["HTz"][lvl][it]) < 1e-7
    np.testing.assert_allclose(g["errors"], o["errors"], rtol=2e-6, atol=1e-3)
    assert_state_close(g["state"], o["state"], rot_tol=1e-8, pos_tol=1e-8, cov_tol=1e-6, rest_tol=1e-8)


def test_image_patch_bit_exact(gpu_ctx, small_vio_frame):
    fr = small_vio_frame
    _setup(gpu_ctx, fr)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    rng = np.random.default_rng(0)
    pc = np.stack([rng.uniform(90, 550, 64), rng.uniform(90, 420, 64)], 1)
    for level in range(4):
        g = gpu_ctx.vio_get_image_patch(pc, level)
        for i in range(len(pc)):
            assert np.array_equal(g[i], vio.get_image_patch(fr["img"], pc[i], level))


def test_warp_matrix_and_warp_affine(gpu_ctx, small_vio_frame):
    fr = small_vio_frame
    _setup(gpu_ctx, fr)
    prior = _vio_prior(fr)
    g = _gpu_warp(gpu_ctx, fr, prior)
    o = O.oracle_warp_patches(fr, prior)
    np.testing.assert_allclose(g["A_cur_ref"], o["A_cur_ref"], rtol=1e-10, atol=1e-12)
    assert np.array_equal(g["search_levels"], o["search_levels"])
    # the warp itself (the inverse through the rounded-products determinant, then float arithmetic without contraction) is
    # bit-exact given the same A: feed the oracle the GPU's A
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    for i in range(len(fr["vis_pos"])):
        ref = vio.warp_affine(fr["img_ref"], g["A_cur_ref"][i], fr["px_ref"][i], g["search_levels"][i])
        assert np.array_equal(ref, g["warp_patch"][i]), i


@pytest.mark.parametrize("seed", [2, 6])
def test_vio_matches_oracle(gpu_ctx, seed):
    fr = get_frame(seed=seed, n_pts=2000, n_map=120_000, n_patches=150, scene_scale=0.5)
    _setup(gpu_ctx, fr)
    prior = _vio_prior(fr, seed)
    w = _gpu_warp(gpu_ctx, fr, prior)
    g = gpu_ctx.vio_update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    o = vio.update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    _compare_vio(g, o, fr["vio_cfg"].levels)


def test_vio_literal_solve_mode(gpu_ctx, small_vio_frame):
    fr = small_vio_frame
    _setup(gpu_ctx, fr)
    prior = _vio_prior(fr)
    w = _gpu_warp(gpu_ctx, fr, prior)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    o = vio.update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    gpu_ctx.set_solve_mode(1)
    g = gpu_ctx.vio_update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    gpu_ctx.set_solve_mode(0)
    _compare_vio(g, o, fr["vio_cfg"].levels)


def test_vio_exposure_off_search_levels_and_distortion(gpu_ctx):
    """exposure_estimate_en = false (zero 7th column), mixed search levels, radtan distortion in world2cam."""
    cam = S.CamCfg(d=(-0.076160, 0.123001, -0.00113, 0.000251, 0.0))
    vcfg = S.VioCfg(levels=3, exposure_estimate_en=False, img_point_cov=1000.0)
    fr = get_frame(seed=8, n_pts=1000, n_map=100_000, n_patches=120, scene_scale=0.5, cam=cam, vio=vcfg)
    _setup(gpu_ctx, fr)
    prior = _vio_prior(fr, 8)
    w = _gpu_warp(gpu_ctx, fr, prior)
    sl = w["search_levels"].copy()
    sl[::3] = 1  # stride doubles for a third of the patches (border = 40 px keeps taps inside the image at level<=2)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    o = vio.update(fr["img"], fr["vis_pos"], w["warp_patch"], sl, fr["inv_ref_expo"], prior, prior)
    g = gpu_ctx.vio_update(fr["img"], fr["vis_pos"], w["warp_patch"], sl, fr["inv_ref_expo"], prior, prior)
    _compare_vio(g, o, 3)
    assert g["state"][12] == prior[12] or abs(g["state"][12] - o["state"][12]) < 1e-10


def test_vio_fisheye_camera(gpu_ctx):
    cam = S.CamCfg(model=1, width=720, height=540, fx=351.31400364193297, fy=351.4911744656785, cx=367.8522793375995, cy=253.8402144980996,
                   d=(-0.03696737352869157, -0.008917880497032812, 0.008912969593422046, -0.0037685977496087313, 0.0))
    vcfg = S.VioCfg(img_point_cov=1000.0)
    fr = get_frame(seed=9, n_pts=1000, n_map=100_000, n_patches=100, scene_scale=0.5, cam=cam, vio=vcfg, ext=S.hilti_extrinsics())
    _setup(gpu_ctx, fr)
    prior = _vio_prior(fr, 9)
    w = _gpu_warp(gpu_ctx, fr, prior)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    o = vio.update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    g = gpu_ctx.vio_update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    _compare_vio(g, o, 4)


def test_vio_edge_cases(gpu_ctx, small_vio_frame):
    fr = small_vio_frame
    _setup(gpu_ctx, fr)
    prior = _vio_prior(fr)
    # total_points == 0: state untouched (vio.cpp:786)
    L = fr["vio_cfg"].levels
    g = gpu_ctx.vio_update(fr["img"], np.zeros((0, 3)), np.zeros((0, 64 * L), np.float32), np.zeros(0, np.int32), np.zeros(0), prior, prior)
    assert np.array_equal(g["state"], prior) and g["total_iters"] == 0
    # one patch
    w = _gpu_warp(gpu_ctx, fr, prior)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    args = (fr["img"], fr["vis_pos"][:1], w["warp_patch"][:1], w["search_levels"][:1], fr["inv_ref_expo"][:1], prior, prior)
    _compare_vio(gpu_ctx.vio_update(*args), vio.update(*args), L)
    # image size mismatch is an argument error, not a crash
    with pytest.raises(api.EsikfError):
        gpu_ctx.vio_set_image(fr["img"][:100])


def test_vio_full_size_properties(gpu_ctx):
    """BASELINE config 2 visual size (2 k patches, 640x512, 4 levels): reproducible, symmetric PSD H^T H, agrees with the oracle."""
    fr = get_frame(seed=0, n_pts=1000, n_map=300_000, n_patches=2000, scene_scale=0.7)
    _setup(gpu_ctx, fr)
    prior = _vio_prior(fr, 0)
    w = _gpu_warp(gpu_ctx, fr, prior)
    args = (fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    a = gpu_ctx.vio_update(*args)
    b = gpu_ctx.vio_update(*args)
    assert np.array_equal(a["state"], b["state"]) and np.array_equal(a["HTH"], b["HTH"]) and np.array_equal(a["errors"], b["errors"])
    H = a["HTH"][3][0]
    assert rel(H, H.T) < 1e-12 and np.linalg.eigvalsh(0.5 * (H + H.T)).min() > -1e-9 * np.abs(H).max()
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"], threads=1)
    _compare_vio(a, vio.update(*args), 4)


def test_persistent_and_per_iteration_loops_are_bit_identical(gpu_ctx, small_vio_frame):
    fr = small_vio_frame
    _setup(gpu_ctx, fr)
    prior = _vio_prior(fr)
    w = _gpu_warp(gpu_ctx, fr, prior)
    args = (fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    try:
        gpu_ctx.set_loop_mode(2)
        a2 = gpu_ctx.vio_update(*args)
        gpu_ctx.set_loop_mode(1)
        a = gpu_ctx.vio_update(*args)
        gpu_ctx.set_loop_mode(0)
        b = gpu_ctx.vio_update(*args)
    finally:
        gpu_ctx.set_loop_mode(api.DEFAULT_LOOP_MODE)
    for x in (a, a2):
        assert x["total_iters"] == b["total_iters"]
        assert np.array_equal(x["state"], b["state"]) and np.array_equal(x["HTH"], b["HTH"]) and np.array_equal(x["errors"], b["errors"])
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    _compare_vio(b, vio.update(*args), fr["vio_cfg"].levels)


def test_config5_five_levels_4k_patches(gpu_ctx):
    """BASELINE config 5 visual size (MARS_LVIG camera 612x512, 4 k patches, 5 pyramid levels, img_point_cov 1000):
    two patches per warp and a coarsest stride of 16 pixels."""
    cam = S.CamCfg(width=612, height=512, fx=612.0 * 0.72, fy=612.0 * 0.72, cx=306.0, cy=256.0)
    vcfg = S.VioCfg(levels=5, img_point_cov=1000.0)
    fr = get_frame(seed=13, n_pts=1000, n_map=300_000, n_patches=4000, scene_scale=0.7, cam=cam, vio=vcfg)
    assert len(fr["vis_pos"]) > 3000
    _setup(gpu_ctx, fr)
    prior = _vio_prior(fr, 13)
    w = _gpu_warp(gpu_ctx, fr, prior)
    args = (fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    g = gpu_ctx.vio_update(*args)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    _compare_vio(g, vio.update(*args), 5)


@pytest.mark.parametrize("name", ["small", "exposure"])
def test_vio_matches_reference_source_golden(gpu_ctx, name):
    """The CUDA path against the committed outputs of the REFERENCE SOURCE (src/vio.cpp compiled against stand-in headers,
    tests/golden/ref_vio_golden.npz — tests/test_oracle_ref_pin_vio.py): posterior state / covariance and the per-patch
    photometric errors of VIOManager::computeJacobianAndUpdateEKF; the warp patches of the same inputs agree sample by sample."""
    from test_oracle_ref_pin_vio import CASES, GOLDEN

    g = np.load(GOLDEN)
    fr = get_frame(**CASES[name])
    prior = g[f"{name}_prior"]
    _setup(gpu_ctx, fr)
    w = _gpu_warp(gpu_ctx, fr, prior)
    assert np.array_equal(w["search_levels"], g[f"{name}_search_levels"])
    # getWarpMatrixAffineHomography + warpAffine on the device: A agrees to 1e-10, so nearly every float sample is identical
    np.testing.assert_allclose(w["warp_patch"], g[f"{name}_warp_patch"], atol=2e-3)
    assert np.mean(w["warp_patch"] == g[f"{name}_warp_patch"]) > 0.98
    v = gpu_ctx.vio_update(fr["img"], fr["vis_pos"], g[f"{name}_warp_patch"], g[f"{name}_search_levels"], fr["inv_ref_expo"], prior, prior)
    assert_state_close(v["state"], g[f"{name}_state"], rot_tol=1e-8, pos_tol=1e-8, cov_tol=1e-6, rest_tol=1e-8)
    np.testing.assert_allclose(v["errors"], g[f"{name}_errors"], rtol=2e-6, atol=1e-3)
