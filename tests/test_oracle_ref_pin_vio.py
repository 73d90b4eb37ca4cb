"""Pins the VIO oracle (oracle/orc_vio.cpp, a restatement) against the REFERENCE'S OWN SOURCE: FAST-LIVO2's src/vio.cpp (+
frame.cpp, visual_point.cpp) compiled from where it lies against stand-in headers (oracle/ref_shim/: matrix library, cv::Mat,
Sophus::SE3, boost::noncopyable, PCL / ROS shells; oracle/ref_vio.cpp -> oracle/_ref/libfl2_ref_vio.so).

What this pins: everything VIOManager::computeJacobianAndUpdateEKF -> updateState (projection, bilinear weights, taps, the
Jacobian chain, H^T H, the gain, boxplus, the error-gated accept / rollback, P -= G P), the inverse-compositional variant
(precomputeReferencePatches, updateStateInverse), getImagePatch, warpAffine, getWarpMatrixAffineHomography / getBestSearchLevel
compute — the reference's own arithmetic. What it cannot pin: vikit (un-vendored, no version pin): the pinhole model and
vk::interpolateMat_8u inside the stand-in are restatements of the published algorithm, shared by both sides.

Calls the library where it is built (oracle/Makefile, from a FAST-LIVO2 source tree); elsewhere every case compares with
the reference's stored outputs (tests/golden/ref_pin/vio.npz, written by a run with FL2_RECORD_REF_PIN=1 where the library is
built; see oracle_bind.RefPin). tests/golden/ref_vio_golden.npz carries full outputs for two cases (make_ref_golden.py)."""
import dataclasses
import os

import numpy as np
import pytest

import oracle_bind as O
import vio_border as VB
from conftest import get_frame
from fast_livo2_b200 import synthetic as S
from parity_util import assert_state_close

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_vio_golden.npz")
PIN = O.RefPin("vio")
needs_ref = pytest.mark.skipif(not O.RefPin.available("vio"), reason="neither oracle/_ref/libfl2_ref_vio.so nor tests/golden/ref_pin/vio.npz")

CASES = {
    "small": dict(seed=2, n_pts=2000, n_map=120_000, n_patches=150, scene_scale=0.5),
    "exposure": dict(seed=6, n_pts=1000, n_map=120_000, n_patches=200, scene_scale=0.5, vio=S.VioCfg(exposure_estimate_en=True)),
    "three_levels": dict(seed=8, n_pts=1000, n_map=120_000, n_patches=300, scene_scale=0.5, vio=S.VioCfg(levels=3, img_point_cov=400.0)),
    "distorted_pinhole": dict(seed=9, n_pts=1000, n_map=120_000, n_patches=200, scene_scale=0.5,
                              cam=S.CamCfg(d=(-0.05, 0.02, 0.001, -0.0005, 0.0))),
    # config 3's camera (HILTI22 fisheye, vk::EquidistantCamera) behind the same abstract interface
    "fisheye": dict(seed=10, n_pts=1000, n_map=120_000, n_patches=200, scene_scale=0.5, vio=S.VioCfg(img_point_cov=1000.0),
                    cam=S.CamCfg(model=1, width=720, height=540, fx=351.31400364193297, fy=351.4911744656785, cx=367.8522793375995, cy=253.8402144980996,
                                 d=(-0.03696737352869157, -0.008917880497032812, 0.008912969593422046, -0.0037685977496087313, 0.0))),
}


def _prior(fr, seed=3):
    rng = np.random.default_rng(seed)
    t = S.unpack_state(fr["state_true"])
    return S.pack_state(t["R"] @ S.so3_exp(rng.normal(0, np.deg2rad(0.15), 3)), t["p"] + rng.normal(0, 0.01, 3), 1.0 + rng.normal(0, 0.01), t["v"], g=t["g"],
                        cov=S.random_prior_cov(rng, scale=0.2))


def _inputs(name):
    fr = get_frame(**CASES[name])
    prior = _prior(fr)
    w = O.oracle_warp_patches(fr, prior)
    return fr, prior, w


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_oracle_vio_update_reproduces_the_reference_source(name):
    fr, prior, w = _inputs(name)
    args = (fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    ref = PIN.get(f"update/{name}", lambda: {k: v for k, v in O.RefVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args).items() if k in ("state", "errors", "H_T_H")})
    orc = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args)
    assert orc["total_iters"] >= 4
    # same decisions (accept / rollback / stop) or the states would differ grossly; the sums differ only in association order
    assert_state_close(orc["state"], ref["state"], rot_tol=1e-11, pos_tol=1e-11, cov_tol=1e-9, rest_tol=1e-11)
    # per-patch photometric error: float accumulation in both, same order (one thread)
    np.testing.assert_allclose(orc["errors"], ref["errors"], rtol=1e-6, atol=1e-4)
    # the H_T_H member (vio.h:121) holds the normal matrix of the last ACCEPTED iteration: one of the oracle's per-iteration blocks
    blocks = orc["HTH"].reshape(-1, 7, 7)
    blocks = blocks[np.abs(blocks).max(axis=(1, 2)) > 0]
    want = ref["H_T_H"][:7, :7]
    rel = [np.abs(b - want).max() / np.abs(want).max() for b in blocks]
    assert min(rel) < 1e-10, min(rel)


@needs_ref
def test_oracle_inverse_compositional_variant_reproduces_the_reference_source():
    fr, prior, w = _inputs("small")
    refs = O.inverse_refs_from_frame(fr)
    n = len(fr["vis_pos"])
    args = (fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], np.ones(n))
    ref = PIN.get("update_inverse", lambda: O.RefVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update_inverse(*args, refs, prior, prior))
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], dataclasses.replace(fr["vio_cfg"], inverse_composition_en=True))
    vio.set_inverse_refs(**refs)
    vio.set_inverse(True)
    orc = vio.update(*args, prior, prior)
    assert_state_close(orc["state"], ref["state"], rot_tol=1e-11, pos_tol=1e-11, cov_tol=1e-9, rest_tol=1e-11)
    np.testing.assert_allclose(orc["errors"], ref["errors"], rtol=1e-6, atol=1e-4)


@needs_ref
def test_oracle_patch_producers_reproduce_the_reference_source():
    """getImagePatch, getWarpMatrixAffineHomography + getBestSearchLevel, warpAffine (vio.cpp:203-331)."""
    fr, prior, w = _inputs("distorted_pinhole")
    orc = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    st = S.unpack_state(prior)
    T_cur = S.camera_pose(fr["ext"], st["R"], st["p"])
    rng = np.random.default_rng(1)
    idx = list(range(0, len(fr["vis_pos"]), 7))
    pcs = [np.array([rng.uniform(40, fr["cam_cfg"].width - 40), rng.uniform(40, fr["cam_cfg"].height - 40)]) for _ in idx]
    L = fr["vio_cfg"].levels

    def ref_producers():
        ref = O.RefVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
        A, sl = zip(*[ref.warp_matrix(fr["px_ref"][i], fr["vis_pos"][i], fr["vis_normal"][i], fr["T_ref"], T_cur) for i in idx])
        warp = [ref.warp_affine(fr["img_ref"], A[k], fr["px_ref"][i], sl[k]) for k, i in enumerate(idx)]
        patch = [[ref.get_image_patch(fr["img"], pc, lvl) for lvl in range(L)] for pc in pcs]
        return dict(A=np.array(A), search_level=np.array(sl, np.int32), warp=np.array(warp), patch=np.array(patch))

    r = PIN.get("patch_producers", ref_producers, exact=("search_level", "warp", "patch"))
    Ao, so = zip(*[orc.warp_matrix(fr["px_ref"][i], fr["vis_pos"][i], fr["vis_normal"][i], fr["T_ref"], T_cur) for i in idx])
    assert O.same(np.array(so, np.int32), r, "search_level")
    np.testing.assert_allclose(np.array(Ao), r["A"], rtol=1e-11, atol=1e-13)
    assert O.same(np.array([orc.warp_affine(fr["img_ref"], r["A"][k], fr["px_ref"][i], int(r["search_level"][k]))
                            for k, i in enumerate(idx)]), r, "warp")
    assert O.same(np.array([[orc.get_image_patch(fr["img"], pc, lvl) for lvl in range(L)] for pc in pcs]), r, "patch")


def test_oracle_matches_reference_vio_golden():
    """The reference library's own outputs, committed: the pin survives where the library cannot be built."""
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/ref_vio_golden.npz not generated")
    g = np.load(GOLDEN, allow_pickle=False)
    for name in ("small", "exposure"):
        fr, prior, w = _inputs(name)
        np.testing.assert_array_equal(w["warp_patch"], g[f"{name}_warp_patch"])  # same inputs as when the vectors were made
        orc = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
        assert_state_close(orc["state"], g[f"{name}_state"], rot_tol=1e-11, pos_tol=1e-11, cov_tol=1e-9, rest_tol=1e-11)
        np.testing.assert_allclose(orc["errors"], g[f"{name}_errors"], rtol=1e-6, atol=1e-4)


BASELINE_COUNTS = {  # per-iteration matched points / VIO iterations the CUDA bench lines report for these frames
    "cfg2": ([99663, 99869, 99883, 99892, 99896], 18),
    "cfg3": (None, -1),  # HILTI fisheye + corridor scene: no CUDA bench line this round, the pin itself is what is checked
    "cfg4": ([259473, 259653, 259654, 259637, 259637], None),
    "cfg5": ([299848, 299903, 299906, 299902, 299902], 13),
}


@needs_ref
@pytest.mark.parametrize("name", ["cfg2", "cfg3", "cfg4", "cfg5"])
def test_oracle_reproduces_the_reference_source_on_the_baseline_configs(name):
    """The frames bench.py times (BASELINE config 2: 100 k points against a 1 M-point map + 2 000 patches; config 4: 260 k
    points; config 5: 300 k points + 4 000 patches, 5 levels, voxel 2.0): VoxelMapManager::StateEstimation and
    VIOManager::computeJacobianAndUpdateEKF of the REFERENCE SOURCE against the oracle — the per-iteration matched counts the
    CUDA path reports in its bench lines, posteriors and per-patch errors. (The large frames are generated once and cached
    in synthetic.frame_cache_dir(); without the cache configs 3 to 5 are skipped unless ESIKF_BIG_FRAMES=1.)"""
    import glob

    from fast_livo2_b200 import workloads as W

    if name != "cfg2" and len(glob.glob(os.path.join(S.frame_cache_dir(), "frame_*.pkl"))) < 3 and os.environ.get("ESIKF_BIG_FRAMES") != "1":
        pytest.skip("large frames are not cached in this checkout")
    fr = W.frame(name)
    want_M, want_vio = BASELINE_COUNTS[name]
    r = PIN.get(f"baseline/{name}/lio", lambda: {k: v for k, v in O.ref_lio_state_estimation(fr).items() if k in ("iters", "M", "state")})
    lio = O.OracleLIO(fr["lio_cfg"], fr["ext"])
    lio.set_map(fr["map"])
    o = lio.state_estimation(fr["pts"], fr["state_prior"], fr["state_prior"])
    assert o["iters"] == r["iters"] and np.array_equal(o["M"], r["M"]) and (want_M is None or o["M"].tolist() == want_M)
    assert_state_close(o["state"], r["state"], rot_tol=1e-12, pos_tol=1e-12, cov_tol=1e-10, rest_tol=1e-12)
    if want_vio is None:
        return
    w = O.oracle_warp_patches(fr, o["state"])
    args = (fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], o["state"], o["state"])
    rv = PIN.get(f"baseline/{name}/vio", lambda: {k: v for k, v in O.RefVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args).items() if k in ("state", "errors")})
    ov = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args)
    assert want_vio < 0 or ov["total_iters"] == want_vio
    assert_state_close(ov["state"], rv["state"], rot_tol=1e-11, pos_tol=1e-11, cov_tol=1e-9, rest_tol=1e-11)
    np.testing.assert_allclose(ov["errors"], rv["errors"], rtol=1e-6, atol=1e-4)


# ---------------------------------------------------------------------------------------------------------------------
# The border rule (DESIGN §4): taps use the reference's linear addressing and read 0 outside [0, w·h). Where the reference is
# well defined — a footprint that wraps to the neighbouring row but stays inside the buffer, and warpAffine's explicit
# in-frame test — the oracle must reproduce it bit for bit. Beyond the buffer the reference reads outside img.data
# (undefined), so those cases are checked against the oracle only (tests/test_oracle_numpy_crosscheck.py, tests/test_gpu_vio_border.py).
BORDER_FRAME = dict(seed=2, n_pts=2000, n_map=120_000, n_patches=250, scene_scale=0.5)


def warp_affine_border_cases(cols, rows):
    """(A_cur_ref, px_ref, search_level) whose warpAffine samples fall on both sides of 0 / cols-1 / rows-1 and exactly on
    them: dyadic matrices (exact inverses and determinants, so the sample positions are exact) around reference pixels at
    integer and half-integer distances from the edges, plus a zero matrix (NaN inverse: the patch is left untouched)."""
    mats = [np.eye(2), 2.0 * np.eye(2), 0.5 * np.eye(2), np.array([[1.25, -0.5], [0.5, 1.25]]), np.array([[1.0, 0.5], [0.25, 1.0]])]
    pxs = [(cols - 4.0, 200.0), (cols - 3.5, 300.5), (cols - 1.0, 250.25), (cols - 1.5, 260.0), (0.0, 220.0), (3.0, 230.5), (0.5, 240.0),
           (320.0, rows - 4.0), (321.5, rows - 2.5), (300.25, rows - 1.0), (310.0, 0.0), (305.5, 2.0), (cols - 3.0, rows - 3.0), (2.0, 1.0),
           (cols - 1.0, rows - 1.0), (0.0, 0.0)]
    cases = [(A, np.array(px), sl) for sl in range(3) for A in mats for px in pxs]
    cases.append((np.zeros((2, 2)), np.array([cols - 4.0, 200.0]), 0))
    return cases


def _border_inputs(in_buffer_only):
    fr = get_frame(**BORDER_FRAME)
    prior = _prior(fr)
    return fr, prior, VB.border_patch_set(fr, prior, in_buffer_only=in_buffer_only)


@needs_ref
def test_oracle_image_patch_at_the_border_reproduces_the_reference_source():
    """getImagePatch (vio.cpp:203-225) at left / right edge pixels, levels 0..3: reads that wrap to the neighbouring row."""
    fr = get_frame(**BORDER_FRAME)
    cam, L = fr["cam_cfg"], fr["vio_cfg"].levels
    pcs, _ = VB.edge_pixels(cam.width, cam.height, L, np.random.default_rng(4))
    # getImagePatch reads columns x0 + s .. x1 - s of updateState's footprint box
    wraps = sum(int(((x0 + (1 << l) < 0) | (x1 - (1 << l) > cam.width - 1)).sum()) for l in range(L)
                for x0, x1, _, _ in [VB.footprint_box(pcs, 1 << l)])
    assert wraps >= 60, wraps  # patch reads that leave the image row (counted here, independently of both sides)

    def ref():
        r = O.RefVIO(cam, fr["ext"], fr["vio_cfg"])
        return dict(patch=np.array([[r.get_image_patch(fr["img"], pc, lvl) for lvl in range(L)] for pc in pcs]))

    r = PIN.get("border/image_patch", ref, exact=("patch",))
    orc = O.OracleVIO(cam, fr["ext"], fr["vio_cfg"])
    assert O.same(np.array([[orc.get_image_patch(fr["img"], pc, lvl) for lvl in range(L)] for pc in pcs]), r, "patch")


@needs_ref
def test_oracle_warp_affine_at_the_border_reproduces_the_reference_source():
    """warpAffine (vio.cpp:292-318): samples across and exactly on 0 / cols-1 / rows-1, search levels 0..2, all levels."""
    fr = get_frame(**BORDER_FRAME)
    cam = fr["cam_cfg"]
    cases = warp_affine_border_cases(cam.width, cam.height)

    def ref():
        r = O.RefVIO(cam, fr["ext"], fr["vio_cfg"])
        return dict(warp=np.array([r.warp_affine(fr["img_ref"], A, px, sl) for A, px, sl in cases]))

    r = PIN.get("border/warp_affine", ref, exact=("warp",))
    orc = O.OracleVIO(cam, fr["ext"], fr["vio_cfg"])
    got = np.array([orc.warp_affine(fr["img_ref"], A, px, sl) for A, px, sl in cases])
    assert O.same(got, r, "warp")
    assert not got[-1].any()  # singular: untouched
    # both sides of the limits are really sampled: zeros from the in-frame test next to interpolated values in one patch
    mixed = sum(bool((g == 0).any() and (g != 0).any()) for g in got)
    assert mixed >= len(cases) // 3, mixed


@needs_ref
def test_oracle_vio_update_with_border_footprints_reproduces_the_reference_source():
    """computeJacobianAndUpdateEKF on interior patches plus left / right edge patches whose footprints wrap to the neighbouring
    row at every stride 1..32 (search levels forced across 0..2), inside the buffer: the tolerances of
    test_oracle_vio_update_reproduces_the_reference_source."""
    fr, prior, bs = _border_inputs(in_buffer_only=True)
    assert bs["n_leave"] >= 30, bs["n_leave"]
    args = (fr["img"], bs["vis_pos"], bs["warp_patch"], bs["search_levels"], bs["inv_ref_expo"], prior, prior)
    ref = PIN.get("border/update", lambda: {k: v for k, v in O.RefVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args).items() if k in ("state", "errors", "H_T_H")})
    orc = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args)
    assert orc["total_iters"] >= 4 and (orc["accepted_per_level"] < orc["iters_per_level"]).any()  # real accept / rollback decisions
    assert_state_close(orc["state"], ref["state"], rot_tol=1e-11, pos_tol=1e-11, cov_tol=1e-9, rest_tol=1e-11)
    np.testing.assert_allclose(orc["errors"], ref["errors"], rtol=1e-6, atol=1e-4)
    blocks = orc["HTH"].reshape(-1, 7, 7)
    blocks = blocks[np.abs(blocks).max(axis=(1, 2)) > 0]
    want = ref["H_T_H"][:7, :7]
    assert min(np.abs(b - want).max() / np.abs(want).max() for b in blocks) < 1e-10
