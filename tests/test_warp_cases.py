"""The oracle's VIO warp producers on the hand-built sets of tests/warp_cases.py, and the reference source on a subset of
them (through oracle_bind.RefPin, stored under warp/* in tests/golden/ref_pin/vio.npz)."""
import numpy as np
import pytest

import oracle_bind as O
import warp_cases as W
from fast_livo2_b200 import synthetic as S
from parity_util import assert_state_close
from test_oracle_ref_pin_vio import PIN, needs_ref

EXT = S.avia_extrinsics()


def oracle_warp_matrix(camera, case, idx=None, levels=4):
    vio = O.OracleVIO(W.CAMERAS[camera], EXT, S.VioCfg(levels=levels))
    idx = range(len(case["px_ref"])) if idx is None else idx
    A, sl = zip(*[vio.warp_matrix(case["px_ref"][i], case["pos_w"][i], case["normal_w"][i], (case["T_ref"][0][i], case["T_ref"][1][i]), W.T_CUR) for i in idx])
    return np.array(A), np.array(sl, np.int32)


@pytest.fixture(scope="module", params=[(c, t) for c in W.CAMERAS for t in W.THRESHOLDS], ids=lambda p: f"{p[0]}-{p[1]:g}")
def threshold(request):
    camera, thr = request.param
    case = W.threshold_set(camera, thr)
    return camera, thr, case, oracle_warp_matrix(camera, case)


def test_search_level_rule():
    D = np.array([np.nextafter(3.0, 0), 3.0, np.nextafter(3.0, 4), np.nextafter(12.0, 0), 12.0, np.nextafter(12.0, 13), 48.5, 1e300, -5.0, np.nan])
    assert W.search_level(D).tolist() == [0, 0, 1, 1, 1, 2, 2, 2, 0, 0]
    # a00 a11 = 1 + 2^-29 + 2^-60: rounded first it loses the 2^-60, the single-rounded form keeps it
    a = 1.0 + 2.0 ** -30
    A = np.array([[a, 1.0], [1.0, a]])
    assert W.det_rounded(A)[0] == 2.0 ** -29 and W.det_contracted(A)[0] == 2.0 ** -29 + 2.0 ** -60


def test_oracle_search_level_is_the_rule_on_its_own_A(threshold):
    """getBestSearchLevel of the oracle, on geometries bisected onto D = 3 / 12: the rule on its own A, and both reach flags
    (|D - thr| <= 1 ulp; the contracted determinant deciding differently) occur."""
    camera, thr, case, (A, sl) = threshold
    assert len(A) >= 20_000
    assert np.array_equal(sl, W.search_level(W.det_rounded(A)))
    near, split = W.reach(A, thr)
    assert near.sum() >= 50 and split.sum() >= 5, (near.sum(), split.sum())
    # the oracle follows the restatement here to well below the 1e-10 the device is held to
    np.testing.assert_allclose(A, case["A"], rtol=0, atol=1e-12)


@pytest.mark.parametrize("camera", list(W.CAMERAS))
def test_oracle_edge_geometries(camera):
    e = W.edge_set(camera)
    A, sl = oracle_warp_matrix(camera, e)
    assert np.array_equal(sl, W.search_level(W.det_rounded(A)))
    for i, want in enumerate(e["want_level"]):
        assert want is None or sl[i] == want, (e["name"][i], sl[i])
    h0 = np.array([nm.startswith("h_zero") for nm in e["name"]])
    assert np.isnan(A[h0]).all() and not np.isnan(A[~h0]).any()
    # warpAffine leaves the patch of a NaN matrix untouched
    vio = O.OracleVIO(W.CAMERAS[camera], EXT, S.VioCfg(levels=4))
    img = np.full((W.CAMERAS[camera].height, W.CAMERAS[camera].width), 200, np.uint8)
    for i in np.nonzero(h0)[0]:
        assert not vio.warp_affine(img, A[i], e["px_ref"][i], int(sl[i])).any()
    assert (W.det_rounded(A)[~h0] < 0).sum() >= 2


def test_caller_matrices_are_cancelling():
    A, px, sl, img = W.caller_matrices()
    n = len(A)
    fr = W.float_inverse(A.reshape(n, 4), W.det_rounded(A))
    fc = W.float_inverse(A.reshape(n, 4), W.det_contracted(A))
    assert (fr != fc).any(1).all()
    assert (np.abs(A) >= 2.0 ** 22).all() and (np.abs(fr) < 64).all()
    inside = W.samples_inside(A, px, sl, *img.shape)
    assert (inside[sl == 0] > 0).all() and set(sl.tolist()) == set(W.CALLER_SEARCH_LEVELS)


# ---------------------------------------------------------------------------------------------------------------------
# the reference source
@needs_ref
@pytest.mark.parametrize("camera", list(W.CAMERAS))
def test_reference_search_level_on_threshold_cases(camera):
    """getWarpMatrixAffineHomography + getBestSearchLevel of the reference source on the near-threshold cases: its level is
    the rule on its own A, and its A is within 1e-11 of the oracle's (near a threshold the two levels may differ, since the
    A differ in the last bits)."""
    sub = {}
    for thr in W.THRESHOLDS:
        case = W.threshold_set(camera, thr)
        sub[thr] = (case, np.nonzero(np.abs(W.det_rounded(case["A"]) - thr) <= 4 * np.spacing(thr))[0][:150])

    def ref():
        r = O.RefVIO(W.CAMERAS[camera], EXT, S.VioCfg(levels=4))
        out = {}
        for thr, (case, idx) in sub.items():
            A, sl = zip(*[r.warp_matrix(case["px_ref"][i], case["pos_w"][i], case["normal_w"][i], (case["T_ref"][0][i], case["T_ref"][1][i]), W.T_CUR) for i in idx])
            out[f"A_{thr:g}"], out[f"level_{thr:g}"] = np.array(A), np.array(sl, np.int32)
        return out

    r = PIN.get(f"warp/threshold/{camera}", ref)
    for thr, (case, idx) in sub.items():
        assert len(idx) >= 100
        Ar, slr = r[f"A_{thr:g}"], r[f"level_{thr:g}"]
        assert np.array_equal(slr, W.search_level(W.det_rounded(Ar)))
        Ao, _ = oracle_warp_matrix(camera, case, idx)
        np.testing.assert_allclose(Ar, Ao, rtol=0, atol=1e-11)


@needs_ref
def test_reference_warp_affine_on_caller_matrices():
    """warpAffine of the reference source on the cancelling matrices, pyramid depths 1..8: bit for bit."""
    A, px, sl, img = W.caller_matrices()

    def ref():
        out = {}
        for L in range(1, 9):
            r = O.RefVIO(W.CAMERAS["pinhole"], EXT, S.VioCfg(levels=L))
            out[f"warp_{L}"] = np.array([r.warp_affine(img, A[i], px[i], int(sl[i])) for i in range(len(A))])
        return out

    r = PIN.get("warp/caller", ref, exact=tuple(f"warp_{L}" for L in range(1, 9)))
    for L in range(1, 9):
        vio = O.OracleVIO(W.CAMERAS["pinhole"], EXT, S.VioCfg(levels=L))
        got = np.array([vio.warp_affine(img, A[i], px[i], int(sl[i])) for i in range(len(A))])
        assert O.same(got, r, f"warp_{L}"), L
        assert (got != 0).any()


@needs_ref
def test_reference_vio_update_at_eight_levels_and_eight_iterations():
    """computeJacobianAndUpdateEKF of the reference source over 8 pyramid levels, 8 iterations each, on central patches whose
    taps stay inside the image buffer at every level (tap strides up to 128): the tolerances of
    test_oracle_vio_update_reproduces_the_reference_source."""
    fr, prior, pt = W.deep_frame(8, pinned=True)
    args = (fr["img"], pt["vis_pos"], pt["warp_patch"], pt["search_levels"], pt["inv_ref_expo"], prior, prior)
    ref = PIN.get("warp/deep8", lambda: {k: v for k, v in O.RefVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args).items() if k in ("state", "errors")})
    orc = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args)
    assert (orc["iters_per_level"][:8] > 0).all() and orc["total_iters"] > 8
    assert_state_close(orc["state"], ref["state"], rot_tol=1e-11, pos_tol=1e-11, cov_tol=1e-9, rest_tol=1e-11)
    np.testing.assert_allclose(orc["errors"], ref["errors"], rtol=1e-6, atol=1e-4)
