"""CPU: the oracle's restatement of the visual sub-map selection (oracle/orc_select.cpp, the per-candidate tail of
retrieveFromVisualSparseMap) — its depth-form warp matrix, search level and calculateNCC bit for bit against the reference
source's own (live where oracle/_ref is built, else tests/golden/ref_pin/select.npz), the warp_map cache owner, and the gate
boundaries."""
import os

import numpy as np
import pytest

import select_cases as SC
from oracle_bind import OracleVIO

HAVE_PIN = SC.ref_select_available() or os.path.exists(SC.GOLDEN)


def _oracle_pins():
    out = {}
    for camera in SC.PIN_CAMERAS:
        o = SC.OracleSelect(SC.W.CAMERAS[camera])
        cases = SC.pin_matrix_cases(o, camera)
        res = [o.warp_matrix_affine(**k) for k in cases]
        out[f"{camera}/A"] = np.array([r[0] for r in res])
        out[f"{camera}/level"] = np.array([r[1] for r in res], np.int32)
    ref, cur = SC.pin_ncc_cases()
    o = SC.OracleSelect(SC.W.CAMERAS["radtan"])
    out["ncc"] = np.array([o.ncc(ref[i], cur[i]) for i in range(len(ref))])
    return out


def reference_pins():
    """The reference source's outputs on the pin cases (the generator of tests/golden/ref_pin/select.npz calls this)."""
    out = {}
    for camera in SC.PIN_CAMERAS:
        o = SC.OracleSelect(SC.W.CAMERAS[camera])  # only to bisect the det crossings; the inputs are then fixed
        r = SC.RefSelect(SC.W.CAMERAS[camera])
        res = [r.warp_matrix_affine(**k) for k in SC.pin_matrix_cases(o, camera)]
        out[f"{camera}/A"] = np.array([x[0] for x in res])
        out[f"{camera}/level"] = np.array([x[1] for x in res], np.int32)
    ref, cur = SC.pin_ncc_cases()
    r = SC.RefSelect(SC.W.CAMERAS["radtan"])
    out["ncc"] = np.array([r.ncc(ref[i], cur[i]) for i in range(len(ref))])
    return out


@pytest.mark.skipif(not HAVE_PIN, reason="needs oracle/_ref (reference source) or the stored pin")
def test_depth_warp_matrix_and_ncc_are_pinned_to_the_reference_source():
    got = _oracle_pins()
    want = reference_pins() if SC.ref_select_available() else dict(np.load(SC.GOLDEN))
    for camera in SC.PIN_CAMERAS:
        A, lv = got[f"{camera}/A"], got[f"{camera}/level"]
        assert np.array_equal(A.view(np.uint64), want[f"{camera}/A"].view(np.uint64)), camera
        assert np.array_equal(lv, want[f"{camera}/level"]), camera
        assert set(lv.tolist()) == {0, 1, 2}, camera
        # the det crossings: the last four cases straddle 3 and 12 on adjacent inputs
        assert lv[-4] == 0 and lv[-3] == 1 and lv[-2] == 1 and lv[-1] == 2, lv[-4:]
        assert np.isfinite(A).all()
    assert np.array_equal(got["ncc"].view(np.uint64), want["ncc"].view(np.uint64))
    assert abs(got["ncc"][0]) < 1e-3 and abs(got["ncc"][2]) == 0.0  # zero-variance patches: the 1e-10 keeps the quotient finite


def test_depth_form_cache_owner_is_the_first_candidate_of_each_key():
    """Candidates sharing a ref_key take the first one's A and level, even where their own geometry gives another A."""
    c = SC.candidates("radtan", 64, n_frames=5, seed=3)
    o = SC.OracleSelect(c["camcfg"])
    r = o.select(c, normal_en=False, outlier_threshold=1e30)
    seen = {}
    differ = 0
    for i, key in enumerate(c["ref_key"].tolist()):
        own, own_sl = o.warp_matrix_affine(c["px_ref"][i], c["ref_f"][i], c["ref_pos"][i], c["pos_w"][i], c["T_ref"][i], c["T_cur"], c["ref_level"][i])
        if key not in seen:
            seen[key] = i
            assert np.array_equal(r["A_cur_ref"][i].ravel(), own) and r["search_levels"][i] == own_sl
        else:
            j = seen[key]
            assert np.array_equal(r["A_cur_ref"][i], r["A_cur_ref"][j]) and r["search_levels"][i] == r["search_levels"][j]
            differ += not np.array_equal(r["A_cur_ref"][i].ravel(), own)
    assert len(seen) == 5 and differ > 40
    assert r["keep"].all() and np.array_equal(r["kept"], np.arange(64))


def test_gate_boundaries():
    """error == outlier_threshold * 64 is kept, one double ulp below the error it is dropped; ncc == ncc_thre is kept, one
    ulp above it is dropped; survivors keep candidate order."""
    c = SC.candidates("pinhole", 40, seed=4)
    o = SC.OracleSelect(c["camcfg"])
    base = o.select(c, outlier_threshold=1e30)
    err = base["errors"].astype(np.float64)
    j = int(np.argsort(err)[20])
    at = o.select(c, outlier_threshold=err[j] / 64)
    assert at["keep"][j] and np.array_equal(at["kept"], np.nonzero(err <= err[j])[0])
    below = o.select(c, outlier_threshold=np.nextafter(err[j], -np.inf) / 64)
    assert not below["keep"][j] and np.array_equal(below["kept"], np.nonzero(err < err[j])[0])
    v = OracleVIO(c["camcfg"], SC.W.EXT, SC.S.VioCfg(levels=4))  # getImagePatch of the current patches
    ncc = np.array([o.ncc(base["warp_patch"][i][:64], v.get_image_patch(c["img"], c["pc"][i], 0)) for i in range(40)])
    on = o.select(c, ncc_en=True, ncc_thre=ncc[j], outlier_threshold=1e30)
    assert on["keep"][j] and np.array_equal(on["kept"], np.nonzero(ncc >= ncc[j])[0])
    off = o.select(c, ncc_en=True, ncc_thre=np.nextafter(ncc[j], np.inf), outlier_threshold=1e30)
    assert not off["keep"][j] and np.array_equal(off["kept"], np.nonzero(ncc > ncc[j])[0])
