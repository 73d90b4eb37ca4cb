"""CPU: the oracle's restatement of the coloured scan (oracle/orc_color.cpp: the world cloud of RGBpointBodyToWorld and
publish_frame_world's gates and getInterpolatedPixel) bit for bit against the reference source's own pieces (live where
oracle/_ref is built, else tests/golden/ref_pin/color.npz), on the pinhole, distorted-pinhole and fisheye cameras and on
hand-built points at every gate boundary."""
import os

import numpy as np
import pytest

import color_cases as CC

HAVE_PIN = CC.ref_color_available() or os.path.exists(CC.GOLDEN)


def _run(lib_class):
    out = {}
    for name, sc in CC.pin_scenes().items():
        r = lib_class(sc).publish(sc)
        for k in CC.PIN_KEYS:
            out[f"{name}/{k}"] = np.ascontiguousarray(r[k])
    return out


def reference_pins():
    """The reference source's outputs on the pin scenes (the generator of tests/golden/ref_pin/color.npz calls this)."""
    return _run(CC.RefColor)


def oracle_pins():
    return _run(CC.OracleColor)


@pytest.mark.skipif(not HAVE_PIN, reason="needs oracle/_ref (reference source) or the stored pin")
def test_coloured_scan_is_pinned_to_the_reference_source():
    got = oracle_pins()
    want = reference_pins() if CC.ref_color_available() else dict(np.load(CC.GOLDEN))
    assert set(got) == set(want)
    for k in got:
        assert got[k].shape == want[k].shape and got[k].tobytes() == want[k].tobytes(), k
    for name in CC.PIN_SCENES:
        assert len(got[f"{name}/index"]) > 150, name  # every camera keeps a real share of the cloud


def test_stored_pin_matches_the_live_reference():
    if not (CC.ref_color_available() and os.path.exists(CC.GOLDEN)):
        pytest.skip("needs both oracle/_ref and the stored pin")
    want, live = dict(np.load(CC.GOLDEN)), reference_pins()
    assert set(want) == set(live)
    for k in want:
        assert want[k].tobytes() == live[k].tobytes(), k


def test_hand_built_points_fall_where_the_gates_put_them():
    """Behind the camera, pf[2] == 0, pc in (-1, 0), (int)pc at 3 / width - 4 / width - 3 (and rows), exact integers,
    pf.norm() == blind_rgb_points (strict), the saturated corners."""
    sc = CC.edge_scene()
    r = CC.OracleColor(sc).publish(sc)
    kept = np.zeros(len(sc["pts"]), bool)
    kept[r["index"]] = True
    assert np.array_equal(kept, sc["keep"]), np.nonzero(kept != sc["keep"])[0]
    assert np.array_equal(r["index"], np.nonzero(sc["keep"])[0])  # cloud order
    assert np.array_equal(r["xyz"], sc["pts"][r["index"]])
    img = sc["img"]
    for i, k in enumerate(r["index"]):
        x, y, z = sc["pts"][k].astype(np.float64)
        u, v = 512.0 * x / z + 320.0, 512.0 * y / z + 256.0
        if u == int(u) and v == int(v):  # all the weight on one tap: the pixel itself
            assert np.array_equal(r["bgr"][i], img[int(v), int(u)]), (k, u, v)
        if u < 8 and v < 8:  # inside a saturated corner block
            assert (r["bgr"][i] >= 254).all(), (k, r["bgr"][i])


def test_world_cloud_is_the_float_of_the_double_transform():
    sc = CC.scene("fisheye", 500, seed=9)
    w = CC.OracleColor(sc).world(sc["pts"], sc["lio_state"])
    st = sc["lio_state"]
    R, t = st[:9].reshape(3, 3), st[9:12]
    e = sc["ext"]
    p = sc["pts"].astype(np.float64)
    want = ((p @ e.extR.T + e.extT) @ R.T + t).astype(np.float32)
    assert np.abs(w.astype(np.float64) - want).max() <= 4e-6 * np.abs(want).max()
