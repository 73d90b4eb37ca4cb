"""CPU: the oracle's restatement of generateVisualMapPoints (oracle/orc_generate.cpp: the isInFrame gate, the grid cell, the
TYPE_MAP mask, vk::shiTomasiScore, the strict per-cell maximum over the scan then add_from, the cos_theta sign of the normal
and the level-0 patch) bit for bit against the reference source's own generateVisualMapPoints (live where oracle/_ref is
built, else tests/golden/ref_pin/generate.npz), on the pinhole, distorted-pinhole and fisheye cameras and on hand-built
points at every boundary."""
import os

import numpy as np
import pytest

import generate_cases as GC

HAVE_PIN = GC.ref_generate_available() or os.path.exists(GC.GOLDEN)


def _run(lib_class):
    out = {}
    for name, sc in GC.pin_scenes().items():
        r = lib_class(sc).run(sc)
        for k in GC.PIN_KEYS:
            out[f"{name}/{k}"] = np.ascontiguousarray(r[k])
    return out


def reference_pins():
    """The reference source's outputs on the pin scenes (the generator of tests/golden/ref_pin/generate.npz calls this)."""
    return _run(GC.RefGenerate)


def oracle_pins():
    return _run(GC.OracleGenerate)


@pytest.mark.skipif(not HAVE_PIN, reason="needs oracle/_ref (reference source) or the stored pin")
def test_new_points_are_pinned_to_the_reference_source():
    got = oracle_pins()
    want = reference_pins() if GC.ref_generate_available() else dict(np.load(GC.GOLDEN))
    assert set(got) == set(want)
    for k in got:
        assert got[k].shape == want[k].shape and got[k].tobytes() == want[k].tobytes(), k
    for name in GC.PIN_SCENES:
        assert len(got[f"{name}/cell"]) > 100, name  # most cells of every camera get a point
    assert len(got["pinhole_n10/cell"]) == 0 and len(got["pinhole_n11/cell"]) > 0


def test_stored_pin_matches_the_live_reference():
    if not (GC.ref_generate_available() and os.path.exists(GC.GOLDEN)):
        pytest.skip("needs both oracle/_ref and the stored pin")
    want, live = dict(np.load(GC.GOLDEN)), reference_pins()
    assert set(want) == set(live)
    for k in want:
        assert want[k].tobytes() == live[k].tobytes(), k


@pytest.mark.parametrize("border", [80, 0])
def test_hand_built_points_win_the_cells_they_should(border):
    """Exact ties (the first point wins), a flat patch, zero normals, TYPE_MAP cells, border and cell edges, add_from ties
    (the scan keeps the cell) and wins (strictly greater, or the first of tied add_from points in an empty cell)."""
    sc = GC.edge_scene(border)
    r = GC.OracleGenerate(sc).run(sc)
    won = dict(zip(r["cell"].tolist(), r["source"].tolist()))
    for c, s in sc["expect"].items():
        assert won.get(c) == s, (c, won.get(c), s)
    assert sc["c_add"] in won.values()  # the better add_from pixel took its cell from the scan
    assert np.all(np.diff(r["cell"]) > 0)  # cell order
    assert (r["score"] > 0).all() and not (sc["mask"][r["cell"]]).any()
    n = len(sc["point_w"])
    for i, s in enumerate(r["source"]):
        src = sc["point_w"][s] if s < n else sc["add_pos"][s ^ GC.ADD_FROM]
        nv = sc["normal"][s] if s < n else sc["add_normal"][s ^ GC.ADD_FROM]
        assert np.array_equal(r["pos"][i], src)
        assert np.array_equal(np.abs(r["normal"][i]), np.abs(nv)) and (r["normal"][i] @ r["pos"][i]) >= 0  # turned away from the camera
        assert np.array_equal(r["var"][i], sc["var"][s] if s < n else np.zeros((3, 3)))
    if border:
        u = r["pc"][:, 0].astype(int)
        assert u.min() >= border and u.max() < 640 - border


def test_pg_of_ten_points_gives_nothing():
    sc = GC.scene("pinhole", 200, seed=8, n_add=50, map_share=0.0)
    orc = GC.OracleGenerate(sc)
    assert len(orc.run(GC.truncated(sc, 10))["cell"]) == 0
    assert len(orc.run(GC.truncated(sc, 11))["cell"]) > 0
