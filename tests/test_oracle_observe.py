"""CPU: the oracle's restatement of updateVisualMapPoints (oracle/orc_observe.cpp: the converged skip, w2c, delta_pose of the
oldest observation, delta_p, delta_theta, the pixel distance and the level-0 patch of every added entry) bit for bit against
the reference source's own updateVisualMapPoints (live where oracle/_ref is built, else tests/golden/ref_pin/observe.npz), on
the pinhole, distorted-pinhole and fisheye cameras and on hand-built entries at every boundary of the add rule."""
import math
import os

import numpy as np
import pytest

import observe_cases as OC

HAVE_PIN = OC.ref_observe_available() or os.path.exists(OC.GOLDEN)


def _run(lib_class, keys):
    out = {}
    for name, sc in OC.pin_scenes().items():
        r = lib_class(sc).run(sc)
        for k in keys:
            out[f"{name}/{k}"] = np.ascontiguousarray(r[k])
    return out


def reference_pins():
    """The reference source's outputs on the pin scenes (the generator of tests/golden/ref_pin/observe.npz calls this)."""
    return _run(OC.RefObserve, OC.PIN_KEYS)


def oracle_pins():
    return _run(OC.OracleObserve, OC.FIELDS)


def _want():
    return reference_pins() if OC.ref_observe_available() else dict(np.load(OC.GOLDEN))


@pytest.mark.skipif(not HAVE_PIN, reason="needs oracle/_ref (reference source) or the stored pin")
def test_new_observations_are_pinned_to_the_reference_source():
    got, want = oracle_pins(), _want()
    assert set(want) == {f"{name}/{k}" for name in OC.pin_scenes() for k in OC.PIN_KEYS}
    for k in got:
        assert got[k].shape == want[k].shape and got[k].tobytes() == want[k].tobytes(), k
    scenes = OC.pin_scenes()
    for name, sc in scenes.items():
        flag, entry = want[f"{name}/update_flag"], want[f"{name}/entry"]
        assert 0 < flag.sum() < len(flag) - sc["converged"].sum(), name  # some entries are added, some are not
        assert not flag[sc["converged"] == 1].any(), name
        # the new Feature's level is the selection's search level of its entry
        assert np.array_equal(want[f"{name}/level"], sc["search_levels"][entry]), name
    assert np.array_equal(want["edge/update_flag"], scenes["edge"]["expect"])


def test_stored_pin_matches_the_live_reference():
    if not (OC.ref_observe_available() and os.path.exists(OC.GOLDEN)):
        pytest.skip("needs both oracle/_ref and the stored pin")
    want, live = dict(np.load(OC.GOLDEN)), reference_pins()
    assert set(want) == set(live)
    for k in want:
        assert want[k].tobytes() == live[k].tobytes(), k


def test_hand_built_entries_get_the_flags_they_should():
    """delta_p exactly 0.5 and one ulp above, delta_theta on both sides of 0.3 (from the host's acos bound), the trace on
    both sides of 3 - 1e-6, acos's NaN below x = -1, the pixel distance exactly 40 and one ulp above, converged entries,
    border footprints, and observation counts of 29, 30 and 31."""
    sc = OC.edge_scene()
    r = OC.OracleObserve(sc).run(sc)
    assert np.array_equal(r["update_flag"], sc["expect"])
    assert np.array_equal(r["entry"], np.nonzero(sc["expect"])[0])
    p = sc["pos"][r["entry"]]
    assert np.array_equal(r["pc"], np.stack([512.0 * p[:, 0] / p[:, 2] + 320.0, 512.0 * p[:, 1] / p[:, 2] + 256.0], 1))  # exact projections
    assert (r["patch"] >= 0).all() and (r["patch"] <= 255).all()


def test_the_acos_bound_splits_the_host_acos():
    """acos(x) > 0.3 exactly when -1 <= x <= c*, on the ulps around c*, the grid of 0.5 * (trace - 1) near it, and -1."""
    c = OC.acos_bound()
    x = c
    for _ in range(2000):
        x = np.nextafter(x, -np.inf)
    for _ in range(4001):
        assert (math.acos(x) > 0.3) == (x <= c), x
        x = np.nextafter(x, np.inf)
    for t in np.linspace(2.9, 2.92, 20001):
        xt = 0.5 * (float(t) - 1.0)
        assert (math.acos(xt) > 0.3) == (-1.0 <= xt <= c), t
    assert math.acos(-1.0) > 0.3
    with pytest.raises(ValueError):  # NaN in C: no add
        math.acos(float(np.nextafter(-1.0, -np.inf)))
