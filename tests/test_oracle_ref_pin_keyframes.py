"""Pins the VIO oracle against the REFERENCE'S OWN SOURCE (oracle/_ref/libfl2_ref_vio.so, see test_oracle_ref_pin_vio.py) on
visual sub-maps drawn from many keyframes (tests/keyframe_cases.py): K = 12 keyframes rendered from the frame's own scene
with exposure gains over [0.6, 1.5], so every patch has its own inverse reference exposure, reference image and reference
pose, and a current image rendered with a gain of 1.25 (true inverse exposure 0.8, prior near 1). Forward update with
exposure estimation on and off, three levels with mixed search levels, a distorted pinhole; the inverse-compositional
variant with per-patch ref_R / ref_pos / ref_f and 12 reference images.

Where oracle/_ref is built the reference runs live; elsewhere the cases compare with its stored outputs
(tests/golden/ref_pin/keyframes.npz, re-recorded with FL2_RECORD_REF_PIN=1). The discrimination checks at the end show that
these inputs catch an update that reads the wrong patch's exposure or reference data."""
import numpy as np
import pytest

import keyframe_cases as KC
import oracle_bind as O
from fast_livo2_b200 import synthetic as S
from parity_util import assert_state_close

KF_PIN = O.RefPin("keyframes")
needs_ref = pytest.mark.skipif(not O.RefPin.available("keyframes"), reason="neither oracle/_ref/libfl2_ref_vio.so nor tests/golden/ref_pin/keyframes.npz")

FORWARD = ["pinhole", "pinhole_gain", "pinhole_expo_off", "pinhole_gain_expo_off", "three_levels_mixed", "distorted_gain"]
INVERSE = ["pinhole_gain", "distorted_gain"]
STATE_TOL = dict(rot_tol=1e-11, pos_tol=1e-11, cov_tol=1e-9, rest_tol=1e-11)


def _pos_diff(a, b):
    return float(np.linalg.norm(S.unpack_state(a)["p"] - S.unpack_state(b)["p"]))


@needs_ref
@pytest.mark.parametrize("name", FORWARD)
def test_oracle_keyframe_update_reproduces_the_reference_source(name):
    c = KC.build(name)
    args = KC.update_args(c)
    ref = KF_PIN.get(f"update/{name}", lambda: {k: v for k, v in O.RefVIO(c["cam_cfg"], c["ext"], c["vio_cfg"]).update(*args).items() if k in ("state", "errors")})
    orc = KC.oracle(c).update(*args)
    assert orc["total_iters"] >= 4
    assert_state_close(orc["state"], ref["state"], **STATE_TOL)
    np.testing.assert_allclose(orc["errors"], ref["errors"], rtol=1e-6, atol=1e-4)


@needs_ref
@pytest.mark.parametrize("name", INVERSE)
def test_oracle_keyframe_inverse_variant_reproduces_the_reference_source(name):
    c = KC.build(name)
    args = KC.update_args(c)
    ref = KF_PIN.get(f"update_inverse/{name}", lambda: O.RefVIO(c["cam_cfg"], c["ext"], c["vio_cfg"]).update_inverse(*args[:5], c["refs"], c["prior"], c["prior"]))
    orc = KC.oracle(c, inverse=True).update(*args)
    assert orc["total_iters"] >= 4
    assert_state_close(orc["state"], ref["state"], **STATE_TOL)
    np.testing.assert_allclose(orc["errors"], ref["errors"], rtol=1e-6, atol=1e-4)


def test_keyframe_sub_map_shape():
    """Every keyframe serves patches, neighbours (one warp's patches) and a point's replicas come from different keyframes,
    the exposures span the gain range, and the exposure of the current image is estimated towards its truth."""
    c = KC.build("pinhole_gain")
    idx = c["ref_idx"]
    assert set(idx.tolist()) == set(range(c["K"]))
    assert np.mean(idx[1:] != idx[:-1]) > 0.9
    np.testing.assert_array_equal(c["inv_ref_expo"], 1.0 / c["gains"][idx])
    assert c["inv_ref_expo"].min() < 0.7 and c["inv_ref_expo"].max() > 1.6
    for i in np.nonzero(idx[1:] != idx[:-1])[0][:8]:  # a warp's neighbouring patches read different reference images
        assert not np.array_equal(c["ref_imgs"][idx[i]], c["ref_imgs"][idx[i + 1]])
    o = KC.oracle(c).update(*KC.update_args(c))
    assert abs(o["state"][12] - 0.8) < abs(c["prior"][12] - 0.8) / 4  # the prior starts near 1
    r = KC.build("pinhole_5k")
    assert len(r["rep"]) > 4224 and np.bincount(r["rep"]).min() >= 12
    for p in range(0, 300, 37):  # the replicas of one point: different keyframes, so different warp patches and exposures
        ks = r["ref_idx"][r["rep"] == p]
        assert np.all(ks[1:] != ks[:-1]) and len(np.unique(ks)) >= c["K"] - 1, ks
    s = KC.build("pinhole_sorted")["ref_idx"]
    assert np.all(np.diff(s) >= 0)


def test_keyframe_inputs_discriminate_the_exposure_list():
    """An update that reads inv_ref_expo = 1 (or another patch's entry) ends far outside compare_vio's tolerances."""
    for name in ("pinhole_gain", "distorted_gain"):
        c = KC.build(name)
        good = KC.oracle(c).update(*KC.update_args(c))
        ones = KC.oracle(c).update(*KC.update_args(c, np.ones(len(c["vis_pos"]))))
        shifted = KC.oracle(c).update(*KC.update_args(c, np.roll(c["inv_ref_expo"], 1)))
        assert _pos_diff(good["state"], ones["state"]) > 1e-4, name
        assert _pos_diff(good["state"], shifted["state"]) > 1e-4, name
        assert np.abs(good["errors"] - ones["errors"]).max() > 1e2


def test_keyframe_inputs_discriminate_the_inverse_reference_data():
    """The inverse variant with reference image 0 and patch 0's ref_R / ref_pos for every patch (a precompute that reads the
    wrong patch's reference data) ends far outside compare_vio's tolerances; so does one that reads only the wrong image."""
    c = KC.build("pinhole_gain")
    n = len(c["ref_idx"])
    args = KC.update_args(c)
    good = KC.oracle(c, inverse=True).update(*args)
    refs = c["refs"]
    bad_all = dict(refs, ref_img_index=np.zeros(n, np.int32), ref_R=np.tile(refs["ref_R"][0], (n, 1)), ref_pos=np.tile(refs["ref_pos"][0], (n, 1)))
    bad_img = dict(refs, ref_img_index=np.zeros(n, np.int32))
    bad_pose = dict(refs, ref_R=np.tile(refs["ref_R"][0], (n, 1)), ref_pos=np.tile(refs["ref_pos"][0], (n, 1)))
    for bad in (bad_all, bad_img, bad_pose):
        o = KC.oracle(c, inverse=True, refs=bad).update(*args)
        assert _pos_diff(good["state"], o["state"]) > 1e-4
