"""CPU: the oracle's restatement of the scan side of retrieveFromVisualSparseMap (oracle/orc_retrieve.cpp: the voxel keys in
first-occurrence order, the depth image, the map-side walk on a persistent sub_feat_map and the depth check) bit for bit
against the reference source's own resetGrid + retrieveFromVisualSparseMap (live where oracle/_ref is built, else
tests/golden/ref_pin/retrieve.npz), on pinhole, distorted-pinhole and fisheye (config 3) frames, on hand-built points at every
boundary, and over two consecutive frames of one VIOManager."""
import os

import numpy as np
import pytest

import retrieve_cases as RC

HAVE_PIN = RC.ref_retrieve_available() or os.path.exists(RC.GOLDEN)


def _oracle_sequence(scenes):
    """The oracle on consecutive frames with ONE persistent sub_feat_map, as the reference's VIOManager member."""
    orc = RC.OracleRetrieve(scenes[0])
    return [orc.retrieve(sc) for sc in scenes]


def _ref_sequence(scenes):
    ref = RC.RefRetrieve(scenes[0])
    return [ref.run(sc) for sc in scenes]


def _runs(oracle):
    out = {}
    for name, sc in RC.pin_scenes().items():
        r = (_oracle_sequence if oracle else _ref_sequence)([sc])[0]
        out.update({f"{name}/{k}": np.ascontiguousarray(r[k]) for k in RC.PIN_KEYS})
    for i, r in enumerate((_oracle_sequence if oracle else _ref_sequence)(RC.pin_sequence())):
        out.update({f"sequence{i}/{k}": np.ascontiguousarray(r[k]) for k in RC.PIN_KEYS})
    return out


def reference_pins():
    """The reference source's outputs (the generator of tests/golden/ref_pin/retrieve.npz calls this)."""
    return _runs(oracle=False)


def oracle_pins():
    return _runs(oracle=True)


def _want():
    return reference_pins() if RC.ref_retrieve_available() else dict(np.load(RC.GOLDEN))


@pytest.mark.skipif(not HAVE_PIN, reason="needs oracle/_ref (reference source) or the stored pin")
def test_retrieval_is_pinned_to_the_reference_source():
    """sub_feat_map after the walk (iteration order), grid_num, retrieve_voxel_points and the points past the depth check."""
    got, want = oracle_pins(), _want()
    assert set(got) == set(want)
    for k in got:
        assert got[k].shape == want[k].shape and got[k].tobytes() == want[k].tobytes(), k
    for name in list(RC.pin_scenes()) + ["sequence0", "sequence1"]:
        cells = want[f"{name}/grid_type"].sum()
        assert 0 < len(want[f"{name}/survivors"]) < cells, name  # the depth check drops some retrieved points, keeps others


def test_stored_pin_matches_the_live_reference():
    if not (RC.ref_retrieve_available() and os.path.exists(RC.GOLDEN)):
        pytest.skip("needs both oracle/_ref and the stored pin")
    want, live = dict(np.load(RC.GOLDEN)), reference_pins()
    assert set(want) == set(live)
    for k in want:
        assert want[k].tobytes() == live[k].tobytes(), k


def test_first_occurrence_keys_give_the_reference_iteration_order():
    """The keys of orc_retrieve_scan are the scan's distinct keys in first-occurrence order; inserted in that order into the
    persistent map that the previous frame left (its bucket count carries through clear()), they iterate as the reference's
    sub_feat_map does (checked through the pin above, which walks that map), while another insertion order does not."""
    seq = RC.pin_sequence()
    orc = RC.OracleRetrieve(seq[0])
    got = [orc.retrieve(sc) for sc in seq]
    for sc, g in zip(seq, got):
        assert np.array_equal(g["keys"], RC.first_occurrence(RC.voxel_keys(sc["pg"])))
    # the same keys in sorted order, after the same first frame, iterate differently
    orc2 = RC.OracleRetrieve(seq[0])
    orc2.retrieve(seq[0])
    s1 = orc2.scan(seq[1])
    shuffled = orc2.walk(seq[1], np.sort(s1["keys"].view("i8,i8,i8"), axis=0).view(np.int64).reshape(-1, 3))
    assert set(map(tuple, shuffled["sub_keys"].tolist())) == set(map(tuple, got[1]["sub_keys"].tolist()))
    assert not np.array_equal(shuffled["sub_keys"], got[1]["sub_keys"])


def test_hand_built_points():
    """Keys at -0.5, -0.25, -0.0, 0.0 and one ulp around voxel faces; pt_c[2] at 0 and one ulp above; int(px) at border - 1,
    border and width - border; two points on one pixel; |delta| at 0.5 and one ulp above, 0.75; a discontinuous depth only at
    the centre tap; empty taps; a map_dist tie of two voxels in one cell."""
    sc = RC.edge_scene()
    orc = RC.OracleRetrieve(sc)
    s = orc.scan(sc)
    keys = [tuple(k) for k in s["keys"].tolist()]
    for c, k in ((-0.5, -2), (-0.25, -2), (-0.0, 0), (0.0, 0), (np.nextafter(0.5, 0), 0), (0.5, 1), (np.nextafter(-0.5, 0), -2),
                 (np.nextafter(-0.5, -1), -3), (-1.0, -3), (np.nextafter(-1.0, 0), -3), (1e-300, 0), (-1e-300, -2)):
        assert (k, k, -3) in keys, c
        assert RC.voxel_keys(np.array([c]))[0] == k, c
    assert len(keys) == len(set(keys))
    d = s["depth"]
    b = sc["border"]
    assert d[256, 320] == 0.0  # pt_c[2] one ulp above 0: float(5e-324) == 0
    assert d[200, b - 1] == 0.0 and d[200, b] == 4.0 and d[200, 640 - b] == 0.0 and d[200, 640 - b - 1] == 4.0
    assert d[b - 1, 300] == 0.0 and d[512 - b, 300] == 0.0
    assert d[100, 100] == 6.0 and d[100, 200] == 4.0  # the later point wins its pixel
    r = orc.retrieve(sc)
    pos = sc["pos"][r["cell_pt"][r["cells"]]]
    vis = [tuple(p) for p in sc["vis_unsorted"].tolist()]
    expect = sc["expect_flag"][[vis.index(tuple(p)) for p in pos.tolist()]]
    tie = expect == -1
    assert tie.sum() == 1  # one of the two tied points holds the cell
    assert np.array_equal(r["flag"][~tie], expect[~tie])
