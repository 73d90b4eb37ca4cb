"""The placement restatement of tests/vmap_retrieve_cases.py: insertPointIntoVoxelMap's key rule (src/vio.cpp:227-250) and the
voxel-list order, on hand-derived values. No GPU."""
import numpy as np

import retrieve_cases as RC
import vmap_retrieve_cases as VR


def test_insertion_key_rule():
    nxt, prv = (lambda x: np.nextafter(x, np.inf)), (lambda x: np.nextafter(x, -np.inf))  # noqa: E731
    c = np.array([-0.3, 0.3, -0.0, 0.0, -1e-9, -0.5, -0.5000000001, 0.4999999999, prv(0.5), 0.5, nxt(-1.0), -1.0, 2.0 ** 19 - 0.25])
    want = np.array([-1, 0, 0, 0, -1, -2, -2, 1, 1, 1, -3, -3, 2 ** 20 - 1])
    got = VR.insertion_keys(np.stack([c, c, c], 1))
    assert np.array_equal(got, np.stack([want] * 3, 1))
    scan = RC.voxel_keys(c)
    # the scan's floor rule differs for negative coordinates, and where the float narrowing rounds the quotient up
    assert scan[0] == -2 and scan[4] == -2 and scan[6] == -3 and scan[7] == 0


def test_voxel_lists_keep_placement_order():
    pos = np.array([[0.1, 0.1, 0.1], [3.0, 3.0, 3.0], [0.2, 0.2, 0.2], [0.1, 0.1, 0.1], [3.1, 3.1, 3.1]])
    vis = VR.placed_visual_map(pos, np.ones(5, np.int32), [3, 4, 0, 2, 1])
    assert vis["vkeys"].tolist() == [[0, 0, 0], [6, 6, 6]]
    assert vis["vcount"].tolist() == [3, 2]
    assert vis["ids"].tolist() == [3, 0, 2, 4, 1]
