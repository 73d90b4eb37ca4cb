"""CPU: the restatement of the map side of the retrieval (tests/vmap_retrieve_cases.py: the placement, walk -> depth check ->
skip, then the reference choice of oracle/orc_vmap.cpp) bit for bit against the reference source's own
insertPointIntoVoxelMap + retrieveFromVisualSparseMap on one VIOManager over three ticks of a growing visual map (live where
oracle/_ref is built, else tests/golden/ref_pin/vmap_retrieve.npz), with normal_en on and off: feat_map's keys and
voxel_points order after every tick (negative coordinates and keys the float narrowing moves included), sub_feat_map after the
walk, grid_num, retrieve_voxel_points, the points reaching visual_submap and, with normal_en, their ref_patch."""
import os

import numpy as np
import pytest

import vmap_retrieve_cases as VR

HAVE_PIN = VR.ref_vretrieve_available() or os.path.exists(VR.GOLDEN)
FIELDS = ("sub_keys", "grid_type", "cell_pt", "survivors", "ref")


def _flat_feat_map(d):
    keys = sorted(d)
    first = np.concatenate([[0], np.cumsum([len(d[k]) for k in keys])]).astype(np.int32)
    return dict(keys=np.array(keys, np.int64).reshape(-1, 3), first=first, ids=np.array([i for k in keys for i in d[k]], np.int32))


def _placed_lists(vis):
    return VR.feat_map_lists(vis["vkeys"], np.append(vis["vfirst"], len(vis["ids"])), vis["ids"])


def reference_pins():
    """The reference source's outputs (the generator of tests/golden/ref_pin/vmap_retrieve.npz calls this)."""
    tks, out = VR.ticks(), {}
    for ne in (1, 0):
        ref = VR.RefVretrieve(tks[0]["sc"])
        for t, tk in enumerate(tks):
            ref.place(tk)
            if ne:
                out.update({f"feat_map{t}/{k}": v for k, v in _flat_feat_map(VR.feat_map_lists(*ref.feat_map())).items()})
            r = ref.retrieve(tk["sc"], ne)
            if not ne:
                r["ref"] = np.zeros(0, np.int32)  # without normal_en the choice is not stored
            out.update({f"normal_en{ne}/tick{t}/{k}": np.ascontiguousarray(r[k]) for k in FIELDS})
    return out


def oracle_pins():
    tks, out = VR.ticks(), {}
    for ne in (1, 0):
        runs, _ = VR.restate_ticks(tks, ne)
        for t, r in enumerate(runs):
            if not ne:
                r["ref"] = np.zeros(0, np.int32)
            out.update({f"normal_en{ne}/tick{t}/{k}": np.ascontiguousarray(r[k]) for k in FIELDS})
    order, P, NO = [], [], []
    for t, tk in enumerate(tks):
        order += tk["order"].tolist()
        P.append(tk["pos"]), NO.append(tk["n_obs"])
        vis = VR.placed_visual_map(np.concatenate(P), np.concatenate(NO), order)
        out.update({f"feat_map{t}/{k}": v for k, v in _flat_feat_map(_placed_lists(vis)).items()})
    return out


def _want():
    return reference_pins() if VR.ref_vretrieve_available() else dict(np.load(VR.GOLDEN))


@pytest.mark.skipif(not HAVE_PIN, reason="needs oracle/_ref (reference source) or the stored pin")
def test_map_side_retrieval_is_pinned_to_the_reference_source():
    got, want = oracle_pins(), _want()
    assert set(got) == set(want)
    for k in sorted(got):
        assert got[k].shape == want[k].shape and got[k].tobytes() == want[k].tobytes(), k
    ins = VR.insertion_keys(VR.HAND)
    keys = {tuple(k) for k in want["feat_map0/keys"].tolist()}
    assert all(tuple(k) in keys for k in ins.tolist())
    for ne in (1, 0):
        for t in range(3):
            cells, surv = want[f"normal_en{ne}/tick{t}/grid_type"].sum(), len(want[f"normal_en{ne}/tick{t}/survivors"])
            assert 0 < surv < cells, (ne, t)
    # the map holds voxels of more than one point, and later ticks walk voxels placed by earlier ones
    assert (np.diff(want["feat_map2/first"]) > 1).sum() > 10
