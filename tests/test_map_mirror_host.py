"""CPU: the export of a tick's touched roots (map_export_root, fast_livo2_b200/csrc/esikf_map.cuh, replayed on the host by
tests/map_mirror_harness.cu) and the shim's host mirror built from it (ApplyMapExport, EraseRootsOutside, find_correspond)
against the oracle, on the room scenes and every stream of tests/map_streams.py; the oracle's find_correspond against the
reference source's."""
import os

import numpy as np
import pytest

import map_bind as MB
import map_mirror as MM
import map_streams as MS
from fast_livo2_b200 import synthetic as S
from fast_livo2_b200.synthetic import NODE_DTYPE

ROOM_CFGS = [S.LioCfg(), S.LioCfg(voxel_size=0.4, max_layer=3, max_points_num=20), S.LioCfg(voxel_size=2.0, max_layer=1, min_eigen_value=0.0005)]
ROOM_IDS = ["avia_defaults", "voxel0.4_layer3_max20", "voxel2.0_layer1"]


def test_node_record_layout():
    assert NODE_DTYPE.itemsize == 312
    off = {k: NODE_DTYPE.fields[k][1] for k in NODE_DTYPE.names}
    assert off == dict(key=0, layer=24, path=28, parent=32, leaf=36, voxel_center=40, quater_length=64, init_octo=68, octo_state=69, update_enable=70, is_plane=71,
                       new_points=72, points_size=76, temp_points=80, pad_=84, center=88, normal=112, plane_var=136, d=304, radius=308)


def room_ticks(cfg, n_ticks=6, seed=5):
    rng = np.random.default_rng(seed)
    rects = S.make_scene("room", 0.5)
    for tick in range(n_ticks):
        lo = np.array([-10.0 + 1.5 * tick, -8.0, -2.0])
        yield MB.tick_points(rng, rects, 4000, lo, lo + np.array([8.0, 16.0, 6.0]))


def check_ticks(cfg, ticks, slides=None, queries=True):
    """Every tick through the host replay, the oracle and a mirror fed only by the exports (and the slide bounds): the export
    equals both sides' dumps and candidate planes of its roots, the mirror equals the oracle's whole map, and find_correspond
    on the mirror equals the oracle's."""
    hm, orc, mirror = MM.HarnessMap(cfg), MS.OracleSide(cfg), MM.Mirror(cfg)
    rng = np.random.default_rng(3)
    n_nodes = 0
    for t, (pw, var) in enumerate(ticks):
        slots = hm.apply_touched(pw, var)
        orc.apply(pw, var)
        exp = hm.export(slots)
        # the export is a pure read: a second one gives the same bytes
        assert hm.export(slots)["nodes"].tobytes() == exp["nodes"].tobytes()
        what = (f"export, tick {t}", "host replay")
        got = MM.export_dump(exp)
        MB.compare_node_dumps(got, MM.rows_of(hm.dump_nodes(), exp["keys"]), what, a_releases_cut_lists=True)
        MB.compare_node_dumps(got, MM.rows_of(orc.dump_nodes(), exp["keys"]), (what[0], "oracle"), a_releases_cut_lists=True)
        MB.compare_flat_maps(MM.export_flat(exp), MM.flat_of(orc.flatten(), exp["keys"]), what=(what[0], "oracle"), exact=True)
        assert mirror.apply(exp) == 0
        if slides and t in slides:
            hm.slide(*slides[t]), orc.slide(*slides[t]), mirror.erase(*slides[t])
        MB.compare_node_dumps(mirror.dump_nodes(), orc.dump_nodes(), (f"mirror, tick {t}", "oracle"), a_releases_cut_lists=True)
        MB.compare_flat_maps(mirror.flatten(), orc.flatten(), what=(f"mirror, tick {t}", "oracle"), exact=True)
        if queries and len(exp["nodes"]):
            q = MM.query_points(exp["nodes"], cfg, rng)
            a, b = mirror.find(q), MM.oracle_find(orc, q)
            bad = np.nonzero(np.any(a != b, axis=1))[0]
            assert len(bad) == 0, f"tick {t}: find_correspond differs on {len(bad)} of {len(q)} points; first {q[bad[0]]}: mirror {a[bad[0]]}, oracle {b[bad[0]]}"
        n_nodes += len(exp["nodes"])
    return n_nodes


@pytest.mark.parametrize("cfg", ROOM_CFGS, ids=ROOM_IDS)
def test_room_ticks_export_and_mirror_match_the_oracle(cfg):
    assert check_ticks(cfg, list(room_ticks(cfg))) > 1000


@pytest.mark.parametrize("name", list(MS.CASES))
def test_stream_export_and_mirror_match_the_oracle(name):
    c = MS.case(name)
    assert check_ticks(c["cfg"], c["ticks"], c.get("slides")) > 0


def export_all(hm, keys):
    """The host replay's export of the given roots (all of a map's)."""
    import ctypes as C

    hm.lib.maph_slot_of_key.argtypes = [C.c_void_p, C.c_longlong, C.c_longlong, C.c_longlong]
    return hm.export(np.array([hm.lib.maph_slot_of_key(hm.h, *map(int, k)) for k in keys], np.int32))


def test_find_correspond_reaches_every_stop():
    """The queries reach every way find_correspond stops: an absent root, a plane, a non-plane node at max_layer, and a
    non-plane node above it (a null leaf below a cut node, or a root not yet cut)."""
    outs = []
    blob = MS.case("deep_blob_L3")  # non-planar blobs: non-plane nodes down to max_layer
    for cfg, ticks in ((ROOM_CFGS[1], list(room_ticks(ROOM_CFGS[1], 4))), (blob["cfg"], blob["ticks"])):
        hm, orc = MM.HarnessMap(cfg), MS.OracleSide(cfg)
        for pw, var in ticks:
            hm.apply_touched(pw, var), orc.apply(pw, var)
        q = MM.query_points(export_all(hm, orc.flatten()["keys"])["nodes"], cfg, np.random.default_rng(1))
        o = MM.oracle_find(orc, q)
        o[:, 1] -= cfg.max_layer  # layer relative to max_layer
        outs.append(o)
    out = np.concatenate(outs)
    found = out[out[:, 0] == 1]
    assert (out[:, 0] == 0).any(), "no query in an absent root"
    assert (found[:, 3] == 1).any(), "no query ends at a plane"
    assert ((found[:, 3] == 0) & (found[:, 1] == 0)).any(), "no query ends at a non-plane node of max_layer"
    assert ((found[:, 3] == 0) & (found[:, 1] < 0)).any(), "no query stops above max_layer at a non-plane node"


def pin_case():
    """The pinned scene: three room ticks of the layer-3 configuration, queries on every node of the map."""
    cfg = ROOM_CFGS[1]
    return cfg, list(room_ticks(cfg, 3, seed=21))


def pin_queries(cfg, ticks, ref=None):
    orc, hm = MS.OracleSide(cfg), MM.HarnessMap(cfg)
    for pw, var in ticks:
        orc.apply(pw, var), hm.apply_touched(pw, var)
        if ref is not None:
            ref.update(pw, var)
    return orc, MM.query_points(export_all(hm, orc.flatten()["keys"])["nodes"], cfg, np.random.default_rng(2))


@pytest.mark.skipif(not MM.ref_find_available() and not os.path.exists(MM.GOLDEN), reason="needs oracle/_ref (reference source) or the stored pin")
def test_oracle_find_correspond_is_pinned_to_the_reference_source():
    """orc_lio_find_correspond restates src/voxel_map.cpp:292-305: the reference's own find_correspond on the reference's own
    map returns the same node for every query (live where oracle/_ref was built, else its stored outputs)."""
    cfg, ticks = pin_case()
    ref = MM.RefFindMap(cfg) if MM.ref_find_available() else None
    orc, q = pin_queries(cfg, ticks, ref)
    got = MM.oracle_find(orc, q)
    if ref is not None:
        want = ref.find(q)
    else:
        g = np.load(MM.GOLDEN)
        assert np.array_equal(g["points"], q), "the stored pin was made on other query points"
        want = g["ref"]
    assert len(q) > 1000 and np.array_equal(got, want)
