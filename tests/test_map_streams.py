"""CPU: the device voxel-map state machine (fast_livo2_b200/csrc/esikf_map.cuh, compiled for the host by
tests/map_host_harness.cu) against the oracle on the hand-built streams of tests/map_streams.py: after every tick the node
dumps are equal (every node, plane or not: layer, path, init_octo, octo_state, update_enable, is_plane, new_points, list size,
points_size) and every candidate plane is equal bit for bit. Every case must reach the branch it was built for."""
import numpy as np
import pytest

import map_bind as MB
import map_streams as MS


def _replay(name, **caps):
    c = MS.case(name)
    h = MS.replay(c, {"dev": MB.HostMap(c["cfg"], **caps), "orc": MS.OracleSide(c["cfg"])})
    return c, h


@pytest.mark.parametrize("name", list(MS.CASES))
def test_stream_node_dumps_and_planes_match_the_oracle_every_tick(name):
    c, h = _replay(name)
    for t, (a, b) in enumerate(zip(h["dev"], h["orc"])):
        what = (f"device state machine, tick {t}", "oracle")
        MB.compare_node_dumps(a["dump"], b["dump"], what, a_releases_cut_lists=True)
        MB.compare_flat_maps(a["flat"], b["flat"], what=what, exact=True)
        if "slid" in a:
            MB.compare_node_dumps(a["slid_dump"], b["slid_dump"], (what[0] + " after the slide", "oracle"), a_releases_cut_lists=True)
            MB.compare_flat_maps(a["slid"], b["slid"], what=what, exact=True)
    assert all(x["usage"]["roots"] == len(y["flat"]["keys"]) for x, y in zip(h["dev"], h["orc"]))
    for what, f in c["reach"].items():
        assert f(h["dev"]) > 0, f"{name}: does not reach '{what}'"


def test_layer_init_num_mutation_is_visible():
    """The per-layer thresholds are what the cases exercise: with a uniform layer_init_num the same streams build another
    tree (a node that used its parent's threshold would pass a uniform-threshold test)."""
    c = MS.case("layer_init_cut")
    c2 = dict(c, cfg=MS.S.LioCfg(**{**c["cfg"].__dict__, "layer_init_num": (64, 64, 64, 64)}))
    a = MS.replay(c, {"d": MB.HostMap(c["cfg"])})["d"][-1]["dump"]
    b = MS.replay(c2, {"d": MB.HostMap(c2["cfg"])})["d"][-1]["dump"]
    assert a.shape != b.shape or not np.array_equal(a, b)


@pytest.mark.parametrize("ax", [0, 1, 2])
@pytest.mark.parametrize("side", [-1, 1])
def test_key_one_past_the_range_is_an_error(ax, side):
    """Keys -2^20 and 2^20 - 1 are roots (test above); one past either end is MAP_ERR_KEY (the oracle has no range)."""
    cfg = MS.S.LioCfg(voxel_size=0.5)
    pw, var = MS.beyond_key(ax, side)
    assert MB.HostMap(cfg).apply(pw, var) & 16


@pytest.mark.parametrize("extra,err", [(-1, 0), (0, 0), (1, 8)], ids=["capacity-1", "capacity", "capacity+1"])
def test_hash_table_filled_to_capacity(extra, err):
    """A 64-slot table with 63, 64 and 65 roots in one tick: up to capacity every probe sequence finds its slot (some of them
    wrap around the end of the table) and the map equals the oracle's; one root over is MAP_ERR_HASH."""
    cap = 64
    cfg, keys, pw = MS.hash_keys(cap + extra)
    var = np.tile(MS.VAR, (len(pw), 1, 1))
    hm = MB.HostMap(cfg, hash_cap=cap)
    assert hm.apply(pw, var) == err
    if err:
        return
    assert MS.probe_wraps([tuple(k) for k in MS.key_order(pw, cfg)], cap) > 0
    orc = MS.OracleSide(cfg)
    orc.apply(pw, var)
    assert hm.slots_used() == len(keys) == hm.usage()["roots"]
    MB.compare_node_dumps(hm.dump_nodes(), orc.dump_nodes(), ("device state machine", "oracle"), a_releases_cut_lists=True)
    MB.compare_flat_maps(hm.flatten(), orc.flatten(), exact=True)
