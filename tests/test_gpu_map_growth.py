"""GPU: capacity growth of the device-resident voxel map (esikf_map_cfg.grow = 1). A map that starts from tiny capacities and
grows whenever a tick would not fit must hold, after every tick, exactly the map of a context with large fixed capacities and
the oracle's: the update loop, the build form, the LIO tick loop (which reads the map through the hash probe and the
relocated records), sliding, and a tick that inserts more new roots than the table had room for."""
import contextlib

import numpy as np
import pytest

import map_bind as MB
import map_streams as MS
import oracle_bind as O
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from map_bind import oracle_map, oracle_update_map, tick_points
from parity_util import assert_state_close

pytestmark = pytest.mark.gpu

TINY = dict(root_capacity=1, node_capacity=16, record_capacity=4, point_capacity=64, grow=True)
CAPS = ("root_capacity", "node_capacity", "record_capacity", "point_capacity")


@contextlib.contextmanager
def second_context():
    ctx = api.Context(0)
    try:
        yield ctx
    finally:
        ctx.close()


def _grew_from_tiny(cap):
    """every capacity is above TINY's (root_capacity 1 opens the smallest table, 1024 slots: 512 roots)"""
    start = dict(TINY, root_capacity=512)
    return all(cap[k] > start[k] for k in CAPS)


def test_update_points_from_tiny_capacities_equals_the_oracle_and_a_fixed_map(gpu_ctx):
    cfg = S.LioCfg()
    rng, rects = np.random.default_rng(5), S.make_scene("room", 0.5)
    orc = oracle_map(cfg)
    with second_context() as fixed:
        fixed.map_device_init(cfg, root_capacity=1 << 16)
        gpu_ctx.map_device_init(cfg, **TINY)
        first = gpu_ctx.map_device_capacity()
        assert first["grow"] and first["node_capacity"] == 16
        for tick in range(10):
            lo = np.array([-10.0 + 1.5 * tick, -8.0, -2.0])
            pw, var = tick_points(rng, rects, 6000, lo, lo + np.array([8.0, 16.0, 6.0]))
            oracle_update_map(orc, pw, var)
            gpu_ctx.map_device_update_points(pw, var)
            fixed.map_device_update_points(pw, var)
            g = gpu_ctx.map_device_download()
            MB.compare_flat_maps(g, orc.flatten(), what=(f"grown device map, tick {tick}", "oracle"), exact=True)
            MB.compare_flat_maps(g, fixed.map_device_download(), what=(f"grown device map, tick {tick}", "fixed-capacity device map"), exact=True)
            assert gpu_ctx.map_device_stats()["errors"] == 0
        last = gpu_ctx.map_device_capacity()
        assert _grew_from_tiny(last), (first, last)
        st = gpu_ctx.map_device_stats()
        assert st["roots"] == len(orc.flatten()["keys"]) and st["nodes"] <= last["node_capacity"] and st["pool_points"] <= last["point_capacity"]


def _poses(k):
    R = S.so3_exp(np.array([0.002 * k, -0.001 * k, 0.01 * k]))
    p = np.array([-2.0 + 0.12 * k, 0.5 - 0.05 * k, 0.3 + 0.01 * k])
    return R, p


def test_lio_tick_loop_on_a_growing_map_equals_the_fixed_map(gpu_ctx):
    """The tick loop of test_gpu_map's LIO test on a fixed-capacity context and on one grown from tiny capacities, side by
    side. The build scan is small so that the hash table also grows on an update tick (where pv.normal must be snapshotted
    before the copy moves the records). Iterations, matched counts, states, pv.normal before and after the map update, and
    the final maps agree bit for bit; the states also track the oracle."""
    cfg = S.LioCfg()
    ext = S.avia_extrinsics()
    rng, rects = np.random.default_rng(21), S.make_scene("room", 0.5)
    orc = O.OracleLIO(cfg, ext)
    cov0 = S.random_prior_cov(np.random.default_rng(3), scale=0.05)
    R0, p0 = _poses(0)
    st0 = S.pack_state(R0, p0, cov=cov0, g=np.array([0, 0, -9.81]))
    scan0 = S.scan_at(rects, ext, R0, p0, 8000, cfg, rng)
    with second_context() as grow:
        ctxs = {"fixed": gpu_ctx, "grow": grow}
        for name, c in ctxs.items():
            c.set_extrinsics(ext)
            c.map_device_init(cfg, **(dict(root_capacity=1 << 16) if name == "fixed" else TINY))
            c.lio_set_scan(scan0)
            c.map_device_build(st0)
        orc.tick_build_map(scan0, st0)
        MB.compare_flat_maps(grow.map_device_download(), gpu_ctx.map_device_download(), exact=True)
        first = grow.map_device_capacity()
        state = st0.copy()
        hash_grew_on_update = 0
        for k in range(1, 11):
            Rk, pk = _poses(k)
            scan = S.scan_at(rects, ext, Rk, pk, 20000, cfg, rng)
            s = S.unpack_state(state)
            pr = S.pack_state(Rk @ S.so3_exp(np.array([0.002, -0.003, 0.002])), pk + np.array([0.02, -0.015, 0.01]), cov=s["cov"] + np.eye(19) * 1e-6,
                              g=np.array([0, 0, -9.81]))
            out = {name: c.lio_update(scan, pr, pr, cfg) for name, c in ctxs.items()}
            a, b = out["fixed"], out["grow"]
            assert a["iters"] == b["iters"] and np.array_equal(a["M"], b["M"]), (k, a["M"], b["M"])
            assert np.array_equal(np.asarray(a["state"]).view(np.uint64), np.asarray(b["state"]).view(np.uint64)), k
            assert np.array_equal(a["match_plane"] >= 0, b["match_plane"] >= 0) and np.array_equal(a["dis_to_plane"], b["dis_to_plane"])
            o = orc.state_estimation(scan, pr, pr)
            assert a["iters"] == o["iters"] and np.array_equal(np.asarray(a["M"])[:a["iters"]], o["M"]), (k, a["M"], o["M"])
            assert_state_close(a["state"], o["state"], rot_tol=1e-9, pos_tol=2e-9, cov_tol=1e-7, rest_tol=1e-9)
            before = {name: c.lio_fetch_normals() for name, c in ctxs.items()}
            cap0 = grow.map_device_capacity()
            for c in ctxs.values():
                c.map_device_update()
            orc.tick_update_map()
            hash_grew_on_update += grow.map_device_capacity()["root_capacity"] > cap0["root_capacity"]
            after = {name: c.lio_fetch_normals() for name, c in ctxs.items()}
            for name in ctxs:
                assert np.array_equal(before[name], after[name]), (k, name)
            assert np.array_equal(before["fixed"], before["grow"]), k
            MB.compare_flat_maps(grow.map_device_download(), gpu_ctx.map_device_download(), what=(f"grown map, tick {k}", "fixed map"), exact=True)
            state = a["state"]
        assert hash_grew_on_update > 0
        assert _grew_from_tiny(first) and grow.map_device_stats()["errors"] == 0
        MB.compare_flat_maps(grow.map_device_download(), orc.flatten(), rtol=1e-6, what=("grown map after 10 ticks", "oracle"))


def test_build_of_a_60k_scan_from_tiny_capacities_equals_the_fixed_build(gpu_ctx):
    cfg = S.LioCfg()
    ext = S.avia_extrinsics()
    rng, rects = np.random.default_rng(21), S.make_scene("room", 0.5)
    R0, p0 = _poses(0)
    st0 = S.pack_state(R0, p0, cov=S.random_prior_cov(np.random.default_rng(3), scale=0.05), g=np.array([0, 0, -9.81]))
    scan0 = S.scan_at(rects, ext, R0, p0, 60000, cfg, rng)
    with second_context() as grow:
        for c, kw in ((gpu_ctx, dict(root_capacity=1 << 16)), (grow, TINY)):
            c.set_extrinsics(ext)
            c.map_device_init(cfg, **kw)
            c.lio_set_scan(scan0)
            c.map_device_build(st0)
        g = grow.map_device_download()
        assert len(g["planes"]) > 500
        MB.compare_flat_maps(g, gpu_ctx.map_device_download(), what=("grown build", "fixed-capacity build"), exact=True)
        assert _grew_from_tiny(grow.map_device_capacity())


def test_more_new_roots_than_the_table_holds_grow_it(gpu_ctx):
    """1025 new roots in one tick (7 points each, concurrent inserts of the same and colliding keys) into a context that
    starts with a 1024-slot table: with growth on it is no error, and the map equals the oracle's."""
    cfg, keys, pw = MS.hash_keys(1025)
    var = np.tile(MS.VAR, (len(pw), 1, 1))
    gpu_ctx.map_device_init(cfg, root_capacity=512, grow=True)
    gpu_ctx.map_device_update_points(pw, var)
    orc = MS.OracleSide(cfg)
    orc.apply(pw, var)
    MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten(), exact=True)
    st = gpu_ctx.map_device_stats()
    assert st["errors"] == 0 and st["roots"] == len(keys) == 1025
    assert gpu_ctx.map_device_capacity()["root_capacity"] > 512


def test_sliding_a_growing_map_matches_the_oracle(gpu_ctx):
    """test_gpu_map's slide scenario with growth on from tiny capacities: six ticks, a slide, four ticks, a compaction."""
    cfg = S.LioCfg()
    rng, rects = np.random.default_rng(17), S.make_scene("room", 0.5)
    orc = oracle_map(cfg)
    gpu_ctx.map_device_init(cfg, **TINY)
    lo_w, hi_w = np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0])
    for tick in range(6):
        pw, var = tick_points(rng, rects, 6000, lo_w, hi_w)
        oracle_update_map(orc, pw, var)
        gpu_ctx.map_device_update_points(pw, var)
    before = gpu_ctx.map_device_stats()
    c, half = np.array([4, -2, 1]), 12
    deleted = orc.lib.orc_lio_clear_out_of_map(orc.h, int(c[0] + half), int(c[0] - half), int(c[1] + half), int(c[1] - half), int(c[2] + half), int(c[2] - half))
    gpu_ctx.map_device_slide(c - half, c + half)
    after = gpu_ctx.map_device_stats()
    assert deleted > 0 and after["roots"] == before["roots"] - deleted and after["errors"] == 0
    MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten(), exact=True)
    for tick in range(4):
        pw, var = tick_points(rng, rects, 6000, lo_w - 4, hi_w + 4)
        oracle_update_map(orc, pw, var)
        gpu_ctx.map_device_update_points(pw, var)
        MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten(), exact=True)
    gpu_ctx.map_device_slide()
    MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten(), exact=True)
    assert gpu_ctx.map_device_stats()["errors"] == 0


def test_key_range_is_still_an_error_with_growth(gpu_ctx):
    """A key outside +-2^20 is not a capacity: with growth on it is still a status (MAP_ERR_KEY), also on a tick that grows
    the hash table first."""
    cfg = S.LioCfg()
    rng, rects = np.random.default_rng(2), S.make_scene("room", 0.5)
    pw, var = tick_points(rng, rects, 5000, np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0]))
    pw[0] = [3e6, 0, 0]
    gpu_ctx.map_device_init(cfg, **TINY)
    with pytest.raises(api.EsikfError):
        gpu_ctx.map_device_update_points(pw, var)
    assert gpu_ctx.map_device_stats()["errors"] & 16
    # and a fresh growing map works
    gpu_ctx.map_device_init(cfg, **TINY)
    gpu_ctx.map_device_update_points(pw[1:], var[1:])
    assert gpu_ctx.map_device_stats()["errors"] == 0
