"""CPU: the device voxel-map state machine (fast_livo2_b200/csrc/esikf_map.cuh: UpdateOctoTree / init_octo_tree /
cut_octo_tree / init_plane / candidate emission, src/voxel_map.cpp:55-290, 532-641) compiled for the host and replayed against
the oracle's BuildVoxelMap / UpdateVoxelMap tick by tick — the same functions the GPU runs one warp per touched root."""
import numpy as np
import pytest

import map_bind as MB
import oracle_bind as O
from fast_livo2_b200 import synthetic as S
from map_bind import oracle_map, oracle_update_map, tick_points


@pytest.mark.parametrize("cfg", [S.LioCfg(), S.LioCfg(voxel_size=0.4, max_layer=3, max_points_num=20), S.LioCfg(voxel_size=2.0, max_layer=1, min_eigen_value=0.0005)],
                         ids=["avia_defaults", "voxel0.4_layer3_max20", "voxel2.0_layer1"])
def test_ten_ticks_of_update_voxel_map_match_the_oracle(cfg):
    rng = np.random.default_rng(5)
    rects = S.make_scene("room", 0.5)
    orc, hm = oracle_map(cfg), MB.HostMap(cfg)
    total = 0
    for tick in range(10):
        # a window that slides through the room: old voxels keep receiving points (refits, max_points_num), new ones appear
        lo = np.array([-10.0 + 1.5 * tick, -8.0, -2.0])
        hi = lo + np.array([8.0, 16.0, 6.0])
        pw, var = tick_points(rng, rects, 6000, lo, hi)
        total += len(pw)
        oracle_update_map(orc, pw, var)
        assert hm.apply(pw, var) == 0
        n = MB.compare_flat_maps(hm.flatten(), orc.flatten(), what=("device state machine", "oracle"), exact=True)  # serial policy: bit for bit
        assert n > 0
    u = hm.usage()
    assert u["roots"] == len(orc.flatten()["keys"]) and total > 30000
    # octrees were cut and planes refitted: several candidates per root exist, lists were released at max_points_num
    f = hm.flatten()
    assert f["count"].max() > 1 and (f["planes"]["layer"] > 0).any()


def test_build_voxel_map_form_matches_the_oracle():
    """BuildVoxelMap (src/voxel_map.cpp:532-591): every point pushed first, init_octo_tree afterwards (large lists, the
    recursive cut), followed by incremental ticks on the same map."""
    cfg = S.LioCfg()
    rng = np.random.default_rng(9)
    rects = S.make_scene("room", 0.5)
    orc, hm = oracle_map(cfg), MB.HostMap(cfg)
    pw, var = tick_points(rng, rects, 40000, np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0]))
    # the oracle's BuildVoxelMap recomputes var from body points; the build FORM (push all, then init) is what is compared:
    # an empty oracle map fed through UpdateVoxelMap differs (it inits at the 6th point) — so build the oracle map by hand
    orc2 = oracle_map(cfg)
    oracle_update_map(orc2, pw[:0], var[:0])
    assert hm.apply(pw, var, build=True) == 0
    fb = hm.flatten()
    # reference for the build form: the oracle's own BuildVoxelMap needs (world, body, state); give it an identity pose so that
    # world == body and var == calcBodyCov + prior blocks, and feed the harness the same var
    st = S.pack_state(np.eye(3), np.zeros(3), cov=np.eye(19) * 1e-4)
    ext = S.Extrinsics(extR=np.eye(3), extT=np.zeros(3), Rcl=np.eye(3), Pcl=np.zeros(3))
    orc3 = O.OracleLIO(cfg, ext)
    pb = pw.astype(np.float32)
    orc3.build_map(pb, pb, st)
    body = S.calc_body_cov_np(pb.astype(np.float64), cfg.dept_err, cfg.beam_err)
    P = np.eye(19) * 1e-4
    cm = np.zeros((len(pb), 3, 3))
    p64 = pb.astype(np.float64)
    cm[:, 0, 1], cm[:, 0, 2], cm[:, 1, 0], cm[:, 1, 2], cm[:, 2, 0], cm[:, 2, 1] = -p64[:, 2], p64[:, 1], p64[:, 2], -p64[:, 0], -p64[:, 1], p64[:, 0]
    var3 = body + (-cm) @ P[:3, :3] @ (-cm).transpose(0, 2, 1) + P[3:6, 3:6]
    hm3 = MB.HostMap(cfg)
    assert hm3.apply(p64, var3, build=True) == 0
    n = MB.compare_flat_maps(hm3.flatten(), orc3.flatten(), rtol=1e-7, what=("device state machine (build form)", "oracle BuildVoxelMap"))
    assert n > 500 and len(fb["keys"]) > 0
    # then five incremental ticks on both
    for tick in range(5):
        pw2, var2 = tick_points(rng, rects, 5000, np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0]))
        oracle_update_map(orc3, pw2, var2)
        assert hm3.apply(pw2, var2) == 0
        MB.compare_flat_maps(hm3.flatten(), orc3.flatten(), rtol=1e-7)


def test_map_sliding_keeps_the_box_and_later_ticks_still_match():
    """mapSliding / clearMemOutOfMap (src/voxel_map.cpp:924-971): roots outside the box around the sensor are dropped. The device
    form copies the survivors into a fresh arena (which also reclaims dead record blocks and list slack); the map must equal the
    oracle's after the deletion AND keep tracking it through the following ticks (node state, point lists and counters survived)."""
    cfg = S.LioCfg()
    rng = np.random.default_rng(17)
    rects = S.make_scene("room", 0.5)
    orc, hm = oracle_map(cfg), MB.HostMap(cfg)
    lo_w, hi_w = np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0])
    for tick in range(6):
        pw, var = tick_points(rng, rects, 6000, lo_w, hi_w)
        oracle_update_map(orc, pw, var)
        assert hm.apply(pw, var) == 0
    before = hm.usage()
    # sensor at voxel (4, -2, 1), half_map_size 12 voxels
    c, half = np.array([4, -2, 1]), 12
    deleted = orc.lib.orc_lio_clear_out_of_map(orc.h, int(c[0] + half), int(c[0] - half), int(c[1] + half), int(c[1] - half), int(c[2] + half), int(c[2] - half))
    assert hm.slide(c - half, c + half) == 0
    after = hm.usage()
    assert deleted > 0 and after["roots"] == before["roots"] - deleted
    assert after["pool_points"] < before["pool_points"] and after["recs"] <= before["recs"]  # compaction
    MB.compare_flat_maps(hm.flatten(), orc.flatten(), exact=True)
    for tick in range(4):
        pw, var = tick_points(rng, rects, 6000, lo_w, hi_w)
        oracle_update_map(orc, pw, var)
        assert hm.apply(pw, var) == 0
        MB.compare_flat_maps(hm.flatten(), orc.flatten(), exact=True)


def test_capacity_errors_are_reported_not_ignored():
    cfg = S.LioCfg()
    rng = np.random.default_rng(2)
    rects = S.make_scene("room", 0.5)
    pw, var = tick_points(rng, rects, 5000, np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0]))
    assert MB.HostMap(cfg, node_cap=16).apply(pw, var) & 1       # MAP_ERR_NODES
    assert MB.HostMap(cfg, pool_cap=64).apply(pw, var) & 2       # MAP_ERR_POOL
    assert MB.HostMap(cfg, hash_cap=64).apply(pw, var) & 8       # MAP_ERR_HASH
    far = pw.copy()
    far[0] = [3e6, 0, 0]
    assert MB.HostMap(cfg).apply(far, var) & 16                  # MAP_ERR_KEY: outside the +-2^20 key range


@pytest.mark.parametrize("voxel_size", [0.5, 0.4, 2.0])
def test_root_voxel_keys_on_voxel_faces_and_negative_coordinates(voxel_size):
    """The key of UpdateVoxelMap (src/voxel_map.cpp:620-625): (float)(p / (double)(float)voxel_size), "-1 if negative", truncation.
    World points (float-rounded, like TransformLidar's output) exactly on voxel faces, one ulp either side, around zero and at
    negative integers of the quotient: the device code must open exactly the root voxels the oracle opens."""
    cfg = S.LioCfg(voxel_size=voxel_size)
    ks = np.arange(-6, 7, dtype=np.float64)
    face = (ks * np.float64(np.float32(voxel_size))).astype(np.float32)
    vals = np.concatenate([face, np.nextafter(face, np.float32(np.inf)), np.nextafter(face, np.float32(-np.inf)), np.float32([0.0, -0.0, 1e-30, -1e-30])])
    grid = np.stack(np.meshgrid(vals, vals[::5], vals[::7], indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    var = np.tile(np.eye(3) * 1e-4, (len(grid), 1, 1))
    orc, hm = oracle_map(cfg), MB.HostMap(cfg)
    oracle_update_map(orc, grid, var)
    assert hm.apply(grid, var) == 0
    a, b = hm.flatten(), orc.flatten()
    assert len(a["keys"]) == len(b["keys"]) > 50
    assert set(map(tuple, a["keys"].tolist())) == set(map(tuple, b["keys"].tolist()))
    assert (a["keys"] < 0).any()
