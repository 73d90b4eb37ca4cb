"""GPU: the device-resident voxel map (SURVEY §8 f1 — BuildVoxelMap / UpdateVoxelMap / UpdateOctoTree / init_plane,
src/voxel_map.cpp:55-290, 532-641, kept and refitted on the GPU by esikf_map_device_*) against the oracle:

  * the same lists of (point_w, var) through esikf_map_device_update_points and the oracle's UpdateVoxelMap for ten ticks:
    plane by plane after every tick;
  * the whole LIO tick loop (LIVMapper.cpp:356-428): first frame BuildVoxelMap, then per tick StateEstimation on the device
    map + device-side map refresh, against the oracle's StateEstimation + UpdateVoxelMap on its own native octrees — states to
    1e-9 every tick, maps plane by plane at the end; no map data crosses PCIe in the loop;
  * capacity errors surface as a status, never as a silently truncated map."""
import numpy as np
import pytest

import map_bind as MB
import oracle_bind as O
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from map_bind import oracle_map, oracle_update_map, tick_points
from parity_util import assert_state_close

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cfg", [S.LioCfg(), S.LioCfg(voxel_size=0.4, max_layer=3, max_points_num=20)], ids=["avia_defaults", "voxel0.4_layer3_max20"])
def test_device_update_voxel_map_matches_the_oracle_for_ten_ticks(gpu_ctx, cfg):
    rng = np.random.default_rng(5)
    rects = S.make_scene("room", 0.5)
    orc = oracle_map(cfg)
    gpu_ctx.map_device_init(cfg, root_capacity=1 << 16)
    for tick in range(10):
        lo = np.array([-10.0 + 1.5 * tick, -8.0, -2.0])
        pw, var = tick_points(rng, rects, 6000, lo, lo + np.array([8.0, 16.0, 6.0]))
        oracle_update_map(orc, pw, var)
        gpu_ctx.map_device_update_points(pw, var)
        # refits add the per-point terms in point order without FMA contraction: bit-identical to the serial evaluation
        n = MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten(), what=("device map", "oracle"), exact=True)
        assert n > 0
    st = gpu_ctx.map_device_stats()
    assert st["errors"] == 0 and st["roots"] == len(orc.flatten()["keys"]) and st["touched_roots"] > 0


def _poses(k):
    R = S.so3_exp(np.array([0.002 * k, -0.001 * k, 0.01 * k]))
    p = np.array([-2.0 + 0.12 * k, 0.5 - 0.05 * k, 0.3 + 0.01 * k])
    return R, p


def test_lio_tick_loop_with_device_side_map_refresh_tracks_the_oracle(gpu_ctx):
    """10 ticks: scan at a moving pose -> StateEstimation -> map absorbs the scan. Device: esikf_lio_update on the device map +
    esikf_map_device_update (nothing but the scan and two states cross PCIe). Oracle: its own StateEstimation and
    UpdateVoxelMap on native octrees."""
    cfg = S.LioCfg()
    ext = S.avia_extrinsics()
    rng = np.random.default_rng(21)
    rects = S.make_scene("room", 0.5)
    orc = O.OracleLIO(cfg, ext)
    n_pts = 20000
    cov0 = S.random_prior_cov(np.random.default_rng(3), scale=0.05)
    # first frame: BuildVoxelMap at the true pose
    R0, p0 = _poses(0)
    st0 = S.pack_state(R0, p0, cov=cov0, g=np.array([0, 0, -9.81]))
    scan0 = S.scan_at(rects, ext, R0, p0, 60000, cfg, rng)
    gpu_ctx.set_extrinsics(ext)
    gpu_ctx.map_device_init(cfg, root_capacity=1 << 16)
    gpu_ctx.lio_set_scan(scan0)
    gpu_ctx.map_device_build(st0)
    orc.tick_build_map(scan0, st0)
    MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten(), rtol=1e-7, what=("device map after BuildVoxelMap", "oracle"))
    state_dev = st0.copy()
    state_orc = st0.copy()
    matched = []
    for k in range(1, 11):
        Rk, pk = _poses(k)
        scan = S.scan_at(rects, ext, Rk, pk, n_pts, cfg, rng)
        # prior of the tick: the previous posterior pushed towards the new pose with some error (stands in for IMU propagation)
        def prior(prev):
            s = S.unpack_state(prev)
            return S.pack_state(Rk @ S.so3_exp(np.array([0.002, -0.003, 0.002])), pk + np.array([0.02, -0.015, 0.01]), cov=s["cov"] + np.eye(19) * 1e-6,
                                g=np.array([0, 0, -9.81]))
        pr_dev, pr_orc = prior(state_dev), prior(state_orc)
        g = gpu_ctx.lio_update(scan, pr_dev, pr_dev, cfg)
        o = orc.state_estimation(scan, pr_orc, pr_orc)
        assert g["iters"] == o["iters"] and np.array_equal(np.asarray(g["M"])[:g["iters"]], o["M"]), (k, g["M"], o["M"])
        assert_state_close(g["state"], o["state"], rot_tol=1e-9, pos_tol=2e-9, cov_tol=1e-7, rest_tol=1e-9)
        matched.append(int(o["M"][-1]))
        # pv.normal of every point (zero when unmatched) before and after the map moved the records
        nb = gpu_ctx.lio_fetch_normals()
        gpu_ctx.map_device_update()      # LIVMapper.cpp:413-424 on the device, posterior resident
        orc.tick_update_map()
        na = gpu_ctx.lio_fetch_normals()
        assert np.array_equal(nb, na)
        assert np.array_equal(np.linalg.norm(nb, axis=1) > 0, g["normal_plane"] >= 0)
        state_dev, state_orc = g["state"], o["state"]
    assert min(matched) > 0.8 * n_pts
    n = MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten(), rtol=1e-6, what=("device map after 10 ticks", "oracle"))
    st = gpu_ctx.map_device_stats()
    assert n > 1000 and st["errors"] == 0


def test_device_map_sliding_matches_clear_mem_out_of_map_and_keeps_tracking(gpu_ctx):
    """esikf_map_device_slide (mapSliding / clearMemOutOfMap, src/voxel_map.cpp:924-971) against the oracle's deletion, then more
    ticks on the compacted map."""
    cfg = S.LioCfg()
    rng = np.random.default_rng(17)
    rects = S.make_scene("room", 0.5)
    orc = oracle_map(cfg)
    gpu_ctx.map_device_init(cfg, root_capacity=1 << 16)
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
    assert deleted > 0 and after["roots"] == before["roots"] - deleted and after["pool_points"] < before["pool_points"] and after["errors"] == 0
    MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten())
    for tick in range(4):
        pw, var = tick_points(rng, rects, 6000, lo_w, hi_w)
        oracle_update_map(orc, pw, var)
        gpu_ctx.map_device_update_points(pw, var)
        MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten())
    # compaction only
    gpu_ctx.map_device_slide()
    MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten())


def test_device_map_capacity_errors_are_statuses(gpu_ctx):
    cfg = S.LioCfg()
    rng = np.random.default_rng(2)
    rects = S.make_scene("room", 0.5)
    pw, var = tick_points(rng, rects, 5000, np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0]))
    for kw, flag in ((dict(root_capacity=1 << 12, node_capacity=16), 1), (dict(root_capacity=1 << 12, point_capacity=64), 2), (dict(root_capacity=1 << 12, record_capacity=4), 4),
                     (dict(root_capacity=128), 8)):
        gpu_ctx.map_device_init(cfg, **kw)
        with pytest.raises(api.EsikfError):
            gpu_ctx.map_device_update_points(pw, var)
        assert gpu_ctx.map_device_stats()["errors"] & flag
    # and the context recovers with a fresh map
    gpu_ctx.map_device_init(cfg, root_capacity=1 << 16)
    gpu_ctx.map_device_update_points(pw, var)
    assert gpu_ctx.map_device_stats()["errors"] == 0
    # host-owned maps cannot be patched into a device-resident one
    with pytest.raises(api.EsikfError):
        gpu_ctx.map_patch(np.zeros(1, np.int32), np.zeros(1, S.PLANE_DTYPE))
