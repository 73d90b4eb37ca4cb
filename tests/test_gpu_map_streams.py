"""GPU: the device-resident voxel map (esikf_map_device_*, csrc/esikf_map.cu / esikf_map.cuh: one warp per touched root)
on the hand-built streams of tests/map_streams.py, against the oracle bit for bit after every tick, and against the host
harness's counters (the same state machine under the serial policy). Then LIO updates on the maps the device built: deep
octrees, roots with 64 / 72 candidates whose record blocks were relocated, the equal-eigenvalue plane (NaN plane_var), and
maps after one and after two slides (the residual kernel must read the swapped arena)."""
import numpy as np
import pytest

import map_bind as MB
import map_streams as MS
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from parity_util import assert_state_close

pytestmark = pytest.mark.gpu


def _lio_compare(g, o):
    assert g["iters"] == o["iters"] and np.array_equal(np.asarray(g["M"])[:g["iters"]], o["M"]), (g["M"], o["M"])
    # association bit for bit: which points matched and their point-to-plane distances (plane ids differ by construction:
    # record slots on the device, flat ids in the oracle)
    assert np.array_equal(g["match_plane"] >= 0, o["match_plane"] >= 0)
    assert np.array_equal(g["dis_to_plane"], o["dis_to_plane"])
    assert_state_close(g["state"], o["state"], rot_tol=1e-9, pos_tol=2e-9, cov_tol=1e-7, rest_tol=1e-9)


def _lio(ctx, orc, c, seed=0, n=3000):
    pts, prior = MS.lio_scan(c, np.random.default_rng(seed), n)
    g = ctx.lio_update(pts, prior, prior, c["cfg"])
    o = orc.o.state_estimation(pts, prior, prior)
    _lio_compare(g, o)
    return g, o, pts


@pytest.mark.parametrize("name", [n for n in MS.CASES if n != "slide"])
def test_device_streams_match_the_oracle_every_tick(gpu_ctx, name):
    c = MS.case(name)
    gpu_ctx.set_extrinsics(MS.IDENTITY_EXT)
    sides = {"gpu": MS.DeviceSide(gpu_ctx, c["cfg"]), "orc": MS.OracleSide(c["cfg"], MS.IDENTITY_EXT), "host": MB.HostMap(c["cfg"])}
    h = MS.replay(c, sides)
    for t in range(len(c["ticks"])):
        MB.compare_flat_maps(h["gpu"][t]["flat"], h["orc"][t]["flat"], what=(f"device map, tick {t}", "oracle"), exact=True)
        u, hu = h["gpu"][t]["usage"], h["host"][t]["usage"]
        assert u["errors"] == 0 and u["roots"] == len(h["orc"][t]["flat"]["keys"])
        assert (u["nodes"], u["recs"], u["pool_points"], u["roots"]) == (hu["nodes"], hu["recs"], hu["pool_points"], hu["roots"]), (u, hu)
    if name in ("deep_blob_L7", "deep_cut", "candidates_growth", "candidates_layer3"):
        g, o, pts = _lio(gpu_ctx, sides["orc"], c)
        assert o["M"][0] == 0 if name.startswith("deep") else o["M"][0] > 0.9 * len(pts)  # the deep blobs hold no plane
    if name == "box_corners":
        # a scan on the mid-planes of the boxes: the equal-eigenvalue plane (NaN plane_var) never matches, the valid one does
        pts, prior = MS.box_scan()
        g = gpu_ctx.lio_update(pts, prior, prior, c["cfg"])
        _lio_compare(g, sides["orc"].o.state_estimation(pts, prior, prior))
        k = MS.voxel_keys(pts, c["cfg"])
        at = lambda name: np.all(k == np.array(MS.BOX_KEYS[name]), axis=1)
        assert at("equal_min").sum() > 0 and not (g["match_plane"][at("equal_min")] >= 0).any()
        assert (g["match_plane"][at("below")] >= 0).all()


def test_device_slides_twice_and_lio_reads_the_swapped_arena(gpu_ctx):
    """mapSliding on the slide stream: faces through occupied roots, a second slide into the first arena's storage, a box that
    keeps nothing; after each slide and after the updates that follow, the device map equals the oracle's and a LIO update on
    it equals the oracle's StateEstimation on its own map."""
    c = MS.case("slide")
    gpu_ctx.set_extrinsics(MS.IDENTITY_EXT)
    dev, orc = MS.DeviceSide(gpu_ctx, c["cfg"]), MS.OracleSide(c["cfg"], MS.IDENTITY_EXT)
    rng = np.random.default_rng(5)
    lio_runs = 0
    for t, (pw, var) in enumerate(c["ticks"]):
        dev.apply(pw, var)
        orc.apply(pw, var)
        MB.compare_flat_maps(dev.flatten(), orc.flatten(), what=(f"device map, tick {t}", "oracle"), exact=True)
        if t in c["slides"]:
            lo, hi = c["slides"][t]
            before = dev.usage()
            dev.slide(lo, hi)
            deleted = orc.slide(lo, hi)
            after = dev.usage()
            assert after["errors"] == 0 and after["roots"] == before["roots"] - deleted
            MB.compare_flat_maps(dev.flatten(), orc.flatten(), what=(f"device map after slide {t}", "oracle"), exact=True)
            if after["roots"]:
                pts, prior = MS.lio_scan(c, rng, 4000)
                o = orc.o.state_estimation(pts, prior, prior)
                _lio_compare(gpu_ctx.lio_update(pts, prior, prior, c["cfg"]), o)
                assert o["M"][0] > 100
                lio_runs += 1
    assert lio_runs == 2
    pts, prior = MS.lio_scan(c, rng, 4000)  # after the empty box and the rebuild
    _lio_compare(gpu_ctx.lio_update(pts, prior, prior, c["cfg"]), orc.o.state_estimation(pts, prior, prior))


@pytest.mark.parametrize("name", ["deep_blob_L7", "candidates_layer3"])
def test_device_build_form_on_hand_built_streams(gpu_ctx, name):
    """BuildVoxelMap (map_device_build: every point pushed, then init_octo_tree with the recursive cut) with identity pose and
    extrinsics on all the stream's points, against the oracle's BuildVoxelMap at the build tolerance, and the device's node
    count against the oracle's."""
    c = MS.case(name)
    cfg = c["cfg"]
    pb = np.concatenate([t[0] for t in c["ticks"]]).astype(np.float32)
    st = S.pack_state(np.eye(3), np.zeros(3), cov=np.eye(19) * 1e-4)
    gpu_ctx.set_extrinsics(MS.IDENTITY_EXT)
    gpu_ctx.map_device_init(cfg, root_capacity=1 << 12)
    gpu_ctx.lio_set_scan(pb)
    gpu_ctx.map_device_build(st)
    orc = MS.OracleSide(cfg, MS.IDENTITY_EXT)
    orc.o.build_map(pb, pb, st)
    n = MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten(), rtol=1e-7, what=("device map (build form)", "oracle BuildVoxelMap"))
    dump = orc.dump_nodes()
    assert gpu_ctx.map_device_stats()["nodes"] == len(dump) and gpu_ctx.map_device_stats()["errors"] == 0
    if name == "deep_blob_L7":
        assert (dump[:, MS.LAYER] == 7).any() and n == 0
    else:
        assert n == 72


@pytest.mark.parametrize("extra", [-1, 0, 1], ids=["capacity-1", "capacity", "capacity+1"])
def test_device_hash_table_to_capacity_with_concurrent_inserts(gpu_ctx, extra):
    """root_capacity 512 -> a 1024-slot table; 1023, 1024 and 1025 new roots in one tick, 7 points each, so that many warps
    insert the same and colliding keys at once (atomicCAS). Up to capacity the map equals the oracle's; one over is a status
    (MAP_ERR_HASH), and a fresh map_device_init recovers."""
    cfg, keys, pw = MS.hash_keys(1024 + extra)
    var = np.tile(MS.VAR, (len(pw), 1, 1))
    gpu_ctx.map_device_init(cfg, root_capacity=512)
    if extra > 0:
        with pytest.raises(api.EsikfError):
            gpu_ctx.map_device_update_points(pw, var)
        assert gpu_ctx.map_device_stats()["errors"] & 8
    else:
        gpu_ctx.map_device_update_points(pw, var)
        orc = MS.OracleSide(cfg)
        orc.apply(pw, var)
        MB.compare_flat_maps(gpu_ctx.map_device_download(), orc.flatten(), exact=True)
        assert gpu_ctx.map_device_stats()["roots"] == len(keys)
    gpu_ctx.map_device_init(cfg, root_capacity=1 << 12)
    gpu_ctx.map_device_update_points(pw, var)
    assert gpu_ctx.map_device_stats()["errors"] == 0 and gpu_ctx.map_device_stats()["roots"] == len(keys)


@pytest.mark.parametrize("ax", [0, 1, 2])
@pytest.mark.parametrize("side", [-1, 1])
def test_device_key_one_past_the_range_is_a_status(gpu_ctx, ax, side):
    cfg = S.LioCfg(voxel_size=0.5)
    gpu_ctx.map_device_init(cfg, root_capacity=1 << 10)
    pw, var = MS.beyond_key(ax, side)
    with pytest.raises(api.EsikfError):
        gpu_ctx.map_device_update_points(pw, var)
    assert gpu_ctx.map_device_stats()["errors"] & 16
