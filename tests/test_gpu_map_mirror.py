"""GPU: esikf_map_device_export (map_export_count_kernel / map_export_kernel) against the oracle, its refusals, and the
shim's host mirror of the device map (VoxelMapConfig::device_map_mirror_) through LIO ticks, failures, growth and slides."""
import numpy as np
import pytest

import map_bind as MB
import map_mirror as MM
import map_streams as MS
import oracle_bind as O
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from test_map_mirror_host import ROOM_CFGS, ROOM_IDS, room_ticks

pytestmark = pytest.mark.gpu


def _export_matches_oracle(cfg, ticks, slides=None, **caps):
    ctx, orc = api.Context(0), MS.OracleSide(cfg)
    try:
        ctx.map_device_init(cfg, root_capacity=caps.pop("root_capacity", 1 << 14), **caps)
        with pytest.raises(api.EsikfError):
            ctx.map_device_export()  # nothing to export after init
        for t, (pw, var) in enumerate(ticks):
            ctx.map_device_update_points(pw, var)
            orc.apply(pw, var)
            exp = ctx.map_device_export()
            assert ctx.map_device_export()["nodes"].tobytes() == exp["nodes"].tobytes()
            assert len(exp["keys"]) == ctx.map_device_stats()["touched_roots"]
            what = (f"device export, tick {t}", "oracle")
            MB.compare_node_dumps(MM.export_dump(exp), MM.rows_of(orc.dump_nodes(), exp["keys"]), what, a_releases_cut_lists=True)
            MB.compare_flat_maps(MM.export_flat(exp), MM.flat_of(orc.flatten(), exp["keys"]), what=what, exact=True)
            if slides and t in slides:
                ctx.map_device_slide(*slides[t]), orc.slide(*slides[t])
                with pytest.raises(api.EsikfError):
                    ctx.map_device_export()  # the slide's bounds say what went
    finally:
        ctx.close()


@pytest.mark.parametrize("cfg", ROOM_CFGS, ids=ROOM_IDS)
def test_device_export_equals_the_oracle_on_room_scenes(cfg):
    _export_matches_oracle(cfg, list(room_ticks(cfg)))


@pytest.mark.parametrize("name", list(MS.CASES))
def test_device_export_equals_the_oracle_on_streams(name):
    c = MS.case(name)
    _export_matches_oracle(c["cfg"], c["ticks"], c.get("slides"))


def test_export_is_refused_after_a_failed_update():
    cfg = ROOM_CFGS[0]
    ticks = list(room_ticks(cfg, 2))
    ctx = api.Context(0)
    try:
        ctx.map_device_init(cfg, root_capacity=1 << 12, node_capacity=64)
        with pytest.raises(api.EsikfError):
            ctx.map_device_update_points(*ticks[0])  # 64 nodes are too few, growth is off
        with pytest.raises(api.EsikfError, match="no build / update"):
            ctx.map_device_export()
    finally:
        ctx.close()


def _lio_loop_poses(k):
    R = S.so3_exp(np.array([0.002 * k, -0.001 * k, 0.01 * k]))
    p = np.array([-2.0 + 0.12 * k, 0.5 - 0.05 * k, 0.3 + 0.01 * k])
    return R, p


def _queries(keys, cfg, rng, n_roots=300):
    """find_correspond queries in a sample of roots: the root centre, its faces, the centres of every layer-1 and layer-2
    node, and random points, plus a point of an absent root."""
    keys = keys[rng.choice(len(keys), min(n_roots, len(keys)), replace=False)].astype(np.float64)
    vs = cfg.voxel_size
    offs = [(np.array(o) - 1) * vs / 4 for o in np.ndindex(3, 3, 3)]  # the centre, points on its split planes, layer-1 centres
    offs += [np.array([i, j, k]) * vs / 8 for i in (-3, -1, 1, 3) for j in (-3, -1, 1, 3) for k in (-3, -1, 1, 3)]  # layer-2 centres
    c = (keys + 0.5) * vs
    pts = [c + o for o in offs] + [c - vs / 2, c + rng.uniform(-0.5, 0.5, c.shape) * vs, c + 1000.0]  # + the root's lower corner
    return np.concatenate(pts)


def test_shim_mirror_through_lio_ticks_tracks_the_oracle():
    """The LIO tick loop of test_gpu_map (BuildVoxelMap, then per tick StateEstimation and UpdateVoxelMap() at a moving pose)
    through two shim sessions, mirror on and off, next to the oracle's StateEstimation + UpdateVoxelMap on native octrees.
    After every tick: the mirror's node dump equals the oracle's (every node, every counter), its planes equal the oracle's
    to test_gpu_map's tolerance and flatten to exactly the device map's download, its find_correspond answers equal the
    oracle's; the posteriors of the two sessions are bit-identical; and the mirror-off session launches per tick what the
    same calls on a plain C-ABI context launch."""
    cfg, ext = S.LioCfg(), S.avia_extrinsics()
    rng, qrng = np.random.default_rng(21), np.random.default_rng(5)
    rects = S.make_scene("room", 0.5)
    orc = O.OracleLIO(cfg, ext)
    R0, p0 = _lio_loop_poses(0)
    st0 = S.pack_state(R0, p0, cov=S.random_prior_cov(np.random.default_rng(3), scale=0.05), g=np.array([0, 0, -9.81]))
    scan0 = S.scan_at(rects, ext, R0, p0, 60000, cfg, rng)
    lib = MM.shim_sessions()
    hs = [MM.session(lib, cfg, ext), MM.session(lib, cfg, ext)]
    plain = api.Context(0)
    try:
        for h, mirror in zip(hs, (1, 0)):
            lib.fl2_shim_session_point_lists(h, 2)  # StateEstimation = esikf_lio_update, as on the plain context
            assert lib.fl2_shim_session_device_map_mirror(h, MM.vp(scan0), len(scan0), MM.vp(st0), cfg.min_eigen_value, cfg.max_points_num, 1 << 16, 0, mirror) == 0
        plain.set_extrinsics(ext)
        plain.map_device_init(cfg, root_capacity=1 << 16)
        plain.lio_set_scan(scan0)
        plain.map_device_build(st0)
        orc.tick_build_map(scan0, st0)
        view = MM.MirrorView(hs[0], lib)
        state = st0
        for k in range(1, 11):
            Rk, pk = _lio_loop_poses(k)
            scan = S.scan_at(rects, ext, Rk, pk, 20000, cfg, rng)
            s = S.unpack_state(state)
            prior = S.pack_state(Rk @ S.so3_exp(np.array([0.002, -0.003, 0.002])), pk + np.array([0.02, -0.015, 0.01]), cov=s["cov"] + np.eye(19) * 1e-6,
                                 g=np.array([0, 0, -9.81]))
            outs, launches = [], []
            for h in hs:
                with MM.SessionContext(lib, h) as c:
                    before = c.launch_count()
                    out = np.zeros(386)
                    assert lib.fl2_shim_session_step(h, MM.vp(scan), len(scan), MM.vp(prior), MM.vp(prior), None, 0, None, None, None, None, MM.vp(out),
                                                     MM.vp(np.zeros(386)), MM.vp(np.zeros(2, np.int32))) == 0
                    assert lib.fl2_shim_session_update_map(h) == 0
                    outs.append(out), launches.append(c.launch_count() - before)
            before = plain.launch_count()
            plain.lio_update(scan, prior, prior, cfg)
            plain.map_device_update()
            assert launches[1] == plain.launch_count() - before, f"tick {k}: the mirror-off session launched {launches[1]}, the C ABI {plain.launch_count() - before}"
            assert launches[0] > launches[1]  # the export
            assert outs[0].tobytes() == outs[1].tobytes(), f"tick {k}: the mirror changed the posterior"
            orc.state_estimation(scan, prior, prior)
            orc.tick_update_map()
            what = (f"mirror, tick {k}", "oracle")
            MB.compare_node_dumps(view.dump_nodes(), orc.dump_nodes(), what, a_releases_cut_lists=True)
            flat = view.flatten()
            MB.compare_flat_maps(flat, orc.flatten(), rtol=1e-6, what=what)
            with MM.SessionContext(lib, hs[0]) as c:
                MB.compare_flat_maps(flat, c.map_device_download(), what=(f"mirror, tick {k}", "device"), exact=True)
            q = _queries(flat["keys"], cfg, qrng)
            got, want = view.find(q), MM.oracle_find(orc, q)
            assert np.array_equal(got, want), f"tick {k}: find_correspond differs on {int(np.any(got != want, axis=1).sum())} of {len(q)} points"
            assert (want[:, 0] == 0).any() and (want[:, 3] == 1).any() and ((want[:, 0] == 1) & (want[:, 3] == 0)).any()
            state = outs[0]
    finally:
        plain.close()
        for h in hs:
            lib.fl2_shim_session_destroy(h)


def test_a_failed_update_voids_the_mirror_until_the_map_is_rebuilt(small_vio_frame):
    """UpdateVoxelMap() refused (the scan has not been through StateEstimation) leaves the device map as it was, but the
    mirror misses a tick from then on: it stays empty and every later UpdateVoxelMap() reports an error, also one that
    succeeds on the device, until EnableDeviceMap() + BuildVoxelMap() rebuild it."""
    fr = small_vio_frame
    cfg, ext, rects = fr["lio_cfg"], fr["ext"], fr["rects"]
    lib = MM.shim_sessions()
    h = MM.session(lib, cfg, ext)
    try:
        rng = np.random.default_rng(8)
        t = S.unpack_state(fr["state_true"])
        st0 = S.pack_state(t["R"], t["p"], cov=S.random_prior_cov(np.random.default_rng(1), scale=0.05), g=np.array([0, 0, -9.81]))
        scan0 = S.scan_at(rects, ext, t["R"], t["p"], 30000, cfg, rng)
        build = lambda: lib.fl2_shim_session_device_map_mirror(h, MM.vp(scan0), len(scan0), MM.vp(st0), cfg.min_eigen_value, cfg.max_points_num, 1 << 15, 0, 1)
        assert build() == 0
        view = MM.MirrorView(h, lib)
        assert len(view.flatten()["keys"]) > 0
        assert lib.fl2_shim_session_update_map(h) != 0  # refused: no StateEstimation on this scan yet
        assert len(view.dump_nodes()) == 0
        prior = S.pack_state(t["R"], t["p"] + np.array([0.01, -0.01, 0.005]), cov=S.unpack_state(st0)["cov"], g=np.array([0, 0, -9.81]))
        for _ in range(2):
            scan = S.scan_at(rects, ext, t["R"], t["p"], 8000, cfg, rng)
            assert lib.fl2_shim_session_step(h, MM.vp(scan), len(scan), MM.vp(prior), MM.vp(prior), None, 0, None, None, None, None, MM.vp(np.zeros(386)),
                                             MM.vp(np.zeros(386)), MM.vp(np.zeros(2, np.int32))) == 0
            assert lib.fl2_shim_session_update_map(h) != 0, "a mirror that missed a tick reports success"
            assert len(view.dump_nodes()) == 0, "a mirror that missed a tick holds a partial map"
        assert build() == 0  # EnableDeviceMap + BuildVoxelMap: a new map, mirrored from its first tick
        with MM.SessionContext(lib, h) as c:
            MB.compare_flat_maps(view.flatten(), c.map_device_download(), what=("rebuilt mirror", "device"), exact=True)
    finally:
        lib.fl2_shim_session_destroy(h)


SLIDES = {1: ((0, 0, 1), 2), 3: ((0, 1, 0), 1)}  # after tick t: (sensor voxel, half_map_size)


@pytest.mark.parametrize("grow", [0, 1], ids=["fixed", "growing"])
def test_shim_mirror_with_updates_slides_and_growth_equals_the_oracle(small_vio_frame, grow):
    """UpdateVoxelMap(input_points) ticks of the slide stream, with mapSliding between them, through a session whose map starts
    tiny and grows (a hash growth on an update tick included) or is large and fixed: after every step the mirror's node dump,
    flattening and find_correspond answers equal the oracle's (UpdateVoxelMap + clearMemOutOfMap)."""
    c = MS.case("slide")
    cfg = c["cfg"]
    lcfg = S.LioCfg(**{**small_vio_frame["lio_cfg"].__dict__, "voxel_size": cfg.voxel_size, "max_layer": cfg.max_layer})
    lib = MM.shim_sessions()
    h = MM.session(lib, lcfg, small_vio_frame["ext"])
    orc = MS.OracleSide(cfg)
    try:
        empty = np.zeros((0, 3), np.float32)
        state = np.ascontiguousarray(small_vio_frame["state_true"])
        assert lib.fl2_shim_session_device_map_mirror(h, MM.vp(empty), 0, MM.vp(state), cfg.min_eigen_value, cfg.max_points_num, 16 if grow else 1 << 14, grow, 1) == 0
        view = MM.MirrorView(h, lib)
        rng = np.random.default_rng(4)
        for t, (pw, var) in enumerate(c["ticks"]):
            pw, var = np.ascontiguousarray(pw, np.float64), np.ascontiguousarray(np.asarray(var).reshape(-1, 9), np.float64)
            assert lib.fl2_shim_session_update_points(h, MM.vp(pw), MM.vp(var), len(pw)) == 0
            orc.apply(pw, var)
            steps = [f"tick {t}"]
            if t in SLIDES:  # mapSliding keeps [loc - half, loc + half] around the sensor's voxel loc
                loc, half = SLIDES[t]
                pos = (np.array(loc, np.float64) + 0.5) * cfg.voxel_size
                assert lib.fl2_shim_session_map_sliding(h, MM.vp(pos), half, 0.0) == 0
                orc.slide(np.array(loc) - half, np.array(loc) + half)
                steps.append("slide")
            what = (f"mirror after {' + '.join(steps)}", "oracle")
            MB.compare_node_dumps(view.dump_nodes(), orc.dump_nodes(), what, a_releases_cut_lists=True)
            MB.compare_flat_maps(view.flatten(), orc.flatten(), what=what, exact=True)
            d = orc.flatten()
            if len(d["keys"]):
                q = np.concatenate([(d["keys"] + 0.5) * cfg.voxel_size, (d["keys"] + rng.uniform(0, 1, d["keys"].shape)) * cfg.voxel_size])
                assert np.array_equal(view.find(q), MM.oracle_find(orc, q))
        if grow:
            with MM.SessionContext(lib, h) as ctx:
                assert ctx.map_device_capacity()["root_capacity"] > 16
    finally:
        lib.fl2_shim_session_destroy(h)
