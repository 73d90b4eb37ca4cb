"""GPU: esikf_map_device_find (map_find_kernel, K12), the find_correspond lookups of updateReferencePatch (rule A) and of the
retrieval's ray casting (rule B) on the device-resident voxel map, against the oracle's keyed restatement
(oracle/orc_find_keyed.cpp) and the device map's own export; the map left untouched by queries; the call's refusals; and the
shim's VoxelMapManager::FindCorrespond against the host mirror's find_correspond."""

import numpy as np
import pytest

import map_bind as MB
import map_find as MF
import map_mirror as MM
import map_streams as MS
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from fast_livo2_b200.synthetic import PLANE_DTYPE
from parity_util import assert_state_close
from test_map_mirror_host import ROOM_CFGS, ROOM_IDS, room_ticks

pytestmark = pytest.mark.gpu


def _queries(exp, cfg, rng):
    """map_mirror.query_points on the tick's exported nodes (centres, faces, negatives, absent roots, random points), every
    node centre again at the 0.5 m grid the lookups key with, and the key rules' edges (NaN and infinities included)."""
    q = [MM.query_points(exp["nodes"], cfg, rng, n_random=1000), MF.boundary_points(cfg.voxel_size)]
    if len(exp["nodes"]):
        c = np.asarray(exp["nodes"]["voxel_center"], np.float64)
        q.append(np.round(c / 0.5) * 0.5)  # on the faces of the 0.5 m keys
    return np.concatenate(q)


def _check(ctx, orc, q, what, exp=None):
    checked = 0
    for name, rule in MF.RULES.items():
        got = ctx.map_device_find(q, rule)
        out, f = MF.oracle_find_keyed(orc, q, rule)
        MF.compare_with_oracle(got, out, f, f"{what}, rule {name}")
        if exp is not None:
            checked += MF.plane_bytes_equal_export(got, exp)
    return checked


def _run(cfg, ticks, slides=None, grow=False, root_capacity=1 << 14):
    ctx, orc = api.Context(0), MS.OracleSide(cfg)
    rng = np.random.default_rng(17)
    stat, checked = np.zeros(3, np.int64), 0
    try:
        ctx.map_device_init(cfg, root_capacity=root_capacity, grow=grow)
        for t, (pw, var) in enumerate(ticks):
            ctx.map_device_update_points(pw, var)  # the find below is enqueued after it with no host synchronisation in between
            orc.apply(pw, var)
            exp = ctx.map_device_export()
            q = _queries(exp, cfg, rng)
            checked += _check(ctx, orc, q, f"tick {t}", exp)
            stat += np.bincount(ctx.map_device_find(q, 0)["status"], minlength=3)
            if slides and t in slides:
                ctx.map_device_slide(*slides[t]), orc.slide(*slides[t])
                _check(ctx, orc, q, f"after the slide of tick {t}")
        return stat, checked
    finally:
        ctx.close()


@pytest.mark.parametrize("cfg", ROOM_CFGS, ids=ROOM_IDS)
def test_find_equals_the_oracle_on_room_scenes(cfg):
    """Room ticks at voxel 0.5, 0.4 and 2.0 (where the 0.5 m lookups key other roots than the map inserts), on a map that
    starts small and grows, with a slide after the third tick."""
    lo = [int(np.floor(-6.0 / cfg.voxel_size)), -10**6, -10**6]
    stat, checked = _run(cfg, list(room_ticks(cfg)), slides={2: (lo, [10**6] * 3)}, grow=True, root_capacity=1 << 9)
    assert stat[0] > 0 and stat[2] > 0
    assert checked > 0 or cfg.voxel_size != 0.5  # at 2.0 the 0.5 m keys rarely name a root the map holds


@pytest.mark.parametrize("name", list(MS.CASES))
def test_find_equals_the_oracle_on_streams(name):
    c = MS.case(name)
    _run(c["cfg"], c["ticks"], c.get("slides"))


def test_find_reaches_every_answer():
    """Both rules, on the layer-3 room and the deep blobs: no root, a plane, and a node that is not a plane."""
    seen = np.zeros(3, np.int64)
    for cfg, ticks in ((ROOM_CFGS[1], list(room_ticks(ROOM_CFGS[1], 4))), (MS.case("deep_blob_L3")["cfg"], MS.case("deep_blob_L3")["ticks"])):
        seen += _run(cfg, ticks)[0]
    assert (seen > 0).all(), seen


def _room_lio(cfg, n_ticks=3):
    """A LIO tick loop on the room scene: the first scan builds the map, every later one is a lio_update + map_device_update."""
    ext = S.avia_extrinsics()
    rng = np.random.default_rng(2)
    rects = S.make_scene("room", 0.5)
    R, p = np.eye(3), np.array([-1.0, 0.4, 0.3])
    st = S.pack_state(R, p, cov=S.random_prior_cov(np.random.default_rng(3), scale=0.05), g=np.array([0, 0, -9.81]))
    scans = [S.scan_at(rects, ext, R, p + np.array([0.1 * k, 0, 0]), 20000, cfg, rng) for k in range(n_ticks)]
    return ext, st, scans


def _map_bytes(ctx):
    d = ctx.map_device_download()
    order = np.lexsort((d["keys"][:, 2], d["keys"][:, 1], d["keys"][:, 0]))
    planes = [d["planes"][d["first"][i]:d["first"][i] + d["count"][i]].tobytes() for i in order]
    return d["keys"][order].tobytes() + b"".join(planes)


def test_queries_leave_the_map_untouched():
    """A map queried with thousands of absent roots (more than its hash table holds) is byte-identical before and after:
    download and export; a map update after the queries still fits the small table and gives the map of a context that made
    no queries; the LIO updates and map updates after it agree with that context's."""
    cfg = S.LioCfg()
    ext, st, scans = _room_lio(cfg)
    ctxs = [api.Context(0), api.Context(0)]
    try:
        for c in ctxs:
            c.set_extrinsics(ext)
            c.map_device_init(cfg, root_capacity=1 << 12)
            c.lio_set_scan(scans[0])
            c.map_device_build(st)
        q, absent = ctxs[0], np.random.default_rng(9).uniform(-3e4, 3e4, (20000, 3))
        before, exp0 = _map_bytes(q), q.map_device_export()
        for rule in MF.RULES.values():
            for _ in range(2):
                q.map_device_find(absent, rule)
        assert _map_bytes(q) == before
        exp1 = q.map_device_export()
        assert exp1["nodes"].tobytes() == exp0["nodes"].tobytes() and exp1["keys"].tobytes() == exp0["keys"].tobytes()
        assert q.map_device_stats() == ctxs[1].map_device_stats()
        # a map update first: an inserting lookup would have filled the small table, and this tick would not fit it
        pw, var = next(room_ticks(cfg, 1, seed=12))
        for c in ctxs:
            c.map_device_update_points(pw, var)
        assert _map_bytes(ctxs[0]) == _map_bytes(ctxs[1])
        for scan in scans[1:]:
            outs = []
            for c in ctxs:
                g = c.lio_update(scan, st, st, cfg)
                c.map_device_update()
                outs.append(g)
            # two contexts lay the same map out in different record slots (concurrent inserts), and their LIO posteriors
            # have been seen to differ in the last bits: this step is compared to the tolerance of test_gpu_map
            assert_state_close(outs[0]["state"], outs[1]["state"])
            MB.compare_flat_maps(ctxs[0].map_device_download(), ctxs[1].map_device_download(), rtol=1e-6, what=("queried", "not queried"))
    finally:
        for c in ctxs:
            c.close()


def test_find_after_a_lio_tick_without_synchronising():
    """lio_update + map_device_update, then the query straight away with no host synchronisation: it answers from the
    updated map (the export of that update, taken afterwards, holds the same plane bytes)."""
    cfg = S.LioCfg()
    ext, st, scans = _room_lio(cfg, 2)
    ctx = api.Context(0)
    try:
        ctx.set_extrinsics(ext)
        ctx.map_device_init(cfg, root_capacity=1 << 14)
        ctx.lio_set_scan(scans[0])
        ctx.map_device_build(st)
        q = _queries(ctx.map_device_export(), cfg, np.random.default_rng(1))
        ctx.lio_update(scans[1], st, st, cfg)
        ctx.map_device_update()
        got = ctx.map_device_find(q, 0)
        exp = ctx.map_device_export()
        assert (got["status"] == 2).sum() > 100
        assert MF.plane_bytes_equal_export(got, exp) > 100
    finally:
        ctx.close()


def _raw(ctx, pts, n, rule, bufs):
    st, keys, rows = bufs
    return ctx.lib.esikf_map_device_find(ctx.h, None if pts is None else pts.ctypes.data, n, rule, None if st is None else st.ctypes.data,
                                         None if keys is None else keys.ctypes.data, None if rows is None else rows.ctypes.data)


def test_find_refusals_write_nothing():
    cfg = S.LioCfg()
    pts = np.array([[0.3, 0.3, 0.3], [1.2, -0.7, 0.1]], np.float64)

    def bufs():
        return np.full(2, 0xAB, np.uint8), np.full((2, 3), 7, np.int64), np.frombuffer(np.full(2 * PLANE_DTYPE.itemsize, 0xCD, np.uint8).tobytes(), PLANE_DTYPE).copy()

    def untouched(b):
        return (b[0] == 0xAB).all() and (b[1] == 7).all() and (b[2].view(np.uint8) == 0xCD).all()

    ctx = api.Context(0)
    try:
        b = bufs()
        assert _raw(ctx, pts, 2, 0, b) == -4 and untouched(b)  # no map
        ctx.map_upload(dict(keys=np.zeros((0, 3), np.int64), first=np.zeros(0, np.int32), count=np.zeros(0, np.int32), planes=np.zeros(0, PLANE_DTYPE)), 0.5)
        assert _raw(ctx, pts, 2, 0, b) == -4 and untouched(b)  # a host-uploaded map is not a device map
        ctx.map_device_init(cfg, root_capacity=1 << 10)
        ctx.map_device_update_points(*next(room_ticks(cfg, 1)))
        assert _raw(ctx, pts, 2, 0, b) == 0 and not untouched(b)
        for args in ((pts, -1, 0), (pts, 2, 2), (pts, 2, -1)):
            b = bufs()
            assert _raw(ctx, *args, b) == -3 and untouched(b)
        for k in range(4):  # a NULL buffer with n > 0
            b = bufs()
            nb = tuple(None if j == k - 1 else x for j, x in enumerate(b))
            assert _raw(ctx, None if k == 0 else pts, 2, 1, nb) == -3 and untouched(b)
        assert _raw(ctx, None, 0, 0, (None, None, None)) == 0  # n == 0
        assert len(ctx.map_device_find(np.zeros((0, 3)), 1)["status"]) == 0
        ctx.map_upload(dict(keys=np.zeros((0, 3), np.int64), first=np.zeros(0, np.int32), count=np.zeros(0, np.int32), planes=np.zeros(0, PLANE_DTYPE)), 0.5)
        b = bufs()
        assert _raw(ctx, pts, 2, 0, b) == -4 and untouched(b)  # replaced by esikf_map_upload
    finally:
        ctx.close()
    ctx = api.Context(0)
    try:
        ctx.map_device_init(cfg, root_capacity=1 << 12, node_capacity=64)
        with pytest.raises(api.EsikfError):
            ctx.map_device_update_points(*next(room_ticks(cfg, 1)))  # 64 nodes are too few, growth is off
        b = bufs()
        assert _raw(ctx, pts, 2, 0, b) == -4 and untouched(b)  # invalidated by the failed update
    finally:
        ctx.close()


def _shim_find(lib, h, q, rule):
    q = np.ascontiguousarray(q, np.float64)
    st, rows = np.zeros(len(q), np.uint8), np.zeros(len(q), PLANE_DTYPE)
    assert lib.fl2_shim_session_find_correspond(h, q.ctypes.data, len(q), rule, st.ctypes.data, rows.ctypes.data) == 0
    return st, rows


def test_shim_find_correspond_equals_the_mirror_and_needs_none():
    """Two sessions on the same LIO ticks at voxel 0.5, mirror on and off: on the first, FindCorrespond (rule A) finds the node
    the mirror's find_correspond finds, with the device's plane fields; on both it answers what esikf_map_device_find does."""
    cfg = S.LioCfg()
    ext, st, scans = _room_lio(cfg, 3)
    lib = MM.shim_sessions()
    hs = [MM.session(lib, cfg, ext), MM.session(lib, cfg, ext)]
    try:
        for h, mirror in zip(hs, (1, 0)):
            lib.fl2_shim_session_point_lists(h, 2)
            assert lib.fl2_shim_session_device_map_mirror(h, MM.vp(scans[0]), len(scans[0]), MM.vp(st), cfg.min_eigen_value, cfg.max_points_num, 1 << 16, 0, mirror) == 0
        for scan in scans[1:]:
            for h in hs:
                assert lib.fl2_shim_session_step(h, MM.vp(scan), len(scan), MM.vp(st), MM.vp(st), None, 0, None, None, None, None, MM.vp(np.zeros(386)),
                                                 MM.vp(np.zeros(386)), MM.vp(np.zeros(2, np.int32))) == 0
                assert lib.fl2_shim_session_update_map(h) == 0
        view = MM.MirrorView(hs[0], lib)
        flat = view.flatten()
        q = np.concatenate([(flat["keys"] + 0.5) * 0.5,
                            (flat["keys"] + np.random.default_rng(3).uniform(0, 1, flat["keys"].shape)) * 0.5, MF.boundary_points()])
        mirror = view.find(q)
        answers = []
        for h in hs:
            with MM.SessionContext(lib, h) as c:
                dev = {name: c.map_device_find(q, rule) for name, rule in MF.RULES.items()}
            for name, rule in MF.RULES.items():
                s, rows = _shim_find(lib, h, q, rule)
                d = dev[name]
                assert np.array_equal(s, d["status"])
                for f in ("center", "normal", "plane_var", "d", "radius"):
                    assert rows[f].tobytes() == d["planes"][f].tobytes(), f
            answers.append(dev["patch"])
        a = answers[0]
        got = np.stack([a["status"] != 0, a["planes"]["layer"], a["planes"]["path"], a["status"] == 2], axis=1).astype(np.int64)
        assert np.array_equal(got, mirror), f"differs from the mirror on {int(np.any(got != mirror, axis=1).sum())} of {len(q)} points"
        assert (mirror[:, 3] == 1).sum() > 100 and (mirror[:, 0] == 0).any()
        # the two sessions ran the same ticks, but their LIO posteriors may differ in the last bits (records land in other
        # slots): the same nodes exactly, their planes to test_gpu_map's tolerance
        b = answers[1]
        assert np.array_equal(a["status"], b["status"]) and np.array_equal(a["planes"]["layer"], b["planes"]["layer"]) and np.array_equal(a["planes"]["path"], b["planes"]["path"])
        for f in ("center", "normal", "plane_var", "d", "radius"):
            np.testing.assert_allclose(a["planes"][f], b["planes"][f], rtol=1e-6, atol=1e-9, err_msg=f)
    finally:
        for h in hs:
            lib.fl2_shim_session_destroy(h)
