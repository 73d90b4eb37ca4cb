"""GPU: the map side of the visual sub-map retrieval (esikf_vmap_place_points / esikf_vmap_retrieve, K15) against the oracle's
walk and depth check (oracle/orc_retrieve.cpp over the map the reference's insertion makes, tests/vmap_retrieve_cases.py) and
against the separate calls it replaces (esikf_vio_depth_check, esikf_vmap_choose_ref)."""
import ctypes as C

import numpy as np
import pytest

import retrieve_cases as RC
import vmap_retrieve_cases as VR
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _store(ctx, n_obs, seed, capacity=1):
    """n store points with n_obs[i] observations each (random patches, ids and camera centres), from a store of `capacity`."""
    rng = np.random.default_rng(seed)
    ctx.vmap_init(capacity)
    first = np.concatenate([[0], np.cumsum(n_obs)]).astype(np.int32)
    m = int(first[-1])
    T = np.zeros((m, 12))
    T[:, [0, 4, 8]] = 1.0
    T[:, 9:] = rng.normal(0, 2.0, (m, 3))
    ids = ctx.vmap_add_points(first, np.zeros((m, 2)), rng.uniform(0, 255, (m, 64)).astype(np.float32), T, rng.integers(0, 5, m).astype(np.int32),
                              np.zeros(m, np.float32), np.zeros(m, np.float32), np.full(len(n_obs), -1, np.int32))
    assert np.array_equal(ids, np.arange(len(n_obs)))


def _frame_pos(sc):
    st = S.unpack_state(sc["state"])
    R, t = S.camera_pose(sc["ext"], st["R"], st["p"])
    return -(R.T @ t)


def _equal(got, want, label):
    """The walk, depth check and skip; a kept point without a reference feature counts as kept here."""
    status = np.where(got["status"] == VR.NO_REF, VR.KEPT, got["status"]).astype(np.int32)
    for f in ("cell", "point_id", "pc"):
        assert np.asarray(got[f]).tobytes() == np.asarray(want[f]).tobytes(), (label, f)
    assert status.tobytes() == want["status"].tobytes(), label


def _grid(sc):
    return [int(sc[k]) for k in ("grid_size", "grid_n_width", "grid_n_height", "border")]


@pytest.mark.parametrize("normal_en", [True, False])
def test_pinhole_scene_matches_the_oracle(normal_en):
    """Points placed over three calls (ascending thirds, shuffled within each) into a store and point arrays grown from capacity
    1, so that each growth carries placed points over: cells, winners,
    pc and statuses equal the oracle's walk and depth check; the refs equal esikf_vmap_choose_ref on the kept points of a
    second context with the same store (and the stored refs after normal_en)."""
    sc = RC.scene("pinhole", 100_000, seed=7, n_vis=6000)
    n = len(sc["pos"])
    rng = np.random.default_rng(1)
    order = np.concatenate([rng.permutation(part) for part in np.array_split(np.arange(n), 3)]).astype(np.int32)  # ascending thirds, shuffled within
    ninit = (rng.random(n) > 0.1).astype(np.uint8)
    ctxs = [api.Context(0), api.Context(0)]
    try:
        for c in ctxs:
            _store(c, sc["n_obs"], seed=2)
            c.set_extrinsics(sc["ext"])
            c.vio_set_camera(sc["cam"], RC.VIO_CFG)
        a, b = ctxs
        for part in np.array_split(order, 3):
            a.vmap_place_points(part, sc["pos"][part], ninit[part])
        scan = a.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"], depth=True)
        orc = RC.OracleRetrieve(sc)
        want_scan = orc.scan(sc)
        assert np.array_equal(scan["keys"].astype(np.int64), want_scan["keys"])
        vis = VR.placed_visual_map(sc["pos"], sc["n_obs"], order)
        walk, want = VR.composed(orc, sc, vis, want_scan["keys"], want_scan["depth"], ninit)
        got = a.vmap_retrieve(walk, *_grid(sc), normal_en)
        _equal(got, want, "pinhole")
        st = want["status"]
        assert len(st) > 200 and (st == VR.KEPT).sum() > 100 and (st == VR.DEPTH).sum() > 0 and (st == VR.NOT_INIT).sum() > 0
        # the reference choice of the kept points, against the separate call on the same store
        kept = got["status"] != VR.DEPTH
        kept &= got["status"] != VR.NOT_INIT
        kept &= got["status"] != VR.NO_WINNER
        pid = got["point_id"][kept]
        ref = b.vmap_choose_ref(pid, normal_en, pos=sc["pos"][pid], frame_pos=_frame_pos(sc))
        assert np.array_equal(got["ref"][kept], ref)
        assert np.array_equal(got["status"][kept] == VR.NO_REF, ref < 0)
        assert (got["ref"][~kept] == -1).all()
        all_ids = np.arange(n, dtype=np.int32)
        assert np.array_equal(a.vmap_download(all_ids)["ref"], b.vmap_download(all_ids)["ref"])
        # the same walk again: the same answers (normal_en: the stored refs are now read back as the refs)
        again = a.vmap_retrieve(walk, *_grid(sc), normal_en)
        for f in got:
            assert np.asarray(again[f]).tobytes() == np.asarray(got[f]).tobytes(), f
    finally:
        for c in ctxs:
            c.close()


def _edge_ctx(ctx, pos, n_obs=None):
    sc = RC.edge_scene()
    ctx.set_extrinsics(sc["ext"])
    ctx.vio_set_camera(sc["cam"], RC.VIO_CFG)
    _store(ctx, np.ones(len(pos), np.int32) if n_obs is None else n_obs, seed=3)
    # a scan 1 mm behind each visual point: the depth image holds no discontinuity at them
    ctx.vio_retrieve_scan(sc["border"], pg=pos + np.array([0.0, 0.0, 0.001]), state=sc["state"])
    return sc


def test_ties_follow_the_walk_order(gpu_ctx):
    """Duplicate positions in one voxel: the point placed last wins, whichever order they were placed in. Equal float distances
    from two voxels (x and y swapped): the point of the key later in the walk wins, and reversing the walk swaps the winner."""
    dup = np.array([[0.3, 0.2, 8.0]] * 3)
    swap = np.array([[4.99, 5.01, 20.0], [5.01, 4.99, 20.0]])  # one grid cell, keys 9 and 10, the same distance
    pos = np.concatenate([dup, swap])
    sc = _edge_ctx(gpu_ctx, pos)
    g = _grid(sc)
    keys = VR.insertion_keys(pos).astype(np.int32)
    assert not np.array_equal(keys[3], keys[4])
    for perm in ([0, 1, 2], [2, 0, 1], [1, 2, 0]):
        ctx = api.Context(0)
        try:
            _edge_ctx(ctx, pos)
            for i in perm:
                ctx.vmap_place_points([i], pos[i:i + 1])
            ctx.vmap_place_points([3, 4], swap)
            for walk, winner in (([keys[0], keys[3], keys[4]], 4), ([keys[4], keys[0], keys[3]], 3)):
                got = ctx.vmap_retrieve(np.array(walk), *g, True)
                cells = {int(c): int(p) for c, p in zip(got["cell"], got["point_id"])}
                assert len(cells) == 2, cells
                assert sorted(cells.values()) == sorted([perm[-1], winner]), (perm, walk, cells)
        finally:
            ctx.close()


def test_negative_coordinates_use_the_insertion_key(gpu_ctx):
    """x = -0.3: insertion key -1, scan key -2. A walk with the scan key finds nothing; with the insertion key the point is
    retrieved. Quotients whose float narrowing moves the key land where the restatement puts them."""
    nxt = lambda x: np.nextafter(x, np.inf)  # noqa: E731
    pos = np.array([[-0.3, -0.2, 6.0], [nxt(-1.0), 0.2, 6.5], [-0.5000000001, 0.3, 7.0], [0.4999999999, -0.3, 7.5], [-1e-9, 0.1, 5.0]])
    sc = _edge_ctx(gpu_ctx, pos)
    gpu_ctx.vmap_place_points(np.arange(len(pos)), pos)
    ins, scn = VR.insertion_keys(pos), RC.voxel_keys(pos)
    assert ins[0, 0] == -1 and scn[0, 0] == -2
    assert (ins != scn).any(axis=1).sum() >= 3
    g = _grid(sc)
    for i in range(len(pos)):
        none = gpu_ctx.vmap_retrieve(scn[i:i + 1].astype(np.int32), *g, True) if (ins[i] != scn[i]).any() else None
        if none is not None:
            assert len(none["cell"]) == 0 or i not in none["point_id"].tolist()
        got = gpu_ctx.vmap_retrieve(ins[i:i + 1].astype(np.int32), *g, True)
        assert i in got["point_id"].tolist(), i


def test_empty_map_and_no_keys(gpu_ctx):
    sc = RC.scene("pinhole", 5000, seed=4)
    gpu_ctx.set_extrinsics(sc["ext"])
    gpu_ctx.vio_set_camera(sc["cam"], RC.VIO_CFG)
    _store(gpu_ctx, sc["n_obs"], seed=1)
    scan = gpu_ctx.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"])
    assert len(gpu_ctx.vmap_retrieve(scan["keys"], *_grid(sc), True)["cell"]) == 0  # nothing placed
    gpu_ctx.vmap_place_points(np.arange(len(sc["pos"])), sc["pos"])
    assert len(gpu_ctx.vmap_retrieve(np.zeros((0, 3), np.int32), *_grid(sc), True)["cell"]) == 0
    assert len(gpu_ctx.vmap_retrieve(scan["keys"], *_grid(sc), True)["cell"]) > 0


def _status(fn):
    with pytest.raises(api.EsikfError) as e:
        fn()
    return int(str(e.value).split(":")[0].split()[1])


def test_refusals_write_nothing():
    sc = RC.scene("pinhole", 20000, seed=5, n_vis=2000)
    n = len(sc["pos"])
    ctx = api.Context(0)
    try:
        ctx.set_extrinsics(sc["ext"])
        ctx.vio_set_camera(sc["cam"], RC.VIO_CFG)
        assert _status(lambda: ctx.vmap_place_points([0], sc["pos"][:1])) == -4  # no store
        _store(ctx, np.maximum(sc["n_obs"], 2), seed=6, capacity=16)
        g = _grid(sc)
        assert _status(lambda: ctx.vmap_retrieve(np.zeros((1, 3), np.int32), *g, True)) == -4  # no scan
        half = np.arange(n // 2, dtype=np.int32)
        ctx.vmap_place_points(half, sc["pos"][half])
        scan = ctx.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"])
        base = ctx.vmap_retrieve(scan["keys"], *g, False)
        refs0 = ctx.vmap_download(np.arange(n, dtype=np.int32))["ref"]
        bad_pos = sc["pos"][n // 2: n // 2 + 2].copy()
        bad_pos[1, 2] = np.nan
        for ids, p in (([n], sc["pos"][:1]), ([3], sc["pos"][3:4]), ([n // 2, n // 2], sc["pos"][:2]), ([n // 2, n // 2 + 1], bad_pos),
                       ([n // 2], np.array([[2.0 ** 19, 0.0, 1.0]]))):
            assert _status(lambda: ctx.vmap_place_points(ids, p)) == -3, ids
        edge = np.array([[2.0 ** 19 - 0.25, 0.0, 1.0]])  # key 2^20 - 1: in range
        dup = np.concatenate([scan["keys"], scan["keys"][:1]])
        gw = list(g)
        gw[1] = (sc["cam"].width - sc["border"]) // g[0] - 1
        for fn in (lambda: ctx.vmap_retrieve(dup, *g, True), lambda: ctx.vmap_retrieve(scan["keys"], *gw, True),
                   lambda: ctx.vmap_retrieve(scan["keys"], *g, True, cap=len(base["cell"]) - 1)):
            assert _status(fn) == -3
        # a refused cap writes only the count
        out = [np.full(4, -7, np.int32) for _ in range(4)]
        pc = np.full((4, 2), -7.0)
        cnt = C.c_int32(-1)
        keys = np.ascontiguousarray(scan["keys"], np.int32)
        rc = ctx.lib.esikf_vmap_retrieve(ctx.h, len(keys), keys.ctypes.data, *g, 1, 4, C.byref(cnt), out[0].ctypes.data, out[1].ctypes.data, pc.ctypes.data,
                                         out[2].ctypes.data, out[3].ctypes.data)
        assert rc == -3 and cnt.value == len(base["cell"]) and all((o == -7).all() for o in out) and (pc == -7.0).all()
        assert np.array_equal(ctx.vmap_download(np.arange(n, dtype=np.int32))["ref"], refs0)  # normal_en refused: no ref stored
        again = ctx.vmap_retrieve(scan["keys"], *g, False)
        for f in base:
            assert np.asarray(again[f]).tobytes() == np.asarray(base[f]).tobytes(), f
        ctx.vmap_place_points([n // 2], edge)
    finally:
        ctx.close()


def _place_ticks(ctx, tks):
    sc0 = tks[0]["sc"]
    ctx.set_extrinsics(sc0["ext"])
    ctx.vio_set_camera(sc0["cam"], RC.VIO_CFG)
    ctx.vmap_init(1)


@pytest.mark.parametrize("normal_en", [True, False])
def test_ticks_match_the_pinned_restatement(gpu_ctx, normal_en):
    """The ticks the CPU test pins to the reference source (tests/test_oracle_vmap_retrieve.py): a growing visual map placed
    in shuffled order, negative coordinates and keys the float narrowing moves, three scans; per tick every cell's point, pc,
    status and ref equal the restatement, and the refs stored with normal_en equal its store."""
    tks = VR.ticks()
    want, _ = VR.restate_ticks(tks, normal_en)
    _place_ticks(gpu_ctx, tks)
    for t, tk in enumerate(tks):
        ids = gpu_ctx.vmap_add_points(tk["first"], np.zeros((len(tk["patch"]), 2)), tk["patch"], tk["T"], tk["fid"], np.zeros(len(tk["patch"]), np.float32),
                                      np.zeros(len(tk["patch"]), np.float32), np.full(len(tk["ids"]), -1, np.int32))
        assert np.array_equal(ids, tk["ids"])
        idx = tk["order"] - tk["ids"][0]
        gpu_ctx.vmap_place_points(tk["order"], tk["pos"][idx], tk["ninit"][idx])
        sc = tk["sc"]
        gpu_ctx.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"])
        w = want[t]
        got = gpu_ctx.vmap_retrieve(w["walk"], *_grid(sc), normal_en)
        _equal(got, w["cells"], f"tick {t}")
        assert np.array_equal(got["ref"], w["ref_all"]), t
        assert np.array_equal(got["status"] == VR.NO_REF, (w["cells"]["status"] == VR.KEPT) & (w["ref_all"] < 0)), t
        assert (got["status"] == VR.KEPT).sum() > 50


def test_cell_without_a_winner(gpu_ctx):
    """A TYPE_MAP cell whose only point lies beyond 10000 m: the cell comes back with point id -1 and status "no winner"; a
    point at 9000 m in another cell wins its cell."""
    pos = np.array([[0.0, 0.0, 20000.0], [3000.0, 3000.0, 9000.0]])
    sc = _edge_ctx(gpu_ctx, pos)
    gpu_ctx.vmap_place_points([0, 1], pos)
    got = gpu_ctx.vmap_retrieve(VR.insertion_keys(pos).astype(np.int32), *_grid(sc), True)
    assert len(got["cell"]) == 2
    far = got["point_id"] == -1
    assert far.sum() == 1 and got["status"][far][0] == VR.NO_WINNER and got["ref"][far][0] == -1 and (got["pc"][far] == 0).all()
    assert got["point_id"][~far][0] == 1 and got["status"][~far][0] == VR.KEPT


def _near_integer(pc):
    return bool((np.abs(pc - np.round(pc)) < 1e-9).any())


def test_fisheye_matches_the_oracle_off_the_edges(gpu_ctx):
    """Config 3's fisheye: the projection calls atan, where CUDA's and glibc's may differ in the last ulp. pc agrees to 1e-9
    px; a cell, winner or status may differ only where a pc (the oracle's or the device's) lies within 1e-9 px of an integer
    (a cell, border or pixel edge). The differing cells are counted and printed."""
    sc = RC.scene("fisheye", 100_000, seed=8, n_vis=6000)
    n = len(sc["pos"])
    rng = np.random.default_rng(4)
    order = rng.permutation(n).astype(np.int32)
    ninit = np.ones(n, np.uint8)
    _store(gpu_ctx, sc["n_obs"], seed=5)
    gpu_ctx.set_extrinsics(sc["ext"])
    gpu_ctx.vio_set_camera(sc["cam"], RC.VIO_CFG)
    gpu_ctx.vmap_place_points(order, sc["pos"][order])
    dev = gpu_ctx.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"], depth=True)
    orc = RC.OracleRetrieve(sc)
    s = orc.scan(sc)
    # the oracle's depth check on the device's depth image, whose fisheye pixels may differ (tests/test_gpu_retrieve_scan.py)
    walk, want = VR.composed(orc, sc, VR.placed_visual_map(sc["pos"], sc["n_obs"], order), s["keys"], dev["depth"], ninit)
    got = gpu_ctx.vmap_retrieve(walk, *_grid(sc), True)
    gs = np.where(got["status"] == VR.NO_REF, VR.KEPT, got["status"])
    g = {int(c): (int(p), tuple(pc), int(st)) for c, p, pc, st in zip(got["cell"], got["point_id"], got["pc"], gs)}
    w = {int(c): (int(p), tuple(pc), int(st)) for c, p, pc, st in zip(want["cell"], want["point_id"], want["pc"], want["status"])}
    differ = 0
    for c in set(g) | set(w):
        a, b = g.get(c), w.get(c)
        if a is not None and b is not None and a[0] == b[0] and a[2] == b[2] and np.allclose(a[1], b[1], rtol=0, atol=1e-9):
            continue
        differ += 1
        assert any(x is not None and _near_integer(np.array(x[1])) for x in (a, b)), (c, a, b)
    print(f"fisheye: {differ} of {len(w)} cells differ from the host's")
    assert len(w) > 100
