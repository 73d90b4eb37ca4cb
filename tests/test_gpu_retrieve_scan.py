"""GPU: the scan side of the visual sub-map retrieval (esikf_vio_retrieve_scan / esikf_vio_depth_check) against the oracle's
restatement (oracle/orc_retrieve.cpp, pinned to the reference source's own retrieveFromVisualSparseMap by
tests/test_oracle_retrieve.py).

Keys and their order are always the oracle's. Pinhole cameras (config 2's, and a distorted one): the depth image and the
depth-check flags are the oracle's bit for bit. Fisheye (config 3's camera and extrinsics): the projection calls atan, where
CUDA's and glibc's may differ in the last ulp, so a point whose int(px) straddles an integer can land one pixel over; the
differing pixels are counted and printed, and each must come from such a point."""
import ctypes as C

import numpy as np
import pytest

import oracle_bind as O
import retrieve_cases as RC
import shim_bind as SB
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _setup(ctx, sc):
    ctx.set_extrinsics(sc["ext"])
    ctx.vio_set_camera(sc["cam"], RC.VIO_CFG)


def _walk_inputs(orc, sc, keys, state=None):
    """The host's map-side walk on the given keys: the retrieved points in cell order and their pc."""
    w = orc.walk(sc, keys, state=state)
    cells = np.nonzero(w["grid_type"])[0]
    return w, sc["pos"][w["cell_pt"][cells]], w["cell_pc"][cells]


def _straddlers(sc, state):
    """Pixels a fisheye projection one ulp off could move a point to: those of scan points with pt_c[2] > 0 whose u or v lies
    within 1e-9 px of an integer (host projection)."""
    cam = sc["cam"]
    Rcw, Pcw = S.camera_pose(sc["ext"], S.unpack_state(state)["R"], S.unpack_state(state)["p"])
    pf = sc["pg"] @ Rcw.T + Pcw
    ok = pf[:, 2] > 0
    x, y = pf[ok, 0] / pf[ok, 2], pf[ok, 1] / pf[ok, 2]
    r = np.hypot(x, y)
    th = np.arctan(r)
    d = cam.d
    thd = th * (1 + d[0] * th ** 2 + d[1] * th ** 4 + d[2] * th ** 6 + d[3] * th ** 8)
    s = np.where(r > 1e-8, thd / np.maximum(r, 1e-300), 1.0)
    u, v = cam.fx * x * s + cam.cx, cam.fy * y * s + cam.cy
    near = (np.abs(u - np.round(u)) < 1e-9) | (np.abs(v - np.round(v)) < 1e-9)
    out = set()
    for uu, vv in zip(u[near], v[near]):
        for a in (np.floor(uu - 1e-9), np.floor(uu + 1e-9)):
            for b in (np.floor(vv - 1e-9), np.floor(vv + 1e-9)):
                out.add((int(b), int(a)))
    return out


def _compare_depth(got, want, sc, label):
    if sc["cam"].model == 0:
        assert got.tobytes() == want.tobytes(), label
        return 0
    diff = np.argwhere(got != want)
    print(f"{label}: {len(diff)} of {int((want != 0).sum())} written pixels differ from the host's")
    allowed = _straddlers(sc, sc["state"])
    for b, a in diff.tolist():  # a pixel that differs is one a straddling point wrote or left on one side
        assert any((b + db, a + da) in allowed for db in (-1, 0, 1) for da in (-1, 0, 1)), (label, b, a)
    return len(diff)


@pytest.mark.parametrize("camera", ["pinhole", "radtan", "fisheye"])
@pytest.mark.parametrize("n", [100_000, 300_000])
def test_host_scans_match_the_oracle(gpu_ctx, camera, n):
    sc = RC.scene(camera, n, seed=n // 1000 + 1, n_vis=6000)
    _setup(gpu_ctx, sc)
    got = gpu_ctx.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"], depth=True)
    orc = RC.OracleRetrieve(sc)
    want = orc.scan(sc)
    assert len(want["keys"]) > 1000
    assert np.array_equal(got["keys"].astype(np.int64), want["keys"]), camera
    ndiff = _compare_depth(got["depth"], want["depth"], sc, f"{camera}-{n}")
    _, pos, pc = _walk_inputs(orc, sc, want["keys"])
    flags = gpu_ctx.vio_depth_check(pos, pc)
    wflags = orc.depth_check(sc, got["depth"], pos, pc)  # the oracle's check on the device's image: exact on every camera
    assert 0 < flags.sum() < len(flags)
    assert flags.tobytes() == wflags.tobytes(), camera
    if ndiff == 0:
        assert flags.tobytes() == orc.depth_check(sc, want["depth"], pos, pc).tobytes()


def test_hand_built_points_match_the_oracle(gpu_ctx):
    """Key boundaries, pt_c[2] at 0, the border, pixel overwrites, |delta| at 0.5, centre-only and empty taps, a map_dist tie."""
    sc = RC.edge_scene()
    _setup(gpu_ctx, sc)
    got = gpu_ctx.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"], depth=True)
    orc = RC.OracleRetrieve(sc)
    want = orc.retrieve(sc)
    assert np.array_equal(got["keys"].astype(np.int64), want["keys"])
    assert got["depth"].tobytes() == want["depth"].tobytes()
    pos = sc["pos"][want["cell_pt"][want["cells"]]]
    flags = gpu_ctx.vio_depth_check(pos, want["cell_pc"][want["cells"]])
    assert flags.tobytes() == want["flag"].tobytes()
    assert 0 < flags.sum() < len(flags)


def _tick(ctx, fr, sc, post, retrieve):
    cfg = fr["lio_cfg"]
    ctx.set_extrinsics(fr["ext"])
    ctx.map_device_init(cfg, root_capacity=1 << 16, grow=True)
    ctx.lio_set_scan(fr["pts"])
    ctx.map_device_build(fr["state_prior"])
    out = {"lio": ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], cfg)}
    ctx.map_device_update(post)
    ctx.vio_set_camera(sc["cam"], RC.VIO_CFG)
    if retrieve:
        out["resident"] = ctx.vio_retrieve_scan(sc["border"], state=None, depth=True)   # the LIO posterior on the device
        out["explicit"] = ctx.vio_retrieve_scan(sc["border"], state=out["lio"]["state"], depth=True)
    out["stats"] = ctx.map_device_stats()
    out["map"] = ctx.map_device_download()
    out["normals"] = ctx.lio_fetch_normals()
    return out


def test_chained_tick_on_the_resident_scan(small_vio_frame):
    """lio_update -> map_device_update -> vio_retrieve_scan(pg = NULL) -> the host's walk -> vio_depth_check against the oracle's
    whole retrieval on the pv list of the same update; state = NULL against the explicit LIO posterior; the resident scan
    against the same points from the host; and the LIO outputs, map stats, map download and pv normals byte-identical to the
    same tick without the calls."""
    fr = small_vio_frame
    orc_lio = O.OracleLIO(fr["lio_cfg"], fr["ext"])
    orc_lio.tick_build_map(fr["pts"], fr["state_prior"])
    o = orc_lio.state_estimation(fr["pts"], fr["state_prior"], fr["state_prior"])
    pw, _ = orc_lio.tick_update_map(want_lists=True)
    # a visual map on the scan points in front of the LIO posterior's camera (the host scans above cover the discontinuities)
    post = S.unpack_state(o["state"])
    cam, ext = RC.CAMERAS["pinhole"][0], fr["ext"]
    Rcw, Pcw = S.camera_pose(ext, post["R"], post["p"])
    rng = np.random.default_rng(3)
    front = pw @ Rcw.T + Pcw
    front = front[front[:, 2] > 2.0]
    q = front[rng.choice(len(front), min(600, len(front)), replace=False)]
    vis = RC.flat_visual_map((q - Pcw) @ Rcw, (-q / np.linalg.norm(q, axis=1, keepdims=True)) @ Rcw, np.ones(len(q), np.int32))
    sc = dict(cam=cam, ext=ext, state=o["state"], pg=pw, **RC.grid(cam), **vis)
    ctx_a, ctx_b = api.Context(0), api.Context(0)
    try:
        a = _tick(ctx_a, fr, sc, o["state"], True)
        b = _tick(ctx_b, fr, sc, o["state"], False)
        host = ctx_a.vio_retrieve_scan(sc["border"], pg=pw, state=a["lio"]["state"], depth=True)
        orc = RC.OracleRetrieve(sc)
        want = orc.retrieve(dict(sc, state=a["lio"]["state"]))
        _, pos, pc = _walk_inputs(orc, dict(sc, state=a["lio"]["state"]), a["resident"]["keys"])
        flags = ctx_a.vio_depth_check(pos, pc)
    finally:
        ctx_a.close(), ctx_b.close()
    for k in ("keys", "depth"):
        assert a["resident"][k].tobytes() == a["explicit"][k].tobytes() == host[k].tobytes(), k
    assert np.array_equal(a["resident"]["keys"].astype(np.int64), want["keys"])
    assert a["resident"]["depth"].tobytes() == want["depth"].tobytes()
    assert len(pos) > 10 and flags.tobytes() == want["flag"].tobytes()
    survivors = want["cell_pt"][want["cells"]][flags == 0]
    assert np.array_equal(survivors, want["survivors"]) and len(survivors) > 0
    for k in ("state", "dis_to_plane", "M", "HTH", "HTz", "solution"):
        assert np.ascontiguousarray(a["lio"][k]).tobytes() == np.ascontiguousarray(b["lio"][k]).tobytes(), k
    assert a["stats"] == b["stats"] and a["normals"].tobytes() == b["normals"].tobytes()
    keys = a["map"]["keys"][np.lexsort(a["map"]["keys"].T[::-1])]
    ma, mb = O.flat_map_subset(a["map"], keys), O.flat_map_subset(b["map"], keys)
    assert len(b["map"]["keys"]) == len(keys)
    for k in ("keys", "count", "planes"):
        assert ma[k].tobytes() == mb[k].tobytes(), k


def test_retrieval_leaves_the_vio_update_unchanged(gpu_ctx):
    """vio_retrieve_scan + vio_depth_check between vio_set_patches and vio_run leave the VIO posterior byte-identical."""
    sc = RC.scene("pinhole", 20000, seed=9)
    n = 300
    rng = np.random.default_rng(1)
    pos = sc["pg"][rng.choice(len(sc["pg"]), n, replace=False)]
    wp = rng.uniform(0, 255, (n, 64)).astype(np.float32)
    outs = []
    for retrieve in (True, False):
        _setup(gpu_ctx, sc)
        gpu_ctx.vio_set_image(sc["img"])
        gpu_ctx.vio_set_patches(pos, wp, np.zeros(n, np.int32), np.ones(n))
        if retrieve:
            gpu_ctx.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"])
            gpu_ctx.vio_depth_check(pos[:50], np.full((50, 2), 100.0))
        gpu_ctx.vio_run(sc["state"], sc["state"])
        outs.append(gpu_ctx.vio_fetch())
    for k in ("state", "errors", "HTH", "HTz", "solution", "iters_per_level"):
        assert np.ascontiguousarray(outs[0][k]).tobytes() == np.ascontiguousarray(outs[1][k]).tobytes(), k


# ----------------------------------------------------------------------------------------------------- errors
def _status(fn):
    with pytest.raises(api.EsikfError) as e:
        fn()
    return int(str(e.value).split(":")[0].split()[1])


def test_errors():
    sc = RC.scene("pinhole", 5000, seed=4)
    pg, st = np.ascontiguousarray(sc["pg"]), np.ascontiguousarray(sc["state"])
    ctx = api.Context(0)
    try:
        ctx.set_extrinsics(sc["ext"])
        ctx.cam_size = (sc["cam"].width, sc["cam"].height)
        assert _status(lambda: ctx.vio_retrieve_scan(sc["border"], pg=pg, state=st)) == -4  # no camera
        _setup(ctx, sc)
        assert _status(lambda: ctx.vio_depth_check(sc["pos"][:3], np.full((3, 2), 50.0))) == -4  # before retrieve_scan
        assert _status(lambda: ctx.vio_retrieve_scan(sc["border"], state=st)) == -4  # no resident pv list
        assert _status(lambda: ctx.vio_retrieve_scan(sc["border"], pg=pg)) == -4  # no LIO posterior on the device
        full = ctx.vio_retrieve_scan(sc["border"], pg=pg, state=st)
        k = len(full["keys"])
        assert 100 < k < len(pg)
        # cap too small: only the count
        keys = np.full((k, 3), -7, np.int32)
        cnt = C.c_int32(-1)
        call = lambda cap, n_out, border=sc["border"], p=pg: ctx.lib.esikf_vio_retrieve_scan(ctx.h, p.ctypes.data, len(p), border, st.ctypes.data, cap,  # noqa: E731
                                                                                             n_out, keys.ctypes.data, None)
        assert call(k - 1, C.byref(cnt)) == -3 and cnt.value == k and (keys == -7).all()
        assert call(k, C.byref(cnt)) == 0 and cnt.value == k and np.array_equal(keys, full["keys"])
        # bad arguments write nothing
        cnt.value = -1
        assert call(k, None) == -3 and call(-1, C.byref(cnt)) == -3 and call(k, C.byref(cnt), border=-1) == -3 and cnt.value == -1
        assert ctx.lib.esikf_vio_retrieve_scan(ctx.h, pg.ctypes.data, len(pg), sc["border"], st.ctypes.data, 5, C.byref(cnt), None, None) == -3
        assert ctx.lib.esikf_vio_depth_check(ctx.h, 3, None, None, None) == -3 and ctx.lib.esikf_vio_depth_check(ctx.h, -1, None, None, None) == -3
        # a key out of range: the call fails, and leaves no depth image behind it
        far = pg.copy()
        far[17, 1] = -(2.0 ** 19) + 0.25  # floor(-2^20 + 0.5) = -2^20, one less: -2^20 - 1
        assert call(len(pg), C.byref(cnt), p=far) == -3
        assert _status(lambda: ctx.vio_depth_check(sc["pos"][:3], np.full((3, 2), 50.0))) == -4
        edge = pg.copy()
        edge[17, 1] = -(2.0 ** 19) + 0.75  # floor(-2^20 + 1.5) = -2^20 + 1, one less: -2^20, still in range
        assert call(len(pg), C.byref(cnt), p=edge) == 0
        # state = NULL after a VIO run: the device holds the VIO posterior
        ctx.vio_set_image(sc["img"])
        ctx.vio_set_patches(pg[:10], np.zeros((10, 64), np.float32), np.zeros(10, np.int32), np.ones(10))
        ctx.vio_run(st, st)
        assert _status(lambda: ctx.vio_retrieve_scan(sc["border"], pg=pg)) == -4
        # vio_set_camera forgets the depth image
        ctx.vio_retrieve_scan(sc["border"], pg=pg, state=st)
        assert len(ctx.vio_depth_check(sc["pos"][:3], np.full((3, 2), 50.0))) == 3
        _setup(ctx, sc)
        assert _status(lambda: ctx.vio_depth_check(sc["pos"][:3], np.full((3, 2), 50.0))) == -4
    finally:
        ctx.close()


def test_shim_gives_the_c_abi_results(gpu_ctx):
    """VIOManager::RetrieveScanVoxels / CheckDepthContinuity (fl2_shim) against the C ABI on the same scan and points."""
    api.load_library()
    shim = SB.load()
    sc = RC.scene("radtan", 50_000, seed=12)
    _setup(gpu_ctx, sc)
    want = gpu_ctx.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"])
    orc = RC.OracleRetrieve(sc)
    _, pos, pc = _walk_inputs(orc, sc, want["keys"])
    wflags = gpu_ctx.vio_depth_check(pos, pc)
    cam, ext = sc["cam"], sc["ext"]
    c = api.CameraC(cam.model, cam.width, cam.height, 0, cam.fx, cam.fy, cam.cx, cam.cy)
    c.d[:] = list(cam.d)
    v = api.VioCfgC(RC.VIO_CFG.img_point_cov, RC.VIO_CFG.levels, RC.VIO_CFG.max_iterations, 1, 0)
    e = api.ExtrinsicsC()
    for f in ("extR", "extT", "Rcl", "Pcl"):
        getattr(e, f)[:] = list(np.ascontiguousarray(getattr(ext, f), np.float64).reshape(-1))
    pg, st, pos, pc = [np.ascontiguousarray(x, np.float64) for x in (sc["pg"], sc["state"], pos, pc)]
    keys = np.zeros((len(pg), 3), np.int64)
    flags = np.zeros(len(pos), np.uint8)
    nk = C.c_int32(0)
    rc = shim.fl2_shim_retrieve_run(C.byref(c), C.byref(v), C.byref(e), st.ctypes.data_as(C.c_void_p), pg.ctypes.data_as(C.c_void_p), len(pg), sc["border"],
                                    pos.ctypes.data_as(C.c_void_p), pc.ctypes.data_as(C.c_void_p), len(pos), C.byref(nk), keys.ctypes.data_as(C.c_void_p),
                                    flags.ctypes.data_as(C.c_void_p))
    assert rc == 0
    assert np.array_equal(keys[:nk.value], want["keys"].astype(np.int64))
    assert flags.tobytes() == wflags.tobytes()
