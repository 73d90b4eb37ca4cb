"""GPU: the new observations of the visual sub-map in a VIO tick (esikf_vio_update_points, updateVisualMapPoints on the
device) against the oracle's restatement (oracle/orc_observe.cpp, pinned to the reference source by
tests/test_oracle_observe.py).

Pinhole cameras (config 2's, and a distorted one): the flags, the added entries, pc and the patches are the oracle's bit for
bit. Fisheye (config 3's camera and extrinsics): the projection calls atan, where CUDA's and glibc's may differ in the last
ulp, so pc may differ by an ulp and the patch by its bilinear weights there; the flags and entries are compared exactly (the
count of such entries is printed)."""
import ctypes as C

import numpy as np
import pytest

import generate_cases as GC
import observe_cases as OC
import oracle_bind as O
import select_cases as SC
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S

pytestmark = pytest.mark.gpu
SUB = ("pos", "converged", "last_T", "last_px")


def _install(ctx, sc):
    """The scene's sub-map through esikf_vio_set_patches (zero warp patches, unit exposure)."""
    n = len(sc["pos"])
    ctx.set_extrinsics(sc["ext"])
    ctx.vio_set_camera(sc["cam"], S.VioCfg())
    ctx.vio_set_image(sc["img"])
    ctx.vio_set_patches(np.ascontiguousarray(sc["pos"]), np.zeros((n, 4 * 64), np.float32), np.ascontiguousarray(sc["search_levels"]), np.ones(n))


def _update(ctx, sc, state="scene"):
    return ctx.vio_update_points(sc["converged"], sc["last_T"], sc["last_px"], state=sc["state"] if isinstance(state, str) else state)


def _compare(got, want, fisheye=False, label=""):
    assert got["update_flag"].tobytes() == want["update_flag"].tobytes(), label
    assert got["entry"].tobytes() == want["entry"].tobytes(), label
    if not fisheye:
        assert got["pc"].tobytes() == want["pc"].tobytes() and got["patch"].tobytes() == want["patch"].tobytes(), label
        return
    off = np.any(got["pc"] != want["pc"], axis=1)
    assert np.abs(got["pc"] - want["pc"]).max(initial=0) <= 1e-9 * np.abs(want["pc"]).max(initial=1), label
    assert np.abs(got["patch"] - want["patch"]).max(initial=0) <= 1e-3, label
    assert np.array_equal(got["patch"][~off], want["patch"][~off]), label
    print(f"{label}: {int(off.sum())} of {len(got['entry'])} added entries have pc 1 ulp apart")


@pytest.mark.parametrize("camera", ["pinhole", "radtan", "fisheye"])
@pytest.mark.parametrize("n", [2000, 10000])
def test_set_patches_sub_maps_match_the_oracle(gpu_ctx, camera, n):
    sc = OC.scene(camera, n, seed=n // 1000)
    _install(gpu_ctx, sc)
    got = _update(gpu_ctx, sc)
    want = OC.OracleObserve(sc).run(sc)
    assert 0.2 * n < len(want["entry"]) < 0.9 * n
    _compare(got, want, fisheye=(camera == "fisheye"), label=f"{camera}-{n}")


def test_hand_built_entries_match_the_oracle(gpu_ctx):
    """Every boundary of the add rule (delta_p, delta_theta from the acos bound, the trace test, acos's NaN, the pixel
    distance), converged entries, footprints on the image border and observation counts of 29 to 31."""
    sc = OC.edge_scene()
    _install(gpu_ctx, sc)
    got = _update(gpu_ctx, sc)
    _compare(got, OC.OracleObserve(sc).run(sc), label="edge")
    assert np.array_equal(got["update_flag"], sc["expect"])


@pytest.mark.parametrize("camera", ["pinhole", "fisheye"])
def test_resident_posterior_equals_the_explicit_state(gpu_ctx, camera):
    """state = NULL reads the posterior esikf_vio_run left on the device: the same result as that posterior passed from the host,
    and the oracle's on it."""
    sc = OC.scene(camera, 2000, seed=7)
    _install(gpu_ctx, sc)
    # a large image noise keeps the posterior near the prior, so every entry stays inside the image (the reference's
    # getImagePatch reads outside the buffer otherwise)
    gpu_ctx.vio_set_camera(sc["cam"], S.VioCfg(img_point_cov=1e12))
    gpu_ctx.vio_run(sc["state"], sc["state"])
    post = gpu_ctx.vio_fetch()["state"]
    got = _update(gpu_ctx, sc, state=None)
    explicit = _update(gpu_ctx, sc, state=post)
    for k in ("update_flag", "entry", "pc", "patch"):
        assert got[k].tobytes() == explicit[k].tobytes(), k
    _compare(got, OC.OracleObserve(sc).run(dict(sc, state=post)), fisheye=(camera == "fisheye"), label=f"resident {camera}")


def _moved(c, Rcw, Pcw):
    """The candidates with the world moved so that the current frame's pose is (Rcw, Pcw): the pixels stay where they are."""
    R_cur, t_cur = c["T_cur"][:9].reshape(3, 3), c["T_cur"][9:]
    A, b = Rcw.T @ R_cur, Rcw.T @ (t_cur - Pcw)  # pos' = A pos + b
    R_ref = c["T_ref"][:, :9].reshape(-1, 3, 3) @ A.T
    t_ref = c["T_ref"][:, 9:] - np.einsum("nij,j->ni", R_ref, b)
    return dict(c, pos_w=c["pos_w"] @ A.T + b, normal_w=c["normal_w"] @ A.T, T_ref=SC.pack_T(R_ref, t_ref), T_cur=SC.pack_T(Rcw, Pcw)[0])


def _select(ctx, c):
    ctx.vio_set_camera(c["camcfg"], S.VioCfg())
    ctx.vio_set_image(c["img"])
    ctx.vio_set_ref_images(c["ref_imgs"])
    return ctx.vio_select_patches(c["ref_idx"], c["px_ref"], c["pos_w"], c["T_ref"], c["ref_inv_expo"], c["pc"], c["T_cur"], c["inv_expo"],
                                  normal_w=c["normal_w"])["kept"]


@pytest.mark.parametrize("camera", ["pinhole", "radtan", "fisheye"])
def test_select_patches_sub_maps_match_the_oracle(gpu_ctx, camera):
    """The sub-map esikf_vio_select_patches installed (its kept candidates, in candidate order), seen from the frame pose of
    the state."""
    cam, ext = OC.CAMERAS[camera]
    rng = np.random.default_rng(5)
    R, p = S.so3_exp(rng.normal(0, 0.4, 3)), rng.normal(0, 2.0, 3)
    Rcw, Pcw = S.camera_pose(ext, R, p)
    c = _moved(SC.candidates(camera, 2000, seed=3), Rcw, Pcw)
    gpu_ctx.set_extrinsics(ext)
    kept = _select(gpu_ctx, c)
    assert 100 < len(kept) < 2000
    sc = dict(cam=cam, ext=ext, img=c["img"], state=S.pack_state(R, p, 1.02), pos=c["pos_w"][kept], **OC.last_observations(Rcw, Pcw, c["pc"][kept], seed=11))
    got = _update(gpu_ctx, sc)
    want = OC.OracleObserve(sc).run(sc)
    assert 0 < len(want["entry"]) < len(kept)
    _compare(got, want, fisheye=(camera == "fisheye"), label=f"select {camera}")


def test_chained_tick_next_to_the_oracle(small_vio_frame):
    """lio_update -> map_device_update -> vio_select_patches + vio_run -> vio_generate_points -> vio_update_points(state = NULL)
    against the oracle at the VIO posterior; and the LIO / VIO outputs and the new visual map points byte-identical to the
    same tick without the call."""
    fr = small_vio_frame
    orc = O.OracleLIO(fr["lio_cfg"], fr["ext"])
    orc.tick_build_map(fr["pts"], fr["state_prior"])
    o = orc.state_estimation(fr["pts"], fr["state_prior"], fr["state_prior"])
    orc.tick_update_map(want_lists=True)
    post = S.unpack_state(o["state"])
    Rcw, Pcw = S.camera_pose(fr["ext"], post["R"], post["p"])
    c = _moved(SC.candidates("radtan", 300, seed=1), Rcw, Pcw)  # the candidates in view of the LIO posterior's frame
    g = GC.grid_geometry(c["camcfg"].width, c["camcfg"].height, levels=2)
    mask = np.zeros(g["grid_n_width"] * g["grid_n_height"], np.uint8)

    def tick(ctx, observe):
        cfg = fr["lio_cfg"]
        ctx.set_extrinsics(fr["ext"])
        ctx.map_device_init(cfg, root_capacity=1 << 16, grow=True)
        ctx.lio_set_scan(fr["pts"])
        ctx.map_device_build(fr["state_prior"])
        out = {"lio": ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], cfg)}
        ctx.map_device_update(o["state"])
        out["kept"] = _select(ctx, c)
        ctx.vio_run(out["lio"]["state"], out["lio"]["state"])
        out["gen"] = ctx.vio_generate_points(mask, *[g[k] for k in ("grid_size", "grid_n_width", "grid_n_height", "border")])
        out["vio"] = ctx.vio_fetch()
        if observe:
            out["obs_in"] = OC.last_observations(Rcw, Pcw, c["pc"][out["kept"]], seed=12)
            out["obs"] = ctx.vio_update_points(out["obs_in"]["converged"], out["obs_in"]["last_T"], out["obs_in"]["last_px"])
        return out

    ctx_a, ctx_b = api.Context(0), api.Context(0)
    try:
        a, b = tick(ctx_a, True), tick(ctx_b, False)
    finally:
        ctx_a.close(), ctx_b.close()
    assert len(a["kept"]) > 50
    sc = dict(a["obs_in"], cam=c["camcfg"], ext=fr["ext"], img=c["img"], pos=c["pos_w"][a["kept"]], state=a["vio"]["state"])
    want = OC.OracleObserve(sc).run(sc)
    assert len(want["entry"]) > 5
    _compare(a["obs"], want, label="chained")
    for k in ("state", "errors", "HTH", "HTz", "solution", "iters_per_level"):
        assert np.ascontiguousarray(a["vio"][k]).tobytes() == np.ascontiguousarray(b["vio"][k]).tobytes(), k
    for k in GC.FIELDS:
        assert a["gen"][k].tobytes() == b["gen"][k].tobytes(), k
    assert np.array_equal(a["kept"], b["kept"])


# ----------------------------------------------------------------------------------------------------- errors
def _status(fn):
    with pytest.raises(api.EsikfError) as e:
        fn()
    return int(str(e.value).split(":")[0].split()[1])


def test_count_sub_map_and_capacity_errors():
    sc = OC.scene("pinhole", 3000, seed=2)
    n = len(sc["pos"])
    ctx = api.Context(0)
    try:
        ctx.set_extrinsics(sc["ext"])
        ctx.vio_set_camera(sc["cam"], S.VioCfg())
        ctx.vio_set_image(sc["img"])
        assert _status(lambda: _update(ctx, sc)) == -4  # no sub-map installed
        _install(ctx, sc)
        assert _status(lambda: _update(ctx, sc, state=None)) == -4  # no VIO posterior
        cut = {k: v[:-1] for k, v in sc.items() if k in SUB}
        assert _status(lambda: ctx.vio_update_points(cut["converged"], cut["last_T"], cut["last_px"], state=sc["state"])) == -3  # wrong n
        full = _update(ctx, sc)
        k = len(full["entry"])
        assert 10 < k < n
        # cap too small: only *n_out is written; a failed argument check writes nothing
        conv, T, px, st = [np.ascontiguousarray(sc[f], dt) for f, dt in (("converged", np.uint8), ("last_T", np.float64), ("last_px", np.float64), ("state", np.float64))]
        flag = np.full(n, 7, np.uint8)
        entry = np.full(k, -5, np.int32)
        pc = np.full((k, 2), 9.0)
        cnt = C.c_int32(-1)
        call = lambda m, cap, n_out: ctx.lib.esikf_vio_update_points(ctx.h, m, conv.ctypes.data, T.ctypes.data, px.ctypes.data, st.ctypes.data, cap, n_out,  # noqa: E731
                                                                  flag.ctypes.data, entry.ctypes.data, pc.ctypes.data, None)
        assert call(n, k - 1, C.byref(cnt)) == -3 and cnt.value == k
        assert (flag == 7).all() and (entry == -5).all() and (pc == 9.0).all()
        cnt.value = -1
        assert call(n - 1, k, C.byref(cnt)) == -3 and cnt.value == -1
        assert call(n, k, None) == -3
        assert (flag == 7).all() and (entry == -5).all()
        assert call(n, k, C.byref(cnt)) == 0 and cnt.value == k
        assert flag.tobytes() == full["update_flag"].tobytes() and entry.tobytes() == full["entry"].tobytes() and pc.tobytes() == full["pc"].tobytes()
        # an empty installed sub-map: nothing to do
        ctx.vio_set_patches(np.zeros((0, 3)), np.zeros((0, 256), np.float32), np.zeros(0, np.int32), np.zeros(0))
        empty = ctx.vio_update_points(np.zeros(0, np.uint8), np.zeros((0, 12)), np.zeros((0, 2)), state=sc["state"])
        assert len(empty["entry"]) == 0 and len(empty["update_flag"]) == 0
    finally:
        ctx.close()
