"""GPU: the new visual map points of a VIO tick (esikf_vio_generate_points, generateVisualMapPoints on the device) against the
oracle's restatement (oracle/orc_generate.cpp, pinned to the reference source by tests/test_oracle_generate.py).

Pinhole cameras (config 2's, and a distorted one): the winners, their order, pos, pc, score, signed normal, var and patch are the
oracle's bit for bit. Fisheye (config 3's camera and extrinsics): the projection calls atan, where CUDA's and glibc's may differ
in the last ulp, so pc may differ by an ulp and the patch by its bilinear weights there; every other output is compared
exactly (the count of such points is printed)."""
import ctypes as C

import numpy as np
import pytest

import color_cases as CC
import generate_cases as GC
import oracle_bind as O
import select_cases as SC
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S

pytestmark = pytest.mark.gpu
GEOM = ("grid_size", "grid_n_width", "grid_n_height", "border")


def _setup(ctx, sc):
    ctx.set_extrinsics(sc["ext"])
    ctx.vio_set_camera(sc["cam"], S.VioCfg())
    ctx.vio_set_image(sc["img"])


def _host(ctx, sc, pg=None, state="scene"):
    pg = (sc["point_w"], sc["normal"], sc["var"]) if pg is None else pg
    return ctx.vio_generate_points(sc["mask"], *[sc[k] for k in GEOM], pg=pg, add_from=(sc["add_pos"], sc["add_normal"]),
                                   state=sc["state"] if state == "scene" else state)


def _compare(got, want, fisheye=False, label="", skip=()):
    assert len(got["cell"]) == len(want["cell"]), (label, len(got["cell"]), len(want["cell"]))
    for k in GC.FIELDS:
        if k in skip or (fisheye and k in ("pc", "patch")):
            continue
        assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(want[k]).tobytes(), (label, k)
    if fisheye:
        off = np.any(got["pc"] != want["pc"], axis=1)
        assert np.abs(got["pc"] - want["pc"]).max(initial=0) <= 1e-9 * np.abs(want["pc"]).max(initial=1), label
        assert np.abs(got["patch"] - want["patch"]).max(initial=0) <= 1e-3, label
        assert np.array_equal(got["patch"][~off], want["patch"][~off]), label
        print(f"{label}: {int(off.sum())} of {len(got['cell'])} new points have pc 1 ulp apart")


@pytest.mark.parametrize("case", ["pinhole-100k", "pinhole-300k", "radtan-50k", "fisheye-100k"])
def test_scans_from_the_host_match_the_oracle(gpu_ctx, case):
    camera, size = case.split("-")
    n = int(size[:-1]) * 1000
    sc = GC.scene(camera, n, seed=n // 1000)
    _setup(gpu_ctx, sc)
    got = _host(gpu_ctx, sc)
    want = GC.OracleGenerate(sc).run(sc)
    assert len(want["cell"]) > 150
    _compare(got, want, fisheye=(camera == "fisheye"), label=case)


@pytest.mark.parametrize("name", ["edge80", "edge0", "pinhole_n10", "pinhole_n11"])
def test_hand_built_and_cut_scans_match_the_oracle(gpu_ctx, name):
    sc = GC.pin_scenes()[name]
    _setup(gpu_ctx, sc)
    got = _host(gpu_ctx, sc)
    want = GC.OracleGenerate(sc).run(sc)
    _compare(got, want, label=name)
    if name.startswith("edge"):
        won = dict(zip(got["cell"].tolist(), got["source"].tolist()))
        assert all(won.get(c) == s for c, s in sc["expect"].items())
    assert (len(got["cell"]) == 0) == (name == "pinhole_n10")


# ----------------------------------------------------------------------------------------------------- the chained tick
def _tick(ctx, fr, c, o_state, gen, mask, add):
    """A LIO tick on the device-resident map (its update with the oracle's posterior, so both hold the same pv list), the
    coloured scan's cloud, and a VIO tick on a selected sub-map; with `gen`, esikf_vio_generate_points on the resident scan
    right after the VIO update. Returns every output of the ticks."""
    cfg = fr["lio_cfg"]
    ctx.set_extrinsics(fr["ext"])
    ctx.map_device_init(cfg, root_capacity=1 << 16, grow=True)
    ctx.lio_set_scan(fr["pts"])
    ctx.map_device_build(fr["state_prior"])
    out = {"lio": ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], cfg)}
    ctx.map_device_update(o_state)
    ctx.rgb_set_cloud(None, o_state)
    ctx.vio_set_camera(c["camcfg"], S.VioCfg())
    ctx.vio_set_image(c["img"])
    ctx.vio_set_ref_images(c["ref_imgs"])
    sel = ctx.vio_select_patches(c["ref_idx"], c["px_ref"], c["pos_w"], c["T_ref"], c["ref_inv_expo"], c["pc"], c["T_cur"], c["inv_expo"], normal_w=c["normal_w"])
    out["kept"] = sel["kept"]
    ctx.vio_run(out["lio"]["state"], out["lio"]["state"])
    g = GC.grid_geometry(c["camcfg"].width, c["camcfg"].height, levels=2)
    if gen:
        out["gen"] = ctx.vio_generate_points(mask, *[g[k] for k in GEOM], add_from=add)
    out["vio"] = ctx.vio_fetch()
    out["rgb"] = ctx.rgb_colorize(CC.bgr_image(c["camcfg"], 3), 0.05)
    out["stats"] = ctx.map_device_stats()
    out["map"] = ctx.map_device_download()
    out["normals"] = ctx.lio_fetch_normals()
    if gen:
        out["gen_explicit"] = ctx.vio_generate_points(mask, *[g[k] for k in GEOM], add_from=add, state=out["vio"]["state"])
    return out


def test_chained_tick_on_the_resident_scan(small_vio_frame):
    """lio_update -> map_device_update -> vio_select_patches + vio_run -> vio_generate_points(pg = NULL, state = NULL) against
    the oracle on the pv list of the same update; NULL state against the explicit one; the resident scan against the same
    points from the host; and the LIO / VIO outputs, coloured scan, map stats, map download and pv normals byte-identical to
    the same ticks without the call."""
    fr = small_vio_frame
    c = SC.candidates("radtan", 300, seed=1)
    orc = O.OracleLIO(fr["lio_cfg"], fr["ext"])
    orc.tick_build_map(fr["pts"], fr["state_prior"])
    o = orc.state_estimation(fr["pts"], fr["state_prior"], fr["state_prior"])
    pw, var = orc.tick_update_map(want_lists=True)
    g = GC.grid_geometry(c["camcfg"].width, c["camcfg"].height, levels=2)  # border 20
    rng = np.random.default_rng(5)
    mask = (rng.random(g["grid_n_width"] * g["grid_n_height"]) < 0.15).astype(np.uint8)
    add = (pw[::37] + rng.normal(0, 0.02, (len(pw[::37]), 3)), rng.normal(size=(len(pw[::37]), 3)))
    ctx_a, ctx_b = api.Context(0), api.Context(0)
    try:
        a = _tick(ctx_a, fr, c, o["state"], True, mask, add)
        b = _tick(ctx_b, fr, c, o["state"], False, mask, add)
        # the same points from the host; var plays no part in the choice: the winners' rows carry the device's own var
        hvar = var.reshape(-1, 3, 3).copy()
        win = a["gen"]["source"][a["gen"]["source"] < GC.ADD_FROM]
        hvar[win] = a["gen"]["var"][a["gen"]["source"] < GC.ADD_FROM]
        sc = dict(g, cam=c["camcfg"], ext=fr["ext"], img=c["img"], state=a["vio"]["state"],
                  point_w=pw, normal=a["normals"], var=hvar, add_pos=add[0], add_normal=add[1], mask=mask)
        host = _host(ctx_a, sc)
    finally:
        ctx_a.close(), ctx_b.close()
    gen = a["gen"]
    assert len(gen["cell"]) > 5
    _compare(gen, host, label="resident vs host")
    _compare(a["gen_explicit"], gen, label="explicit state")
    want = GC.OracleGenerate(sc).run(dict(sc, var=var.reshape(-1, 3, 3)))
    _compare(gen, want, label="chained", skip=("var",))
    # var: the device's recomputation of LIVMapper.cpp:420-421 against the oracle's (the body covariance may differ by an ulp)
    assert np.allclose(gen["var"], want["var"], rtol=1e-11, atol=1e-20)
    for k in ("state", "dis_to_plane", "M", "HTH", "HTz", "solution"):
        assert np.ascontiguousarray(a["lio"][k]).tobytes() == np.ascontiguousarray(b["lio"][k]).tobytes(), k
    for k in ("state", "errors", "HTH", "HTz", "solution", "iters_per_level"):
        assert np.ascontiguousarray(a["vio"][k]).tobytes() == np.ascontiguousarray(b["vio"][k]).tobytes(), k
    for k in ("xyz", "bgr", "index"):
        assert a["rgb"][k].tobytes() == b["rgb"][k].tobytes(), k
    assert np.array_equal(a["kept"], b["kept"]) and a["stats"] == b["stats"] and a["normals"].tobytes() == b["normals"].tobytes()
    keys = a["map"]["keys"][np.lexsort(a["map"]["keys"].T[::-1])]
    ma, mb = O.flat_map_subset(a["map"], keys), O.flat_map_subset(b["map"], keys)
    assert len(b["map"]["keys"]) == len(keys)
    for k in ("keys", "count", "planes"):
        assert ma[k].tobytes() == mb[k].tobytes(), k


# ----------------------------------------------------------------------------------------------------- errors
def _status(fn):
    with pytest.raises(api.EsikfError) as e:
        fn()
    return int(str(e.value).split(":")[0].split()[1])


def test_call_order_mask_length_and_capacity_errors():
    sc = GC.scene("pinhole", 5000, seed=2)
    geo = [sc[k] for k in GEOM]
    pg = (sc["point_w"], sc["normal"], sc["var"])
    ctx = api.Context(0)
    try:
        ctx.set_extrinsics(sc["ext"])
        assert _status(lambda: ctx.vio_generate_points(sc["mask"], *geo, pg=pg, state=sc["state"])) == -4  # no camera
        ctx.vio_set_camera(sc["cam"], S.VioCfg())
        assert _status(lambda: ctx.vio_generate_points(sc["mask"], *geo, pg=pg, state=sc["state"])) == -4  # no image
        ctx.vio_set_image(sc["img"])
        assert _status(lambda: ctx.vio_generate_points(sc["mask"], *geo, pg=pg)) == -4                      # no VIO posterior
        assert _status(lambda: ctx.vio_generate_points(sc["mask"], *geo, state=sc["state"])) == -4          # no resident pv list
        assert _status(lambda: ctx.vio_generate_points(sc["mask"][:-1], *geo, pg=pg, state=sc["state"])) == -3  # mask length
        assert _status(lambda: ctx.vio_generate_points(sc["mask"], 0, *geo[1:], pg=pg, state=sc["state"])) == -3  # grid size
        full = ctx.vio_generate_points(sc["mask"], *geo, pg=pg, state=sc["state"])
        k = len(full["cell"])
        assert k > 10
        # cap too small: only *n_out is written
        src = np.full(k, -5, np.int32)
        pos = np.full((k, 3), 7.0)
        n = C.c_int32(-1)
        pw, nv, var, st = [np.ascontiguousarray(x, np.float64) for x in (sc["point_w"], sc["normal"], sc["var"], sc["state"])]
        mask = np.ascontiguousarray(sc["mask"], np.uint8)
        call = lambda cap, n_out: ctx.lib.esikf_vio_generate_points(ctx.h, pw.ctypes.data, nv.ctypes.data, var.ctypes.data, len(pw), None, None, 0,  # noqa: E731
                                                                      mask.ctypes.data, len(mask), *geo, st.ctypes.data, cap, n_out, src.ctypes.data, None,
                                                                      pos.ctypes.data, None, None, None, None, None)
        assert call(k - 1, C.byref(n)) == -3 and n.value == k
        assert (src == -5).all() and (pos == 7.0).all()
        assert call(k, None) == -3  # missing n_out
        assert call(k, C.byref(n)) == 0 and n.value == k and pos.tobytes() == full["pos"].tobytes() and src.tobytes() == full["source"].tobytes()
        # after the device map is rewritten by a host tick, the resident pv list is gone
        cfg = S.LioCfg()
        ctx.map_device_init(cfg, root_capacity=1 << 12)
        ctx.map_device_update_points(sc["point_w"][:100], sc["var"][:100].reshape(-1, 9))
        ctx.vio_set_patches(np.zeros((0, 3)), np.zeros((0, 256), np.float32), np.zeros(0, np.int32), np.zeros(0))
        ctx.vio_run(sc["state"], sc["state"])
        assert _status(lambda: ctx.vio_generate_points(sc["mask"], *geo)) == -4
        nul = ctx.vio_generate_points(sc["mask"], *geo, pg=pg)  # the VIO posterior (here the state the empty update kept)
        assert nul["pos"].tobytes() == full["pos"].tobytes()
    finally:
        ctx.close()
