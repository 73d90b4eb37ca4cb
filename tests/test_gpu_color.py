"""GPU: the coloured scan (esikf_rgb_set_cloud / esikf_rgb_colorize, publish_frame_world on the device) against the oracle's
restatement (oracle/orc_color.cpp, pinned to the reference source by tests/test_oracle_color.py).

Pinhole cameras (config 2's, and a distorted one): the kept set, its order, xyz and B G R are the oracle's bit for bit.
Fisheye (config 3's camera and extrinsics): the projection calls atan, where CUDA's and glibc's may differ in the last ulp, so
the kept set, its order and xyz are identical and B G R is identical except where the two float pixel positions differ,
where it is within 1 (the count of such points is printed)."""
import ctypes as C

import numpy as np
import pytest

import color_cases as CC
import oracle_bind as O
import select_cases as SC
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _setup(ctx, sc):
    ctx.set_extrinsics(sc["ext"])
    ctx.vio_set_camera(sc["cam"], S.VioCfg())


def _device(ctx, sc, resident=False):
    """The pass on the device: the scene's body points as the resident scan (lio_set_scan) or from the host."""
    _setup(ctx, sc)
    if resident:
        ctx.lio_set_scan(sc["pts"])
        ctx.rgb_set_cloud(None, sc["lio_state"])
    else:
        ctx.rgb_set_cloud(sc["pts"], sc["lio_state"])
    return ctx.rgb_colorize(sc["img"], sc["blind"], state=sc["vio_state"])


def _compare(got, want, fisheye=False, label=""):
    assert np.array_equal(got["index"], want["index"]), (label, len(got["index"]), len(want["index"]))
    assert got["xyz"].tobytes() == want["xyz"].tobytes(), label
    if not fisheye:
        assert got["bgr"].tobytes() == want["bgr"].tobytes(), label
        return 0
    d = np.abs(got["bgr"].astype(int) - want["bgr"].astype(int))
    assert d.max(initial=0) <= 1, label
    off = int((d > 0).any(1).sum())
    print(f"{label}: {off} of {len(got['index'])} kept points differ by 1 in a channel (pixel position 1 ulp apart)")
    return off


@pytest.mark.parametrize("case", ["pinhole-resident-100k", "pinhole-host-300k", "radtan-host-100k", "fisheye-resident-50k", "fisheye-host-300k"])
def test_config_clouds_match_the_oracle(gpu_ctx, case):
    camera, where, size = case.split("-")
    n = int(size[:-1]) * 1000
    sc = CC.scene(camera, n, seed=n // 1000)
    got = _device(gpu_ctx, sc, resident=(where == "resident"))
    want = CC.OracleColor(sc).publish(sc)
    assert len(want["index"]) > n // 40
    _compare(got, want, fisheye=(camera == "fisheye"), label=case)


@pytest.mark.parametrize("camera", ["edge", "edge_radtan", "edge_fisheye"])
def test_hand_built_points_match_the_oracle(gpu_ctx, camera):
    sc = CC.pin_scenes()[camera]
    got = _device(gpu_ctx, sc)
    want = CC.OracleColor(sc).publish(sc)
    _compare(got, want, fisheye=(camera == "edge_fisheye"), label=camera)
    if camera == "edge":
        assert np.array_equal(got["index"], np.nonzero(sc["keep"])[0])


def test_resident_scan_equals_the_same_points_from_the_host(gpu_ctx):
    sc = CC.scene("radtan", 20_000, seed=4)
    a = _device(gpu_ctx, sc, resident=True)
    b = _device(gpu_ctx, sc, resident=False)
    for k in ("xyz", "bgr", "index"):
        assert a[k].tobytes() == b[k].tobytes(), k


# ----------------------------------------------------------------------------------------------------- the chained tick
def _tick(ctx, fr, c, with_color, blind=0.05):
    """One LIO tick on the device-resident map and one VIO tick on a selected sub-map, the colour calls interleaved where
    a LIVO loop makes them (with_color) or left out. Returns every output of the ticks."""
    cfg = fr["lio_cfg"]
    ctx.set_extrinsics(fr["ext"])
    ctx.map_device_init(cfg, root_capacity=1 << 16, grow=True)
    ctx.lio_set_scan(fr["pts"])
    ctx.map_device_build(fr["state_prior"])
    out = {}
    g = ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], cfg)
    out["lio"] = g
    ctx.map_device_update(None)
    if with_color:
        ctx.rgb_set_cloud(None, None)  # the resident scan and the LIO posterior left on the device
        dense = np.concatenate([fr["pts"], fr["pts"] * np.float32(1.01)])  # a "dense" cloud of another size, from the host
    ctx.vio_set_camera(c["camcfg"], S.VioCfg())
    ctx.vio_set_image(c["img"])
    ctx.vio_set_ref_images(c["ref_imgs"])
    sel = ctx.vio_select_patches(c["ref_idx"], c["px_ref"], c["pos_w"], c["T_ref"], c["ref_inv_expo"], c["pc"], c["T_cur"], c["inv_expo"], normal_w=c["normal_w"])
    out["kept"] = sel["kept"]
    ctx.vio_run(g["state"], g["state"])
    if with_color:
        rgb = CC.bgr_image(c["camcfg"], 3)
        out["rgb"] = ctx.rgb_colorize(rgb, blind)
    out["vio"] = ctx.vio_fetch()
    out["stats"] = ctx.map_device_stats()
    out["map"] = ctx.map_device_download()
    if with_color:
        out["rgb_explicit"] = ctx.rgb_colorize(rgb, blind, state=out["vio"]["state"])
        ctx.rgb_set_cloud(fr["pts"], g["state"])
        out["rgb_host"] = ctx.rgb_colorize(rgb, blind, state=out["vio"]["state"])
        ctx.rgb_set_cloud(dense, g["state"])
        out["rgb_dense"] = ctx.rgb_colorize(rgb, blind, state=out["vio"]["state"])
        out["dense"] = dense
    return out


def test_chained_tick_matches_the_oracle_and_disturbs_nothing(small_vio_frame):
    """lio_update -> map_device_update(NULL) -> rgb_set_cloud(NULL, NULL) -> vio_select_patches + vio_run ->
    rgb_colorize(NULL) against the oracle chained the same way (world cloud with the LIO posterior, colours with the VIO
    posterior); NULL states equal the explicit ones; and the LIO / VIO outputs, map stats and map download are byte-identical
    to the same ticks without the colour calls."""
    fr = small_vio_frame
    c = SC.candidates("radtan", 300, seed=1)
    ctx_a, ctx_b = api.Context(0), api.Context(0)
    try:
        a = _tick(ctx_a, fr, c, with_color=True)
        b = _tick(ctx_b, fr, c, with_color=False)
    finally:
        ctx_a.close(), ctx_b.close()
    for k in ("state", "dis_to_plane", "M", "HTH", "HTz", "solution"):
        assert np.ascontiguousarray(a["lio"][k]).tobytes() == np.ascontiguousarray(b["lio"][k]).tobytes(), k
    for k in ("match_plane", "normal_plane"):  # record slots of a device-built map: which points matched, not the slot numbers
        assert np.array_equal(a["lio"][k] >= 0, b["lio"][k] >= 0), k
    for k in ("state", "errors", "HTH", "HTz", "solution", "iters_per_level"):
        assert np.ascontiguousarray(a["vio"][k]).tobytes() == np.ascontiguousarray(b["vio"][k]).tobytes(), k
    assert np.array_equal(a["kept"], b["kept"]) and a["stats"] == b["stats"]
    # roots come out in no particular order: compare them in key order, each with its planes
    keys = a["map"]["keys"][np.lexsort(a["map"]["keys"].T[::-1])]
    ma, mb = O.flat_map_subset(a["map"], keys), O.flat_map_subset(b["map"], keys)
    assert len(b["map"]["keys"]) == len(keys)
    for k in ("keys", "count", "planes"):
        assert ma[k].tobytes() == mb[k].tobytes(), k
    # the oracle chained on the posteriors the device left
    sc = dict(cam=c["camcfg"], ext=fr["ext"], pts=fr["pts"], lio_state=a["lio"]["state"], vio_state=a["vio"]["state"], img=CC.bgr_image(c["camcfg"], 3),
              blind=0.05)
    want = CC.OracleColor(sc).publish(sc)
    assert len(want["index"]) > 20
    _compare(a["rgb"], want, label="chained")
    for k in ("rgb_explicit", "rgb_host"):
        for f in ("xyz", "bgr", "index"):
            assert a[k][f].tobytes() == a["rgb"][f].tobytes(), (k, f)
    dense = CC.OracleColor(sc).publish(dict(sc, pts=a["dense"]))
    _compare(a["rgb_dense"], dense, label="dense")


# ----------------------------------------------------------------------------------------------------- errors
def _status(fn):
    with pytest.raises(api.EsikfError) as e:
        fn()
    return int(str(e.value).split(":")[0].split()[1])


def test_call_order_image_size_and_capacity_errors():
    sc = CC.scene("pinhole", 5000, seed=2)
    ctx = api.Context(0)
    try:
        assert _status(lambda: ctx.rgb_set_cloud(sc["pts"], sc["lio_state"])) == -4  # before set_extrinsics
        ctx.set_extrinsics(sc["ext"])
        assert _status(lambda: ctx.rgb_set_cloud(None, sc["lio_state"])) == -4      # no resident scan
        assert _status(lambda: ctx.rgb_set_cloud(sc["pts"], None)) == -4             # no LIO posterior yet
        assert _status(lambda: ctx.rgb_colorize(sc["img"], 0.01, state=sc["vio_state"])) == -4  # no cloud
        ctx.rgb_set_cloud(sc["pts"], sc["lio_state"])
        assert _status(lambda: ctx.rgb_colorize(sc["img"], 0.01, state=sc["vio_state"])) == -4  # no camera
        ctx.vio_set_camera(sc["cam"], S.VioCfg())
        assert _status(lambda: ctx.rgb_colorize(sc["img"], 0.01)) == -4              # no VIO posterior yet
        assert _status(lambda: ctx.rgb_colorize(sc["img"][:-1], 0.01, state=sc["vio_state"])) == -3  # image size
        lib = ctx.lib
        neg = lib.esikf_rgb_set_cloud(ctx.h, sc["pts"].ctypes.data, -1, sc["lio_state"].ctypes.data)
        assert neg == -3
        full = ctx.rgb_colorize(sc["img"], 0.01, state=sc["vio_state"])
        k = len(full["index"])
        assert k > 10
        # cap too small: only *n_out is written
        xyz, bgr, idx = np.full((k, 3), 7.0, np.float32), np.full((k, 3), 9, np.uint8), np.full(k, -5, np.int32)
        n = C.c_int32(-1)
        img, st = np.ascontiguousarray(sc["img"]), np.ascontiguousarray(sc["vio_state"])
        rc = lib.esikf_rgb_colorize(ctx.h, img.ctypes.data, img.shape[1], img.shape[0], st.ctypes.data, 0.01, k - 1, C.byref(n), xyz.ctypes.data,
                                    bgr.ctypes.data, idx.ctypes.data)
        assert rc == -3 and n.value == k
        assert (xyz == 7.0).all() and (bgr == 9).all() and (idx == -5).all()
        assert lib.esikf_rgb_colorize(ctx.h, img.ctypes.data, img.shape[1], img.shape[0], st.ctypes.data, 0.01, k, None, xyz.ctypes.data, bgr.ctypes.data,
                                      None) == -3  # missing n_out
        rc = lib.esikf_rgb_colorize(ctx.h, img.ctypes.data, img.shape[1], img.shape[0], st.ctypes.data, 0.01, k, C.byref(n), xyz.ctypes.data, bgr.ctypes.data, None)
        assert rc == 0 and n.value == k and xyz.tobytes() == full["xyz"].tobytes()
        # after a VIO update the LIO posterior is gone: rgb_set_cloud(state = NULL) refuses
        ctx.vio_set_image(np.zeros((sc["cam"].height, sc["cam"].width), np.uint8))
        ctx.vio_set_patches(np.zeros((0, 3)), np.zeros((0, 256), np.float32), np.zeros(0, np.int32), np.zeros(0))
        ctx.vio_run(sc["vio_state"], sc["vio_state"])
        assert _status(lambda: ctx.rgb_set_cloud(sc["pts"], None)) == -4
        nul = ctx.rgb_colorize(sc["img"], 0.01)  # the VIO posterior (here the state the empty update kept)
        assert nul["index"].tobytes() == full["index"].tobytes()
    finally:
        ctx.close()
