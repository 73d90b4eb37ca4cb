"""GPU: esikf_vio_select_patches (the per-candidate tail of retrieveFromVisualSparseMap on the device) against the oracle's
restatement (oracle/orc_select.cpp) on seeded candidate sets of config-2 shape (2 k candidates, pinhole-radtan) and config-3
shape (1 k, fisheye), exposure times != 1, several candidates per reference frame; both warp forms, NCC on and off.

The warp matrices are evaluated by the device's own camera arithmetic, which nvcc contracts (as in warp_matrix_kernel): A is
compared within 1e-10 of the oracle's, and every later step (warps, current patch, error, gates, append) bit for bit against
the oracle evaluated on the device's A and levels."""
import numpy as np
import pytest

import select_cases as SC
import shim_bind as SB
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from harness import VIO_KEYS, bits_equal, variant

pytestmark = pytest.mark.gpu
SHAPES = {"config2": ("radtan", 2000), "config3": ("fisheye", 1000)}


def _setup(ctx, c, levels=4):
    ctx.set_extrinsics(S.avia_extrinsics())
    ctx.vio_set_camera(c["camcfg"], S.VioCfg(levels=levels))
    ctx.vio_set_image(c["img"])
    ctx.vio_set_ref_images(c["ref_imgs"])


def _select(ctx, c, **kw):
    return ctx.vio_select_patches(c["ref_idx"], c["px_ref"], c["pos_w"], c["T_ref"], c["ref_inv_expo"], c["pc"], c["T_cur"], c["inv_expo"], normal_w=c["normal_w"],
                                  ref_level=c["ref_level"], ref_f=c["ref_f"], ref_pos=c["ref_pos"], ref_key=c["ref_key"], **kw)


def _check(ctx, c, normal_en, ncc_en, quantile=0.5):
    """Select on the device and on the oracle; returns (device result, oracle result, outlier_threshold)."""
    n = len(c["px_ref"])
    o = SC.OracleSelect(c["camcfg"])
    everything = _select(ctx, c, normal_en=normal_en, outlier_threshold=1e30, want_patches=True)
    assert np.array_equal(everything["kept"], np.arange(n))
    A, sl = everything["A_cur_ref"], everything["search_levels"]
    own = o.select(c, normal_en=normal_en, outlier_threshold=1e30)
    np.testing.assert_allclose(A, own["A_cur_ref"], rtol=0, atol=1e-10)
    assert np.array_equal(sl, own["search_levels"])
    on_dev = o.select(c, normal_en=normal_en, outlier_threshold=1e30, A_in=A, sl_in=sl)
    assert np.array_equal(everything["warp_patch"], on_dev["warp_patch"])
    assert np.array_equal(everything["errors"].view(np.uint32), on_dev["errors"].view(np.uint32))
    thr = float(np.quantile(on_dev["errors"], quantile)) / 64
    v = SC.OracleSelect(c["camcfg"])
    want = v.select(c, normal_en=normal_en, ncc_en=ncc_en, ncc_thre=0.05, outlier_threshold=thr, A_in=A, sl_in=sl)
    got = _select(ctx, c, normal_en=normal_en, ncc_en=ncc_en, ncc_thre=0.05, outlier_threshold=thr, want_patches=True)
    assert np.array_equal(got["kept"], want["kept"]), (len(got["kept"]), len(want["kept"]))
    k = want["kept"]
    assert np.array_equal(got["errors"].view(np.uint32), want["errors"][k].view(np.uint32))
    assert np.array_equal(got["search_levels"], want["search_levels"][k])
    assert np.array_equal(got["A_cur_ref"].view(np.uint64), A[k].view(np.uint64))
    assert np.array_equal(got["warp_patch"], want["warp_patch"][k])
    return got, want, thr


@pytest.mark.parametrize("ncc_en", [False, True])
@pytest.mark.parametrize("normal_en", [True, False])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_select_matches_oracle(gpu_ctx, shape, normal_en, ncc_en):
    camera, n = SHAPES[shape]
    c = SC.candidates(camera, n, n_frames=40, seed=7)
    _setup(gpu_ctx, c)
    got, want, _ = _check(gpu_ctx, c, normal_en, ncc_en)
    assert 0.4 * n < len(got["kept"]) < 0.6 * n or (ncc_en and len(got["kept"]) > 0)
    if ncc_en:
        assert (~want["keep"]).sum() > n // 2  # the NCC gate removed some candidates below the error quantile too


def test_all_none_and_border(gpu_ctx):
    """All kept, none kept (the next run is that of an empty sub-map) and current patches that reach past the image border."""
    c = SC.candidates("radtan", 300, seed=9)
    cam = c["camcfg"]
    edge = np.array([[0.2, 0.3], [cam.width - 1.4, cam.height - 0.6], [-2.5, 100.0], [100.0, cam.height + 1.5], [3.9, 3.9], [cam.width - 4.1, 4.0]])
    c["pc"][:len(edge)] = edge
    c["px_ref"][len(edge):2 * len(edge)] = edge  # reference footprints at the border too
    _setup(gpu_ctx, c)
    _check(gpu_ctx, c, True, False)
    a = _select(gpu_ctx, c, outlier_threshold=1e30)
    assert len(a["kept"]) == 300
    none = _select(gpu_ctx, c, outlier_threshold=-1.0)
    assert len(none["kept"]) == 0
    prior = S.pack_state(np.eye(3), np.zeros(3), 1.0, cov=S.random_prior_cov(np.random.default_rng(0), scale=0.2))
    gpu_ctx.vio_run(prior, prior)
    e = gpu_ctx.vio_fetch()
    z = gpu_ctx.vio_update(c["img"], np.zeros((0, 3)), np.zeros((0, 256), np.float32), np.zeros(0, np.int32), np.zeros(0), prior, prior)
    bits_equal(e, z, VIO_KEYS)


@pytest.mark.parametrize("loop_mode", [0, 2])
@pytest.mark.parametrize("normal_en", [True, False])
def test_select_then_run_equals_set_patches(gpu_ctx, loop_mode, normal_en):
    """select_patches + vio_run gives the posterior and stats of set_patches with the oracle's survivors + vio_run."""
    c = SC.candidates("radtan", 2000, n_frames=40, seed=11)
    _setup(gpu_ctx, c)
    got, want, thr = _check(gpu_ctx, c, normal_en, False)
    k = want["kept"]
    prior = S.pack_state(np.eye(3), np.zeros(3), 0.9, cov=S.random_prior_cov(np.random.default_rng(2), scale=0.05))
    with variant(gpu_ctx, loop_mode=loop_mode):
        _select(gpu_ctx, c, normal_en=normal_en, outlier_threshold=thr)
        gpu_ctx.vio_run(prior, prior)
        a = gpu_ctx.vio_fetch()
        b = gpu_ctx.vio_update(c["img"], c["pos_w"][k], want["warp_patch"][k], want["search_levels"][k], c["ref_inv_expo"][k], prior, prior)
    bits_equal(a, b, VIO_KEYS)
    assert a["total_iters"] > 0


def test_bad_arguments_leave_the_sub_map(gpu_ctx):
    c = SC.candidates("radtan", 64, seed=13)
    _setup(gpu_ctx, c)
    first = _select(gpu_ctx, c, outlier_threshold=1e30)
    prior = S.pack_state(np.eye(3), np.zeros(3), 0.9, cov=S.random_prior_cov(np.random.default_rng(2), scale=0.05))
    gpu_ctx.vio_run(prior, prior)
    before = gpu_ctx.vio_fetch()
    bad = [dict(ref_idx=np.full(64, 3, np.int32)), dict(ref_idx=np.full(64, -1, np.int32)), dict(ref_level=np.full(64, 9, np.int32))]
    for b in bad:
        cc = dict(c, **b)
        with pytest.raises(api.EsikfError, match="status -3"):
            _select(gpu_ctx, cc, normal_en=False)
    with pytest.raises(api.EsikfError, match="status -3"):  # the depth form without its inputs
        gpu_ctx.vio_select_patches(c["ref_idx"], c["px_ref"], c["pos_w"], c["T_ref"], c["ref_inv_expo"], c["pc"], c["T_cur"], 1.0, normal_en=False)
    lib = gpu_ctx.lib
    assert lib.esikf_vio_select_patches(gpu_ctx.h, -1, *([None] * 12), 1.0, None, None, None, None, None, None, None) == -3
    gpu_ctx.vio_run(prior, prior)
    bits_equal(gpu_ctx.vio_fetch(), before, VIO_KEYS)
    assert len(first["kept"]) == 64
    fresh = api.Context(0)
    try:
        fresh.set_extrinsics(S.avia_extrinsics())
        fresh.vio_set_camera(c["camcfg"], S.VioCfg(levels=4))
        with pytest.raises(api.EsikfError, match="status -4"):  # no current image yet
            _select(fresh, c)
    finally:
        fresh.close()


CAND_DTYPE = np.dtype([("ref_img_index", "<i4"), ("ref_level", "<i4"), ("ref_key", "<i4"), ("pad_", "<i4"), ("px_ref", "<f8", 2), ("ref_f", "<f8", 3),
                       ("ref_pos", "<f8", 3), ("pos_w", "<f8", 3), ("normal_w", "<f8", 3), ("T_ref_w", "<f8", 12), ("ref_inv_expo", "<f8"), ("pc", "<f8", 2)])


@pytest.mark.parametrize("normal_en", [True, False])
def test_shim_select_then_update_equals_host_sub_map(gpu_ctx, normal_en):
    """VIOManager::SelectSubSparseMap + computeJacobianAndUpdateEKF (no sub-map upload) equals the update on the same sub-map
    assembled on the host (MaterializeWarpPatches, set_patches path), bit for bit; the kept set, errors and patches are those
    of esikf_vio_select_patches."""
    import ctypes as C
    import os
    assert CAND_DTYPE.itemsize == 248
    c = SC.candidates("radtan", 1500, n_frames=30, seed=17)
    _setup(gpu_ctx, c)
    n = len(c["px_ref"])
    everything = _select(gpu_ctx, c, normal_en=normal_en, outlier_threshold=1e30)
    thr = float(np.sort(everything["errors"])[n // 2]) / 64
    direct = _select(gpu_ctx, c, normal_en=normal_en, outlier_threshold=thr, want_patches=True)
    cand = np.zeros(n, CAND_DTYPE)
    for f, k in (("ref_img_index", "ref_idx"), ("ref_level", "ref_level"), ("ref_key", "ref_key"), ("px_ref", "px_ref"), ("ref_f", "ref_f"), ("ref_pos", "ref_pos"),
                 ("pos_w", "pos_w"), ("normal_w", "normal_w"), ("T_ref_w", "T_ref"), ("ref_inv_expo", "ref_inv_expo"), ("pc", "pc")):
        cand[f] = c[k]
    cam, ext = c["camcfg"], S.avia_extrinsics()
    cc = api.CameraC(cam.model, cam.width, cam.height, 0, cam.fx, cam.fy, cam.cx, cam.cy)
    cc.d[:] = list(cam.d)
    vc = api.VioCfgC(100.0, 4, 5, 1, 0)
    ec = api.ExtrinsicsC()
    ec.extR[:], ec.extT[:], ec.Rcl[:], ec.Pcl[:] = ext.extR.reshape(9), ext.extT, ext.Rcl.reshape(9), ext.Pcl
    imgs = [np.ascontiguousarray(im) for im in c["ref_imgs"]]
    arr = (C.c_void_p * len(imgs))(*[im.ctypes.data for im in imgs])
    prior = S.pack_state(np.eye(3), np.zeros(3), c["inv_expo"], cov=S.random_prior_cov(np.random.default_rng(2), scale=0.05))
    gate = np.array([float(normal_en), 0.0, 0.0, thr])
    nk = C.c_int32(0)
    kept, e_sel, e_host = np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(n, np.float32)
    s_sel, s_host, wp, counts = np.zeros(386), np.zeros(386), np.zeros((n, 256), np.float32), np.zeros(4, np.int64)
    img, T_cur = np.ascontiguousarray(c["img"]), np.ascontiguousarray(c["T_cur"])
    shim = SB.load()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = shim.fl2_shim_select_run(C.byref(cc), C.byref(vc), C.byref(ec), vp(img), C.cast(arr, C.c_void_p), len(imgs), vp(cand), n, vp(T_cur), vp(prior),
                                  vp(gate), C.byref(nk), vp(kept), vp(s_sel), vp(e_sel), vp(s_host), vp(e_host), vp(wp), vp(counts))
    assert rc == 0
    k = nk.value
    assert k == len(direct["kept"]) and 0 < k < n
    assert np.array_equal(kept[:k], direct["kept"])
    assert np.array_equal(wp[:k], direct["warp_patch"])
    assert np.array_equal(s_sel.view(np.uint64), s_host.view(np.uint64))
    assert np.array_equal(e_sel[:k].view(np.uint32), e_host[:k].view(np.uint32))
    # the selected sub-map's update uploads no sub-map; the host-assembled one uploads it once; both launch the same update
    assert counts[1] == 0 and counts[3] == 1 and counts[0] == counts[2] > 0, counts
    assert not np.array_equal(e_sel[:k], direct["errors"])  # the update wrote its own errors over the gate's


def test_gate_ties_on_the_device(gpu_ctx):
    """error == outlier_threshold * 64 is kept and one double ulp lower it is dropped; ncc == ncc_thre is kept and one ulp
    higher it is dropped — on the device's own errors and on the NCC of the device's patches."""
    c = SC.candidates("radtan", 400, seed=19)
    _setup(gpu_ctx, c)
    everything = _select(gpu_ctx, c, outlier_threshold=1e30, want_patches=True)
    err = everything["errors"].astype(np.float64)
    j = int(np.argsort(err)[200])
    at = _select(gpu_ctx, c, outlier_threshold=err[j] / 64)
    assert j in at["kept"] and np.array_equal(at["kept"], np.nonzero(err <= err[j])[0])
    below = _select(gpu_ctx, c, outlier_threshold=np.nextafter(err[j], -np.inf) / 64)
    assert j not in below["kept"] and np.array_equal(below["kept"], np.nonzero(err < err[j])[0])
    o = SC.OracleSelect(c["camcfg"])
    cur = gpu_ctx.vio_get_image_patch(c["pc"], 0)
    ncc = np.array([o.ncc(everything["warp_patch"][i][:64], cur[i]) for i in range(len(err))])
    on = _select(gpu_ctx, c, ncc_en=True, ncc_thre=ncc[j], outlier_threshold=1e30)
    assert j in on["kept"] and np.array_equal(on["kept"], np.nonzero(ncc >= ncc[j])[0])
    off = _select(gpu_ctx, c, ncc_en=True, ncc_thre=np.nextafter(ncc[j], np.inf), outlier_threshold=1e30)
    assert j not in off["kept"] and np.array_equal(off["kept"], np.nonzero(ncc > ncc[j])[0])
