"""GPU: entry points added (or first tested) at the end of round 1 — esikf_vio_warp_affine, the shim's per-patch
getImagePatch / warpAffine mirrors, esikf_map_patch and the shim's incremental map refresh."""
import ctypes as C

import numpy as np
import pytest

import oracle_bind as O
import shim_bind as SB
from fast_livo2_b200 import api
from harness import compare_lio, lio_gpu, lio_oracle, vio_prior, vio_setup, vio_warp

pytestmark = pytest.mark.gpu


def test_warp_affine_alone_with_caller_matrices(gpu_ctx, small_vio_frame):
    """esikf_vio_warp_affine (include/vio.h:161-162): the same kernel as warp_patches fed with caller-provided matrices —
    identical to the batched producer for its own matrices, and equal to the oracle's warpAffine for arbitrary ones
    (rotation + anisotropic scale, search levels 0 / 1; a zero matrix leaves zeros)."""
    fr = small_vio_frame
    vio_setup(gpu_ctx, fr)
    prior = vio_prior(fr)
    g = vio_warp(gpu_ctx, fr, prior)
    n = len(fr["vis_pos"])
    again = gpu_ctx.vio_warp_affine(np.zeros(n, np.int32), fr["px_ref"], g["A_cur_ref"], g["search_levels"])
    assert np.array_equal(again, g["warp_patch"])
    m = 24
    rng = np.random.default_rng(5)
    ang = rng.uniform(-0.6, 0.6, m)
    A = np.stack([np.stack([1.3 * np.cos(ang), -0.8 * np.sin(ang)], 1), np.stack([1.3 * np.sin(ang), 0.8 * np.cos(ang)], 1)], 1)  # (m, 2, 2)
    A[-1] = 0.0  # singular with A_ref_cur(0, 0) = NaN: the patch is left untouched (vio.cpp:297-301)
    sl = (np.arange(m) % 2).astype(np.int32)
    out = gpu_ctx.vio_warp_affine(np.zeros(m, np.int32), fr["px_ref"][:m], A, sl)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    exact = 0
    for i in range(m - 1):
        ref = vio.warp_affine(fr["img_ref"], A[i], fr["px_ref"][i], sl[i])
        np.testing.assert_allclose(out[i], ref, atol=2e-3)
        exact += np.array_equal(out[i], ref)
    assert exact >= m // 2  # float products without contraction on both sides: mostly bit-exact
    assert not out[-1].any()


def test_shim_patch_helpers_match_oracle(small_vio_frame):
    """VIOManager::getImagePatch / VIOManager::warpAffine mirrors (include/vio.h:151, 161-162): one patch each through the
    shim class; only the addressed pyramid level of the caller's buffer is written."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    fr = small_vio_frame
    shim = SB.load()
    L = fr["vio_cfg"].levels
    cam = api.CameraC(fr["cam_cfg"].model, fr["cam_cfg"].width, fr["cam_cfg"].height, 0, fr["cam_cfg"].fx, fr["cam_cfg"].fy, fr["cam_cfg"].cx, fr["cam_cfg"].cy)
    cam.d[:] = list(fr["cam_cfg"].d)
    vcfg = api.VioCfgC(fr["vio_cfg"].img_point_cov, L, fr["vio_cfg"].max_iterations, int(fr["vio_cfg"].exposure_estimate_en), 0)
    img, img_ref = np.ascontiguousarray(fr["img"]), np.ascontiguousarray(fr["img_ref"])
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    pc = np.array([301.37, 222.81])
    A = np.array([[1.1, -0.2], [0.15, 0.9]])
    px_ref = np.ascontiguousarray(fr["px_ref"][0], dtype=np.float64)
    for level, search_level in ((0, 0), (2, 1), (L - 1, 0)):
        patch = np.full(64 * L, -7.0, np.float32)
        warp = np.full(64 * L, -7.0, np.float32)
        rc = shim.fl2_shim_patch_helpers(C.byref(cam), C.byref(vcfg), vp(img), img.shape[1], img.shape[0], vp(pc), level, vp(patch), vp(A), vp(img_ref), vp(px_ref),
                                         search_level, level, vp(warp))
        assert rc == 0
        sel = slice(64 * level, 64 * level + 64)
        assert np.array_equal(patch[sel], vio.get_image_patch(img, pc, level))
        np.testing.assert_allclose(warp[sel], vio.warp_affine(img_ref, A, px_ref, search_level)[sel], atol=2e-3)
        untouched = np.ones(64 * L, bool)
        untouched[sel] = False
        assert (patch[untouched] == -7.0).all() and (warp[untouched] == -7.0).all()


def _refit(planes, rng, frac=0.05):
    """Planes as UpdateVoxelMap would leave them after refitting a few: nudged offsets / normals, same structure."""
    out = planes.copy()
    ids = np.sort(rng.choice(len(out), max(3, int(frac * len(out))), replace=False))
    out["d"][ids] += rng.normal(0, 0.01, len(ids)).astype(np.float32)
    out["center"][ids] += rng.normal(0, 0.005, (len(ids), 3))
    out["plane_var"][ids] *= 1.1
    return out, ids


def test_map_patch_equals_full_upload(small_frame):
    """esikf_map_patch: patching the refitted plane records in place gives the same update, bit for bit, as uploading the
    whole modified map into a fresh context."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    fr = small_frame
    m = fr["map"]
    rng = np.random.default_rng(8)
    planes_b, ids = _refit(np.ascontiguousarray(m["planes"]), rng)
    a = api.Context(0)
    b = api.Context(0)
    try:
        for ctx in (a, b):
            ctx.set_extrinsics(fr["ext"])
        a.map_upload(m, fr["lio_cfg"].voxel_size)
        before = a.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], fr["lio_cfg"])
        a.map_patch(ids.astype(np.int32), planes_b[ids])
        ra = a.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], fr["lio_cfg"])
        b.map_upload(dict(m, planes=planes_b), fr["lio_cfg"].voxel_size)
        rb = b.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], fr["lio_cfg"])
    finally:
        a.close()
        b.close()
    assert not np.array_equal(before["state"], ra["state"])  # the refit matters
    for key in ("state", "match_plane", "normal_plane", "dis_to_plane", "M", "HTH"):
        assert np.array_equal(np.asarray(ra[key]), np.asarray(rb[key])), key


def test_shim_incremental_map_sync_equals_fresh_upload(small_frame):
    """VoxelMapManager::SyncDeviceMap after the host map was refitted under it: the changed records are patched (no full
    upload) and StateEstimation matches a fresh manager built on the refitted map."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    fr = small_frame
    shim = SB.load()
    m = fr["map"]
    k, f, c = (np.ascontiguousarray(m["keys"], dtype=np.int64), np.ascontiguousarray(m["first"], dtype=np.int32), np.ascontiguousarray(m["count"], dtype=np.int32))
    pa = np.ascontiguousarray(m["planes"])
    pb, ids = _refit(pa, np.random.default_rng(9))
    lcfg = api.lio_cfg_c(fr["lio_cfg"])
    ext = api.ExtrinsicsC()
    ext.extR[:] = fr["ext"].extR.reshape(9)
    ext.extT[:] = fr["ext"].extT
    ext.Rcl[:] = fr["ext"].Rcl.reshape(9)
    ext.Pcl[:] = fr["ext"].Pcl
    pts = np.ascontiguousarray(fr["pts"])
    sp = np.ascontiguousarray(fr["state_prior"])
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    out_inc, out_fresh = np.zeros(386), np.zeros(386)
    npatched = C.c_int32(-2)
    rc = shim.fl2_shim_resync_run(vp(k), vp(f), vp(c), len(f), vp(pa), vp(pb), len(pa), C.byref(lcfg), C.byref(ext), vp(pts), len(pts), vp(sp), vp(out_inc),
                                  C.byref(npatched))
    assert rc == 0 and npatched.value == len(ids)
    n2 = C.c_int32(-2)
    rc = shim.fl2_shim_resync_run(vp(k), vp(f), vp(c), len(f), vp(pb), vp(pb), len(pb), C.byref(lcfg), C.byref(ext), vp(pts), len(pts), vp(sp), vp(out_fresh),
                                  C.byref(n2))
    assert rc == 0 and n2.value == 0  # nothing changed between the two syncs
    assert np.array_equal(out_inc, out_fresh)


@pytest.mark.parametrize("kind", ["voxel_0.5", "voxel_0.4", "voxel_2.0"])
def test_lio_association_on_voxel_boundaries_and_negative_keys(gpu_ctx, kind):
    """Bit-exact voxel indexing and neighbour rule where they are fragile (parity_util.edge_scan: points exactly on voxel
    corners / faces with both signs, one float ulp to either side, z == 0, and off-plane points that send the lookup to
    the one neighbour voxel the unit-mixing rule picks), for the three voxel sizes of the shipped configs: 0.5 (exact
    reciprocal: multiply), 0.4 (true fp64 division) and 2.0. The same scans go through the reference source on the CPU in
    tests/test_oracle_ref_pin.py::test_edge_scan_oracle_reproduces_the_reference_source."""
    from conftest import get_frame
    from parity_util import edge_scan
    from ref_pin_cases import EDGE_FRAMES

    fr = get_frame(**EDGE_FRAMES[kind])
    pts, ext, state = edge_scan(fr)
    fe = dict(fr, pts=pts, ext=ext, state_prior=state)
    o = lio_oracle(fe)
    assert o["M"][0] > 20
    compare_lio(lio_gpu(gpu_ctx, fe), o)
