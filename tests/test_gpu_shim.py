"""GPU: the C++ shim (VoxelMapManager::StateEstimation / VIOManager::computeJacobianAndUpdateEKF mirrors) gives the same
states as the direct C-ABI calls and as the oracle."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_bind as O
import shim_bind as SB
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from parity_util import assert_state_close

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shim_lio_and_vio_match_oracle(gpu_ctx, small_vio_frame):
    fr = small_vio_frame
    shim = SB.load()
    m = fr["map"]
    k, f, c, p = (np.ascontiguousarray(m["keys"]), np.ascontiguousarray(m["first"]), np.ascontiguousarray(m["count"]), np.ascontiguousarray(m["planes"]))
    lcfg = api.lio_cfg_c(fr["lio_cfg"])
    ext = api.ExtrinsicsC()
    ext.extR[:] = fr["ext"].extR.reshape(9)
    ext.extT[:] = fr["ext"].extT
    ext.Rcl[:] = fr["ext"].Rcl.reshape(9)
    ext.Pcl[:] = fr["ext"].Pcl
    cam = api.CameraC(fr["cam_cfg"].model, fr["cam_cfg"].width, fr["cam_cfg"].height, 0, fr["cam_cfg"].fx, fr["cam_cfg"].fy, fr["cam_cfg"].cx, fr["cam_cfg"].cy)
    cam.d[:] = list(fr["cam_cfg"].d)
    vcfg = api.VioCfgC(fr["vio_cfg"].img_point_cov, fr["vio_cfg"].levels, fr["vio_cfg"].max_iterations, int(fr["vio_cfg"].exposure_estimate_en), 0)
    pts = np.ascontiguousarray(fr["pts"])
    n = len(pts)
    # oracle LIO first: its posterior is what the warp patches are built for
    lio = O.OracleLIO(fr["lio_cfg"], fr["ext"])
    lio.set_map(m)
    o = lio.state_estimation(pts, fr["state_prior"], fr["state_prior"])
    w = O.oracle_warp_patches(fr, o["state"])
    npatch = len(fr["vis_pos"])
    lio_out, vio_out = np.zeros(386), np.zeros(386)
    neff, nptpl = C.c_int32(0), C.c_int32(0)
    normals = np.zeros((n, 3))
    errs = np.zeros(npatch, np.float32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    img = np.ascontiguousarray(fr["img"])
    pos, wp, sl, ie = (np.ascontiguousarray(fr["vis_pos"]), np.ascontiguousarray(w["warp_patch"]), np.ascontiguousarray(w["search_levels"]),
                       np.ascontiguousarray(fr["inv_ref_expo"]))
    sp = np.ascontiguousarray(fr["state_prior"])
    rc = shim.fl2_shim_run(vp(k), vp(f), vp(c), len(f), vp(p), len(p), C.byref(lcfg), C.byref(ext), vp(pts), n, vp(sp), vp(sp), vp(lio_out), C.byref(neff),
                           C.byref(nptpl), vp(normals), C.byref(cam), C.byref(vcfg), vp(img), npatch, vp(pos), vp(wp), vp(sl), vp(ie), vp(vio_out), vp(errs))
    assert rc == 0
    assert neff.value == o["M"][-1] and nptpl.value == o["M"][-1]
    assert_state_close(lio_out, o["state"])
    # pv.normal: the matched plane's normal, zero when the point never matched
    want = np.where(o["normal_plane"][:, None] >= 0, m["planes"]["normal"][np.maximum(o["normal_plane"], 0)], 0.0)
    assert np.array_equal(normals, want)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    ov = vio.update(img, pos, wp, sl, ie, lio_out, lio_out)
    assert_state_close(vio_out, ov["state"], rot_tol=1e-8, pos_tol=1e-8, cov_tol=1e-6, rest_tol=1e-8)
    np.testing.assert_allclose(errs, ov["errors"], rtol=2e-6, atol=1e-3)


def test_shim_session_with_device_resident_map_equals_the_c_abi_tick_loop(small_vio_frame):
    """fl2b200::VoxelMapManager in device-map mode (EnableDeviceMap, BuildVoxelMap, StateEstimation, UpdateVoxelMap() per tick)
    against the same sequence issued directly through the C ABI on a second context: identical posteriors every tick, and
    pv_list_ / ptpl_list_ materialise from device data (no host VoxelPlane exists in this mode)."""
    fr = small_vio_frame
    cfg, ext = fr["lio_cfg"], fr["ext"]
    shim = SB.load()
    m = fr["map"]
    k, f, c, p = (np.ascontiguousarray(m["keys"]), np.ascontiguousarray(m["first"]), np.ascontiguousarray(m["count"]), np.ascontiguousarray(m["planes"]))
    lcfg = api.lio_cfg_c(cfg)
    extc = api.ExtrinsicsC()
    extc.extR[:], extc.extT[:], extc.Rcl[:], extc.Pcl[:] = ext.extR.reshape(9), ext.extT, ext.Rcl.reshape(9), ext.Pcl
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    h = shim.fl2_shim_session_create(vp(k), vp(f), vp(c), len(f), vp(p), len(p), C.addressof(lcfg), C.addressof(extc), None, None, 0)
    assert h
    rng = np.random.default_rng(8)
    rects = fr["rects"]
    t = S.unpack_state(fr["state_true"])
    st0 = S.pack_state(t["R"], t["p"], cov=S.random_prior_cov(np.random.default_rng(1), scale=0.05), g=np.array([0, 0, -9.81]))
    scan0 = S.scan_at(rects, ext, t["R"], t["p"], 30000, cfg, rng)
    ctx = api.Context(0)
    try:
        assert shim.fl2_shim_session_device_map(h, vp(scan0), len(scan0), vp(st0), cfg.min_eigen_value, cfg.max_points_num, 1 << 15) == 0
        shim.fl2_shim_session_point_lists(h, 1)  # lazy lists
        ctx.set_extrinsics(ext)
        ctx.map_device_init(cfg, root_capacity=1 << 15)
        ctx.lio_set_scan(scan0)
        ctx.map_device_build(st0)
        prev = st0
        for tick in range(4):
            scan = S.scan_at(rects, ext, t["R"], t["p"], 8000, cfg, rng)
            s = S.unpack_state(prev)
            prior = S.pack_state(t["R"] @ S.so3_exp(np.array([0.003, -0.002, 0.002])), t["p"] + np.array([0.02, -0.01, 0.015]), cov=s["cov"] + np.eye(19) * 1e-6,
                                 g=np.array([0, 0, -9.81]))
            lio_out, vio_out, iters = np.zeros(386), np.zeros(386), np.zeros(2, np.int32)
            assert shim.fl2_shim_session_step(h, vp(scan), len(scan), vp(prior), vp(prior), None, 0, None, None, None, None, vp(lio_out), vp(vio_out), vp(iters)) == 0
            assert shim.fl2_shim_session_update_map(h) == 0
            g = ctx.lio_update(scan, prior, prior, cfg)
            ctx.map_device_update()
            assert iters[0] == g["iters"] and np.array_equal(lio_out, g["state"]), tick
            prev = g["state"]
        npv, nptpl = C.c_int32(0), C.c_int32(0)
        assert shim.fl2_shim_session_materialize(h, C.byref(npv), C.byref(nptpl)) == 0
        assert npv.value == 8000 and nptpl.value == int(np.asarray(g["M"])[g["iters"] - 1])
    finally:
        ctx.close()
        shim.fl2_shim_session_destroy(h)


def test_example_tick_loop_runs_on_the_device(tmp_path):
    import subprocess

    exe = str(tmp_path / "tick_loop")
    pkg = os.path.join(ROOT, "fast_livo2_b200")
    cmd = ["/usr/bin/g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "tick_loop.cpp"), "-L" + pkg, "-lfl2_shim", "-lesikf_b200",
           "-Wl,-rpath," + pkg, "-o", exe]
    assert subprocess.run(cmd, capture_output=True, text=True).returncode == 0
    run = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "BuildVoxelMap: status 0" in run.stdout and "tick 3 LIO: status 0" in run.stdout and "tick 3 VIO: status 0" in run.stdout, run.stdout
