"""ctypes binding of the CPU oracle (oracle/liborc_parity.so). TEST INFRASTRUCTURE ONLY:
imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg — never by
fast_livo2_b200/."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
STATE_PACK = 386

_libs = {}


def build_oracle():
    subprocess.run(["make", "-s", "-C", ORACLE_DIR], check=True)


def load(kind="parity"):
    if kind in _libs:
        return _libs[kind]
    path = os.path.join(ORACLE_DIR, f"liborc_{kind}.so")
    if kind == "baseline" and os.environ.get("ORC_BASELINE_SO") and os.path.exists(os.environ["ORC_BASELINE_SO"]):
        path = os.environ["ORC_BASELINE_SO"]  # built on the host the timing runs on (bench.py native_baseline_build)
    if not os.path.exists(path):
        build_oracle()
    lib = C.CDLL(path)
    vp, dp, fp, ip, i64p, u8p = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
    lib.orc_lio_create.restype = vp
    lib.orc_lio_create.argtypes = [dp, dp, dp, C.c_int]
    lib.orc_lio_destroy.argtypes = [vp]
    lib.orc_lio_set_map_flat.argtypes = [vp, i64p, ip, ip, C.c_int, vp, C.c_int]
    lib.orc_lio_build_map.argtypes = [vp, fp, fp, C.c_int, dp]
    lib.orc_lio_update_map.argtypes = [vp, dp, dp, C.c_int]
    lib.orc_lio_tick_build_map.argtypes = [vp, fp, C.c_int, dp]
    lib.orc_lio_tick_update_map.argtypes = [vp, dp, dp]
    lib.orc_lio_flatten.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), i64p, ip, ip, vp]
    lib.orc_lio_set_layer_init_num.argtypes = [vp, ip, C.c_int]
    lib.orc_lio_dump_nodes.restype = C.c_int
    lib.orc_lio_dump_nodes.argtypes = [vp, i64p, C.c_int]
    lib.orc_lio_state_estimation.restype = C.c_double
    lib.orc_lio_state_estimation.argtypes = [vp, fp, C.c_int, dp, dp, dp, ip, ip, fp, dp, dp, dp]
    lib.orc_lio_single_pass.argtypes = [vp, fp, C.c_int, dp, dp, ip, fp, dp, dp, dp, dp]
    lib.orc_vio_create.restype = vp
    lib.orc_vio_create.argtypes = [dp, dp, dp, dp, dp, dp, C.c_int]
    lib.orc_vio_destroy.argtypes = [vp]
    lib.orc_vio_update.restype = C.c_double
    lib.orc_vio_update.argtypes = [vp, u8p, C.c_int, dp, fp, ip, dp, dp, dp, dp, fp, dp]
    lib.orc_vio_get_image_patch.argtypes = [vp, u8p, dp, C.c_int, fp]
    lib.orc_vio_set_inverse_refs.argtypes = [vp, vp, C.c_int, C.c_int, ip, dp, dp, dp, dp]
    lib.orc_vio_set_inverse.argtypes = [vp, C.c_int]
    lib.orc_vio_get_h_sub_inv.restype = C.c_int
    lib.orc_vio_get_h_sub_inv.argtypes = [vp, dp, C.c_int]
    lib.orc_vio_precompute_reference_patches.argtypes = [vp, C.c_int, dp, C.c_int]
    lib.orc_vio_warp_affine.argtypes = [vp, u8p, C.c_int, C.c_int, dp, dp, C.c_int, fp]
    lib.orc_vio_warp_matrix.restype = C.c_int
    lib.orc_vio_warp_matrix.argtypes = [vp, dp, dp, dp, dp, dp, dp, dp, dp]
    lib.orc_cam_world2cam.argtypes = [vp, dp, dp]
    lib.orc_cam_cam2world.argtypes = [vp, dp, dp]
    for name in ("orc_boxplus", "orc_boxminus"):
        getattr(lib, name).argtypes = [dp, dp, dp]
    lib.orc_exp.argtypes = [dp, dp]
    lib.orc_log.argtypes = [dp, dp]
    lib.orc_inverse19.argtypes = [dp, dp]
    lib.orc_calc_body_cov.argtypes = [dp, C.c_float, C.c_float, dp, dp]
    lib.orc_default_state.argtypes = [dp]
    lib.orc_max_threads.restype = C.c_int
    _libs[kind] = lib
    return lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def dptr(a):
    return _p(a, C.c_double)


def fptr(a):
    return _p(a, C.c_float)


def iptr(a):
    return _p(a, C.c_int32)


def c64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def layer_init_num8(cfg):
    """lio/layer_init_num as the 8 entries (one per possible layer) every side of the map tests is given: padded with its last."""
    lin = list(cfg.layer_init_num)
    return np.array((lin + [lin[-1]] * 8)[:8], np.int32)


# one row of a node dump (oracle, reference source, host harness): the state of a VoxelOctoTree node
NODE_COLS = ("kx", "ky", "kz", "layer", "path", "init_octo", "octo_state", "update_enable", "is_plane", "new_points", "temp_points", "points_size")


def _dump_nodes(fill):
    n = fill(np.zeros((1, 12), np.int64), 0)
    out = np.zeros((max(n, 1), 12), np.int64)
    assert fill(out, n) == n
    out = out[:n]
    # roots in key order (a stable sort keeps every root's DFS order)
    return out[np.lexsort((out[:, 2], out[:, 1], out[:, 0]))] if n else out


class OracleLIO:
    def __init__(self, lio_cfg, ext, threads=1, kind="parity"):
        self.lib = load(kind)
        self.cfg = lio_cfg
        self.h = self.lib.orc_lio_create(dptr(lio_cfg.as_array()), dptr(c64(ext.extR)), dptr(c64(ext.extT)), threads)
        lin = layer_init_num8(lio_cfg)
        self.lib.orc_lio_set_layer_init_num(self.h, iptr(lin), len(lin))

    def __del__(self):
        try:
            self.lib.orc_lio_destroy(self.h)
        except Exception:
            pass

    def set_map(self, vmap):
        self._map = vmap  # keep alive
        k, f, c, p = vmap["keys"], vmap["first"], vmap["count"], vmap["planes"]
        self.lib.orc_lio_set_map_flat(self.h, _p(k, C.c_int64), iptr(f), iptr(c), len(f), p.ctypes.data, len(p))

    def build_map(self, pts_world_f32, pts_body_f32, state):
        pw = np.ascontiguousarray(pts_world_f32, dtype=np.float32)
        pb = np.ascontiguousarray(pts_body_f32, dtype=np.float32)
        self.lib.orc_lio_build_map(self.h, fptr(pw), fptr(pb), len(pw), dptr(c64(state)))

    def tick_build_map(self, pts_body_f32, state):
        """First LiDAR frame, LIVMapper.cpp:356-366."""
        pb = np.ascontiguousarray(pts_body_f32, dtype=np.float32)
        self.lib.orc_lio_tick_build_map(self.h, fptr(pb), len(pb), dptr(c64(state)))

    def tick_update_map(self, want_lists=False):
        """LIVMapper.cpp:413-424 after state_estimation(): UpdateVoxelMap with the posterior; optionally the lists it used."""
        if not want_lists:
            self.lib.orc_lio_tick_update_map(self.h, None, None)
            return None
        n = self._last_n
        pw, var = np.zeros((n, 3)), np.zeros((n, 9))
        self.lib.orc_lio_tick_update_map(self.h, dptr(pw), dptr(var))
        return pw, var

    def flatten(self):
        from fast_livo2_b200.synthetic import PLANE_DTYPE

        nr, npl = C.c_int(0), C.c_int(0)
        self.lib.orc_lio_flatten(self.h, C.byref(nr), C.byref(npl), None, None, None, None)
        keys = np.zeros((nr.value, 3), np.int64)
        first = np.zeros(nr.value, np.int32)
        count = np.zeros(nr.value, np.int32)
        planes = np.zeros(npl.value, PLANE_DTYPE)
        self.lib.orc_lio_flatten(self.h, C.byref(nr), C.byref(npl), _p(keys, C.c_int64), iptr(first), iptr(count), planes.ctypes.data)
        return dict(keys=keys, first=first, count=count, planes=planes)

    def dump_nodes(self):
        """Every octree node (see NODE_COLS), roots in key order, nodes in DFS pre-order."""
        return _dump_nodes(lambda out, cap: self.lib.orc_lio_dump_nodes(self.h, _p(out, C.c_int64), cap))

    def state_estimation(self, pts, state_in, state_prop):
        pts = np.ascontiguousarray(pts, dtype=np.float32)
        n = len(pts)
        self._last_n = n
        out = np.zeros(STATE_PACK)
        match = np.zeros(n, np.int32)
        normal = np.zeros(n, np.int32)
        dis = np.zeros(n, np.float32)
        stats = np.zeros(520)
        secs = self.lib.orc_lio_state_estimation(self.h, fptr(pts), n, dptr(c64(state_in)), dptr(c64(state_prop)), dptr(out), iptr(match),
                                                 iptr(normal), fptr(dis), dptr(stats), None, None)
        iters = int(stats[0])
        return dict(state=out, match_plane=match, normal_plane=normal, dis_to_plane=dis, iters=iters, M=stats[1:9].astype(int)[:iters],
                    total_residual=stats[9:17][:iters], HTH=stats[17:305].reshape(8, 6, 6)[:iters], HTz=stats[305:353].reshape(8, 6)[:iters],
                    solution=stats[353:505].reshape(8, 19)[:iters], converged=stats[505:513].astype(int)[:iters], secs=secs)

    def single_pass(self, pts, state_cur, state_prop):
        pts = np.ascontiguousarray(pts, dtype=np.float32)
        n = len(pts)
        plane = np.zeros(n, np.int32)
        dis = np.zeros(n, np.float32)
        H = np.zeros((n, 6))
        rinv = np.zeros(n)
        pw = np.zeros((n, 3))
        var = np.zeros((n, 3, 3))
        self.lib.orc_lio_single_pass(self.h, fptr(pts), n, dptr(c64(state_cur)), dptr(c64(state_prop)), iptr(plane), fptr(dis), dptr(H),
                                     dptr(rinv), dptr(pw), dptr(var))
        return dict(plane=plane, dis=dis, H=H, R_inv=rinv, point_w=pw, var=var)


class OracleVIO:
    def __init__(self, cam_cfg, ext, vio_cfg, threads=1, kind="parity"):
        self.lib = load(kind)
        self.cam, self.cfg = cam_cfg, vio_cfg
        self.h = self.lib.orc_vio_create(dptr(cam_cfg.as_array()), dptr(c64(ext.extR)), dptr(c64(ext.extT)), dptr(c64(ext.Rcl)),
                                         dptr(c64(ext.Pcl)), dptr(vio_cfg.as_array()), threads)

    def __del__(self):
        try:
            self.lib.orc_vio_destroy(self.h)
        except Exception:
            pass

    def update(self, img, pos, warp_patch, search_levels, inv_expo, state_in, state_prop):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        pos = c64(pos)
        n = len(pos)
        wp = np.ascontiguousarray(warp_patch, dtype=np.float32)
        sl = np.ascontiguousarray(search_levels, dtype=np.int32)
        ie = c64(inv_expo)
        out = np.zeros(STATE_PACK)
        err = np.zeros(n, np.float32)
        stats = np.zeros(4881)
        secs = self.lib.orc_vio_update(self.h, _p(img, C.c_uint8), n, dptr(pos), fptr(wp), iptr(sl), dptr(ie), dptr(c64(state_in)),
                                       dptr(c64(state_prop)), dptr(out), fptr(err), dptr(stats))
        return dict(state=out, errors=err, total_iters=int(stats[0]), iters_per_level=stats[1:9].astype(int),
                    accepted_per_level=stats[9:17].astype(int), error_trace=stats[17:81].reshape(8, 8),
                    HTH=stats[81:3217].reshape(8, 8, 7, 7), HTz=stats[3217:3665].reshape(8, 8, 7), solution=stats[3665:4881].reshape(8, 8, 19),
                    secs=secs)

    def set_inverse_refs(self, ref_imgs, ref_img_index, ref_px, ref_f, ref_R, ref_pos, ref_t=None):
        """Reference-feature data of the inverse-compositional variant (Feature::img_, px_, f_, T_f_w_ rotation, pos())."""
        self._ref_imgs = [np.ascontiguousarray(im, dtype=np.uint8) for im in ref_imgs]
        arr = (C.c_void_p * len(self._ref_imgs))(*[im.ctypes.data for im in self._ref_imgs])
        idx = np.ascontiguousarray(ref_img_index, dtype=np.int32)
        n = len(idx)
        self.lib.orc_vio_set_inverse_refs(self.h, arr, len(self._ref_imgs), n, iptr(idx), dptr(c64(ref_px)), dptr(c64(ref_f)),
                                          dptr(c64(np.asarray(ref_R).reshape(n, 9))), dptr(c64(ref_pos)))

    def set_inverse(self, enable):
        self.lib.orc_vio_set_inverse(self.h, int(bool(enable)))

    def precompute_reference_patches(self, pos, level):
        pos = c64(pos)
        n = len(pos)
        self.lib.orc_vio_precompute_reference_patches(self.h, n, dptr(pos), level)
        out = np.zeros(n * 64 * 6)
        got = self.lib.orc_vio_get_h_sub_inv(self.h, dptr(out), out.size)
        assert got == out.size
        return out.reshape(n, 64, 6)

    def get_image_patch(self, img, pc, level):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        out = np.zeros(64 * self.cfg.levels, np.float32)
        self.lib.orc_vio_get_image_patch(self.h, _p(img, C.c_uint8), dptr(c64(pc)), level, fptr(out))
        return out[64 * level: 64 * level + 64].copy()

    def warp_affine(self, img_ref, A_cur_ref, px_ref, search_level):
        img_ref = np.ascontiguousarray(img_ref, dtype=np.uint8)
        out = np.zeros(64 * self.cfg.levels, np.float32)
        self.lib.orc_vio_warp_affine(self.h, _p(img_ref, C.c_uint8), img_ref.shape[1], img_ref.shape[0], dptr(c64(A_cur_ref)), dptr(c64(px_ref)),
                                     int(search_level), fptr(out))
        return out

    def warp_matrix(self, px_ref, pos_w, normal_w, T_ref, T_cur):
        A = np.zeros(4)
        sl = self.lib.orc_vio_warp_matrix(self.h, dptr(c64(px_ref)), dptr(c64(pos_w)), dptr(c64(normal_w)), dptr(c64(T_ref[0])),
                                          dptr(c64(T_ref[1])), dptr(c64(T_cur[0])), dptr(c64(T_cur[1])), dptr(A))
        return A.reshape(2, 2), sl

    def world2cam(self, xyz):
        px = np.zeros(2)
        self.lib.orc_cam_world2cam(self.h, dptr(c64(xyz)), dptr(px))
        return px

    def cam2world(self, px):
        f = np.zeros(3)
        self.lib.orc_cam_cam2world(self.h, dptr(c64(px)), dptr(f))
        return f


def oracle_warp_patches(frame, state_for_cur_pose, threads=1):
    """Build the VIO inputs (A_cur_ref, search_level, warp_patch) with the oracle's
    getWarpMatrixAffineHomography / warpAffine. The 'current frame pose' used for the warp
    is the one implied by `state_for_cur_pose` (vio.cpp:1800 updateFrameState before retrieve)."""
    from fast_livo2_b200.synthetic import camera_pose, unpack_state

    vio = OracleVIO(frame["cam_cfg"], frame["ext"], frame["vio_cfg"], threads)
    st = unpack_state(state_for_cur_pose)
    T_cur = camera_pose(frame["ext"], st["R"], st["p"])
    n = len(frame["vis_pos"])
    L = frame["vio_cfg"].levels
    wp = np.zeros((n, L * 64), np.float32)
    sl = np.zeros(n, np.int32)
    A_all = np.zeros((n, 2, 2))
    for i in range(n):
        A, s = vio.warp_matrix(frame["px_ref"][i], frame["vis_pos"][i], frame["vis_normal"][i], frame["T_ref"], T_cur)
        A_all[i], sl[i] = A, s
        wp[i] = vio.warp_affine(frame["img_ref"], A, frame["px_ref"][i], s)
    return dict(warp_patch=wp, search_levels=sl, A_cur_ref=A_all)


def rot_err(Ra, Rb):
    v = np.zeros(3)
    load().orc_log(dptr(c64(Ra.T @ Rb)), dptr(v))
    return float(np.linalg.norm(v))


def inverse_refs_from_frame(fr):
    """Reference-feature arrays of the inverse-compositional variant for a synthetic frame (one reference frame):
    T_f_w_ = (Rcw_ref, Pcw_ref), pos() = -R^T t, f_ = unit bearing of the point in the reference camera."""
    R, t = fr["T_ref"]
    n = len(fr["vis_pos"])
    pc = fr["vis_pos"] @ R.T + t
    f = pc / np.linalg.norm(pc, axis=1, keepdims=True)
    return dict(ref_imgs=[fr["img_ref"]], ref_img_index=np.zeros(n, np.int32), ref_px=np.ascontiguousarray(fr["px_ref"], dtype=np.float64),
                ref_f=np.ascontiguousarray(f), ref_R=np.tile(R.reshape(1, 9), (n, 1)), ref_pos=np.tile(-R.T @ t, (n, 1)), ref_t=np.tile(t, (n, 1)))


# ---------------------------------------------------------------------------------------------------------------------
# oracle/_ref: the reference's own src/voxel_map.cpp compiled against stand-in headers (oracle/ref_voxel_map.cpp). Present
# only where it was built (the build container has /root/reference; the .so travels with the snapshot).
REF_LIO_SO = os.path.join(ORACLE_DIR, "_ref", "libfl2_ref_lio.so")


REF_LIO_DRIVER = "ref_lio_driver_version_2"  # oracle/ref_voxel_map.cpp's C API version the tests are written against
_ref_lio_ok = None


def ref_lio_available():
    """The reference-source library exists and was built from the current driver. A library built from an older driver (one
    that lacks the node dump, say) is not used live: the tests then compare with the stored outputs instead."""
    global _ref_lio_ok
    if _ref_lio_ok is None:
        _ref_lio_ok = os.path.exists(REF_LIO_SO) and hasattr(C.CDLL(REF_LIO_SO), REF_LIO_DRIVER)
    return _ref_lio_ok


def ref_lio_state_estimation(fr, state_in=None, state_prop=None, cfg=None, pts=None, so=None):
    """VoxelMapManager::StateEstimation of the REFERENCE SOURCE on a synthetic frame's flat map / scan."""
    lib = C.CDLL(so or REF_LIO_SO)
    cfg = cfg or fr["lio_cfg"]
    m = fr["map"]
    k, f, c, p = (np.ascontiguousarray(m["keys"], dtype=np.int64), np.ascontiguousarray(m["first"], dtype=np.int32), np.ascontiguousarray(m["count"], dtype=np.int32),
                  np.ascontiguousarray(m["planes"]))
    pts = np.ascontiguousarray(fr["pts"] if pts is None else pts, dtype=np.float32)
    n = len(pts)
    si = c64(fr["state_prior"] if state_in is None else state_in)
    sp = c64(fr["state_prior"] if state_prop is None else state_prop)
    cf = np.array([cfg.voxel_size, cfg.max_layer, cfg.max_iterations, cfg.sigma_num, cfg.dept_err, cfg.beam_err], dtype=np.float64)
    out = np.zeros(STATE_PACK)
    M = np.zeros(8, np.int32)
    iters, nptpl = C.c_int32(0), C.c_int32(0)
    normals = np.zeros((n, 3))
    centers = np.zeros((n, 3))
    dis = np.zeros(n, np.float32)
    pb = np.zeros((n, 3), np.float32)
    secs = C.c_double(0)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib.ref_lio_state_estimation(vp(k), vp(f), vp(c), len(f), vp(p), len(p), vp(cf), vp(c64(fr["ext"].extR)), vp(c64(fr["ext"].extT)), vp(pts), n, vp(si), vp(sp),
                                      vp(out), vp(M), C.byref(iters), vp(normals), C.byref(nptpl), vp(centers), vp(dis), vp(pb), C.byref(secs))
    assert rc == 0
    kk = nptpl.value
    return dict(state=out, iters=iters.value, M=M[:iters.value].copy(), normals=normals, ptpl_center=centers[:kk], ptpl_dis=dis[:kk], ptpl_point_b=pb[:kk], secs=secs.value)


class RefMap:
    """The REFERENCE SOURCE's map construction (VoxelMapManager::UpdateVoxelMap / UpdateOctoTree / init_plane of
    oracle/_ref/libfl2_ref_lio.so) fed with caller-supplied (point_w, var) lists, flattened like OracleLIO.flatten."""

    def __init__(self, cfg):
        self.lib = C.CDLL(REF_LIO_SO)
        self.lib.ref_map_create.restype = C.c_void_p
        self.lib.ref_map_create.argtypes = [C.c_void_p]
        self.lib.ref_map_destroy.argtypes = [C.c_void_p]
        self.lib.ref_map_update.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        self.lib.ref_map_flatten.argtypes = [C.c_void_p] * 7
        self.lib.ref_map_dump_nodes.restype = C.c_int
        self.lib.ref_map_dump_nodes.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        a = c64([cfg.voxel_size, cfg.max_layer, cfg.min_eigen_value, cfg.max_points_num] + layer_init_num8(cfg).tolist())
        self.h = self.lib.ref_map_create(a.ctypes.data)

    def __del__(self):
        try:
            self.lib.ref_map_destroy(self.h)
        except Exception:
            pass

    def update(self, pw, var):
        pw, var = c64(np.asarray(pw).reshape(-1, 3)), c64(np.asarray(var).reshape(-1, 9))
        self.lib.ref_map_update(self.h, pw.ctypes.data, var.ctypes.data, len(pw))

    def build(self, pts_body_f32, state, ext, cfg):
        """First LiDAR frame: TransformLidar + BuildVoxelMap of the reference source (LIVMapper.cpp:356-366)."""
        self.lib.ref_map_build.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_double]
        pb, st, R, t = np.ascontiguousarray(pts_body_f32, dtype=np.float32), c64(state), c64(ext.extR), c64(ext.extT)
        self.lib.ref_map_build(self.h, pb.ctypes.data, len(pb), st.ctypes.data, R.ctypes.data, t.ctypes.data, float(cfg.dept_err), float(cfg.beam_err))

    def flatten(self):
        from fast_livo2_b200.synthetic import PLANE_DTYPE

        nr, npl = C.c_int(0), C.c_int(0)
        self.lib.ref_map_flatten(self.h, C.addressof(nr), C.addressof(npl), None, None, None, None)
        keys, first, count = np.zeros((nr.value, 3), np.int64), np.zeros(nr.value, np.int32), np.zeros(nr.value, np.int32)
        planes = np.zeros(npl.value, PLANE_DTYPE)
        self.lib.ref_map_flatten(self.h, C.addressof(nr), C.addressof(npl), keys.ctypes.data, first.ctypes.data, count.ctypes.data, planes.ctypes.data)
        return dict(keys=keys, first=first, count=count, planes=planes)

    def dump_nodes(self):
        return _dump_nodes(lambda out, cap: self.lib.ref_map_dump_nodes(self.h, out.ctypes.data, cap))

    def clear_out_of_map(self, lo, hi):
        self.lib.ref_map_clear_out_of_map(C.c_void_p(self.h), int(hi[0]), int(lo[0]), int(hi[1]), int(lo[1]), int(hi[2]), int(lo[2]))


# ---------------------------------------------------------------------------------------------------------------------
# oracle/_ref/libfl2_ref_vio.so: the reference's own src/vio.cpp (+ frame.cpp, visual_point.cpp) compiled against stand-in
# headers (oracle/ref_vio.cpp). vikit's pinhole model and interpolateMat_8u are restatements (un-vendored dependency).
REF_VIO_SO = os.path.join(ORACLE_DIR, "_ref", "libfl2_ref_vio.so")


REF_VIO_DRIVER = "ref_vio_driver_version_2"  # oracle/ref_vio.cpp + stand-in headers the tests are written against
_ref_vio_ok = None


def ref_vio_available():
    """The reference-source VIO library exists and was built at the current version. An older build (whose stand-in inverted
    2 x 2 matrices by LU, not by Eigen's closed form) is not used live: the tests then compare with the stored outputs."""
    global _ref_vio_ok
    if _ref_vio_ok is None:
        _ref_vio_ok = os.path.exists(REF_VIO_SO) and hasattr(C.CDLL(REF_VIO_SO), REF_VIO_DRIVER)
    return _ref_vio_ok


class RefVIO:
    """VIOManager of the REFERENCE SOURCE (pinhole camera only)."""

    def __init__(self, cam_cfg, ext, vio_cfg, so=None):
        self.lib = C.CDLL(so or REF_VIO_SO)
        L = self.lib
        L.ref_vio_create.restype = C.c_void_p
        L.ref_vio_create.argtypes = [C.c_void_p] * 6
        L.ref_vio_destroy.argtypes = [C.c_void_p]
        L.ref_vio_update.restype = C.c_double
        L.ref_vio_update.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 10
        L.ref_vio_update_inverse.restype = C.c_double
        L.ref_vio_update_inverse.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 5 + [C.c_int] + [C.c_void_p] * 9
        L.ref_vio_get_image_patch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.ref_vio_warp_affine.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.ref_vio_warp_matrix.restype = C.c_int
        L.ref_vio_warp_matrix.argtypes = [C.c_void_p] * 9
        self.cam, self.cfg = cam_cfg, vio_cfg
        a = lambda x: c64(x).ctypes.data
        self._keep = [c64(cam_cfg.as_array()), c64(ext.extR), c64(ext.extT), c64(ext.Rcl), c64(ext.Pcl), c64(vio_cfg.as_array())]
        self.h = L.ref_vio_create(*[k.ctypes.data for k in self._keep])
        assert self.h, "ref_vio_create failed (only the pinhole model is available in the stand-in vikit)"

    def __del__(self):
        try:
            self.lib.ref_vio_destroy(self.h)
        except Exception:
            pass

    def update(self, img, pos, warp_patch, search_levels, inv_expo, state_in, state_prop):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        pos, wp = c64(pos), np.ascontiguousarray(warp_patch, dtype=np.float32)
        sl, ie = np.ascontiguousarray(search_levels, dtype=np.int32), c64(inv_expo)
        n = len(pos)
        out, err, G, HTH = np.zeros(STATE_PACK), np.zeros(n, np.float32), np.zeros((19, 19)), np.zeros((19, 19))
        si, sp = c64(state_in), c64(state_prop)
        secs = self.lib.ref_vio_update(self.h, img.ctypes.data, n, pos.ctypes.data, wp.ctypes.data, sl.ctypes.data, ie.ctypes.data, si.ctypes.data, sp.ctypes.data,
                                       out.ctypes.data, err.ctypes.data, G.ctypes.data, HTH.ctypes.data)
        return dict(state=out, errors=err, G=G, H_T_H=HTH, secs=secs)

    def update_inverse(self, img, pos, warp_patch, search_levels, inv_expo, refs, state_in, state_prop):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        pos, wp = c64(pos), np.ascontiguousarray(warp_patch, dtype=np.float32)
        sl, ie = np.ascontiguousarray(search_levels, dtype=np.int32), c64(inv_expo)
        n = len(pos)
        imgs = [np.ascontiguousarray(im, dtype=np.uint8) for im in refs["ref_imgs"]]
        arr = (C.c_void_p * len(imgs))(*[im.ctypes.data for im in imgs])
        idx = np.ascontiguousarray(refs["ref_img_index"], dtype=np.int32)
        # the reference's Feature holds T_f_w_ = (R, t); pos() is derived from it. ref_t, when present, is that t; else t = -R pos
        R = c64(np.asarray(refs["ref_R"]).reshape(n, 9))
        t = refs["ref_t"] if "ref_t" in refs else -np.einsum("nij,nj->ni", R.reshape(n, 3, 3), np.asarray(refs["ref_pos"]))
        px, f, rp = c64(refs["ref_px"]), c64(refs["ref_f"]), c64(t)
        out, err = np.zeros(STATE_PACK), np.zeros(n, np.float32)
        si, sp = c64(state_in), c64(state_prop)
        self.lib.ref_vio_update_inverse(self.h, img.ctypes.data, n, pos.ctypes.data, wp.ctypes.data, sl.ctypes.data, ie.ctypes.data, C.cast(arr, C.c_void_p), len(imgs),
                                        idx.ctypes.data, px.ctypes.data, f.ctypes.data, R.ctypes.data, rp.ctypes.data, si.ctypes.data, sp.ctypes.data, out.ctypes.data,
                                        err.ctypes.data)
        return dict(state=out, errors=err)

    def get_image_patch(self, img, pc, level):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        out = np.zeros(64 * self.cfg.levels, np.float32)
        pc = c64(pc)
        self.lib.ref_vio_get_image_patch(self.h, img.ctypes.data, pc.ctypes.data, level, out.ctypes.data)
        return out[64 * level: 64 * level + 64].copy()

    def warp_affine(self, img_ref, A_cur_ref, px_ref, search_level):
        img_ref = np.ascontiguousarray(img_ref, dtype=np.uint8)
        out = np.zeros(64 * self.cfg.levels, np.float32)
        A, px = c64(A_cur_ref), c64(px_ref)
        for lvl in range(self.cfg.levels):  # retrieveFromVisualSparseMap loops the pyramid levels (vio.cpp:739-742)
            self.lib.ref_vio_warp_affine(self.h, img_ref.ctypes.data, img_ref.shape[1], img_ref.shape[0], A.ctypes.data, px.ctypes.data, int(search_level), lvl, out.ctypes.data)
        return out

    def warp_matrix(self, px_ref, pos_w, normal_w, T_ref, T_cur):
        A = np.zeros(4)
        args = [c64(px_ref), c64(pos_w), c64(normal_w), c64(T_ref[0]), c64(T_ref[1]), c64(T_cur[0]), c64(T_cur[1])]
        sl = self.lib.ref_vio_warp_matrix(self.h, *[x.ctypes.data for x in args], A.ctypes.data)
        return A.reshape(2, 2), sl


# ---------------------------------------------------------------------------------------------------------------------
# Stored outputs of the reference source, so that the tests that compare the oracle with it run on every checkout.
# Where oracle/_ref is built the tests call the reference live; FL2_RECORD_REF_PIN=1 then rewrites tests/golden/ref_pin/.
# Elsewhere they compare with what was stored. Exact (bit-for-bit) comparisons of arrays above 4 KB are stored as a
# SHA-256 of the array, which asserts the same equality; values compared with a tolerance are stored in full.
REF_PIN_DIR = os.path.join(ROOT, "tests", "golden", "ref_pin")


def digest(a):
    a = np.ascontiguousarray(a)
    h = __import__("hashlib").sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


class RefPin:
    """The reference source's outputs for one test, by key: live (and optionally recorded) where the libraries are built,
    else read from tests/golden/ref_pin/<name>.npz."""

    def __init__(self, name):
        self.path = os.path.join(REF_PIN_DIR, f"{name}.npz")
        self.live = ref_lio_available() and ref_vio_available()
        self.record = self.live and os.environ.get("FL2_RECORD_REF_PIN") == "1"
        # recording merges into what is stored: re-recording some cases (pytest -k) keeps the others' outputs
        self.store = dict(np.load(self.path, allow_pickle=False)) if (self.record and os.path.exists(self.path)) else {}
        self.stored = dict(np.load(self.path, allow_pickle=False)) if (not self.live and os.path.exists(self.path)) else {}

    @staticmethod
    def available(name):
        return (ref_lio_available() and ref_vio_available()) or os.path.exists(os.path.join(REF_PIN_DIR, f"{name}.npz"))

    def get(self, key, compute, exact=()):
        """compute() -> dict of arrays. Keys listed in `exact` are compared bit for bit by the caller (see same())."""
        if self.live:
            out = compute()
            if self.record:
                for k in [k for k in self.store if k.startswith(key + "/")]:
                    del self.store[k]  # this key's previous outputs, replaced as a whole
                for k, v in out.items():
                    v = np.asarray(v)
                    if k in exact and v.nbytes > 4096:
                        self.store[f"{key}/{k}#sha256"] = np.array(digest(v))
                    else:
                        self.store[f"{key}/{k}"] = v
                np.savez_compressed(self.path, **self.store)
            return out
        pre = key + "/"
        out = {}
        for k, v in self.stored.items():
            if k.startswith(pre):
                out[k[len(pre):]] = str(v) if k.endswith("#sha256") else v
        assert out, f"{self.path} holds no outputs for {key!r}: regenerate with FL2_RECORD_REF_PIN=1 where oracle/_ref is built"
        return out


def same(a, ref, k):
    """Bit-for-bit equality of `a` with ref[k], or with the stored digest of ref[k]."""
    if k + "#sha256" in ref:
        return digest(a) == ref[k + "#sha256"]
    return np.array_equal(a, ref[k])


def flat_map_sample(flat, n_roots=24, seed=0):
    """A fixed seeded sample of a flattened map's root voxels that hold planes, with those planes, plus digests of the whole key
    set and of the candidate count of every root (in key order)."""
    order = np.lexsort(flat["keys"].T[::-1])
    keys, count = flat["keys"][order], flat["count"][order]
    with_planes = order[count > 0]  # roots without a candidate plane are covered by the count digest
    pick = np.sort(np.random.default_rng(seed).choice(len(with_planes), size=min(n_roots, len(with_planes)), replace=False))
    sel = with_planes[pick]
    planes = np.concatenate([flat["planes"][f:f + c] for f, c in zip(flat["first"][sel], flat["count"][sel])])
    first = np.concatenate([[0], np.cumsum(flat["count"][sel])[:-1]]).astype(np.int32)
    return dict(keys=flat["keys"][sel], first=first, count=flat["count"][sel].astype(np.int32), planes=planes,
                all_keys_sha=np.array(digest(keys.astype(np.int64))), all_counts_sha=np.array(digest(count.astype(np.int32))))


def flat_map_subset(flat, keys):
    """The roots `keys` of a flattened map (in that order) with their candidate planes."""
    where = {tuple(k): i for i, k in enumerate(flat["keys"].tolist())}
    sel = np.array([where[tuple(k)] for k in np.asarray(keys).tolist()], np.int64)
    planes = np.concatenate([flat["planes"][f:f + c] for f, c in zip(flat["first"][sel], flat["count"][sel])])
    first = np.concatenate([[0], np.cumsum(flat["count"][sel])[:-1]]).astype(np.int32)
    return dict(keys=flat["keys"][sel], first=first, count=flat["count"][sel].astype(np.int32), planes=planes)


def compare_with_map_sample(MB, flat, sample, rtol, what):
    """compare_flat_maps of `flat` against a flat_map_sample of the other side: the same key set and counts (digests), and
    the sampled roots' planes within rtol. Returns the number of planes compared."""
    order = np.lexsort(flat["keys"].T[::-1])
    assert digest(flat["keys"][order].astype(np.int64)) == str(sample["all_keys_sha"]), f"root voxels differ between {what[0]} and {what[1]}"
    assert digest(flat["count"][order].astype(np.int32)) == str(sample["all_counts_sha"]), "candidate counts per root differ"
    sub = {k: sample[k] for k in ("keys", "first", "count", "planes")}
    MB.compare_flat_maps(flat_map_subset(flat, sub["keys"]), sub, rtol=rtol, what=what)
    return int(flat["count"].sum())
