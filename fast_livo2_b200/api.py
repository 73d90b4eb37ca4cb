"""ctypes binding of the C ABI in include/esikf_b200.h (libesikf_b200.so).

This is plumbing for tests and bench.py — the product is the CUDA library. There is no CPU
fallback: importing works anywhere, but creating a context without the compiled library or
without an sm_90 device raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ESIKF_LIB") or os.path.join(_HERE, "libesikf_b200.so")  # ESIKF_LIB: A/B builds of the same sources (measurement)
STATE_DOUBLES = 386


class EsikfError(RuntimeError):
    pass


class LioCfgC(C.Structure):
    _fields_ = [("voxel_size", C.c_double), ("sigma_num", C.c_double), ("dept_err", C.c_double), ("beam_err", C.c_double),
                ("max_layer", C.c_int32), ("max_iterations", C.c_int32)]


class ExtrinsicsC(C.Structure):
    _fields_ = [("extR", C.c_double * 9), ("extT", C.c_double * 3), ("Rcl", C.c_double * 9), ("Pcl", C.c_double * 3)]


class CameraC(C.Structure):
    _fields_ = [("model", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("pad_", C.c_int32), ("fx", C.c_double),
                ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double), ("d", C.c_double * 5)]


class VioCfgC(C.Structure):
    _fields_ = [("img_point_cov", C.c_double), ("patch_pyrimid_level", C.c_int32), ("max_iterations", C.c_int32),
                ("exposure_estimate_en", C.c_int32), ("inverse_composition_en", C.c_int32)]


class VioSelectCfgC(C.Structure):
    _fields_ = [("normal_en", C.c_int32), ("ncc_en", C.c_int32), ("ncc_thre", C.c_double), ("outlier_threshold", C.c_double)]


class LioStatsC(C.Structure):
    _fields_ = [("iters", C.c_int32), ("effct_feat_num", C.c_int32 * 8), ("converged", C.c_int32 * 8), ("pad_", C.c_int32),
                ("total_residual", C.c_double * 8), ("HTH", C.c_double * (8 * 36)), ("HTz", C.c_double * (8 * 6)),
                ("solution", C.c_double * (8 * 19))]


class VioStatsC(C.Structure):
    _fields_ = [("total_iters", C.c_int32), ("iters_per_level", C.c_int32 * 8), ("accepted_per_level", C.c_int32 * 8),
                ("pad_", C.c_int32), ("error_trace", C.c_float * 64), ("HTH", C.c_double * (64 * 49)), ("HTz", C.c_double * (64 * 7)),
                ("solution", C.c_double * (64 * 19))]


_lib = None


def load_library():
    """Load libesikf_b200.so; raises EsikfError if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EsikfError(f"{LIB_PATH} is missing — run __graft_entry__.build() (nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, dp, fp, ip, i64p, u8p = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(
        C.c_int64), C.POINTER(C.c_uint8)
    lib.esikf_create.argtypes = [C.POINTER(vp), C.c_int]
    lib.esikf_destroy.argtypes = [vp]
    lib.esikf_last_error.argtypes = [vp]
    lib.esikf_last_error.restype = C.c_char_p
    lib.esikf_stream.argtypes = [vp]
    lib.esikf_stream.restype = vp
    lib.esikf_synchronize.argtypes = [vp]
    lib.esikf_launch_count.argtypes = [vp]
    lib.esikf_launch_count.restype = C.c_int64
    lib.esikf_set_solve_mode.argtypes = [vp, C.c_int]
    lib.esikf_set_loop_mode.argtypes = [vp, C.c_int]
    lib.esikf_set_tuning.argtypes = [vp, C.c_uint32]
    lib.esikf_set_extrinsics.argtypes = [vp, C.POINTER(ExtrinsicsC)]
    lib.esikf_set_lidar_extrinsics.argtypes = [vp, dp, dp]
    lib.esikf_map_upload.argtypes = [vp, i64p, ip, ip, C.c_int32, vp, C.c_int32, C.c_double]
    lib.esikf_map_patch.argtypes = [vp, ip, vp, C.c_int32]
    lib.esikf_map_device_init.argtypes = [vp, vp]
    lib.esikf_map_device_build.argtypes = [vp, vp]
    lib.esikf_map_device_update.argtypes = [vp, vp]
    lib.esikf_map_device_update_points.argtypes = [vp, vp, vp, C.c_int32]
    lib.esikf_map_device_stats.argtypes = [vp, vp]
    lib.esikf_map_device_capacity.argtypes = [vp, vp]
    lib.esikf_map_device_slide.argtypes = [vp, vp, vp]
    lib.esikf_map_device_download.argtypes = [vp, vp, vp, vp, C.c_int32, vp, C.c_int32, vp, vp]
    lib.esikf_map_device_export.argtypes = [vp, vp, vp, vp, C.c_int32, vp, C.c_int32, vp, vp]
    lib.esikf_map_device_find.argtypes = [vp, vp, C.c_int32, C.c_int32, vp, vp, vp]
    lib.esikf_lio_fetch_normals.argtypes = [vp, vp]
    lib.esikf_lio_set_scan.argtypes = [vp, vp, C.c_int32]
    lib.esikf_lio_run.argtypes = [vp, vp, vp, C.POINTER(LioCfgC)]
    lib.esikf_lio_fetch.argtypes = [vp, vp, C.POINTER(LioStatsC), vp, vp, vp]
    lib.esikf_lio_update.argtypes = [vp, vp, C.c_int32, vp, vp, C.POINTER(LioCfgC), vp, C.POINTER(LioStatsC), vp, vp, vp]
    lib.esikf_lio_fetch_point_cov.argtypes = [vp, vp, vp]
    lib.esikf_vio_set_camera.argtypes = [vp, C.POINTER(CameraC), C.POINTER(VioCfgC)]
    lib.esikf_vio_set_image.argtypes = [vp, vp, C.c_int32, C.c_int32]
    lib.esikf_vio_set_patches.argtypes = [vp, vp, vp, vp, vp, C.c_int32]
    lib.esikf_vio_run.argtypes = [vp, vp, vp]
    lib.esikf_vio_fetch.argtypes = [vp, vp, C.POINTER(VioStatsC), vp]
    lib.esikf_vio_update.argtypes = [vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, C.c_int32, vp, vp, vp, C.POINTER(VioStatsC), vp]
    lib.esikf_vio_get_image_patch.argtypes = [vp, vp, C.c_int32, C.c_int32, vp]
    lib.esikf_vio_set_ref_images.argtypes = [vp, C.POINTER(vp), C.c_int32, C.c_int32, C.c_int32]
    lib.esikf_vio_warp_patches.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int32]
    lib.esikf_vio_warp_affine.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp]
    lib.esikf_vio_set_inverse_refs.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp]
    lib.esikf_vio_select_patches.argtypes = [vp, C.c_int32] + [vp] * 12 + [C.c_double, C.POINTER(VioSelectCfgC), ip, vp, vp, vp, vp, vp]
    lib.esikf_rgb_set_cloud.argtypes = [vp, vp, C.c_int32, vp]
    lib.esikf_rgb_colorize.argtypes = [vp, vp, C.c_int32, C.c_int32, vp, C.c_double, C.c_int32, ip, vp, vp, vp]
    lib.esikf_vio_generate_points.argtypes = [vp, vp, vp, vp, C.c_int32, vp, vp, C.c_int32, vp] + [C.c_int32] * 5 + [vp, C.c_int32, ip] + [vp] * 8
    lib.esikf_vio_update_points.argtypes = [vp, C.c_int32, vp, vp, vp, vp, C.c_int32, ip, vp, vp, vp, vp]
    lib.esikf_vio_retrieve_scan.argtypes = [vp, vp, C.c_int32, C.c_int32, vp, C.c_int32, ip, vp, vp]
    lib.esikf_vio_depth_check.argtypes = [vp, C.c_int32, vp, vp, vp]
    lib.esikf_vio_score_ref_patches.argtypes = [vp, C.c_int32, vp, C.c_int32] + [vp] * 9
    lib.esikf_vmap_init.argtypes = [vp, C.c_int64]
    lib.esikf_vmap_add_points.argtypes = [vp, C.c_int32, vp, C.c_int32] + [vp] * 8
    lib.esikf_vmap_update_points.argtypes = [vp, C.c_int32, vp, vp, vp, C.c_int32, vp, C.c_int32, ip] + [vp] * 6
    lib.esikf_vmap_score.argtypes = [vp, C.c_int32] + [vp] * 6
    lib.esikf_vmap_choose_ref.argtypes = [vp, C.c_int32, vp, vp, vp, C.c_int32, vp]
    lib.esikf_vmap_download.argtypes = [vp, C.c_int32, vp, C.c_int32] + [vp] * 8
    lib.esikf_vmap_stats.argtypes = [vp, vp, vp]
    lib.esikf_vmap_place_points.argtypes = [vp, C.c_int32, vp, vp, vp]
    lib.esikf_vmap_retrieve.argtypes = [vp, C.c_int32, vp] + [C.c_int32] * 6 + [ip] + [vp] * 5
    lib.esikf_comm_unique_id.argtypes = [C.c_char_p]
    lib.esikf_comm_init.argtypes = [vp, C.c_int32, C.c_int32, C.c_char_p]
    lib.esikf_comm_rank.argtypes = [vp, ip, ip]
    lib.esikf_peer_export.argtypes = [vp, C.c_char_p]
    lib.esikf_peer_attach.argtypes = [vp, C.c_int32, C.c_int32, C.c_char_p]
    lib.esikf_shard_range.argtypes = [C.c_int32, C.c_int32, C.c_int32, ip, ip]
    lib.esikf_profile_kernel.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, fp]
    lib.esikf_set_kernel_timing.argtypes = [vp, C.c_int32]
    lib.esikf_set_phase_stamps.argtypes = [vp, C.c_int32]
    lib.esikf_get_phase_stamps.argtypes = [vp, C.POINTER(C.c_uint64)]
    lib.esikf_get_vio_chain_stamps.argtypes = [vp, C.POINTER(C.c_uint64)]
    lib.esikf_get_kernel_timing.argtypes = [vp, fp, fp, fp, fp]
    _lib = lib
    return lib


TUNE_STAGE_LDG = 1
TUNE_VIO_TMA = 2  # esikf_set_tuning flag: stage LIO plane records with __ldg copies instead of cp.async.bulk (measurement variant)
GEN_ADD_FROM = 0x40000000  # esikf_vio_generate_points: the source of a winner from the add_from list
FIND_RULE_PATCH, FIND_RULE_RAYCAST = 0, 1  # esikf_map_device_find: updateReferencePatch's key, the ray casting's key
FIND_NO_ROOT, FIND_NODE, FIND_PLANE = 0, 1, 2  # esikf_map_device_find's status per point
# esikf_vmap_retrieve's status per cell: kept, depth-discontinuous, not normal-initialised, no reference feature, no winner
RETRIEVE_KEPT, RETRIEVE_DEPTH, RETRIEVE_NOT_INIT, RETRIEVE_NO_REF, RETRIEVE_NO_WINNER = 0, 1, 2, 3, 4
# esikf_get_vio_chain_stamps (csrc/esikf_fused.cu): 8 words per (level, iteration) slot, then from VIO_CHAIN_CTA on
# VIO_CHAIN_MAX_CTAS words per slot, one per CTA
VIO_CHAIN_CTA, VIO_CHAIN_MAX_CTAS = 8 * 64, 160
VIO_CHAIN_STAMP_WORDS = VIO_CHAIN_CTA + VIO_CHAIN_MAX_CTAS * 64  # ESIKF_VIO_CHAIN_STAMP_WORDS
DEFAULT_LOOP_MODE = 2  # esikf_set_loop_mode: 2 (alias 1) persistent kernel per update, 0 per-iteration launches

class MapCfgC(C.Structure):
    _fields_ = [("voxel_size", C.c_double), ("min_eigen_value", C.c_double), ("dept_err", C.c_double), ("beam_err", C.c_double), ("max_layer", C.c_int32),
                ("max_points_num", C.c_int32), ("layer_init_num", C.c_int32 * 8), ("grow", C.c_int32), ("root_capacity", C.c_int64), ("node_capacity", C.c_int64),
                ("record_capacity", C.c_int64), ("point_capacity", C.c_int64)]


class MapStatsC(C.Structure):
    _fields_ = [("roots", C.c_int32), ("nodes", C.c_int32), ("records", C.c_int32), ("touched_roots", C.c_int32), ("errors", C.c_int32), ("pad", C.c_int32),
                ("pool_points", C.c_int64)]


EXPORTED_SYMBOLS = [
    "esikf_create", "esikf_destroy", "esikf_last_error", "esikf_stream", "esikf_synchronize", "esikf_host_alloc", "esikf_host_free", "esikf_launch_count", "esikf_set_solve_mode", "esikf_set_loop_mode", "esikf_set_tuning",
    "esikf_set_extrinsics", "esikf_set_lidar_extrinsics", "esikf_map_upload", "esikf_map_patch", "esikf_map_device_init", "esikf_map_device_build", "esikf_map_device_update", "esikf_map_device_update_points", "esikf_map_device_slide", "esikf_map_device_stats", "esikf_map_device_capacity", "esikf_map_device_download", "esikf_map_device_export", "esikf_map_device_find", "esikf_lio_fetch_normals", "esikf_lio_set_scan", "esikf_lio_run", "esikf_lio_fetch",
    "esikf_lio_update", "esikf_lio_fetch_point_cov", "esikf_vio_set_camera", "esikf_vio_set_image", "esikf_vio_set_patches",
    "esikf_vio_run", "esikf_vio_fetch", "esikf_vio_update", "esikf_vio_get_image_patch", "esikf_vio_set_ref_images",
    "esikf_vio_warp_patches", "esikf_vio_select_patches", "esikf_vio_warp_affine", "esikf_vio_set_inverse_refs", "esikf_rgb_set_cloud", "esikf_rgb_colorize", "esikf_vio_generate_points", "esikf_vio_update_points", "esikf_vio_retrieve_scan", "esikf_vio_depth_check", "esikf_vio_score_ref_patches",
    "esikf_vmap_init", "esikf_vmap_add_points", "esikf_vmap_update_points", "esikf_vmap_score", "esikf_vmap_choose_ref", "esikf_vmap_download", "esikf_vmap_stats", "esikf_vmap_place_points", "esikf_vmap_retrieve", "esikf_comm_unique_id", "esikf_comm_init", "esikf_comm_rank", "esikf_shard_range", "esikf_peer_export", "esikf_peer_attach", "esikf_profile_kernel", "esikf_set_kernel_timing", "esikf_get_kernel_timing", "esikf_set_phase_stamps", "esikf_get_phase_stamps",
    "esikf_get_vio_chain_stamps",
]


def _addr(a):
    """Raw address of a numpy array or torch tensor (host memory)."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()  # torch tensor (pinned host memory in bench.py)


def _c(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def lio_cfg_c(cfg) -> LioCfgC:
    return LioCfgC(cfg.voxel_size, cfg.sigma_num, cfg.dept_err, cfg.beam_err, cfg.max_layer, cfg.max_iterations)


class Context:
    """One ESIKF context = one CUDA device + stream (one process per GPU)."""

    def __init__(self, device: int = 0):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.esikf_create(C.byref(h), device)
        if rc != 0:
            raise EsikfError(f"esikf_create(device={device}) failed with status {rc} (no sm_90 CUDA device?) — no CPU fallback")
        self.h = h
        self.n_pts = 0
        self.n_patches = 0
        self.levels = 4
        self._rgb_n = 0  # points of the last rgb_set_cloud

    def close(self):
        if getattr(self, "h", None):
            self.lib.esikf_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise EsikfError(f"status {rc}: {self.lib.esikf_last_error(self.h).decode()}")

    @property
    def stream(self):
        return self.lib.esikf_stream(self.h)

    def synchronize(self):
        self._ck(self.lib.esikf_synchronize(self.h))

    def launch_count(self):
        return int(self.lib.esikf_launch_count(self.h))

    def set_solve_mode(self, mode):
        self._ck(self.lib.esikf_set_solve_mode(self.h, mode))

    def set_loop_mode(self, mode):
        self._ck(self.lib.esikf_set_loop_mode(self.h, mode))

    def set_tuning(self, flags):
        """OR of the TUNE_* measurement variants; 0 = none."""
        self._ck(self.lib.esikf_set_tuning(self.h, flags))

    def set_extrinsics(self, ext):
        e = ExtrinsicsC()
        e.extR[:] = _c(ext.extR, np.float64).reshape(9)
        e.extT[:] = _c(ext.extT, np.float64)
        e.Rcl[:] = _c(ext.Rcl, np.float64).reshape(9)
        e.Pcl[:] = _c(ext.Pcl, np.float64)
        self._ck(self.lib.esikf_set_extrinsics(self.h, C.byref(e)))

    def set_lidar_extrinsics(self, extR, extT):
        """Only the lidar -> IMU part; the camera part set before is kept (Rcl = I, Pcl = 0 if none was)."""
        R, t = _c(extR, np.float64).reshape(9), _c(extT, np.float64).reshape(3)
        self._ck(self.lib.esikf_set_lidar_extrinsics(self.h, R.ctypes.data_as(C.POINTER(C.c_double)), t.ctypes.data_as(C.POINTER(C.c_double))))

    # ------------------------------------------------------------------ map
    def map_upload(self, vmap, voxel_size):
        k, f, c, p = _c(vmap["keys"], np.int64), _c(vmap["first"], np.int32), _c(vmap["count"], np.int32), np.ascontiguousarray(vmap["planes"])
        assert p.dtype.itemsize == 256
        self._ck(self.lib.esikf_map_upload(self.h, k.ctypes.data_as(C.POINTER(C.c_int64)), f.ctypes.data_as(C.POINTER(C.c_int32)),
                                           c.ctypes.data_as(C.POINTER(C.c_int32)), len(f), p.ctypes.data, len(p), float(voxel_size)))

    def map_patch(self, ids, planes):
        ids = _c(ids, np.int32)
        planes = np.ascontiguousarray(planes)
        self._ck(self.lib.esikf_map_patch(self.h, ids.ctypes.data_as(C.POINTER(C.c_int32)), planes.ctypes.data, len(ids)))

    # ------------------------------------------------------------------ device-resident map
    def map_device_init(self, cfg, root_capacity=0, node_capacity=0, record_capacity=0, point_capacity=0, grow=False):
        """cfg: synthetic.LioCfg (voxel_size, min_eigen_value, dept_err, beam_err, max_layer, max_points_num, layer_init_num).
        grow: the capacities are starting sizes and the map grows when a tick would exceed one (else they are fixed)."""
        m = MapCfgC()
        m.voxel_size, m.min_eigen_value, m.dept_err, m.beam_err = cfg.voxel_size, cfg.min_eigen_value, cfg.dept_err, cfg.beam_err
        m.max_layer, m.max_points_num = cfg.max_layer, cfg.max_points_num
        for k in range(8):
            m.layer_init_num[k] = cfg.layer_init_num[min(k, len(cfg.layer_init_num) - 1)]
        m.root_capacity, m.node_capacity, m.record_capacity, m.point_capacity = root_capacity, node_capacity, record_capacity, point_capacity
        m.grow = 1 if grow else 0
        self._ck(self.lib.esikf_map_device_init(self.h, C.byref(m)))

    def map_device_capacity(self):
        """The device map's current capacities (root_capacity = hash slots / 2) and whether it grows."""
        m = MapCfgC()
        self._ck(self.lib.esikf_map_device_capacity(self.h, C.byref(m)))
        return dict(root_capacity=m.root_capacity, node_capacity=m.node_capacity, record_capacity=m.record_capacity, point_capacity=m.point_capacity,
                    grow=bool(m.grow))

    def map_device_build(self, state):
        self._ck(self.lib.esikf_map_device_build(self.h, _c(state, np.float64).ctypes.data))

    def map_device_update(self, state=None):
        self._ck(self.lib.esikf_map_device_update(self.h, None if state is None else _c(state, np.float64).ctypes.data))

    def map_device_update_points(self, point_w, var):
        pw, v = _c(point_w, np.float64).reshape(-1, 3), _c(var, np.float64).reshape(-1, 9)
        self._ck(self.lib.esikf_map_device_update_points(self.h, pw.ctypes.data, v.ctypes.data, len(pw)))

    def map_device_slide(self, key_min=None, key_max=None):
        lo = None if key_min is None else _c(key_min, np.int64)
        hi = None if key_max is None else _c(key_max, np.int64)
        self._ck(self.lib.esikf_map_device_slide(self.h, None if lo is None else lo.ctypes.data, None if hi is None else hi.ctypes.data))

    def map_device_stats(self):
        st = MapStatsC()
        self._ck(self.lib.esikf_map_device_stats(self.h, C.byref(st)))
        return {f: getattr(st, f) for f, _ in MapStatsC._fields_ if f != "pad"}

    def map_device_download(self):
        from .synthetic import PLANE_DTYPE

        nr, npl = C.c_int32(0), C.c_int32(0)
        self._ck(self.lib.esikf_map_device_download(self.h, None, None, None, 0, None, 0, C.byref(nr), C.byref(npl)))
        keys, first, count = np.zeros((max(nr.value, 1), 3), np.int64), np.zeros(max(nr.value, 1), np.int32), np.zeros(max(nr.value, 1), np.int32)
        planes = np.zeros(max(npl.value, 1), PLANE_DTYPE)
        self._ck(self.lib.esikf_map_device_download(self.h, keys.ctypes.data, first.ctypes.data, count.ctypes.data, len(first), planes.ctypes.data, len(planes),
                                                    C.byref(nr), C.byref(npl)))
        return dict(keys=keys[:nr.value], first=first[:nr.value], count=count[:nr.value], planes=planes[:npl.value])

    def map_device_export(self):
        """The subtrees of the roots the last build / update replayed: root r owns nodes[first[r]:first[r] + count[r]]
        (synthetic.NODE_DTYPE, DFS pre-order, leaves 0..7); roots in hash-slot order."""
        from .synthetic import NODE_DTYPE

        nr, nn = C.c_int32(0), C.c_int32(0)
        self._ck(self.lib.esikf_map_device_export(self.h, None, None, None, 0, None, 0, C.byref(nr), C.byref(nn)))
        keys, first, count = np.zeros((max(nr.value, 1), 3), np.int64), np.zeros(max(nr.value, 1), np.int32), np.zeros(max(nr.value, 1), np.int32)
        nodes = np.zeros(max(nn.value, 1), NODE_DTYPE)
        self._ck(self.lib.esikf_map_device_export(self.h, keys.ctypes.data, first.ctypes.data, count.ctypes.data, len(first), nodes.ctypes.data, len(nodes),
                                                  C.byref(nr), C.byref(nn)))
        return dict(keys=keys[:nr.value], first=first[:nr.value], count=count[:nr.value], nodes=nodes[:nn.value])

    def map_device_find(self, points, rule):
        """find_correspond on the device map for world points (n x 3) from the root voxel the call site's key rule gives
        (FIND_RULE_PATCH / FIND_RULE_RAYCAST): status (FIND_*), key (n x 3, INT64_MIN when out of range) and planes
        (synthetic.PLANE_DTYPE: the found node's layer, path and plane fields, zero where there is no root)."""
        from .synthetic import PLANE_DTYPE

        pts = _c(points, np.float64).reshape(-1, 3)
        n = len(pts)
        status, keys, rows = np.zeros(n, np.uint8), np.zeros((n, 3), np.int64), np.zeros(n, PLANE_DTYPE)
        self._ck(self.lib.esikf_map_device_find(self.h, pts.ctypes.data, n, rule, status.ctypes.data, keys.ctypes.data, rows.ctypes.data))
        return dict(status=status, key=keys, planes=rows)

    def lio_fetch_normals(self):
        out = np.zeros((self.n_pts, 3), np.float64)
        self._ck(self.lib.esikf_lio_fetch_normals(self.h, out.ctypes.data))
        return out

    # ------------------------------------------------------------------ LIO
    def lio_set_scan(self, pts):
        """pts: (n,3) float32 numpy array or pinned torch tensor (kept alive by the caller until the copy is done)."""
        n = int(pts.shape[0])
        self._ck(self.lib.esikf_lio_set_scan(self.h, _addr(pts), n))
        self.n_pts = n

    def lio_run(self, state_in, state_prop, cfg):
        self._cfg_keep = lio_cfg_c(cfg) if not isinstance(cfg, LioCfgC) else cfg
        self._ck(self.lib.esikf_lio_run(self.h, _addr(state_in), _addr(state_prop), C.byref(self._cfg_keep)))

    def lio_fetch(self, per_point=True, state_out=None, match=None, normal=None, dis=None):
        """Outputs may be caller-provided (e.g. pinned torch tensors); otherwise numpy arrays are allocated."""
        out = np.zeros(STATE_DOUBLES) if state_out is None else state_out
        st = LioStatsC()
        n = self.n_pts
        if per_point:
            match = np.zeros(n, np.int32) if match is None else match
            normal = np.zeros(n, np.int32) if normal is None else normal
            dis = np.zeros(n, np.float32) if dis is None else dis
        self._ck(self.lib.esikf_lio_fetch(self.h, _addr(out), C.byref(st), _addr(match), _addr(normal), _addr(dis)))
        return self._lio_result(out, st, match, normal, dis)

    @staticmethod
    def _lio_result(out, st, match, normal, dis):
        it = st.iters
        return dict(state=out, match_plane=match, normal_plane=normal, dis_to_plane=dis, iters=it, M=np.array(st.effct_feat_num[:it]),
                    total_residual=np.array(st.total_residual[:it]), HTH=np.array(st.HTH[:]).reshape(8, 6, 6)[:it],
                    HTz=np.array(st.HTz[:]).reshape(8, 6)[:it], solution=np.array(st.solution[:]).reshape(8, 19)[:it],
                    converged=np.array(st.converged[:it]))

    def lio_update(self, pts, state_in, state_prop, cfg):
        """One-shot host-buffer call (esikf_lio_update): H2D + loop + D2H."""
        pts = _c(pts, np.float32)
        n = len(pts)
        self.n_pts = n
        out = np.zeros(STATE_DOUBLES)
        st = LioStatsC()
        match, normal, dis = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32)
        cfgc = lio_cfg_c(cfg)
        si, sp = _c(state_in, np.float64), _c(state_prop, np.float64)
        self._ck(self.lib.esikf_lio_update(self.h, pts.ctypes.data, n, si.ctypes.data, sp.ctypes.data, C.byref(cfgc), out.ctypes.data, C.byref(st),
                                           match.ctypes.data, normal.ctypes.data, dis.ctypes.data))
        return self._lio_result(out, st, match, normal, dis)

    def lio_update_into(self, pts, state_in, state_prop, cfg, state_out, match, normal, dis):
        """esikf_lio_update with caller-owned (e.g. pinned) input AND output buffers: one C call per LIO tick."""
        n = int(pts.shape[0])
        self.n_pts = n
        st = LioStatsC()
        cfgc = lio_cfg_c(cfg) if not isinstance(cfg, LioCfgC) else cfg
        self._ck(self.lib.esikf_lio_update(self.h, _addr(pts), n, _addr(state_in), _addr(state_prop), C.byref(cfgc), _addr(state_out), C.byref(st),
                                           _addr(match), _addr(normal), _addr(dis)))
        return st.iters

    def vio_update_into(self, img, pos, warp_patch, search_levels, inv_expo, state_in, state_prop, state_out, errors):
        n = int(pos.shape[0])
        self.n_patches = n
        st = VioStatsC()
        self._ck(self.lib.esikf_vio_update(self.h, _addr(img), int(img.shape[1]), int(img.shape[0]), _addr(pos), _addr(warp_patch), _addr(search_levels),
                                           _addr(inv_expo), n, _addr(state_in), _addr(state_prop), _addr(state_out), C.byref(st), _addr(errors)))
        return st.total_iters

    def lio_fetch_point_cov(self):
        bc = np.zeros((self.n_pts, 3, 3))
        cm = np.zeros((self.n_pts, 3, 3))
        self._ck(self.lib.esikf_lio_fetch_point_cov(self.h, bc.ctypes.data, cm.ctypes.data))
        return bc, cm

    # ------------------------------------------------------------------ VIO
    def vio_set_camera(self, cam, vio):
        c = CameraC(cam.model, cam.width, cam.height, 0, cam.fx, cam.fy, cam.cx, cam.cy)
        c.d[:] = list(cam.d)
        v = VioCfgC(vio.img_point_cov, vio.levels, vio.max_iterations, int(vio.exposure_estimate_en), int(getattr(vio, "inverse_composition_en", False)))
        self._ck(self.lib.esikf_vio_set_camera(self.h, C.byref(c), C.byref(v)))
        self.levels = vio.levels
        self.cam_size = (cam.width, cam.height)

    def vio_set_image(self, img):
        h, w = int(img.shape[0]), int(img.shape[1])
        self._ck(self.lib.esikf_vio_set_image(self.h, _addr(img), w, h))

    def vio_set_patches(self, pos, warp_patch, search_levels, inv_expo):
        n = int(pos.shape[0])
        self._ck(self.lib.esikf_vio_set_patches(self.h, _addr(pos), _addr(warp_patch), _addr(search_levels), _addr(inv_expo), n))
        self.n_patches = n

    def vio_run(self, state_in, state_prop):
        self._ck(self.lib.esikf_vio_run(self.h, _addr(state_in), _addr(state_prop)))

    def vio_fetch(self, errors=True, state_out=None, err=None):
        out = np.zeros(STATE_DOUBLES) if state_out is None else state_out
        st = VioStatsC()
        if errors and err is None:
            err = np.zeros(self.n_patches, np.float32)
        self._ck(self.lib.esikf_vio_fetch(self.h, _addr(out), C.byref(st), _addr(err)))
        return self._vio_result(out, st, err)

    @staticmethod
    def _vio_result(out, st, err):
        return dict(state=out, errors=err, total_iters=st.total_iters, iters_per_level=np.array(st.iters_per_level[:]),
                    accepted_per_level=np.array(st.accepted_per_level[:]), error_trace=np.array(st.error_trace[:]).reshape(8, 8),
                    HTH=np.array(st.HTH[:]).reshape(8, 8, 7, 7), HTz=np.array(st.HTz[:]).reshape(8, 8, 7),
                    solution=np.array(st.solution[:]).reshape(8, 8, 19))

    def vio_update(self, img, pos, warp_patch, search_levels, inv_expo, state_in, state_prop):
        img = _c(img, np.uint8)
        pos, wp = _c(pos, np.float64), _c(warp_patch, np.float32)
        sl, ie = _c(search_levels, np.int32), _c(inv_expo, np.float64)
        n = len(pos)
        self.n_patches = n
        out = np.zeros(STATE_DOUBLES)
        st = VioStatsC()
        err = np.zeros(n, np.float32)
        si, sp = _c(state_in, np.float64), _c(state_prop, np.float64)
        self._ck(self.lib.esikf_vio_update(self.h, img.ctypes.data, img.shape[1], img.shape[0], pos.ctypes.data, wp.ctypes.data, sl.ctypes.data,
                                           ie.ctypes.data, n, si.ctypes.data, sp.ctypes.data, out.ctypes.data, C.byref(st), err.ctypes.data))
        return self._vio_result(out, st, err)

    def vio_get_image_patch(self, pc, level):
        pc = _c(pc, np.float64).reshape(-1, 2)
        out = np.zeros((len(pc), 64), np.float32)
        self._ck(self.lib.esikf_vio_get_image_patch(self.h, pc.ctypes.data, len(pc), level, out.ctypes.data))
        return out

    def vio_set_ref_images(self, imgs):
        imgs = [_c(im, np.uint8) for im in imgs]
        self._ref_keep = imgs
        arr = (C.c_void_p * len(imgs))(*[im.ctypes.data for im in imgs])
        self._ck(self.lib.esikf_vio_set_ref_images(self.h, arr, len(imgs), imgs[0].shape[1], imgs[0].shape[0]))

    def vio_warp_patches(self, ref_idx, px_ref, pos_w, normal_w, T_ref, T_cur, keep_on_device=False):
        n = len(px_ref)
        ref_idx = _c(ref_idx, np.int32)
        px_ref, pos_w, normal_w = _c(px_ref, np.float64), _c(pos_w, np.float64), _c(normal_w, np.float64)
        T_ref = _c(T_ref, np.float64).reshape(n, 12)
        T_cur = _c(T_cur, np.float64).reshape(12)
        A = np.zeros((n, 2, 2))
        sl = np.zeros(n, np.int32)
        wp = np.zeros((n, 64 * self.levels), np.float32)
        self._ck(self.lib.esikf_vio_warp_patches(self.h, n, ref_idx.ctypes.data, px_ref.ctypes.data, pos_w.ctypes.data, normal_w.ctypes.data,
                                                 T_ref.ctypes.data, T_cur.ctypes.data, A.ctypes.data, sl.ctypes.data, wp.ctypes.data,
                                                 int(keep_on_device)))
        if keep_on_device:
            self.n_patches = n
        return dict(A_cur_ref=A, search_levels=sl, warp_patch=wp)

    def vio_select_patches(self, ref_idx, px_ref, pos_w, T_ref, ref_inv_expo, pc, T_cur, inv_expo_time, normal_w=None, ref_level=None, ref_f=None,
                           ref_pos=None, ref_key=None, normal_en=True, ncc_en=False, ncc_thre=0.0, outlier_threshold=1000.0, want_patches=False):
        """The per-candidate tail of the visual sub-map retrieval (esikf_vio_select_patches): warp matrices (homography form
        from normal_w when normal_en, else the depth form from ref_f / ref_pos / ref_level cached per ref_key), warps, the
        photometric / NCC gates; the survivors become the sub-map of the next vio_run. Returns kept (candidate indices),
        errors, search_levels, A_cur_ref (n_kept, 2, 2) and, with want_patches, warp_patch (n_kept, levels*64)."""
        n = len(px_ref)
        d = lambda a, shape: None if a is None else _c(a, np.float64).reshape(shape)
        i32 = lambda a: None if a is None else _c(a, np.int32).reshape(n)
        args = [i32(ref_idx), d(px_ref, (n, 2)), i32(ref_level), d(ref_f, (n, 3)), d(ref_pos, (n, 3)), d(pos_w, (n, 3)), d(normal_w, (n, 3)),
                d(T_ref, (n, 12)), d(ref_inv_expo, (n,)), i32(ref_key), d(pc, (n, 2)), d(T_cur, (12,))]
        cfg = VioSelectCfgC(int(normal_en), int(ncc_en), float(ncc_thre), float(outlier_threshold))
        nk = C.c_int32(0)
        kept, err, sl, A = np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(n, np.int32), np.zeros((n, 2, 2))
        wp = np.zeros((n, 64 * self.levels), np.float32) if want_patches else None
        self._ck(self.lib.esikf_vio_select_patches(self.h, n, *[_addr(a) for a in args], float(inv_expo_time), C.byref(cfg), C.byref(nk), kept.ctypes.data,
                                                   err.ctypes.data, sl.ctypes.data, A.ctypes.data, _addr(wp)))
        k = nk.value
        self.n_patches = k
        out = dict(kept=kept[:k], errors=err[:k], search_levels=sl[:k], A_cur_ref=A[:k])
        if want_patches:
            out["warp_patch"] = wp[:k]
        return out

    # ------------------------------------------------------------------ coloured scan (publish_frame_world)
    def rgb_set_cloud(self, pts=None, state=None):
        """The world cloud of this LIO tick (esikf_rgb_set_cloud): pts (n, 3) float32 body points, or None for the resident
        scan of lio_set_scan / lio_update; state: a packed state, or None for the posterior the last LIO update left on the
        device. Call after the LIO update and before the VIO update."""
        p = None if pts is None else _c(pts, np.float32).reshape(-1, 3)
        s = None if state is None else _c(state, np.float64)
        self._ck(self.lib.esikf_rgb_set_cloud(self.h, _addr(p), 0 if p is None else len(p), _addr(s)))
        self._rgb_n = self.n_pts if p is None else len(p)

    def rgb_colorize(self, bgr, blind_rgb_points=0.01, state=None, cap=None):
        """publish_frame_world on the cloud of rgb_set_cloud (esikf_rgb_colorize): bgr (height, width, 3) uint8 B G R of the
        camera's size; state: a packed state, or None for the posterior the last VIO update left on the device. Returns
        xyz (k, 3) float32, bgr (k, 3) uint8 (B, G, R) and index (k,) int32 of the kept points in cloud order. cap: room for
        that many points (default: every point of the cloud); fewer than the kept points raises."""
        img = _c(bgr, np.uint8)
        assert img.ndim == 3 and img.shape[2] == 3
        s = None if state is None else _c(state, np.float64)
        cap = self._rgb_n if cap is None else int(cap)
        xyz, col, idx = np.zeros((max(cap, 1), 3), np.float32), np.zeros((max(cap, 1), 3), np.uint8), np.zeros(max(cap, 1), np.int32)
        n = C.c_int32(0)
        self._ck(self.lib.esikf_rgb_colorize(self.h, img.ctypes.data, img.shape[1], img.shape[0], _addr(s), float(blind_rgb_points), cap, C.byref(n),
                                             xyz.ctypes.data, col.ctypes.data, idx.ctypes.data))
        k = n.value
        return dict(xyz=xyz[:k], bgr=col[:k], index=idx[:k])

    # ------------------------------------------------------------------ new visual map points (generateVisualMapPoints)
    def vio_generate_points(self, type_map, grid_size, grid_n_width, grid_n_height, border, pg=None, add_from=None, state=None, cap=None):
        """generateVisualMapPoints on the device (esikf_vio_generate_points), after vio_run. type_map: (grid_n_height *
        grid_n_width,) bool / uint8, True where the retrieval set TYPE_MAP; grid_size .. border as initializeVIO left them.
        pg: None for the pv list the last map_device_update left on the device, else (point_w (n, 3), normal (n, 3), var (n, 3, 3))
        float64; add_from: None or (pos (m, 3), normal (m, 3)); state: a packed state, or None for the VIO posterior on the device.
        Returns the winners in cell order: source (int32: scan index, or api.GEN_ADD_FROM | add_from index), cell, pos (k, 3),
        pc (k, 2), score (k,) float32, normal (k, 3) (sign-flipped as the reference does), var (k, 3, 3), patch (k, 64) float32.
        cap: room for that many (default: one per cell); fewer than the winners raises."""
        mask = _c(type_map, np.uint8).reshape(-1)
        if pg is None:
            pw = nv = var = None
            n = 0
        else:
            pw, nv, var = _c(pg[0], np.float64).reshape(-1, 3), _c(pg[1], np.float64).reshape(-1, 3), _c(pg[2], np.float64).reshape(-1, 9)
            n = len(pw)
            assert len(nv) == n and len(var) == n
        if add_from is None:
            ap = an = None
            m = 0
        else:
            ap, an = _c(add_from[0], np.float64).reshape(-1, 3), _c(add_from[1], np.float64).reshape(-1, 3)
            m = len(ap)
            assert len(an) == m
        s = None if state is None else _c(state, np.float64)
        cap = len(mask) if cap is None else int(cap)
        k = max(cap, 1)
        out = dict(source=np.zeros(k, np.int32), cell=np.zeros(k, np.int32), pos=np.zeros((k, 3)), pc=np.zeros((k, 2)), score=np.zeros(k, np.float32),
                   normal=np.zeros((k, 3)), var=np.zeros((k, 3, 3)), patch=np.zeros((k, 64), np.float32))
        cnt = C.c_int32(0)
        self._ck(self.lib.esikf_vio_generate_points(self.h, _addr(pw), _addr(nv), _addr(var), n, _addr(ap), _addr(an), m, mask.ctypes.data, len(mask),
                                                    int(grid_size), int(grid_n_width), int(grid_n_height), int(border), _addr(s), cap, C.byref(cnt),
                                                    *[out[f].ctypes.data for f in ("source", "cell", "pos", "pc", "score", "normal", "var", "patch")]))
        return {f: v[:cnt.value] for f, v in out.items()}

    # ------------------------------------------------------------------ new observations of the sub-map (updateVisualMapPoints)
    def vio_update_points(self, converged, last_T, last_px, state=None, cap=None):
        """updateVisualMapPoints on the device (esikf_vio_update_points), after vio_run, for the sub-map installed on the device
        (n entries). converged: (n,) bool / uint8, is_converged_; last_T: (n, 12) float64, obs_.back()->T_f_w_ as R (row-major)
        then t; last_px: (n, 2) float64, obs_.back()->px_; state: a packed state, or None for the VIO posterior on the device.
        Returns update_flag (n,) uint8 and, for the added entries in entry order, entry (int32 sub-map index), pc (k, 2) and
        patch (k, 64) float32. cap: room for that many (default n); fewer than the added entries raises."""
        conv = _c(converged, np.uint8).reshape(-1)
        n = len(conv)
        T = _c(last_T, np.float64).reshape(-1, 12)
        px = _c(last_px, np.float64).reshape(-1, 2)
        assert len(T) == n and len(px) == n
        s = None if state is None else _c(state, np.float64)
        cap = n if cap is None else int(cap)
        k = max(cap, 1)
        flag = np.zeros(max(n, 1), np.uint8)
        out = dict(entry=np.zeros(k, np.int32), pc=np.zeros((k, 2)), patch=np.zeros((k, 64), np.float32))
        cnt = C.c_int32(0)
        self._ck(self.lib.esikf_vio_update_points(self.h, n, conv.ctypes.data, T.ctypes.data, px.ctypes.data, _addr(s), cap, C.byref(cnt),
                                                  flag.ctypes.data, *[out[f].ctypes.data for f in ("entry", "pc", "patch")]))
        return dict(update_flag=flag[:n], **{f: v[:cnt.value] for f, v in out.items()})

    # ------------------------------------------------------------------ scan side of the retrieval (retrieveFromVisualSparseMap)
    def vio_retrieve_scan(self, border, pg=None, state=None, depth=False, cap=None):
        """The scan's voxel keys and depth image (esikf_vio_retrieve_scan, vio.cpp:386-428). pg: (n, 3) float64 world points, or
        None for the pv list the last map_device_update left on the device; state: the frame's packed state (the VIO prior), or
        None for the LIO posterior on the device. Returns keys (k, 3) int32 in first-occurrence order and, with depth=True, the
        depth image (height, width) float32. cap: room for that many keys (fewer raises); by default the scan size, or for the
        resident scan whatever a first call reports."""
        p = None if pg is None else _c(pg, np.float64).reshape(-1, 3)
        s = None if state is None else _c(state, np.float64)
        n = 0 if p is None else len(p)
        w, h = self.cam_size
        img = np.zeros((h, w), np.float32) if depth else None
        cnt = C.c_int32(-1)

        def call(k):
            keys = np.zeros((max(k, 1), 3), np.int32)
            rc = self.lib.esikf_vio_retrieve_scan(self.h, _addr(p), n, int(border), _addr(s), k, C.byref(cnt), keys.ctypes.data, _addr(img))
            return rc, keys

        rc, keys = call(n if cap is None and p is not None else int(cap or 0))
        if rc == -3 and cap is None and p is None and cnt.value > 0:  # ESIKF_ERR_ARG with the count of the resident scan's keys
            rc, keys = call(cnt.value)
        self._ck(rc)
        return dict(keys=keys[:cnt.value], depth=img) if depth else dict(keys=keys[:cnt.value])

    def vio_depth_check(self, pos, pc):
        """The depth-continuity flags of n retrieved points (esikf_vio_depth_check, vio.cpp:614-640) against the depth image of
        the last vio_retrieve_scan: pos (n, 3) VisualPoint::pos_, pc (n, 2) the caller's w2c(pos_). Returns (n,) uint8, 1 = the
        point is dropped."""
        pos = _c(pos, np.float64).reshape(-1, 3)
        pc = _c(pc, np.float64).reshape(-1, 2)
        assert len(pos) == len(pc)
        out = np.zeros(max(len(pos), 1), np.uint8)
        self._ck(self.lib.esikf_vio_depth_check(self.h, len(pos), pos.ctypes.data, pc.ctypes.data, out.ctypes.data))
        return out[:len(pos)]

    # ------------------------------------------------------------------ reference patches (updateReferencePatch)
    def vio_score_ref_patches(self, first, pos, normal, patch, mean, id_, T_f_w):
        """The patch scoring of updateReferencePatch (esikf_vio_score_ref_patches, vio.cpp:1036-1097) for n visual points:
        first (n + 1,) int32 offsets of each point's observations in obs_ order; pos, normal (n, 3) float64 (pos_, and normal_
        after the plane half); per observation patch (m, 64) float32, mean (m,) float32 (mean_), id_ (m,) int32 and T_f_w
        (m, 12) float64 (R row-major, then t). Returns score (m,) float32 (score_), mean (m,) float32 (mean_ afterwards) and
        ref (n,) int32, the position of ref_patch within the point's list or -1 when no score beats -1000."""
        first = _c(first, np.int32).reshape(-1)
        n = len(first) - 1
        pos, normal = _c(pos, np.float64).reshape(-1, 3), _c(normal, np.float64).reshape(-1, 3)
        patch, mean = _c(patch, np.float32).reshape(-1, 64), _c(mean, np.float32).reshape(-1)
        id_, T = _c(id_, np.int32).reshape(-1), _c(T_f_w, np.float64).reshape(-1, 12)
        m = len(patch)
        assert n >= 0 and len(pos) == n and len(normal) == n and len(mean) == m and len(id_) == m and len(T) == m
        score, mean_out, ref = np.zeros(max(m, 1), np.float32), np.zeros(max(m, 1), np.float32), np.zeros(max(n, 1), np.int32)
        self._ck(self.lib.esikf_vio_score_ref_patches(self.h, n, first.ctypes.data, m, pos.ctypes.data, normal.ctypes.data, patch.ctypes.data,
                                                      mean.ctypes.data, id_.ctypes.data, T.ctypes.data, score.ctypes.data, mean_out.ctypes.data,
                                                      ref.ctypes.data))
        return dict(score=score[:m], mean=mean_out[:m], ref=ref[:n])

    # ------------------------------------------------------------------ the visual map's observations on the device (K14)
    def vmap_init(self, point_capacity):
        """An empty observation store with room for point_capacity points (esikf_vmap_init); it grows by doubling."""
        self._ck(self.lib.esikf_vmap_init(self.h, int(point_capacity)))

    def vmap_stats(self):
        """(points, capacity) of the observation store."""
        pts, cap = C.c_int64(0), C.c_int64(0)
        self._ck(self.lib.esikf_vmap_stats(self.h, C.byref(pts), C.byref(cap)))
        return pts.value, cap.value

    def vmap_add_points(self, first, px, patch, T_f_w, id, mean, score, ref):  # noqa: A002 (vmap_download's field names)
        """Append n points (esikf_vmap_add_points): first (n + 1,) int32 offsets of each point's observations in obs_ order;
        per observation px (m, 2) float64, patch (m, 64) float32, T_f_w (m, 12) float64, id (m,) int32, mean, score (m,)
        float32; ref (n,) int32, the position of ref_patch or -1. Returns the new points' ids (n,) int32."""
        first = _c(first, np.int32).reshape(-1)
        n = len(first) - 1
        px, patch, T = _c(px, np.float64).reshape(-1, 2), _c(patch, np.float32).reshape(-1, 64), _c(T_f_w, np.float64).reshape(-1, 12)
        id_, mean, score, ref = _c(id, np.int32).reshape(-1), _c(mean, np.float32).reshape(-1), _c(score, np.float32).reshape(-1), _c(ref, np.int32).reshape(-1)
        m = len(px)
        assert n >= 0 and len(ref) == n and len(patch) == m and len(T) == m and len(id_) == m and len(mean) == m and len(score) == m
        ids = np.zeros(max(n, 1), np.int32)
        self._ck(self.lib.esikf_vmap_add_points(self.h, n, first.ctypes.data, m, px.ctypes.data, patch.ctypes.data, T.ctypes.data, id_.ctypes.data,
                                                mean.ctypes.data, score.ctypes.data, ref.ctypes.data, ids.ctypes.data))
        return ids[:n]

    def vmap_update_points(self, point_id, converged, frame_id, T_f_w=None, state=None, cap=None):
        """updateVisualMapPoints on the store (esikf_vmap_update_points) for the installed sub-map, entry i being store point
        point_id[i]. T_f_w (12,): the new observations' T_f_w_, None for the frame pose of the flags; state: a packed state, or
        None for the VIO posterior on the device. Returns vio_update_points' update_flag, entry, pc and patch, and per entry
        evicted (the list position removed, or -1) and count (the count afterwards)."""
        pid = _c(point_id, np.int32).reshape(-1)
        conv = _c(converged, np.uint8).reshape(-1)
        n = len(pid)
        assert len(conv) == n
        T = None if T_f_w is None else _c(T_f_w, np.float64).reshape(12)
        s = None if state is None else _c(state, np.float64)
        cap = n if cap is None else int(cap)
        k = max(cap, 1)
        flag, evicted, count = np.zeros(max(n, 1), np.uint8), np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
        out = dict(entry=np.zeros(k, np.int32), pc=np.zeros((k, 2)), patch=np.zeros((k, 64), np.float32))
        cnt = C.c_int32(0)
        self._ck(self.lib.esikf_vmap_update_points(self.h, n, pid.ctypes.data, conv.ctypes.data, _addr(T), int(frame_id), _addr(s), cap, C.byref(cnt),
                                                   flag.ctypes.data, *[out[f].ctypes.data for f in ("entry", "pc", "patch")], evicted.ctypes.data,
                                                   count.ctypes.data))
        return dict(update_flag=flag[:n], evicted=evicted[:n], count=count[:n], **{f: v[:cnt.value] for f, v in out.items()})

    def vmap_score(self, point_id, pos, normal):
        """The patch scoring of updateReferencePatch on the store (esikf_vmap_score): pos, normal (n, 3) float64 per entry.
        Returns ref (n,) int32 (stored where >= 0) and the store's score and mean rows (n, 30) float32 afterwards."""
        pid = _c(point_id, np.int32).reshape(-1)
        n = len(pid)
        pos, normal = _c(pos, np.float64).reshape(-1, 3), _c(normal, np.float64).reshape(-1, 3)
        assert len(pos) == n and len(normal) == n
        ref, score, mean = np.zeros(max(n, 1), np.int32), np.zeros((max(n, 1), 30), np.float32), np.zeros((max(n, 1), 30), np.float32)
        self._ck(self.lib.esikf_vmap_score(self.h, n, pid.ctypes.data, pos.ctypes.data, normal.ctypes.data, ref.ctypes.data, score.ctypes.data,
                                           mean.ctypes.data))
        return dict(ref=ref[:n], score=score[:n], mean=mean[:n])

    def vmap_choose_ref(self, point_id, normal_en, pos=None, frame_pos=None):
        """The reference feature of the retrieval (esikf_vmap_choose_ref, vio.cpp:651-697): normal_en, or getCloseViewObs from
        frame_pos (3,) with pos (n, 3). Returns ref (n,) int32, -1 where none is chosen."""
        pid = _c(point_id, np.int32).reshape(-1)
        n = len(pid)
        p = None if pos is None else _c(pos, np.float64).reshape(-1, 3)
        fp = None if frame_pos is None else _c(frame_pos, np.float64).reshape(3)
        ref = np.zeros(max(n, 1), np.int32)
        self._ck(self.lib.esikf_vmap_choose_ref(self.h, n, pid.ctypes.data, _addr(p), _addr(fp), int(bool(normal_en)), ref.ctypes.data))
        return ref[:n]

    def vmap_place_points(self, point_id, pos, normal_init=None):
        """Place store points in their visual voxels (esikf_vmap_place_points, insertPointIntoVoxelMap): pos (n, 3) float64
        pos_, normal_init (n,) is_normal_initialized_ (None: all true)."""
        pid = _c(point_id, np.int32).reshape(-1)
        n = len(pid)
        pos = _c(pos, np.float64).reshape(-1, 3)
        ni = None if normal_init is None else _c(normal_init, np.uint8).reshape(-1)
        assert len(pos) == n and (ni is None or len(ni) == n)
        self._ck(self.lib.esikf_vmap_place_points(self.h, n, pid.ctypes.data, pos.ctypes.data, _addr(ni)))

    def vmap_retrieve(self, keys, grid_size, grid_n_width, grid_n_height, border, normal_en, cap=None):
        """The walk of the retrieval over the placed points, its depth check, skip and reference choice (esikf_vmap_retrieve)
        for the pose and depth image of the last vio_retrieve_scan: keys (k, 3) in sub_feat_map iteration order. Returns per
        TYPE_MAP cell, in cell order: cell, point_id (-1 none), pc (m, 2), status (RETRIEVE_*) and ref (-1 unless kept).
        cap: room for that many cells (fewer raises); by default the grid's length."""
        keys = _c(keys, np.int32).reshape(-1, 3)
        cap = int(grid_n_width) * int(grid_n_height) if cap is None else int(cap)
        k = max(cap, 1)
        out = dict(cell=np.zeros(k, np.int32), point_id=np.zeros(k, np.int32), pc=np.zeros((k, 2)), status=np.zeros(k, np.int32), ref=np.zeros(k, np.int32))
        cnt = C.c_int32(0)
        self._ck(self.lib.esikf_vmap_retrieve(self.h, len(keys), keys.ctypes.data, int(grid_size), int(grid_n_width), int(grid_n_height), int(border),
                                              int(bool(normal_en)), cap, C.byref(cnt), *[out[f].ctypes.data for f in ("cell", "point_id", "pc", "status", "ref")]))
        return {f: v[:cnt.value] for f, v in out.items()}

    def vmap_download(self, point_id):
        """The lists of the given points (esikf_vmap_download), in vmap_add_points' form: first, px, patch, T_f_w, id, mean,
        score, ref."""
        pid = _c(point_id, np.int32).reshape(-1)
        n = len(pid)
        first = np.zeros(n + 1, np.int32)
        rc = self.lib.esikf_vmap_download(self.h, n, pid.ctypes.data, 0, first.ctypes.data, *([None] * 6), np.zeros(max(n, 1), np.int32).ctypes.data)
        if rc != 0 and first[n] == 0:
            self._ck(rc)
        m = int(first[n])
        out = dict(px=np.zeros((max(m, 1), 2)), patch=np.zeros((max(m, 1), 64), np.float32), T_f_w=np.zeros((max(m, 1), 12)), id=np.zeros(max(m, 1), np.int32),
                   mean=np.zeros(max(m, 1), np.float32), score=np.zeros(max(m, 1), np.float32))
        ref = np.zeros(max(n, 1), np.int32)
        self._ck(self.lib.esikf_vmap_download(self.h, n, pid.ctypes.data, m, first.ctypes.data, *[out[f].ctypes.data for f in ("px", "patch", "T_f_w", "id", "mean", "score")],
                                              ref.ctypes.data))
        return dict(first=first, ref=ref[:n], **{f: v[:m] for f, v in out.items()})

    # ------------------------------------------------------------------ multi-GPU / measurement
    def vio_set_inverse_refs(self, ref_img_index, ref_px, ref_f, ref_R, ref_pos):
        """Reference-feature data of the inverse-compositional variant (esikf_vio_set_inverse_refs); images via vio_set_ref_images."""
        idx = _c(ref_img_index, np.int32)
        n = len(idx)
        px, f, R, pos = _c(ref_px, np.float64), _c(ref_f, np.float64), _c(np.asarray(ref_R).reshape(n, 9), np.float64), _c(ref_pos, np.float64)
        self._ck(self.lib.esikf_vio_set_inverse_refs(self.h, n, idx.ctypes.data, px.ctypes.data, f.ctypes.data, R.ctypes.data, pos.ctypes.data))

    def vio_warp_affine(self, ref_idx, px_ref, A_cur_ref, search_levels):
        """warpAffine alone (esikf_vio_warp_affine): caller-provided 2x2 matrices and search levels -> (n, levels*64) float32."""
        n = len(px_ref)
        ref_idx, sl = _c(ref_idx, np.int32), _c(search_levels, np.int32)
        px_ref, A = _c(px_ref, np.float64), _c(A_cur_ref, np.float64).reshape(n, 4)
        wp = np.zeros((n, 64 * self.levels), np.float32)
        self._ck(self.lib.esikf_vio_warp_affine(self.h, n, ref_idx.ctypes.data, px_ref.ctypes.data, A.ctypes.data, sl.ctypes.data, wp.ctypes.data))
        return wp

    def comm_init(self, rank, nranks, unique_id: bytes):
        self._ck(self.lib.esikf_comm_init(self.h, rank, nranks, unique_id))

    def set_phase_stamps(self, enable):
        self._ck(self.lib.esikf_set_phase_stamps(self.h, int(enable)))

    def get_phase_stamps(self):
        out = np.zeros(800, np.uint64)
        self._ck(self.lib.esikf_get_phase_stamps(self.h, out.ctypes.data_as(C.POINTER(C.c_uint64))))
        self.debug_stamps = out[576:640].copy()
        self.cta_stamps = out[640:].copy()
        return out[:576].reshape(72, 8)

    def get_vio_chain_stamps(self):
        """The VIO kernel's chain stamps (esikf_get_vio_chain_stamps): written only by a library built with
        -DESIKF_VIO_CHAIN_STAMPS, by a persistent update run while phase stamps are on."""
        out = np.zeros(VIO_CHAIN_STAMP_WORDS, np.uint64)
        self._ck(self.lib.esikf_get_vio_chain_stamps(self.h, out.ctypes.data_as(C.POINTER(C.c_uint64))))
        return out

    def set_kernel_timing(self, enable):
        self._ck(self.lib.esikf_set_kernel_timing(self.h, int(enable)))

    def get_kernel_timing(self):
        a, b, c, d = (np.zeros(8, np.float32), np.zeros(8, np.float32), np.zeros(64, np.float32), np.zeros(64, np.float32))
        f = lambda x: x.ctypes.data_as(C.POINTER(C.c_float))
        self._ck(self.lib.esikf_get_kernel_timing(self.h, f(a), f(b), f(c), f(d)))
        return dict(lio_residual_ms=a, lio_solve_ms=b, vio_patch_ms=c, vio_solve_ms=d)

    def peer_export(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._ck(self.lib.esikf_peer_export(self.h, buf))
        return buf.raw

    def peer_attach(self, rank, nranks, handles):
        """handles: list of the 64-byte IPC handles of every rank, in rank order."""
        self._ck(self.lib.esikf_peer_attach(self.h, rank, nranks, b"".join(handles)))

    def profile_kernel(self, which, arg=0, reps=20, flush_l2=True):
        ms = C.c_float(0)
        self._ck(self.lib.esikf_profile_kernel(self.h, which, arg, reps, int(flush_l2), C.byref(ms)))
        return float(ms.value)


def shard_range(n, rank, nranks):
    lib = load_library()
    b, c = C.c_int32(0), C.c_int32(0)
    if lib.esikf_shard_range(n, rank, nranks, C.byref(b), C.byref(c)) != 0:
        raise EsikfError("esikf_shard_range: bad argument")
    return b.value, c.value


def comm_unique_id() -> bytes:
    lib = load_library()
    buf = C.create_string_buffer(128)
    rc = lib.esikf_comm_unique_id(buf)
    if rc != 0:
        raise EsikfError(f"esikf_comm_unique_id failed: {rc}")
    return buf.raw


def pack_T(Rcw, Pcw):
    return np.concatenate([np.asarray(Rcw, np.float64).reshape(9), np.asarray(Pcw, np.float64).reshape(3)])
