"""Candidate sets of the visual sub-map selection (esikf_vio_select_patches: the per-candidate tail of
retrieveFromVisualSparseMap, src/vio.cpp:645-770) and ctypes bindings of its oracle (oracle/liborc_select.so) and of the
reference source's pieces it is pinned to (oracle/_ref/libfl2_ref_select.so), both built by oracle/select.mk.

candidates(camera, n, ...) draws n visual points in front of a current camera pose (not the identity), each observed in one of
several reference frames (several candidates per frame, keys = frame ids) with its own exposure time, pyramid level and image."""
import ctypes as C
import os

import numpy as np

import warp_cases as W
from fast_livo2_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORC_SELECT_SO = os.path.join(ROOT, "oracle", "liborc_select.so")
REF_SELECT_SO = os.path.join(ROOT, "oracle", "_ref", "libfl2_ref_select.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pin", "select.npz")
vp = C.c_void_p


def _a(x, dt=np.float64):
    return None if x is None else np.ascontiguousarray(x, dtype=dt)


def _ptr(x):
    return None if x is None else x.ctypes.data


def texture(cam, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:cam.height, 0:cam.width]
    return (127.5 + 60 * np.sin(xx / 9.7 + seed) * np.cos(yy / 6.3) + rng.normal(0, 25, (cam.height, cam.width))).clip(0, 255).astype(np.uint8)


def pack_T(R, t):
    return np.concatenate([np.asarray(R).reshape(-1, 9), np.asarray(t).reshape(-1, 3)], 1)


def candidates(camera, n, n_frames=12, n_imgs=3, seed=0, margin=24.0):
    """n candidates in grid-cell-like order. Returns a dict with the esikf_vio_select_patches inputs (T as R(9) t(3)), the
    current image `img`, the reference images `ref_imgs` and the camera `cam`."""
    cam = W.CAMERAS[camera]
    rng = np.random.default_rng(seed)
    R_cur = W._rot(rng.normal(0, 0.05, 3))
    t_cur = rng.normal(0, 0.3, 3)
    px = np.stack([rng.uniform(margin, cam.width - margin, n), rng.uniform(margin, cam.height - margin, n)], 1)
    depth = rng.uniform(1.5, 9.0, n)
    P_cur = W.cam2world(cam, px[:, 0], px[:, 1]) * depth[:, None]
    pos_w = np.einsum("ji,nj->ni", R_cur, P_cur - t_cur)  # R_cur^T (P - t)
    pc = np.stack(W.world2cam(cam, np.einsum("ij,nj->ni", R_cur, pos_w) + t_cur), 1)
    # reference frames near the current pose (the warps stay well conditioned)
    R_k = W._rot(rng.normal(0, 0.08, (n_frames, 3))) @ R_cur
    t_k = t_cur + rng.normal(0, 0.25, (n_frames, 3))
    frame = rng.integers(0, n_frames, n)
    R_ref, t_ref = R_k[frame], t_k[frame]
    P_ref = np.einsum("nij,nj->ni", R_ref, pos_w) + t_ref
    px_ref = np.stack(W.world2cam(cam, P_ref), 1)
    ref_f = W.cam2world(cam, px_ref[:, 0], px_ref[:, 1])
    ref_pos = -np.einsum("nji,nj->ni", R_ref, t_ref)
    normal = rng.normal(0, 0.3, (n, 3)) - P_cur / depth[:, None]
    normal_w = np.einsum("ji,nj->ni", R_cur, normal / np.linalg.norm(normal, axis=1, keepdims=True))
    expo = rng.uniform(0.6, 1.6, n_frames)
    return dict(cam=camera, camcfg=cam, img=texture(cam, 100 + seed), ref_imgs=[texture(cam, 200 + seed + k) for k in range(n_imgs)],
                ref_idx=(frame % n_imgs).astype(np.int32), px_ref=px_ref, ref_level=rng.integers(0, 3, n).astype(np.int32), ref_f=ref_f, ref_pos=ref_pos,
                pos_w=pos_w, normal_w=normal_w, T_ref=pack_T(R_ref, t_ref), ref_inv_expo=expo[frame], ref_key=(1000 + 7 * frame).astype(np.int32), pc=pc,
                T_cur=pack_T(R_cur, t_cur)[0], inv_expo=0.9)


class OracleSelect:
    """The oracle's restatement of the tail (oracle/orc_select.cpp) on one camera and pyramid depth."""

    def __init__(self, cam, levels=4):
        self.lib = C.CDLL(ORC_SELECT_SO)
        L = self.lib
        L.orc_vio_create.restype = vp
        L.orc_vio_create.argtypes = [vp] * 6 + [C.c_int]
        L.orc_vio_destroy.argtypes = [vp]
        L.orc_select_warp_matrix_affine.restype = C.c_int
        L.orc_select_warp_matrix_affine.argtypes = [vp] * 7 + [C.c_int, vp]
        L.orc_select_calculate_ncc.restype = C.c_double
        L.orc_select_calculate_ncc.argtypes = [vp, vp]
        L.orc_select_patches.restype = C.c_int
        L.orc_select_patches.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int] + [vp] * 13 + [C.c_double, C.c_int, C.c_int, C.c_double, C.c_double] + [vp] * 8
        ext = S.avia_extrinsics()
        self.levels = levels
        self._keep = [_a(cam.as_array()), _a(ext.extR), _a(ext.extT), _a(ext.Rcl), _a(ext.Pcl), _a(S.VioCfg(levels=levels).as_array())]
        self.h = L.orc_vio_create(*[_ptr(k) for k in self._keep], 1)

    def __del__(self):
        try:
            self.lib.orc_vio_destroy(self.h)
        except Exception:
            pass

    def warp_matrix_affine(self, px_ref, f_ref, ref_pos, pos_w, T_ref, T_cur, level_ref):
        A = np.zeros(4)
        args = [_a(px_ref), _a(f_ref), _a(ref_pos), _a(pos_w), _a(T_ref), _a(T_cur)]
        sl = self.lib.orc_select_warp_matrix_affine(self.h, *[_ptr(x) for x in args], int(level_ref), _ptr(A))
        return A, sl

    def ncc(self, ref_patch, cur_patch):
        r, c = _a(ref_patch, np.float32), _a(cur_patch, np.float32)
        return self.lib.orc_select_calculate_ncc(_ptr(r), _ptr(c))

    def select(self, c, normal_en=True, ncc_en=False, ncc_thre=0.0, outlier_threshold=1000.0, A_in=None, sl_in=None):
        """The tail over the candidate set `c`. A_in / sl_in: evaluate the later steps on these warp matrices and levels."""
        n = len(c["px_ref"])
        L = self.levels
        imgs = [np.ascontiguousarray(im) for im in c["ref_imgs"]]
        arr = (vp * len(imgs))(*[im.ctypes.data for im in imgs])
        img = np.ascontiguousarray(c["img"])
        ins = [_a(c["ref_idx"], np.int32), _a(c["px_ref"]), _a(c["ref_level"], np.int32), _a(c["ref_f"]), _a(c["ref_pos"]), _a(c["pos_w"]),
               _a(c["normal_w"]), _a(c["T_ref"]), _a(c["ref_inv_expo"]), _a(c["ref_key"], np.int32), _a(c["pc"]), _a(c["T_cur"])]
        A_in, sl_in = _a(A_in), _a(sl_in, np.int32)
        A, sl, wp = np.zeros((n, 2, 2)), np.zeros(n, np.int32), np.zeros((n, 64 * L), np.float32)
        err, keep, kept = np.zeros(n, np.float32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        ref_h, ref_w = imgs[0].shape
        k = self.lib.orc_select_patches(self.h, n, C.cast(arr, vp), ref_w, ref_h, img.ctypes.data, *[_ptr(x) for x in ins], float(c["inv_expo"]), int(normal_en),
                                        int(ncc_en), float(ncc_thre), float(outlier_threshold), _ptr(A_in), _ptr(sl_in), _ptr(A), _ptr(sl), _ptr(wp), _ptr(err),
                                        _ptr(keep), _ptr(kept))
        return dict(A_cur_ref=A, search_levels=sl, warp_patch=wp, errors=err, keep=keep.astype(bool), kept=kept[:k])


def ref_select_available():
    return os.path.exists(REF_SELECT_SO)


class RefSelect:
    """The reference source's own getWarpMatrixAffine + getBestSearchLevel and calculateNCC (oracle/ref_select.cpp)."""

    def __init__(self, cam, levels=4):
        self.lib = C.CDLL(REF_SELECT_SO)
        L = self.lib
        L.ref_vio_create.restype = vp
        L.ref_vio_create.argtypes = [vp] * 6
        L.ref_vio_destroy.argtypes = [vp]
        L.ref_vio_warp_matrix_affine.restype = C.c_int
        L.ref_vio_warp_matrix_affine.argtypes = [vp] * 7 + [C.c_int, vp]
        L.ref_vio_calculate_ncc.restype = C.c_double
        L.ref_vio_calculate_ncc.argtypes = [vp] * 3
        ext = S.avia_extrinsics()
        self._keep = [_a(cam.as_array()), _a(ext.extR), _a(ext.extT), _a(ext.Rcl), _a(ext.Pcl), _a(S.VioCfg(levels=levels).as_array())]
        self.h = L.ref_vio_create(*[_ptr(k) for k in self._keep])
        assert self.h

    def __del__(self):
        try:
            self.lib.ref_vio_destroy(self.h)
        except Exception:
            pass

    def warp_matrix_affine(self, px_ref, f_ref, ref_pos, pos_w, T_ref, T_cur, level_ref):
        A = np.zeros(4)
        args = [_a(px_ref), _a(f_ref), _a(ref_pos), _a(pos_w), _a(T_ref), _a(T_cur)]
        sl = self.lib.ref_vio_warp_matrix_affine(self.h, *[_ptr(x) for x in args], int(level_ref), _ptr(A))
        return A, sl

    def ncc(self, ref_patch, cur_patch):
        r, c = _a(ref_patch, np.float32), _a(cur_patch, np.float32)
        return self.lib.ref_vio_calculate_ncc(self.h, _ptr(r), _ptr(c))


# ----------------------------------------------------------------------------------------------- pin cases
PIN_CAMERAS = ("radtan", "fisheye")


def det_crossing(o, camera, thr, level_ref=0):
    """Two depth-form geometries on either side of det(A) = thr, adjacent in the bisected parameter (the current camera's
    distance along the reference ray): pure approach along the optical axis scales A by about z_ref / z_cur."""
    cam = W.CAMERAS[camera]
    px = np.array([cam.cx + 13.25, cam.cy - 7.5])
    f = W.cam2world(cam, px[:1], px[1:])[0]
    pos = f * 4.0
    T_ref = pack_T(np.eye(3), np.zeros(3))[0]

    def D(s):
        A, _ = o.warp_matrix_affine(px, f, np.zeros(3), pos, T_ref, pack_T(np.eye(3), np.array([0, 0, -s]))[0], level_ref)
        return A[0] * A[3] - A[1] * A[2]

    lo, hi = 0.0, 3.9  # D(lo) < thr < D(hi)
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if mid in (lo, hi):
            break
        lo, hi = (mid, hi) if D(mid) <= thr else (lo, mid)
    return [dict(px_ref=px, f_ref=f, ref_pos=np.zeros(3), pos_w=pos, T_ref=T_ref, T_cur=pack_T(np.eye(3), np.array([0, 0, -s]))[0], level_ref=level_ref)
            for s in (lo, hi)]


def pin_matrix_cases(o, camera):
    """Depth-form warp-matrix inputs: the random candidates at level_ref 0..2, near (0.3 m) and far (60 m) points, a
    near-singular A (reference and current rays almost parallel to the image plane) and the crossings of det = 3 and 12."""
    c = candidates(camera, 48, seed=5)
    out = []
    for i in range(48):
        out.append(dict(px_ref=c["px_ref"][i], f_ref=c["ref_f"][i], ref_pos=c["ref_pos"][i], pos_w=c["pos_w"][i], T_ref=c["T_ref"][i], T_cur=c["T_cur"],
                        level_ref=i % 3))
    for scale in (0.3, 60.0):
        for i in range(6):
            d = c["pos_w"][i] - c["ref_pos"][i]
            out.append(dict(out[i], pos_w=c["ref_pos"][i] + d / np.linalg.norm(d) * scale))
    T_side = pack_T(W._rot(np.array([0.0, 1.5707, 0.0])), np.array([0.0, 0.0, 3.0]))[0]
    out.append(dict(out[0], T_cur=T_side))
    for thr in (3.0, 12.0):
        out += det_crossing(o, camera, thr)
    return out


def pin_ncc_cases(seed=0):
    rng = np.random.default_rng(seed)
    ref = rng.uniform(0, 255, (16, 64)).astype(np.float32)
    cur = (ref * rng.uniform(0.5, 1.5, (16, 1)) + rng.normal(0, 20, (16, 64))).astype(np.float32)
    ref[0] = 77.0  # constant (zero-variance) reference patch
    cur[1] = 13.5  # constant current patch
    ref[2] = cur[2] = 0.0
    return ref, cur
