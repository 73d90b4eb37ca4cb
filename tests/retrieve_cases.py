"""Inputs of the scan side of the visual sub-map retrieval (esikf_vio_retrieve_scan / esikf_vio_depth_check:
retrieveFromVisualSparseMap, src/vio.cpp:352-640) and ctypes bindings of its oracle (oracle/liborc_retrieve.so) and of the
reference source's own resetGrid + retrieveFromVisualSparseMap (oracle/_ref/libfl2_ref_retrieve.so), both built by
oracle/retrieve.mk.

scene(camera, n, ...) draws a world scan around a frame (points behind the camera and outside the image included), the frame's
state and a flat visual map whose points sit on or off the scan's surfaces (so the depth check goes both ways); edge_scene()
holds hand-built points on every boundary of the keys, the depth image and the depth check."""
import ctypes as C
import os

import numpy as np

import color_cases as CC
import generate_cases as GC
import observe_cases as OC
import warp_cases as W
from fast_livo2_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORC_RETRIEVE_SO = os.path.join(ROOT, "oracle", "liborc_retrieve.so")
REF_RETRIEVE_SO = os.path.join(ROOT, "oracle", "_ref", "libfl2_ref_retrieve.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pin", "retrieve.npz")
vp = C.c_void_p
CAMERAS = CC.CAMERAS
EDGE_CAM = CC.EDGE_CAM  # 640 x 512, fx = 512, c = (320, 256): pixel u of (x, y, z) is 512 x / z + 320 exactly
VIO_CFG = S.VioCfg(levels=1)  # the reference's retrieval warps the reference patch at every level: one keeps its taps near the point
BORDER = 10  # (patch_size_half + 1) << 1


def grid(cam):
    """initializeVIO's grid for the default vio/grid_size 5, vio/grid_n_height 17 (integer divisions included), and a border of at
    least BORDER that keeps every pixel isInFrame passes inside the grid (the reference indexes past grid_num otherwise)."""
    g = GC.grid_geometry(cam.width, cam.height, levels=1)
    b = BORDER
    while (cam.width - b - 1) // g["grid_size"] >= g["grid_n_width"] or (cam.height - b - 1) // g["grid_size"] >= g["grid_n_height"]:
        b += 1
    return dict(g, border=b)
PIN_KEYS = ("sub_keys", "grid_type", "cell_pt", "survivors")


def _a(x, dt=np.float64):
    return np.ascontiguousarray(x, dtype=dt)


def voxel_keys(p):
    """The retrieval's key of every point (:392-396): floor(c / 0.5) in double, one less when negative (-0.0 gives 0)."""
    k = np.floor(np.asarray(p, np.float64) / 0.5).astype(np.int64)
    return np.where(k < 0, k - 1, k)


def first_occurrence(keys):
    _, first = np.unique(keys, axis=0, return_index=True)
    return keys[np.sort(first)]


def flat_visual_map(pos, normal, n_obs):
    """Group visual points by the retrieval's voxel key: vkeys, vfirst, vcount and the points in voxel order."""
    k = voxel_keys(pos)
    order = np.lexsort(k.T[::-1])
    ks = k[order]
    head = np.ones(len(ks), bool)
    head[1:] = np.any(ks[1:] != ks[:-1], axis=1)
    first = np.nonzero(head)[0].astype(np.int32)
    count = np.diff(np.append(first, len(ks))).astype(np.int32)
    return dict(vkeys=_a(ks[first], np.int64), vfirst=first, vcount=count, pos=_a(pos[order]), normal=_a(normal[order]), n_obs=_a(n_obs[order], np.int32))


def scene(camera, n, seed=0, n_vis=4000):
    """n world points on a few surfaces around a frame (a VIO prior), a flat visual map of n_vis points: half on the scan's
    surfaces, a quarter 1 to 3 m in front of them, a quarter with no observation or behind the camera."""
    cam, ext = CAMERAS[camera]
    rng = np.random.default_rng(seed)
    R, p = S.so3_exp(rng.normal(0, 0.4, 3)), rng.normal(0, 2.0, 3)
    state = S.pack_state(R, p, 1.02)
    Rcw, Pcw = S.camera_pose(ext, R, p)
    # surfaces in the camera frame: bearings through the image (and some outside it) at a depth that jumps between patches
    u, v = rng.uniform(-0.2 * cam.width, 1.2 * cam.width, n), rng.uniform(-0.2 * cam.height, 1.2 * cam.height, n)
    f = W.cam2world(cam, np.clip(u, 0, cam.width - 1), np.clip(v, 0, cam.height - 1))
    f[:, :2] += np.stack([u - np.clip(u, 0, cam.width - 1), v - np.clip(v, 0, cam.height - 1)], 1) / cam.fx
    z = np.where((np.floor(u / 60) + np.floor(v / 50)) % 3 == 0, 3.0, 7.0) + rng.normal(0, 0.05, n)
    pf = f / f[:, 2:3] * z[:, None]
    back = rng.random(n) < 0.05
    pf[back] *= -1.0
    pw = (pf - Pcw) @ Rcw
    pick = rng.choice(n, n_vis, replace=False)
    q = pf[pick].copy()
    q[n_vis // 2: 3 * n_vis // 4] *= (1.0 - rng.uniform(1.0, 3.0, n_vis // 4) / np.abs(q[n_vis // 2: 3 * n_vis // 4, 2]))[:, None]
    q += rng.normal(0, 0.02, q.shape)
    n_obs = rng.integers(1, 4, n_vis)
    n_obs[3 * n_vis // 4:] = rng.integers(0, 2, n_vis - 3 * n_vis // 4)
    # normals facing the camera: the reference's homography warp of each point stays near the identity
    vis = flat_visual_map((q - Pcw) @ Rcw, (-q / np.linalg.norm(q, axis=1, keepdims=True)) @ Rcw, n_obs)
    return dict(camera=camera, cam=cam, ext=ext, state=state, pg=pw, img=OC.grey_image(cam, 30 + seed), **grid(cam), **vis)


def edge_scene():
    """Hand-built scan and visual points under the identity frame pose on a 640 x 512 pinhole (pt_c = p_w). `expect_flag`:
    the depth-check flag of every visual point that is retrieved alone in its cell, by point index."""
    nxt, prv = (lambda x: np.nextafter(x, np.inf)), (lambda x: np.nextafter(x, -np.inf))  # noqa: E731
    pts = []

    def at(u, v, z):  # a point whose pixel is (u, v) exactly
        pts.append(((u - 320.0) * z / 512.0, (v - 256.0) * z / 512.0, z))

    # keys: both sides of 0, -0.25, -0.5 and one ulp around voxel faces, behind the camera (no depth)
    for c in (-0.5, -0.25, -0.0, 0.0, prv(0.5), 0.5, nxt(0.5), prv(-0.5), nxt(-0.5), prv(-1.0), -1.0, 1e-300, -1e-300):
        pts.append((c, c, -1.0))
        pts.append((1.5, c, -2.0))
    # pt_c[2] exactly 0, one ulp above (float depth 0: the pixel stays empty), and a tiny positive depth
    pts += [(0.0, 0.0, 0.0), (0.0, 0.0, 5e-324), (1e-300, 0.0, 5e-324)]
    # int(px) at border - 1, border and width - border, height - border (only the middle one writes)
    for u in (BORDER - 1 + 0.5, BORDER + 0.25, 640 - BORDER + 0.5, 640 - BORDER - 0.5):
        at(u, 200.5, 4.0)
    for v in (BORDER - 0.75, 512 - BORDER + 0.25):
        at(300.5, v, 4.0)
    # two points on one pixel: the later one wins (100, 100) with 6 m and (200, 100) with 4 m
    at(100.5, 100.5, 4.0), at(100.25, 100.75, 6.0)
    at(200.5, 100.5, 6.0), at(200.25, 100.75, 4.0)
    # a plain 4 m depth around (300, 300), a 9 m depth only at (400, 300) with empty taps around it, and empty (500, 300)
    at(301.5, 300.5, 4.0), at(400.5, 300.5, 9.0)
    vis, flag = [], []

    def vpoint(u, v, z, f):
        vis.append(((u - 320.0) * z / 512.0, (v - 256.0) * z / 512.0, z))
        flag.append(f)

    vpoint(100.5, 103.5, 4.1, 1)            # the 6 m point won (100, 100): 1.9 m away
    vpoint(200.5, 103.5, 4.1, 0)            # the 4 m point won (200, 100)
    vpoint(300.5, 300.5, 4.5, 0)            # |4.5 - 4| = 0.5 exactly
    vpoint(300.5, 340.5, 4.0, 0)            # no depth within 4 px: empty taps
    vpoint(400.5, 300.5, 4.0, 0)            # discontinuous depth only at the centre tap
    vpoint(500.5, 300.5, 4.0, 0)            # empty
    # |pt_cam[2] - depth| = 0.75 two pixels away: std::abs(double) (an int abs would give 0)
    vpoint(140.5, 420.5, 4.0, 1)
    at(142.5, 420.5, 4.75)
    # one ulp above 0.5: 4 m two rows below
    vpoint(301.5, 260.5, nxt(4.5), 1)
    at(301.5, 262.5, 4.0)
    # two visual points of different voxels, one grid cell, the same distance from the frame (x and y swapped): a map_dist tie
    vis += [(0.49, 0.51, 20.0), (0.51, 0.49, 20.0)]
    flag += [-1, -1]
    vis = np.array(vis)
    # the scan reaches every visual voxel (a point 1 mm behind each visual point, first, so the hand-built points win their pixels)
    scan = np.concatenate([vis + np.array([0.0, 0.0, 0.001]), np.array(pts)])
    n_vis = len(vis)
    fv = flat_visual_map(vis, np.tile([0.0, 0.0, -1.0], (n_vis, 1)), np.ones(n_vis, np.int32))
    return dict(camera="edge", cam=EDGE_CAM, ext=CC.IDENTITY_EXT, state=S.pack_state(np.eye(3), np.zeros(3)), pg=scan, img=OC.grey_image(EDGE_CAM, 3),
                vis_unsorted=vis, expect_flag=np.array(flag), **grid(EDGE_CAM), **fv)


def _cam_ext(sc):
    cam, ext = sc["cam"], sc["ext"]
    return [_a(cam.as_array()), _a(ext.extR), _a(ext.extT), _a(ext.Rcl), _a(ext.Pcl), _a(VIO_CFG.as_array())]


def _grid(sc):
    return [int(sc[k]) for k in ("grid_size", "grid_n_width", "grid_n_height", "border")]


class OracleRetrieve:
    """The oracle's restatement (oracle/orc_retrieve.cpp) on the scene's camera and extrinsics, with one persistent sub_feat_map."""

    def __init__(self, sc):
        L = self.lib = C.CDLL(ORC_RETRIEVE_SO)
        L.orc_vio_create.restype = vp
        L.orc_vio_create.argtypes = [vp] * 6 + [C.c_int]
        L.orc_vio_destroy.argtypes = [vp]
        L.orc_submap_create.restype = vp
        L.orc_submap_destroy.argtypes = [vp]
        L.orc_submap_keys.restype = C.c_int
        L.orc_submap_keys.argtypes = [vp, vp]
        L.orc_submap_fill.argtypes = [vp, vp, C.c_int]
        L.orc_retrieve_scan.restype = C.c_int
        L.orc_retrieve_scan.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp]
        L.orc_retrieve_walk.restype = C.c_int
        L.orc_retrieve_walk.argtypes = [vp, vp, vp, vp, C.c_int, vp, vp, vp, C.c_int, vp, vp] + [C.c_int] * 4 + [vp] * 3
        L.orc_depth_check.argtypes = [vp, vp, vp, C.c_int, vp, vp, vp]
        self.cam = sc["cam"]
        self._keep = _cam_ext(sc)
        self.h = L.orc_vio_create(*[k.ctypes.data for k in self._keep], 1)
        self.s = L.orc_submap_create()

    def scan(self, sc, pg=None, state=None):
        pg = _a(sc["pg"] if pg is None else pg)
        st = _a(sc["state"] if state is None else state)
        keys = np.zeros((max(len(pg), 1), 3), np.int64)
        depth = np.zeros((self.cam.height, self.cam.width), np.float32)
        k = self.lib.orc_retrieve_scan(self.h, st.ctypes.data, pg.ctypes.data, len(pg), int(sc["border"]), keys.ctypes.data, depth.ctypes.data)
        assert k >= 0, "a voxel key leaves the map's key range"
        return dict(keys=keys[:k], depth=depth)

    def walk(self, sc, keys, state=None):
        """The map-side walk on the persistent sub_feat_map, with the keys inserted in the given order."""
        st = _a(sc["state"] if state is None else state)
        keys = _a(keys, np.int64).reshape(-1, 3)
        L = sc["grid_n_width"] * sc["grid_n_height"]
        out = dict(grid_type=np.zeros(L, np.uint8), cell_pt=np.zeros(L, np.int32), cell_pc=np.zeros((L, 2)))
        args = [sc[k] for k in ("vkeys", "vfirst", "vcount")]
        m = self.lib.orc_retrieve_walk(self.h, self.s, st.ctypes.data, keys.ctypes.data, len(keys), args[0].ctypes.data, args[1].ctypes.data, args[2].ctypes.data,
                                       len(args[0]), sc["pos"].ctypes.data, sc["n_obs"].ctypes.data, *_grid(sc), *[out[f].ctypes.data for f in out])
        sub = np.zeros((max(m, 1), 3), np.int64)
        self.lib.orc_submap_keys(self.s, sub.ctypes.data)
        out["sub_keys"] = sub[:m]
        return out

    def depth_check(self, sc, depth, pos, pc, state=None):
        st = _a(sc["state"] if state is None else state)
        pos, pc, depth = _a(pos).reshape(-1, 3), _a(pc).reshape(-1, 2), _a(depth, np.float32)
        flag = np.zeros(max(len(pos), 1), np.uint8)
        self.lib.orc_depth_check(self.h, st.ctypes.data, depth.ctypes.data, len(pos), pos.ctypes.data, pc.ctypes.data, flag.ctypes.data)
        return flag[:len(pos)]

    def retrieve(self, sc, state=None):
        """The whole retrieval up to the reference-feature choice: scan, walk, depth check. survivors: the retrieved points
        (cell order) past the depth check."""
        s = self.scan(sc, state=state)
        w = self.walk(sc, s["keys"], state=state)
        cells = np.nonzero(w["grid_type"])[0]
        pt = w["cell_pt"][cells]
        flag = self.depth_check(sc, s["depth"], sc["pos"][pt], w["cell_pc"][cells], state=state)
        return dict(s, **w, cells=cells, flag=flag, survivors=pt[flag == 0].astype(np.int32))

    def __del__(self):
        try:
            self.lib.orc_submap_destroy(self.s)
            self.lib.orc_vio_destroy(self.h)
        except Exception:
            pass


def ref_retrieve_available():
    return os.path.exists(REF_RETRIEVE_SO)


class RefRetrieve:
    """The reference source's own resetGrid + retrieveFromVisualSparseMap (oracle/ref_retrieve.cpp) on one VIOManager."""

    def __init__(self, sc):
        L = self.lib = C.CDLL(REF_RETRIEVE_SO)
        L.ref_vio_create.restype = vp
        L.ref_vio_create.argtypes = [vp] * 6
        L.ref_vio_destroy.argtypes = [vp]
        L.ref_retrieve.restype = C.c_int
        L.ref_retrieve.argtypes = [vp] * 4 + [C.c_int] + [vp] * 3 + [C.c_int] + [vp] * 3 + [C.c_int] * 4 + [vp] * 5
        self._keep = _cam_ext(sc)
        self.h = L.ref_vio_create(*[k.ctypes.data for k in self._keep])
        assert self.h

    def run(self, sc):
        pg = _a(sc["pg"])
        L = sc["grid_n_width"] * sc["grid_n_height"]
        out = dict(sub_keys=np.zeros((max(len(pg), 1), 3), np.int64), grid_type=np.zeros(L, np.uint8), cell_pt=np.zeros(L, np.int32),
                   survivors=np.zeros(L, np.int32))
        ns = C.c_int32(0)
        args = [sc[k] for k in ("vkeys", "vfirst", "vcount")]
        k = self.lib.ref_retrieve(self.h, _a(sc["img"], np.uint8).ctypes.data, _a(sc["state"]).ctypes.data, pg.ctypes.data, len(pg), args[0].ctypes.data,
                                  args[1].ctypes.data, args[2].ctypes.data, len(args[0]), sc["pos"].ctypes.data, sc["normal"].ctypes.data, sc["n_obs"].ctypes.data,
                                  *_grid(sc), *[out[f].ctypes.data for f in PIN_KEYS], C.byref(ns))
        out["sub_keys"] = out["sub_keys"][:k]
        out["survivors"] = out["survivors"][:ns.value]
        return out

    def __del__(self):
        try:
            self.lib.ref_vio_destroy(self.h)
        except Exception:
            pass


# ----------------------------------------------------------------------------------------------- pin cases
PIN_SCENES = ("pinhole", "radtan", "fisheye")
PIN_POINTS = 20000


def pin_scenes():
    out = {name: scene(name, PIN_POINTS, seed=5) for name in PIN_SCENES}
    out["edge"] = edge_scene()
    return out


def pin_sequence():
    """Two consecutive frames of config 2's camera for one VIOManager: the second scan is larger, so the bucket count sub_feat_map
    keeps through clear() is the first frame's."""
    return [scene("pinhole", 6000, seed=21, n_vis=1500), scene("pinhole", 30000, seed=22, n_vis=3000)]
