"""Inputs of the coloured scan (esikf_rgb_set_cloud / esikf_rgb_colorize: publish_frame_world, src/LIVMapper.cpp:1140-1173)
and ctypes bindings of its oracle (oracle/liborc_color.so) and of the reference source's pieces it is pinned to
(oracle/_ref/libfl2_ref_color.so), both built by oracle/color.mk.

scene(camera, n, ...) draws a body-frame LiDAR cloud around the sensor, a LIO posterior and a VIO posterior near it, and a
textured BGR image with saturated corners; edge_scene(camera) holds hand-built points on every boundary of the gates."""
import ctypes as C
import os

import numpy as np

import warp_cases as W
from fast_livo2_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORC_COLOR_SO = os.path.join(ROOT, "oracle", "liborc_color.so")
REF_COLOR_SO = os.path.join(ROOT, "oracle", "_ref", "libfl2_ref_color.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pin", "color.npz")
vp = C.c_void_p

# config 2 (avia, pinhole 640 x 512), a distorted pinhole, config 3 (HILTI22 fisheye, non-identity extrinsics)
CAMERAS = {"pinhole": (W.CAMERAS["pinhole"], S.avia_extrinsics()), "radtan": (W.CAMERAS["radtan"], S.avia_extrinsics()),
           "fisheye": (W.CAMERAS["fisheye"], S.hilti_extrinsics())}
# the hand-built cases: a pinhole whose projection of the chosen points is exact (fx = 512, z = 2 or 4, no distortion)
EDGE_CAM = S.CamCfg(width=640, height=512, fx=512.0, fy=512.0, cx=320.0, cy=256.0)
IDENTITY_EXT = S.Extrinsics(extR=np.eye(3), extT=np.zeros(3), Rcl=np.eye(3), Pcl=np.zeros(3))
EDGE_BLIND = 2.0


def _a(x, dt=np.float64):
    return None if x is None else np.ascontiguousarray(x, dtype=dt)


def _ptr(x):
    return None if x is None else x.ctypes.data


def bgr_image(cam, seed):
    """A textured B G R image with 8 x 8 blocks of 255 in all three channels at the four corners."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:cam.height, 0:cam.width]
    chans = [127.5 + 70 * np.sin(xx / (7.3 + 2 * k) + seed + k) * np.cos(yy / (5.1 + k)) + rng.normal(0, 30, (cam.height, cam.width)) for k in range(3)]
    img = np.stack(chans, 2).clip(0, 255).astype(np.uint8)
    for r in (slice(0, 8), slice(cam.height - 8, cam.height)):
        for c in (slice(0, 8), slice(cam.width - 8, cam.width)):
            img[r, c] = 255
    return img


def scene(camera, n, seed=0):
    """n body points (float32) in all directions at 0.3 to 40 m, the LIO posterior they are moved to the world with, a VIO
    posterior near it (the frame pose of the colouring) and the image."""
    cam, ext = CAMERAS[camera]
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pts = (d * rng.uniform(0.3, 40.0, (n, 1))).astype(np.float32)
    R = S.so3_exp(rng.normal(0, 0.4, 3))
    p = rng.normal(0, 2.0, 3)
    lio = S.pack_state(R, p)
    vio = S.pack_state(R @ S.so3_exp(rng.normal(0, 0.002, 3)), p + rng.normal(0, 0.01, 3), 1.02)
    return dict(camera=camera, cam=cam, ext=ext, pts=pts, lio_state=lio, vio_state=vio, img=bgr_image(cam, 50 + seed), blind=0.01)


def edge_scene():
    """World points (the state and the extrinsics are identities, so pf = p_w) on the boundaries of publish_frame_world's
    gates, with the expected keep flag of each. Pixel u of a point (x, y, z) is 512 x / z + 320 exactly."""
    pts, keep = [], []

    def px(u, v, z=4.0, k=True):
        pts.append(((u - 320.0) * z / 512.0, (v - 256.0) * z / 512.0, z))
        keep.append(k)

    pts += [(0.5, 0.2, -1.0), (0.5, 0.2, -1e-30), (0.3, 0.1, 0.0), (0.0, 0.0, 0.0)]  # behind the camera; pf[2] == 0 exactly
    keep += [False, False, False, False]
    px(-0.5, 100.0, k=False)       # pc in (-1, 0): truncates to 0, outside the border of 3
    px(100.0, -0.25, k=False)
    for u, k in ((2.75, False), (3.0, True), (3.5, True), (636.0, True), (636.99609375, True), (637.0, False), (637.5, False)):
        px(u, 200.0, k=k)          # (int)pc at 2, 3, width - 4, width - 3
    for v, k in ((2.75, False), (3.0, True), (508.0, True), (508.99609375, True), (509.0, False)):
        px(300.0, v, k=k)          # the same for rows
    for u, v in ((100.0, 200.0), (321.0, 257.0), (4.0, 4.0), (630.0, 500.0)):
        px(u, v)                   # exact integers (all weight on one tap)
    for u, v in ((4.5, 4.5), (5.25, 6.75), (633.5, 4.5), (4.5, 505.5), (634.75, 505.25)):
        px(u, v)                   # inside the saturated corners: 255 weighted by rounded weights
    pts.append((0.0, 0.0, EDGE_BLIND))                                # pf.norm() == blind_rgb_points: dropped (strict)
    keep.append(False)
    pts.append((0.0, 0.0, float(np.nextafter(np.float32(EDGE_BLIND), np.float32(3)))))  # the next float above: kept
    keep.append(True)
    pts.append((0.0, 0.0, float(np.nextafter(np.float32(EDGE_BLIND), np.float32(0)))))  # below: dropped
    keep.append(False)
    pts = np.array(pts, np.float32)
    return dict(camera="edge", cam=EDGE_CAM, ext=IDENTITY_EXT, pts=pts, lio_state=S.pack_state(np.eye(3), np.zeros(3)),
                vio_state=S.pack_state(np.eye(3), np.zeros(3)), img=bgr_image(EDGE_CAM, 7), blind=EDGE_BLIND, keep=np.array(keep))


def _cam_ext(sc):
    cam, ext = sc["cam"], sc["ext"]
    return [_a(cam.as_array()), _a(ext.extR), _a(ext.extT), _a(ext.Rcl), _a(ext.Pcl), _a(S.VioCfg().as_array())]


class _Lib:
    prefix = None

    def __init__(self, path, sc):
        self.lib = C.CDLL(path)
        L, p = self.lib, self.prefix
        getattr(L, f"{p}_color_world").argtypes = [vp] * 4 + [C.c_int, vp]
        getattr(L, f"{p}_color_colorize").restype = C.c_int
        getattr(L, f"{p}_color_colorize").argtypes = [vp, vp, C.c_int, vp, vp, C.c_double, vp, vp, vp]
        self.ext = sc["ext"]
        self._keep = _cam_ext(sc)

    def world(self, pts, state):
        pts, st = _a(pts, np.float32).reshape(-1, 3), _a(state)
        out = np.zeros_like(pts)
        eR, eT = _a(self.ext.extR), _a(self.ext.extT)
        getattr(self.lib, f"{self.prefix}_color_world")(_ptr(eR), _ptr(eT), _ptr(st), _ptr(pts), len(pts), _ptr(out))
        return out

    def colorize(self, cloud, img, state, blind):
        cloud, img, st = _a(cloud, np.float32).reshape(-1, 3), _a(img, np.uint8), _a(state)
        n = len(cloud)
        xyz, bgr, idx = np.zeros((max(n, 1), 3), np.float32), np.zeros((max(n, 1), 3), np.uint8), np.zeros(max(n, 1), np.int32)
        k = getattr(self.lib, f"{self.prefix}_color_colorize")(self.h, _ptr(cloud), n, _ptr(img), _ptr(st), float(blind), _ptr(xyz), _ptr(bgr), _ptr(idx))
        return dict(xyz=xyz[:k], bgr=bgr[:k], index=idx[:k])

    def publish(self, sc, cloud=None):
        """The whole pass on a scene: world cloud with the LIO posterior, colours with the VIO posterior."""
        world = self.world(sc["pts"], sc["lio_state"]) if cloud is None else cloud
        return dict(world=world, **self.colorize(world, sc["img"], sc["vio_state"], sc["blind"]))


class OracleColor(_Lib):
    """The oracle's restatement (oracle/orc_color.cpp) on the scene's camera and extrinsics."""
    prefix = "orc"

    def __init__(self, sc):
        super().__init__(ORC_COLOR_SO, sc)
        L = self.lib
        L.orc_vio_create.restype = vp
        L.orc_vio_create.argtypes = [vp] * 6 + [C.c_int]
        L.orc_vio_destroy.argtypes = [vp]
        self.h = L.orc_vio_create(*[_ptr(k) for k in self._keep], 1)

    def __del__(self):
        try:
            self.lib.orc_vio_destroy(self.h)
        except Exception:
            pass


def ref_color_available():
    return os.path.exists(REF_COLOR_SO)


class RefColor(_Lib):
    """The reference source's own updateFrameState / w2f / w2c / isInFrame / getInterpolatedPixel (oracle/ref_color.cpp)."""
    prefix = "ref"

    def __init__(self, sc):
        super().__init__(REF_COLOR_SO, sc)
        L = self.lib
        L.ref_vio_create.restype = vp
        L.ref_vio_create.argtypes = [vp] * 6
        L.ref_vio_destroy.argtypes = [vp]
        self.h = L.ref_vio_create(*[_ptr(k) for k in self._keep])
        assert self.h

    def __del__(self):
        try:
            self.lib.ref_vio_destroy(self.h)
        except Exception:
            pass


# ----------------------------------------------------------------------------------------------- pin cases
PIN_SCENES = ("pinhole", "radtan", "fisheye")
PIN_POINTS = 4000


def pin_scenes():
    """The scenes the oracle is pinned to the reference source on: random clouds of every camera and the hand-built set
    (also projected through each camera)."""
    out = {name: scene(name, PIN_POINTS, seed=3) for name in PIN_SCENES}
    e = edge_scene()
    out["edge"] = e
    for name in ("radtan", "fisheye"):
        cam, ext = CAMERAS[name]
        out[f"edge_{name}"] = dict(e, camera=f"edge_{name}", cam=cam, img=bgr_image(cam, 8))
    return out


PIN_KEYS = ("world", "xyz", "bgr", "index")
