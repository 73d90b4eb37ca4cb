"""Inputs of the new observations of the visual sub-map in a VIO tick (esikf_vio_update_points: updateVisualMapPoints,
src/vio.cpp:908-967) and ctypes bindings of its oracle (oracle/liborc_observe.so) and of the reference source's own
updateVisualMapPoints (oracle/_ref/libfl2_ref_observe.so), both built by oracle/observe.mk.

scene(camera, n, ...) draws a sub-map seen by the camera (some entries converged), each entry's oldest observation at a pose
and pixel near the current frame's (so that every part of the add rule fires), a VIO posterior and a textured grey image;
edge_scene() holds hand-built entries on every boundary of the rule (delta_p, delta_theta, the trace test, the NaN of acos,
the pixel distance), patches whose footprint reaches the image border and observation counts around the eviction at 30."""
import ctypes as C
import math
import os
import struct

import numpy as np

import color_cases as CC
import warp_cases as W
from fast_livo2_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORC_OBSERVE_SO = os.path.join(ROOT, "oracle", "liborc_observe.so")
REF_OBSERVE_SO = os.path.join(ROOT, "oracle", "_ref", "libfl2_ref_observe.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pin", "observe.npz")
vp = C.c_void_p
CAMERAS = CC.CAMERAS
EDGE_CAM = CC.EDGE_CAM  # fx = 512, c = (320, 256), 640 x 512: pixel u of a point (x, y, z) is 512 x / z + 320 exactly
IDENTITY_EXT = CC.IDENTITY_EXT
FIELDS = ("update_flag", "entry", "pc", "patch")


def _bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def _float(b):
    return struct.unpack("<d", struct.pack("<q", b))[0]


def acos_bound():
    """The largest double x with acos(x) > 0.3 under the host's acos (bisection over the bit patterns of [0.5, 1])."""
    lo, hi = _bits(0.5), _bits(1.0)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if math.acos(_float(mid)) > 0.3:
            lo = mid
        else:
            hi = mid
    return _float(lo)


def grey_image(cam, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:cam.height, 0:cam.width]
    img = 127.5 + 60 * np.sin(xx / 5.3 + seed) * np.cos(yy / 7.1) + 25 * np.sin((2 * xx + yy) / 13.0) + rng.normal(0, 20, (cam.height, cam.width))
    return img.clip(0, 255).astype(np.uint8)


def pack_T(R, t):
    return np.concatenate([np.asarray(R).reshape(-1, 9), np.asarray(t).reshape(-1, 3)], 1)


def last_observations(Rcw, Pcw, pc, seed=0):
    """Per entry projected at pc by the frame pose (Rcw, Pcw): its oldest observation at that pose moved by a rotation of up to
    0.45 rad and a translation of up to 0.75 m, at a pixel up to 60 px from pc; 10 % of the entries are converged. n_obs
    (1 to 31), has_ref and search_levels feed the reference's object code."""
    n = len(pc)
    rng = np.random.default_rng(seed)
    ang = rng.normal(size=(n, 3))
    ang *= (rng.uniform(0, 0.45, n) / np.linalg.norm(ang, axis=1))[:, None]
    dR = W._rot(ang)
    dt = rng.normal(size=(n, 3))
    dt *= (rng.uniform(0, 0.75, n) / np.linalg.norm(dt, axis=1))[:, None]
    off = rng.normal(size=(n, 2))
    off *= (rng.uniform(0, 60.0, n) / np.linalg.norm(off, axis=1))[:, None]
    return dict(converged=(rng.random(n) < 0.1).astype(np.uint8), last_T=pack_T(dR @ Rcw, np.einsum("nij,j->ni", dR, Pcw) + dt), last_px=pc + off,
                n_obs=rng.integers(1, 32, n).astype(np.int32), has_ref=(rng.random(n) < 0.5).astype(np.uint8),
                search_levels=rng.integers(0, 3, n).astype(np.int32))


def scene(camera, n, seed=0, margin=8.0):
    """n sub-map entries in front of the frame of a VIO posterior, at least `margin` pixels inside the image, with the last
    observations of last_observations()."""
    cam, ext = CAMERAS[camera]
    rng = np.random.default_rng(seed)
    R, p = S.so3_exp(rng.normal(0, 0.4, 3)), rng.normal(0, 2.0, 3)
    state = S.pack_state(R, p, 1.02)
    Rcw, Pcw = S.camera_pose(ext, R, p)
    u, v = rng.uniform(margin, cam.width - margin, n), rng.uniform(margin, cam.height - margin, n)
    z = rng.uniform(1.0, 20.0, n)
    pf = W.cam2world(cam, u, v) * (z / W.cam2world(cam, u, v)[:, 2])[:, None]
    pos = (pf - Pcw) @ Rcw  # Rcw^T (pf - Pcw)
    return dict(camera=camera, cam=cam, ext=ext, state=state, img=grey_image(cam, 70 + seed), pos=pos,
                **last_observations(Rcw, Pcw, np.stack([u, v], 1), seed=seed + 1000))


def edge_scene():
    """Hand-built entries under an identity frame pose (pf = p_w, pose_cur = identity, so delta_pose is the oldest observation's
    pose itself) on a 640 x 512 pinhole. `expect` holds every entry's flag."""
    c_max = acos_bound()
    img = grey_image(EDGE_CAM, 9)
    pos, conv, Ts, pxs, n_obs, expect = [], [], [], [], [], []
    I = np.eye(3)

    def entry(u, v, flag, R=I, t=(0.0, 0.0, 0.0), px=None, z=4.0, converged=0, obs=3):
        pos.append(((u - 320.0) * z / 512.0, (v - 256.0) * z / 512.0, z))
        conv.append(converged), Ts.append(np.concatenate([np.asarray(R, np.float64).reshape(9), t])), n_obs.append(obs)
        pxs.append((u, v) if px is None else px)
        expect.append(flag)

    nxt = lambda x: np.nextafter(x, np.inf)  # noqa: E731
    prv = lambda x: np.nextafter(x, -np.inf)  # noqa: E731
    # nothing moved, and converged entries whatever moved
    entry(100.25, 100.5, 0)
    entry(110.5, 100.5, 0, t=(5.0, 0, 0), px=(0.0, 0.0), converged=1)
    entry(120.75, 100.5, 0, R=np.diag([-1.0, -1.0, 1.0]), converged=1)
    # delta_p = |t|: exactly 0.5, and one ulp above
    entry(130.25, 110.5, 0, t=(0.5, 0.0, 0.0))
    entry(140.25, 110.5, 1, t=(nxt(0.5), 0.0, 0.0))
    entry(150.25, 110.5, 0, t=(0.0, -0.5, 0.0))
    # the trace test: trace exactly 3 - 1e-6 (acos of 1 - 5e-7: about 1e-3) and one ulp of the trace above it (0); above 3 (0)
    T0 = 3.0 - 1e-6
    entry(160.25, 120.5, 0, R=np.diag([1.0, 1.0, T0 - 2.0]))
    entry(170.25, 120.5, 0, R=np.diag([1.0, 1.0, nxt(T0) - 2.0]))
    entry(180.25, 120.5, 0, R=np.diag([1.0, 1.5, 1.0]))
    # delta_theta = acos(0.5 * (trace - 1)) at 0.3: the largest trace whose x is at most c_max (> 0.3), and the next (<= 0.3)
    T_lo = 2.0 * c_max + 1.0
    while 0.5 * (T_lo - 1.0) > c_max:
        T_lo = prv(T_lo)
    while 0.5 * (nxt(T_lo) - 1.0) <= c_max:
        T_lo = nxt(T_lo)
    assert math.acos(0.5 * (T_lo - 1.0)) > 0.3 >= math.acos(0.5 * (nxt(T_lo) - 1.0))
    entry(190.25, 130.5, 1, R=np.diag([1.0, 1.0, T_lo - 2.0]))
    entry(200.25, 130.5, 0, R=np.diag([1.0, 1.0, nxt(T_lo) - 2.0]))
    # ... and where acos is NaN: x = -1 exactly (pi), x one ulp below -1 (trace -1 - 2^-51; a trace of -1 - 2^-52 still
    # rounds to x = -1) and far below (NaN > 0.3 is false)
    entry(210.25, 130.5, 1, R=np.diag([-1.0, -1.0, 1.0]))
    entry(215.25, 130.5, 1, R=np.diag([-1.0, -1.0, 1.0 - 2.0 ** -52]))
    entry(220.25, 130.5, 0, R=np.diag([-1.0, -1.0, 1.0 - 2.0 ** -51]))
    entry(230.25, 130.5, 0, R=np.diag([-1.0, -1.0, -1.5]))
    # a plain rotation by 0.31 rad and by 0.29 rad about an axis
    entry(240.25, 140.5, 1, R=S.so3_exp(np.array([0.0, 0.31, 0.0])))
    entry(250.25, 140.5, 0, R=S.so3_exp(np.array([0.29, 0.0, 0.0])))
    # pixel distance exactly 40, and one ulp above (du = -40, dv small enough to round onto it)
    entry(260.25, 150.5, 0, px=(300.25, 150.5))
    entry(270.25, 150.5, 0, px=(270.25, 110.5))
    dv = next(k * 2.0 ** -23 for k in range(1, 256) if math.sqrt(0.0 + 1600.0 + (150.5 - (150.5 - k * 2.0 ** -23)) ** 2) == nxt(40.0))
    entry(280.25, 150.5, 1, px=(320.25, 150.5 - dv))
    # patches whose footprint reaches the image border (the reference reads the neighbouring row there), added by distance
    for u, v in ((0.25, 200.5), (639.5, 300.25), (320.5, 4.25), (330.75, 507.25), (4.0, 6.5), (635.25, 505.75)):
        entry(u, v, 1, px=(u + 41.0, v))
    # observation counts around the eviction at 30: added and not added
    for k, obs in enumerate((29, 30, 31)):
        entry(300.25 + 10 * k, 200.5, 1, t=(0.6, 0, 0), obs=obs)
        entry(300.25 + 10 * k, 220.5, 0, obs=obs)
        entry(300.25 + 10 * k, 240.5, 0, t=(9.0, 0, 0), obs=obs, converged=1)
    n = len(pos)
    rng = np.random.default_rng(4)
    return dict(camera="edge", cam=EDGE_CAM, ext=IDENTITY_EXT, state=S.pack_state(np.eye(3), np.zeros(3)), img=img, pos=np.array(pos),
                converged=np.array(conv, np.uint8), last_T=np.array(Ts), last_px=np.array(pxs, np.float64), n_obs=np.array(n_obs, np.int32),
                has_ref=(np.arange(n) % 2).astype(np.uint8), search_levels=rng.integers(0, 3, n).astype(np.int32), expect=np.array(expect, np.uint8))


def _a(x, dt=np.float64):
    return np.ascontiguousarray(x, dtype=dt)


def _cam_ext(sc):
    cam, ext = sc["cam"], sc["ext"]
    return [_a(cam.as_array()), _a(ext.extR), _a(ext.extT), _a(ext.Rcl), _a(ext.Pcl), _a(S.VioCfg().as_array())]


def _inputs(sc):
    return [_a(sc["img"], np.uint8), _a(sc["state"]), _a(sc["pos"]), _a(sc["converged"], np.uint8), _a(sc["last_T"]), _a(sc["last_px"])]


def _outputs(n):
    return dict(update_flag=np.zeros(max(n, 1), np.uint8), entry=np.zeros(max(n, 1), np.int32), pc=np.zeros((max(n, 1), 2)),
                patch=np.zeros((max(n, 1), 64), np.float32))


class OracleObserve:
    """The oracle's restatement (oracle/orc_observe.cpp) on the scene's camera and extrinsics."""

    def __init__(self, sc):
        L = self.lib = C.CDLL(ORC_OBSERVE_SO)
        L.orc_vio_create.restype = vp
        L.orc_vio_create.argtypes = [vp] * 6 + [C.c_int]
        L.orc_vio_destroy.argtypes = [vp]
        L.orc_update_points.restype = C.c_int
        L.orc_update_points.argtypes = [vp] * 7 + [C.c_int] + [vp] * 4
        self._keep = _cam_ext(sc)
        self.h = L.orc_vio_create(*[k.ctypes.data for k in self._keep], 1)

    def run(self, sc):
        args = _inputs(sc)
        n = len(sc["converged"])
        out = _outputs(n)
        k = self.lib.orc_update_points(self.h, *[x.ctypes.data for x in args], n, *[out[f].ctypes.data for f in FIELDS])
        return dict(update_flag=out["update_flag"][:n], **{f: out[f][:k] for f in FIELDS[1:]})

    def __del__(self):
        try:
            self.lib.orc_vio_destroy(self.h)
        except Exception:
            pass


def ref_observe_available():
    return os.path.exists(REF_OBSERVE_SO)


class RefObserve:
    """The reference source's own updateVisualMapPoints (oracle/ref_observe.cpp): the flags, the new Feature's px_, patch_ and
    level_ of every added entry, and every entry's observation count after the call."""

    def __init__(self, sc):
        L = self.lib = C.CDLL(REF_OBSERVE_SO)
        L.ref_vio_create.restype = vp
        L.ref_vio_create.argtypes = [vp] * 6
        L.ref_vio_destroy.argtypes = [vp]
        L.ref_update_points.restype = C.c_int
        L.ref_update_points.argtypes = [vp] * 10 + [C.c_int] + [vp] * 6
        self._keep = _cam_ext(sc)
        self.h = L.ref_vio_create(*[k.ctypes.data for k in self._keep])
        assert self.h

    def run(self, sc):
        args = _inputs(sc) + [_a(sc["n_obs"], np.int32), _a(sc["has_ref"], np.uint8), _a(sc["search_levels"], np.int32)]
        n = len(sc["converged"])
        out = _outputs(n)
        out["level"] = np.zeros(max(n, 1), np.int32)
        out["obs_left"] = np.zeros(max(n, 1), np.int32)
        k = self.lib.ref_update_points(self.h, *[x.ctypes.data for x in args], n, *[out[f].ctypes.data for f in FIELDS + ("level", "obs_left")])
        return dict(update_flag=out["update_flag"][:n], obs_left=out["obs_left"][:n], **{f: out[f][:k] for f in FIELDS[1:] + ("level",)})

    def __del__(self):
        try:
            self.lib.ref_vio_destroy(self.h)
        except Exception:
            pass


# ----------------------------------------------------------------------------------------------- pin cases
PIN_SCENES = ("pinhole", "radtan", "fisheye")
PIN_ENTRIES = 800
PIN_KEYS = FIELDS + ("level", "obs_left")


def pin_scenes():
    """The scenes the oracle is pinned to the reference source on: random sub-maps of every camera and the hand-built entries."""
    out = {name: scene(name, PIN_ENTRIES, seed=3) for name in PIN_SCENES}
    out["edge"] = edge_scene()
    return out
