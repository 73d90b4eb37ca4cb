"""Inputs of the new visual map points of a VIO tick (esikf_vio_generate_points: generateVisualMapPoints, src/vio.cpp:804-906)
and ctypes bindings of its oracle (oracle/liborc_generate.so) and of the reference source's own generateVisualMapPoints
(oracle/_ref/libfl2_ref_generate.so), both built by oracle/generate.mk.

scene(camera, n, ...) draws a pv list seen by the camera (float-narrowed world points, normals with some zero, random var), an
add_from list, a TYPE_MAP mask, a VIO posterior and a textured grey image with a flat block; edge_scene(border) holds
hand-built points on every boundary of the pass (ties, flat patches, border and cell edges, zero normals, TYPE_MAP cells,
add_from ties and wins)."""
import ctypes as C
import os

import numpy as np

import color_cases as CC
from fast_livo2_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORC_GENERATE_SO = os.path.join(ROOT, "oracle", "liborc_generate.so")
REF_GENERATE_SO = os.path.join(ROOT, "oracle", "_ref", "libfl2_ref_generate.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pin", "generate.npz")
ADD_FROM = 0x40000000
vp = C.c_void_p
CAMERAS = CC.CAMERAS
EDGE_CAM = CC.EDGE_CAM  # fx = 512, c = (320, 256), 640 x 512: pixel u of a point (x, y, z) is 512 x / z + 320 exactly
IDENTITY_EXT = CC.IDENTITY_EXT
FIELDS = ("source", "cell", "pos", "pc", "score", "normal", "var", "patch")


def grid_geometry(width, height, grid_size=5, grid_n_height=17, levels=4):
    """grid_size, grid_n_width, grid_n_height, border as initializeVIO (vio.cpp:66-80, 154) leaves them from the vio/grid_size
    and vio/grid_n_height parameters (LIVMapper.cpp:66-67 defaults), integer divisions included."""
    if grid_size > 10:
        gw, gh = width // grid_size, height // grid_size
    else:
        grid_size = height // grid_n_height
        gh, gw = height // grid_size, width // grid_size
    return dict(grid_size=grid_size, grid_n_width=gw, grid_n_height=gh, border=5 * (1 << levels))


def grey_image(cam, seed):
    """Texture of several scales with noise, and a flat block (shiTomasiScore 0) in the middle of the image."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:cam.height, 0:cam.width]
    img = 127.5 + 60 * np.sin(xx / 6.1 + seed) * np.cos(yy / 4.3) + 30 * np.sin((xx + 2 * yy) / 17.0) + rng.normal(0, 25, (cam.height, cam.width))
    img = img.clip(0, 255).astype(np.uint8)
    img[200:260, 300:360] = 128
    return img


def _rot(rng, s):
    return S.so3_exp(rng.normal(0, s, 3))


def scene(camera, n, seed=0, n_add=300, map_share=0.15, geometry=None):
    """n scan points (about 90 % in front of the camera), n_add add_from points, the mask and the VIO posterior."""
    cam, ext = CAMERAS[camera]
    rng = np.random.default_rng(seed)
    R, p = _rot(rng, 0.4), rng.normal(0, 2.0, 3)
    state = S.pack_state(R, p, 1.02)
    Rcw, Pcw = S.camera_pose(ext, R, p)

    def in_view(k):
        u, v = rng.uniform(-40, cam.width + 40, k), rng.uniform(-40, cam.height + 40, k)
        z = rng.uniform(0.5, 30.0, k)
        pf = np.stack([(u - cam.cx) / cam.fx * z, (v - cam.cy) / cam.fy * z, z], 1)
        return (pf - Pcw) @ Rcw  # Rcw^T (pf - Pcw)

    pts = in_view(n)
    far = rng.random(n) < 0.1
    pts[far] = rng.normal(0, 15.0, (int(far.sum()), 3))
    point_w = pts.astype(np.float32).astype(np.float64)  # the pv list holds float-narrowed world points
    normal = rng.normal(size=(n, 3))
    normal /= np.linalg.norm(normal, axis=1, keepdims=True)
    normal[rng.random(n) < 0.05] = 0.0
    a = rng.normal(0, 0.01, (n, 3, 3))
    var = a @ a.transpose(0, 2, 1)
    add_pos = in_view(n_add)
    add_normal = rng.normal(size=(n_add, 3))
    g = geometry or grid_geometry(cam.width, cam.height)
    mask = (rng.random(g["grid_n_width"] * g["grid_n_height"]) < map_share).astype(np.uint8)
    return dict(camera=camera, cam=cam, ext=ext, state=state, img=grey_image(cam, 40 + seed), point_w=point_w, normal=normal, var=var, add_pos=add_pos,
                add_normal=add_normal, mask=mask, **g)


def edge_scene(border=80):
    """Hand-built points under identity poses (pf = p_w) on a 640 x 512 pinhole with 30-pixel cells (21 x 17) and the given
    border. Each entry of `expect` names a cell and the source that must win it (None: the cell gets no point)."""
    g = dict(grid_size=30, grid_n_width=21, grid_n_height=17, border=border)
    img = grey_image(EDGE_CAM, 5)
    pts, nrm, add, add_nrm = [], [], [], []
    up, down = (0.0, 0.0, -1.0), (0.0, 0.0, 1.0)  # towards / away from the camera: cos_theta < 0 flips the second

    def w(u, v, z=4.0):
        return ((u - 320.0) * z / 512.0, (v - 256.0) * z / 512.0, z)

    def scan(u, v, z=4.0, n=down):
        pts.append(w(u, v, z)), nrm.append(n)
        return len(pts) - 1

    def add_from(u, v, z=4.0, n=down):
        add.append(w(u, v, z)), add_nrm.append(n)
        return ADD_FROM | (len(add) - 1)

    cell = lambda u, v: int(v / 30) * 21 + int(u / 30)  # noqa: E731
    mask = np.zeros(21 * 17, np.uint8)
    expect = {}
    # exact ties in one cell: the same pixel at three depths, the first wins; normals both ways
    a = scan(100.25, 100.5, 2.0, up)
    scan(100.25, 100.5, 4.0)
    scan(100.25, 100.5, 8.0, up)
    expect[cell(100.25, 100.5)] = a
    # a flat patch (score 0) alone in its cell: no point
    scan(330.0, 230.0)
    expect[cell(330.0, 230.0)] = None
    # zero normals are skipped (even the better pixel), the rest of the cell competes
    pts.append(w(130.0, 130.0)), nrm.append((0.0, 0.0, 0.0))
    pts.append(w(131.0, 131.0)), nrm.append((-0.0, 0.0, -0.0))
    scan(134.0, 134.0)
    # a TYPE_MAP cell
    scan(190.5, 190.5)
    mask[cell(190.5, 190.5)] = 1
    expect[cell(190.5, 190.5)] = None
    if border > 0:
        # (int)pc on the border: border and width - border - 1 are in, one pixel further is out; rows the same
        for u, v in ((border, 250.0), (border - 0.25, 280.0), (639.0 - border + 0.75, 250.0), (640.0 - border, 280.0), (250.0, border), (280.0, border - 0.5),
                     (250.0, 511.0 - border + 0.5), (280.0, 512.0 - border)):
            scan(u, v)
    else:
        # negative pixel coordinates truncate to 0 and pass isInFrame(·, 0); the score is 0 there (its box leaves the image)
        for u, v in ((-0.75, 100.0), (100.0, -0.5), (-0.25, -0.25)):
            scan(u, v)
    # cell edges: 30 pixels is the first pixel of the next cell
    for u, v in ((390.0, 400.0), (389.75, 400.0), (400.0, 390.0), (400.0, 389.875)):
        scan(u, v)
    # add_from: a tie with the scan winner keeps it, a better pixel in the same cell replaces it, an empty cell takes the first
    # of two tied add_from points, a TYPE_MAP cell stays empty
    b = scan(460.5, 300.5)
    add_from(460.5, 300.5, 2.0)
    expect[cell(460.5, 300.5)] = b
    scan(460.5, 150.5)
    add_from(470.25, 160.5)
    c = add_from(475.0, 165.0, 4.0, up)
    add_from(475.0, 165.0, 8.0)
    d = add_from(200.5, 320.5, 4.0, up)
    add_from(200.5, 320.5, 2.0)
    expect[cell(200.5, 320.5)] = d
    add_from(250.5, 440.5)
    mask[cell(250.5, 440.5)] = 1
    expect[cell(250.5, 440.5)] = None
    # fill up with points of ordinary cells
    rng = np.random.default_rng(border)
    taken = {cell(512.0 * x / z + 320.0, 512.0 * y / z + 256.0) for x, y, z in pts + add}
    for u, v in rng.uniform(100, 400, (40, 2)):
        if cell(u, v) not in taken:
            scan(float(u), float(v), float(rng.uniform(1, 9)), up if rng.random() < 0.5 else down)
    n = len(pts)
    rng = np.random.default_rng(11)
    a = rng.normal(0, 0.01, (n, 3, 3))
    return dict(camera=f"edge{border}", cam=EDGE_CAM, ext=IDENTITY_EXT, state=S.pack_state(np.eye(3), np.zeros(3)), img=img,
                point_w=np.array(pts, np.float64), normal=np.array(nrm, np.float64), var=a @ a.transpose(0, 2, 1), add_pos=np.array(add, np.float64).reshape(-1, 3),
                add_normal=np.array(add_nrm, np.float64).reshape(-1, 3), mask=mask, expect=expect, c_add=c, **g)


def truncated(sc, n):
    """The scene with its first n scan points only (pg.size() <= 10 returns before add_from is looked at)."""
    return dict(sc, camera=f"{sc['camera']}_n{n}", point_w=sc["point_w"][:n], normal=sc["normal"][:n], var=sc["var"][:n])


def _a(x, dt=np.float64):
    return None if x is None else np.ascontiguousarray(x, dtype=dt)


def _ptr(x):
    return None if x is None else x.ctypes.data


def _cam_ext(sc):
    cam, ext = sc["cam"], sc["ext"]
    return [_a(cam.as_array()), _a(ext.extR), _a(ext.extT), _a(ext.Rcl), _a(ext.Pcl), _a(S.VioCfg().as_array())]


def _inputs(sc):
    n = len(sc["point_w"])
    return [_a(sc["img"], np.uint8), _a(sc["state"]), _a(sc["point_w"]), _a(sc["normal"]), _a(np.reshape(sc["var"], (n, 9))), n, _a(sc["add_pos"]),
            _a(sc["add_normal"]), len(sc["add_pos"]), _a(sc["mask"], np.uint8), sc["grid_size"], sc["grid_n_width"], sc["grid_n_height"], sc["border"]]


def _outputs(L, fields):
    shapes = dict(source=((L,), np.int32), cell=((L,), np.int32), pos=((L, 3), np.float64), pc=((L, 2), np.float64), score=((L,), np.float32),
                  normal=((L, 3), np.float64), var=((L, 3, 3), np.float64), patch=((L, 64), np.float32))
    return {f: np.zeros(*shapes[f]) for f in fields}


def _call(fn, h, sc, fields):
    args = _inputs(sc)
    L = sc["grid_n_width"] * sc["grid_n_height"]
    out = _outputs(L, fields)
    k = fn(h, *[_ptr(x) if isinstance(x, np.ndarray) or x is None else x for x in args], *[_ptr(out[f]) for f in fields])
    return {f: v[:k] for f, v in out.items()}


_ARGS = [vp] * 6 + [C.c_int, vp, vp, C.c_int, vp] + [C.c_int] * 4


class OracleGenerate:
    """The oracle's restatement (oracle/orc_generate.cpp) on the scene's camera and extrinsics."""

    def __init__(self, sc):
        L = self.lib = C.CDLL(ORC_GENERATE_SO)
        L.orc_vio_create.restype = vp
        L.orc_vio_create.argtypes = [vp] * 6 + [C.c_int]
        L.orc_vio_destroy.argtypes = [vp]
        L.orc_generate_points.restype = C.c_int
        L.orc_generate_points.argtypes = _ARGS + [vp] * 8
        self._keep = _cam_ext(sc)
        self.h = L.orc_vio_create(*[_ptr(k) for k in self._keep], 1)

    def run(self, sc):
        return _call(self.lib.orc_generate_points, self.h, sc, FIELDS)

    def __del__(self):
        try:
            self.lib.orc_vio_destroy(self.h)
        except Exception:
            pass


def ref_generate_available():
    return os.path.exists(REF_GENERATE_SO)


class RefGenerate:
    """The reference source's own generateVisualMapPoints (oracle/ref_generate.cpp): everything but the source index."""
    fields = tuple(f for f in FIELDS if f != "source")

    def __init__(self, sc):
        L = self.lib = C.CDLL(REF_GENERATE_SO)
        L.ref_vio_create.restype = vp
        L.ref_vio_create.argtypes = [vp] * 6
        L.ref_vio_destroy.argtypes = [vp]
        L.ref_generate_points.restype = C.c_int
        L.ref_generate_points.argtypes = _ARGS + [vp] * 7
        self._keep = _cam_ext(sc)
        self.h = L.ref_vio_create(*[_ptr(k) for k in self._keep])
        assert self.h

    def run(self, sc):
        return _call(self.lib.ref_generate_points, self.h, sc, self.fields)

    def __del__(self):
        try:
            self.lib.ref_vio_destroy(self.h)
        except Exception:
            pass


# ----------------------------------------------------------------------------------------------- pin cases
PIN_SCENES = ("pinhole", "radtan", "fisheye")
PIN_POINTS = 6000


def pin_scenes():
    """The scenes the oracle is pinned to the reference source on: random scans of every camera, the hand-built sets with a
    border of 80 and of 0, and a scene cut to 10 and to 11 scan points."""
    out = {name: scene(name, PIN_POINTS, seed=3) for name in PIN_SCENES}
    for border in (80, 0):
        e = edge_scene(border)
        out[e["camera"]] = e
    small = scene("pinhole", 11, seed=6, n_add=40, map_share=0.0)
    for n in (10, 11):
        t = truncated(small, n)
        out[t["camera"]] = t
    return out


PIN_KEYS = RefGenerate.fields
