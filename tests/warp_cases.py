"""Hand-built inputs of the VIO warp producers (getWarpMatrixAffineHomography + getBestSearchLevel, warpAffine) at their
decisions, and VIO frames down to eight pyramid levels.

getBestSearchLevel picks the search level from D = det(A): one step for D > 3, two for D > 12 (the loop quarters D and
stops at 2). warpAffine inverts A through the same determinant. The reference rounds both products of a00 a11 - a01 a10;
evaluated with one FMA the determinant can land on the other side of 3 or 12, or give a different float inverse when the
products cancel. Every set below records on the A it is evaluated on how often it reaches those decisions, so the tests can
assert that the cases are really there:

  near  : |D - thr| <= 1 ulp of thr
  split : fma(a00, a11, -round(a01 a10)) (evaluated exactly) picks a different level than the rounded-products rule

a. threshold_set(camera, thr): random geometries (reference pixel, depth, plane tilt, roll, motion direction) whose current
   camera position is bisected, vectorised, to the crossing of D = thr. One ulp of the camera position moves D by tens of
   ulps (A's entries are differences of pixel coordinates near 300), so only a fraction lands within an ulp: many geometries.
b. edge_set(camera): grazing planes (D tiny, either sign), a mirrored warp (D < 0), D >> 48 (the cap of two steps), no
   motion with the plane through the reference centre (H = 0: A is NaN, level 0, the patch is left untouched) and, on the
   fisheye camera, the equidistant cam2world evaluated at the principal point.
c. caller_matrices(): matrices with entries near 2^24 whose determinant cancels by about 26 bits, kept only where the
   contracted and the rounded determinant give different float inverses; search levels 0, 1, 2 and 8.
d. deep_frame(levels): a 2048 x 2048 frame whose central patches are updated over 6 to 8 pyramid levels, 8 iterations each.

All geometry lives in the current camera's frame: T_cur_w is the identity and every case has its own reference pose, so one
vio_warp_patches call evaluates a whole set."""
import dataclasses
import functools
from fractions import Fraction

import numpy as np

from fast_livo2_b200 import synthetic as S

THRESHOLDS = (3.0, 12.0)
CAMERAS = {
    "pinhole": S.CamCfg(),
    "radtan": S.CamCfg(d=(-0.076160, 0.123001, -0.00113, 0.000251, 0.0)),
    # config 3's camera (HILTI22, vk::EquidistantCamera)
    "fisheye": S.CamCfg(model=1, width=720, height=540, fx=351.31400364193297, fy=351.4911744656785, cx=367.8522793375995, cy=253.8402144980996,
                        d=(-0.03696737352869157, -0.008917880497032812, 0.008912969593422046, -0.0037685977496087313, 0.0)),
}
N_GEOMETRIES = 34_000  # per camera and threshold, before the geometries without a crossing are dropped
T_CUR = (np.eye(3), np.zeros(3))


# ----------------------------------------------------------------------------------------------- the rule and the reach flags
def search_level(D):
    """getBestSearchLevel(A, 2) on determinants D: quartering is exact, so the loop is (D > 3) + (D > 12); NaN gives 0."""
    D = np.asarray(D, np.float64)
    return (D > 3.0).astype(np.int32) + (D > 12.0)


def det_rounded(A):
    """a00 a11 - a01 a10 with both products rounded (numpy does not contract)."""
    A = np.asarray(A, np.float64).reshape(-1, 4)
    return A[:, 0] * A[:, 3] - A[:, 1] * A[:, 2]


def det_contracted(A):
    """fma(a00, a11, -round(a01 a10)): the exact value, rounded once (Fraction -> float is correctly rounded)."""
    A = np.asarray(A, np.float64).reshape(-1, 4)
    out = np.empty(len(A))
    for i, (a00, a01, a10, a11) in enumerate(A):
        if not np.isfinite([a00, a01, a10, a11]).all():
            out[i] = a00 * a11 - a01 * a10
            continue
        out[i] = float(Fraction(a00) * Fraction(a11) - Fraction(float(a01 * a10)))
    return out


def reach(A, thr):
    """(near, split) masks of matrices A (N, 2, 2) at threshold thr."""
    D = det_rounded(A)
    near = np.abs(D - thr) <= np.spacing(thr)
    split = np.zeros(len(D), bool)
    cand = np.nonzero(np.abs(D - thr) <= 16 * np.spacing(thr))[0]  # an FMA moves D by at most an ulp of the products
    if len(cand):
        split[cand] = search_level(det_contracted(np.asarray(A).reshape(-1, 4)[cand])) != search_level(D[cand])
    return near, split


# ----------------------------------------------------------------------------------------------- numpy restatement of the producer
def cam2world(cam, u, v):
    """Unit bearings of pixels (u, v), as the device evaluates vk::*Camera::cam2world."""
    x0, y0 = (u - cam.cx) / cam.fx, (v - cam.cy) / cam.fy
    x, y = x0.copy(), y0.copy()
    d = cam.d
    if cam.model == 0:
        if abs(d[0]) > 1e-7:
            for _ in range(5):
                r2 = x * x + y * y
                icd = 1.0 / (1 + ((d[4] * r2 + d[1]) * r2 + d[0]) * r2)
                dx = 2 * d[2] * x * y + d[3] * (r2 + 2 * x * x)
                dy = d[2] * (r2 + 2 * y * y) + 2 * d[3] * x * y
                x, y = (x0 - dx) * icd, (y0 - dy) * icd
    else:
        td = np.sqrt(x0 * x0 + y0 * y0)
        th = td.copy()
        for _ in range(10):
            t2 = th * th
            t4 = t2 * t2
            th = td / (1 + d[0] * t2 + d[1] * t4 + d[2] * t4 * t2 + d[3] * t4 * t4)
        sc = np.where(td > 1e-8, np.tan(th) / np.where(td > 1e-8, td, 1.0), 1.0)
        x, y = x0 * sc, y0 * sc
    n = np.sqrt(x * x + y * y + 1.0)
    return np.stack([x / n, y / n, 1.0 / n], -1)


def world2cam(cam, P):
    with np.errstate(invalid="ignore", divide="ignore"):  # H = 0 projects 0 / 0, as on the device
        return _world2cam(cam, P)


def _world2cam(cam, P):
    x, y = P[..., 0] / P[..., 2], P[..., 1] / P[..., 2]
    d = cam.d
    if cam.model == 0:
        if abs(d[0]) > 1e-7:
            r2 = x * x + y * y
            r4 = r2 * r2
            cd = 1 + d[0] * r2 + d[1] * r4 + d[4] * r4 * r2
            a1, a2, a3 = 2 * x * y, r2 + 2 * x * x, r2 + 2 * y * y
            x, y = x * cd + d[2] * a1 + d[3] * a2, y * cd + d[2] * a3 + d[3] * a1
        return cam.fx * x + cam.cx, cam.fy * y + cam.cy
    r = np.sqrt(x * x + y * y)
    th = np.arctan(r)
    t2 = th * th
    t4 = t2 * t2
    thd = th * (1 + d[0] * t2 + d[1] * t4 + d[2] * t4 * t2 + d[3] * t4 * t4)
    sc = np.where(r > 1e-8, thd / np.where(r > 1e-8, r, 1.0), 1.0)
    return cam.fx * x * sc + cam.cx, cam.fy * y * sc + cam.cy


def warp_matrix(cam, px_ref, pos_w, normal_w, T_ref):
    """getWarpMatrixAffineHomography with T_cur_w = identity, vectorised: T_ref = (R (N, 3, 3), t (N, 3)). Returns A (N, 2, 2)."""
    Rr, tr = T_ref
    nv = np.einsum("nij,nj->ni", Rr, normal_w)
    nv /= np.linalg.norm(nv, axis=1, keepdims=True)
    pf = np.einsum("nij,nj->ni", Rr, pos_w) + tr
    R = np.transpose(Rr, (0, 2, 1))  # T_cur_ref = T_ref^-1
    t = -np.einsum("nij,nj->ni", R, tr)
    ti = -np.einsum("nji,nj->ni", R, t)
    ndx = np.sum(nv * pf, 1)
    B = ndx[:, None, None] * np.eye(3) - ti[:, :, None] * nv[:, None, :]
    H = R @ B
    f_u = cam2world(cam, px_ref[:, 0] + 4.0, px_ref[:, 1])
    f_v = cam2world(cam, px_ref[:, 0], px_ref[:, 1] + 4.0)
    cu, cv = world2cam(cam, np.einsum("nij,nj->ni", H, pf))
    uu, uv = world2cam(cam, np.einsum("nij,nj->ni", H, f_u))
    vu, vv = world2cam(cam, np.einsum("nij,nj->ni", H, f_v))
    return np.stack([(uu - cu) / 4, (vu - cu) / 4, (uv - cv) / 4, (vv - cv) / 4], 1).reshape(-1, 2, 2)


def _rot(axis_angle):
    th = np.linalg.norm(axis_angle, axis=-1, keepdims=True)
    k = axis_angle / np.where(th > 0, th, 1.0)
    K = np.zeros(axis_angle.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 2] = -k[..., 2], k[..., 1], -k[..., 0]
    K = K - np.swapaxes(K, -1, -2)
    th = th[..., None]
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


def _look_at(c, p, roll):
    """Rotations R (reference -> current camera) whose optical axis runs from c towards p, rolled by `roll`."""
    z = p - c
    z /= np.linalg.norm(z, axis=1, keepdims=True)
    a = np.where(np.abs(z[:, :1]) < 0.9, np.array([[1.0, 0, 0]]), np.array([[0, 1.0, 0]]))
    x = np.cross(a, z)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    y = np.cross(z, x)
    R = np.stack([x, y, z], 1)
    return _rot(roll[:, None] * np.array([[0, 0, 1.0]])) @ R


def _inputs(R, c, pf, n):
    """Device inputs of a geometry given in the reference camera's frame: current camera at c with X_cur = R (X_ref - c).
    The world is the current camera's frame, so T_ref_w = (R^T, c) and T_cur_w = identity."""
    pos_w = np.einsum("nij,nj->ni", R, pf - c)
    normal_w = np.einsum("nij,nj->ni", R, n)
    return dict(pos_w=pos_w, normal_w=normal_w, T_ref=(np.ascontiguousarray(np.transpose(R, (0, 2, 1))), np.ascontiguousarray(c)))


def T_ref_packed(case):
    """(N, 12) rows [R row-major, t] as vio_warp_patches takes them."""
    R, t = case["T_ref"]
    return np.ascontiguousarray(np.concatenate([R.reshape(-1, 9), t], 1))


# ----------------------------------------------------------------------------------------------- a. threshold sets
@functools.lru_cache(maxsize=None)
def threshold_set(camera, thr, n=N_GEOMETRIES, seed=0):
    """Geometries whose rounded-products determinant (as restated here) is bisected onto thr. Returns px_ref, pos_w, normal_w,
    T_ref, A (numpy's), D_bisected and the reach masks of numpy's A."""
    cam = CAMERAS[camera]
    rng = np.random.default_rng([seed, int(thr), cam.model, int(abs(cam.d[0]) > 0)])
    m = 40.0
    px = np.stack([rng.uniform(m, cam.width - m, n), rng.uniform(m, cam.height - m, n)], 1)
    depth = rng.uniform(1.0, 10.0, n)
    pf = cam2world(cam, px[:, 0], px[:, 1]) * depth[:, None]
    # plane normal: facing the reference camera, tilted by up to 60 degrees about a random axis normal to the bearing
    b = pf / depth[:, None]
    ax = np.cross(b, rng.normal(size=(n, 3)))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    nrm = np.einsum("nij,nj->ni", _rot(ax * rng.uniform(-np.pi / 3, np.pi / 3, n)[:, None]), -b)
    # the current camera moves from the reference centre towards the point (with a lateral component), looking at it
    d = 0.85 * pf + rng.normal(0, 0.08, (n, 3)) * depth[:, None]
    roll = rng.uniform(-np.pi, np.pi, n)
    rot_jitter = _rot(rng.normal(0, np.deg2rad(3.0), (n, 3)))

    def det_at(s):
        c = s[:, None] * d
        R = rot_jitter @ _look_at(c, pf, roll)
        inp = _inputs(R, c, pf, nrm)
        return det_rounded(warp_matrix(cam, px, inp["pos_w"], inp["normal_w"], inp["T_ref"])), inp

    lo, hi = np.zeros(n), np.ones(n)
    D_lo, _ = det_at(lo)
    D_hi, _ = det_at(hi)
    ok = (D_lo < thr) & (D_hi > thr)
    for _ in range(64):
        mid = 0.5 * (lo + hi)
        Dm, _ = det_at(mid)
        above = Dm > thr
        hi, lo = np.where(above, mid, hi), np.where(above, lo, mid)
    D_lo, _ = det_at(lo)
    D_hi, _ = det_at(hi)
    s = np.where(np.abs(D_lo - thr) <= np.abs(D_hi - thr), lo, hi)
    D, inp = det_at(s)
    ok &= np.isfinite(D) & (np.abs(D - thr) < 1e-9)
    idx = np.nonzero(ok)[0]
    out = dict(px_ref=np.ascontiguousarray(px[idx]), pos_w=np.ascontiguousarray(inp["pos_w"][idx]), normal_w=np.ascontiguousarray(inp["normal_w"][idx]),
               T_ref=(np.ascontiguousarray(inp["T_ref"][0][idx]), np.ascontiguousarray(inp["T_ref"][1][idx])), thr=thr, camera=camera)
    out["A"] = warp_matrix(cam, out["px_ref"], out["pos_w"], out["normal_w"], out["T_ref"])
    assert len(idx) >= 20_000, (camera, thr, len(idx))
    return out


# ----------------------------------------------------------------------------------------------- b. degenerate and edge geometries
@functools.lru_cache(maxsize=None)
def edge_set(camera):
    """Named single geometries. Returns px_ref, pos_w, normal_w, T_ref, name (list), want_level (list, None where only the
    rule on the device's own A is asserted), A (numpy's)."""
    cam = CAMERAS[camera]
    names, rows = [], []

    def add(name, px, R, c, pf, n):
        names.append(name)
        rows.append((np.asarray(px, float), np.asarray(R, float), np.asarray(c, float), np.asarray(pf, float), np.asarray(n, float)))

    px0 = np.array([cam.cx + 37.25, cam.cy - 21.5])
    pf0 = cam2world(cam, px0[:1], px0[1:])[0] * 4.0
    b0 = pf0 / np.linalg.norm(pf0)
    # a plane normal tilted 40 degrees from the bearing, and a direction inside the plane
    n0 = _rot(np.cross(b0, [0.0, 1.0, 0.0])[None] / np.linalg.norm(np.cross(b0, [0.0, 1.0, 0.0])) * np.deg2rad(40.0))[0] @ -b0
    inplane = np.cross(n0, [0.0, 1.0, 0.0])
    inplane /= np.linalg.norm(inplane)
    for sgn in (1.0, -1.0):
        for k, eps in enumerate((1e-7, 1e-9)):
            # the current camera (almost) inside the plane, looking at the point along it: the patch collapses to a line
            c = pf0 - 3.0 * inplane * (1 if k == 0 else -1) + sgn * eps * n0
            add(f"grazing_{k}", px0, None, c, pf0, n0)
    # the current camera behind the plane: the patch is seen mirrored
    add("mirrored", px0, None, pf0 + 2.0 * (-n0) + 0.5 * inplane, pf0, n0)
    # very close to the point along the bearing: D ~ (1 / 0.03)^2 >> 48
    add("det_above_48", px0, np.eye(3), 0.97 * pf0, pf0, n0)
    add("det_just_above_48", px0, np.eye(3), 0.86 * pf0, pf0, -b0)
    # no motion, plane through the reference centre: n . p_ref = 0 exactly, H = 0, A = NaN
    add("h_zero_axis", [cam.cx, cam.cy], np.eye(3), np.zeros(3), [0.0, 0.0, 5.0], [1.0, 0.0, 0.0])
    add("h_zero_offaxis", [cam.cx + 200.0, cam.cy + 400.0], np.eye(3), np.zeros(3), [1.0, 2.0, 5.0], [2.0 / np.sqrt(5), -1.0 / np.sqrt(5), 0.0])
    if cam.model == 1:
        # px_ref + (4, 0) is the principal point: theta_d = 0, the branch that skips the undistortion
        pc = np.array([cam.cx - 4.0, cam.cy])
        pfc = cam2world(cam, pc[:1], pc[1:])[0] * 3.0
        add("fisheye_principal_point", pc, None, 0.3 * pfc + np.array([0.05, -0.02, 0.0]), pfc, -pfc / np.linalg.norm(pfc))
    px = np.array([r[0] for r in rows])
    c = np.array([r[2] for r in rows])
    pf = np.array([r[3] for r in rows])
    nrm = np.array([r[4] for r in rows])
    look = _look_at(c, pf, np.full(len(rows), 0.3))
    R = np.array([r[1] if r[1].ndim == 2 else look[i] for i, r in enumerate(rows)])
    out = _inputs(R, c, pf, nrm)
    # exact inputs where the geometry is meant to be exact (H = 0 needs n . p_ref == 0 to the last bit)
    for i, nm in enumerate(names):
        if nm.startswith("h_zero"):
            out["pos_w"][i], out["normal_w"][i] = pf[i], nrm[i]
            out["T_ref"][0][i], out["T_ref"][1][i] = np.eye(3), np.zeros(3)
    out.update(px_ref=px, name=names)
    A = warp_matrix(cam, px, out["pos_w"], out["normal_w"], out["T_ref"])
    D = det_rounded(A)
    want = []
    for i, nm in enumerate(names):
        if nm.startswith("grazing"):
            assert 0 < abs(D[i]) < 1e-3, (nm, D[i])
            names[i] = nm.replace("grazing", "grazing_pos" if D[i] > 0 else "grazing_neg")
            want.append(0)
        elif nm == "mirrored":
            assert D[i] < -0.1, D[i]
            want.append(0)
        elif nm.startswith("det_"):
            assert D[i] > 48 and D[i] / 16 > 3, (nm, D[i])
            want.append(2)
        elif nm.startswith("h_zero"):
            assert np.isnan(A[i]).all(), A[i]
            want.append(0)
        else:
            want.append(None)
    assert any(nm.startswith("grazing_pos") for nm in names) and any(nm.startswith("grazing_neg") for nm in names), names
    out.update(A=A, want_level=want)
    return out


# ----------------------------------------------------------------------------------------------- c. caller matrices
CALLER_SEARCH_LEVELS = (0, 1, 2, 8)  # 8: the largest esikf_vio_warp_affine accepts
CALLER_IMAGE = (512, 640)


def float_inverse(A, det):
    id_ = 1.0 / det
    return np.stack([(A[:, 3] * id_), (-A[:, 1] * id_), (-A[:, 2] * id_), (A[:, 0] * id_)], 1).astype(np.float32)


@functools.lru_cache(maxsize=None)
def caller_matrices(n=48, seed=0):
    """(A (n, 2, 2), px_ref (n, 2), search_level (n,), ref image): entries in [2^22, 2^25), determinant about 2^21..2^23 (the
    products cancel by about 26 bits), inverse entries O(1). Only matrices whose float inverse differs between the contracted
    and the rounded determinant are kept."""
    rng = np.random.default_rng(seed)
    keep = []
    while len(keep) < n:
        m = 4000
        a00, a01, a11 = (rng.uniform(2.0 ** 23, 2.0 ** 24, m) * rng.choice([-1.0, 1.0], m) for _ in range(3))
        T = rng.uniform(2.0 ** 21, 2.0 ** 23, m) * rng.choice([-1.0, 1.0], m)
        a10 = (a00 * a11 - T) / a01
        A = np.stack([a00, a01, a10, a11], 1)
        fu = float_inverse(A, det_rounded(A))
        cand = np.nonzero((np.abs(det_rounded(A)) > 2.0 ** 20) & (np.abs(a10) >= 2.0 ** 22) & (np.abs(a10) < 2.0 ** 25))[0]
        fc = float_inverse(A[cand], det_contracted(A[cand]))
        diff = cand[(fc != fu[cand]).any(1)]
        keep.extend(A[diff].tolist())
    A = np.array(keep[:n]).reshape(n, 2, 2)
    assert (float_inverse(A.reshape(n, 4), det_rounded(A)) != float_inverse(A.reshape(n, 4), det_contracted(A))).any(1).all()
    h, w = CALLER_IMAGE
    px = np.stack([rng.uniform(0.35 * w, 0.65 * w, n), rng.uniform(0.35 * h, 0.65 * h, n)], 1)
    sl = np.array([CALLER_SEARCH_LEVELS[i % len(CALLER_SEARCH_LEVELS)] for i in range(n)], np.int32)
    # integer arithmetic only: the stored digests of the reference's warps must not depend on a platform's sin / cos
    yy, xx = np.mgrid[0:h, 0:w]
    img = ((xx * 7 + yy * 13) % 97 + (xx // 5 + yy // 3) % 61 + rng.integers(0, 97, (h, w))).astype(np.uint8)
    return A, px, sl, img


def samples_inside(A, px, sl, h, w):
    """Per matrix: how many of its level-0 samples land inside [0, w-1) x [0, h-1) (float arithmetic of warpAffine)."""
    inv = float_inverse(A.reshape(-1, 4), det_rounded(A))
    g = np.arange(8, dtype=np.float32) - 4
    X, Y = np.meshgrid(g, g)
    s = (2.0 ** sl).astype(np.float32)[:, None, None]
    u = inv[:, 0, None, None] * (X * s) + inv[:, 1, None, None] * (Y * s) + px[:, 0, None, None].astype(np.float32)
    v = inv[:, 2, None, None] * (X * s) + inv[:, 3, None, None] * (Y * s) + px[:, 1, None, None].astype(np.float32)
    return ((u >= 0) & (v >= 0) & (u < w - 1) & (v < h - 1)).sum((1, 2))


# ----------------------------------------------------------------------------------------------- d. deep frames
DEEP_CAM = S.CamCfg(width=2048, height=2048, fx=1400.0, fy=1400.0, cx=1023.5, cy=1024.5)
DEEP_BASE = dict(seed=21, n_pts=1000, n_map=100_000, n_patches=40, scene_scale=0.5, cam=DEEP_CAM, vio=S.VioCfg(levels=4, img_point_cov=1000.0))
DEEP_LEVELS = (6, 7, 8)


def _prior(fr, seed=3):
    rng = np.random.default_rng(seed)
    t = S.unpack_state(fr["state_true"])
    return S.pack_state(t["R"] @ S.so3_exp(rng.normal(0, np.deg2rad(0.15), 3)), t["p"] + rng.normal(0, 0.01, 3), 1.0 + rng.normal(0, 0.01), t["v"], g=t["g"],
                        cov=S.random_prior_cov(rng, scale=0.2))


def in_buffer(px, search_levels, levels, width, height, margin=16.0):
    """Per patch: every tap index of updateState's footprint (all levels, anchors of px moved by up to `margin` px) lies inside
    the image buffer [0, w·h)."""
    import vio_border as VB

    ok = np.ones(len(px), bool)
    for du in (-margin, margin):
        for dv in (-margin, margin):
            q = px + np.array([du, dv])
            for lvl in range(levels):
                x0, x1, y0, y1 = VB.footprint_box(q, 1 << (lvl + np.asarray(search_levels)))
                ok &= (y0 * width + x0 >= 0) & (y1 * width + x1 < width * height)
    return ok


def deep_frame(levels, pinned=False, n=96, seed=0):
    """A frame updated over `levels` pyramid levels with 8 iterations each: n central patches (prior projections within 300 px
    of the centre) with search levels 0, 1, 2 in turn. pinned=True keeps only the patches whose every tap index lies inside the
    image buffer (the reference reads outside it otherwise), which at 8 levels leaves search level 0."""
    from conftest import get_frame
    import vio_border as VB

    fr = get_frame(**DEEP_BASE)
    vcfg = dataclasses.replace(fr["vio_cfg"], levels=levels, max_iterations=8)
    fr = dict(fr, vio_cfg=vcfg)
    prior = _prior(fr)
    rng = np.random.default_rng([seed, levels])
    cam = fr["cam_cfg"]
    px = np.stack([rng.uniform(cam.cx - 300, cam.cx + 300, n), rng.uniform(cam.cy - 300, cam.cy + 300, n)], 1)
    sl = (np.arange(n) % 3).astype(np.int32)
    inb = in_buffer(px, sl, levels, cam.width, cam.height)
    if pinned:
        px, sl, inb = px[inb], sl[inb], inb[inb]
        assert len(px) >= 24 and inb.all()
    pt = VB.patches_at(fr, prior, px, sl)
    pt["inv_ref_expo"] = np.ones(len(px))
    pt["in_buffer"] = inb
    return fr, prior, pt
