"""The patch scoring of updateReferencePatch (src/vio.cpp:1036-1097, esikf_vio_score_ref_patches): hand-built observation
sets at every edge of the scoring, the oracle's restatement (oracle/orc_refpatch.cpp), a numpy spelling of it, and the
reference source's own updateReferencePatch (oracle/_ref/libfl2_ref_refpatch.so), all built by oracle/refpatch.mk.

A case is a dict of the call's inputs: first (n + 1 offsets), pos / normal (n x 3), and per observation patch (m x 64 float32),
mean (float32 mean_), id (int32 id_) and T (m x 12: R row-major, then t)."""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORC_SO = os.path.join(ROOT, "oracle", "liborc_refpatch.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libfl2_ref_refpatch.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pin", "refpatch.npz")
INPUTS = ("first", "pos", "normal", "patch", "mean", "id", "T")
F32_1E6 = np.float32(1e-6)  # 9.99999997e-07: below the double 1e-6, so a cached mean_ of this value is recomputed
vp = C.c_void_p


def _a(x, dt):
    return np.ascontiguousarray(x, dtype=dt)


def rot(axis, ang):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def concat(points):
    """One case from a list of points, each a dict pos, normal, patch (k x 64), mean (k), id (k), T (k x 12)."""
    first = np.concatenate([[0], np.cumsum([len(p["patch"]) for p in points])]).astype(np.int32)
    return dict(first=first, pos=_a([p["pos"] for p in points], np.float64).reshape(-1, 3), normal=_a([p["normal"] for p in points], np.float64).reshape(-1, 3),
                patch=_a(np.concatenate([p["patch"] for p in points]) if points else np.zeros((0, 64)), np.float32).reshape(-1, 64),
                mean=_a(np.concatenate([p["mean"] for p in points]) if points else [], np.float32),
                id=_a(np.concatenate([p["id"] for p in points]) if points else [], np.int32),
                T=_a(np.concatenate([p["T"] for p in points]) if points else np.zeros((0, 12)), np.float64).reshape(-1, 12))


def views(rng, k, pos, spread=0.4):
    """k camera poses T_f_w (R, t) looking at pos from about 3 m, rotated up to `spread` rad about random axes."""
    T = np.zeros((k, 12))
    for j in range(k):
        R = rot(rng.normal(size=3), rng.uniform(0, spread))
        t = np.array([0.0, 0.0, 3.0]) + rng.normal(0, 0.3, 3) - R @ pos
        T[j] = np.concatenate([R.reshape(9), t])
    return T


def zero_sum_patch(rng, scale=30.0):
    """64 float32 taps whose double sum is exactly 0 (32 values and their negatives, shuffled): mean_ computes to 0."""
    v = (rng.normal(0, scale, 32)).astype(np.float32)
    p = np.concatenate([v, -v])
    return p[rng.permutation(64)]


def small_mean_patch(rng, scale=30.0, delta=None):
    """A zero-sum patch with one tap moved so that the mean is nonzero and below 1e-6 in magnitude (either sign)."""
    p = zero_sum_patch(rng, scale)
    delta = rng.choice([-1, 1]) * rng.uniform(5e-6, 6e-5) if delta is None else delta
    k = int(np.argmin(np.abs(p)))  # the faintest tap: its ulp is far below delta
    p[k] = np.float32(p[k] + delta)
    m = np.float32(np.float32(p.astype(np.float64).sum()) / np.float32(64))
    assert m != 0 and abs(float(m)) < 1e-6, m
    return p


def point(rng, k, kind="zero", ids=None, mean_in=0.0, scale=30.0):
    pos = rng.uniform(-2, 2, 3)
    nrm = rng.normal(size=3)
    nrm /= np.linalg.norm(nrm)
    make = zero_sum_patch if kind == "zero" else small_mean_patch
    patch = np.stack([make(rng, scale) for _ in range(k)])
    return dict(pos=pos, normal=nrm, patch=patch, mean=np.full(k, mean_in, np.float32), id=np.arange(k, dtype=np.int32) + 100 if ids is None else np.asarray(ids, np.int32),
                T=views(rng, k, pos))


def tie_point(rng, k=8):
    """Two adjacent identical observations (same patch, same pose, different ids) seen head-on along the normal: their running
    sums see the same sequence of other patches, so their scores tie exactly, and their cosine of 1 puts the tie on top."""
    p = point(rng, k)
    pos = p["pos"]
    R = rot(rng.normal(size=3), 0.2)
    t = np.array([0.0, 0.0, 3.0]) - R @ pos
    p["normal"] = R.T @ np.array([0.0, 0.0, 1.0])  # R normal = +z, the viewing ray of pos in that frame
    T2 = np.concatenate([R.reshape(9), t])
    a = 2 + int(rng.integers(0, k - 3))
    p["T"][a] = p["T"][a + 1] = T2
    p["patch"][a + 1] = p["patch"][a]
    return p


def pin_case():
    """The inputs on which the reference's scoring is defined (every mean_ is below 1e-6 and recomputes below 1e-6, so ref_mean
    and other_mean are assigned at every read), one point per property: zero-sum and sub-1e-6-mean patches; 6, 7, 30 and 64
    observations; ids shared by some observations (a reduced count) and by all (count 0: every score NaN, nothing chosen); a
    flat zero patch (0 / 0), patches so faint that d1 * d2 underflows (x / 0 = inf); exact score ties; cached means of +-0,
    +-1e-6f and below; and random sets."""
    rng = np.random.default_rng(20)
    pts = []
    for k in (6, 7, 30, 64):
        pts.append(point(rng, k, "zero"))
        pts.append(point(rng, k, "small"))
    p = point(rng, 12, "zero", ids=[5, 5, 6, 7, 7, 7, 8, 9, 9, 10, 11, 5])
    pts.append(p)
    pts.append(point(rng, 9, "small", ids=[3, 4, 3, 4, 3, 4, 3, 4, 5]))
    pts.append(point(rng, 7, "zero", ids=[42] * 7))  # count 0 for every observation
    p = point(rng, 8, "zero")
    p["patch"][0] = 0.0  # flat: the first pair of every other observation is 0 / 0
    pts.append(p)
    p = point(rng, 8, "zero")
    p["patch"][3] = 0.0
    pts.append(p)
    pts.append(point(rng, 6, "zero", scale=1e-13))  # d1 * d2 underflows to 0 while up does not: inf
    p = point(rng, 10, "zero")
    p["patch"][4] = zero_sum_patch(rng, 1e-13)
    pts.append(p)
    for _ in range(4):
        pts.append(tie_point(rng, int(rng.integers(7, 14))))
    for m_in in (F32_1E6, -F32_1E6, 5e-7, -5e-7, -0.0, 1e-30):  # cached means that are recomputed
        pts.append(point(rng, int(rng.integers(6, 12)), "small", mean_in=m_in))
    for _ in range(30):
        pts.append(point(rng, int(rng.integers(6, 31)), "zero" if rng.random() < 0.5 else "small", scale=float(rng.choice([1.0, 30.0, 255.0]))))
    return concat(pts)


def mean_case():
    """Inputs for mean_ alone (the reference's scores read uninitialised means here): real-intensity patches (0..255) with
    mean_ 0, and cached means just below and just above 1e-6 in magnitude, both signs, on zero-sum and real patches."""
    rng = np.random.default_rng(21)
    pts = []
    above = np.nextafter(F32_1E6, np.float32(1))
    edge = [F32_1E6, above, -F32_1E6, -above, np.float32(1e-6 * 0.999), np.float32(2e-6), np.float32(-2e-6), 0.0, -0.0, 127.25, -3.5]
    for m_in in edge:
        p = point(rng, 6, "zero", mean_in=m_in)
        p["patch"][1::2] = rng.integers(0, 256, (3, 64)).astype(np.float32)
        pts.append(p)
    for _ in range(20):
        p = point(rng, int(rng.integers(6, 31)), "zero")
        p["patch"] = rng.integers(0, 256, p["patch"].shape).astype(np.float32)
        pts.append(p)
    return concat(pts)


def gpu_only_case():
    """Counts the reference skips (fewer than 6 observations) and well above the eviction limit: 1 to 5, 31 to 33, 100, 200."""
    rng = np.random.default_rng(22)
    pts = [point(rng, k, "zero" if k % 2 else "small") for k in (1, 2, 3, 4, 5, 31, 32, 33, 100, 200)]
    for k in (1, 5, 40):
        p = point(rng, k, "zero")
        p["patch"] = rng.integers(0, 256, p["patch"].shape).astype(np.float32)
        p["mean"] = (p["patch"].astype(np.float64).sum(1).astype(np.float32) / np.float32(64)).astype(np.float32)
        pts.append(p)
    return concat(pts)


K_FRAMES = 30


def realistic_case(ctx, n_points, seed, lo=6, hi=30):
    """n_points visual points of the PINHOLE keyframe frame (replicas of its 1000 points), each observed in lo..hi of
    K_FRAMES keyframes that see it, in a random list order; the patches cut from those keyframes' images by the device's
    image_patch_kernel at level 0; id_ the keyframe's; mean_ 0 for about half the observations and the patch's own mean for
    the rest (cached: real intensities have means far above 1e-6). ctx: an api.Context, whose camera and image this sets."""
    import keyframe_cases as KC
    from conftest import get_frame
    from fast_livo2_b200 import synthetic as S

    fr = get_frame(**KC.PINHOLE)
    poses, _, imgs = KC.keyframes(fr, K_FRAMES, seed=7)
    cam = fr["cam_cfg"]
    ctx.vio_set_camera(cam, fr["vio_cfg"])
    pos_all, nrm_all = fr["vis_pos"], fr["vis_normal"]
    b = 8
    pc = np.stack([pos_all @ R.T + P for R, P in poses])
    px = np.stack([S.cam_project(cam, p) for p in pc])
    ok = (pc[..., 2] > 0.1) & (px[..., 0] > b) & (px[..., 0] < cam.width - b) & (px[..., 1] > b) & (px[..., 1] < cam.height - b)
    rng = np.random.default_rng(seed)
    pts, counts, obs = [], [], []  # obs: (keyframe, point index into pos_all) per observation, point by point
    for j in range(10 * n_points):
        if len(pts) == n_points:
            break
        p = j % len(pos_all)
        see = np.nonzero(ok[:, p])[0]
        if len(see) < lo:
            continue
        k = int(rng.integers(lo, min(hi, len(see)) + 1))
        pts.append(p), counts.append(k)
        obs += [(int(f), p) for f in rng.permutation(see)[:k]]
    assert len(pts) == n_points
    obs = np.array(obs)
    patch = np.zeros((len(obs), 64), np.float32)
    for f in range(K_FRAMES):
        sel = np.nonzero(obs[:, 0] == f)[0]
        if len(sel):
            ctx.vio_set_image(imgs[f])
            patch[sel] = ctx.vio_get_image_patch(px[f, obs[sel, 1]], 0)
    own = (patch.astype(np.float64).sum(1).astype(np.float32) / np.float32(64)).astype(np.float32)
    mean = np.where(rng.random(len(obs)) < 0.5, own, np.float32(0)).astype(np.float32)
    first = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    T = np.stack([np.concatenate([poses[f][0].reshape(9), poses[f][1]]) for f in obs[:, 0]])
    return dict(first=first, pos=np.ascontiguousarray(pos_all[pts]), normal=np.ascontiguousarray(nrm_all[pts]), patch=patch, mean=mean,
                id=(1000 + obs[:, 0]).astype(np.int32), T=T)


# ----------------------------------------------------------------------------------------------- the oracle and the reference
def oracle(c):
    L = C.CDLL(ORC_SO)
    L.orc_score_ref_patches.argtypes = [C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    n, m = len(c["first"]) - 1, len(c["patch"])
    out = dict(score=np.zeros(max(m, 1), np.float32), mean=np.zeros(max(m, 1), np.float32), ref=np.zeros(max(n, 1), np.int32))
    ins = [_a(c["first"], np.int32), _a(c["pos"], np.float64), _a(c["normal"], np.float64), _a(c["patch"], np.float32), _a(c["mean"], np.float32),
           _a(c["id"], np.int32), _a(c["T"], np.float64)]
    L.orc_score_ref_patches(n, *[x.ctypes.data for x in ins], out["score"].ctypes.data, out["mean"].ctypes.data, out["ref"].ctypes.data)
    return dict(score=out["score"][:m], mean=out["mean"][:m], ref=out["ref"][:n])


def ref_available():
    return os.path.exists(REF_SO)


def reference(c, cam, ext, vio_cfg, timed=False):
    """The reference source's own updateReferencePatch with an empty plane map: score_, mean_, the chosen position (-1: none)
    and has_ref_patch_; with timed=True also the seconds of the call."""
    L = C.CDLL(REF_SO)
    L.ref_vio_create.restype = vp
    L.ref_vio_create.argtypes = [vp] * 6
    L.ref_vio_destroy.argtypes = [vp]
    L.ref_score_ref_patches.restype = C.c_double
    L.ref_score_ref_patches.argtypes = [vp, C.c_int] + [vp] * 11
    keep = [_a(cam.as_array(), np.float64), _a(ext.extR, np.float64), _a(ext.extT, np.float64), _a(ext.Rcl, np.float64), _a(ext.Pcl, np.float64),
            _a(vio_cfg.as_array(), np.float64)]
    h = L.ref_vio_create(*[k.ctypes.data for k in keep])
    assert h
    n, m = len(c["first"]) - 1, len(c["patch"])
    out = dict(score=np.zeros(max(m, 1), np.float32), mean=np.zeros(max(m, 1), np.float32), ref=np.zeros(max(n, 1), np.int32), has_ref=np.zeros(max(n, 1), np.uint8))
    ins = [_a(c["first"], np.int32), _a(c["pos"], np.float64), _a(c["normal"], np.float64), _a(c["patch"], np.float32), _a(c["mean"], np.float32),
           _a(c["id"], np.int32), _a(c["T"], np.float64)]
    try:
        sec = L.ref_score_ref_patches(h, n, *[x.ctypes.data for x in ins], *[out[f].ctypes.data for f in ("score", "mean", "ref", "has_ref")])
    finally:
        L.ref_vio_destroy(h)
    r = dict(score=out["score"][:m], mean=out["mean"][:m], ref=out["ref"][:n], has_ref=out["has_ref"][:n])
    return (r, sec) if timed else r


# ----------------------------------------------------------------------------------------------- numpy spelling
def numpy_score(c, sqrt_in_double=False, mean_recompute=False, reset_per_pair=False):
    """The scoring spelled in numpy float32 / float64 operations, vectorised over a point's reference observations.
    sqrt_in_double: sqrt resolved to the double overload (the quotient, fabs and the NCC sum then run in double and narrow at
    +=); mean_recompute: ignore a cached mean_ (always the patch's own mean); reset_per_pair: the three sums restarted for every
    other observation (the reference does not restart them)."""
    f32, f64 = np.float32, np.float64
    n = len(c["first"]) - 1
    score, mean, ref = np.zeros(len(c["patch"]), f32), np.zeros(len(c["patch"]), f32), np.full(n, -1, np.int32)
    with np.errstate(all="ignore"):
        for i in range(n):
            b, e = int(c["first"][i]), int(c["first"][i + 1])
            k = e - b
            if k == 0:
                continue
            P = c["patch"][b:e].astype(f32)
            mu_in = c["mean"][b:e].astype(f32)
            own = (P.astype(f64).sum(1).astype(f32) / f32(64)).astype(f32)
            recompute = (np.abs(mu_in).astype(f64) < 1e-6) | mean_recompute
            mu = np.where(recompute, own, mu_in).astype(f32)
            mean[b:e] = mu
            Cc = (P - mu[:, None]).astype(f32)
            ids = c["id"][b:e]
            up = np.zeros(k, f32)
            d1 = np.zeros(k, f32)
            d2 = np.zeros(k, f32)
            ncc = np.zeros(k, f32)
            cnt = np.zeros(k, np.int64)
            for j in range(k):
                act = ids != ids[j]
                if reset_per_pair:
                    up, d1, d2 = np.where(act, f32(0), up), np.where(act, f32(0), d1), np.where(act, f32(0), d2)
                for t in range(64):
                    a, bb = Cc[:, t], Cc[j, t]
                    up = np.where(act, (up + (a * bb).astype(f32)).astype(f32), up)
                    d1 = np.where(act, (d1 + (a * a).astype(f32)).astype(f32), d1)
                    d2 = np.where(act, (d2 + f32(bb * bb)).astype(f32), d2)
                if sqrt_in_double:
                    term = np.abs(up.astype(f64) / np.sqrt((d1 * d2).astype(f32).astype(f64)))
                    ncc = np.where(act, (ncc.astype(f64) + term).astype(f32), ncc)
                else:
                    term = np.abs((up / np.sqrt((d1 * d2).astype(f32))).astype(f32))
                    ncc = np.where(act, (ncc + term).astype(f32), ncc)
                cnt += act
            nccf = (ncc / cnt.astype(f32)).astype(f32)
            T = c["T"][b:e]
            R = T[:, :9].reshape(-1, 3, 3)
            pw, nw = c["pos"][i], c["normal"][i]
            cos = np.zeros(k)
            for r in range(k):  # left-to-right sums as the stand-in Eigen
                pf = [R[r, q, 0] * pw[0] + R[r, q, 1] * pw[1] + R[r, q, 2] * pw[2] + T[r, 9 + q] for q in range(3)]
                nv = [R[r, q, 0] * nw[0] + R[r, q, 1] * nw[1] + R[r, q, 2] * nw[2] for q in range(3)]
                ln = np.sqrt(pf[0] * pf[0] + pf[1] * pf[1] + pf[2] * pf[2])
                cos[r] = (pf[0] / ln) * nv[0] + (pf[1] / ln) * nv[1] + (pf[2] / ln) * nv[2]
            s = (nccf.astype(f64) + cos).astype(f32)
            score[b:e] = s
            best = f32(-1000)
            for r in range(k):
                if s[r] > best:
                    best, ref[i] = s[r], r
    return dict(score=score, mean=mean, ref=ref)


def same_bits(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def same_bits_but_nan(a, b):
    """Bit for bit, except that a NaN equals any NaN: the host's 0 / 0 gives the x86 default NaN (sign set, and fabs clears it
    again), the device's gives CUDA's canonical NaN, and the scoring does not define a payload."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind != "f":
        return same_bits(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()
