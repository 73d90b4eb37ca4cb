"""The visual map's observation store (esikf_vmap_*) on the host: OracleStore keeps the same per-point slots as the device
and applies each call with the oracle's restatements (orc_update_points for the flags and the new observations,
oracle/orc_vmap.cpp for the list edits and the reference choice, orc_score_ref_patches for the scoring). A seeded sequence of
VIO ticks (generate -> sub-map -> update points -> score -> choose) and hand-built states drive both."""
import ctypes as C
import os

import numpy as np

import observe_cases as OC
import refpatch_cases as RC
import warp_cases as W
from fast_livo2_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORC_VMAP_SO = os.path.join(ROOT, "oracle", "liborc_vmap.so")
REF_VMAP_SO = os.path.join(ROOT, "oracle", "_ref", "libfl2_ref_vmap.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pin", "vmap.npz")
SLOTS = 30
FLT_MAX = np.finfo(np.float32).max
vp = C.c_void_p
LIST_FIELDS = ("first", "px", "patch", "T_f_w", "id", "mean", "score", "ref")


def _a(x, dt=np.float64):
    return np.ascontiguousarray(x, dtype=dt)


class OracleStore:
    """A host copy of the observation store: count, ref (P,) and per slot T (P, 30, 12), px (P, 30, 2), patch (P, 30, 64),
    mean, score (P, 30) float32, id (P, 30) int32."""

    def __init__(self, cam, ext, capacity=4096):
        self.L = C.CDLL(ORC_VMAP_SO)
        self.L.orc_vmap_edit.argtypes = [C.c_int] + [vp] * 6 + [C.c_int32] + [vp] * 10
        self.L.orc_vmap_choose_ref.argtypes = [C.c_int, vp, vp, vp, C.c_int] + [vp] * 6
        self.cam, self.ext = cam, ext
        self.obs = None
        P = capacity
        self.count, self.ref = np.zeros(P, np.int32), np.full(P, -1, np.int32)
        self.T, self.px, self.patch = np.zeros((P, SLOTS, 12)), np.zeros((P, SLOTS, 2)), np.zeros((P, SLOTS, 64), np.float32)
        self.mean, self.score, self.id = np.zeros((P, SLOTS), np.float32), np.zeros((P, SLOTS), np.float32), np.zeros((P, SLOTS), np.int32)
        self.points = 0

    def add(self, first, px, patch, T_f_w, id, mean, score, ref):  # noqa: A002 (the download's field names)
        n = len(first) - 1
        ids = np.arange(self.points, self.points + n, dtype=np.int32)
        for i, p in enumerate(ids):
            b, e = first[i], first[i + 1]
            c = e - b
            self.count[p], self.ref[p] = c, ref[i]
            self.T[p, :c], self.px[p, :c], self.patch[p, :c] = T_f_w[b:e], px[b:e], patch[b:e]
            self.mean[p, :c], self.score[p, :c], self.id[p, :c] = mean[b:e], score[b:e], id[b:e]
        self.points += n
        return ids

    def download(self, pid):
        pid = np.asarray(pid, np.int32)
        c = self.count[pid]
        first = np.concatenate([[0], np.cumsum(c)]).astype(np.int32)
        out = dict(first=first, ref=self.ref[pid].copy())
        for f, a in (("px", self.px), ("patch", self.patch), ("T_f_w", self.T), ("id", self.id), ("mean", self.mean), ("score", self.score)):
            out[f] = np.concatenate([a[p, :k] for p, k in zip(pid, c)]) if len(pid) else a[:0, 0]
        return out

    def update(self, pid, converged, sc, frame_id, T_new):
        """updateVisualMapPoints for the entries pid of the sub-map whose positions, image and state `sc` holds."""
        pid, converged = _a(pid, np.int32), _a(converged, np.uint8)
        n = len(pid)
        c = self.count[pid]
        last_T = np.where((c > 0)[:, None], self.T[pid, np.maximum(c - 1, 0)], np.nan)
        last_px = np.where((c > 0)[:, None], self.px[pid, np.maximum(c - 1, 0)], np.nan)
        if self.obs is None:
            self.obs = OC.OracleObserve(dict(cam=self.cam, ext=self.ext))
        o = self.obs.run(dict(img=sc["img"], state=sc["state"], pos=sc["pos"], converged=converged, last_T=last_T, last_px=last_px))
        new_pc, new_patch = np.zeros((max(n, 1), 2)), np.zeros((max(n, 1), 64), np.float32)
        new_pc[o["entry"]], new_patch[o["entry"]] = o["pc"], o["patch"]
        evicted, count = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
        flag = _a(o["update_flag"], np.uint8)
        self.L.orc_vmap_edit(n, pid.ctypes.data, converged.ctypes.data, flag.ctypes.data, new_pc.ctypes.data, new_patch.ctypes.data,
                             _a(T_new).ctypes.data, int(frame_id), *[a.ctypes.data for a in (self.count, self.ref, self.T, self.px, self.patch,
                                                                                          self.mean, self.score, self.id)],
                             evicted.ctypes.data, count.ctypes.data)
        return dict(o, evicted=evicted[:n], count=count[:n])

    def score_points(self, pid, pos, normal):
        pid = np.asarray(pid, np.int32)
        d = self.download(pid)
        r = RC.oracle(dict(first=d["first"], pos=pos, normal=normal, patch=d["patch"], mean=d["mean"], id=d["id"], T=d["T_f_w"]))
        rows_s, rows_m = np.zeros((len(pid), SLOTS), np.float32), np.zeros((len(pid), SLOTS), np.float32)
        for i, p in enumerate(pid):
            b, e = d["first"][i], d["first"][i + 1]
            self.score[p, :e - b], self.mean[p, :e - b] = r["score"][b:e], r["mean"][b:e]
            rows_s[i, :e - b], rows_m[i, :e - b] = r["score"][b:e], r["mean"][b:e]
            if r["ref"][i] >= 0:
                self.ref[p] = r["ref"][i]
        return dict(ref=r["ref"], score=rows_s, mean=rows_m)

    def choose(self, pid, normal_en, pos=None, frame_pos=None):
        pid = _a(pid, np.int32)
        n = len(pid)
        pos = np.zeros((max(n, 1), 3)) if pos is None else _a(pos).reshape(-1, 3)
        fp = np.zeros(3) if frame_pos is None else _a(frame_pos)
        out = np.zeros(max(n, 1), np.int32)
        self.L.orc_vmap_choose_ref(n, pid.ctypes.data, pos.ctypes.data, fp.ctypes.data, int(bool(normal_en)), self.count.ctypes.data,
                                   self.ref.ctypes.data, self.T.ctypes.data, self.patch.ctypes.data, self.id.ctypes.data, out.ctypes.data)
        return out[:n]


class RefStore:
    """The reference's own VisualPoint / Feature objects kept across calls (oracle/ref_vmap.cpp): updateVisualMapPoints,
    updateReferencePatch (empty plane map) and getCloseViewObs run as they are."""

    def __init__(self, cam, ext):
        L = self.lib = C.CDLL(REF_VMAP_SO)
        L.ref_vio_create.restype = vp
        L.ref_vio_create.argtypes = [vp] * 6
        L.ref_vio_destroy.argtypes = [vp]
        L.ref_vmap_add.argtypes = [vp, C.c_int] + [vp] * 9
        L.ref_vmap_update.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp]
        L.ref_vmap_set_scores.argtypes = [vp, C.c_int] + [vp] * 5
        L.ref_vmap_close_view.argtypes = [vp, C.c_int, vp, vp, vp]
        L.ref_vmap_download.restype = C.c_int
        L.ref_vmap_download.argtypes = [vp] * 10
        self._keep = OC._cam_ext(dict(cam=cam, ext=ext))
        self.h = L.ref_vio_create(*[k.ctypes.data for k in self._keep])
        assert self.h

    def add(self, pos, first, px, patch, T_f_w, id, mean, score, ref):  # noqa: A002
        ins = [_a(pos), _a(first, np.int32), _a(px), _a(patch, np.float32), _a(T_f_w), _a(id, np.int32), _a(mean, np.float32), _a(score, np.float32),
               _a(ref, np.int32)]
        self.lib.ref_vmap_add(self.h, len(first) - 1, *[x.ctypes.data for x in ins])

    def update(self, pid, converged, sc, frame_id):
        pid, conv = _a(pid, np.int32), _a(converged, np.uint8)
        flag, T = np.zeros(max(len(pid), 1), np.uint8), np.zeros(12)
        img, state = _a(sc["img"], np.uint8), _a(sc["state"])
        self.lib.ref_vmap_update(self.h, img.ctypes.data, state.ctypes.data, int(frame_id), len(pid), pid.ctypes.data, conv.ctypes.data, flag.ctypes.data,
                                 T.ctypes.data)
        return flag[:len(pid)], T

    def score(self, pid, pos, normal):
        """updateReferencePatch's write-back of the restatement's scores (orc_score_ref_patches, pinned by
        tests/test_oracle_refpatch.py where the reference is defined) into the reference's objects"""
        pid = _a(pid, np.int32)
        d = self.download()
        c = np.diff(d["first"])[pid]
        first = np.concatenate([[0], np.cumsum(c)]).astype(np.int32)
        sl = [slice(d["first"][p], d["first"][p + 1]) for p in pid]
        cat = lambda k, dt: _a(np.concatenate([d[k][x] for x in sl]) if len(pid) else d[k][:0], dt)  # noqa: E731
        r = RC.oracle(dict(first=first, pos=pos, normal=normal, patch=cat("patch", np.float32), mean=cat("mean", np.float32), id=cat("id", np.int32),
                           T=cat("T_f_w", np.float64)))
        sc, mu, ref = _a(r["score"], np.float32), _a(r["mean"], np.float32), _a(r["ref"], np.int32)
        self.lib.ref_vmap_set_scores(self.h, len(pid), pid.ctypes.data, first.ctypes.data, sc.ctypes.data, mu.ctypes.data, ref.ctypes.data)

    def close_view(self, pid, frame_pos):
        pid, fp = _a(pid, np.int32), _a(frame_pos)
        out = np.zeros(max(len(pid), 1), np.int32)
        self.lib.ref_vmap_close_view(self.h, len(pid), pid.ctypes.data, fp.ctypes.data, out.ctypes.data)
        return out[:len(pid)]

    def download(self):
        n = self.lib.ref_vmap_download(self.h, *([None] * 9))
        m = 30 * n
        out = dict(first=np.zeros(n + 1, np.int32), px=np.zeros((max(m, 1), 2)), patch=np.zeros((max(m, 1), 64), np.float32), T_f_w=np.zeros((max(m, 1), 12)),
                   id=np.zeros(max(m, 1), np.int32), mean=np.zeros(max(m, 1), np.float32), score=np.zeros(max(m, 1), np.float32), ref=np.zeros(max(n, 1), np.int32),
                   has_ref=np.zeros(max(n, 1), np.uint8))
        self.lib.ref_vmap_download(self.h, *[out[f].ctypes.data for f in LIST_FIELDS + ("has_ref",)])
        k = int(out["first"][n])
        return dict(first=out["first"], ref=out["ref"][:n], has_ref=out["has_ref"][:n], **{f: out[f][:k] for f in LIST_FIELDS[1:-1]})

    def __del__(self):
        try:
            self.lib.ref_vio_destroy(self.h)
        except Exception:
            pass


def ref_available():
    return os.path.exists(REF_VMAP_SO)


def scored(update_flag, converged, count):
    """The points updateReferencePatch scores: flagged, not converged, more than 5 observations (vio.cpp:977-980)."""
    return (np.asarray(update_flag) == 1) & (np.asarray(converged) == 0) & (np.asarray(count) > 5)


def list_digests(d):
    import hashlib

    return np.array([hashlib.sha256(np.ascontiguousarray(d[f]).tobytes()).hexdigest() for f in LIST_FIELDS])


def reference_sequence():
    """The reference driver over the tick sequence (the scores written back as updateReferencePatch does, from the scoring's
    restatement): per tick the flags, the frame's T_f_w_, getCloseViewObs of the retrieved
    points and the digests of every list afterwards (LIST_FIELDS order), and has_ref_patch_ against ref."""
    cam, ext, ticks = sequence()
    R = RefStore(cam, ext)
    out = dict(flag=[], T=[], close=[], digest=[], has_ref_ok=[])
    for tk in ticks:
        R.add(tk["pos_new"], **tk["add"])
        flag, T = R.update(tk["sub"], tk["converged"], tk, tk["t"])
        d = R.download()
        count = np.diff(d["first"])[tk["sub"]]
        sel = scored(flag, tk["converged"], count)
        R.score(tk["sub"][sel], tk["pos"][sel], tk["normal"][tk["sub"][sel]])
        close = R.close_view(tk["ret"], tk["frame_pos"])
        d = R.download()
        out["flag"].append(flag), out["T"].append(T), out["close"].append(close), out["digest"].append(list_digests(d))
        out["has_ref_ok"].append(bool(np.array_equal(d["has_ref"], (d["ref"] >= 0).astype(np.uint8))))
    return out


def hand_case():
    """The hand-built update of hand_lists and the getCloseViewObs lists of choose_lists, as the tests run them."""
    cam, ext = OC.CAMERAS["pinhole"]
    R, p = S.so3_exp(np.array([0.01, -0.02, 0.03])), np.array([0.3, -0.2, 0.1])
    T_near, pts = hand_lists(np.random.default_rng(3), cam, ext, R, p)
    sc = dict(img=OC.grey_image(cam, 9), state=S.pack_state(R, p, 1.0), pos=np.array([q["pos"] for q in pts]))
    cpos, fp = np.array([1.0, -2.0, 14.0]), np.array([0.2, 0.1, -0.3])
    return cam, ext, T_near, pts, sc, choose_lists(np.random.default_rng(4), cpos, fp), cpos, fp


def reference_hand():
    """The reference driver on hand_case(): the flags, the frame's T_f_w_ and the lists after the update (has_ref_patch_
    included), and getCloseViewObs of the choice lists."""
    cam, ext, T_near, pts, sc, lists, cpos, fp = hand_case()
    R = RefStore(cam, ext)
    R.add(sc["pos"], **lists_of(pts))
    flag, T = R.update(np.arange(len(pts)), [q["conv"] for q in pts], sc, 77)
    d = R.download()
    C2 = RefStore(cam, ext)
    C2.add(np.tile(cpos, (len(lists), 1)), **lists_of(lists))
    close = C2.close_view(np.arange(len(lists)), fp)
    return dict(flag=flag, T=T, close=close, **{f"list_{k}": v for k, v in d.items()})


def same_lists(a, b):
    """Two downloads are equal bit for bit (NaN scores by their bits too: both sides move them without arithmetic)."""
    for f in LIST_FIELDS:
        if np.asarray(a[f]).tobytes() != np.asarray(b[f]).tobytes():
            return f
    return None


# ---------------------------------------------------------------------------------------------------------------- the tick sequence
def frame(t, ticks):
    """The frame of tick t: the IMU on a circle of radius 1.2 m, looking along +z with a small sway."""
    a = 2 * np.pi * t / ticks * 1.7
    R = S.so3_exp(np.array([0.02 * np.sin(a), 0.03 * np.cos(a), 0.0]))
    p = np.array([1.2 * np.cos(a), 1.2 * np.sin(a), 0.0])
    return R, p


def new_points(rng, cam, ext, R, p, k, frame_id, img):
    """k new points of one tick (esikf_vio_generate_points' winners): one observation each, at the frame's pose."""
    Rcw, Pcw = S.camera_pose(ext, R, p)
    u, v = rng.uniform(160, cam.width - 160, k), rng.uniform(140, cam.height - 140, k)
    z = rng.uniform(12.0, 25.0, k)
    ray = W.cam2world(cam, u, v)
    pf = ray * (z / ray[:, 2])[:, None]
    pos = (pf - Pcw) @ Rcw
    patch = np.stack([img[int(y) - 4:int(y) + 4, int(x) - 4:int(x) + 4].astype(np.float32).reshape(64) for x, y in zip(u, v)])
    T = np.tile(OC.pack_T(Rcw, Pcw), (k, 1))
    return pos, dict(first=np.arange(k + 1, dtype=np.int32), px=np.stack([u, v], 1), patch=patch, T_f_w=T, id=np.full(k, frame_id, np.int32),
                     mean=np.zeros(k, np.float32), score=np.zeros(k, np.float32), ref=np.full(k, -1, np.int32))


def sequence(ticks=44, seed=5, per_tick=24):
    """The inputs of every tick, seeded: new points, the sub-map (every point of tick 0, which thus reaches 30 observations,
    and a random subset of the others), convergence from tick 25 on for a third of the points, normals for the scoring (which
    takes the points scored() selects) and the retrieved points of getCloseViewObs."""
    cam, ext = OC.CAMERAS["pinhole"]
    rng = np.random.default_rng(seed)
    pos_all, ticks_out, conv = [], [], np.zeros(0, np.uint8)
    for t in range(ticks):
        R, p = frame(t, ticks)
        Rcw, Pcw = S.camera_pose(ext, R, p)
        img = OC.grey_image(cam, 300 + t)
        pos_new, add = new_points(rng, cam, ext, R, p, 40 if t == 0 else per_tick, t, img)
        base = len(pos_all)
        pos_all.extend(pos_new)
        conv = np.concatenate([conv, np.zeros(len(pos_new), np.uint8)])
        if t >= 25:
            conv[np.arange(len(conv)) % 3 == 1] = 1
        old = np.arange(40, base)
        sub = np.concatenate([np.arange(min(40, base)), rng.choice(old, size=min(len(old), 60), replace=False) if len(old) else old]).astype(np.int32)
        rng.shuffle(sub)
        pos = np.array(pos_all)
        normal = rng.normal(size=(len(pos), 3))
        normal /= np.linalg.norm(normal, axis=1)[:, None]
        normal[:, 2] = -np.abs(normal[:, 2])
        ret = rng.choice(len(pos), size=min(len(pos), 80), replace=False).astype(np.int32)
        ticks_out.append(dict(t=t, add=add, pos_new=pos_new, sub=sub, converged=conv[sub].copy(), img=img, state=S.pack_state(R, p, 1.0), pos=pos[sub],
                              T_new=OC.pack_T(Rcw, Pcw)[0], normal=normal, all_pos=pos, ret=ret, frame_pos=-(Rcw.T @ Pcw)))
    return cam, ext, ticks_out


# ---------------------------------------------------------------------------------------------------------------- hand-built states
def hand_lists(rng, cam, ext, R, p):
    """Hand-built points at the frame (R, p). Observation j of a point is 'near' (the frame's own pose and pixel: adds nothing)
    unless listed in `far` (2 m away: adds the frame). Returns the lists, the points' pos and what each case expects."""
    Rcw, Pcw = S.camera_pose(ext, R, p)
    T_near = OC.pack_T(Rcw, Pcw)[0]
    T_far = OC.pack_T(Rcw, Pcw + np.array([2.0, 0.0, 0.0]))[0]
    pts = []

    def point(name, c, scores, ref=-1, far=(), ids=None, conv=0, uv=(320.0, 256.0)):
        u, v = uv
        ray = W.cam2world(cam, np.array([u]), np.array([v]))[0]
        pos = (ray * (15.0 / ray[2]) - Pcw) @ Rcw
        T = np.tile(T_near, (c, 1))
        for j in far:
            T[j] = T_far
        px = np.tile([u, v], (c, 1)).astype(np.float64)
        pts.append(dict(name=name, c=c, pos=pos, T=T, px=px, patch=rng.normal(100, 20, (c, 64)).astype(np.float32), score=np.asarray(scores, np.float32),
                        ref=ref, id=np.arange(c, dtype=np.int32) if ids is None else np.asarray(ids, np.int32), conv=conv))

    nan, inf = np.float32(np.nan), np.float32(np.inf)
    s = np.linspace(5, 1, 30)
    tie = s.copy()
    tie[[3, 7]] = 0.5  # tied minimum: the first goes
    point("tie", 30, tie, ref=10)
    point("nan", 30, np.full(30, nan), ref=4)  # every score NaN: the newest goes
    point("flt_max", 30, np.full(30, FLT_MAX), ref=0)  # nothing below FLT_MAX: the newest goes, and it was the ref
    mix = np.full(30, inf)
    mix[12] = FLT_MAX
    mix[20] = nan
    point("inf", 30, mix, ref=25)
    ev = s.copy()
    ev[15] = -3.0
    point("evict_ref", 30, ev, ref=15)
    last_min = s.copy()
    last_min[29] = -9.0
    point("oldest_decides", 30, last_min, ref=2, far=(29,))  # the oldest is far and evicted: the flag reads it first
    point("far_29", 29, s[:29], ref=1, far=(28,))  # 29 observations: no eviction, an addition
    point("conv_ref", 8, s[:8], ref=3, conv=1)
    point("conv_noref", 8, s[:8], ref=-1, conv=1)
    point("near", 5, s[:5], ref=-1)
    return T_near, pts


def lists_of(pts):
    first = np.concatenate([[0], np.cumsum([q["c"] for q in pts])]).astype(np.int32)
    cat = lambda k: np.concatenate([q[k] for q in pts])  # noqa: E731
    return dict(first=first, px=cat("px"), patch=cat("patch"), T_f_w=cat("T"), id=cat("id"), mean=np.zeros(first[-1], np.float32), score=cat("score"),
                ref=np.array([q["ref"] for q in pts], np.int32))


def choose_lists(rng, pos, frame_pos):
    """Points for the reference choice: 1 observation; no ref; a ref; every id_ equal (0 / 0); and for getCloseViewObs,
    camera centres whose viewing-ray cosines lie on both sides of 0.5 (59 and 61 degrees)."""
    fp = np.asarray(frame_pos, np.float64)
    d0 = (fp - pos) / np.linalg.norm(fp - pos)
    e = np.cross(d0, [0.0, 0.0, 1.0])
    e /= np.linalg.norm(e)

    def centre(deg):  # a camera centre whose ray to pos makes `deg` degrees with the frame's
        a = np.deg2rad(deg)
        return pos + 5.0 * (np.cos(a) * d0 + np.sin(a) * e)

    def T_at(c):  # T_f_w_ of a camera at centre c with R = I: t = -c
        return np.concatenate([np.eye(3).reshape(9), -c])

    lists = []
    for name, degs, ids, ref in (("one", [10], [0], -1), ("noref", [10, 20, 30, 40], [0, 1, 2, 3], -1), ("ref", [70, 20, 10], [0, 1, 2], 1),
                                 ("same_ids", [30, 20, 10], [4, 4, 4], -1), ("wide", [80, 65, 61], [0, 1, 2], -1),
                                 ("mixed", [75, 59, 45, 89], [0, 1, 1, 2], -1), ("behind", [120, 170], [0, 1], -1)):
        c = len(degs)
        lists.append(dict(name=name, c=c, pos=pos, T=np.stack([T_at(centre(d)) for d in degs]), px=np.zeros((c, 2)),
                          patch=rng.normal(100, 20, (c, 64)).astype(np.float32), score=np.zeros(c, np.float32), ref=ref, id=np.asarray(ids, np.int32), conv=0))
    return lists
