"""Hand-built voxel maps and scans for the LIO plane association (voxel_map.cpp:643-786).

The maps of synthetic.build_voxel_map hold at most a handful of candidate planes per root voxel, no exact probability
ties and hardly any deep octree, so the code that arbitrates between candidates (on the device the warp-cooperative
cold path of csrc/esikf_lio.cu: the (owner lane, candidate) pairs of a warp dealt in chunks of 32, the lowest-index tie
break across lanes and chunks, the neighbour voxel) is barely reached by them. These helpers build flat maps
(synthetic.PLANE_DTYPE, `keys / first / count / planes`) and scans where it is:

  * root voxels with 1, 2-9, 33, 34, 64 (layer-2 leaves) and 130 (layer-3 leaves) candidates, and roots without a plane;
  * byte-identical planes in different leaves (exact probability ties), at candidate 0 and further down the DFS list;
  * candidates that fail the range gate, the sigma gate, and the range gate by one float ulp of `radius`;
  * neighbour voxels with 1, 2, 5, 9, 34, 64 or 130 candidates, with an exact tie, without a plane, or absent, reached
    through the unit-mixing rule (:680-691) diagonally and along faces from home voxels where nothing passes (all planes a
    metre off, or none); points in voxels without a root next to occupied ones;
  * with sigma_num = 40, candidates that pass the gate 38.7-39.9 sigma off the plane, where this_prob underflows to 0.

The scan is laid out by warp: points 32w .. 32w+31 are one warp of the device (one shard, CTA slices start on 32-point
boundaries). Every point is checked in plain numpy to stay clear of the rounding the device and the oracle may
legitimately differ in (sigma_l and the probabilities are tolerance-level, DESIGN §4): the top two probabilities of a
point differ by more than 1e-9 relative unless they come from identical planes, and no candidate sits within 1e-9 of the
sigma gate. World points are placed exactly: identity extrinsics and an identity prior pose make p_w the scan point."""
import numpy as np

from fast_livo2_b200 import synthetic as S

f32 = np.float32
VOXEL = 0.5
MARGIN = 1e-9
ZERO_PROB_K = (38.7, 39.9)  # sigma distances where exp(-k^2 / 2) underflows to 0 but k < sigma_num = 40 passes the gate


# ---------------------------------------------------------------------------------------------------------------------
# map validity
def dfs_digits(layer, path):
    return tuple((int(path) >> (3 * l)) & 7 for l in range(int(layer)))


def validate_map(vm, max_layer):
    """The rules under which a flat map means the same octree to the device (which walks each root's records in order)
    and to the oracle / reference driver (which rebuild the octree from layer / path and walk it depth first): records in
    DFS order, unique (layer, path), no plane above another plane, layer <= max_layer, and unique root keys."""
    keys = [tuple(k) for k in np.asarray(vm["keys"]).tolist()]
    assert len(set(keys)) == len(keys), "duplicate root keys"
    planes = vm["planes"]
    for r, (f, c) in enumerate(zip(vm["first"], vm["count"])):
        assert c >= 0 and (c == 0 or 0 <= f and f + c <= len(planes)), f"root {keys[r]}: bad range"
        prev = None
        for j in range(f, f + c):
            L, p = int(planes["layer"][j]), int(planes["path"][j])
            assert 0 <= L <= max_layer, f"root {keys[r]} record {j}: layer {L} > max_layer {max_layer}"
            assert 0 <= p < 8 ** L or (L == 0 and p == 0), f"root {keys[r]} record {j}: path {p} has bits above layer {L}"
            d = dfs_digits(L, p)
            if prev is not None:
                assert prev < d, f"root {keys[r]} record {j}: not in DFS order or duplicate (layer, path)"
                assert d[:len(prev)] != prev, f"root {keys[r]} record {j}: a plane below another plane"
            prev = d
    first_ok = np.concatenate([[0], np.cumsum(vm["count"])[:-1]])
    assert np.array_equal(vm["first"], first_ok) and int(np.sum(vm["count"])) == len(planes), "records not packed root by root"


def tree_paths(k, max_layer, rng, root_plane_ok=True):
    """k distinct (layer, path) in DFS order with no plane above another: a random octree with layers up to max_layer."""

    def rec(k, depth, digits):
        if k == 0:
            return []
        if k == 1 and (depth == max_layer or (depth > 0 and rng.random() < 0.5) or (depth == 0 and root_plane_ok and rng.random() < 0.5)):
            return [digits]
        cap = 8 ** (max_layer - depth - 1)
        assert k <= 8 * cap
        cnt = np.zeros(8, int)
        for _ in range(k):
            free = np.nonzero(cnt < cap)[0]
            cnt[rng.choice(free)] += 1
        return [x for i in range(8) for x in rec(int(cnt[i]), depth + 1, digits + (i,))]

    out = rec(k, 0, ())
    return [(len(d), sum(x << (3 * l) for l, x in enumerate(d))) for d in out]


# ---------------------------------------------------------------------------------------------------------------------
# numpy restatement of the gates (float-exact where the reference narrows to float) and of the association rule
def point_var(p, cfg, P):
    """pv.var of a world point at the identity pose with identity extrinsics (voxel_map.cpp:376-390)."""
    pz = np.array(p, np.float64)
    if pz[2] == 0:
        pz[2] = 0.001
    rng_f = float(f32(np.sqrt(pz @ pz)))
    dv = np.sin(float(f32(cfg.beam_err)) * 0.017453293) ** 2
    d = pz / np.linalg.norm(pz)
    b1 = np.array([1.0, 1.0, -(d[0] + d[1]) / d[2]])
    b1 /= np.linalg.norm(b1)
    b2 = np.cross(b1, d)
    b2 /= np.linalg.norm(b2)
    A = rng_f * S.skew(d) @ np.stack([b1, b2], 1)
    bc = np.outer(d, d) * float(f32(cfg.dept_err) * f32(cfg.dept_err)) + dv * (A @ A.T)
    cm = S.skew(pz)
    return bc + cm @ P[0:3, 0:3] @ cm.T + P[3:6, 3:6]


IU = np.triu_indices(6)


def plane_var6(pl):
    pv = np.empty((6, 6))
    pv[IU] = pl["plane_var"]
    pv[IU[1], IU[0]] = pl["plane_var"]
    return pv


def range_dis(pl, pw):
    """dis_to_plane, signed distance and range_dis of build_single_residual (:723-727), in the reference's precision."""
    n, c = [float(x) for x in pl["normal"]], [float(x) for x in pl["center"]]
    sd = n[0] * pw[0] + n[1] * pw[1] + n[2] * pw[2] + float(pl["d"])
    dtp = f32(abs(sd))
    e = [c[k] - pw[k] for k in range(3)]
    dtc = f32(e[0] * e[0] + e[1] * e[1] + e[2] * e[2])
    with np.errstate(invalid="ignore"):
        rd = np.sqrt(f32(dtc - f32(dtp * dtp)))
    return dtp, f32(sd), rd


def evaluate(pl, pw, var, sigma_num):
    """One candidate: range gate, sigma_l, sigma gate (as the ratio dtp / (sigma_num sqrt(sigma_l))) and this_prob."""
    dtp, sd, rd = range_dis(pl, pw)
    in_range = bool(float(rd) <= 3.0 * float(pl["radius"]))
    if not in_range:
        return dict(in_range=False, passed=False, prob=None, dis=sd, ratio=None)
    J = np.concatenate([np.asarray(pw) - pl["center"], -pl["normal"]])
    sig = J @ plane_var6(pl) @ J + pl["normal"] @ var @ pl["normal"]
    ratio = float(dtp) / (sigma_num * np.sqrt(sig))
    passed = bool(float(dtp) < sigma_num * np.sqrt(sig))
    prob = 1.0 / np.sqrt(sig) * np.exp(-0.5 * float(dtp) * float(dtp) / sig) if passed else None
    return dict(in_range=True, passed=passed, prob=prob, dis=sd, ratio=ratio, k=float(dtp) / np.sqrt(sig))


def voxel_loc(pw, vs=VOXEL):
    """The float voxel coordinate and key of a world point (:665-671): double quotient narrowed to float, -1 if negative,
    truncation."""
    loc = np.zeros(3, f32)
    for j in range(3):
        loc[j] = f32(pw[j] / vs)
        if loc[j] < 0:
            loc[j] = f32(float(loc[j]) - 1.0)
    return loc, tuple(int(np.trunc(float(x))) for x in loc)


def neighbour_key(pw, vs=VOXEL):
    """The one neighbour voxel the reference probes (:680-691): voxel units compared with metres, reproduced literally."""
    loc, key = voxel_loc(pw, vs)
    vsf, ql = float(f32(vs)), float(f32(f32(vs) / f32(4)))
    nk = list(key)
    for a in range(3):
        center = (0.5 + key[a]) * vsf
        if float(loc[a]) > center + ql:
            nk[a] += 1
        elif float(loc[a]) < center - ql:
            nk[a] -= 1
    return tuple(nk)


def content_key(pl):
    return b"".join(np.ascontiguousarray(pl[f]).tobytes() for f in ("center", "normal", "plane_var", "d", "radius"))


def associate(vm, roots, pw, var, sigma_num, vs=VOXEL):
    """The reference's association of one point with world position pw and covariance var (any pose): home root depth
    first, strict '>' on this_prob starting from 0 (the first of equal probabilities wins, a probability of 0 is never
    chosen), the neighbour probed only when no candidate of the home root passed. `roots`: key -> (first, count). Returns a
    dict with the chosen plane (-1: none), its signed distance, and what led to it."""
    _, key = voxel_loc(pw, vs)
    out = dict(key=key, home=key in roots, plane=-1, dis=f32(0), passed=False, via=None, nb_key=None, nb=False, cands=[], evals=[])
    if not out["home"]:
        return out
    for where, k in (("home", key), ("nb", None)):
        if where == "nb":
            if out["passed"]:
                break
            k = out["nb_key"] = neighbour_key(pw, vs)
            if k not in roots:
                break
            out["nb"] = True
        f, c = roots[k]
        prob, cands = 0.0, []
        for j in range(f, f + c):
            e = evaluate(vm["planes"][j], pw, var, sigma_num)
            out["evals"].append((j, e))
            if e["passed"]:
                out["passed"] = True
                cands.append((j, e["prob"]))
                if e["prob"] > prob:
                    prob, out["plane"], out["dis"], out["via"] = e["prob"], j, e["dis"], where
        out["cands"] = cands
        out["count"] = c
    return out


def margin_ok(vm, a):
    """Clear of the rounding the device and the oracle may differ in: no candidate within MARGIN of the sigma gate, and the
    winning probability more than MARGIN (relative) above the best probability of a plane with different content."""
    for _, e in a["evals"]:
        if e["in_range"] and abs(e["ratio"] - 1.0) <= MARGIN:
            return False
    if a["plane"] < 0:
        return True
    win = content_key(vm["planes"][a["plane"]])
    best = max(p for _, p in a["cands"])
    others = [p for j, p in a["cands"] if content_key(vm["planes"][j]) != win]
    return not others or max(others) < best * (1.0 - MARGIN)


# ---------------------------------------------------------------------------------------------------------------------
# construction
def _unit(rng):
    while True:
        v = rng.normal(size=3)
        v /= np.linalg.norm(v)
        if np.abs(v).min() > 0.15:  # never axis-aligned: every coordinate enters the distances
            return v


def _inplane(n):
    a = np.cross(n, [1.0, 0.0, 0.0])
    a /= np.linalg.norm(a)
    return a, np.cross(n, a)


def _pv(rng, scale=1e-5):
    A = rng.normal(size=(6, 6))
    pv = A @ A.T / 6.0 * scale
    pv[:3, :3] *= 0.1  # centre block: sigma_l depends weakly on where the point is
    return pv[np.triu_indices(6)]


def centre_of(key):
    return (0.5 + np.asarray(key, np.float64)) * VOXEL


class Builder:
    """Roots: key -> plane records in DFS order, with the stack parameters they were made from."""

    def __init__(self, cfg, seed):
        self.cfg = cfg
        self.rng = np.random.default_rng(seed)
        self.roots = {}
        self.meta = {}  # key -> dict(n, anchor, t)

    def root(self, key, t, radius=None, max_layer=None, dups=(), anchor=None, n=None, root_plane_ok=True, inplane_r=0.04):
        """A root whose candidate j is the plane through anchor + t[j] n (plus a small in-plane shift of its centre), all
        with normal n. radius[j] < 0.05 pushes candidate j's centre 0.3 m off in the plane: it fails the range gate.
        dups: (src, dst) pairs, record dst becomes a byte-identical copy of src's plane content."""
        key = tuple(int(x) for x in key)
        assert key not in self.roots
        rng = self.rng
        k = len(t)
        n = _unit(rng) if n is None else n
        anchor = centre_of(key) if anchor is None else np.asarray(anchor, np.float64)
        radius = [0.5] * k if radius is None else list(radius)
        ml = self.cfg.max_layer if max_layer is None else max_layer
        paths = tree_paths(k, ml, rng, root_plane_ok)
        a, b = _inplane(n)
        recs = np.zeros(k, S.PLANE_DTYPE)
        for j in range(k):
            off = 0.3 if radius[j] < 0.05 else rng.uniform(0.5, 1.0) * inplane_r  # never 0: range_dis would cancel to NaN
            ang = rng.uniform(0, 2 * np.pi)
            c = anchor + t[j] * n + off * (np.cos(ang) * a + np.sin(ang) * b)
            recs[j]["center"] = c
            recs[j]["normal"] = n
            recs[j]["plane_var"] = _pv(rng)
            recs[j]["d"] = f32(-(n @ c))
            recs[j]["radius"] = f32(radius[j])
            recs[j]["layer"], recs[j]["path"] = paths[j]
        t = list(t)
        for s, d in dups:
            for f in ("center", "normal", "plane_var", "d", "radius"):
                recs[d][f] = recs[s][f]
            t[d] = t[s]
        self.roots[key] = recs
        self.meta[key] = dict(n=n, anchor=anchor, t=t)
        return key

    def flat(self):
        keys = sorted(self.roots)
        count = np.array([len(self.roots[k]) for k in keys], np.int32)
        first = np.concatenate([[0], np.cumsum(count)[:-1]]).astype(np.int32)
        planes = np.concatenate([self.roots[k] for k in keys]) if keys else np.zeros(0, S.PLANE_DTYPE)
        return dict(keys=np.array(keys, np.int64).reshape(-1, 3), first=first, count=count, planes=planes)


def place(key, n, anchor, h, rng, tries=400, pred=None, box=((0.06, 0.94),) * 3):
    """A float point inside voxel `key` at height h above the plane (anchor, n), i.e. n.(p - anchor) = h, for which
    pred(p) holds, tried from starting points in `box` (per axis, fractions of the voxel). None when none is found."""
    lo = np.asarray(key, np.float64) * VOXEL
    blo, bhi = np.array(box).T
    for _ in range(tries):
        q = lo + rng.uniform(blo, bhi) * VOXEL
        q = q - (n @ (q - anchor) - h) * n
        p = q.astype(f32)
        if voxel_loc(p.astype(np.float64))[1] != tuple(key):
            continue
        if pred is None or pred(p):
            return p
    return None


class Scene:
    """A map, its roots index and the per-point numpy association for a config / covariance."""

    def __init__(self, vm, cfg, P):
        self.vm, self.cfg, self.P = vm, cfg, P
        self.roots = {tuple(k): (int(f), int(c)) for k, f, c in zip(vm["keys"].tolist(), vm["first"], vm["count"])}

    def assoc(self, p):
        pw = np.asarray(p, np.float64)
        return associate(self.vm, self.roots, pw, point_var(pw, self.cfg, self.P), self.cfg.sigma_num)

    def sigma(self, p, key=None, j=None):
        """sqrt(sigma_l) of point p against record j (the first record of its root by default)."""
        pw = np.asarray(p, np.float64)
        if j is None:
            j = self.roots[key][0]
        pl = self.vm["planes"][j]
        J = np.concatenate([pw - pl["center"], -pl["normal"]])
        return float(np.sqrt(J @ plane_var6(pl) @ J + pl["normal"] @ point_var(pw, self.cfg, self.P) @ pl["normal"]))


# ---------------------------------------------------------------------------------------------------------------------
# the designed cases
def base_state(rng, scale=0.5):
    return S.pack_state(np.eye(3), np.zeros(3), 1.0, v=np.zeros(3), g=np.array([0, 0, -9.81]), cov=S.random_prior_cov(rng, scale))


def identity_ext():
    a = S.avia_extrinsics()
    return S.Extrinsics(np.eye(3), np.zeros(3), a.Rcl, a.Pcl)


def _cluster(rng, k, idx, span=0.09, far=0.45):
    """Offsets of a stack of k parallel planes: the planes `idx` within +-span of the anchor (several can pass for one
    point), every other one at least `far` away (never passes)."""
    t = [(far + 0.03 * j) * (1 if j % 2 else -1) for j in range(k)]
    idx = sorted(set(idx))
    vals = np.linspace(-span, span, len(idx)) if len(idx) > 1 else [0.0]
    vals = rng.permutation(vals)
    for i, v in zip(idx, vals):
        t[i] = float(v)
    return t


def build_main(seed=0, cfg=None):
    """The sigma_num = 3 case: every root kind, neighbours, ties, range-gate boundaries; points grouped into designed warps.
    Returns a frame dict (map, pts, state_prior, lio_cfg, ext) plus `tags` (what each point was placed for)."""
    cfg = cfg or S.LioCfg(voxel_size=VOXEL, max_layer=3, max_iterations=5)
    B = Builder(cfg, seed)
    rng = B.rng
    state = base_state(rng)
    P = S.unpack_state(state)["cov"]

    # ---- home roots on a grid of positive keys (their unit-mixing neighbour is the diagonal +1 voxel), zero-coordinate keys
    # (neighbours along faces / edges) and negative keys (diagonal -1)
    homes = [(3 * i + 1, 3 * j + 1, 3 * k + 1) for i in range(4) for j in range(3) for k in range(3)]
    homes += [(3 * i + 1, 0, 0) for i in range(3)] + [(0, 3 * j + 1, 0) for j in range(1, 3)] + [(3 * i + 1, 3, 0) for i in range(2)]
    homes += [(-3 * i - 2, -3 * j - 2, -3 * k - 2) for i in range(2) for j in range(2) for k in range(2)]
    homes = [homes[i] for i in rng.permutation(len(homes))]

    kinds = []
    for k in (2, 3, 4, 5, 6, 7, 8, 9):
        kinds.append(("multi", k, dict(idx=list(range(k)))))
    kinds += [("single", 1, {}), ("single", 1, {}), ("single", 1, {}), ("single", 1, {})]
    kinds += [("zero", 0, {}), ("zero", 0, {})]
    kinds += [("wide", 33, dict(idx=[0, 1, 16, 31, 32])), ("wide", 34, dict(idx=[0, 2, 17, 32, 33])), ("wide", 64, dict(idx=[0, 5, 31, 32, 33, 40, 63])),
              ("wide", 64, dict(idx=[50])), ("wide", 34, dict(idx=[33])), ("deep", 130, dict(idx=[0, 3, 31, 32, 64, 65, 100, 129])),
              ("deep", 131, dict(idx=[1, 33, 64, 96, 130]))]
    # exact duplicates: at candidate 0 and later; two extras whose pairs share a chunk; two extras in different chunks
    kinds += [("dup", 9, dict(idx=[0, 2, 4], dups=[(0, 5)])), ("dup", 8, dict(idx=[1, 3, 6], dups=[(3, 7)])), ("dup", 40, dict(idx=[0, 10, 20], dups=[(10, 35)])),
              ("dup", 64, dict(idx=[0, 12, 30], dups=[(0, 45), (12, 13)])), ("dup", 2, dict(idx=[0], dups=[(0, 1)])), ("dup", 130, dict(idx=[3, 70], dups=[(70, 101), (3, 4)]))]
    # range-gate failures among the candidates (radius 0.01, centre 0.3 m off in the plane)
    kinds += [("rangefail", 6, dict(idx=[0, 1, 2, 3, 4, 5], fail=[0, 2])), ("rangefail", 34, dict(idx=[0, 1, 20, 32, 33], fail=[0, 32])), ("rangefail", 1, dict(idx=[0], fail=[0]))]
    assert len(kinds) <= len(homes)
    nb_kinds = [("single", 1, {}), ("multi", 5, dict(idx=[0, 1, 2, 3, 4])), ("wide", 34, dict(idx=[0, 15, 33])), ("wide", 64, dict(idx=[31, 32, 63])),
                ("deep", 130, dict(idx=[0, 64, 129])), ("dup", 9, dict(idx=[0, 3], dups=[(0, 6)])), ("zero", 0, {}), ("absent", 0, {})]

    def make_root(key, kind, k, opt, anchor=None, n=None):
        if kind == "absent":
            return None
        if kind == "zero":
            return B.root(key, [])
        idx = opt.get("idx", [0])
        t = _cluster(rng, k, idx)
        radius = [0.5] * k
        for j in opt.get("fail", []):
            radius[j] = 0.01
        ml = 3 if k > 64 else 2 if (kind == "wide" or k > 8) else int(rng.integers(1, 3))
        return B.root(key, t, radius=radius, max_layer=ml, dups=opt.get("dups", ()), anchor=anchor, n=n)

    home_kind = {}
    for key, (kind, k, opt) in zip(homes, kinds):
        make_root(key, kind, k, opt)
        home_kind[key] = kind

    # ---- neighbour fallback cells: a home root that nothing in its voxel can match (every plane a metre or more off, or no
    # plane at all) next to a neighbour root of each kind whose planes run through the home voxel. Positive keys reach the
    # diagonal +1 neighbour, keys with zero coordinates a face / edge neighbour, negative keys the diagonal -1 neighbour.
    nb_specs = [("single", 1, {}), ("single", 1, {}), ("multi", 2, dict(idx=[0, 1])), ("multi", 5, dict(idx=[0, 1, 2, 3, 4])),
                ("multi", 9, dict(idx=[2, 5, 8])), ("wide", 34, dict(idx=[0, 15, 33])), ("wide", 64, dict(idx=[31, 32, 63])),
                ("deep", 130, dict(idx=[0, 64, 129])), ("dup", 9, dict(idx=[0], dups=[(0, 6)])), ("dup", 40, dict(idx=[3], dups=[(3, 35)])),
                ("zero", 0, {}), ("absent", 0, {})]
    dead_homes = [("dead", 1), ("dead", 4), ("dead", 34), ("zero", 0)]
    cells = [(3 * i + 1, 3 * j + 1, 22) for i in range(3) for j in range(2)] + [(10, 0, 0), (13, 0, 0), (0, 10, 0)]
    cells += [(-3 * i - 2, -3 * j - 2, -12) for i in range(2) for j in range(2)]
    assert len(cells) >= len(nb_specs)
    nb_cells = []
    for ci, (nkind, k, opt) in enumerate(nb_specs):
        key = cells[ci]
        hkind, hk = dead_homes[ci % len(dead_homes)]
        if hkind == "zero":
            B.root(key, [])
        else:
            B.root(key, _cluster(rng, hk, [], far=1.0), max_layer=2)
        lo = np.asarray(key, np.float64) * VOXEL
        frac = rng.uniform(0.3, 0.7, 3)
        box = [(0.06, 0.94)] * 3
        for a in range(3):
            if key[a] == 0:  # loc in [0.125, 0.375]: no shift along that axis; above 0.375: +1
                frac[a] = 0.25 if ci % 2 else 0.9
                box[a] = (0.15, 0.35) if ci % 2 else (0.6, 0.94)
        nk = neighbour_key((lo + frac * VOXEL).astype(f32).astype(np.float64))
        assert nk != key and nk not in B.roots
        # its planes run through the part of the home voxel whose points have that neighbour
        make_root(nk, nkind, k, opt, anchor=lo + np.mean(box, axis=1) * VOXEL)
        nb_cells.append((key, nk, nkind, hkind, box))

    # ---- absent voxels next to occupied roots (the reference probes no neighbour for them)
    absent = []
    for key in list(B.roots)[:12]:
        ak = tuple(x - 1 for x in key) if min(key) >= 1 else tuple(x + 1 for x in key)
        if ak not in B.roots and all(x != 0 and x != -1 for x in ak):
            absent.append((ak, key))

    # ---- range-gate boundary roots: one point each, radius the smallest float that passes / the float below it
    boundary = []
    for bi in range(8):
        key = (20 + 3 * bi, 21, 22)
        k = 1 if bi % 2 == 0 else 5  # hot path (first and only candidate) and an extra candidate
        boundary.append((key, k, bi // 2 % 2 == 0))

    pts, tags = [], []

    def add(p, tag):
        pts.append(np.asarray(p, f32))
        tags.append(tag)

    def near_target(key, j, spread=0.35):  # a height near candidate j of the root's stack
        m = B.meta[key]
        p0 = centre_of(key)
        s = sc.sigma(p0, key=key, j=sc.roots[key][0] + j)
        return m["t"][j] + rng.uniform(-spread, spread) * s

    # points in home roots (re-built once the neighbours and boundary roots exist)
    boundary_roots = []
    for key, k, passes in boundary:
        t = [0.0] + [0.5 + 0.05 * j for j in range(k - 1)]
        # the boundary candidate is the last (k == 5: an extra of the pair layout, cold path) or the only one (hot path)
        B.root(key, t[::-1] if k > 1 else t, max_layer=2, root_plane_ok=False)
        boundary_roots.append((key, k, passes))
    vm = B.flat()
    sc = Scene(vm, cfg, P)

    for key in homes[:len(kinds)]:
        kind = home_kind[key]
        n_pts = 6 if kind in ("wide", "deep", "dup") else 4
        for q in range(n_pts):
            if kind == "zero":
                p = place(key, _unit(rng), centre_of(key), 0.0, rng)
                add(p, "zero")
                continue
            m = B.meta[key]
            idx = [j for j in range(len(m["t"])) if abs(m["t"][j]) < 0.2]
            j = idx[q % len(idx)]
            h = near_target(key, j)
            p = place(key, m["n"], m["anchor"], h, rng, pred=lambda p: margin_ok(vm, sc.assoc(p)))
            if p is not None:
                add(p, kind)
    for key, nk, nkind, hkind, box in nb_cells:
        placed = 0
        for q in range(4):
            if nk in B.meta and len(B.meta[nk]["t"]):
                m = B.meta[nk]
                idx = [j for j in range(len(m["t"])) if abs(m["t"][j]) < 0.2]
                h = m["t"][idx[q % len(idx)]] + rng.uniform(-0.3, 0.3) * 0.03
                n, anc = m["n"], m["anchor"]
            else:
                h, n, anc = 0.0, _unit(rng), centre_of(key)

            def want(p, nk=nk, match=nkind not in ("zero", "absent")):
                a = sc.assoc(p)
                # matched in the neighbour (so no home candidate passed), or nothing passed at home nor in the neighbour
                return a["nb_key"] == nk and (a["via"] == "nb" if match else not a["passed"]) and margin_ok(vm, a)

            p = place(key, n, anc, h, rng, tries=1000, pred=want, box=box)
            if p is not None:
                add(p, f"nb_{nkind}_from_{hkind}")
                placed += 1
        assert placed >= 2, f"neighbour cell {key} -> {nk} ({nkind}): {placed} points placed"
    for ak, occ in absent:
        m = B.meta.get(occ)
        if m is None or not len(m["t"]):
            continue
        p = place(ak, m["n"], m["anchor"], m["t"][0], rng)
        if p is not None:
            add(p, "absent")
    # range-gate boundary: choose the radius from the point
    for key, k, passes in boundary_roots:
        f, c = sc.roots[key]
        j = f + c - 1
        pl = vm["planes"][j]
        p = place(key, pl["normal"], pl["center"], 0.3 * 0.03, rng)
        rd = range_dis(pl, p.astype(np.float64))[2]
        r = f32(float(rd) / 3.0)
        while not float(rd) <= 3.0 * float(r):
            r = np.nextafter(r, f32(np.inf))
        while float(rd) <= 3.0 * float(np.nextafter(r, f32(0))):
            r = np.nextafter(r, f32(0))
        B.roots[key][c - 1]["radius"] = r if passes else np.nextafter(r, f32(0))
        add(p, "range_pass" if passes else "range_fail")
    vm = B.flat()
    sc = Scene(vm, cfg, P)
    pts = np.array(pts, f32)
    tags = np.array(tags)
    return _finish(dict(map=vm, lio_cfg=cfg, ext=identity_ext(), state_prior=state), pts, tags, rng)


def build_zero_prob(seed=1):
    """sigma_num = 40: candidates that pass the gate 38.7-39.9 sigma off the plane, where this_prob = exp(-k^2/2)/sqrt(sigma_l)
    underflows to 0. The reference then sets is_sucess (so the neighbour is not probed) but chooses no plane, and the
    point is unmatched. Single-plane and multi-plane roots, each with a neighbour voxel that would match; and home roots
    that fail outright next to neighbours whose only passing candidate has this_prob == 0."""
    # one iteration: the 38.7-39.9 sigma margins hold at the prior only. Once the pose has moved, a point can sit where
    # exp(-k^2 / 2) just underflows, a rounding-level decision, and a match 39 sigma off swings the next update.
    cfg = S.LioCfg(voxel_size=VOXEL, max_layer=2, max_iterations=1, sigma_num=40.0)
    B = Builder(cfg, seed)
    rng = B.rng
    state = base_state(rng)
    P = S.unpack_state(state)["cov"]
    # (prob-0 offsets in sigma units, normal offsets) per root: the first entry is candidate 0
    layouts = [("z",), ("z",), ("z", "far"), ("far", "z"), ("z", "z"), ("far", "z", "z"), ("z", "ok"), ("ok", "z"), ("far", "far", "z", "far")]
    pts, tags = [], []
    keys = [(3 * i + 1, 3 * j + 1, 1) for i in range(4) for j in range(4)]
    specs = []
    for key, lay in zip(keys, layouts * 2):
        p = (centre_of(key) + rng.uniform(-0.08, 0.08, 3)).astype(f32)
        n = _unit(rng)
        specs.append((key, lay, p, n))
    def stack(key, lay, pw, n, var, root_plane_ok):
        """A root whose planes lie the wanted number of sigmas from pw: "z" passes with this_prob == 0, "far" fails the gate,
        "ok" passes with a positive probability."""
        t, pv = [], _pv(rng)
        pvm = np.zeros((6, 6))
        pvm[np.triu_indices(6)] = pv
        pvm = pvm + pvm.T - np.diag(np.diag(pvm))
        for what in lay:
            k = {"z": rng.uniform(*ZERO_PROB_K), "far": 45.0 + rng.uniform(0, 5), "ok": rng.uniform(1.0, 6.0)}[what]
            sgn = rng.choice([-1.0, 1.0])
            tt = sgn * k * np.sqrt(n @ var @ n)
            for _ in range(4):  # sigma_l includes J plane_var J^T with J = p - c: iterate the offset to the wanted k
                J = np.concatenate([tt * n, -n])
                tt = sgn * k * np.sqrt(J @ pvm @ J + n @ var @ n)
            t.append(-tt)  # the plane through pw - tt n: n.(pw - c) = tt, dis_to_plane = |tt|
        B.root(key, t, anchor=pw, n=n, inplane_r=0.05, max_layer=2, root_plane_ok=root_plane_ok)
        for j in range(len(t)):
            B.roots[key][j]["plane_var"] = pv

    for key, lay, p, n in specs:
        pw = p.astype(np.float64)
        stack(key, lay, pw, n, point_var(pw, cfg, P), len(lay) == 1)
        # the neighbour voxel holds a plane right through the point: it would match if it were probed
        B.root(neighbour_key(pw), [0.0], anchor=pw, n=_unit(rng))
        pts.append(p)
        tags.append("zero_prob_" + "_".join(lay))
    # home candidates that all fail the gate, and a neighbour whose only passing candidate has this_prob == 0 (alone, and
    # as an extra between failing ones): the neighbour is probed, and the point stays unmatched
    for i, nlay in enumerate([("z",), ("far", "z", "far"), ("z",), ("far", "far", "z")]):
        key = (3 * i + 1, 13, 1)
        p = (centre_of(key) + rng.uniform(-0.08, 0.08, 3)).astype(f32)
        pw = p.astype(np.float64)
        var = point_var(pw, cfg, P)
        stack(key, ("far", "far") if i % 2 else ("far",), pw, _unit(rng), var, True)
        stack(neighbour_key(pw), nlay, pw, _unit(rng), var, len(nlay) == 1)
        pts.append(p)
        tags.append("zero_prob_nb_" + "_".join(nlay))
    # ordinary points within a few millimetres of further planes, so that the update has matches to work with
    for i in range(16):
        key = (3 * i + 1, 25, 1 + 3 * (i % 3))
        n = _unit(rng)
        B.root(key, [0.0], n=n)
        for q in range(6):
            p = place(key, n, centre_of(key), rng.uniform(-0.005, 0.005), rng)
            pts.append(p)
            tags.append("plain")
    vm = B.flat()
    return _finish(dict(map=vm, lio_cfg=cfg, ext=identity_ext(), state_prior=state), np.array(pts, f32), np.array(tags), rng)


def _finish(fr, pts, tags, rng):
    """Validate the map, check the margins of every point and lay the points out in warps of 32: the designed mixtures
    (pending lanes next to non-pending ones, lanes that fall back to the neighbour next to lanes that resolve at home,
    warps whose pair total exceeds 32, 64 and 256)."""
    validate_map(fr["map"], fr["lio_cfg"].max_layer)
    sc = Scene(fr["map"], fr["lio_cfg"], S.unpack_state(fr["state_prior"])["cov"])
    bad = [i for i, p in enumerate(pts) if not margin_ok(fr["map"], sc.assoc(p))]
    assert not bad, f"{len(bad)} points too close to a rounding-level decision: {tags[bad][:5]}"
    count = {k: c for k, (_, c) in sc.roots.items()}
    pend = np.array([count.get(voxel_loc(p.astype(np.float64))[1], 0) > 1 for p in pts])
    wide = np.array([count.get(voxel_loc(p.astype(np.float64))[1], 0) >= 33 for p in pts])
    order = []
    # warps of wide-root points only (pair totals far above 256), then random mixtures of everything
    w_idx = rng.permutation(np.nonzero(wide)[0])
    order += list(w_idx[: (len(w_idx) // 32) * 32][:64])
    rest = [i for i in rng.permutation(len(pts)) if i not in set(order)]
    order += rest
    pad = (-len(order)) % 32
    order += list(rng.choice(len(pts), pad)) if pad else []
    order = np.array(order)
    return dict(fr, pts=np.ascontiguousarray(pts[order]), tags=tags[order])


# ---------------------------------------------------------------------------------------------------------------------
# coverage, in numpy from the map, the scan and the oracle's outputs
def pair_layout(counts_pending):
    """Per lane of one warp: (exclusive prefix, number of pairs) of the (owner lane, extra candidate) pairs."""
    npairs = np.array([max(c - 1, 0) for c in counts_pending])
    excl = np.concatenate([[0], np.cumsum(npairs)[:-1]])
    return excl, npairs


def coverage(fr, first_iter_plane, final_plane):
    """How often each case the device's cold path must get right occurs at the prior pose (first iteration). Returns a dict
    of counts: points whose home root has > 33 candidates, warps whose pair total is > 32 / 64 / 256, lanes whose pair range
    straddles a chunk of 32, points with >= 2 passing candidates, exact-tie points (and where the tie lies: candidate 0
    against an extra, two extras in one chunk, two extras in different chunks), neighbour matches by the neighbour root's
    kind (one candidate, 2-9, more than 33, an exact tie), zero-probability passes at home and in the neighbour, the
    one-ulp radius points on the right side of the range gate (range_boundary_wrong: on the wrong side), and points whose
    final match differs from their first-iteration match."""
    vm, cfg = fr["map"], fr["lio_cfg"]
    sc = Scene(vm, cfg, S.unpack_state(fr["state_prior"])["cov"])
    pts = fr["pts"].astype(np.float64)
    n = len(pts)
    A = [sc.assoc(p) for p in pts]
    assert np.array_equal(np.array([a["plane"] for a in A]), first_iter_plane), "numpy association differs from the oracle's first iteration"
    c = dict.fromkeys(("home_over_33", "warp_pairs_over_32", "warp_pairs_over_64", "warp_pairs_over_256", "straddling_lanes", "multi_pass", "ties",
                       "tie_with_first", "tie_same_chunk", "tie_cross_chunk", "nb_single", "nb_multi", "nb_wide", "nb_dup", "zero_prob_pass",
                       "zero_prob_nb", "range_boundary_pass", "range_boundary_fail", "changed_match"), 0)
    for w in range(0, n, 32):
        lanes = range(w, min(w + 32, n))
        cnt = [sc.roots[A[i]["key"]][1] if A[i]["home"] and sc.roots[A[i]["key"]][1] > 1 else 0 for i in lanes]
        excl, npairs = pair_layout(cnt)
        tot = int(npairs.sum())
        c["warp_pairs_over_32"] += tot > 32
        c["warp_pairs_over_64"] += tot > 64
        c["warp_pairs_over_256"] += tot > 256
        for li, i in enumerate(lanes):
            if npairs[li] and excl[li] // 32 != (excl[li] + npairs[li] - 1) // 32:
                c["straddling_lanes"] += 1
            a = A[i]
            if not a["home"]:
                continue
            f, cc = sc.roots[a["key"]]
            c["home_over_33"] += cc > 33
            c["multi_pass"] += len(a["cands"]) >= 2
            c["zero_prob_pass"] += any(p == 0.0 for _, p in a["cands"])
            if a["via"] == "nb":  # matched in the neighbour voxel, by the neighbour root's candidate count
                nc = sc.roots[a["nb_key"]][1]
                kind = "nb_single" if nc == 1 else "nb_multi" if nc <= 9 else "nb_wide" if nc > 33 else "nb_other"
                c[kind] = c.get(kind, 0) + 1
            if a["nb"] and a["plane"] < 0:
                f2 = sc.roots[a["nb_key"]][0]
                c["zero_prob_nb"] += any(j >= f2 and e["passed"] and e["prob"] == 0.0 for j, e in a["evals"])
            tag = str(fr["tags"][i])
            if tag in ("range_pass", "range_fail"):  # the one-ulp radius boundary decides the point's only close candidate
                on = a["plane"] == f + cc - 1
                kind = "range_boundary_pass" if (tag, on) == ("range_pass", True) else "range_boundary_fail" if (tag, on) == ("range_fail", False) else "range_boundary_wrong"
                c[kind] = c.get(kind, 0) + 1
            if a["plane"] >= 0:
                win = content_key(vm["planes"][a["plane"]])
                best = max(p for _, p in a["cands"])
                tied = [j for j, p in a["cands"] if p == best and content_key(vm["planes"][j]) == win]
                if len(tied) >= 2:
                    c["ties"] += 1
                    c["nb_dup"] += a["via"] == "nb"
                    base = sc.roots[a["key"] if a["via"] == "home" else a["nb_key"]][0]
                    ranks = [j - base for j in tied]
                    if ranks[0] == 0:
                        c["tie_with_first"] += 1
                    if a["via"] == "home":
                        chunks = {(excl[li] + r - 1) // 32 for r in ranks if r > 0}
                        if len([r for r in ranks if r > 0]) >= 2:
                            c["tie_same_chunk" if len(chunks) == 1 else "tie_cross_chunk"] += 1
    c["changed_match"] = int((np.asarray(first_iter_plane) != np.asarray(final_plane)).sum())
    return c


# ---------------------------------------------------------------------------------------------------------------------
# the cases, built once per session
CASES = ("main", "displaced", "zero_prob")
REF_CASES = ("main", "displaced")  # zero_prob: the reference pushes an uninitialised PointToPlane there (DESIGN §4)
_cases = {}


def displaced(fr, rot=(0.004, -0.003, 0.005), shift=(0.03, -0.02, 0.025)):
    """The main case with a prior pose a few centimetres / a few tenths of a degree off the pose the scan was placed at:
    points start in other voxels or off their planes and change voxel and match between iterations."""
    st = S.unpack_state(fr["state_prior"])
    state = S.pack_state(S.so3_exp(np.array(rot)), np.array(shift), 1.0, v=st["v"], g=st["g"], cov=st["cov"])
    return dict(fr, state_prior=state)


def case(name):
    """The named case; the generated ones are cached in the frame cache directory (keyed by this file's source)."""
    if name not in _cases:
        if name == "displaced":
            _cases[name] = displaced(case("main"))
        else:
            import hashlib
            import os
            import pickle

            with open(os.path.abspath(__file__), "rb") as f:
                src = hashlib.sha1(f.read() + open(S.__file__, "rb").read()).hexdigest()[:16]
            path = os.path.join(S.frame_cache_dir(), f"lio_assoc_{name}_{src}.pkl")
            try:
                with open(path, "rb") as f:
                    _cases[name] = pickle.load(f)
            except Exception:
                _cases[name] = {"main": build_main, "zero_prob": build_zero_prob}[name]()
                try:
                    os.makedirs(os.path.dirname(path), exist_ok=True)
                    with open(path + f".{os.getpid()}.tmp", "wb") as f:
                        pickle.dump(_cases[name], f, protocol=4)
                    os.replace(path + f".{os.getpid()}.tmp", path)
                except Exception:
                    pass
    return _cases[name]


SMEM_LANES, LANES = 704, 768  # lanes per CTA of the LIO kernels in shared-memory slots / in all (csrc/esikf_lio.cu)


def l2_lane_layout(fr, G, start):
    """A scan of G * 768 points (every CTA exactly 24 chunks of 32) built from the case's designed warps: CTA b runs the
    case's warps start + 2b and start + 2b + 1 in its L2-slot warps and the 22 warps after them in its shared-slot warps."""
    pts, tags = fr["pts"], np.asarray(fr["tags"])
    W = len(pts) // 32
    order = []
    for b in range(G):
        ws = [(start + 2 * b + 2 + j) % W for j in range(SMEM_LANES // 32)] + [(start + 2 * b) % W, (start + 2 * b + 1) % W]
        order += [np.arange(32 * w, 32 * w + 32) for w in ws]
    order = np.concatenate(order)
    return dict(fr, pts=np.ascontiguousarray(pts[order]), tags=tags[order])


def tiled(fr, n):
    """The case's scan repeated warp by warp to n points (the designed warps keep their lanes)."""
    pts = fr["pts"]
    reps = -(-n // len(pts))
    return dict(fr, pts=np.ascontiguousarray(np.tile(pts, (reps, 1))[:n]))
