"""Hand-built point streams for the voxel map (UpdateVoxelMap / UpdateOctoTree / init_octo_tree / cut_octo_tree / init_plane,
src/voxel_map.cpp:55-290, 609-641, and mapSliding's clearMemOutOfMap, :924-971): the device state machine
(fast_livo2_b200/csrc/esikf_map.cuh) is held to the oracle on every tick of every stream, node by node and plane by plane.

The synthetic room scene never builds a plane below layer 1, a root with more than 8 candidates, a per-layer layer_init_num or
a list that meets max_points_num at a refit. Each case here is built to reach one of those decisions, and `reach` names what
it must reach: a count over the node dumps / flattened maps / usage of the replay, which the tests assert is non-zero, so a
case cannot silently drift away from its branch.

Coordinates are float32 (world points are float in the product). Voxel sizes 2.0 and 0.5 are dyadic, so node centres and
split planes are exact; where a case needs exact covariances (the box corners) every coordinate is dyadic as well.
"""
import numpy as np

from fast_livo2_b200 import synthetic as S

VAR = np.diag([2.0 ** -14, 2.0 ** -14, 2.0 ** -13])  # the per-point covariance of every stream (SPD, exact)
NORMAL = np.array([0.3, -0.2, 1.0]) / np.linalg.norm([0.3, -0.2, 1.0])  # tilt of the planar patches
_T1 = np.cross(NORMAL, [0.0, 1.0, 0.0])
_T1 /= np.linalg.norm(_T1)
_T2 = np.cross(NORMAL, _T1)

# dump columns (oracle_bind.NODE_COLS)
KX, KY, KZ, LAYER, PATH, INIT, OCTO, ENABLE, PLANE, NEWP, TEMP, PSIZE = range(12)


def f32(p):
    return np.asarray(p, np.float64).astype(np.float32).astype(np.float64)


def node_center(cfg, key, path):
    """Centre and half side of the node reached from root `key` through leaves `path` (the reference's float quarter lengths)."""
    v = np.float32(cfg.voxel_size)
    c = (0.5 + np.asarray(key, np.float64)) * np.float64(v)
    q = np.float32(v / np.float32(4))
    for leaf in path:
        b = np.array([(leaf >> 2) & 1, (leaf >> 1) & 1, leaf & 1])
        c = c + np.float64(np.float32(2 * b - 1) * q)
        q = np.float32(q / np.float32(2))
    return c, 2.0 * float(q)


def blob(cfg, key, path, n, rng, spread=0.7):
    """n points spread uniformly over the inner `spread` of a node (isotropic: never planar at a tiny min_eigen_value)."""
    c, h = node_center(cfg, key, path)
    return f32(c + rng.uniform(-spread, spread, (n, 3)) * h)


def patch(cfg, key, path, n, rng, jitter=0.0):
    """n points on a tilted plane through the centre of a node (anisotropic in the plane: distinct eigenvalues), optionally
    `jitter` (fraction of the half side) off the plane."""
    c, h = node_center(cfg, key, path)
    # the first nine on a 3 x 3 grid, corners first (any three of a patch already span the plane), then random
    g = np.array([(-1, -1), (1, 1), (1, -1), (-1, 1), (0, 0), (-1, 0), (1, 0), (0, -1), (0, 1)], np.float64)
    uw = np.concatenate([g, rng.uniform(-1, 1, (max(n - 9, 0), 2))])[:n] + rng.uniform(-0.1, 0.1, (n, 2))
    u, w = uw[:, 0] * 0.55 * h, uw[:, 1] * 0.27 * h
    off = rng.uniform(-1.0, 1.0, n) * jitter * h
    return f32(c + u[:, None] * _T1 + w[:, None] * _T2 + off[:, None] * NORMAL)


def interleave(groups):
    """Round-robin over the groups (point j of every group, then point j + 1, ...): a node's first points come from all of
    its sub-cells, so that an interior node is not fitted on one patch alone."""
    out, j = [], 0
    while any(j < len(g) for g in groups):
        out += [g[j] for g in groups if j < len(g)]
        j += 1
    return np.array(out).reshape(-1, 3)


def tick(pw):
    pw = np.asarray(pw, np.float64).reshape(-1, 3)
    return pw, np.tile(VAR, (len(pw), 1, 1))


def cell2(i, j, k):
    """Leaf path of the layer-2 cell (i, j, k) of a root, i, j, k in 0..3."""
    return [4 * (i >> 1) + 2 * (j >> 1) + (k >> 1), 4 * (i & 1) + 2 * (j & 1) + (k & 1)]


def cell3(i, j, k):
    """Leaf path of the layer-3 cell (i, j, k) of a root, i, j, k in 0..7."""
    return [4 * ((i >> 2) & 1) + 2 * ((j >> 2) & 1) + ((k >> 2) & 1), 4 * ((i >> 1) & 1) + 2 * ((j >> 1) & 1) + ((k >> 1) & 1), 4 * (i & 1) + 2 * (j & 1) + (k & 1)]


# ---------------------------------------------------------------------------------------------------------------- reach
def _nodes(d, key=None, path=None, layer=None):
    m = np.ones(len(d), bool)
    if key is not None:
        m &= np.all(d[:, :3] == np.asarray(key), axis=1)
    if path is not None:
        p = 0
        for l, leaf in enumerate(path):
            p |= leaf << (3 * l)
        m &= (d[:, PATH] == p) & (d[:, LAYER] == len(path))
    if layer is not None:
        m &= d[:, LAYER] == layer
    return d[m]


def _count(flat, key):
    i = np.nonzero(np.all(flat["keys"] == np.asarray(key), axis=1))[0]
    return int(flat["count"][i[0]]) if len(i) else 0


def _one(d, key, path, **want):
    """1 if the node exists and every named column has the wanted value."""
    n = _nodes(d, key, path)
    cols = dict(init=INIT, octo=OCTO, enable=ENABLE, plane=PLANE, newp=NEWP, temp=TEMP, psize=PSIZE)
    return int(len(n) == 1 and all(n[0][cols[k]] == v for k, v in want.items()))


# ---------------------------------------------------------------------------------------------------------------- cases
def deep_blob(max_layer, seed=0):
    """Isotropic blobs at min_eigen_value 1e-12: no node is ever planar, so every node with enough points is cut, down to
    max_layer. A dense cluster on the leaf path 7, 0, 7, 0, ... makes one chain reach the last layer; the uniform part fills
    the upper layers with up to 8 non-planar children each (the widest DFS / cut stack)."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=max_layer, min_eigen_value=1e-12, max_points_num=100000)
    rng = np.random.default_rng(seed)
    key = (1, -2, 0)
    chain = [7, 0] * 4
    ticks = []
    for t in range(3):
        pw = np.concatenate([blob(cfg, key, [], 700, rng, 0.999), blob(cfg, key, chain[:8], 100, rng, 0.9)])
        ticks.append(tick(pw[rng.permutation(len(pw))]))
    reach = {f"a node of layer {max_layer} fitted": lambda h: int(((h[-1]["dump"][:, LAYER] == max_layer) & (h[-1]["dump"][:, INIT] == 1)).sum()),
             "no plane anywhere": lambda h: int(h[-1]["dump"][:, PLANE].sum() == 0)}
    if max_layer >= 2:
        reach["a node with 8 cut children"] = lambda h: int(max(np.bincount(_parent_ids(h[-1]["dump"]), minlength=1)) == 8)
    return dict(cfg=cfg, ticks=ticks, reach=reach)


def _parent_ids(d):
    """Index of every node's parent in a dump (roots: -1 dropped)."""
    par, stack = [], []
    for i, r in enumerate(d):
        while stack and d[stack[-1]][LAYER] >= r[LAYER]:
            stack.pop()
        if stack:
            par.append(stack[-1])
        stack.append(i)
    return np.array(par, np.int64)


def deep_cut():
    """The same blob with layer_init_num[0] = 1500: the root's first fit sees 1501 points and cut_octo_tree recurses seven
    layers down within one call (map_cut's explicit stack, not the per-point descent)."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=7, min_eigen_value=1e-12, max_points_num=100000, layer_init_num=(1500, 5, 5, 5, 5, 5, 5, 5))
    rng = np.random.default_rng(3)
    key = (0, 0, 0)
    pw = np.concatenate([blob(cfg, key, [], 1200, rng, 0.999), blob(cfg, key, [7, 0] * 4, 301, rng, 0.9)])
    reach = {"the root cut at its first fit, down to layer 7": lambda h: int(_one(h[0]["dump"], key, [], init=1, octo=1) and (h[0]["dump"][:, LAYER] == 7).any()),
             "a cut child cut again in the same call (octo_state 1 below the root)": lambda h: int(((h[0]["dump"][:, OCTO] == 1) & (h[0]["dump"][:, LAYER] > 0)).sum())}
    return dict(cfg=cfg, ticks=[tick(pw[rng.permutation(len(pw))])], reach=reach)


def candidates_growth():
    """One root whose candidate list grows 1 -> 8 -> 9 -> 16 -> 17 -> 64 over six ticks: small tilted patches in distinct
    layer-2 cells, two z levels in every layer-1 parent, so no ancestor is ever planar. The record block of the root moves
    1 -> 8 -> 16 -> 32 -> 64 slots (map_emit_root)."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=2, min_eigen_value=2.0 ** -12, max_points_num=1000)
    rng = np.random.default_rng(7)
    key = (0, 0, 0)
    par = lambda p: [(2 * (p >> 2) + (q >> 2), 2 * ((p >> 1) & 1) + ((q >> 1) & 1), 2 * (p & 1) + (q & 1)) for q in range(8)]  # the 8 cells of parent p
    P = [par(p) for p in range(8)]
    full = lambda c: patch(cfg, key, cell2(*c), 9, rng)
    part = lambda c, n: patch(cfg, key, cell2(*c), n, rng)
    pend = {}

    def half(c):  # 3 points now, 6 later: the cell stays unfitted until its second part arrives
        pts = part(c, 9)
        pend[c] = pts[3:]
        return pts[:3]

    t0 = interleave([full(P[0][0]), half(P[0][1])])
    t1 = interleave([pend.pop(P[0][1])] + [full(c) for c in P[0][2:]])
    t2 = interleave([full(P[1][0]), half(P[1][1])])
    t3 = interleave([pend.pop(P[1][1])] + [full(c) for c in P[1][2:]])
    t4 = interleave([full(P[2][0]), half(P[2][1])])
    t5 = interleave([pend.pop(P[2][1])] + [full(c) for c in P[2][2:]] + [full(c) for p in range(3, 8) for c in P[p]])
    ticks = [tick(t) for t in (t0, t1, t2, t3, t4, t5)]
    reach = {"candidate counts 1, 8, 9, 16, 17, 64": lambda h: int([_count(x["flat"], key) for x in h] == [1, 8, 9, 16, 17, 64]),
             "every candidate at layer 2": lambda h: int((h[-1]["flat"]["planes"]["layer"] == 2).all()),
             # record blocks of 1, 8, 16, 32 and 64 slots: each relocation allocated exactly once
             "record blocks 1 + 8 + 16 + 32 + 64": lambda h: int(h[-1]["usage"]["recs"] == 1 + 8 + 16 + 32 + 64)}
    return dict(cfg=cfg, ticks=ticks, reach=reach, key=key)


def candidates_layer3():
    """72 candidate planes of one root, all at layer 3 (9 layer-2 parents with a patch in each of their 8 cells)."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=3, min_eigen_value=2.0 ** -12, max_points_num=1000)
    rng = np.random.default_rng(11)
    key = (-1, 0, 2)
    parents = [(0, 0, 0), (1, 0, 0), (0, 1, 1), (2, 3, 0), (3, 3, 3), (1, 2, 2), (3, 0, 1), (2, 1, 3), (0, 3, 2)]
    cells = [(2 * a + (q >> 2), 2 * b + ((q >> 1) & 1), 2 * c + (q & 1)) for a, b, c in parents for q in range(8)]
    pw = interleave([patch(cfg, key, cell3(*c), 8, rng) for c in cells])
    reach = {"72 candidates at layer 3": lambda h: int(_count(h[-1]["flat"], key) == 72 and (h[-1]["flat"]["planes"]["layer"] == 3).all())}
    return dict(cfg=cfg, ticks=[tick(pw)], reach=reach, key=key)


def layer_init_update():
    """layer_init_num (5, 7, 11, 13): layer-k nodes that receive exactly layer_init_num[k] points one by one (no fit) and one
    more (fitted) through UpdateOctoTree, for k = 1, 2, 3."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=3, min_eigen_value=1e-12, max_points_num=10000, layer_init_num=(5, 7, 11, 13))
    rng = np.random.default_rng(13)
    key = (0, 1, 0)
    b = lambda path, n: blob(cfg, key, path, n, rng, 0.6)
    t0 = np.concatenate([b([o, 3], 1) for o in range(6)])                   # root fitted at 6, one point in each of 6 leaves
    t1 = np.concatenate([b([0], 6), b([1, 0], 4), b([1, 7, 3], 3)])          # leaf 0 at 7 (= 7: not fitted), leaf 1 at 8 (fitted, cut)
    t2 = np.concatenate([b([1, 0], 7), b([1, 7, 0], 5), b([1, 7, 7], 4)])    # [1,0] at 11 (not fitted), [1,7] at 12 (fitted, cut)
    t3 = np.concatenate([b([1, 7, 0], 8), b([1, 7, 7], 10)])                 # [1,7,0] at 13 (not fitted), [1,7,7] at 14 (fitted)
    ticks = [tick(t) for t in (t0, t1, t2, t3)]
    d = lambda h: h[-1]["dump"]
    reach = {"layer 1 at 7 points unfitted": lambda h: _one(d(h), key, [0], init=0, temp=7),
             "layer 1 at 8 points fitted": lambda h: _one(d(h), key, [1], init=1, psize=8),
             "layer 2 at 11 points unfitted": lambda h: _one(d(h), key, [1, 0], init=0, temp=11),
             "layer 2 at 12 points fitted": lambda h: _one(d(h), key, [1, 7], init=1, psize=12),
             "layer 3 at 13 points unfitted": lambda h: _one(d(h), key, [1, 7, 0], init=0, temp=13),
             "layer 3 at 14 points fitted": lambda h: _one(d(h), key, [1, 7, 7], init=1, psize=14)}
    return dict(cfg=cfg, ticks=ticks, reach=reach)


def layer_init_cut():
    """layer_init_num (64, 7, 11, 13): the root's first fit sees 65 points and cut_octo_tree hands layer-k children exactly
    layer_init_num[k] points (not fitted) and one more (fitted, cut further), for k = 1, 2, 3."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=3, min_eigen_value=1e-12, max_points_num=10000, layer_init_num=(64, 7, 11, 13))
    rng = np.random.default_rng(17)
    key = (2, 0, -1)
    b = lambda path, n: blob(cfg, key, path, n, rng, 0.6)
    pw = np.concatenate([b([0], 7), b([1], 8), b([2, 0], 11), b([3, 0], 12), b([4, 0, 0], 13), b([4, 0, 7], 14)])
    assert len(pw) == 65
    d = lambda h: h[-1]["dump"]
    reach = {"cut: layer 1 at 7 unfitted": lambda h: _one(d(h), key, [0], init=0, temp=7, newp=7),
             "cut: layer 1 at 8 fitted": lambda h: _one(d(h), key, [1], init=1, psize=8),
             "cut: layer 2 at 11 unfitted": lambda h: _one(d(h), key, [2, 0], init=0, temp=11),
             "cut: layer 2 at 12 fitted": lambda h: _one(d(h), key, [3, 0], init=1, psize=12),
             "cut: layer 3 at 13 unfitted": lambda h: _one(d(h), key, [4, 0, 0], init=0, temp=13),
             "cut: layer 3 at 14 fitted": lambda h: _one(d(h), key, [4, 0, 7], init=1, psize=14)}
    return dict(cfg=cfg, ticks=[tick(pw[rng.permutation(65)])], reach=reach)


def max_points_last_layer():
    """max_layer 0, max_points_num 20. Plane roots fed 19, 20 and 21 points over three ticks (a plane stops at size >= 20),
    non-plane roots fed 19, 20, 21 and 22 (a last-layer non-plane node stops at size > 20), and a jittered root that is not a
    plane at its first fit or its first refit and becomes one at its second (then stops at >= 20)."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=0, min_eigen_value=2.0 ** -12, max_points_num=20)
    rng = np.random.default_rng(19)
    roots = {("plane", n): (n, 0, 0) for n in (19, 20, 21)}
    roots.update({("blob", n): (n, 1, 0) for n in (19, 20, 21, 22)})
    pts = {k: (patch(cfg, key, [], k[1], rng) if k[0] == "plane" else blob(cfg, key, [], k[1], rng)) for k, key in roots.items()}
    flip_key = (0, 5, 0)
    c, _ = node_center(cfg, flip_key, [])
    # 6 points +-j off the plane, uncorrelated with their in-plane coordinates and centred: the normal stays an eigenvector,
    # with eigenvalue 6 j^2 / n after n points (the rest on the plane): above 2^-12 at n = 6 and 12, below it at 18
    j = 0.0245
    uwo = np.array([(0.3, 0.1, j), (-0.3, -0.1, j), (0.3, -0.1, -j), (-0.3, 0.1, -j), (0.0, 0.0, j), (0.0, 0.0, -j)])
    jit = f32(c + uwo[:, :1] * _T1 + uwo[:, 1:2] * _T2 + uwo[:, 2:] * NORMAL)
    flip = [jit, patch(cfg, flip_key, [], 6, rng), patch(cfg, flip_key, [], 6, rng), patch(cfg, flip_key, [], 4, rng)]
    ticks = []
    for t, (a, e) in enumerate([(0, 8), (8, 16), (16, 22)]):
        ticks.append(tick(np.concatenate([p[a:e] for p in pts.values()] + [flip[t] if t < 2 else np.concatenate(flip[2:])])))
    d = lambda h: h[-1]["dump"]
    reach = {"plane at 19 enabled": lambda h: _one(d(h), roots[("plane", 19)], [], plane=1, enable=1, temp=19),
             "plane at 20 stopped (>=)": lambda h: _one(d(h), roots[("plane", 20)], [], plane=1, enable=0, temp=0),
             "plane at 21 stopped at 20": lambda h: _one(d(h), roots[("plane", 21)], [], plane=1, enable=0, temp=0, psize=18),
             "non-plane at 20 enabled (>)": lambda h: _one(d(h), roots[("blob", 20)], [], plane=0, enable=1, temp=20),
             "non-plane at 21 stopped": lambda h: _one(d(h), roots[("blob", 21)], [], plane=0, enable=0, temp=0),
             "last-layer non-plane became a plane": lambda h: int(_one(h[1]["dump"], flip_key, [], plane=0) and _one(d(h), flip_key, [], plane=1, enable=0))}
    return dict(cfg=cfg, ticks=ticks, reach=reach)


def max_points_cut():
    """max_points_num 20 inside one init list: layer_init_num[0] = 44, the root's cut hands a planar patch of 20 points to
    leaf 0 (fitted, kept: 20 > 20 is false) and one of 21 to leaf 1 (fitted, stopped); the next tick brings leaf 0 to 21."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=2, min_eigen_value=2.0 ** -12, max_points_num=20, layer_init_num=(44, 5, 5))
    rng = np.random.default_rng(23)
    key = (0, 0, 3)
    pw = np.concatenate([patch(cfg, key, [0], 20, rng), patch(cfg, key, [1], 21, rng), blob(cfg, key, [6], 4, rng)])
    t1 = np.concatenate([patch(cfg, key, [0], 1, rng), patch(cfg, key, [1], 1, rng)])
    reach = {"cut child at 20 kept": lambda h: _one(h[0]["dump"], key, [0], plane=1, enable=1, temp=20),
             "cut child at 21 stopped": lambda h: _one(h[0]["dump"], key, [1], plane=1, enable=0, temp=0, psize=21),
             "kept child stopped at 21 (>=)": lambda h: _one(h[1]["dump"], key, [0], plane=1, enable=0, temp=0)}
    return dict(cfg=cfg, ticks=[tick(pw[rng.permutation(45)]), tick(t1)], reach=reach)


def refit_flip():
    """max_points_num 12: a plane root whose refit at exactly 12 points makes it non-planar. It took the plane branch, so it
    stops (>= 12) although it is no longer a plane; the following points go to fresh leaves of the non-plane root."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=2, min_eigen_value=2.0 ** -12, max_points_num=12)
    rng = np.random.default_rng(29)
    key = (3, 3, 3)
    t0 = patch(cfg, key, [], 6, rng)
    t1 = np.concatenate([blob(cfg, key, [o], 1, rng) for o in (0, 3, 5, 6, 7, 2)])
    t2 = np.concatenate([blob(cfg, key, [1], 8, rng), blob(cfg, key, [4], 3, rng)])
    reach = {"plane refit to non-plane at max_points_num, stopped": lambda h: _one(h[1]["dump"], key, [], plane=0, enable=0, temp=0, psize=12),
             "later points in fresh leaves": lambda h: _one(h[2]["dump"], key, [1], init=1, plane=0, octo=1) * _one(h[2]["dump"], key, [4], init=0, temp=3)}
    return dict(cfg=cfg, ticks=[tick(t0), tick(t1), tick(t2)], reach=reach)


def on_centre():
    """Points with coordinates exactly on the split planes of fitted non-plane nodes of layers 0, 1 and 2 (the test is
    p > centre): they go to the low leaf."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=3, min_eigen_value=1e-12, max_points_num=1000)
    rng = np.random.default_rng(31)
    key = (0, 0, 0)
    t0 = blob(cfg, key, [7, 7, 7], 6, rng, 0.6)  # root, [7] and [7, 7]: fitted, not planar, cut (all into leaf 7)
    on = []
    for path in ([], [7], [7, 7]):
        c, h = node_center(cfg, key, path)
        lo = c - 0.5 * h
        on += [[c[0], lo[1], lo[2]], [lo[0], c[1], lo[2]], [lo[0], lo[1], c[2]], list(c)]
    on = f32(on)
    assert np.all(on == np.asarray(on, np.float32))
    reach = {f"layer {len(p)}: on-centre points in the low leaf": (lambda p: lambda h: _one(h[1]["dump"], key, p + [0], init=0, temp=4))(p) for p in ([], [7], [7, 7])}
    return dict(cfg=cfg, ticks=[tick(t0), tick(on)], reach=reach)


BOX_A, BOX_B = 2.0 ** -2, 2.0 ** -3
BOX_H = {"below": 2.0 ** -6 - 2.0 ** -16, "at": 2.0 ** -6, "above": 2.0 ** -6 + 2.0 ** -16, "equal_min": 2.0 ** -7}
BOX_KEYS = {"below": (0, 0, 0), "at": (1, 0, 0), "above": (2, 0, 0), "equal_min": (3, 0, 0)}


def box_corners():
    """8 corners (c +- a, c +- b, c +- h) of dyadic boxes around root centres: the covariance is exactly diag(a^2, b^2, h^2).
    layer_init_num[0] = 7, so the first fit sees exactly the 8 corners. min_eigen_value 2^-12: h^2 one step below, exactly at
    (not a plane: the test is strict) and above it; and b = h, two equal smallest eigenvalues, where 1 / (l_min - l_mid)
    divides by zero: the reference keeps a plane whose plane_var holds inf / NaN."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=0, min_eigen_value=2.0 ** -12, max_points_num=1000, layer_init_num=(7,))
    pw = []
    for name, key in BOX_KEYS.items():
        c, _ = node_center(cfg, key, [])
        h = BOX_H[name]
        b = h if name == "equal_min" else BOX_B
        pw += [c + np.array([sx * BOX_A, sy * b, sz * h]) for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]
    pw = np.array(pw)
    assert np.array_equal(pw, f32(pw))
    d = lambda h: h[-1]["dump"]
    reach = {"h^2 below min_eigen_value: plane": lambda h: _one(d(h), BOX_KEYS["below"], [], plane=1, psize=8),
             "h^2 at min_eigen_value: no plane": lambda h: _one(d(h), BOX_KEYS["at"], [], plane=0, init=1, psize=8),
             "h^2 above: no plane": lambda h: _one(d(h), BOX_KEYS["above"], [], plane=0, init=1, psize=8),
             "equal smallest eigenvalues: plane with NaN in plane_var": lambda h: int(np.isnan(h[-1]["flat"]["planes"]["plane_var"]).any(axis=1).sum() == 1)}
    return dict(cfg=cfg, ticks=[tick(pw)], reach=reach)


def big_list(n=4500):
    """One plane root that receives n points in one tick (max_points_num above n): its list grows 8 -> 16 -> ... -> 8192 inside
    one replay, and each refit sums the whole list (on the GPU: n / 32 rounds of 32 lanes)."""
    cfg = S.LioCfg(voxel_size=2.0, max_layer=0, min_eigen_value=2.0 ** -12, max_points_num=100000)
    rng = np.random.default_rng(37)
    key = (-3, 2, 1)
    reach = {f"a list of {n} points, refitted": lambda h: _one(h[0]["dump"], key, [], plane=1, enable=1, temp=n) * int(h[0]["dump"][0, PSIZE] > 4096)}
    return dict(cfg=cfg, ticks=[tick(patch(cfg, key, [], n, rng))], reach=reach)


KEY_LIMIT = 1 << 20


def key_edges():
    """Roots at keys -2^20 and 2^20 - 1 (the ends of [-2^20, 2^20)) on every axis, voxel 0.5: their points are float32-exact
    (centre +- multiples of 1/32)."""
    cfg = S.LioCfg(voxel_size=0.5, max_layer=1, max_points_num=100)
    rng = np.random.default_rng(41)
    keys = []
    for ax in range(3):
        for k in (-KEY_LIMIT, KEY_LIMIT - 1):
            key = [0, 0, 0]
            key[ax] = k
            keys.append(tuple(key))
    pw = []
    offs = np.array([[a, b, c] for a in (-3, 3) for b in (-5, 1, 4) for c in (-2, 3)]) / 32.0
    for key in keys:
        c, _ = node_center(cfg, key, [])
        pw.append(c + offs[rng.permutation(len(offs))])
    pw = np.concatenate(pw)
    assert np.array_equal(pw, f32(pw))
    reach = {"roots at both ends of the key range on every axis": lambda h: int(all(len(_nodes(h[-1]["dump"], k, [])) == 1 for k in keys))}
    return dict(cfg=cfg, ticks=[tick(pw)], reach=reach)


def beyond_key(ax, side):
    """One point whose key is one past the end of the key range on one axis (MAP_ERR_KEY)."""
    key = [0, 0, 0]
    key[ax] = KEY_LIMIT if side > 0 else -KEY_LIMIT - 1
    c, _ = node_center(S.LioCfg(voxel_size=0.5), key, [])
    return tick(f32([c]))


def hash_keys(n_roots, seed=43):
    """n_roots distinct root keys (voxel 0.5), 7 points each, all in one tick."""
    cfg = S.LioCfg(voxel_size=0.5, max_layer=1)
    rng = np.random.default_rng(seed)
    side = int(np.ceil(n_roots ** (1 / 3)))
    keys = np.array([(i, j, k) for i in range(side) for j in range(side) for k in range(side)])[:n_roots] - side // 2
    pw = np.concatenate([patch(cfg, tuple(k), [], 7, rng) for k in keys])
    return cfg, keys, pw[rng.permutation(len(pw))]


def hash_slot(key, mask):
    """hash_key(pack_key(key)) & mask, as esikf_dev.cuh computes it."""
    x, y, z = (int(v) + KEY_LIMIT for v in key)
    k = (x << 42) | (y << 21) | z
    M = (1 << 64) - 1
    k ^= k >> 33
    k = (k * 0xFF51AFD7ED558CCD) & M
    k ^= k >> 33
    k = (k * 0xC4CEB9FE1A85EC53) & M
    k ^= k >> 33
    return (k & 0xFFFFFFFF) & mask


def voxel_keys(pw, cfg):
    """Root key of every point, the float quotient of UpdateVoxelMap (src/voxel_map.cpp:620-625)."""
    loc = (np.asarray(pw, np.float64) / np.float64(np.float32(cfg.voxel_size))).astype(np.float32)
    loc = np.where(loc < 0, (loc.astype(np.float64) - 1.0).astype(np.float32), loc)
    return np.trunc(loc).astype(np.int64)


def key_order(pw, cfg):
    """The distinct root keys of a tick in the order of their first point (the order the host harness inserts them)."""
    k = voxel_keys(pw, cfg)
    _, first = np.unique(k, axis=0, return_index=True)
    return k[np.sort(first)]


def probe_wraps(keys, cap):
    """Linear probing of `keys` inserted in order into a table of cap slots: how many probe sequences run past the last slot."""
    used, wraps = np.zeros(cap, bool), 0
    for key in keys:
        s = hash_slot(key, cap - 1)
        start = s
        while used[s]:
            s = (s + 1) & (cap - 1)
        wraps += s < start
        used[s] = True
    return wraps


SLIDE_BOXES = [((-2, -1, 0), (1, 2, 2)), ((-1, -1, 1), (1, 1, 2))]


def slide():
    """Roots on the key grid [-3, 3]^3 (voxel 0.5, a tilted patch in each), then mapSliding to a box whose faces pass through
    occupied roots on every axis (keys equal to lo / hi stay, keys one past go), updates, a second slide into a smaller box
    (which reuses the first arena's storage on the device), updates, and a box that keeps nothing, then updates."""
    cfg = S.LioCfg(voxel_size=0.5, max_layer=2, max_points_num=40)
    rng = np.random.default_rng(47)
    keys = [(i, j, k) for i in range(-3, 4) for j in range(-3, 4) for k in range(-3, 4)]
    pts = lambda n: interleave([patch(cfg, key, [], n, rng) for key in keys])
    ticks = [tick(pts(8)), tick(pts(4)), tick(pts(7)), tick(pts(6)), tick(pts(6))]
    slides = {1: SLIDE_BOXES[0], 2: SLIDE_BOXES[1], 3: ((10, 10, 10), (11, 11, 11))}  # after tick i
    kb = np.array(keys)

    def on_faces(h):
        lo, hi = map(np.array, SLIDE_BOXES[0])
        kept = set(map(tuple, h[1]["slid"]["keys"].tolist()))
        n = 0
        for ax in range(3):
            n += all(tuple(k) in kept for k in kb[(kb[:, ax] == lo[ax]) & np.all((kb >= lo) & (kb <= hi), axis=1)])
            n += all(tuple(k) in kept for k in kb[(kb[:, ax] == hi[ax]) & np.all((kb >= lo) & (kb <= hi), axis=1)])
            n += not any(tuple(k) in kept for k in kb[(kb[:, ax] == lo[ax] - 1) | (kb[:, ax] == hi[ax] + 1)])
        return int(n == 9)

    reach = {"faces through occupied roots: on-face kept, one past dropped": on_faces,
             "second slide keeps a non-empty subset": lambda h: int(0 < len(h[2]["slid"]["keys"]) < len(h[1]["slid"]["keys"])),
             "empty box then updates rebuild the map": lambda h: int(len(h[3]["slid"]["keys"]) == 0 and len(h[4]["flat"]["keys"]) == len(keys))}
    return dict(cfg=cfg, ticks=ticks, slides=slides, reach=reach)


CASES = {
    **{f"deep_blob_L{L}": (lambda L: lambda: deep_blob(L))(L) for L in (0, 1, 2, 3, 7)},
    "deep_cut": deep_cut,
    "candidates_growth": candidates_growth,
    "candidates_layer3": candidates_layer3,
    "layer_init_update": layer_init_update,
    "layer_init_cut": layer_init_cut,
    "max_points_last_layer": max_points_last_layer,
    "max_points_cut": max_points_cut,
    "refit_flip": refit_flip,
    "on_centre": on_centre,
    "box_corners": box_corners,
    "big_list": big_list,
    "key_edges": key_edges,
    "slide": slide,
}


def case(name):
    return CASES[name]()


def key_box(lo, hi):
    """clearMemOutOfMap's arguments (x_max, x_min, y_max, y_min, z_max, z_min) of the box [lo, hi]."""
    return [int(hi[0]), int(lo[0]), int(hi[1]), int(lo[1]), int(hi[2]), int(lo[2])]


class OracleSide:
    """The oracle's UpdateVoxelMap / clearMemOutOfMap in the interface replay() drives."""

    def __init__(self, cfg, ext=None):
        import oracle_bind as O

        self.o = O.OracleLIO(cfg, ext or S.avia_extrinsics())

    def apply(self, pw, var):
        import oracle_bind as O

        pw, var = np.ascontiguousarray(pw, np.float64), np.ascontiguousarray(np.asarray(var).reshape(-1, 9), np.float64)
        self.o.lib.orc_lio_update_map(self.o.h, O.dptr(pw), O.dptr(var), len(pw))

    def slide(self, lo, hi):
        return self.o.lib.orc_lio_clear_out_of_map(self.o.h, *key_box(lo, hi))

    def flatten(self):
        return self.o.flatten()

    def dump_nodes(self):
        return self.o.dump_nodes()

    def usage(self):
        return None


class RefSide:
    """The reference source's UpdateVoxelMap / clearMemOutOfMap (oracle/_ref) in the interface replay() drives."""

    def __init__(self, cfg):
        import oracle_bind as O

        self.r = O.RefMap(cfg)

    def apply(self, pw, var):
        self.r.update(pw, var)

    def slide(self, lo, hi):
        self.r.clear_out_of_map(lo, hi)

    def flatten(self):
        return self.r.flatten()

    def dump_nodes(self):
        return self.r.dump_nodes()

    def usage(self):
        return None


class DeviceSide:
    """esikf_map_device_update_points / _slide / _download of a GPU context in the interface replay() drives (no node dump:
    the device keeps its nodes in HBM; their state shows through the planes, the counters and the harness's dump)."""

    def __init__(self, ctx, cfg, **caps):
        self.ctx = ctx
        ctx.map_device_init(cfg, root_capacity=caps.pop("root_capacity", 1 << 12), **caps)

    def apply(self, pw, var):
        self.ctx.map_device_update_points(pw, var)

    def slide(self, lo, hi):
        self.ctx.map_device_slide(lo, hi)

    def flatten(self):
        return self.ctx.map_device_download()

    def dump_nodes(self):
        return None

    def usage(self):
        st = self.ctx.map_device_stats()
        return dict(nodes=st["nodes"], recs=st["records"], pool_points=st["pool_points"], roots=st["roots"], errors=st["errors"])


IDENTITY_EXT = S.Extrinsics(extR=np.eye(3), extT=np.zeros(3), Rcl=np.eye(3), Pcl=np.zeros(3))


def lio_scan(c, rng, n=None):
    """A scan of the stream's own points (identity extrinsics and pose: body = world), 1 mm off their place, and a prior
    displaced by a few mm / mrad: what the LIO update on the stream's map is run with."""
    pw = np.concatenate([t[0] for t in c["ticks"]])
    if n is not None and len(pw) > n:
        pw = pw[rng.choice(len(pw), n, replace=False)]
    pts = (pw + rng.normal(0, 1e-3, pw.shape)).astype(np.float32)
    prior = S.pack_state(S.so3_exp(np.array([0.002, -0.001, 0.0015])), np.array([0.004, -0.003, 0.002]), cov=np.eye(19) * 1e-4)
    return pts, prior


def box_scan():
    """Points on the mid-plane of every box of box_corners() (the plane a valid fit finds: z = c_z, or y = c_y for the
    equal-eigenvalue box) and the prior of lio_scan()."""
    cfg = box_corners()["cfg"]
    g = np.array([(x, y) for x in (-0.2, -0.1, 0.0, 0.1, 0.2) for y in (-0.1, 0.0, 0.1)])
    pts = []
    for name, key in BOX_KEYS.items():
        c, _ = node_center(cfg, key, [])
        if name == "equal_min":
            pts += [c + np.array([x, 0.0, y]) for x, y in g]
        else:
            pts += [c + np.array([x, y, 0.0]) for x, y in g]
    prior = S.pack_state(S.so3_exp(np.array([0.002, -0.001, 0.0015])), np.array([0.004, -0.003, 0.002]), cov=np.eye(19) * 1e-4)
    return np.array(pts, np.float32), prior


def replay(c, sides):
    """Feed every tick of case c to every side (objects with apply(pw, var) and flatten() / dump_nodes(), and slide(lo, hi));
    returns per side the history [{flat, dump, usage, slid}] after every tick."""
    hist = {name: [] for name in sides}
    for t, (pw, var) in enumerate(c["ticks"]):
        for name, s in sides.items():
            s.apply(pw, var)
            rec = dict(flat=s.flatten(), dump=s.dump_nodes(), usage=s.usage())
            if t in c.get("slides", {}):
                s.slide(*c["slides"][t])
                rec["slid"] = s.flatten()
                rec["slid_dump"] = s.dump_nodes()
            hist[name].append(rec)
    return hist
