"""Seeded synthetic frames for the ESIKF update (SURVEY.md §8d "Synthetic inputs").

A frame is everything one LIO + VIO tick of LIVMapper hands to the hot path:

  * a flattened adaptive voxel map (root voxel keys -> ordered candidate-plane list,
    256-byte plane records) built by a vectorised numpy restatement of
    VoxelMapManager::BuildVoxelMap / VoxelOctoTree::init_plane
    (reference src/voxel_map.cpp:532-591, 55-135, 137-217),
  * a body-frame LiDAR scan (float32 xyz, the post-downsample `feats_down_body_`),
  * the prior state + 19x19 covariance (`state_propagat`),
  * a u8 image rendered at the true pose, visual map points and a reference image
    rendered from a displaced pose (the inputs of warpAffine / updateState).

This module is a data generator, not the oracle and not the product: it never imports
anything from oracle/ and performs no ESIKF arithmetic.
"""
from __future__ import annotations

import dataclasses
import numpy as np
import torch


def _bmm(a, b):
    """Batched small matmul (numpy's stacked @ is slow for 3x3 blocks)."""
    ta = torch.from_numpy(np.ascontiguousarray(a))
    tb = torch.from_numpy(np.ascontiguousarray(b))
    return torch.matmul(ta, tb).numpy()

STATE_PACK = 386  # R[9] p[3] inv_expo v[3] bg[3] ba[3] g[3] cov[361]

PLANE_DTYPE = np.dtype(
    [
        ("center", "<f8", (3,)),
        ("normal", "<f8", (3,)),
        ("plane_var", "<f8", (21,)),
        ("d", "<f4"),
        ("radius", "<f4"),
        ("layer", "<i4"),
        ("path", "<i4"),
        ("pad", "<i4", (6,)),
    ],
    align=False,
)
assert PLANE_DTYPE.itemsize == 256

# esikf_map_node (include/esikf_b200.h): one octree node of the device map as esikf_map_device_export writes it
NODE_DTYPE = np.dtype(
    [
        ("key", "<i8", (3,)),
        ("layer", "<i4"),
        ("path", "<i4"),
        ("parent", "<i4"),
        ("leaf", "<i4"),
        ("voxel_center", "<f8", (3,)),
        ("quater_length", "<f4"),
        ("init_octo", "u1"),
        ("octo_state", "u1"),
        ("update_enable", "u1"),
        ("is_plane", "u1"),
        ("new_points", "<i4"),
        ("points_size", "<i4"),
        ("temp_points", "<i4"),
        ("pad_", "<i4"),
        ("center", "<f8", (3,)),
        ("normal", "<f8", (3,)),
        ("plane_var", "<f8", (21,)),
        ("d", "<f4"),
        ("radius", "<f4"),
    ],
    align=False,
)


# ----------------------------------------------------------------------------- configs
@dataclasses.dataclass
class LioCfg:
    voxel_size: float = 0.5
    max_layer: int = 2
    max_iterations: int = 5
    sigma_num: float = 3.0
    dept_err: float = 0.02
    beam_err: float = 0.05
    min_eigen_value: float = 0.0025
    max_points_num: int = 50
    layer_init_num: tuple = (5, 5, 5, 5, 5)

    def as_array(self):
        return np.array(
            [self.voxel_size, self.max_layer, self.max_iterations, self.sigma_num, self.dept_err, self.beam_err,
             self.min_eigen_value, self.max_points_num], dtype=np.float64)


@dataclasses.dataclass
class VioCfg:
    levels: int = 4
    max_iterations: int = 5
    img_point_cov: float = 100.0
    exposure_estimate_en: bool = True
    inverse_composition_en: bool = False  # vio/inverse_composition_en (LIVMapper.cpp:60); false in every shipped config

    def as_array(self):
        return np.array([self.levels, self.max_iterations, self.img_point_cov, float(self.exposure_estimate_en)], dtype=np.float64)


@dataclasses.dataclass
class CamCfg:
    model: int = 0  # 0 pinhole(radtan), 1 equidistant
    width: int = 640
    height: int = 512
    fx: float = 646.78472
    fy: float = 646.65775
    cx: float = 313.456795
    cy: float = 261.399612
    d: tuple = (0.0, 0.0, 0.0, 0.0, 0.0)

    def as_array(self):
        return np.array([self.model, self.width, self.height, self.fx, self.fy, self.cx, self.cy, *self.d], dtype=np.float64)


@dataclasses.dataclass
class Extrinsics:
    extR: np.ndarray  # lidar -> imu rotation (config extrinsic_R)
    extT: np.ndarray
    Rcl: np.ndarray  # lidar -> camera
    Pcl: np.ndarray


def avia_extrinsics():  # config/avia.yaml:10-15
    return Extrinsics(
        extR=np.eye(3),
        extT=np.array([0.04165, 0.02326, -0.0284]),
        Rcl=np.array([[0.00610193, -0.999863, -0.0154172], [-0.00615449, 0.0153796, -0.999863], [0.999962, 0.00619598, -0.0060598]]),
        Pcl=np.array([0.0194384, 0.104689, -0.0251952]),
    )


def hilti_extrinsics():  # config/HILTI22.yaml (non-identity extrinsic_R)
    R = np.array([[-0.0028, -0.0076, -1.0], [-0.9999, 0.0115, 0.0027], [0.0115, 0.9999, -0.0076]])
    u, _, vt = np.linalg.svd(R)
    R = u @ vt
    return Extrinsics(
        extR=R,
        extT=np.array([-0.001, -0.00855, 0.055]),
        Rcl=np.array([[0.00610193, -0.999863, -0.0154172], [-0.00615449, 0.0153796, -0.999863], [0.999962, 0.00619598, -0.0060598]]),
        Pcl=np.array([0.0194384, 0.104689, -0.0251952]),
    )


# ----------------------------------------------------------------------------- small math
def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], dtype=np.float64)


def so3_exp(w):
    th = np.linalg.norm(w)
    if th < 1e-12:
        return np.eye(3)
    K = skew(w / th)
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def pack_state(R, p, inv_expo=1.0, v=None, bg=None, ba=None, g=None, cov=None):
    s = np.zeros(STATE_PACK)
    s[0:9] = np.asarray(R).reshape(9)
    s[9:12] = p
    s[12] = inv_expo
    s[13:16] = 0 if v is None else v
    s[16:19] = 0 if bg is None else bg
    s[19:22] = 0 if ba is None else ba
    s[22:25] = 0 if g is None else g
    s[25:] = np.asarray(np.eye(19) * 0.01 if cov is None else cov).reshape(361)
    return s


def unpack_state(s):
    return dict(R=s[0:9].reshape(3, 3).copy(), p=s[9:12].copy(), inv_expo=float(s[12]), v=s[13:16].copy(), bg=s[16:19].copy(),
                ba=s[19:22].copy(), g=s[22:25].copy(), cov=s[25:].reshape(19, 19).copy())


# ----------------------------------------------------------------------------- scene
@dataclasses.dataclass
class Rect:
    p0: np.ndarray  # centre
    n: np.ndarray  # unit normal
    u: np.ndarray  # in-plane unit axes
    v: np.ndarray
    hu: float  # half extents
    hv: float
    tex_seed: int


def _rect(p0, n, u, hu, hv, seed):
    n = np.asarray(n, float)
    n /= np.linalg.norm(n)
    u = np.asarray(u, float)
    u = u - n * (u @ n)
    u /= np.linalg.norm(u)
    v = np.cross(n, u)
    return Rect(np.asarray(p0, float), n, u, v, hu, hv, seed)


def make_scene(kind="room", scale=1.0):
    """Closed room of axis-aligned walls plus two tilted planes (>=6 non-parallel normals),
    or the degenerate 'corridor' scene (floor + ONE long wall) of BASELINE config 3."""
    s = scale
    X, Y, Z0, Z1 = 20.0 * s, 15.0 * s, -1.5 * s, 6.5 * s
    zc, zh = 0.5 * (Z0 + Z1), 0.5 * (Z1 - Z0)
    if kind == "corridor":
        return [
            _rect([0, 0, Z0], [0, 0, 1], [1, 0, 0], 60 * s, 60 * s, 1),
            _rect([0, Y, zc], [0, -1, 0], [1, 0, 0], 60 * s, zh * 4, 2),
        ]
    rects = [
        _rect([0, 0, Z0], [0, 0, 1], [1, 0, 0], X, Y, 1),
        _rect([0, 0, Z1], [0, 0, -1], [1, 0, 0], X, Y, 2),
        _rect([X, 0, zc], [-1, 0, 0], [0, 1, 0], Y, zh, 3),
        _rect([-X, 0, zc], [1, 0, 0], [0, 1, 0], Y, zh, 4),
        _rect([0, Y, zc], [0, -1, 0], [1, 0, 0], X, zh, 5),
        _rect([0, -Y, zc], [0, 1, 0], [1, 0, 0], X, zh, 6),
        # two tilted panels inside the room
        _rect([9 * s, 5 * s, Z0 + 1.2 * s], [-0.5, -0.2, 0.84], [1, 0, 0.6], 4 * s, 3 * s, 7),
        _rect([-8 * s, -6 * s, zc], [0.7, 0.6, 0.39], [0, 0, 1], 3.5 * s, 3 * s, 8),
    ]
    return rects


def raycast(rects, o, d):
    """o: (3,) or (N,3); d: (N,3) unit. Returns t (N,), plane index (N,), hit (N,3)."""
    o = np.broadcast_to(np.asarray(o, float), d.shape)
    best_t = np.full(d.shape[0], np.inf)
    best_i = np.full(d.shape[0], -1, dtype=np.int64)
    for i, r in enumerate(rects):
        denom = d @ r.n
        with np.errstate(divide="ignore", invalid="ignore"):
            t = ((r.p0 - o) @ r.n) / denom
        hit = o + d * t[:, None]
        rel = hit - r.p0
        ok = (np.abs(denom) > 1e-9) & (t > 1e-3) & (np.abs(rel @ r.u) <= r.hu) & (np.abs(rel @ r.v) <= r.hv) & (t < best_t)
        best_t = np.where(ok, t, best_t)
        best_i = np.where(ok, i, best_i)
    hit = o + d * np.where(np.isfinite(best_t), best_t, 0.0)[:, None]
    return best_t, best_i, hit


def texture(rects, idx, hit):
    """Band-limited procedural texture on each plane, in [30, 225]."""
    out = np.zeros(hit.shape[0])
    for i, r in enumerate(rects):
        m = idx == i
        if not m.any():
            continue
        rel = hit[m] - r.p0
        a, b = rel @ r.u, rel @ r.v
        rng = np.random.Generator(np.random.PCG64(1000 + r.tex_seed))
        val = np.zeros(a.shape[0])
        for _ in range(10):
            f = rng.uniform(0.6, 5.0)  # cycles / m  (kept low: smooth at every pyramid level)
            ang = rng.uniform(0, np.pi)
            ph = rng.uniform(0, 2 * np.pi)
            amp = rng.uniform(0.4, 1.0) / f ** 0.5
            val += amp * np.sin(2 * np.pi * f * (a * np.cos(ang) + b * np.sin(ang)) + ph)
        out[m] = val
    out = 127.5 + 97.5 * np.tanh(out / 1.6)
    return out


def sample_on_rects(rects, n, rng):
    areas = np.array([4 * r.hu * r.hv for r in rects])
    which = rng.choice(len(rects), size=n, p=areas / areas.sum())
    a = rng.uniform(-1, 1, n)
    b = rng.uniform(-1, 1, n)
    P0 = np.stack([r.p0 for r in rects])[which]
    U = np.stack([r.u * r.hu for r in rects])[which]
    V = np.stack([r.v * r.hv for r in rects])[which]
    return P0 + U * a[:, None] + V * b[:, None], which


# ----------------------------------------------------------------------------- sensor noise (body frame)
def calc_body_cov_np(pb, range_inc, degree_inc):
    """Vectorised calcBodyCov (src/voxel_map.cpp:15-34). pb: (N,3) float64 (z==0 already fixed)."""
    pb = pb.copy()
    pb[pb[:, 2] == 0, 2] = 0.0001
    rng_f = np.sqrt((pb ** 2).sum(1)).astype(np.float32)
    range_var = np.float32(range_inc) * np.float32(range_inc)
    dv = np.sin(np.float64(np.float32(degree_inc)) * 0.017453293) ** 2
    dirn = pb / np.linalg.norm(pb, axis=1, keepdims=True)
    b1 = np.stack([np.ones(len(pb)), np.ones(len(pb)), -(dirn[:, 0] + dirn[:, 1]) / dirn[:, 2]], 1)
    b1 /= np.linalg.norm(b1, axis=1, keepdims=True)
    b2 = np.cross(b1, dirn)
    b2 /= np.linalg.norm(b2, axis=1, keepdims=True)
    Nm = np.stack([b1, b2], 2)  # (N,3,2)
    dh = np.zeros((len(pb), 3, 3))
    dh[:, 0, 1], dh[:, 0, 2] = -dirn[:, 2], dirn[:, 1]
    dh[:, 1, 0], dh[:, 1, 2] = dirn[:, 2], -dirn[:, 0]
    dh[:, 2, 0], dh[:, 2, 1] = -dirn[:, 1], dirn[:, 0]
    A = rng_f.astype(np.float64)[:, None, None] * _bmm(dh, Nm)
    cov = dirn[:, :, None] * float(range_var) * dirn[:, None, :] + dv * _bmm(A, A.transpose(0, 2, 1))
    return cov


def add_sensor_noise(p_sensor, dept_err, beam_err_deg, rng):
    """Perturb points expressed in the sensor frame: range sigma + bearing sigma."""
    r = np.linalg.norm(p_sensor, axis=1, keepdims=True)
    d = p_sensor / r
    r_n = r + rng.normal(0, dept_err, r.shape)
    a = np.where(np.abs(d[:, [2]]) < 0.9, np.array([[0.0, 0.0, 1.0]]), np.array([[1.0, 0.0, 0.0]]))
    t1 = np.cross(d, a)
    t1 /= np.linalg.norm(t1, axis=1, keepdims=True)
    t2 = np.cross(d, t1)
    sb = np.sin(np.deg2rad(beam_err_deg))
    d_n = d + t1 * rng.normal(0, sb, r.shape) + t2 * rng.normal(0, sb, r.shape)
    d_n /= np.linalg.norm(d_n, axis=1, keepdims=True)
    return d_n * r_n


# ----------------------------------------------------------------------------- voxel keys
def voxel_keys(pw, voxel_size, float_voxel_size):
    """loc = (float)(p / voxel_size); if (loc < 0) loc -= 1.0; key = (int64)loc
    (src/voxel_map.cpp:561-567 uses a float voxel_size, :665-671 a double one)."""
    vs = np.float64(np.float32(voxel_size)) if float_voxel_size else np.float64(voxel_size)
    loc = (pw / vs).astype(np.float32)
    neg = loc < 0
    loc = np.where(neg, (loc.astype(np.float64) - 1.0).astype(np.float32), loc)
    return np.trunc(loc.astype(np.float64)).astype(np.int64)


# ----------------------------------------------------------------------------- map build (vectorised BuildVoxelMap)
def _fit_planes(pw, var, seg_start, seg_len, thr):
    """Batched init_plane (src/voxel_map.cpp:55-135) for segments of the sorted point array."""
    ns = seg_len.astype(np.float64)
    P2 = pw[:, :, None] * pw[:, None, :]
    sum_pp = np.add.reduceat(P2.reshape(-1, 9), seg_start, axis=0).reshape(-1, 3, 3)
    sum_p = np.add.reduceat(pw, seg_start, axis=0)
    center = sum_p / ns[:, None]
    covm = sum_pp / ns[:, None, None] - center[:, :, None] * center[:, None, :]
    covm = 0.5 * (covm + covm.transpose(0, 2, 1))
    evals, evecs = np.linalg.eigh(covm)  # ascending: min = 0, mid = 1, max = 2
    is_plane = evals[:, 0] < np.float32(thr)
    seg_id = np.repeat(np.arange(len(seg_start)), seg_len)
    dlt = pw - center[seg_id]  # (N,3)
    umin = evecs[:, :, 0]
    F = np.zeros((pw.shape[0], 3, 3))
    for m in (1, 2):
        um = evecs[:, :, m]
        S = um[:, :, None] * umin[:, None, :] + umin[:, :, None] * um[:, None, :]  # (S,3,3)
        with np.errstate(divide="ignore", invalid="ignore"):
            coef = 1.0 / (ns * (evals[:, 0] - evals[:, m]))
        coef = np.where(np.isfinite(coef), coef, 0.0)
        F[:, m, :] = _bmm(dlt[:, None, :], S[seg_id])[:, 0, :] * coef[seg_id][:, None]
    J = np.zeros((pw.shape[0], 6, 3))
    J[:, 0:3, :] = _bmm(evecs[seg_id], F)
    J[:, 3:6, :] = np.eye(3)[None] / ns[seg_id][:, None, None]
    JV = _bmm(_bmm(J, var), J.transpose(0, 2, 1))
    plane_var = np.add.reduceat(JV.reshape(-1, 36), seg_start, axis=0).reshape(-1, 6, 6)
    normal = umin
    radius = np.sqrt(np.maximum(evals[:, 2], 0)).astype(np.float32)
    d = (-(normal * center).sum(1)).astype(np.float32)
    return is_plane, center, normal, plane_var, radius, d


def build_voxel_map(pw, var, cfg: LioCfg):
    """Vectorised BuildVoxelMap + init_octo_tree + cut_octo_tree. pw: (N,3) float64 world
    points (float32-valued), var: (N,3,3). Returns a dict of flat arrays."""
    keys = voxel_keys(pw, cfg.voxel_size, float_voxel_size=True)
    order = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    pw, var, keys = pw[order], var[order], keys[order]
    chg = np.any(keys[1:] != keys[:-1], axis=1)
    root_start = np.concatenate([[0], np.nonzero(chg)[0] + 1])
    root_keys = keys[root_start]
    n_roots = len(root_start)
    root_of_pt = np.repeat(np.arange(n_roots), np.diff(np.concatenate([root_start, [len(pw)]])))
    vs_f = np.float64(np.float32(cfg.voxel_size))
    center0 = (0.5 + root_keys.astype(np.float64)) * vs_f
    ql0 = np.float32(np.float32(cfg.voxel_size) / np.float32(4))

    records = []  # tuples of arrays: root, layer, path, center, normal, plane_var, radius, d

    # level-synchronous recursion: each entry is a set of nodes with (point subset sorted by node)
    node_of_pt = root_of_pt.copy()  # node ids at the current layer, contiguous & sorted
    node_root = np.arange(n_roots)
    node_center = center0
    node_path = np.zeros(n_roots, dtype=np.int64)
    ql = ql0
    cur_pw, cur_var = pw, var
    for layer in range(cfg.max_layer + 1):
        if len(cur_pw) == 0:
            break
        chg = node_of_pt[1:] != node_of_pt[:-1]
        seg_start = np.concatenate([[0], np.nonzero(chg)[0] + 1])
        seg_len = np.diff(np.concatenate([seg_start, [len(cur_pw)]]))
        seg_node = node_of_pt[seg_start]
        enough = seg_len > cfg.layer_init_num[layer]
        is_plane, c, nrm, pv, rad, d = _fit_planes(cur_pw, cur_var, seg_start, seg_len, cfg.min_eigen_value)
        plane_mask = enough & is_plane
        if plane_mask.any():
            sn = seg_node[plane_mask]
            records.append((node_root[sn], np.full(sn.shape, layer), node_path[sn], c[plane_mask], nrm[plane_mask], pv[plane_mask],
                            rad[plane_mask], d[plane_mask]))
        if layer == cfg.max_layer:
            break
        # nodes to subdivide: enough points, not a plane
        sub = enough & ~is_plane
        sub_pt = np.repeat(sub, seg_len)
        if not sub_pt.any():
            break
        p_sub, v_sub = cur_pw[sub_pt], cur_var[sub_pt]
        n_sub = node_of_pt[sub_pt]
        cc = node_center[n_sub]
        xyz = (p_sub > cc).astype(np.int64)
        leaf = 4 * xyz[:, 0] + 2 * xyz[:, 1] + xyz[:, 2]
        child_id = n_sub * 8 + leaf
        o2 = np.argsort(child_id, kind="stable")
        p_sub, v_sub, child_id, leaf, n_sub, xyz = p_sub[o2], v_sub[o2], child_id[o2], leaf[o2], n_sub[o2], xyz[o2]
        uniq, first_idx, inv = np.unique(child_id, return_index=True, return_inverse=True)
        new_center = node_center[n_sub[first_idx]] + (2 * xyz[first_idx] - 1) * np.float64(ql)
        new_root = node_root[n_sub[first_idx]]
        new_path = node_path[n_sub[first_idx]] | (leaf[first_idx] << (3 * layer))
        node_of_pt = inv
        node_root, node_center, node_path = new_root, new_center, new_path
        cur_pw, cur_var = p_sub, v_sub
        ql = np.float32(ql / np.float32(2))

    if records:
        root = np.concatenate([r[0] for r in records])
        layer = np.concatenate([r[1] for r in records])
        path = np.concatenate([r[2] for r in records])
        center = np.concatenate([r[3] for r in records])
        normal = np.concatenate([r[4] for r in records])
        plane_var = np.concatenate([r[5] for r in records])
        radius = np.concatenate([r[6] for r in records])
        d = np.concatenate([r[7] for r in records])
    else:
        root = layer = path = np.zeros(0, np.int64)
        center = normal = np.zeros((0, 3))
        plane_var = np.zeros((0, 6, 6))
        radius = d = np.zeros(0, np.float32)
    # DFS order inside a root = lexicographic (leaf at layer 1, leaf at layer 2, ...); a plane
    # node terminates its branch so no prefix ambiguity exists.
    sort_keys = [((path >> (3 * l)) & 7) for l in reversed(range(max(cfg.max_layer, 1)))]
    o = np.lexsort(tuple(sort_keys) + (root,))
    root, layer, path = root[o], layer[o], path[o]
    planes = np.zeros(len(root), dtype=PLANE_DTYPE)
    planes["center"] = center[o]
    planes["normal"] = normal[o]
    iu = np.triu_indices(6)
    planes["plane_var"] = plane_var[o][:, iu[0], iu[1]]
    planes["d"] = d[o]
    planes["radius"] = radius[o]
    planes["layer"] = layer
    planes["path"] = path
    count = np.bincount(root, minlength=n_roots).astype(np.int32)
    first = np.concatenate([[0], np.cumsum(count)[:-1]]).astype(np.int32)
    return dict(keys=np.ascontiguousarray(root_keys, dtype=np.int64), first=first, count=count, planes=planes)


# ----------------------------------------------------------------------------- camera (generator side)
def cam_rays(cam: CamCfg, px):
    """Unit bearing vectors for pixels (N,2). Pinhole without distortion / equidistant."""
    x = (px[:, 0] - cam.cx) / cam.fx
    y = (px[:, 1] - cam.cy) / cam.fy
    if cam.model == 0:
        if abs(cam.d[0]) > 1e-7:
            x0, y0 = x.copy(), y.copy()
            d = cam.d
            for _ in range(8):
                r2 = x * x + y * y
                icd = 1.0 / (1 + ((d[4] * r2 + d[1]) * r2 + d[0]) * r2)
                dx = 2 * d[2] * x * y + d[3] * (r2 + 2 * x * x)
                dy = d[2] * (r2 + 2 * y * y) + 2 * d[3] * x * y
                x, y = (x0 - dx) * icd, (y0 - dy) * icd
        f = np.stack([x, y, np.ones_like(x)], 1)
    else:
        td = np.sqrt(x * x + y * y)
        th = td.copy()
        k = cam.d
        for _ in range(12):
            t2 = th * th
            th = td / (1 + k[0] * t2 + k[1] * t2 ** 2 + k[2] * t2 ** 3 + k[3] * t2 ** 4)
        sc = np.where(td > 1e-8, np.tan(th) / np.maximum(td, 1e-12), 1.0)
        f = np.stack([x * sc, y * sc, np.ones_like(x)], 1)
    return f / np.linalg.norm(f, axis=1, keepdims=True)


def cam_project(cam: CamCfg, pc):
    x, y = pc[:, 0] / pc[:, 2], pc[:, 1] / pc[:, 2]
    if cam.model == 0:
        d = cam.d
        if abs(d[0]) > 1e-7:
            r2 = x * x + y * y
            cd = 1 + d[0] * r2 + d[1] * r2 ** 2 + d[4] * r2 ** 3
            a1, a2, a3 = 2 * x * y, r2 + 2 * x * x, r2 + 2 * y * y
            x, y = x * cd + d[2] * a1 + d[3] * a2, y * cd + d[2] * a3 + d[3] * a1
        return np.stack([cam.fx * x + cam.cx, cam.fy * y + cam.cy], 1)
    r = np.sqrt(x * x + y * y)
    th = np.arctan(r)
    k = cam.d
    thd = th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8)
    sc = np.where(r > 1e-8, thd / np.maximum(r, 1e-12), 1.0)
    return np.stack([cam.fx * x * sc + cam.cx, cam.fy * y * sc + cam.cy], 1)


def camera_pose(ext: Extrinsics, R_wi, p_wi):
    """(Rcw, Pcw) from the IMU pose (src/vio.cpp:57-58, 1542-1543)."""
    Rli = ext.extR.T
    Pli = -ext.extR.T @ ext.extT
    Rci = ext.Rcl @ Rli
    Pci = ext.Rcl @ Pli + ext.Pcl
    Rcw = Rci @ R_wi.T
    Pcw = -Rci @ R_wi.T @ p_wi + Pci
    return Rcw, Pcw


def render(rects, cam: CamCfg, Rcw, Pcw, expo_gain=1.0):
    uu, vv = np.meshgrid(np.arange(cam.width, dtype=np.float64), np.arange(cam.height, dtype=np.float64))
    px = np.stack([uu.ravel(), vv.ravel()], 1)
    f = cam_rays(cam, px)
    d = f @ Rcw  # Rcw^T f
    o = -Rcw.T @ Pcw
    t, idx, hit = raycast(rects, o, d)
    val = texture(rects, idx, hit) * expo_gain
    val[idx < 0] = 0
    img = np.clip(np.rint(val), 0, 255).astype(np.uint8).reshape(cam.height, cam.width)
    return img


# ----------------------------------------------------------------------------- the frame
def random_prior_cov(rng, scale=1.0):
    sig = np.concatenate([np.full(3, np.deg2rad(0.5)), np.full(3, 0.05), [0.01], np.full(3, 0.1), np.full(3, 3e-3), np.full(3, 3e-3),
                          np.full(3, 3e-3)]) * scale
    A = rng.normal(size=(19, 19))
    C = A @ A.T / 19.0
    dC = np.sqrt(np.diag(C))
    C = C / dC[:, None] / dC[None, :]
    C = 0.75 * np.eye(19) + 0.25 * C
    return C * sig[:, None] * sig[None, :]


def make_frame(seed=0, n_pts=5000, n_map=200_000, n_patches=0, lio: LioCfg | None = None, vio: VioCfg | None = None,
               cam: CamCfg | None = None, ext: Extrinsics | None = None, scene="room", scene_scale=1.0, prior_sigma=(0.5, 0.05),
               fov="sphere", make_image=None, ref_offset=(5.0, 0.3)):
    """Build one seeded synthetic LIO(+VIO) frame. Returns a dict of numpy arrays."""
    lio = lio or LioCfg()
    vio = vio or VioCfg()
    cam = cam or CamCfg()
    ext = ext or avia_extrinsics()
    make_image = (n_patches > 0) if make_image is None else make_image
    rng = np.random.Generator(np.random.PCG64(seed))
    rects = make_scene(scene, scene_scale)

    # ground-truth IMU pose
    R_true = so3_exp(rng.normal(0, 0.15, 3))
    p_true = np.array([rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-0.3, 0.8)]) * scene_scale
    R_wl = R_true @ ext.extR
    p_wl = R_true @ ext.extT + p_true

    # ---- map: points on the scene with sensor noise as seen from the true pose, BuildVoxelMap at truth
    P_map_cov = np.zeros((19, 19))
    P_map_cov[0:3, 0:3] = np.eye(3) * np.deg2rad(0.1) ** 2
    P_map_cov[3:6, 3:6] = np.eye(3) * 0.01 ** 2
    mp_w, _ = sample_on_rects(rects, n_map, rng)
    mp_l = (mp_w - p_wl) @ R_wl  # R_wl^T (p - t)
    mp_l = add_sensor_noise(mp_l, lio.dept_err, lio.beam_err, rng).astype(np.float32)
    mp_ld = mp_l.astype(np.float64)
    mp_wn = ((mp_ld @ ext.extR.T + ext.extT) @ R_true.T + p_true).astype(np.float32).astype(np.float64)
    bc = calc_body_cov_np(mp_ld, lio.dept_err, lio.beam_err)
    RE = R_true @ ext.extR
    cm = np.zeros((n_map, 3, 3))
    cm[:, 0, 1], cm[:, 0, 2] = -mp_ld[:, 2], mp_ld[:, 1]
    cm[:, 1, 0], cm[:, 1, 2] = mp_ld[:, 2], -mp_ld[:, 0]
    cm[:, 2, 0], cm[:, 2, 1] = -mp_ld[:, 1], mp_ld[:, 0]
    var = _bmm(_bmm(np.broadcast_to(RE, (n_map, 3, 3)), bc), np.broadcast_to(RE.T, (n_map, 3, 3))) + P_map_cov[0:3, 0:3][0, 0] * _bmm(cm, cm.transpose(0, 2, 1)) + P_map_cov[3:6, 3:6]
    vmap = build_voxel_map(mp_wn, var, lio)

    # ---- scan
    if fov == "sphere":
        d = rng.normal(size=(int(n_pts * 1.15) + 64, 3))
    else:  # forward cone (Avia-like 70 deg)
        d = rng.normal(size=(int(n_pts * 1.15) + 64, 3)) * 0.45 + np.array([1.0, 0, 0])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    dw = d @ R_wl.T
    t, idx, hit = raycast(rects, p_wl, dw)
    ok = (idx >= 0) & (t > 0.8)
    hit = hit[ok][:n_pts]
    while hit.shape[0] < n_pts:  # top up (rare)
        hit = np.concatenate([hit, hit[: n_pts - hit.shape[0]]])
    sc_l = (hit - p_wl) @ R_wl
    sc_l = add_sensor_noise(sc_l, lio.dept_err, lio.beam_err, rng).astype(np.float32)

    # ---- prior
    cov = random_prior_cov(rng)
    dth = rng.normal(0, np.deg2rad(prior_sigma[0]), 3)
    dp = rng.normal(0, prior_sigma[1], 3)
    inv_expo_true = 1.0
    state_true = pack_state(R_true, p_true, inv_expo_true, v=rng.normal(0, 0.5, 3), g=np.array([0, 0, -9.81]), cov=cov)
    state_prior = pack_state(R_true @ so3_exp(dth), p_true + dp, inv_expo_true * (1 + rng.normal(0, 0.02)), v=state_true[13:16],
                             bg=rng.normal(0, 1e-3, 3), ba=rng.normal(0, 1e-3, 3), g=np.array([0, 0, -9.81]), cov=cov)

    frame = dict(seed=seed, lio_cfg=lio, vio_cfg=vio, cam_cfg=cam, ext=ext, map=vmap, pts=np.ascontiguousarray(sc_l),
                 state_true=state_true, state_prior=state_prior, rects=rects)

    if make_image:
        Rcw, Pcw = camera_pose(ext, R_true, p_true)
        img = render(rects, cam, Rcw, Pcw)
        # visual points: pixels inside the border, cast onto the scene
        border = (4 + 1) * (1 << vio.levels) + 8
        px = np.stack([rng.uniform(border, cam.width - border, n_patches * 2), rng.uniform(border, cam.height - border, n_patches * 2)], 1)
        f = cam_rays(cam, px)
        o = -Rcw.T @ Pcw
        t, idx, hit = raycast(rects, o, f @ Rcw)
        ok = idx >= 0
        # reference frame pose
        R_ref = R_true @ so3_exp(rng.normal(0, 1, 3) / np.sqrt(3) * np.deg2rad(ref_offset[0]))
        p_ref = p_true + rng.normal(0, 1, 3) / np.sqrt(3) * ref_offset[1]
        Rcw_r, Pcw_r = camera_pose(ext, R_ref, p_ref)
        pc_ref = hit @ Rcw_r.T + Pcw_r
        px_ref = cam_project(cam, pc_ref)
        ok &= (pc_ref[:, 2] > 0.1) & (px_ref[:, 0] > border) & (px_ref[:, 0] < cam.width - border) & (px_ref[:, 1] > border) & (
            px_ref[:, 1] < cam.height - border)
        sel = np.nonzero(ok)[0][:n_patches]
        normals = np.stack([r.n for r in rects])[idx[sel]]
        img_ref = render(rects, cam, Rcw_r, Pcw_r)
        frame.update(img=img, img_ref=img_ref, vis_pos=np.ascontiguousarray(hit[sel]), vis_normal=np.ascontiguousarray(normals),
                     px_ref=np.ascontiguousarray(px_ref[sel]), T_ref=(Rcw_r, Pcw_r), T_cur_true=(Rcw, Pcw),
                     inv_ref_expo=np.ones(len(sel)))
    return frame


def scan_at(rects, ext: Extrinsics, R_wi, p_wi, n_pts, lio: LioCfg, rng, fov="sphere"):
    """One noisy body-frame scan (float32, n_pts x 3) of the scene from the IMU pose (R_wi, p_wi): the per-tick input of a
    multi-tick run (tests of the device-resident map)."""
    R_wl = R_wi @ ext.extR
    p_wl = R_wi @ ext.extT + p_wi
    hits = np.zeros((0, 3))
    while len(hits) < n_pts:
        d = rng.normal(size=(int(n_pts * 1.3) + 64, 3))
        if fov != "sphere":
            d = d * 0.45 + np.array([1.0, 0, 0])
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        t, idx, hit = raycast(rects, p_wl, d @ R_wl.T)
        hits = np.concatenate([hits, hit[(idx >= 0) & (t > 0.8)]])
    sc_l = (hits[:n_pts] - p_wl) @ R_wl
    return np.ascontiguousarray(add_sensor_noise(sc_l, lio.dept_err, lio.beam_err, rng).astype(np.float32))


# ----------------------------------------------------------------------------- on-disk cache (frames take tens of seconds to build)
def frame_cache_dir():
    """Where seeded frames are cached: $FL2_FRAME_CACHE, else a per-user directory under the system temp dir (never the
    source tree, which may be read-only)."""
    import os
    import tempfile

    return os.environ.get("FL2_FRAME_CACHE") or os.path.join(tempfile.gettempdir(), f"fast_livo2_frames_{os.getuid()}")


def cached_frame(cache_dir=None, **kw):
    """make_frame(**kw) with a pickle cache keyed by the arguments and by this generator's source (defaults to
    frame_cache_dir(), which several checkouts may share: a changed generator never reuses another version's frames)."""
    import hashlib
    import os
    import pickle

    cache_dir = cache_dir or frame_cache_dir()
    with open(os.path.abspath(__file__), "rb") as f:
        src = hashlib.sha1(f.read()).hexdigest()
    key = hashlib.sha1((src + repr(sorted((k, repr(v)) for k, v in kw.items()))).encode()).hexdigest()[:16]
    path = os.path.join(cache_dir, f"frame_{key}.pkl")
    if os.path.exists(path):
        try:
            with open(path, "rb") as f:
                return pickle.load(f)
        except Exception:
            pass
    fr = make_frame(**kw)
    try:
        os.makedirs(cache_dir, exist_ok=True)
        tmp = path + f".{os.getpid()}.tmp"
        with open(tmp, "wb") as f:
            pickle.dump(fr, f, protocol=4)
        os.replace(tmp, path)
    except Exception:
        pass
    return fr
