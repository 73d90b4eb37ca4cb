"""The VIO front end's keyed find_correspond lookups (esikf_map_device_find) on the oracle's map (oracle/orc_find_keyed.cpp),
query sets for them, and the comparison of the device's answers with the oracle's and with the device map's own export."""
import ctypes as C
import os

import numpy as np

import oracle_bind as O

RULES = {"patch": 0, "raycast": 1}  # api.FIND_RULE_PATCH / FIND_RULE_RAYCAST
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pin", "find_keyed.npz")
REF_SO = os.path.join(O.ORACLE_DIR, "_ref", "libfl2_ref_find_keyed.so")
NONE_KEY = np.iinfo(np.int64).min


def oracle_find_keyed(orc, pts, rule):
    """orc_lio_find_correspond_keyed on an oracle map (an OracleLIO, or map_streams.OracleSide): out n x 6 int64 = status, key,
    layer, path; f n x 29 = center, normal, plane_var (upper triangle), d, radius of the found node."""
    h = orc.o.h if hasattr(orc, "o") else orc.h
    lib = C.CDLL(os.path.join(O.ORACLE_DIR, "liborc_find_keyed.so"))
    lib.orc_lio_find_correspond_keyed.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
    out, f = np.zeros((len(pts), 6), np.int64), np.zeros((len(pts), 29), np.float64)
    lib.orc_lio_find_correspond_keyed(C.c_void_p(h), pts.ctypes.data, len(pts), rule, out.ctypes.data, f.ctypes.data)
    return out, f


def key_patch_numpy(p):
    """updateReferencePatch's key (src/vio.cpp:983-989) spelled in numpy: the double quotient by 0.5 narrowed to float32, one
    subtracted in double and narrowed again when negative, truncated. NaN / inf / out of range: NONE_KEY."""
    p = np.asarray(p, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        loc = (p / 0.5).astype(np.float32)
        loc = np.where(loc < 0, (loc.astype(np.float64) - 1.0).astype(np.float32), loc)
        ok = (loc > np.float32(-(2**20) - 1)) & (loc < np.float32(2**20))
        return np.where(ok, np.trunc(np.where(ok, loc, 0)).astype(np.int64), NONE_KEY)


def key_raycast_numpy(p):
    """The ray casting's key (:508-514, int loc_xyz): floor(p / 0.5), one less when negative. Out of range: NONE_KEY."""
    p = np.asarray(p, np.float64)
    with np.errstate(invalid="ignore"):
        f = np.floor(p / 0.5)
        ok = (f >= -(2**20)) & (f < 2**20)
        k = np.where(ok, f, 0).astype(np.int64)
        k = np.where(k < 0, k - 1, k)
        ok &= k >= -(2**20)
        return np.where(ok, k, NONE_KEY)


def boundary_points(voxel_size=0.5):
    """Coordinates at the key rules' edges, for x, y and z in turn (the other two on a root inside the room scenes): a quotient
    that rounds up to an integer in float32 (2 k + 1 - 2^-30 and friends), negative exact multiples of 0.5, -0.0 and 0.0, the
    keys at +-2^20 on both sides, NaN and infinities, and the root faces of the map's voxel size."""
    c = []
    for k in (1, 3, 7, 100, 12345, 2**19):
        q = np.nextafter(np.float32(k), np.float32(0))  # the float below k: its half-ulp neighbours round up to k in float
        for e in (-1e-9, -1e-12, 0.0):
            c += [(k + e) * 0.5, -(k + e) * 0.5]
        c += [float(q) * 0.5, -float(q) * 0.5]
    c += [-0.5 * k for k in range(1, 9)] + [0.5 * k for k in range(0, 9)] + [-0.0, 0.0, 1e-300, -1e-300]
    for b in (2**20, 2**20 + 1, 2**20 - 1):  # key = floor / trunc of 2 p
        for s in (-1, 1):
            for e in (-0.25, -1e-6, 0.0, 1e-6, 0.25):
                c.append(s * (b + e) * 0.5)
    c += [np.nan, np.inf, -np.inf, 1e300, -1e300]
    c += [voxel_size * k + e for k in range(-4, 5) for e in (-1e-12, 0.0, 1e-12)]
    c = np.array(c, np.float64)
    base = np.array([1.3, 0.7, 0.2])
    pts = []
    for ax in range(3):
        p = np.tile(base, (len(c), 1))
        p[:, ax] = c
        pts.append(p)
    return np.concatenate(pts)


def compare_with_oracle(got, orc_out, orc_f, what, rtol=1e-6):
    """Device answers (api.Context.map_device_find) against the oracle's: status, key, layer, path exactly; the plane fields of
    found nodes to test_gpu_map's tolerance (the device refits in its own summation order), zero rows where there is no root."""
    st, key, rows = got["status"], got["key"], got["planes"]
    bad = np.nonzero((st != orc_out[:, 0]) | np.any(key != orc_out[:, 1:4], axis=1))[0]
    assert len(bad) == 0, f"{what}: status / key differ on {len(bad)} points; first {bad[0]}: device {st[bad[0]]} {key[bad[0]]}, oracle {orc_out[bad[0]]}"
    found = st != 0
    assert np.array_equal(rows["layer"][found], orc_out[found, 4]) and np.array_equal(rows["path"][found], orc_out[found, 5]), f"{what}: layer / path differ"
    assert not np.any(rows[~found].view(np.uint8)), f"{what}: a row without a root is not zero"
    planes = st == 2
    f = np.concatenate([rows["center"], rows["normal"], rows["plane_var"], rows["d"][:, None], rows["radius"][:, None]], axis=1)
    np.testing.assert_allclose(f[planes], orc_f[planes], rtol=rtol, atol=1e-9, err_msg=f"{what}: plane fields")


def export_rows_by_node(exp):
    """The export's rows keyed by (root key, layer, path)."""
    n = exp["nodes"]
    return {(int(n["key"][i, 0]), int(n["key"][i, 1]), int(n["key"][i, 2]), int(n["layer"][i]), int(n["path"][i])): i for i in range(len(n))}


def plane_bytes_equal_export(got, exp):
    """Every found node whose root the export holds: the find row's plane fields are the export row's bytes. Returns how many
    rows were checked."""
    idx = export_rows_by_node(exp)
    n, rows, checked = exp["nodes"], got["planes"], 0
    for i in np.nonzero(got["status"] != 0)[0]:
        k = (*map(int, got["key"][i]), int(rows["layer"][i]), int(rows["path"][i]))
        j = idx.get(k)
        if j is None:
            continue
        for f in ("center", "normal", "plane_var", "d", "radius"):
            assert rows[f][i].tobytes() == n[f][j].tobytes(), f"point {i}: {f} differs from the export's row of node {k}"
        checked += 1
    return checked


def ref_available():
    return os.path.exists(REF_SO)


class RefKeyed:
    """The reference source's own updateReferencePatch (rule A) and ray-casting retrieval (rule B) on the reference's own map
    (oracle/ref_find_keyed.cpp), fed with the same (point_w, var) ticks as the oracle's map."""

    def __init__(self, cfg, cam, ext, vio_cfg):
        L = self.lib = C.CDLL(REF_SO)
        vp = C.c_void_p
        L.ref_keyed_create.restype = vp
        L.ref_keyed_create.argtypes = [vp] * 7
        L.ref_keyed_destroy.argtypes = [vp]
        L.ref_keyed_update.argtypes = [vp, vp, vp, C.c_int]
        L.ref_keyed_update_reference_patch.argtypes = [vp, vp, C.c_int, vp]
        L.ref_keyed_raycast.restype = C.c_int
        L.ref_keyed_raycast.argtypes = [vp, vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, C.c_int]
        mc = O.c64([cfg.voxel_size, cfg.max_layer, cfg.min_eigen_value, cfg.max_points_num] + O.layer_init_num8(cfg).tolist())
        self._keep = [mc, O.c64(cam.as_array()), O.c64(ext.extR), O.c64(ext.extT), O.c64(ext.Rcl), O.c64(ext.Pcl), O.c64(vio_cfg.as_array())]
        self.h = L.ref_keyed_create(*[k.ctypes.data for k in self._keep])
        assert self.h

    def __del__(self):
        try:
            self.lib.ref_keyed_destroy(C.c_void_p(self.h))
        except Exception:
            pass

    def update(self, pw, var):
        pw, var = O.c64(pw).reshape(-1, 3), O.c64(var).reshape(-1, 9)
        self.lib.ref_keyed_update(C.c_void_p(self.h), pw.ctypes.data, var.ctypes.data, len(pw))

    def update_reference_patch(self, pos):
        pos = O.c64(pos).reshape(-1, 3)
        out = np.zeros((len(pos), 3))
        self.lib.ref_keyed_update_reference_patch(C.c_void_p(self.h), pos.ctypes.data, len(pos), out.ctypes.data)
        return out

    def raycast(self, state, rays):
        """rays: a list of (k x 3) camera-frame sample arrays, one per grid cell. Returns the samples' world points (concatenated)
        and add_from_voxel_map (m x 6: point_w, normal)."""
        count = np.array([len(r) for r in rays], np.int32)
        first = (np.cumsum(count) - count).astype(np.int32)
        flat = O.c64(np.concatenate(rays))
        sw, add = np.zeros_like(flat), np.zeros((len(rays), 6))
        n = self.lib.ref_keyed_raycast(C.c_void_p(self.h), O.c64(state).ctypes.data, len(rays), first.ctypes.data, count.ctypes.data, flat.ctypes.data, len(flat),
                                       sw.ctypes.data, add.ctypes.data, len(add))
        return sw, add[:n]


def expect_reference_patch(q, out, f):
    """What updateReferencePatch leaves in normal_ under the rule-A pin's set-up, from the keyed restatement's answers: the found
    plane's normal where a plane is found, 0 elsewhere. ambiguous: a plane is found but the gate's float range_dis may be NaN
    (dis_to_center - dis_to_plane^2 at or below 0 in float), where the reference keeps 0."""
    plane = out[:, 0] == 2
    n, c, d = f[:, 3:6], f[:, 0:3], f[:, 27]
    dp = (((n[:, 0] * q[:, 0] + n[:, 1] * q[:, 1]) + n[:, 2] * q[:, 2]) + d).astype(np.float32)
    dc = ((((c[:, 0] - q[:, 0]) ** 2) + (c[:, 1] - q[:, 1]) ** 2) + (c[:, 2] - q[:, 2]) ** 2).astype(np.float32)
    ambiguous = plane & ((dc - dp * dp) <= np.float32(1e-6))
    want = np.where(plane[:, None], n, 0.0)
    return want, ambiguous


def expect_raycast(samples_w, counts, out, f):
    """add_from_voxel_map of the ray-casting branch with an empty scan and feat_map, from the keyed restatement's rule-B answers:
    per cell in order, the centre and normal of the plane found for the first of its samples that finds one."""
    rows, start = [], 0
    for k in counts:
        hit = np.nonzero(out[start:start + k, 0] == 2)[0]
        if len(hit):
            j = start + hit[0]
            rows.append(np.concatenate([f[j, 0:3], f[j, 3:6]]))
        start += k
    return np.array(rows).reshape(-1, 6)
