"""ctypes bindings for the host mirror of the device voxel map: the export of a tick's touched roots replayed on the host
(tests/map_mirror_harness.cu), the shim's mirror (fl2_shim.cpp: ApplyMapExport, find_correspond), and find_correspond on the
oracle's map (oracle/orc_find.cpp) and on the reference source's (oracle/ref_find.cpp)."""
import ctypes as C
import os

import numpy as np

import __graft_entry__
import map_bind as MB
import oracle_bind as O
import shim_bind as SB
from fast_livo2_b200.synthetic import NODE_DTYPE, PLANE_DTYPE

REF_FIND_SO = os.path.join(O.ORACLE_DIR, "_ref", "libfl2_ref_find.so")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pin", "find_correspond.npz")


def _vp(a):
    return None if a is None else a.ctypes.data


class HarnessMap(MB.HostMap):
    """The host build of the device map state machine, with the export of the roots every tick touched."""

    def __init__(self, cfg, hash_cap=1 << 16, node_cap=1 << 16, pool_cap=1 << 19, rec_cap=1 << 16):
        MB.build()
        self.lib = lib = C.CDLL(__graft_entry__.MAP_MIRROR_HARNESS_LIB)  # map_host_harness.cu's entry points are in it too
        lib.maph_create.restype = C.c_void_p
        lib.maph_create.argtypes = [C.c_float, C.c_float, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_int]
        lib.maph_destroy.argtypes = [C.c_void_p]
        lib.maph_flatten.argtypes = [C.c_void_p] * 7
        lib.maph_usage.argtypes = [C.c_void_p, C.c_void_p]
        lib.maph_slide.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.maph_dump_nodes.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        lib.maph_apply_touched.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        lib.maph_export.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        lin = O.layer_init_num8(cfg)
        self.h = lib.maph_create(cfg.voxel_size, cfg.min_eigen_value, cfg.max_layer, cfg.max_points_num, lin.ctypes.data, hash_cap, node_cap, pool_cap, rec_cap)

    def apply_touched(self, pw, var, build=False):
        """The tick, then the slots of the roots it touched (slot order)."""
        pt = np.ascontiguousarray(np.concatenate([np.asarray(pw, np.float64).reshape(-1, 3), np.asarray(var, np.float64).reshape(-1, 9)], axis=1))
        slots, err = np.zeros(max(len(pt), 1), np.int32), C.c_int(0)
        n = self.lib.maph_apply_touched(self.h, pt.ctypes.data, len(pt), 1 if build else 0, slots.ctypes.data, C.byref(err))
        assert err.value == 0, f"host replay error flags {err.value}"
        return slots[:n].copy()

    def export(self, slots):
        slots = np.ascontiguousarray(slots, np.int32)
        nn = self.lib.maph_export(self.h, slots.ctypes.data, len(slots), None, None, None, None, 0)
        keys, first, count = np.zeros((len(slots), 3), np.int64), np.zeros(len(slots), np.int32), np.zeros(len(slots), np.int32)
        nodes = np.zeros(max(nn, 1), NODE_DTYPE)
        assert self.lib.maph_export(self.h, slots.ctypes.data, len(slots), keys.ctypes.data, first.ctypes.data, count.ctypes.data, nodes.ctypes.data, len(nodes)) == nn
        return dict(keys=keys, first=first, count=count, nodes=nodes[:nn])


def export_dump(exp):
    """The export as node-dump rows (oracle_bind.NODE_COLS), roots in key order."""
    n = exp["nodes"]
    rows = np.stack([n["key"][:, 0], n["key"][:, 1], n["key"][:, 2], n["layer"], n["path"], n["init_octo"], n["octo_state"], n["update_enable"], n["is_plane"],
                     n["new_points"], n["temp_points"], n["points_size"]], axis=1).astype(np.int64) if len(n) else np.zeros((0, 12), np.int64)
    return rows[np.lexsort((rows[:, 2], rows[:, 1], rows[:, 0]))] if len(rows) else rows


def export_flat(exp):
    """The candidate planes of the exported roots (a plane node none of whose ancestors is a plane: the walk of
    build_single_residual), in esikf_map_upload's flat form."""
    n = exp["nodes"]
    planes, first, count = [], [], []
    for f, c in zip(exp["first"], exp["count"]):
        blocked = np.zeros(c, bool)  # a plane at or above the row
        first.append(len(planes))
        for j in range(c):
            e = n[f + j]
            above = blocked[e["parent"]] if j else False
            blocked[j] = above or bool(e["is_plane"])
            if e["is_plane"] and not above:
                p = np.zeros(1, PLANE_DTYPE)[0]
                for k in ("center", "normal", "plane_var", "d", "radius", "layer", "path"):
                    p[k] = e[k]
                planes.append(p)
        count.append(len(planes) - first[-1])
    return dict(keys=exp["keys"], first=np.array(first, np.int32), count=np.array(count, np.int32), planes=np.array(planes, PLANE_DTYPE).reshape(-1))


def rows_of(dump, keys):
    """The rows of a node dump that belong to the given roots."""
    want = set(map(tuple, np.asarray(keys).tolist()))
    return dump[np.array([tuple(r) in want for r in dump[:, :3].tolist()], bool)] if len(dump) else dump


def flat_of(flat, keys):
    """The roots `keys` of a flattened map with their candidate planes."""
    ix = {tuple(k): i for i, k in enumerate(flat["keys"].tolist())}
    sel = [ix[tuple(k)] for k in np.asarray(keys).tolist()]
    planes = [flat["planes"][flat["first"][i]:flat["first"][i] + flat["count"][i]] for i in sel]
    count = np.array([flat["count"][i] for i in sel], np.int32)
    first = (np.cumsum(count) - count).astype(np.int32)
    return dict(keys=np.asarray(keys, np.int64).reshape(-1, 3), first=first, count=count, planes=np.concatenate(planes) if planes else np.zeros(0, PLANE_DTYPE))


class MirrorView:
    """The shim's mirror behind a handle (a standalone mirror, or a session's voxel_map_): node dump, flatten, find_correspond."""

    def __init__(self, h, lib=None):
        self.lib, self.h = lib or SB.load(), h

    def dump_nodes(self):
        return O._dump_nodes(lambda out, cap: self.lib.fl2_shim_mirror_dump(self.h, out.ctypes.data, cap))

    def flatten(self):
        nr, npl = C.c_int(0), C.c_int(0)
        assert self.lib.fl2_shim_mirror_flatten(self.h, C.byref(nr), C.byref(npl), None, None, None, None) == 0
        keys, first, count = np.zeros((nr.value, 3), np.int64), np.zeros(nr.value, np.int32), np.zeros(nr.value, np.int32)
        planes = np.zeros(npl.value, PLANE_DTYPE)
        self.lib.fl2_shim_mirror_flatten(self.h, C.byref(nr), C.byref(npl), _vp(keys), _vp(first), _vp(count), _vp(planes))
        return dict(keys=keys, first=first, count=count, planes=planes)

    def find(self, pts):
        pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
        out = np.zeros((len(pts), 4), np.int64)
        self.lib.fl2_shim_mirror_find(self.h, pts.ctypes.data, len(pts), out.ctypes.data)
        return out


class Mirror(MirrorView):
    """A mirror built on the CPU from exports (ApplyMapExport) and slide bounds (EraseRootsOutside)."""

    def __init__(self, cfg):
        lib = SB.load()
        super().__init__(lib.fl2_shim_mirror_create(cfg.voxel_size, cfg.max_layer), lib)

    def __del__(self):
        try:
            self.lib.fl2_shim_session_destroy(self.h)
        except Exception:
            pass

    def apply(self, exp):
        k, f, c = (np.ascontiguousarray(exp[x]) for x in ("keys", "first", "count"))
        n = np.ascontiguousarray(exp["nodes"])
        return self.lib.fl2_shim_mirror_apply(self.h, _vp(k), _vp(f), _vp(c), len(f), _vp(n), len(n))

    def erase(self, lo, hi):
        lo, hi = np.ascontiguousarray(lo, np.int64), np.ascontiguousarray(hi, np.int64)
        self.lib.fl2_shim_mirror_erase(self.h, lo.ctypes.data, hi.ctypes.data)


def oracle_find(orc, pts):
    """orc_lio_find_correspond on an oracle map (an OracleLIO, or map_streams.OracleSide)."""
    h = orc.o.h if hasattr(orc, "o") else orc.h
    lib = C.CDLL(os.path.join(O.ORACLE_DIR, "liborc_find.so"))
    lib.orc_lio_find_correspond.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
    out = np.zeros((len(pts), 4), np.int64)
    lib.orc_lio_find_correspond(C.c_void_p(h), pts.ctypes.data, len(pts), out.ctypes.data)
    return out


def ref_find_available():
    return os.path.exists(REF_FIND_SO)


class RefFindMap(O.RefMap):
    """The reference source's map (the ref_voxel_map.cpp driver) in the library that also has its find_correspond."""

    def __init__(self, cfg):
        lib = C.CDLL(REF_FIND_SO)
        lib.ref_map_create.restype = C.c_void_p
        lib.ref_map_create.argtypes = [C.c_void_p]
        lib.ref_map_destroy.argtypes = [C.c_void_p]
        lib.ref_map_update.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        lib.ref_map_flatten.argtypes = [C.c_void_p] * 7
        lib.ref_map_dump_nodes.restype = C.c_int
        lib.ref_map_dump_nodes.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        lib.ref_map_find_correspond.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        self.lib = lib
        a = O.c64([cfg.voxel_size, cfg.max_layer, cfg.min_eigen_value, cfg.max_points_num] + O.layer_init_num8(cfg).tolist())
        self.h = lib.ref_map_create(a.ctypes.data)

    def find(self, pts):
        pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
        out = np.zeros((len(pts), 4), np.int64)
        self.lib.ref_map_find_correspond(C.c_void_p(self.h), pts.ctypes.data, len(pts), out.ctypes.data)
        return out


def query_points(nodes, cfg, rng, n_random=2000):
    """find_correspond queries for a map whose nodes are `nodes` (NODE_DTYPE): every node's voxel_center_ (the strict `>`
    of every layer decides there), its eight corners at half its extent (root faces for the roots), the same points mirrored
    to negative coordinates (other, often absent roots), points of absent roots far away, and random points inside roots."""
    c = np.asarray(nodes["voxel_center"], np.float64)
    q = np.asarray(nodes["quater_length"], np.float64)[:, None]
    corners = np.array([[i, j, k] for i in (-1, 1) for j in (-1, 1) for k in (-1, 1)], np.float64)
    pts = [c, (c[:, None, :] + 2 * q[:, None, :] * corners[None]).reshape(-1, 3), -c, c + 1000.0]
    if len(c):
        base = c[rng.integers(0, len(c), n_random)]
        pts.append(base + rng.uniform(-1, 1, (n_random, 3)) * cfg.voxel_size / 2)
    return np.concatenate(pts)


# ---- shim sessions (fl2_shim.cpp's ShimSession): the managers as LIVMapper holds them, for the GPU tests and the timing tool
def vp(a):
    return a.ctypes.data_as(C.c_void_p)


def shim_sessions():
    """The shim library (shim_bind.load()), whose session entry points the mirror tests and tools/map_mirror_timing.py call."""
    return SB.load()


def session(lib, cfg, ext, vmap=None):
    """A session over the flat map `vmap` (None: an empty one) with the LIO configuration cfg and extrinsics ext."""
    from fast_livo2_b200 import api

    keys, first, count, planes = (np.ascontiguousarray(vmap[x]) for x in ("keys", "first", "count", "planes")) if vmap is not None else (
        np.zeros((0, 3), np.int64), np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, PLANE_DTYPE))
    lcfg = api.lio_cfg_c(cfg)
    extc = api.ExtrinsicsC()
    extc.extR[:], extc.extT[:], extc.Rcl[:], extc.Pcl[:] = ext.extR.reshape(9), ext.extT, ext.Rcl.reshape(9), ext.Pcl
    h = lib.fl2_shim_session_create(vp(keys), vp(first), vp(count), len(first), vp(planes), len(planes), C.addressof(lcfg), C.addressof(extc), None, None, 0)
    assert h, "fl2_shim_session_create failed"
    return h


class SessionContext:
    """The session's own esikf context behind api.Context's methods (`with SessionContext(lib, h) as ctx:`); the session
    keeps owning it."""

    def __init__(self, lib, h):
        self.lib, self.h = lib, h

    def __enter__(self):
        from fast_livo2_b200 import api

        self.ctx = api.Context.__new__(api.Context)
        self.ctx.lib, self.ctx.h = api.load_library(), C.c_void_p(self.lib.fl2_shim_session_context(self.h))
        return self.ctx

    def __exit__(self, *exc):
        self.ctx.h = None  # not destroyed here
        return False
