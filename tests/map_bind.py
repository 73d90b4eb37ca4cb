"""ctypes binding of tests/map_host_harness.cu (the device voxel-map state machine compiled for the host) + the comparison of
two flattened maps (keys / candidate lists / plane records) used by the CPU and GPU map tests."""
import ctypes as C

import numpy as np

import __graft_entry__
import oracle_bind as O
from fast_livo2_b200.synthetic import PLANE_DTYPE

SO = __graft_entry__.MAP_HARNESS_LIB


def build():
    __graft_entry__.build_map_harness()  # the one recipe (compiler, architecture, flags) build() uses too


class HostMap:
    def __init__(self, cfg, hash_cap=1 << 16, node_cap=1 << 16, pool_cap=1 << 19, rec_cap=1 << 16):
        build()
        self.lib = C.CDLL(SO)
        self.lib.maph_create.restype = C.c_void_p
        self.lib.maph_create.argtypes = [C.c_float, C.c_float, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_int]
        self.lib.maph_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        self.lib.maph_flatten.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        self.lib.maph_usage.argtypes = [C.c_void_p, C.c_void_p]
        self.lib.maph_destroy.argtypes = [C.c_void_p]
        self.lib.maph_slide.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        self.lib.maph_dump_nodes.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        self.lib.maph_slots_used.argtypes = [C.c_void_p]
        lin = O.layer_init_num8(cfg)
        self.h = self.lib.maph_create(cfg.voxel_size, cfg.min_eigen_value, cfg.max_layer, cfg.max_points_num, lin.ctypes.data, hash_cap, node_cap, pool_cap, rec_cap)

    def __del__(self):
        try:
            self.lib.maph_destroy(self.h)
        except Exception:
            pass

    def apply(self, pw, var, build=False):
        pt = np.ascontiguousarray(np.concatenate([np.asarray(pw, np.float64).reshape(-1, 3), np.asarray(var, np.float64).reshape(-1, 9)], axis=1))
        return self.lib.maph_apply(self.h, pt.ctypes.data, len(pt), 1 if build else 0)

    def flatten(self):
        nr, npl = C.c_int(0), C.c_int(0)
        self.lib.maph_flatten(self.h, C.byref(nr), C.byref(npl), None, None, None, None)
        keys, first, count = np.zeros((nr.value, 3), np.int64), np.zeros(nr.value, np.int32), np.zeros(nr.value, np.int32)
        planes = np.zeros(npl.value, PLANE_DTYPE)
        self.lib.maph_flatten(self.h, C.byref(nr), C.byref(npl), keys.ctypes.data, first.ctypes.data, count.ctypes.data, planes.ctypes.data)
        return dict(keys=keys, first=first, count=count, planes=planes)

    def slide(self, lo, hi):
        """mapSliding: keep the roots whose key lies in [lo, hi] (component-wise); everything is rebuilt into a fresh arena."""
        lo, hi = np.ascontiguousarray(lo, np.int64), np.ascontiguousarray(hi, np.int64)
        return self.lib.maph_slide(self.h, lo.ctypes.data, hi.ctypes.data)

    def dump_nodes(self):
        """Every octree node (oracle_bind.NODE_COLS), roots in key order, nodes in DFS pre-order."""
        return O._dump_nodes(lambda out, cap: self.lib.maph_dump_nodes(self.h, out.ctypes.data, cap))

    def slots_used(self):
        return self.lib.maph_slots_used(self.h)

    def usage(self):
        u = np.zeros(4, np.int64)
        self.lib.maph_usage(self.h, u.ctypes.data)
        return dict(nodes=int(u[0]), recs=int(u[1]), pool_points=int(u[2]), roots=int(u[3]))


def compare_flat_maps(a, b, rtol=1e-9, what=("a", "b"), exact=False):
    """Same root keys, same candidate count per root, candidate j of a root = the same plane (centre, +-normal, plane_var, d,
    radius, layer, path) within rtol. Returns the number of planes compared. The eigenvector sign of a fit is free: a flipped
    normal flips d and the normal-position cross block of plane_var."""
    ka = {tuple(k): i for i, k in enumerate(a["keys"].tolist())}
    kb = {tuple(k): i for i, k in enumerate(b["keys"].tolist())}
    assert set(ka) == set(kb), f"root voxels differ: {len(set(ka) - set(kb))} only in {what[0]}, {len(set(kb) - set(ka))} only in {what[1]}"
    ia = np.array([ka[k] for k in ka], np.int64)
    ib = np.array([kb[k] for k in ka], np.int64)
    assert np.array_equal(a["count"][ia], b["count"][ib]), "candidate counts per root differ"
    sel_a = np.concatenate([np.arange(f, f + c) for f, c in zip(a["first"][ia], a["count"][ia])] or [np.zeros(0, np.int64)]).astype(np.int64)
    sel_b = np.concatenate([np.arange(f, f + c) for f, c in zip(b["first"][ib], b["count"][ib])] or [np.zeros(0, np.int64)]).astype(np.int64)
    pa, pb = a["planes"][sel_a].copy(), b["planes"][sel_b].copy()
    # NaN (a plane fitted with two equal smallest eigenvalues keeps 0 / 0 terms in plane_var) must sit in the same fields on
    # both sides; it then compares equal whatever its payload: the CPU and the GPU need not produce the same NaN bits
    for f in ("center", "normal", "plane_var", "d", "radius"):
        na, nb = np.isnan(pa[f]), np.isnan(pb[f])
        assert np.array_equal(na, nb), f"NaN in different {f} fields of {what[0]} and {what[1]}"
        pa[f][na], pb[f][nb] = 0, 0
    if exact:  # every byte of every candidate record (centre, normal incl. its sign, plane_var, d, radius, layer, path)
        bad = np.nonzero(pa.view(np.uint8).reshape(len(pa), pa.dtype.itemsize) != pb.view(np.uint8).reshape(len(pb), pb.dtype.itemsize))[0]
        assert len(bad) == 0, f"{len(np.unique(bad))} of {len(pa)} plane records differ between {what[0]} and {what[1]}"
        return len(pa)
    assert np.array_equal(pa["layer"], pb["layer"]) and np.array_equal(pa["path"], pb["path"]), "candidate order (layer / path) differs"
    if len(pa) == 0:
        return 0
    np.testing.assert_allclose(pa["center"], pb["center"], rtol=rtol, atol=1e-12)
    sign = np.sign((pa["normal"] * pb["normal"]).sum(1))
    assert np.all(sign != 0)
    np.testing.assert_allclose(pa["normal"], pb["normal"] * sign[:, None], rtol=0, atol=1e-8)
    np.testing.assert_allclose(pa["d"], pb["d"] * sign, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(pa["radius"], pb["radius"], rtol=1e-6)
    # plane_var upper triangle: the normal block is rows / cols 0..2, the centre block 3..5; the cross block changes sign with the normal
    tri = [(i, j) for i in range(6) for j in range(i, 6)]
    flip = np.array([-1.0 if (i < 3) != (j < 3) else 1.0 for i, j in tri])
    va, vb = pa["plane_var"], pb["plane_var"] * np.where(sign[:, None] < 0, flip[None, :], 1.0)
    scale = np.abs(vb).max(axis=1, keepdims=True) + 1e-300
    # the refit sums are ill-conditioned where two eigenvalues nearly coincide (1 / (l_min - l_m)): relative to the plane's largest entry
    assert np.max(np.abs(va - vb) / scale) < max(rtol, 1e-7), f"plane_var differs by {np.max(np.abs(va - vb) / scale):.3e} (relative to the largest entry)"
    return len(pa)


def compare_node_dumps(a, b, what=("a", "b"), a_releases_cut_lists=False):
    """Node dumps (oracle_bind.NODE_COLS, roots in key order, DFS pre-order) equal row by row. With a_releases_cut_lists, `a`
    is the device state machine: it frees the temp_points_ of a node it cut (octo_state 1: a non-plane node above the last
    layer, which only forwards points and is never fitted again), where the reference keeps the list it distributed. There
    the list size of `a` must be 0 and the other side's is not compared. Returns the number of nodes."""
    assert a.shape == b.shape, f"{len(a)} nodes in {what[0]}, {len(b)} in {what[1]}"
    a, b = a.copy(), b.copy()
    if a_releases_cut_lists:
        cut = a[:, 6] == 1
        assert np.all(a[cut, 10] == 0), f"{what[0]} keeps the list of a cut node"
        b[cut, 10] = 0
    bad = np.nonzero(np.any(a != b, axis=1))[0]
    if len(bad):
        import oracle_bind as O

        i = bad[0]
        raise AssertionError(f"{len(bad)} of {len(a)} nodes differ between {what[0]} and {what[1]}; first: " +
                             ", ".join(f"{c} {x}/{y}" for c, x, y in zip(O.NODE_COLS, a[i], b[i])))
    return len(a)
