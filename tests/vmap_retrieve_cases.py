"""The map side of the visual sub-map retrieval (esikf_vmap_place_points / esikf_vmap_retrieve) restated on the host.

Placement: insertPointIntoVoxelMap (src/vio.cpp:227-250) keys a point by float(c / 0.5), minus 1.0 in double and narrowed
again when negative, then truncated; a voxel's voxel_points list is its points in placement order. placed_visual_map() builds
the flat visual map of oracle/orc_retrieve.cpp's orc_retrieve_walk from that rule and order, so the walk restated there runs
over the map the reference's insertion makes (retrieve_cases.flat_visual_map groups by the scan's floor rule instead).

Composed retrieval: walk (orc_retrieve_walk) -> depth check (orc_depth_check) -> the is_normal_initialized_ skip, per cell in
cell order, as esikf_vmap_retrieve returns them."""
import ctypes as C
import os

import numpy as np

import retrieve_cases as RC
import vmap_cases as VC
from fast_livo2_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_VRETRIEVE_SO = os.path.join(ROOT, "oracle", "_ref", "libfl2_ref_vretrieve.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pin", "vmap_retrieve.npz")
vp = C.c_void_p
KEPT, DEPTH, NOT_INIT, NO_REF, NO_WINNER = 0, 1, 2, 3, 4


def insertion_keys(p):
    """insertPointIntoVoxelMap's key of every point (n, 3) -> (n, 3) int64."""
    q = (np.asarray(p, np.float64) / 0.5).astype(np.float32)
    q = np.where(q < 0, (q.astype(np.float64) - 1.0).astype(np.float32), q)
    return np.trunc(q).astype(np.int64)


def placed_visual_map(pos, n_obs, order):
    """The flat visual map of the points placed in `order` (point ids, placement order): vkeys, vfirst, vcount, the points'
    pos and n_obs in voxel-list order, and `ids`, the point id of each of them."""
    order = np.asarray(order, np.int64)
    k = insertion_keys(pos[order])
    srt = np.lexsort((np.arange(len(order)),) + tuple(k.T[::-1]))  # by key, then placement order
    ks = k[srt]
    head = np.ones(len(ks), bool)
    head[1:] = np.any(ks[1:] != ks[:-1], axis=1)
    first = np.nonzero(head)[0].astype(np.int32)
    count = np.diff(np.append(first, len(ks))).astype(np.int32)
    ids = order[srt].astype(np.int32)
    return dict(vkeys=np.ascontiguousarray(ks[first]), vfirst=first, vcount=count, pos=np.ascontiguousarray(pos[ids], np.float64),
                n_obs=np.ascontiguousarray(n_obs[ids], np.int32), ids=ids)


def composed(orc, sc, vis, keys, depth, normal_init):
    """walk -> depth check -> skip on the oracle. Returns the walk order the sub_feat_map iterated (its keys after the erase,
    then the erased ones, which hold no candidate) and per TYPE_MAP cell: cell, point_id, pc, status (KEPT for the points the
    choice runs on)."""
    s = dict(sc, **vis)
    w = orc.walk(s, keys)
    cells = np.nonzero(w["grid_type"])[0]
    flat = w["cell_pt"][cells]
    pid = np.where(flat >= 0, vis["ids"][np.maximum(flat, 0)], -1).astype(np.int32)
    pc = w["cell_pc"][cells]
    status = np.full(len(cells), NO_WINNER, np.int32)
    has = pid >= 0
    if has.any():
        flag = orc.depth_check(sc, depth, vis["pos"][flat[has]], pc[has])
        ni = np.asarray(normal_init, bool)[pid[has]]
        status[has] = np.where(flag != 0, DEPTH, np.where(~ni, NOT_INIT, KEPT))
    kept = {tuple(k) for k in w["sub_keys"].tolist()}
    rest = [k for k in np.asarray(keys).tolist() if tuple(k) not in kept]
    order = np.concatenate([w["sub_keys"], np.asarray(rest, np.int64).reshape(-1, 3)]).astype(np.int32)
    return order, dict(cell=cells.astype(np.int32), point_id=pid, pc=pc, status=status, sub_keys=w["sub_keys"], grid_type=w["grid_type"])


# ----------------------------------------------------------------------------------------------- ticks over one visual map
HAND = np.array([[-0.3, -0.2, 6.0], [np.nextafter(-1.0, np.inf), 0.2, 6.5], [-0.5000000001, 0.3, 7.0], [0.4999999999, -0.3, 7.5], [-1e-9, 0.1, 5.0],
                 [-2.7500000001, -3.25, 1.0], [np.nextafter(-0.5, np.inf), 1.0, -2.0]])  # negative, and where the float narrowing moves the key


def frame_pos(sc):
    st = S.unpack_state(sc["state"])
    R, t = S.camera_pose(sc["ext"], st["R"], st["p"])
    return -(R.T @ t)


def ticks(n_ticks=3, n_scan=20000, n_vis=1500, seed=40):
    """Consecutive frames of config 2's camera over one growing visual map: tick t adds its scene's visual points (tick 0 also
    the hand-built HAND points), with ids in order, placed in a shuffled order; each has n_obs observations with random
    patches, a few frame ids and camera centres around the frame's. Per tick: the scene, and the new points' ids, pos, normal,
    normal_init, n_obs, the packed observations (first, patch, id, T_f_w) and the placement order."""
    out, base = [], 0
    for t in range(n_ticks):
        sc = RC.scene("pinhole", n_scan, seed=seed + t, n_vis=n_vis)
        rng = np.random.default_rng(seed + 100 + t)
        pos, normal, n_obs = sc["pos"], sc["normal"], sc["n_obs"]
        if t == 0:
            pos, normal, n_obs = np.concatenate([pos, HAND]), np.concatenate([normal, np.tile([0.0, 0.0, -1.0], (len(HAND), 1))]), np.append(n_obs, np.ones(len(HAND), np.int32))
        n = len(pos)
        st = S.unpack_state(sc["state"])
        Rcw, _ = S.camera_pose(sc["ext"], st["R"], st["p"])
        first = np.concatenate([[0], np.cumsum(n_obs)]).astype(np.int32)
        m = int(first[-1])
        centre = frame_pos(sc) + rng.normal(0, 2.0, (m, 3))
        # a point of several observations has two frame ids at least: with every id_ equal the reference reads an unset
        # ref_ftr (DESIGN.md §4), which the restatement and the device report as no reference feature
        fid = rng.integers(0, 4, m).astype(np.int32)
        two = first[:-1][np.diff(first) >= 2]
        fid[two + 1] = (fid[two] + 1) % 4
        T = np.concatenate([np.tile(Rcw.reshape(1, 9), (m, 1)), -(centre @ Rcw.T)], 1)
        out.append(dict(sc=sc, ids=np.arange(base, base + n, dtype=np.int32), pos=np.ascontiguousarray(pos), normal=np.ascontiguousarray(normal),
                        ninit=(rng.random(n) > 0.1).astype(np.uint8), n_obs=n_obs.astype(np.int32), first=first,
                        patch=rng.uniform(0, 255, (m, 64)).astype(np.float32), fid=fid, T=np.ascontiguousarray(T),
                        order=(base + rng.permutation(n)).astype(np.int32)))
        base += n
    return out


def _cell_arrays(sc, cells):
    L = sc["grid_n_width"] * sc["grid_n_height"]
    cell_pt = np.full(L, -1, np.int32)
    cell_pt[cells["cell"]] = cells["point_id"]
    return cell_pt


def restate_ticks(tks, normal_en):
    """The restatement over the ticks: placement, walk -> depth check -> skip (composed) and the reference choice
    (vmap_cases.OracleStore.choose). Per tick: sub_keys, grid_type, cell_pt (ids), survivors (ids, cell order), ref (their ref
    position; with normal_en the stored ref_patch), the walk order and the per-cell answers; and the final feat_map."""
    sc0 = tks[0]["sc"]
    total = sum(len(tk["ids"]) for tk in tks)
    orc, store = RC.OracleRetrieve(sc0), VC.OracleStore(sc0["cam"], sc0["ext"], capacity=total)
    P, Nm, NO, NI = np.zeros((total, 3)), np.zeros((total, 3)), np.zeros(total, np.int32), np.zeros(total, np.uint8)
    order, out = [], []
    for tk in tks:
        ids = store.add(tk["first"], np.zeros((len(tk["patch"]), 2)), tk["patch"], tk["T"], tk["fid"], np.zeros(len(tk["patch"]), np.float32),
                        np.zeros(len(tk["patch"]), np.float32), np.full(len(tk["ids"]), -1, np.int32))
        assert np.array_equal(ids, tk["ids"])
        P[ids], Nm[ids], NO[ids], NI[ids] = tk["pos"], tk["normal"], tk["n_obs"], tk["ninit"]
        order += tk["order"].tolist()
        n = ids[-1] + 1
        vis = placed_visual_map(P[:n], NO[:n], order)
        sc = tk["sc"]
        s = orc.scan(sc)
        walk, cells = composed(orc, sc, vis, s["keys"], s["depth"], NI[:n])
        kept = cells["status"] == KEPT
        pid = cells["point_id"][kept]
        ref = store.choose(pid, normal_en, pos=P[pid], frame_pos=frame_pos(sc))
        ref_all = np.full(len(cells["cell"]), -1, np.int32)
        ref_all[kept] = ref
        out.append(dict(sub_keys=cells["sub_keys"], grid_type=cells["grid_type"], cell_pt=_cell_arrays(sc, cells), survivors=pid[ref >= 0].astype(np.int32),
                        ref=ref[ref >= 0].astype(np.int32), walk=walk, cells=cells, ref_all=ref_all))
    return out, placed_visual_map(P, NO, order)


def ref_vretrieve_available():
    return os.path.exists(REF_VRETRIEVE_SO)


class RefVretrieve:
    """The reference source's own insertPointIntoVoxelMap + retrieveFromVisualSparseMap on one VIOManager (oracle/ref_vretrieve.cpp)."""

    def __init__(self, sc):
        L = self.lib = C.CDLL(REF_VRETRIEVE_SO)
        L.ref_vrt_create.restype = vp
        L.ref_vrt_create.argtypes = [vp] * 7
        L.ref_vrt_destroy.argtypes = [vp]
        L.ref_vrt_place.argtypes = [vp, C.c_int] + [vp] * 8
        L.ref_vrt_feat_map.restype = C.c_int
        L.ref_vrt_feat_map.argtypes = [vp] * 4
        L.ref_vrt_retrieve.restype = C.c_int
        L.ref_vrt_retrieve.argtypes = [vp, vp, vp] + [C.c_int] * 6 + [vp] * 6
        self._keep = RC._cam_ext(sc) + [np.ascontiguousarray(sc["img"], np.uint8)]
        self.h = L.ref_vrt_create(*[k.ctypes.data for k in self._keep])
        assert self.h
        self.points = 0

    def place(self, tk):
        idx = tk["order"] - tk["ids"][0]  # the new points in placement order
        first = tk["first"]
        cnt = np.diff(first)[idx]
        f2 = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
        obs = np.concatenate([np.arange(first[i], first[i + 1]) for i in idx]).astype(np.int64) if len(idx) else np.zeros(0, np.int64)
        a = [np.ascontiguousarray(x) for x in (tk["order"], tk["pos"][idx], tk["normal"][idx], tk["ninit"][idx], f2, tk["patch"][obs], tk["fid"][obs], tk["T"][obs])]
        self.lib.ref_vrt_place(self.h, len(idx), *[x.ctypes.data for x in a])
        self.points += len(idx)

    def feat_map(self):
        keys, first, ids = np.zeros((max(self.points, 1), 3), np.int64), np.zeros(self.points + 1, np.int32), np.zeros(max(self.points, 1), np.int32)
        k = self.lib.ref_vrt_feat_map(self.h, keys.ctypes.data, first.ctypes.data, ids.ctypes.data)
        return keys[:k], first[:k + 1], ids[:self.points]

    def retrieve(self, sc, normal_en):
        pg = np.ascontiguousarray(sc["pg"], np.float64)
        L = sc["grid_n_width"] * sc["grid_n_height"]
        out = dict(sub_keys=np.zeros((max(len(pg), 1), 3), np.int64), grid_type=np.zeros(L, np.uint8), cell_pt=np.zeros(L, np.int32), survivors=np.zeros(L, np.int32),
                   ref=np.zeros(L, np.int32))
        ns = C.c_int32(0)
        k = self.lib.ref_vrt_retrieve(self.h, np.ascontiguousarray(sc["state"]).ctypes.data, pg.ctypes.data, len(pg), *RC._grid(sc), int(bool(normal_en)),
                                      *[out[f].ctypes.data for f in ("sub_keys", "grid_type", "cell_pt", "survivors", "ref")], C.byref(ns))
        out["sub_keys"] = out["sub_keys"][:k]
        out["survivors"], out["ref"] = out["survivors"][:ns.value], out["ref"][:ns.value]
        return out

    def __del__(self):
        try:
            self.lib.ref_vrt_destroy(self.h)
        except Exception:
            pass


def feat_map_lists(keys, first, ids):
    """feat_map as {key: [point ids in voxel_points order]}."""
    return {tuple(int(x) for x in keys[j]): ids[first[j]:first[j + 1]].tolist() for j in range(len(keys))}
