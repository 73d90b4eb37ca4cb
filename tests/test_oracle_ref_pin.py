"""Pins the LIO oracle (oracle/orc_lio.cpp, a restatement) against the REFERENCE'S OWN SOURCE: FAST-LIVO2's src/voxel_map.cpp
compiled against stand-in headers for Eigen / PCL / ROS (oracle/ref_shim/, oracle/ref_voxel_map.cpp ->
oracle/_ref/libfl2_ref_lio.so). The reference ships no tests or golden vectors of its own; its compiled update loop
(VoxelMapManager::StateEstimation with BuildResidualListOMP / build_single_residual, OpenMP on) is the next best thing.

Where the library is built (oracle/Makefile, from a FAST-LIVO2 source tree) the oracle must reproduce it on every case below: iteration count, effective feature number per iteration (parsed from the reference's own console line),
the final ptpl_list_ (matched plane centres and signed distances, in order), pv.normal of every point — all bit-exact —
and the posterior state / covariance to 1e-12 (the two differ only in the summation order of small fixed-size products).
Without the library every case compares with the reference's stored outputs (tests/golden/ref_pin/lio.npz, written by a
run with FL2_RECORD_REF_PIN=1 where the library is built; see oracle_bind.RefPin). tests/golden/ref_lio_golden.npz
holds the reference's full outputs for two of the cases (test_oracle_matches_reference_golden) — tests/golden/make_ref_golden.py
regenerates it."""
import ctypes as C

import numpy as np
import pytest

import oracle_bind as O
from conftest import get_frame
from fast_livo2_b200 import synthetic as S
from harness import lio_oracle
from map_bind import oracle_update_map, tick_points
from ref_pin_cases import EDGE_FRAMES, LIO_CASES, LIO_GOLDEN, lio_case

PIN = O.RefPin("lio")
needs_ref = pytest.mark.skipif(not O.RefPin.available("lio"), reason="neither oracle/_ref/libfl2_ref_lio.so nor tests/golden/ref_pin/lio.npz")
EXACT = ("M", "ptpl_center", "ptpl_dis", "normals")


def _ref_lio(fr, **kw):
    """The reference's StateEstimation (live, or its stored outputs): what _check compares."""
    r = O.ref_lio_state_estimation(fr, **kw)
    return {k: r[k] for k in ("iters", "M", "ptpl_center", "ptpl_dis", "normals", "state")}


def _check(o, r, planes):
    assert o["iters"] == r["iters"]
    assert O.same(o["M"], r, "M")  # effective feature number of every iteration
    mk = o["match_plane"] >= 0
    # ptpl_list_ keeps the scan order of the matched points: plane by plane and distance by distance (shapes included)
    assert O.same(planes["center"][o["match_plane"][mk]], r, "ptpl_center")
    assert O.same(o["dis_to_plane"][mk], r, "ptpl_dis")
    want = np.where(o["normal_plane"][:, None] >= 0, planes["normal"][np.maximum(o["normal_plane"], 0)], 0.0)
    assert O.same(want, r, "normals")  # pv.normal, zero when the point never matched
    d = np.abs(o["state"] - r["state"])
    assert d[:25].max() <= 1e-12 * max(1.0, np.abs(r["state"][:25]).max())
    assert d[25:].max() <= 1e-12 * np.abs(r["state"][25:]).max()


@needs_ref
@pytest.mark.parametrize("name", list(LIO_CASES))
def test_oracle_reproduces_the_reference_source(name):
    fr, cfg = lio_case(name)
    o = lio_oracle(fr, cfg)
    r = PIN.get(f"state_estimation/{name}", lambda: _ref_lio(fr, cfg=cfg), exact=EXACT)
    assert r["iters"] >= 2
    _check(o, r, fr["map"]["planes"])


@needs_ref
def test_oracle_reproduces_the_reference_source_on_early_stop():
    """A tight prior converges twice in a row: the rematch / stop rule (voxel_map.cpp:477-499) ends the loop after 2 iterations."""
    fr, cfg = lio_case("small")
    st = lio_oracle(fr, cfg)["state"].copy()
    st[25:] = (np.eye(19) * 1e-12).reshape(-1)
    fr2 = dict(fr, state_prior=st)
    o = lio_oracle(fr2, cfg)
    r = PIN.get("early_stop", lambda: _ref_lio(fr2, cfg=cfg), exact=EXACT)
    assert r["iters"] == 2
    _check(o, r, fr["map"]["planes"])


@needs_ref
@pytest.mark.parametrize("kind", list(EDGE_FRAMES))
def test_edge_scan_oracle_reproduces_the_reference_source(kind):
    """Voxel corners / faces with both signs, float neighbours of them, z == 0 and off-plane points that exercise the
    neighbour rule (parity_util.edge_scan), for voxel sizes 0.5 / 0.4 / 2.0: oracle against the reference source."""
    from parity_util import edge_scan

    fr = get_frame(**EDGE_FRAMES[kind])
    pts, ext, state = edge_scan(fr)
    fr2 = dict(fr, ext=ext, pts=pts, state_prior=state)
    lio = O.OracleLIO(fr["lio_cfg"], ext)
    lio.set_map(fr["map"])
    o = lio.state_estimation(pts, state, state)
    r = PIN.get(f"edge_scan/{kind}", lambda: _ref_lio(fr2), exact=EXACT)
    assert o["M"][0] > 20
    # the neighbour rule is exercised: some points match a plane that is not in their own voxel's candidate list
    _check(o, r, fr["map"]["planes"])


@needs_ref
@pytest.mark.parametrize("name", ["main", "displaced"])
def test_hand_built_association_oracle_reproduces_the_reference_source(name):
    """The hand-built maps of tests/lio_assoc.py: roots with up to 131 candidates in layer-2 / layer-3 leaves, byte-identical
    planes (exact probability ties, the first in DFS order wins), range-gate failures and one-ulp radius boundaries,
    neighbour voxels from one to 130 candidates, with ties, without a plane or absent; at the pose the scan was placed at and at a displaced prior. The sigma_num = 40 case of
    the same file is not pinned here: where a candidate passes with this_prob == 0 the reference pushes an uninitialised
    PointToPlane, so its output is undefined; the oracle's documented rule (DESIGN §4) and the numpy restatement
    (test_oracle_numpy_crosscheck.py) are the references there."""
    import lio_assoc

    fr = lio_assoc.case(name)
    o = lio_oracle(fr, fr["lio_cfg"])
    r = PIN.get(f"assoc/{name}", lambda: _ref_lio(fr, cfg=fr["lio_cfg"]), exact=EXACT)
    assert r["iters"] == 5
    _check(o, r, fr["map"]["planes"])


@needs_ref
def test_calc_body_cov_matches_the_reference_source():
    import ctypes as C

    olib = O.load()
    rng = np.random.default_rng(0)
    pts = [np.ascontiguousarray(p.astype(np.float32).astype(np.float64)) for p in np.concatenate([rng.normal(0, 5, (50, 3)), [[1.0, 2.0, 0.001], [0.3, -0.2, 7.0]]])]

    def ref_cov():
        lib = C.CDLL(O.REF_LIO_SO)
        a = np.zeros((len(pts), 9))
        for i, p in enumerate(pts):
            lib.ref_calc_body_cov(p.ctypes.data_as(C.c_void_p), C.c_float(0.02), C.c_float(0.05), a[i].ctypes.data_as(C.c_void_p))
        return dict(cov=a)

    a = PIN.get("calc_body_cov", ref_cov)["cov"]
    for i, p in enumerate(pts):
        b, cm = np.zeros(9), np.zeros(9)
        olib.orc_calc_body_cov(O.dptr(p.copy()), C.c_float(0.02), C.c_float(0.05), O.dptr(b), O.dptr(cm))
        np.testing.assert_allclose(b, a[i], rtol=1e-13, atol=1e-300)


@pytest.mark.parametrize("name", ["small", "hilti_voxel_04_non_identity_extrinsics"])
def test_oracle_matches_reference_golden(name):
    """Same check against the committed outputs of the reference source (generated by tests/golden/make_ref_golden.py)."""
    g = np.load(LIO_GOLDEN)
    fr, cfg = lio_case(name)
    o = lio_oracle(fr, cfg)
    r = dict(iters=int(g[f"{name}_iters"]), M=g[f"{name}_M"], ptpl_center=g[f"{name}_ptpl_center"], ptpl_dis=g[f"{name}_ptpl_dis"], normals=g[f"{name}_normals"],
             state=g[f"{name}_state"])
    _check(o, r, fr["map"]["planes"])


def _compare_map(MB, orc_flat, ref, key, what):
    """The oracle's flattened map against the reference's: every plane where the library is built (a fixed sample of root
    voxels is recorded), else the stored sample plus the digests of the whole key set and candidate counts."""
    if PIN.live:
        rf = ref.flatten()
        PIN.get(key, lambda: O.flat_map_sample(rf, n_roots=8))
        return MB.compare_flat_maps(orc_flat, rf, rtol=1e-9, what=what)
    return O.compare_with_map_sample(MB, orc_flat, PIN.get(key, None), 1e-9, what)


@needs_ref
@pytest.mark.parametrize("cfg", [S.LioCfg(), S.LioCfg(voxel_size=0.4, max_layer=3, max_points_num=20)], ids=["avia_defaults", "voxel0.4_layer3_max20"])
def test_oracle_update_voxel_map_reproduces_the_reference_source(cfg):
    """The map construction (f1's oracle): VoxelMapManager::UpdateVoxelMap / UpdateOctoTree / init_octo_tree / cut_octo_tree /
    init_plane of the REFERENCE SOURCE against the oracle's restatement, tick by tick on the same (point_w, var) lists: the same
    root voxels, the same octree shape (candidate planes per root in DFS order, layer / path), every plane's centre, normal,
    plane_var, d and radius. Tolerance, not bits: the reference calls Eigen::EigenSolver, which here is the stand-in's Jacobi
    and in the oracle another Jacobi — a genuine Eigen would differ in the last bits just the same."""
    import map_bind as MB

    rng = np.random.default_rng(5)
    rects = S.make_scene("room", 0.5)
    cid = "layer%d_max%d_voxel%g" % (cfg.max_layer, cfg.max_points_num, cfg.voxel_size)
    orc, ref = O.OracleLIO(cfg, S.avia_extrinsics()), (O.RefMap(cfg) if PIN.live else None)
    n = 0
    for tick in range(8):
        lo = np.array([-10.0 + 1.5 * tick, -8.0, -2.0])
        pw, var = tick_points(rng, rects, 6000, lo, lo + np.array([8.0, 16.0, 6.0]))
        oracle_update_map(orc, pw, var)
        if ref is not None:
            ref.update(pw, var)
        n = _compare_map(MB, orc.flatten(), ref, f"update_map/{cid}/tick{tick}", ("oracle", "reference source"))
        if tick == 5:
            f = orc.flatten()  # equal to the reference's (compared just above)
            assert f["count"].max() > 1 and (f["planes"]["layer"] > 0).any()  # octrees were cut: several candidates per root
            # mapSliding's clearMemOutOfMap (:950-971) in between, then more ticks on the pruned maps
            c, half = np.array([4, -2, 1]), 14
            b = [int(c[0] + half), int(c[0] - half), int(c[1] + half), int(c[1] - half), int(c[2] + half), int(c[2] - half)]
            deleted = orc.lib.orc_lio_clear_out_of_map(orc.h, *b)
            if ref is not None:
                ref.lib.ref_map_clear_out_of_map(C.c_void_p(ref.h), *b)
            assert deleted > 0
            _compare_map(MB, orc.flatten(), ref, f"update_map/{cid}/cleared", ("oracle after clearMemOutOfMap", "reference source"))
    assert n > 1500


@needs_ref
def test_oracle_build_voxel_map_reproduces_the_reference_source():
    """First LiDAR frame (LIVMapper.cpp:356-366): TransformLidar + BuildVoxelMap (per-point covariance with the raw body point's
    cross matrix and calcBodyCov's own z fix, all points pushed, then init_octo_tree with the recursive cut) of the REFERENCE
    SOURCE against the oracle's tick_build_map on a 60 k-point scan with non-identity extrinsics — the form the device map's
    esikf_map_device_build is held to."""
    import map_bind as MB

    cfg, ext = S.LioCfg(), S.hilti_extrinsics()
    rng = np.random.default_rng(21)
    rects = S.make_scene("room", 0.5)
    R0, p0 = S.so3_exp(np.array([0.01, -0.02, 0.3])), np.array([-2.0, 0.5, 0.3])
    st0 = S.pack_state(R0, p0, cov=S.random_prior_cov(np.random.default_rng(3), scale=0.05), g=np.array([0, 0, -9.81]))
    scan = S.scan_at(rects, ext, R0, p0, 60000, cfg, rng)
    orc, ref = O.OracleLIO(cfg, ext), (O.RefMap(cfg) if PIN.live else None)
    orc.tick_build_map(scan, st0)
    if ref is not None:
        ref.build(scan, st0, ext, cfg)
    n = _compare_map(MB, orc.flatten(), ref, "build_map", ("oracle BuildVoxelMap", "reference source"))
    assert n > 1500


@needs_ref
@pytest.mark.parametrize("name", ["deep_blob_L3", "deep_blob_L7", "deep_cut", "candidates_growth", "candidates_layer3", "layer_init_update", "layer_init_cut",
                                  "max_points_last_layer", "max_points_cut", "refit_flip", "on_centre", "box_corners", "big_list", "key_edges", "slide"])
def test_oracle_map_streams_reproduce_the_reference_source(name):
    """The hand-built streams of tests/map_streams.py (deep octrees, 64 / 72 candidates, per-layer layer_init_num, every
    max_points_num boundary, refits that flip plane / non-plane, points on split planes, box-corner eigenvalues at the
    threshold and equal smallest eigenvalues, slides): the oracle's UpdateVoxelMap / clearMemOutOfMap against the REFERENCE
    SOURCE's after every tick, node by node (every field of the node dump equal) and plane by plane (1e-9; NaN in the same
    fields). The whole maps are stored: they are small."""
    import map_bind as MB
    import map_streams as MS

    c = MS.case(name)
    o = MS.replay(c, {"orc": MS.OracleSide(c["cfg"])})["orc"]
    r = MS.replay(c, {"ref": MS.RefSide(c["cfg"])})["ref"] if PIN.live else None
    for t, x in enumerate(o):
        for stage in ("", "slid") if "slid" in x else ("",):
            flat, dump = (x["slid"], x["slid_dump"]) if stage else (x["flat"], x["dump"])
            key = f"map/{name}/tick{t}{'/' + stage if stage else ''}"
            y = PIN.get(key, lambda: {**(r[t]["slid"] if stage else r[t]["flat"]), "dump": r[t]["slid_dump"] if stage else r[t]["dump"]})
            what = (f"oracle, tick {t} {stage}", "reference source")
            MB.compare_node_dumps(dump, y["dump"], what)
            MB.compare_flat_maps(flat, {k: y[k] for k in ("keys", "first", "count", "planes")}, rtol=1e-9, what=what)
