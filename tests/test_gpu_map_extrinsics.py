"""GPU: the device-resident voxel map and the LIO precompute at non-identity LiDAR extrinsics (HILTI22's extR, benchmarked as
config 3).

With extR = I the per-point stage of the device map (map_points_kernel: the world point R (extR p + extT) + t, M = R extR and
var = M B M^T + (-C) P_rot (-C)^T + P_pos) cannot tell R extR from extR R, extR from extR^T, or the IMU-frame point of the
cross matrix from the raw body point. Here R and extR are far from commuting, so each of those slips moves points or
covariances and the maps stop matching the oracle's.

The second half holds a resident scan (esikf_lio_set_scan once, esikf_lio_run many times) to what StateEstimation does on
every call: recompute calcBodyCov and the cross vector (voxel_map.cpp:349-360) with the extrinsics and noise model of that
call. It also checks that esikf_set_lidar_extrinsics and esikf_set_extrinsics keep the camera part as documented."""
import contextlib
import dataclasses

import numpy as np
import pytest

import harness as H
import map_bind as MB
import map_mirror as MM
import oracle_bind as O
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from parity_util import assert_state_close

pytestmark = pytest.mark.gpu

CFG3 = S.LioCfg(voxel_size=0.4, min_eigen_value=1e-4, max_points_num=100)  # config 3's map settings (HILTI22)
G = np.array([0, 0, -9.81])


@contextlib.contextmanager
def contexts(n):
    cs = [api.Context(0) for _ in range(n)]
    try:
        yield cs
    finally:
        for c in cs:
            c.close()


def first_frame(scene="room", n=60000):
    """The inputs of test_oracle_ref_pin's BuildVoxelMap pin: seed 21, a 60 k-point scan at R0 = Exp(0.01, -0.02, 0.3)."""
    rng = np.random.default_rng(21)
    rects = S.make_scene(scene, 0.5)
    R0, p0 = S.so3_exp(np.array([0.01, -0.02, 0.3])), np.array([-2.0, 0.5, 0.3])
    st0 = S.pack_state(R0, p0, cov=S.random_prior_cov(np.random.default_rng(3), scale=0.05), g=G)
    return rects, rng, st0, (R0, p0)


def device_build(ctx, cfg, ext, scan0, st0):
    ctx.set_extrinsics(ext)
    ctx.map_device_init(cfg, root_capacity=1 << 16, grow=True)
    ctx.lio_set_scan(scan0)
    ctx.map_device_build(st0)


def prior_near(R, p, prev):
    """The previous posterior pushed towards the pose (R, p) with some error (stands in for IMU propagation)."""
    cov = S.unpack_state(prev)["cov"] + np.eye(19) * 1e-6
    return S.pack_state(R @ S.so3_exp(np.array([0.002, -0.003, 0.002])), p + np.array([0.02, -0.015, 0.01]), cov=cov, g=G)


def aligned_planes(a, b):
    """The candidate planes of two flat maps with the same roots, root by root in a's order."""
    kb = {tuple(k): i for i, k in enumerate(b["keys"].tolist())}
    ib = np.array([kb[tuple(k)] for k in a["keys"].tolist()], np.int64)
    sel = lambda m, ix: np.concatenate([np.arange(f, f + c) for f, c in zip(m["first"][ix], m["count"][ix])] or [np.zeros(0, np.int64)]).astype(np.int64)
    return a["planes"][sel(a, np.arange(len(a["keys"])))], b["planes"][sel(b, ib)]


# --------------------------------------------------------------------------------------------------- a. BuildVoxelMap
@pytest.mark.parametrize("scene,cfg", [("room", S.LioCfg()), ("corridor", CFG3)], ids=["room_avia_defaults", "corridor_cfg3"])
def test_device_build_at_hilti_extrinsics_matches_the_oracle(scene, cfg):
    """esikf_map_device_build on the frame test_oracle_build_voxel_map_reproduces_the_reference_source pins the oracle's
    BuildVoxelMap to the reference source on (room scene), and on the corridor scene with config 3's map settings: the same
    root voxels, every octree node (state, counters, list sizes) and every candidate plane at the build tolerance.
    Catches: the world point with extR^T or with extT outside the rotation (points land in other voxels: keys and node
    counters differ), M = extR R or M = R extR^T in the covariance, and a cross matrix other than the raw body point's
    (plane_var differs)."""
    ext = S.hilti_extrinsics()
    rects, rng, st0, (R0, p0) = first_frame(scene)
    scan0 = S.scan_at(rects, ext, R0, p0, 60000, cfg, rng)
    orc = O.OracleLIO(cfg, ext)
    orc.tick_build_map(scan0, st0)
    with contexts(1) as (ctx,):
        device_build(ctx, cfg, ext, scan0, st0)
        st, dump = ctx.map_device_stats(), orc.dump_nodes()
        assert st["errors"] == 0 and st["nodes"] == len(dump), (st, len(dump))
        flat = ctx.map_device_download()
        assert st["roots"] == len(flat["keys"]) == len(orc.flatten()["keys"])
        exp = ctx.map_device_export()  # the build touched every root: the export is the whole map
        assert len(exp["keys"]) == st["roots"]
        MB.compare_node_dumps(MM.export_dump(exp), dump, ("device BuildVoxelMap", "oracle"), a_releases_cut_lists=True)
        n = MB.compare_flat_maps(flat, orc.flatten(), rtol=1e-7, what=("device BuildVoxelMap", "oracle"))
    assert n > 1000 and (dump[:, 3] > 0).any()  # some roots were cut


# --------------------------------------------------------------------------------------------------- b. the per-point stage
def test_device_update_lists_at_hilti_extrinsics_match_the_oracle_lists():
    """One LIO update at Hilti extrinsics, then UpdateVoxelMap twice on the same built map: on context A with the lists
    map_points_kernel makes from the resident scan (world points and covariances with the oracle's posterior, passed as the
    state), on context B with the oracle's own lists (orc_lio_tick_update_map) through esikf_map_device_update_points.

    The two device maps differ only in who computed the lists. The world points agree bit for bit (the same uncontracted
    R (extR p + extT) + t, rounded to float), so the roots, every node, and every plane's centre, normal, d, radius, layer
    and path are byte-identical. plane_var is not, in about a third of the planes: it is the only field the covariances
    reach, and the covariance of the update form starts from the LIO precompute's calcBodyCov and cross vector, which
    lio_precompute_kernel evaluates with FMA contraction where the reference rounds every product. They differ from the
    oracle's by an ulp or two (test_gpu_lio allows the body covariance 1e-11). plane_var sums J var J^T over the points of
    the plane with the same J on both sides, at most max_points_num = 50 of them, so the difference stays below 50 eps
    (1e-14) of the plane's largest entry; on an H100 it is 4e-16.

    Catches: M = extR R (with this R and extR, off by far more than the tolerance), extR^T in place of extR, and the cross
    matrix taken from the raw body point instead of the IMU-frame point of the precompute."""
    cfg, ext = S.LioCfg(), S.hilti_extrinsics()
    rects, rng, st0, (R0, p0) = first_frame()
    scan0 = S.scan_at(rects, ext, R0, p0, 60000, cfg, rng)
    orc = O.OracleLIO(cfg, ext)
    orc.tick_build_map(scan0, st0)
    R1, p1 = R0 @ S.so3_exp(np.array([0.05, -0.04, 0.2])), p0 + np.array([0.3, -0.2, 0.05])
    scan1 = S.scan_at(rects, ext, R1, p1, 20000, cfg, rng)
    prior = prior_near(R1, p1, st0)
    with contexts(2) as (a, b):
        for c in (a, b):
            device_build(c, cfg, ext, scan0, st0)
        MB.compare_flat_maps(a.map_device_download(), b.map_device_download(), what=("build A", "build B"), exact=True)
        g = a.lio_update(scan1, prior, prior, cfg)
        o = orc.state_estimation(scan1, prior, prior)
        assert g["iters"] == o["iters"] and np.array_equal(g["M"], o["M"]), (g["M"], o["M"])
        assert_state_close(g["state"], o["state"], rot_tol=1e-9, pos_tol=2e-9, cov_tol=1e-7, rest_tol=1e-9)
        assert o["M"][-1] > 0.7 * len(scan1)
        a.map_device_update(state=o["state"])
        pw, var = orc.tick_update_map(want_lists=True)
        b.map_device_update_points(pw, var)
        fa, fb = a.map_device_download(), b.map_device_download()
        assert a.map_device_stats()["touched_roots"] == b.map_device_stats()["touched_roots"] > 0
        MB.compare_node_dumps(MM.export_dump(a.map_device_export()), MM.export_dump(b.map_device_export()), ("device lists", "oracle lists"))
    strip = lambda f: dict(f, planes=f["planes"].copy())
    sa, sb = strip(fa), strip(fb)
    sa["planes"]["plane_var"], sb["planes"]["plane_var"] = 0, 0
    n = MB.compare_flat_maps(sa, sb, what=("device lists", "oracle lists"), exact=True)
    pa, pb = aligned_planes(fa, fb)
    va, vb = pa["plane_var"], pb["plane_var"]
    worst = float(np.max(np.abs(va - vb) / (np.abs(vb).max(axis=1, keepdims=True) + 1e-300)))
    print(f"plane_var: device lists vs oracle lists, worst difference {worst:.3e} of the plane's largest entry over {n} planes; "
          f"{int(np.any(va != vb, axis=1).sum())} planes not bit-identical")
    assert worst < 1e-14
    for f, what in ((fa, "device lists"), (fb, "oracle lists")):
        MB.compare_flat_maps(f, orc.flatten(), rtol=1e-7, what=(what, "oracle map"))
    assert n > 1000


# --------------------------------------------------------------------------------------------------- c. the tick loop
def hilti_poses(k):
    """Yaw from 0.3 rad past 90 degrees over ten ticks, roll and pitch near 0.2 rad: R extR and extR R far apart."""
    R = S.so3_exp(np.array([0, 0, 0.3 + 0.17 * k])) @ S.so3_exp(np.array([0, -0.2 + 0.01 * k, 0])) @ S.so3_exp(np.array([0.2 - 0.005 * k, 0, 0]))
    return R, np.array([-2.0 + 0.12 * k, 0.5 - 0.05 * k, 0.3 + 0.01 * k])


def test_lio_tick_loop_at_hilti_extrinsics_tracks_the_oracle():
    """test_gpu_map's tick loop at Hilti extrinsics with config 3's map settings, yaw sweeping past 90 degrees and a
    mapSliding in the middle: every tick the iterations and effective feature counts equal, the posterior at that test's
    tolerances, pv.normal unchanged by the map update, the touched roots node by node and the whole map plane by plane
    against the oracle's StateEstimation + UpdateVoxelMap + clearMemOutOfMap.
    Catches: M = extR R (the covariances of every later tick drift from the oracle's, and the states with them), extR^T in
    the world point (points in the wrong voxels from the first tick), the cross matrix from the raw body point."""
    cfg, ext = CFG3, S.hilti_extrinsics()
    rng = np.random.default_rng(21)
    rects = S.make_scene("room", 0.5)
    orc = O.OracleLIO(cfg, ext)
    R0, p0 = hilti_poses(0)
    st0 = S.pack_state(R0, p0, cov=S.random_prior_cov(np.random.default_rng(3), scale=0.05), g=G)
    scan0 = S.scan_at(rects, ext, R0, p0, 60000, cfg, rng)
    n_pts = 20000
    with contexts(1) as (ctx,):
        device_build(ctx, cfg, ext, scan0, st0)
        orc.tick_build_map(scan0, st0)
        MB.compare_flat_maps(ctx.map_device_download(), orc.flatten(), rtol=1e-7, what=("device map after BuildVoxelMap", "oracle"))
        state_dev = state_orc = st0
        matched, slid = [], False
        for k in range(1, 11):
            Rk, pk = hilti_poses(k)
            scan = S.scan_at(rects, ext, Rk, pk, n_pts, cfg, rng)
            pr_dev, pr_orc = prior_near(Rk, pk, state_dev), prior_near(Rk, pk, state_orc)
            g = ctx.lio_update(scan, pr_dev, pr_dev, cfg)
            o = orc.state_estimation(scan, pr_orc, pr_orc)
            assert g["iters"] == o["iters"] and np.array_equal(np.asarray(g["M"])[:g["iters"]], o["M"]), (k, g["M"], o["M"])
            assert_state_close(g["state"], o["state"], rot_tol=1e-9, pos_tol=2e-9, cov_tol=1e-7, rest_tol=1e-9)
            matched.append(int(o["M"][-1]))
            nb = ctx.lio_fetch_normals()
            ctx.map_device_update()
            orc.tick_update_map()
            assert np.array_equal(nb, ctx.lio_fetch_normals()), f"tick {k}: the map update changed pv.normal"
            assert np.array_equal(np.linalg.norm(nb, axis=1) > 0, g["normal_plane"] >= 0)
            what = (f"device map, tick {k}", "oracle")
            exp = ctx.map_device_export()
            MB.compare_node_dumps(MM.export_dump(exp), MM.rows_of(orc.dump_nodes(), exp["keys"]), what, a_releases_cut_lists=True)
            MB.compare_flat_maps(ctx.map_device_download(), orc.flatten(), rtol=1e-6, what=what)
            if k == 5:  # mapSliding around the sensor's voxel (keys within +-10 voxels = 4 m stay)
                c, half = np.floor(pk / cfg.voxel_size).astype(np.int64), 10
                before = ctx.map_device_stats()["roots"]
                deleted = orc.lib.orc_lio_clear_out_of_map(orc.h, int(c[0] + half), int(c[0] - half), int(c[1] + half), int(c[1] - half), int(c[2] + half), int(c[2] - half))
                ctx.map_device_slide(c - half, c + half)
                st = ctx.map_device_stats()
                assert deleted > 0 and st["roots"] == before - deleted and st["errors"] == 0
                MB.compare_flat_maps(ctx.map_device_download(), orc.flatten(), rtol=1e-6, what=("device map after the slide", "oracle"))
                slid = True
            state_dev, state_orc = g["state"], o["state"]
        assert slid and ctx.map_device_stats()["errors"] == 0
    print(f"matched per tick: {matched}")
    assert min(matched) > 0.3 * n_pts


# --------------------------------------------------------------------------------------------------- d. a resident scan
LIO_OUT = H.LIO_KEYS + ("iters", "body_cov", "cross_mat", "normals")
PLANE_IDS = ("match_plane", "normal_plane")


def lio_outputs(ctx):
    r = ctx.lio_fetch()
    r["body_cov"], r["cross_mat"] = ctx.lio_fetch_point_cov()
    r["normals"] = ctx.lio_fetch_normals()
    return r


def same_lio_across_contexts(a, b):
    """Bit-identical LIO results of two contexts holding the same device-built map. The map's record slots are handed out
    by atomics, so two such maps number their planes differently: plane ids are compared as matched / unmatched, the planes
    themselves through the normals of normal_plane and the distances of match_plane."""
    H.bits_equal(a, b, [k for k in LIO_OUT if k not in PLANE_IDS])
    for k in PLANE_IDS:
        assert np.array_equal(a[k] >= 0, b[k] >= 0), k


def launches(ctx, fn):
    n = ctx.launch_count()
    fn()
    return ctx.launch_count() - n


def moved_lidar(ext):
    """Another lidar mounting: extR turned by a few degrees, extT moved by centimetres."""
    return dataclasses.replace(ext, extR=ext.extR @ S.so3_exp(np.array([0.03, -0.02, 0.05])), extT=ext.extT + np.array([0.02, -0.01, 0.03]))


CHANGES = {"extrinsics": (None, None), "dept_err": ("dept_err", 0.05), "beam_err": ("beam_err", 0.2)}


@pytest.mark.parametrize("change", list(CHANGES))
def test_a_resident_scan_follows_extrinsic_and_noise_model_changes(change):
    """esikf_lio_set_scan(S) + esikf_lio_run with extrinsics / noise model A, then with B on the same resident scan (B's
    extrinsics through esikf_set_lidar_extrinsics, B's dept_err / beam_err through the run's configuration): the second run
    equals a fresh context's set_scan(S) + lio_run with B bit for bit (state, stats, association, distances, the body
    covariances and cross matrices of esikf_lio_fetch_point_cov), and so does the map the following esikf_map_device_update
    makes. A changed run launches the precompute once more; an unchanged repeat launches only the update, and a repeated
    identical esikf_set_lidar_extrinsics launches nothing."""
    ext_a = S.hilti_extrinsics()
    field, value = CHANGES[change]
    cfg_a = S.LioCfg()
    ext_b = moved_lidar(ext_a) if field is None else ext_a
    cfg_b = cfg_a if field is None else dataclasses.replace(cfg_a, **{field: value})
    rects, rng, st0, (R0, p0) = first_frame()
    scan0 = S.scan_at(rects, ext_a, R0, p0, 60000, cfg_a, rng)
    R1, p1 = R0 @ S.so3_exp(np.array([0.05, -0.04, 0.2])), p0 + np.array([0.3, -0.2, 0.05])
    scan = S.scan_at(rects, ext_b, R1, p1, 20000, cfg_b, rng)
    prior = prior_near(R1, p1, st0)
    with contexts(2) as (res, fresh):
        for c in (res, fresh):
            device_build(c, cfg_a, ext_a, scan0, st0)  # the same map on both: built with A
        res.lio_set_scan(scan)
        first_run = launches(res, lambda: res.lio_run(prior, prior, cfg_a))
        first = lio_outputs(res)
        if field is None:
            res.set_lidar_extrinsics(ext_b.extR, ext_b.extT)
        changed = launches(res, lambda: res.lio_run(prior, prior, cfg_b))
        got = lio_outputs(res)
        if field is None:
            fresh.set_lidar_extrinsics(ext_b.extR, ext_b.extT)
        fresh.lio_set_scan(scan)
        fresh_run = launches(fresh, lambda: fresh.lio_run(prior, prior, cfg_b))
        want = lio_outputs(fresh)
        same_lio_across_contexts(got, want)
        # B is a different input: the comparison above would not notice a precompute that was never redone otherwise
        differs = ("cross_mat",) if field is None else ("body_cov", "state")
        assert all(not np.array_equal(first[k], want[k]) for k in differs), differs
        assert changed == fresh_run == first_run, (first_run, changed, fresh_run)
        # nothing changed: the same results and one precompute fewer
        assert launches(res, lambda: res.set_lidar_extrinsics(ext_b.extR, ext_b.extT)) == 0
        unchanged = launches(res, lambda: res.lio_run(prior, prior, cfg_b))
        assert unchanged == changed - 1, (changed, unchanged)
        same_lio_across_contexts(lio_outputs(res), want)
        for c in (res, fresh):
            c.map_device_update()
        n = MB.compare_flat_maps(res.map_device_download(), fresh.map_device_download(), what=("resident scan, map update", "fresh context"), exact=True)
    assert n > 1000


# --------------------------------------------------------------------------------------------------- e. the camera part
def vio_run(ctx, fr, w, prior):
    return ctx.vio_update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)


def vio_camera(ctx, fr):
    ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])
    ctx.vio_set_image(fr["img"])


def test_set_lidar_extrinsics_keeps_the_camera_part(small_vio_frame):
    """esikf_set_lidar_extrinsics replaces extR / extT only: repeated with the lidar part already set it launches nothing and
    the next VIO update is bit-identical to the one before; with another lidar part the VIO update equals a fresh context's
    given the old Rcl / Pcl with the new extR / extT (the VIO reads Rci = Rcl extR^T, Pci = Rcl (-extR^T extT) + Pcl)."""
    fr = small_vio_frame
    ext = fr["ext"]
    moved = dataclasses.replace(ext, extR=ext.extR @ S.so3_exp(np.array([0.004, -0.003, 0.005])), extT=ext.extT + np.array([0.01, -0.005, 0.008]))
    prior = H.vio_prior(fr)
    with contexts(2) as (ctx, fresh):
        H.vio_setup(ctx, fr)
        w = H.vio_warp(ctx, fr, prior)
        before = vio_run(ctx, fr, w, prior)
        assert launches(ctx, lambda: [ctx.set_lidar_extrinsics(ext.extR, ext.extT) for _ in range(3)]) == 0
        H.bits_equal(vio_run(ctx, fr, w, prior), before, H.VIO_KEYS)
        ctx.set_lidar_extrinsics(moved.extR, moved.extT)
        got = vio_run(ctx, fr, w, prior)
        vio_camera(fresh, fr)
        fresh.set_extrinsics(moved)
        H.bits_equal(got, vio_run(fresh, fr, w, prior), H.VIO_KEYS)
        assert not np.array_equal(got["state"], before["state"])


def test_set_lidar_extrinsics_without_a_camera_part_leaves_rcl_identity_and_pcl_zero(small_vio_frame):
    """Before any esikf_set_extrinsics, esikf_set_lidar_extrinsics sets the camera part to Rcl = I, Pcl = 0: the camera frame
    is the lidar frame. Given the lidar mounting that puts the camera where the frame's extrinsics put it (extR' = Rci^T,
    extT' = -extR' Pci), its VIO update equals bit for bit the one of a context given (extR', extT', I, 0) explicitly."""
    fr = small_vio_frame
    e = fr["ext"]
    Rci = e.Rcl @ e.extR.T
    Pci = e.Rcl @ (-e.extR.T @ e.extT) + e.Pcl
    extR, extT = Rci.T.copy(), -Rci.T @ Pci
    prior = H.vio_prior(fr)
    with contexts(2) as (ctx, explicit):
        ctx.set_lidar_extrinsics(extR, extT)
        explicit.set_extrinsics(S.Extrinsics(extR=extR, extT=extT, Rcl=np.eye(3), Pcl=np.zeros(3)))
        outs = []
        for c in (ctx, explicit):
            vio_camera(c, fr)
            c.vio_set_ref_images([fr["img_ref"]])
            outs.append(vio_run(c, fr, H.vio_warp(c, fr, prior), prior))
        H.bits_equal(outs[0], outs[1], H.VIO_KEYS)
        assert outs[0]["total_iters"] > 0


def test_set_extrinsics_changing_only_the_camera_part(small_vio_frame):
    """esikf_set_extrinsics with the lidar part unchanged takes its early return (no copy to the device), yet the next VIO
    update uses the new Rcl / Pcl: bit-identical to a fresh context's with them. A resident LIO scan is not precomputed again
    (its precompute does not depend on the camera) and gives the same results."""
    fr = small_vio_frame
    ext, cfg = fr["ext"], fr["lio_cfg"]
    cam_moved = dataclasses.replace(ext, Rcl=ext.Rcl @ S.so3_exp(np.array([-0.004, 0.003, 0.002])), Pcl=ext.Pcl + np.array([0.005, -0.01, 0.004]))
    prior = H.vio_prior(fr)
    with contexts(2) as (ctx, fresh):
        H.vio_setup(ctx, fr)
        ctx.map_upload(fr["map"], cfg.voxel_size)
        ctx.lio_set_scan(fr["pts"])
        ctx.lio_run(fr["state_prior"], fr["state_prior"], cfg)
        repeat = launches(ctx, lambda: ctx.lio_run(fr["state_prior"], fr["state_prior"], cfg))
        lio_before = lio_outputs(ctx)
        w = H.vio_warp(ctx, fr, prior)
        before = vio_run(ctx, fr, w, prior)
        ctx.set_extrinsics(cam_moved)
        got = vio_run(ctx, fr, w, prior)
        vio_camera(fresh, fr)
        fresh.set_extrinsics(cam_moved)
        H.bits_equal(got, vio_run(fresh, fr, w, prior), H.VIO_KEYS)
        assert not np.array_equal(got["state"], before["state"])
        assert launches(ctx, lambda: ctx.lio_run(fr["state_prior"], fr["state_prior"], cfg)) == repeat
        H.bits_equal(lio_outputs(ctx), lio_before, LIO_OUT)
