"""GPU: esikf_launch_count against what every launching entry point enqueues. Each kernel launch counts one and each CUB
device-wide call counts one, however many kernels it runs (include/esikf_b200.h).

COUNTS holds, per entry point and case, the (kernels, CUB calls) its host code launches. Each row's call runs once, and
launch_count() must grow by kernels + CUB calls. Every row runs inside one torch.profiler session with CPU and CUDA
activities, each call inside a record_function range of its own. The call's launches are the cudaLaunch* runtime events
inside its range, and its kernels are the kernel records with their correlation ids: every launch must have its record,
exactly `kernels` of them must not be CUB's, and there must be at least one CUB kernel per CUB call. One session for all rows
because a session of its own per call sometimes came back without the kernel records of a short call; the runtime events
of the call were there, and launch_count() was right.

Rows whose call goes through a wrapper of fast_livo2_b200.api that calls the C ABI twice (a sizing call, then the filling
call) count both calls."""
import ctypes as C
import dataclasses
import json
import os
import tempfile

import numpy as np
import pytest

import color_cases as CC
import generate_cases as GC
import observe_cases as OC
import oracle_bind as O
import refpatch_cases as RPC
import retrieve_cases as RC
import select_cases as SC
import vmap_cases as VC
import vmap_retrieve_cases as VR
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from harness import variant, vio_prior, vio_setup, vio_warp
from map_bind import tick_points
from test_gpu_map_growth import TINY

pytestmark = pytest.mark.gpu

LIO_IT, VIO_IT, LEVELS = S.LioCfg().max_iterations, S.VioCfg().max_iterations, S.VioCfg().levels
REPS = 2  # profile_kernel: REPS timed launches after 3 warm-up launches
DEFER = dict(TINY, root_capacity=1 << 16)  # every capacity but the hash table's tiny: the first tick is deferred, the table never grows

# (kernels, CUB calls) of one call, read off the host code (esikf_api_*.cu)
COUNTS = {
    # voxel map
    "map_upload": (1, 0),                                      # plane_compact
    "map_patch": (1, 0),                                       # plane_compact
    "map_device_init": (1, 0),                                 # map_reset
    "map_device_build: growth off": (3, 1),                    # points, sort, heads, replay
    "map_device_build: growth on": (4, 1),                     # points, sort, heads, demand, replay
    "map_device_build: deferred": (11, 2),                     # the tick (5), grow: reset, survivors, copy; keys, sort, heads, demand, replay
    "map_device_update: growth off": (3, 1),
    "map_device_update: growth on": (4, 1),
    "map_device_update_points: growth off": (3, 1),            # keys, sort, heads, replay
    "map_device_update_points: deferred": (11, 2),             # keys, sort, heads, demand, replay, grow (3), keys, sort, heads, demand, replay
    "map_device_slide": (3, 0),                                # reset, survivors, copy
    "map_device_download: sizing, filling": (2, 0),            # map_download twice
    "map_device_export: sizing, filling": (3, 2),              # count, scan; count, scan, export
    "map_device_find": (1, 0),
    "lio_fetch_normals: gathered": (1, 0),                     # gather_normals
    # LIO
    "lio_run: loop 2, precompute": (2, 0),                     # precompute, the persistent kernel
    "lio_run: loop 2": (1, 0),
    "lio_run: loop 0, precompute": (1 + 2 * LIO_IT, 0),        # precompute, residual + solve per iteration
    "lio_run: loop 0": (2 * LIO_IT, 0),
    "lio_fetch_point_cov": (1, 0),                             # expand_point_cov
    "profile_kernel: 0, LIO residual": (REPS + 3, 0),
    "profile_kernel: 1, LIO solve": (REPS + 3, 0),
    "profile_kernel: 2, VIO patch": (REPS + 3, 0),
    "profile_kernel: 3, LIO precompute": (REPS + 3, 0),
    # VIO update and the patch producers
    "vio_run: loop 2, forward": (1, 0),
    "vio_run: loop 0, forward": (2 * LEVELS * VIO_IT, 0),      # patch + solve per level and iteration
    "vio_run: loop 2, inverse": (1, 0),
    "vio_run: loop 0, inverse": (LEVELS * (1 + 2 * VIO_IT), 0),  # precompute per level, patch + solve per iteration
    "vio_get_image_patch": (1, 0),
    "vio_warp_patches: answers to the host": (2, 0),           # warp_matrix, warp_affine
    "vio_warp_patches: kept on the device": (2, 0),
    "vio_warp_affine": (1, 0),
    "vio_select_patches: homography": (5, 0),                  # warp_matrix, warp_affine, gate, select_scan, scatter
    "vio_select_patches: depth form": (5, 0),                  # warp_matrix_depth, warp_affine, gate, select_scan, scatter
    # front end
    "rgb_set_cloud": (1, 0),                                   # rgb_world
    "rgb_colorize": (2, 1),                                    # rgb_color, scan, rgb_scatter
    "vio_generate_points: with patches": (5, 0),               # score, cells, select_scan, scatter, image_patch
    "vio_generate_points: without patches": (4, 0),
    "vio_update_points: with patches": (4, 0),                 # flag, select_scan, scatter, image_patch
    "vio_retrieve_scan": (4, 2),                               # ret_scan, ret_depth, sort, ret_head, scan, ret_keys
    "vio_depth_check": (1, 0),
    "vio_score_ref_patches": (1, 0),
    "vmap_add_points": (1, 0),                                 # vmap_pack
    "vmap_update_points: with patches": (6, 0),                # vmap_last, flag, select_scan, scatter, image_patch, vmap_edit
    "vmap_score: with rows": (2, 0),                           # refpatch_score, vmap_rows
    "vmap_choose_ref": (1, 0),
    "vmap_download: sizing, filling": (3, 0),                  # vmap_rows; vmap_rows, vmap_pack
    "vmap_place_points": (2, 0),                               # vpl_key, vpl_commit
    "vmap_retrieve: with survivors": (12, 0),                  # hash, init, walk x3, depth check, cells, select_scan x2, cells; choose, refs
}


def _is_cub(name):
    return "cub::" in name


class _Recorder:
    """Runs each row's call inside a record_function range named after its COUNTS key and keeps its launch_count() growth."""

    PREFIX = "launch_counts/"

    def __init__(self):
        self.launches = {}

    def __call__(self, ctx, key, fn):
        from torch.profiler import record_function

        assert key in COUNTS and key not in self.launches, key
        ctx.synchronize()
        before = ctx.launch_count()
        with record_function(self.PREFIX + key):
            out = fn()
            ctx.synchronize()
        self.launches[key] = ctx.launch_count() - before
        return out


def _kernels_per_row(events):
    """{COUNTS key: (correlation ids of the launches inside its range, {correlation id: kernel name} of the whole trace)}"""
    of = lambda cat: [e for e in events if str(e.get("cat", "")).lower() == cat]  # noqa: E731
    names = {e["args"]["correlation"]: e["name"] for e in of("kernel")}
    launches = [e for e in of("cuda_runtime") if e["name"].startswith("cudaLaunch")]
    rows = {}
    for r in of("user_annotation"):
        if r["name"].startswith(_Recorder.PREFIX):
            inside = {e["args"]["correlation"] for e in launches if r["ts"] <= e["ts"] <= r["ts"] + r["dur"]}
            rows[r["name"][len(_Recorder.PREFIX):]] = (inside, names)
    return rows


def _lio_host_map(m, ctx, fr):
    cfg, prior = fr["lio_cfg"], fr["state_prior"]
    assert cfg.max_iterations == LIO_IT
    ctx.set_extrinsics(fr["ext"])
    m(ctx, "map_upload", lambda: ctx.map_upload(fr["map"], cfg.voxel_size))
    ids = np.arange(0, 96, 3, dtype=np.int32)
    m(ctx, "map_patch", lambda: ctx.map_patch(ids, fr["map"]["planes"][ids]))
    for mode in (2, 0):
        ctx.lio_set_scan(fr["pts"])  # a new scan: the first run makes its precompute
        with variant(ctx, loop_mode=mode):
            m(ctx, f"lio_run: loop {mode}, precompute", lambda: ctx.lio_run(prior, prior, cfg))
            m(ctx, f"lio_run: loop {mode}", lambda: ctx.lio_run(prior, prior, cfg))
    m(ctx, "lio_fetch_point_cov", ctx.lio_fetch_point_cov)
    m(ctx, "lio_fetch_normals: gathered", ctx.lio_fetch_normals)
    for which, what in ((0, "LIO residual"), (1, "LIO solve"), (3, "LIO precompute")):
        m(ctx, f"profile_kernel: {which}, {what}", lambda: ctx.profile_kernel(which, reps=REPS, flush_l2=False))


def _device_map(m, ctx, fr):
    cfg, prior = fr["lio_cfg"], fr["state_prior"]
    ctx.set_extrinsics(fr["ext"])
    m(ctx, "map_device_init", lambda: ctx.map_device_init(cfg, root_capacity=1 << 16))
    ctx.lio_set_scan(fr["pts"])
    m(ctx, "map_device_build: growth off", lambda: ctx.map_device_build(prior))
    ctx.lio_run(prior, prior, cfg)
    m(ctx, "map_device_update: growth off", lambda: ctx.map_device_update())
    m(ctx, "map_device_export: sizing, filling", ctx.map_device_export)
    m(ctx, "map_device_find", lambda: ctx.map_device_find(fr["pts"][:200].astype(np.float64), api.FIND_RULE_PATCH))
    m(ctx, "map_device_download: sizing, filling", ctx.map_device_download)
    pw, var = tick_points(np.random.default_rng(5), S.make_scene("room", 0.5), 6000, np.array([-10.0, -8.0, -2.0]), np.array([-2.0, 8.0, 4.0]))
    m(ctx, "map_device_update_points: growth off", lambda: ctx.map_device_update_points(pw, var))
    m(ctx, "map_device_slide", lambda: ctx.map_device_slide())


def _growing_map(m, ctx, fr):
    cfg, prior = fr["lio_cfg"], fr["state_prior"]
    ctx.set_extrinsics(fr["ext"])
    ctx.map_device_init(cfg, root_capacity=1 << 16, grow=True)
    ctx.lio_set_scan(fr["pts"])
    m(ctx, "map_device_build: growth on", lambda: ctx.map_device_build(prior))
    ctx.lio_run(prior, prior, cfg)
    cap = ctx.map_device_capacity()
    m(ctx, "map_device_update: growth on", lambda: ctx.map_device_update())
    assert ctx.map_device_capacity() == cap  # the tick fitted: not deferred


def _deferred_ticks(m, ctxs, fr):
    a, b = ctxs
    a.set_extrinsics(fr["ext"])
    a.map_device_init(fr["lio_cfg"], **DEFER)
    a.lio_set_scan(fr["pts"])
    cap = a.map_device_capacity()
    m(a, "map_device_build: deferred", lambda: a.map_device_build(fr["state_prior"]))
    grown = a.map_device_capacity()
    assert grown["node_capacity"] > cap["node_capacity"] and grown["root_capacity"] == cap["root_capacity"]
    b.map_device_init(S.LioCfg(), **DEFER)
    pw, var = tick_points(np.random.default_rng(5), S.make_scene("room", 0.5), 6000, np.array([-10.0, -8.0, -2.0]), np.array([-2.0, 8.0, 4.0]))
    cap = b.map_device_capacity()
    m(b, "map_device_update_points: deferred", lambda: b.map_device_update_points(pw, var))
    grown = b.map_device_capacity()
    assert grown["node_capacity"] > cap["node_capacity"] and grown["root_capacity"] == cap["root_capacity"]


def _vio(m, ctx, fr):
    assert (fr["vio_cfg"].levels, fr["vio_cfg"].max_iterations) == (LEVELS, VIO_IT)
    vio_setup(ctx, fr)
    prior = vio_prior(fr)
    n = len(fr["vis_pos"])
    st = S.unpack_state(prior)
    T_cur = api.pack_T(*S.camera_pose(fr["ext"], st["R"], st["p"]))
    T_ref = np.tile(api.pack_T(*fr["T_ref"]), (n, 1))
    w = m(ctx, "vio_warp_patches: answers to the host", lambda: vio_warp(ctx, fr, prior))
    m(ctx, "vio_warp_patches: kept on the device",
      lambda: ctx.vio_warp_patches(np.zeros(n, np.int32), fr["px_ref"], fr["vis_pos"], fr["vis_normal"], T_ref, T_cur, keep_on_device=True))
    m(ctx, "vio_get_image_patch", lambda: ctx.vio_get_image_patch(fr["px_ref"][:16], 0))
    m(ctx, "vio_warp_affine", lambda: ctx.vio_warp_affine(np.zeros(n, np.int32), fr["px_ref"], w["A_cur_ref"], w["search_levels"]))
    m(ctx, "profile_kernel: 2, VIO patch", lambda: ctx.profile_kernel(2, reps=REPS, flush_l2=False))
    refs = O.inverse_refs_from_frame(fr)
    for form in ("forward", "inverse"):
        if form == "inverse":
            ctx.vio_set_camera(fr["cam_cfg"], dataclasses.replace(fr["vio_cfg"], inverse_composition_en=True))
            ctx.vio_set_inverse_refs(refs["ref_img_index"], refs["ref_px"], refs["ref_f"], refs["ref_R"], refs["ref_pos"])
        for mode in (2, 0):
            with variant(ctx, loop_mode=mode):
                m(ctx, f"vio_run: loop {mode}, {form}", lambda: ctx.vio_run(prior, prior))


def _select(m, ctx):
    c = SC.candidates("radtan", 300, seed=9)
    ctx.set_extrinsics(S.avia_extrinsics())
    ctx.vio_set_camera(c["camcfg"], S.VioCfg())
    ctx.vio_set_image(c["img"])
    ctx.vio_set_ref_images(c["ref_imgs"])
    args = (c["ref_idx"], c["px_ref"], c["pos_w"], c["T_ref"], c["ref_inv_expo"], c["pc"], c["T_cur"], c["inv_expo"])
    depth = dict(ref_level=c["ref_level"], ref_f=c["ref_f"], ref_pos=c["ref_pos"], ref_key=c["ref_key"])
    m(ctx, "vio_select_patches: homography", lambda: ctx.vio_select_patches(*args, normal_w=c["normal_w"], normal_en=True))
    m(ctx, "vio_select_patches: depth form", lambda: ctx.vio_select_patches(*args, normal_en=False, **depth))


def _color(m, ctx):
    sc = CC.scene("pinhole", 20_000, seed=4)
    ctx.set_extrinsics(sc["ext"])
    ctx.vio_set_camera(sc["cam"], S.VioCfg())
    m(ctx, "rgb_set_cloud", lambda: ctx.rgb_set_cloud(sc["pts"], sc["lio_state"]))
    got = m(ctx, "rgb_colorize", lambda: ctx.rgb_colorize(sc["img"], sc["blind"], state=sc["vio_state"]))
    assert len(got["index"]) > 0


def _generate(m, ctx):
    sc = GC.scene("pinhole", 5000, seed=2)
    ctx.set_extrinsics(sc["ext"])
    ctx.vio_set_camera(sc["cam"], S.VioCfg())
    ctx.vio_set_image(sc["img"])
    geo = [int(sc[k]) for k in ("grid_size", "grid_n_width", "grid_n_height", "border")]
    got = m(ctx, "vio_generate_points: with patches",
            lambda: ctx.vio_generate_points(sc["mask"], *geo, pg=(sc["point_w"], sc["normal"], sc["var"]), state=sc["state"]))
    assert len(got["cell"]) > 0
    d = lambda a: np.ascontiguousarray(a, np.float64)  # noqa: E731
    pw, nv, var, st, mask = d(sc["point_w"]), d(sc["normal"]), d(sc["var"]), d(sc["state"]), np.ascontiguousarray(sc["mask"], np.uint8)
    cnt = C.c_int32(0)
    rc = m(ctx, "vio_generate_points: without patches",
           lambda: ctx.lib.esikf_vio_generate_points(ctx.h, pw.ctypes.data, nv.ctypes.data, var.ctypes.data, len(pw), None, None, 0, mask.ctypes.data, len(mask),
                                                    *geo, st.ctypes.data, len(mask), C.byref(cnt), *[None] * 8))
    assert rc == 0 and cnt.value == len(got["cell"])


def _update_points(m, ctx):
    sc = OC.scene("pinhole", 2000, seed=7)
    n = len(sc["pos"])
    ctx.set_extrinsics(sc["ext"])
    ctx.vio_set_camera(sc["cam"], S.VioCfg())
    ctx.vio_set_image(sc["img"])
    ctx.vio_set_patches(np.ascontiguousarray(sc["pos"]), np.zeros((n, LEVELS * 64), np.float32), np.ascontiguousarray(sc["search_levels"]), np.ones(n))
    got = m(ctx, "vio_update_points: with patches", lambda: ctx.vio_update_points(sc["converged"], sc["last_T"], sc["last_px"], state=sc["state"]))
    assert len(got["entry"]) > 0
    c = RPC.pin_case()
    m(ctx, "vio_score_ref_patches", lambda: ctx.vio_score_ref_patches(c["first"], c["pos"], c["normal"], c["patch"], c["mean"], c["id"], c["T"]))


def _store(m, ctx):
    cam, ext, ticks = VC.sequence(ticks=12)
    ctx.vmap_init(4096)
    for tk in ticks[:-1]:
        ctx.vmap_add_points(**tk["add"])
    tk = ticks[-1]
    m(ctx, "vmap_add_points", lambda: ctx.vmap_add_points(**tk["add"]))
    sub = tk["sub"]
    n = len(sub)
    ctx.set_extrinsics(ext)
    ctx.vio_set_camera(cam, S.VioCfg())
    ctx.vio_set_image(tk["img"])
    ctx.vio_set_patches(np.ascontiguousarray(tk["pos"]), np.zeros((n, LEVELS * 64), np.float32), np.zeros(n, np.int32), np.ones(n))
    got = m(ctx, "vmap_update_points: with patches", lambda: ctx.vmap_update_points(sub, tk["converged"], tk["t"], T_f_w=tk["T_new"], state=tk["state"]))
    assert len(got["entry"]) > 0
    m(ctx, "vmap_score: with rows", lambda: ctx.vmap_score(sub, tk["pos"], np.tile([0.0, 0.0, 1.0], (n, 1))))
    m(ctx, "vmap_choose_ref", lambda: ctx.vmap_choose_ref(sub, True))
    m(ctx, "vmap_download: sizing, filling", lambda: ctx.vmap_download(sub))


def _retrieve(m, ctx):
    sc = RC.scene("pinhole", 20_000, seed=5, n_vis=2000)
    n_obs = sc["n_obs"]
    first = np.concatenate([[0], np.cumsum(n_obs)]).astype(np.int32)
    k = int(first[-1])
    T = np.zeros((k, 12))
    T[:, [0, 4, 8]] = 1.0
    ctx.vmap_init(len(n_obs))
    ctx.vmap_add_points(first, np.zeros((k, 2)), np.zeros((k, 64), np.float32), T, np.zeros(k, np.int32), np.zeros(k, np.float32), np.zeros(k, np.float32),
                        np.full(len(n_obs), -1, np.int32))
    ctx.set_extrinsics(sc["ext"])
    ctx.vio_set_camera(sc["cam"], RC.VIO_CFG)
    ids = np.arange(len(n_obs), dtype=np.int32)
    m(ctx, "vmap_place_points", lambda: ctx.vmap_place_points(ids, sc["pos"]))
    scan = m(ctx, "vio_retrieve_scan", lambda: ctx.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"]))
    m(ctx, "vio_depth_check", lambda: ctx.vio_depth_check(sc["pos"][:50], np.full((50, 2), 100.0)))
    geo = [int(sc[k]) for k in ("grid_size", "grid_n_width", "grid_n_height", "border")]
    got = m(ctx, "vmap_retrieve: with survivors", lambda: ctx.vmap_retrieve(scan["keys"], *geo, True))
    assert np.isin(got["status"], (VR.KEPT, VR.NO_REF)).any()


@pytest.fixture(scope="module")
def measured(small_frame, small_vio_frame):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from torch.profiler import ProfilerActivity, profile

    m = _Recorder()
    scenarios = [(_lio_host_map, 1, small_frame), (_device_map, 1, small_frame), (_growing_map, 1, small_frame), (_deferred_ticks, 2, small_frame),
                 (_vio, 1, small_vio_frame), (_select, 1, None), (_color, 1, None), (_generate, 1, None), (_update_points, 1, None), (_store, 1, None),
                 (_retrieve, 1, None)]
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for run, k, fr in scenarios:
            ctxs = [api.Context(0) for _ in range(k)]
            try:
                run(m, *(ctxs if k == 1 else [ctxs]), *([fr] if fr is not None else []))
            finally:
                for c in ctxs:
                    c.close()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            rows = _kernels_per_row(json.load(f)["traceEvents"])
    return {key: (n, *rows.get(key, (set(), {}))) for key, n in m.launches.items()}


def test_every_row_was_run(measured):
    assert sorted(measured) == sorted(COUNTS)


@pytest.mark.parametrize("key", list(COUNTS))
def test_launch_count_is_what_the_call_enqueues(measured, key):
    kernels, cub_calls = COUNTS[key]
    launches, launched, names = measured[key]
    assert launches == kernels + cub_calls, (key, launches)
    lost = launched - names.keys()
    assert not lost, (key, f"{len(lost)} of {len(launched)} launches have no kernel record in the trace")
    ran = [names[c] for c in sorted(launched)]
    own = [n for n in ran if not _is_cub(n)]
    cub = [n for n in ran if _is_cub(n)]
    assert len(own) == kernels, (key, own)
    assert len(cub) >= cub_calls and (cub_calls > 0 or not cub), (key, cub)
