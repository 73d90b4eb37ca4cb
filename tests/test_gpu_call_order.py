"""GPU: the context's call-order rules (the input groups of esikf_ctx). A call whose input is missing, or stale after a camera
change, is refused with ESIKF_ERR_STATE before it launches anything; re-setting an identical camera voids nothing the update
reads; profile_kernel(2) takes its pyramid level as an argument in [0, levels)."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import select_cases as SC
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from harness import vio_prior, vio_setup, vio_warp

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = -3, -4


@pytest.fixture
def new_context():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    made = []

    def make():
        made.append(api.Context(0))
        return made[-1]

    yield make
    for ctx in made:
        ctx.close()


def _refused(fn):
    """(status, message) of a refused call."""
    with pytest.raises(api.EsikfError) as e:
        fn()
    return int(str(e.value).split(":")[0].split()[1]), str(e.value)


def test_fresh_context_refuses_every_call_that_needs_an_earlier_input(new_context):
    """Each entry point with a state check, called with valid arguments on a fresh context: ESIKF_ERR_STATE, no launch."""
    ctx = new_context()
    lib, h = ctx.lib, ctx.h
    d = lambda n: np.zeros(n, np.float64)  # noqa: E731
    i = lambda n: np.zeros(n, np.int32)  # noqa: E731
    p = lambda a: a.ctypes.data  # noqa: E731
    st, pts, img = d(api.STATE_DOUBLES), np.ones(3, np.float32), np.zeros((48, 64), np.uint8)
    i1, i2, u1 = C.c_int32(), C.c_int32(), np.zeros(8, np.uint8)
    lio_cfg = api.lio_cfg_c(S.LioCfg())
    sel = api.VioSelectCfgC(1, 0, 0.5, 1e30)
    mask = np.ones(4, np.uint8)
    calls = {
        "map_patch": lambda: lib.esikf_map_patch(h, None, None, 0),
        "map_device_build": lambda: lib.esikf_map_device_build(h, p(st)),
        "map_device_update": lambda: lib.esikf_map_device_update(h, None),
        "map_device_update_points": lambda: lib.esikf_map_device_update_points(h, p(d(3)), p(d(9)), 1),
        "map_device_slide": lambda: lib.esikf_map_device_slide(h, None, None),
        "map_device_capacity": lambda: lib.esikf_map_device_capacity(h, C.byref(api.MapCfgC())),
        "map_device_stats": lambda: lib.esikf_map_device_stats(h, C.byref(api.MapStatsC())),
        "map_device_download": lambda: lib.esikf_map_device_download(h, None, None, None, 0, None, 0, C.byref(i1), C.byref(i2)),
        "map_device_export": lambda: lib.esikf_map_device_export(h, None, None, None, 0, None, 0, C.byref(i1), C.byref(i2)),
        "map_device_find": lambda: lib.esikf_map_device_find(h, p(d(3)), 1, api.FIND_RULE_PATCH, p(u1), p(np.zeros(3, np.int64)), p(np.zeros(32, np.float64))),
        "lio_fetch_normals": lambda: lib.esikf_lio_fetch_normals(h, p(d(3))),
        "lio_run": lambda: lib.esikf_lio_run(h, p(st), p(st), C.byref(lio_cfg)),
        "vio_set_image": lambda: lib.esikf_vio_set_image(h, p(img), 64, 48),
        "vio_set_patches": lambda: lib.esikf_vio_set_patches(h, None, None, None, None, 0),
        "vio_run": lambda: lib.esikf_vio_run(h, p(st), p(st)),
        "vio_get_image_patch": lambda: lib.esikf_vio_get_image_patch(h, p(d(2)), 1, 0, p(np.zeros(64, np.float32))),
        "vio_warp_patches": lambda: lib.esikf_vio_warp_patches(h, 0, None, None, None, None, None, None, None, None, None, 0),
        "vio_select_patches": lambda: lib.esikf_vio_select_patches(h, 0, *[None] * 12, 1.0, C.byref(sel), C.byref(i1), None, None, None, None, None),
        "vio_set_inverse_refs": lambda: lib.esikf_vio_set_inverse_refs(h, 1, p(i(1)), p(d(2)), p(d(3)), p(d(9)), p(d(3))),
        "vio_warp_affine": lambda: lib.esikf_vio_warp_affine(h, 0, None, None, None, None, None),
        "rgb_set_cloud": lambda: lib.esikf_rgb_set_cloud(h, p(pts), 1, p(st)),
        "rgb_colorize": lambda: lib.esikf_rgb_colorize(h, p(np.zeros(64 * 48 * 3, np.uint8)), 64, 48, p(st), 0.01, 0, C.byref(i1), None, None, None),
        "vio_generate_points": lambda: lib.esikf_vio_generate_points(h, p(d(3)), p(d(3)), p(d(9)), 1, None, None, 0, p(mask), 4, 16, 2, 2, 0, p(st), 4,
                                                                     C.byref(i1), *[None] * 8),
        "vio_update_points": lambda: lib.esikf_vio_update_points(h, 0, None, None, None, p(st), 0, C.byref(i1), None, None, None, None),
        "vio_retrieve_scan": lambda: lib.esikf_vio_retrieve_scan(h, p(d(3)), 1, 0, p(st), 0, C.byref(i1), None, None),
        "vio_depth_check": lambda: lib.esikf_vio_depth_check(h, 1, p(d(3)), p(d(2)), p(u1)),
        "vmap_stats": lambda: lib.esikf_vmap_stats(h, C.byref(C.c_int64()), C.byref(C.c_int64())),
        "vmap_add_points": lambda: lib.esikf_vmap_add_points(h, 0, None, 0, *[None] * 8),
        "vmap_update_points": lambda: lib.esikf_vmap_update_points(h, 0, None, None, None, 0, p(st), 0, C.byref(i1), *[None] * 6),
        "vmap_score": lambda: lib.esikf_vmap_score(h, 0, *[None] * 6),
        "vmap_choose_ref": lambda: lib.esikf_vmap_choose_ref(h, 0, None, None, None, 1, None),
        "vmap_download": lambda: lib.esikf_vmap_download(h, 0, None, 0, p(i(1)), *[None] * 7),
        "vmap_place_points": lambda: lib.esikf_vmap_place_points(h, 0, None, None, None),
        "vmap_retrieve": lambda: lib.esikf_vmap_retrieve(h, 0, None, 16, 4, 3, 0, 1, 0, C.byref(i1), *[None] * 5),
        "peer_attach": lambda: lib.esikf_peer_attach(h, 0, 1, b"\0" * 64),
    }
    calls.update({f"profile_kernel({w})": (lambda w=w: lib.esikf_profile_kernel(h, w, 0, 1, 0, C.byref(C.c_float()))) for w in range(4)})
    before = ctx.launch_count()
    got = {name: fn() for name, fn in calls.items()}
    assert got == {name: ERR_STATE for name in calls}
    assert ctx.launch_count() == before
    # the scan is missing only once one is set and not yet run
    ctx.lio_set_scan(np.zeros((4, 3), np.float32))
    assert lib.esikf_lio_fetch_point_cov(h, p(d(36)), p(d(36))) == ERR_STATE
    assert lib.esikf_rgb_set_cloud(h, None, 0, None) == ERR_STATE
    assert ctx.launch_count() == before


def _frame_setup(ctx, fr):
    """Extrinsics, camera, image and reference image of the frame, and its patches installed by set_patches."""
    vio_setup(ctx, fr)
    prior = vio_prior(fr)
    w = vio_warp(ctx, fr, prior)
    ctx.vio_set_patches(fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"])
    return prior, w


def test_a_camera_of_another_size_voids_the_image(new_context, small_vio_frame):
    fr = small_vio_frame
    ctx = new_context()
    prior, _ = _frame_setup(ctx, fr)
    cam = fr["cam_cfg"]
    bigger = dataclasses.replace(cam, width=cam.width + 64, height=cam.height + 32)
    ctx.vio_set_camera(bigger, fr["vio_cfg"])
    c = SC.candidates("radtan", 8, seed=3)
    pg = (fr["vis_pos"][:20], fr["vis_normal"][:20], np.tile(np.eye(3) * 1e-4, (20, 1, 1)))
    before = ctx.launch_count()
    calls = {
        "vio_run": lambda: ctx.vio_run(prior, prior),
        "vio_select_patches": lambda: ctx.vio_select_patches(np.zeros(8, np.int32), c["px_ref"], c["pos_w"], c["T_ref"], c["ref_inv_expo"], c["pc"], c["T_cur"],
                                                             c["inv_expo"], normal_w=c["normal_w"], normal_en=True),
        "vio_get_image_patch": lambda: ctx.vio_get_image_patch(fr["px_ref"][:4], 0),
        "vio_generate_points": lambda: ctx.vio_generate_points(np.ones(4, np.uint8), 16, 2, 2, 0, pg=pg, state=prior),
        "profile_kernel(2)": lambda: ctx.profile_kernel(2, reps=1, flush_l2=False),
    }
    for name, fn in calls.items():
        status, msg = _refused(fn)
        assert status == ERR_STATE and "image" in msg, (name, msg)
    assert ctx.launch_count() == before
    img = np.zeros((bigger.height, bigger.width), np.uint8)
    img[:cam.height, :cam.width] = fr["img"]
    ctx.vio_set_image(img)
    ctx.vio_run(prior, prior)
    assert ctx.vio_fetch()["total_iters"] > 0


def _install_set_patches(ctx, fr, prior):
    w = vio_warp(ctx, fr, prior)
    ctx.vio_set_patches(fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"])


def _install_warp_patches(ctx, fr, prior):
    st = S.unpack_state(prior)
    n = len(fr["vis_pos"])
    T_cur = api.pack_T(*S.camera_pose(fr["ext"], st["R"], st["p"]))
    T_ref = np.tile(api.pack_T(*fr["T_ref"]), (n, 1))
    ctx.vio_warp_patches(np.zeros(n, np.int32), fr["px_ref"], fr["vis_pos"], fr["vis_normal"], T_ref, T_cur, keep_on_device=True)


def _install_select_patches(ctx, fr, prior):
    st = S.unpack_state(prior)
    n = len(fr["vis_pos"])
    T_cur = api.pack_T(*S.camera_pose(fr["ext"], st["R"], st["p"]))
    T_ref = np.tile(api.pack_T(*fr["T_ref"]), (n, 1))
    Rcw, Pcw = S.camera_pose(fr["ext"], st["R"], st["p"])
    pc = S.cam_project(fr["cam_cfg"], fr["vis_pos"] @ Rcw.T + Pcw)
    got = ctx.vio_select_patches(np.zeros(n, np.int32), fr["px_ref"], fr["vis_pos"], T_ref, np.ones(n), pc, T_cur, 1.0, normal_w=fr["vis_normal"],
                                 normal_en=True, outlier_threshold=1e30)
    assert len(got["kept"]) > 0


@pytest.mark.parametrize("install", [_install_set_patches, _install_warp_patches, _install_select_patches], ids=["set_patches", "warp_patches", "select_patches"])
def test_a_camera_of_another_level_count_voids_the_sub_map(new_context, small_vio_frame, install):
    fr = small_vio_frame
    ctx = new_context()
    vio_setup(ctx, fr)
    prior = vio_prior(fr)
    install(ctx, fr, prior)
    ctx.vio_run(prior, prior)  # the installed sub-map is usable at its own level count
    L = fr["vio_cfg"].levels
    ctx.vio_set_camera(fr["cam_cfg"], dataclasses.replace(fr["vio_cfg"], levels=L + 1))
    n = ctx.n_patches
    before = ctx.launch_count()
    calls = {
        "vio_run": lambda: ctx.vio_run(prior, prior),
        "vio_update_points": lambda: ctx.vio_update_points(np.zeros(n, np.uint8), np.zeros((n, 12)), np.zeros((n, 2)), state=prior),
        "profile_kernel(2)": lambda: ctx.profile_kernel(2, reps=1, flush_l2=False),
    }
    for name, fn in calls.items():
        status, msg = _refused(fn)
        assert status == ERR_STATE and "sub-map" in msg, (name, msg)
    assert ctx.launch_count() == before


def test_an_identical_camera_voids_nothing_the_update_reads(new_context, small_vio_frame):
    fr = small_vio_frame
    ctx = new_context()
    prior, _ = _frame_setup(ctx, fr)
    ctx.vio_run(prior, prior)
    a = ctx.vio_fetch()
    ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])
    ctx.vio_run(prior, prior)
    b = ctx.vio_fetch()
    assert a["total_iters"] > 0
    for k in ("state", "errors"):
        assert a[k].tobytes() == b[k].tobytes(), k


def test_profile_kernel_level_is_an_argument(new_context, small_vio_frame):
    fr = small_vio_frame
    ctx = new_context()
    _frame_setup(ctx, fr)
    L = fr["vio_cfg"].levels
    for level in (L, -1):
        status, msg = _refused(lambda: ctx.profile_kernel(2, arg=level, reps=1, flush_l2=False))
        assert status == ERR_ARG, msg
    assert ctx.profile_kernel(2, arg=L - 1, reps=1, flush_l2=False) > 0
