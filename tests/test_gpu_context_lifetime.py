"""GPU: what an ESIKF context owns is released with it. esikf_profile_kernel's error returns can be repeated without end,
and a context that went through every entry point that allocates closes cleanly, several times in one process, with the
next context still matching the oracle. Each test builds its own contexts (not the session's gpu_ctx)."""
import numpy as np
import pytest

import oracle_bind as O
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from harness import compare_lio, compare_vio, lio_gpu, lio_oracle, vio_prior, vio_setup, vio_warp
from map_bind import tick_points

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


def _vio_equals_oracle(ctx, fr):
    vio_setup(ctx, fr)
    prior = vio_prior(fr)
    w = vio_warp(ctx, fr, prior)
    args = (fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    g = ctx.vio_update(*args)
    o = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(*args)
    compare_vio(g, o, fr["vio_cfg"].levels)


def _status(excinfo):
    return int(str(excinfo.value).split(":")[0].split()[1])


def test_profile_kernel_errors_repeat_and_leave_the_context_usable(new_context, small_frame):
    """No resident frame and an unknown kernel id are refused, a thousand times in a row, and the context then still runs
    an LIO update equal to the oracle."""
    ctx = new_context()
    for which, status, msg in ((0, ERR_STATE, "no resident LIO frame"), (1, ERR_STATE, "no resident LIO frame"), (3, ERR_STATE, "no resident LIO frame"),
                               (2, ERR_STATE, "no resident VIO frame"), (7, ERR_ARG, "which=7"), (-1, ERR_ARG, "which=-1")):
        with pytest.raises(api.EsikfError, match=msg) as e:
            ctx.profile_kernel(which, reps=1)
        assert _status(e) == status
    for i in range(1000):
        with pytest.raises(api.EsikfError):
            ctx.profile_kernel(7 if i % 2 else 0, reps=1, flush_l2=False)
    compare_lio(lio_gpu(ctx, small_frame), lio_oracle(small_frame))
    # a resident LIO frame is measurable now; VIO still is not, and an unknown id is still refused
    assert ctx.profile_kernel(0, reps=2, flush_l2=False) > 0
    for which, msg in ((2, "no resident VIO frame"), (9, "which=9")):
        with pytest.raises(api.EsikfError, match=msg):
            ctx.profile_kernel(which, reps=1)


def _walk_allocating_entry_points(ctx, fr):
    """Every call that allocates device memory, events or host staging, on one context."""
    # device-resident map: init, build, update, update_points, two slides (the second frees the arena the first retired), download
    cfg = S.LioCfg()
    ext = S.avia_extrinsics()
    rng = np.random.default_rng(21)
    rects = S.make_scene("room", 0.5)
    R0, p0 = np.eye(3), np.array([-2.0, 0.5, 0.3])
    st0 = S.pack_state(R0, p0, cov=S.random_prior_cov(np.random.default_rng(3), scale=0.05), g=np.array([0, 0, -9.81]))
    ctx.set_extrinsics(ext)
    ctx.map_device_init(cfg, root_capacity=1 << 15)
    ctx.lio_set_scan(S.scan_at(rects, ext, R0, p0, 20000, cfg, rng))
    ctx.map_device_build(st0)
    scan = S.scan_at(rects, ext, R0, p0, 8000, cfg, rng)
    g = ctx.lio_update(scan, st0, st0, cfg)
    assert g["M"][-1] > 0
    bc, _ = ctx.lio_fetch_point_cov()
    assert np.isfinite(bc).all()
    ctx.lio_fetch_normals()
    ctx.map_device_update()
    ctx.lio_fetch_normals()
    pw, var = tick_points(rng, rects, 4000, np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0]))
    ctx.map_device_update_points(pw, var)
    ctx.map_device_slide(np.array([-8, -8, -4]), np.array([8, 8, 6]))
    ctx.map_device_slide()
    flat = ctx.map_device_download()
    assert len(flat["keys"]) > 0 and ctx.map_device_stats()["errors"] == 0

    # kernel timing (per-iteration launches, timing events) and phase stamps (persistent launches)
    ctx.set_kernel_timing(True)
    ctx.lio_update(scan, st0, st0, cfg)
    assert ctx.get_kernel_timing()["lio_residual_ms"][0] > 0
    ctx.set_kernel_timing(False)
    ctx.set_phase_stamps(True)
    ctx.lio_update(scan, st0, st0, cfg)
    ctx.get_phase_stamps()
    ctx.set_phase_stamps(False)
    assert ctx.profile_kernel(0, reps=2) > 0  # L2 flush buffer + measurement events

    # VIO: reference images twice, warp producers, inverse-compositional references, an update with timing
    vio_setup(ctx, fr)
    ctx.vio_set_ref_images([fr["img_ref"], fr["img"]])
    n = len(fr["vis_pos"])
    prior = vio_prior(fr)
    st = S.unpack_state(prior)
    T_cur = api.pack_T(*S.camera_pose(fr["ext"], st["R"], st["p"]))
    T_ref = np.tile(api.pack_T(*fr["T_ref"]), (n, 1))
    w = ctx.vio_warp_patches(np.zeros(n, np.int32), fr["px_ref"], fr["vis_pos"], fr["vis_normal"], T_ref, T_cur, keep_on_device=True)
    again = ctx.vio_warp_affine(np.zeros(n, np.int32), fr["px_ref"], w["A_cur_ref"], w["search_levels"])
    assert np.array_equal(again, w["warp_patch"])
    refs = O.inverse_refs_from_frame(fr)
    ctx.vio_set_inverse_refs(refs["ref_img_index"], refs["ref_px"], refs["ref_f"], refs["ref_R"], refs["ref_pos"])
    ctx.vio_get_image_patch(fr["px_ref"][:16], 1)
    ctx.vio_run(prior, prior)  # on the patches warp_patches installed
    assert ctx.vio_fetch()["total_iters"] > 0
    ctx.set_kernel_timing(True)
    ctx.vio_update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
    ctx.get_kernel_timing()
    ctx.set_kernel_timing(False)
    assert ctx.profile_kernel(2, reps=2, flush_l2=False) > 0

    # the NVLink peer mailbox (allocated by the export)
    assert len(ctx.peer_export()) == 64


def test_contexts_release_everything_they_allocate(new_context, small_vio_frame):
    """Three contexts in a row each walk every allocating entry point and close; a fourth still computes what the oracle
    does, LIO and VIO, bit for bit in association and iteration counts."""
    fr = small_vio_frame
    for _ in range(3):
        ctx = api.Context(0)
        try:
            _walk_allocating_entry_points(ctx, fr)
        finally:
            ctx.close()
    ctx = new_context()
    compare_lio(lio_gpu(ctx, fr), lio_oracle(fr))
    _vio_equals_oracle(ctx, fr)
