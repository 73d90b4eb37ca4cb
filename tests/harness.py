"""What the GPU tests share: launch variants of a context (loop mode, solve mode, tuning flags) that are always put back,
sweeps over them, bit-identity of two results, and the LIO / VIO runs on a synthetic frame with their oracle comparisons.

Collection on a machine without a GPU imports this module, so nothing here imports torch or touches a device at import time."""
import contextlib

import numpy as np

import oracle_bind as O
from fast_livo2_b200 import api

LIO_KEYS = ("state", "match_plane", "normal_plane", "dis_to_plane", "M", "HTH", "HTz", "solution", "total_residual", "converged")
VIO_KEYS = ("state", "errors", "iters_per_level", "accepted_per_level", "error_trace", "HTH", "HTz", "solution")


# ----------------------------------------------------------------------------------------------------- launch variants
@contextlib.contextmanager
def variant(ctx, loop_mode=api.DEFAULT_LOOP_MODE, solve_mode=0, tuning=0):
    """Run the body with these modes; the defaults are back afterwards, also when the body raises (the session's context is
    shared by every later test)."""
    try:
        ctx.set_loop_mode(loop_mode)
        ctx.set_solve_mode(solve_mode)
        ctx.set_tuning(tuning)
        yield ctx
    finally:
        ctx.set_loop_mode(api.DEFAULT_LOOP_MODE)
        ctx.set_solve_mode(0)
        ctx.set_tuning(0)


def sweep(ctx, run, variants):
    """run() once under each variant (a dict of variant()'s keywords), in the order given: the results in that order."""
    out = []
    for v in variants:
        with variant(ctx, **v):
            out.append(run())
    return out


def bits_equal(a, b, keys):
    for k in keys:
        x, y = np.ascontiguousarray(a[k]), np.ascontiguousarray(b[k])
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), k


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------------------------------- LIO
def lio_gpu(ctx, fr, cfg=None, state_in=None):
    cfg = cfg or fr["lio_cfg"]
    ctx.set_extrinsics(fr["ext"])
    ctx.map_upload(fr["map"], cfg.voxel_size)
    s = fr["state_prior"] if state_in is None else state_in
    return ctx.lio_update(fr["pts"], s, fr["state_prior"], cfg)


def lio_oracle(fr, cfg=None, state_in=None):
    cfg = cfg or fr["lio_cfg"]
    lio = O.OracleLIO(cfg, fr["ext"])
    lio.set_map(fr["map"])
    s = fr["state_prior"] if state_in is None else state_in
    return lio.state_estimation(fr["pts"], s, fr["state_prior"])


def compare_lio(g, o, same_plane_ids=True, **state_tol):
    """Iterations, association, counts, distances and per-iteration decisions bit for bit, the information to INFO_RTOL and
    the posterior within assert_state_close(**state_tol). Plane ids are compared as they are, or with same_plane_ids=False
    only as matched / unmatched: on a device-built map they are record slots, in the oracle flat ids."""
    from parity_util import INFO_RTOL, assert_state_close, rel

    assert g["iters"] == o["iters"]
    for k in ("match_plane", "normal_plane"):
        assert np.array_equal(g[k], o[k]) if same_plane_ids else np.array_equal(g[k] >= 0, o[k] >= 0), k
    assert np.array_equal(g["M"], o["M"]), (g["M"], o["M"])
    assert np.array_equal(g["converged"], o["converged"])
    assert np.array_equal(g["dis_to_plane"], o["dis_to_plane"])  # float, same op order
    for it in range(o["iters"]):
        assert rel(g["HTH"][it], o["HTH"][it]) < INFO_RTOL
        assert rel(g["HTz"][it], o["HTz"][it]) < 1e-8
        assert abs(g["total_residual"][it] - o["total_residual"][it]) < 1e-9 * max(1.0, o["total_residual"][it])
    assert_state_close(g["state"], o["state"], **state_tol)


# ----------------------------------------------------------------------------------------------------- VIO
def vio_prior(fr, seed=3, rot_deg=0.15, pos=0.01, cov_scale=0.2):
    from fast_livo2_b200 import synthetic as S

    rng = np.random.default_rng(seed)
    t = S.unpack_state(fr["state_true"])
    cov = S.random_prior_cov(rng, scale=cov_scale)
    return S.pack_state(t["R"] @ S.so3_exp(rng.normal(0, np.deg2rad(rot_deg), 3)), t["p"] + rng.normal(0, pos, 3), 1.0 + rng.normal(0, 0.01), t["v"],
                        g=t["g"], cov=cov)


def vio_setup(ctx, fr):
    ctx.set_extrinsics(fr["ext"])
    ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])
    ctx.vio_set_image(fr["img"])
    ctx.vio_set_ref_images([fr["img_ref"]])


def vio_warp(ctx, fr, state):
    from fast_livo2_b200 import synthetic as S

    st = S.unpack_state(state)
    T_cur = api.pack_T(*S.camera_pose(fr["ext"], st["R"], st["p"]))
    n = len(fr["vis_pos"])
    T_ref = np.tile(api.pack_T(*fr["T_ref"]), (n, 1))
    return ctx.vio_warp_patches(np.zeros(n, np.int32), fr["px_ref"], fr["vis_pos"], fr["vis_normal"], T_ref, T_cur)


def compare_vio(g, o, L):
    from parity_util import assert_state_close, rel

    assert g["total_iters"] == o["total_iters"]
    assert np.array_equal(g["iters_per_level"], o["iters_per_level"])
    assert np.array_equal(g["accepted_per_level"], o["accepted_per_level"])
    for lvl in range(L):
        for it in range(o["iters_per_level"][lvl]):
            # error: a sequential FLOAT accumulation over n_meas terms in the reference (rounding error ~ sqrt(n) * 6e-8, and an
            # unspecified OpenMP order); an fp64 fixed-order sum here -> compare at 1e-5 relative
            assert abs(g["error_trace"][lvl][it] - o["error_trace"][lvl][it]) <= 1e-5 * o["error_trace"][lvl][it]
        for it in range(o["accepted_per_level"][lvl]):
            assert rel(g["HTH"][lvl][it], o["HTH"][lvl][it]) < 1e-9
            assert rel(g["HTz"][lvl][it], o["HTz"][lvl][it]) < 1e-7
    np.testing.assert_allclose(g["errors"], o["errors"], rtol=2e-6, atol=1e-3)
    assert_state_close(g["state"], o["state"], rot_tol=1e-8, pos_tol=1e-8, cov_tol=1e-6, rest_tol=1e-8)
