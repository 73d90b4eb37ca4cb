"""The CUDA solve (through the C ABI) at its decision thresholds and on ill-conditioned priors, in the persistent (loop mode
2) and per-iteration (loop mode 0) forms and both gain forms (solve mode 0: push-through elimination, 1: the literal
inversions). Cases and references: tests/solve_cases.py; the same cases on the oracle: tests/test_solve_cases.py."""
import numpy as np
import pytest

import solve_cases as SC
from fast_livo2_b200 import synthetic as S
from harness import variant

pytestmark = pytest.mark.gpu

MODES = [(2, 0), (0, 0), (2, 1), (0, 1)]  # (loop mode, solve mode)


def gpu_lio_zero(ctx, case):
    ctx.set_extrinsics(S.avia_extrinsics())
    ctx.map_upload(SC.EMPTY_MAP, 0.5)
    return ctx.lio_update(SC.lio_zero_info_scan(), case["state_in"], case["state_prop"], SC.lio_cfg(case))


def gpu_vio_zero(ctx, case):
    cam, vcfg, ext = S.CamCfg(), SC.vio_zero_info_cfg(), S.avia_extrinsics()
    d = SC.vio_zero_info_inputs(cam, ext, vcfg.levels)
    ctx.set_extrinsics(ext)
    ctx.vio_set_camera(cam, vcfg)
    ctx.vio_set_image(d["img"])
    return ctx.vio_update(d["img"], d["pos"], d["warp_patch"], d["search_levels"], d["inv_expo"], case["state_in"], case["state_prop"])


def _exp_identity(R, sols):
    return np.array_equal(R, np.eye(3).reshape(9)) == (not any(SC.exp_taken(s[0:3]) for s in sols))


@pytest.mark.parametrize("loop_mode,solve_mode", MODES)
def test_lio_zero_information(gpu_ctx, loop_mode, solve_mode):
    """Every LIO threshold case: iteration count and per-iteration decisions equal the oracle's, the first solution equals
    the oracle's bit for bit, each decision is the uncontracted rule on the device's own solution, the covariance is the
    prior's bit for bit and the posterior rotation shows whether Exp was taken."""
    with variant(gpu_ctx, loop_mode=loop_mode, solve_mode=solve_mode):
        for case in SC.LIO_CASES:
            g, o = gpu_lio_zero(gpu_ctx, case), SC.oracle_lio_zero(case)
            name = case["name"]
            assert g["iters"] == o["iters"], name
            assert np.array_equal(g["converged"], o["converged"]), name
            assert np.array_equal(g["solution"][0], o["solution"][0]), (name, g["solution"][0][:6], o["solution"][0][:6])
            np.testing.assert_allclose(g["solution"], o["solution"], rtol=1e-12, atol=1e-15, err_msg=name)
            SC.check_lio_rule(g, case["max_iterations"])
            assert np.array_equal(g["state"][25:], case["state_in"][25:]), name
            assert _exp_identity(g["state"][0:9], g["solution"]), name
            assert np.array_equal(g["state"][0:9] == np.eye(3).reshape(9), o["state"][0:9] == np.eye(3).reshape(9)), name


@pytest.mark.parametrize("loop_mode,solve_mode", MODES)
def test_vio_zero_information(gpu_ctx, loop_mode, solve_mode):
    L = SC.vio_zero_info_cfg().levels
    with variant(gpu_ctx, loop_mode=loop_mode, solve_mode=solve_mode):
        for case in SC.VIO_CASES:
            g, o = gpu_vio_zero(gpu_ctx, case), SC.oracle_vio_zero(case)
            name = case["name"]
            assert np.array_equal(g["iters_per_level"][:L], o["iters_per_level"][:L]), name
            assert np.array_equal(g["accepted_per_level"][:L], o["accepted_per_level"][:L]), name
            assert np.array_equal(g["solution"][L - 1][0], o["solution"][L - 1][0]), name
            for lvl in range(L):
                n = int(o["accepted_per_level"][lvl])
                np.testing.assert_allclose(g["solution"][lvl][:n], o["solution"][lvl][:n], rtol=1e-12, atol=1e-15, err_msg=name)
            SC.check_vio_rule(g, L)
            assert np.array_equal(g["state"][25:], case["state_in"][25:]), name
            sols = [g["solution"][l][it] for l in range(L) for it in range(g["accepted_per_level"][l])]
            assert _exp_identity(g["state"][0:9], sols), name


GPU_GAIN_CASES = [("small", c) for c in SC.stress_covs()] + [("corridor", "base"), ("corridor", "tiny_bias_grav")] + \
                 [("vio", "base"), ("vio", "corr_1m1e8"), ("vio", "tiny_bias_grav"), ("vio_expo_off", "base")]


def _gpu_gain_run(ctx, frame_name, fr, st, prop):
    ctx.set_extrinsics(fr["ext"])
    if frame_name.startswith("vio"):
        ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])
        ctx.vio_set_image(fr["img"])
        wp, sl = SC.oracle_vio_warp(fr, prop)
        return ctx.vio_update(fr["img"], fr["vis_pos"], wp, sl, fr["inv_ref_expo"], st, prop)
    ctx.map_upload(fr["map"], fr["lio_cfg"].voxel_size)
    return ctx.lio_update(fr["pts"], st, prop, fr["lio_cfg"])


def _iterations(kind, r, L):
    """(A, HTz, solution) of every accepted iteration in order."""
    if kind == "lio":
        return [(r["HTH"][i], r["HTz"][i], r["solution"][i]) for i in range(r["iters"])]
    return [(r["HTH"][l][i], r["HTz"][l][i], r["solution"][l][i]) for l in range(L - 1, -1, -1) for i in range(int(r["accepted_per_level"][l]))]


def _applied_solutions(kind, r, L):
    """The solutions the posterior pose is made of: a VIO rejection restores old_state, which undoes the level's last
    accepted solution (vio.cpp:1650, 1679)."""
    if kind == "lio":
        return [r["solution"][i] for i in range(r["iters"])]
    out = []
    for l in range(L - 1, -1, -1):
        n = int(r["accepted_per_level"][l])
        keep = n - 1 if int(r["iters_per_level"][l]) > n else n
        out += [r["solution"][l][i] for i in range(keep)]
    return out


def _cov_truth(kind, P, A, img_point_cov):
    m, ps = (6, 1.0) if kind == "lio" else (7, 1.0 / img_point_cov)
    K = SC.mp_gain(P, A, ps, m)
    G = K * SC._mp(np.asarray(A)[:m, :m])
    return SC.to_np(SC.mp_cov_lio(P, G) if kind == "lio" else SC.mp_cov_vio(P, G))


@pytest.mark.parametrize("frame_name,cov_name", [("small", "base"), ("small", "propagated"), ("corridor", "base"), ("vio", "base")])
def test_gain_is_the_emulated_elimination(gpu_ctx, frame_name, cov_name):
    """The first solution of solve mode 0 is the exact emulation of gain_setup / spd_sweep / gain_rows on the device's own
    information, bit for bit. A reciprocal one unit of 2^-50 off moves it by about 1e-15 relative: inside the 40-digit
    bound, but not inside this one. The iterate starts at the prior, so state_propagat (-) state is zero on both sides."""
    kind = "vio" if frame_name.startswith("vio") else "lio"
    fr, _, prop = SC.gain_inputs(frame_name, cov_name)
    m, sign, ps = (6, 1, 1.0) if kind == "lio" else (7, -1, 1.0 / fr["vio_cfg"].img_point_cov)
    g = _gpu_gain_run(gpu_ctx, frame_name, fr, prop, prop)
    A0, z0, s0 = _iterations(kind, g, fr["vio_cfg"].levels)[0]
    emu, _ = SC.emulate_device_solution(prop[25:].reshape(19, 19), A0, z0, np.zeros(19), ps, m, sign)
    assert np.array_equal(s0, emu), (SC.rel_err(s0, emu), s0[:6], emu[:6])


@pytest.mark.parametrize("frame_name,cov_name", GPU_GAIN_CASES)
def test_gain_against_mpmath(gpu_ctx, frame_name, cov_name):
    """On the device's own information: the first solution against 40 digits within the bound fixed on the CPU
    (4 max(oracle error, emulated device error) + 1e-14); the posterior covariance against the truth built from the last
    accepted A within the same rule applied to the oracle; the posterior pose against the boxplus chain of the reported
    solutions. Both loop modes, solve mode 0."""
    kind = "vio" if frame_name.startswith("vio") else "lio"
    b = SC.gain_bound(frame_name, cov_name)
    fr, st, prop = SC.gain_inputs(frame_name, cov_name)
    P = prop[25:].reshape(19, 19)
    L = fr["vio_cfg"].levels
    icov = fr["vio_cfg"].img_point_cov
    o_its = _iterations(kind, b["run"], L)
    cov_orc = SC.rel_err(b["run"]["state"][25:].reshape(19, 19), _cov_truth(kind, P, o_its[-1][0], icov))
    for loop_mode in (2, 0):
        with variant(gpu_ctx, loop_mode=loop_mode):
            g = _gpu_gain_run(gpu_ctx, frame_name, fr, st, prop)
        its = _iterations(kind, g, L)
        assert len(its) == len(o_its)
        A0, z0, s0 = its[0]
        truth, _, _ = SC.gain_truth(kind, P, A0, z0, SC.boxminus(prop, st), icov)
        err = SC.rel_err(s0, truth)
        assert err <= b["bound"], (err, b["oracle"], b["emulation"])
        cov = SC.rel_err(g["state"][25:].reshape(19, 19), _cov_truth(kind, P, its[-1][0], icov))
        assert cov <= 4 * cov_orc + 1e-14, (cov, cov_orc)
        R, p = SC.mp_boxplus_chain(st, _applied_solutions(kind, g, L))
        assert np.abs(g["state"][0:9] - SC.to_np(R).reshape(9)).max() < 1e-14
        assert np.abs(g["state"][9:12] - SC.to_np(p).reshape(3)).max() <= 1e-15 * max(1.0, np.abs(st[9:12]).max()) * len(its)
