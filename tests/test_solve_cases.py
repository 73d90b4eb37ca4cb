"""The ESIKF solve on the CPU oracle at its decision thresholds (tests/solve_cases.py) and on ill-conditioned priors:
every decision equals the reference's rule evaluated on the reported solution, zero information leaves the solution equal
to state_propagat (-) state and the covariance unchanged bit for bit, and the gain of the oracle and of an exact emulation of
the device's elimination stay within a few units of rounding of a 40-digit reference."""
import math

import numpy as np
import pytest

import oracle_bind as O
import solve_cases as SC
from conftest import get_frame
from fast_livo2_b200 import synthetic as S

LIO_CASES = SC.lio_zero_info_cases()
VIO_CASES = SC.vio_zero_info_cases()
EMPTY_MAP = dict(keys=np.zeros((0, 3), np.int64), first=np.zeros(0, np.int32), count=np.zeros(0, np.int32), planes=np.zeros(0, S.PLANE_DTYPE))


def lio_cfg(case):
    return S.LioCfg(max_iterations=case["max_iterations"])


def oracle_lio_zero(case):
    lio = O.OracleLIO(lio_cfg(case), S.avia_extrinsics())
    lio.set_map(EMPTY_MAP)
    return lio.state_estimation(SC.lio_zero_info_scan(), case["state_in"], case["state_prop"])


def oracle_vio_zero(case):
    cam, vcfg, ext = S.CamCfg(), SC.vio_zero_info_cfg(), S.avia_extrinsics()
    d = SC.vio_zero_info_inputs(cam, ext, vcfg.levels)
    vio = O.OracleVIO(cam, ext, vcfg)
    return vio.update(d["img"], d["pos"], d["warp_patch"], d["search_levels"], d["inv_expo"], case["state_in"], case["state_prop"])


def expected_vec0(case):
    """state_propagat (-) state of a zero-information case as the reference computes it (Log of the chosen matrix)."""
    Rp = case["state_prop"][0:9].reshape(3, 3)
    tr = (Rp[0, 0] + Rp[1, 1]) + Rp[2, 2]
    theta = 0.0 if tr > SC.LOG_TR else math.acos(0.5 * (tr - 1))
    K = np.array([Rp[2, 1] - Rp[1, 2], Rp[0, 2] - Rp[2, 0], Rp[1, 0] - Rp[0, 1]])
    f = 0.5 if abs(theta) < 0.001 else 0.5 * theta / math.sin(theta)
    v = np.zeros(19)
    v[0:3] = f * K
    v[3:6] = case["state_prop"][9:12]
    return v


def check_lio_rule(r, m):
    """converged[it] is the rule on solution[it], and the iteration count follows the rematch / stop rule."""
    for it in range(r["iters"]):
        assert bool(r["converged"][it]) == SC.lio_converged(r["solution"][it]), f"iteration {it}"
    assert r["iters"] == SC.expected_lio_iters([bool(c) for c in r["converged"]], m)


def check_vio_rule(r, levels):
    """Each level ends after its first accepted iteration whose solution meets the rule (or at max_iterations); with the
    zero-information tie every iteration is accepted."""
    for lvl in range(levels):
        n_it, n_acc = int(r["iters_per_level"][lvl]), int(r["accepted_per_level"][lvl])
        assert n_acc == n_it
        ends = [SC.vio_end(r["solution"][lvl][it]) for it in range(n_acc)]
        assert not any(ends[:-1])
        assert ends[-1] or n_it == SC.vio_zero_info_cfg().max_iterations


# ----------------------------------------------------------------------------------------------- reach
def test_reach_counts():
    """Every family reaches the decision it is there for."""
    lio = {t: [c for c in LIO_CASES if t in c["tags"]] for t in {t for c in LIO_CASES for t in c["tags"]}}
    vio = {t: [c for c in VIO_CASES if t in c["tags"]] for t in {t for c in VIO_CASES for t in c["tags"]}}
    pos = lambda c: c["state_prop"][9:12]
    rot = lambda c: c["vec0_rot"]
    reach = dict(
        pos_equal=sum(SC.norm_rn(pos(c)) * 100 == 0.015 for c in lio["pos_eq"]),
        pos_below=sum(SC.norm_rn(pos(c)) * 100 < 0.015 for c in lio["pos_ulp"]),
        pos_above=sum(SC.norm_rn(pos(c)) * 100 > 0.015 for c in lio["pos_ulp"]),
        pos_below_001=sum(0.01 < SC.norm_rn(pos(c)) * 100 < 0.015 for c in lio["pos_ulp"]),
        pos_fma=len(lio["pos_fma"]),
        rot_both_sides=len({SC.norm_rn(rot(c)) * 57.3 < 0.01 for c in lio["rot_ulp"]}) - 1,
        rot_fma=len(lio["rot_fma"]),
        exp_both_sides=len({SC.exp_taken(rot(c)) for c in lio["exp_ulp"]}) - 1,
        exp_at_1e5=sum(SC.norm_rn(rot(c)) == 1e-5 for c in lio["exp_ulp"]),
        exp_fma=len(lio["exp_fma"]),
        log_tr_equal=sum(SC.log_branches(c["state_prop"][0:9].reshape(3, 3)) == (False, False) and
                         (c["state_prop"][0] + c["state_prop"][4]) + c["state_prop"][8] == SC.LOG_TR for c in lio["log_tr"]),
        log_tr_above=sum(SC.log_branches(c["state_prop"][0:9].reshape(3, 3))[0] for c in lio["log_tr"]),
        log_theta_window=sum(0.001 < math.acos(0.5 * (((c["state_prop"][0] + c["state_prop"][4]) + c["state_prop"][8]) - 1)) < 0.0011 for c in lio["log_theta"]),
        iters_rematch_at_m_minus_2=sum(c["max_iterations"] >= 2 for c in lio["iters"] if c["name"].endswith("far")),
        vio_rot_573=sum((SC.norm_rn(rot(c)) * SC.F57 < SC.F0001) and not (SC.norm_rn(rot(c)) * 57.3 < SC.F0001) for c in vio["vio_rot_window"]),
        vio_rot_0001=sum((SC.norm_rn(rot(c)) * SC.F57 < SC.F0001) and not (SC.norm_rn(rot(c)) * SC.F57 < 0.001) for c in vio["vio_rot_window"]),
        vio_pos_0001=sum((SC.norm_rn(pos(c)) * 100.0 < SC.F0001) and not (SC.norm_rn(pos(c)) * 100.0 < 0.001) for c in vio["vio_pos_window"]),
        vio_pos_fma=len(vio["vio_pos_fma"]),
        vio_tie=len(vio["tie"]),
    )
    assert all(v > 0 for v in reach.values()), {k: v for k, v in reach.items() if v <= 0}


# ----------------------------------------------------------------------------------------------- zero information
@pytest.mark.parametrize("case", LIO_CASES, ids=[c["name"] for c in LIO_CASES])
def test_lio_zero_information(case):
    r = oracle_lio_zero(case)
    assert r["M"].tolist() == [0] * r["iters"]
    v0 = expected_vec0(case)
    assert np.array_equal(r["solution"][0], v0), (r["solution"][0][:6], v0[:6])
    if case["vec0_rot"] is not None:
        assert np.array_equal(r["solution"][0][0:3], case["vec0_rot"])
    check_lio_rule(r, case["max_iterations"])
    assert np.array_equal(r["state"][25:], case["state_in"][25:]), "G = 0: (I - G) P must be P"
    # Exp's branch shows in the posterior rotation: the identity exactly iff no iteration took it
    took = any(SC.exp_taken(s[0:3]) for s in r["solution"])
    assert np.array_equal(r["state"][0:9], np.eye(3).reshape(9)) == (not took)


@pytest.mark.parametrize("case", VIO_CASES, ids=[c["name"] for c in VIO_CASES])
def test_vio_zero_information(case):
    r = oracle_vio_zero(case)
    L = SC.vio_zero_info_cfg().levels
    assert np.all(r["HTH"] == 0) and np.all(r["HTz"] == 0)
    assert np.array_equal(r["solution"][L - 1][0], expected_vec0(case))
    check_vio_rule(r, L)
    assert np.array_equal(r["state"][25:], case["state_in"][25:]), "G = 0: P - G P must be P"
    took = any(SC.exp_taken(r["solution"][l][it][0:3]) for l in range(L) for it in range(r["accepted_per_level"][l]))
    assert np.array_equal(r["state"][0:9], np.eye(3).reshape(9)) == (not took)


def test_vio_tie_is_accepted():
    """The error is the same in every iteration: `error <= last_error` accepts the tie (vio.cpp:1648)."""
    r = oracle_vio_zero(next(c for c in VIO_CASES if "tie" in c["tags"]))
    L = SC.vio_zero_info_cfg().levels
    assert r["iters_per_level"][L - 1] >= 2 and r["accepted_per_level"][L - 1] == r["iters_per_level"][L - 1]
    assert len(set(r["error_trace"][L - 1][: r["iters_per_level"][L - 1]].tolist())) == 1


# ----------------------------------------------------------------------------------------------- gain against 40 digits
def gain_frames():
    return dict(small=dict(seed=1, n_pts=4000, n_map=150_000, scene_scale=0.5),
                corridor=dict(seed=5, n_pts=6000, n_map=400_000, lio=S.LioCfg(voxel_size=0.4, min_eigen_value=1e-4, max_points_num=100),
                              ext=S.hilti_extrinsics(), scene="corridor", scene_scale=0.25),
                vio=dict(seed=2, n_pts=2000, n_map=120_000, n_patches=150, scene_scale=0.5),
                vio_expo_off=dict(seed=8, n_pts=1000, n_map=100_000, n_patches=120, scene_scale=0.5, vio=S.VioCfg(levels=3, exposure_estimate_en=False)))


GAIN_CASES = [(f, c) for f in ("small", "corridor") for c in SC.stress_covs()] + [(f, c) for f in ("vio", "vio_expo_off") for c in ("base", "corr_1m1e8", "tiny_bias_grav", "info_dominant", "propagated")]


def gain_inputs(frame_name, cov_name):
    """(frame, state_in, state_prop): the frame's prior with the family's covariance, the iterate displaced from it so that
    state_propagat (-) state is not zero."""
    fr = get_frame(**gain_frames()[frame_name])
    P = SC.stress_covs()[cov_name]
    prop = fr["state_prior"].copy()
    prop[25:] = P.reshape(-1)
    st = prop.copy()
    st[0:9] = (prop[0:9].reshape(3, 3) @ S.so3_exp(np.array([2e-4, -1e-4, 3e-4]))).reshape(9)
    st[9:12] += np.array([3e-3, -2e-3, 1e-3])
    return fr, st, prop


def vio_warp(fr, state):
    w = O.oracle_warp_patches(fr, state)
    return w["warp_patch"], w["search_levels"]


def gain_truth(kind, P, HTH, HTz, vec, img_point_cov=None):
    """(mpmath solution, mpmath G, emulated device solution) of one iteration."""
    m, sign, ps = (6, 1, 1.0) if kind == "lio" else (7, -1, 1.0 / img_point_cov)
    sol, G = SC.mp_solution(P, HTH, HTz, vec, ps, m, sign)
    emu, _ = SC.emulate_device_solution(P, HTH, HTz, vec, ps, m, sign)
    return SC.to_np(sol).reshape(19), G, emu


def boxminus(prop, st):
    v = np.zeros(19)
    O.load().orc_boxminus(O.dptr(O.c64(prop)), O.dptr(O.c64(st)), O.dptr(v))
    return v


def oracle_gain_run(frame_name, cov_name):
    fr, st, prop = gain_inputs(frame_name, cov_name)
    if frame_name.startswith("vio"):
        wp, sl = vio_warp(fr, prop)
        vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
        r = vio.update(fr["img"], fr["vis_pos"], wp, sl, fr["inv_ref_expo"], st, prop)
        L = fr["vio_cfg"].levels
        return fr, st, prop, r, r["HTH"][L - 1][0], r["HTz"][L - 1][0], r["solution"][L - 1][0]
    lio = O.OracleLIO(fr["lio_cfg"], fr["ext"])
    lio.set_map(fr["map"])
    r = lio.state_estimation(fr["pts"], st, prop)
    return fr, st, prop, r, r["HTH"][0], r["HTz"][0], r["solution"][0]


def gain_bound(frame_name, cov_name):
    """The device bound of a gain case, fixed on the CPU: 4 max(oracle error, emulated device error) + 1e-14, relative to the
    40-digit solution of the first iteration."""
    fr, st, prop, r, HTH, HTz, sol0 = oracle_gain_run(frame_name, cov_name)
    kind = "vio" if frame_name.startswith("vio") else "lio"
    truth, _, emu = gain_truth(kind, prop[25:].reshape(19, 19), HTH, HTz, boxminus(prop, st), fr["vio_cfg"].img_point_cov)
    e_orc, e_emu = SC.rel_err(sol0, truth), SC.rel_err(emu, truth)
    return dict(oracle=e_orc, emulation=e_emu, bound=4 * max(e_orc, e_emu) + 1e-14, run=r)


@pytest.mark.parametrize("frame_name,cov_name", GAIN_CASES)
def test_gain_against_mpmath(frame_name, cov_name):
    """The first solution of the oracle (two pivoted 19x19 inversions) and of the emulated device elimination (unpivoted
    m x m on S^-1 + A with a correctly rounded reciprocal) against 40 digits, on the same information."""
    b = gain_bound(frame_name, cov_name)
    r = b["run"]
    if frame_name.startswith("vio"):
        assert r["accepted_per_level"].sum() > 0
        if frame_name == "vio_expo_off":
            assert np.all(r["HTH"][2][0][6, :] == 0)  # rank-deficient information: the exposure column is zero
    else:
        assert r["M"][0] > 100
    # measured: at most 3e-12 (oracle) and 5e-12 (emulation), on the 1 - 1e-8 correlation; about 1e-15 elsewhere
    assert b["oracle"] < 1e-10 and b["emulation"] < 1e-10, b


def test_vio_rejection_at_the_last_level_is_reached():
    """The small VIO frame rejects an iteration at level 0, so its final cov -= G cov uses the G an earlier accepted
    iteration stored (vio.cpp:800); tests/test_gpu_solve.py checks that covariance against 40 digits."""
    r = oracle_gain_run("vio", "base")[3]
    assert r["accepted_per_level"][0] < r["iters_per_level"][0]


def test_corridor_information_is_poorly_conditioned():
    """The corridor constrains one direction weakly: the smallest eigenvalue of its information is below 1e-2 of the largest."""
    fr, st, prop, r, HTH, HTz, sol0 = oracle_gain_run("corridor", "base")
    ev = np.linalg.eigvalsh(0.5 * (HTH + HTH.T))
    assert ev.min() < 1e-2 * ev.max()
