"""The ESIKF solve on the CPU oracle at its decision thresholds (tests/solve_cases.py) and on ill-conditioned priors:
every decision equals the reference's rule evaluated on the reported solution, zero information leaves the solution equal
to state_propagat (-) state and the covariance unchanged bit for bit, and the gain of the oracle and of an exact emulation of
the device's elimination stay within a few units of rounding of a 40-digit reference."""
import math

import numpy as np
import pytest

import solve_cases as SC

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


# ----------------------------------------------------------------------------------------------- reach
def test_reach_counts():
    """Every family reaches the decision it is there for."""
    lio = {t: [c for c in SC.LIO_CASES if t in c["tags"]] for t in {t for c in SC.LIO_CASES for t in c["tags"]}}
    vio = {t: [c for c in SC.VIO_CASES if t in c["tags"]] for t in {t for c in SC.VIO_CASES for t in c["tags"]}}
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
@pytest.mark.parametrize("case", SC.LIO_CASES, ids=[c["name"] for c in SC.LIO_CASES])
def test_lio_zero_information(case):
    r = SC.oracle_lio_zero(case)
    assert r["M"].tolist() == [0] * r["iters"]
    v0 = expected_vec0(case)
    assert np.array_equal(r["solution"][0], v0), (r["solution"][0][:6], v0[:6])
    if case["vec0_rot"] is not None:
        assert np.array_equal(r["solution"][0][0:3], case["vec0_rot"])
    SC.check_lio_rule(r, case["max_iterations"])
    assert np.array_equal(r["state"][25:], case["state_in"][25:]), "G = 0: (I - G) P must be P"
    # Exp's branch shows in the posterior rotation: the identity exactly iff no iteration took it
    took = any(SC.exp_taken(s[0:3]) for s in r["solution"])
    assert np.array_equal(r["state"][0:9], np.eye(3).reshape(9)) == (not took)


@pytest.mark.parametrize("case", SC.VIO_CASES, ids=[c["name"] for c in SC.VIO_CASES])
def test_vio_zero_information(case):
    r = SC.oracle_vio_zero(case)
    L = SC.vio_zero_info_cfg().levels
    assert np.all(r["HTH"] == 0) and np.all(r["HTz"] == 0)
    assert np.array_equal(r["solution"][L - 1][0], expected_vec0(case))
    SC.check_vio_rule(r, L)
    assert np.array_equal(r["state"][25:], case["state_in"][25:]), "G = 0: P - G P must be P"
    took = any(SC.exp_taken(r["solution"][l][it][0:3]) for l in range(L) for it in range(r["accepted_per_level"][l]))
    assert np.array_equal(r["state"][0:9], np.eye(3).reshape(9)) == (not took)


def test_vio_tie_is_accepted():
    """The error is the same in every iteration: `error <= last_error` accepts the tie (vio.cpp:1648)."""
    r = SC.oracle_vio_zero(next(c for c in SC.VIO_CASES if "tie" in c["tags"]))
    L = SC.vio_zero_info_cfg().levels
    assert r["iters_per_level"][L - 1] >= 2 and r["accepted_per_level"][L - 1] == r["iters_per_level"][L - 1]
    assert len(set(r["error_trace"][L - 1][: r["iters_per_level"][L - 1]].tolist())) == 1


# ----------------------------------------------------------------------------------------------- gain against 40 digits
GAIN_CASES = [(f, c) for f in ("small", "corridor") for c in SC.stress_covs()] + [(f, c) for f in ("vio", "vio_expo_off") for c in ("base", "corr_1m1e8", "tiny_bias_grav", "info_dominant", "propagated")]


@pytest.mark.parametrize("frame_name,cov_name", GAIN_CASES)
def test_gain_against_mpmath(frame_name, cov_name):
    """The first solution of the oracle (two pivoted 19x19 inversions) and of the emulated device elimination (unpivoted
    m x m on S^-1 + A with a correctly rounded reciprocal) against 40 digits, on the same information."""
    b = SC.gain_bound(frame_name, cov_name)
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
    r = SC.oracle_gain_run("vio", "base")[3]
    assert r["accepted_per_level"][0] < r["iters_per_level"][0]


def test_corridor_information_is_poorly_conditioned():
    """The corridor constrains one direction weakly: the smallest eigenvalue of its information is below 1e-2 of the largest."""
    fr, st, prop, r, HTH, HTz, sol0 = SC.oracle_gain_run("corridor", "base")
    ev = np.linalg.eigvalsh(0.5 * (HTH + HTH.T))
    assert ev.min() < 1e-2 * ev.max()
