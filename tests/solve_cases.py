"""Inputs for the ESIKF solve (fast_livo2_b200/csrc/esikf_solve.cu) where its decisions are close calls, and high-precision
references of the reference's literal formulas.

Zero-information updates. When nothing matches (LIO: an empty map) or the image is flat (VIO: a black image with the
exposure column off, so every Jacobian row is zero), H^T H = 0 and H^T z = 0. Then K_1 H^T z = 0 and G = 0 exactly, and
the first solution is state_propagat (-) state to the last bit on every side. With the state at the identity rotation and
the origin, that difference is whatever the caller picks:
  * position: state_propagat's position itself;
  * rotation: state_propagat's rotation is a (non-orthogonal) matrix with off-diagonals +-w and a chosen diagonal. For a
    unit diagonal the trace is 3, so Log returns 0.5 K = w exactly; another diagonal sets the trace to an exact double.
So every threshold of the solve (the LIO and VIO stop rules, Exp's 1e-5, Log's trace and angle tests) can be placed one
ulp from the boundary, and the decisions are visible in the per-iteration outputs.

The thresholds are evaluated as the reference does, with every product and sum rounded (no FMA contraction): norm_rn.
norm_fma gives the two contracted forms a compiler may emit for the same expression; vectors on which they disagree with
norm_rn are the ones a contracted implementation decides differently.
"""
from __future__ import annotations

import math
from fractions import Fraction

import mpmath
import numpy as np

import oracle_bind as O
from conftest import get_frame
from fast_livo2_b200 import synthetic as S

F57 = float(np.float32(57.3))  # the float constants of vio.cpp:1675, promoted to double against the double norm
F0001 = float(np.float32(0.001))
LOG_TR = 3.0 - 1e-6  # so3_math.h:62
MP_DPS = 40


# ----------------------------------------------------------------------------------------------- arithmetic and the rules
def fma(a, b, c):
    """a b + c rounded once (Fraction is exact; int / int true division rounds to nearest even)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def norm_rn(v):
    """|v| of the reference: (v0 v0 + v1 v1) + v2 v2, every operation rounded (Python floats never contract)."""
    a, b, c = (float(x) for x in v)
    return math.sqrt((a * a + b * b) + c * c)


def norm_fma(v, order):
    """The contracted forms of the same expression: one product rounded, the other two fused."""
    a, b, c = (float(x) for x in v)
    return math.sqrt(fma(c, c, fma(b, b, a * a) if order == 0 else fma(a, a, b * b)))


def lio_converged(sol, norm=norm_rn):
    return (norm(sol[0:3]) * 57.3 < 0.01) and (norm(sol[3:6]) * 100 < 0.015)  # voxel_map.cpp:477


def vio_end(sol, norm=norm_rn):
    return (norm(sol[0:3]) * F57 < F0001) and (norm(sol[3:6]) * 100.0 < F0001)  # vio.cpp:1675


def exp_taken(v, norm=norm_rn):
    return norm(v) > 1e-5  # so3_math.h:48


def log_branches(R):
    """(trace test, angle test) of Log(R), so3_math.h:61-66: tr > 3 - 1e-6 sets theta = 0; |theta| < 0.001 takes 0.5 K."""
    tr = (R[0, 0] + R[1, 1]) + R[2, 2]
    theta = 0.0 if tr > LOG_TR else math.acos(0.5 * (tr - 1))
    return tr > LOG_TR, abs(theta) < 0.001


def fma_disagreeing(norm_target, threshold_ok, rng, want, tries=200_000):
    """Directions scaled to |v| = norm_target on which both contracted norms decide `threshold_ok` differently from norm_rn."""
    out = []
    for _ in range(tries):
        d = rng.normal(size=3)
        v = d / np.linalg.norm(d) * norm_target * (1 + rng.uniform(-4e-16, 4e-16))
        r = threshold_ok(norm_rn(v))
        if all(threshold_ok(norm_fma(v, o)) != r for o in (0, 1)):
            out.append(v)
            if len(out) == want:
                break
    return out


def ulps(x, k):
    """x and its k neighbours on each side."""
    lo, hi, out = x, x, [x]
    for _ in range(k):
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        out += [float(lo), float(hi)]
    return sorted(out)


def exact_product_point(target, scale):
    """The double x nearest target / scale with x * scale == target exactly (searched over the neighbouring doubles)."""
    x = target / scale
    for _ in range(64):
        if x * scale == target:
            return x
        x = float(np.nextafter(x, np.inf if x * scale < target else -np.inf))
    raise AssertionError("no exact point")


# ----------------------------------------------------------------------------------------------- zero-information cases
def rot_prop(w, diag=(1.0, 1.0, 1.0)):
    """A rotation-like matrix whose Log (with the trace test passed, or at the chosen trace) is built from K = 2 w."""
    a, b, c = (float(x) for x in w)
    return np.array([[diag[0], -c, b], [c, diag[1], -a], [-b, a, diag[2]]])


def zero_info_states(w=(0.0, 0.0, 0.0), p=(0.0, 0.0, 0.0), diag=(1.0, 1.0, 1.0), cov=None):
    """(state_in, state_prop): state at the identity / origin, the prior carrying the chosen difference."""
    cov = S.random_prior_cov(np.random.default_rng(7)) if cov is None else cov
    g = np.array([0.0, 0.0, -9.81])
    st = S.pack_state(np.eye(3), np.zeros(3), 1.0, v=np.array([0.1, -0.2, 0.3]), g=g, cov=cov)
    pr = S.pack_state(rot_prop(w, diag), np.asarray(p, float), 1.0, v=np.array([0.1, -0.2, 0.3]), g=g, cov=cov)
    return st, pr


def _case(name, kind, w=(0.0, 0.0, 0.0), p=(0.0, 0.0, 0.0), diag=(1.0, 1.0, 1.0), max_iterations=5, tags=()):
    st, pr = zero_info_states(w, p, diag)
    vec_rot = np.asarray(w, float) if log_branches(rot_prop(w, diag))[0] else None  # exact only where Log takes 0.5 K on a unit-trace split
    return dict(name=name, kind=kind, state_in=st, state_prop=pr, max_iterations=max_iterations, tags=tuple(tags),
                vec0_rot=vec_rot, vec0_pos=np.asarray(p, float))


def lio_zero_info_cases():
    rng = np.random.default_rng(11)
    cases = []
    # |dp| * 100 against 0.015: the double whose product is exactly 0.015 (the rule is strict), and its neighbours
    xp = exact_product_point(0.015, 100.0)
    for i, x in enumerate(ulps(xp, 2)):
        cases.append(_case(f"lio_pos_axis_{i}", "lio", p=(0.0, x, 0.0), tags=("pos_eq",) if x == xp else ("pos_ulp",)))
    for i, v in enumerate(fma_disagreeing(1.5e-4, lambda n: n * 100 < 0.015, rng, 4)):
        cases.append(_case(f"lio_pos_fma_{i}", "lio", p=v, tags=("pos_fma",)))
    # |dtheta| * 57.3 against 0.01
    xr = 0.01 / 57.3
    for i, x in enumerate(ulps(xr, 3)):
        cases.append(_case(f"lio_rot_axis_{i}", "lio", w=(x, 0.0, 0.0), tags=("rot_ulp",)))
    for i, v in enumerate(fma_disagreeing(xr, lambda n: n * 57.3 < 0.01, rng, 4)):
        cases.append(_case(f"lio_rot_fma_{i}", "lio", w=v, tags=("rot_fma",)))
    # Exp: |v| against 1e-5, exactly, by ulps, and where the contracted norm decides differently
    for i, x in enumerate(ulps(1e-5, 2)):
        cases.append(_case(f"lio_exp_axis_{i}", "lio", w=(0.0, 0.0, x), tags=("exp_ulp",)))
    for i, v in enumerate(fma_disagreeing(1e-5, lambda n: n > 1e-5, rng, 4)):
        cases.append(_case(f"lio_exp_fma_{i}", "lio", w=v, tags=("exp_fma",)))
    # Log: the trace at, one ulp either side of, 3 - 1e-6, and angles in (0.001, 0.0011)
    w = (2.0e-4, -1.5e-4, 1.0e-4)
    for i, tr in enumerate([LOG_TR, float(np.nextafter(LOG_TR, 4.0)), float(np.nextafter(LOG_TR, 0.0))]):
        cases.append(_case(f"lio_log_tr_{i}", "lio", w=w, diag=(1.0, 1.0, tr - 2.0), tags=("log_tr",)))
    for i, th in enumerate([0.0010000001, 0.00105, 0.001099]):
        tr = 1.0 + 2.0 * math.cos(th)
        cases.append(_case(f"lio_log_theta_{i}", "lio", w=w, diag=(1.0, 1.0, tr - 2.0), tags=("log_theta",)))
    # every max_iterations with a first step that converges and one that does not
    for m in range(1, 9):
        cases.append(_case(f"lio_iters_{m}_conv", "lio", p=(0.0, 0.0, 1e-5), max_iterations=m, tags=("iters",)))
        cases.append(_case(f"lio_iters_{m}_far", "lio", p=(0.0, 0.0, 1e-2), w=(1e-3, 0.0, 0.0), max_iterations=m, tags=("iters",)))
    return cases


def vio_windows():
    """Norms where the float constants of the VIO rule decide differently from their double spellings:
    rotation: (0.001f / 57.3, 0.001f / 57.3f) ends with 57.3f but not with 57.3, (0.001 / 57.3f, 0.001f / 57.3f) ends with
    0.001f but not with 0.001; position: (0.001 / 100, 0.001f / 100) the same for 0.001f."""
    mid = lambda lo, hi: 0.5 * (lo + hi)
    return dict(rot_573=mid(F0001 / 57.3, F0001 / F57), rot_0001=mid(0.001 / F57, F0001 / F57), pos_0001=mid(0.001 / 100.0, F0001 / 100.0))


def vio_zero_info_cases():
    rng = np.random.default_rng(12)
    win = vio_windows()
    cases = [_case("vio_rot_573", "vio", w=(win["rot_573"], 0.0, 0.0), tags=("vio_rot_window",)),
             _case("vio_rot_0001", "vio", w=(0.0, win["rot_0001"], 0.0), tags=("vio_rot_window",)),
             _case("vio_pos_0001", "vio", p=(0.0, 0.0, win["pos_0001"]), tags=("vio_pos_window",)),
             _case("vio_far", "vio", w=(1e-3, 0.0, 0.0), p=(1e-2, 0.0, 0.0), tags=("tie",))]
    for i, v in enumerate(fma_disagreeing(F0001 / 100.0, lambda n: n * 100.0 < F0001, rng, 3)):
        cases.append(_case(f"vio_pos_fma_{i}", "vio", p=v, tags=("vio_pos_fma",)))
    for i, x in enumerate(ulps(1e-5, 1)):
        cases.append(_case(f"vio_exp_axis_{i}", "vio", w=(x, 0.0, 0.0), tags=("exp_ulp",)))
    return cases


def lio_zero_info_scan(n=256, seed=3):
    """A small scan; the map it meets is empty, so nothing matches."""
    return np.random.default_rng(seed).uniform(-4, 4, (n, 3)).astype(np.float32)


def vio_zero_info_inputs(cam, ext, levels, n=24):
    """Black image, patches well inside it at the identity pose, warp patches of ones: every residual is -1 and every
    Jacobian row is zero, so the error is 1 in every iteration (an exact tie) and the information is zero."""
    Rcw, Pcw = S.camera_pose(ext, np.eye(3), np.zeros(3))
    g = np.stack(np.meshgrid(np.linspace(200, cam.width - 200, 6), np.linspace(180, cam.height - 180, 4)), -1).reshape(-1, 2)[:n]
    rays = np.stack([(g[:, 0] - cam.cx) / cam.fx, (g[:, 1] - cam.cy) / cam.fy, np.ones(len(g))], 1) * 4.0
    pos = (rays - Pcw) @ Rcw  # Rcw^T (pc - Pcw)
    img = np.zeros((cam.height, cam.width), np.uint8)
    return dict(img=img, pos=np.ascontiguousarray(pos), warp_patch=np.ones((len(pos), 64 * levels), np.float32),
                search_levels=np.zeros(len(pos), np.int32), inv_expo=np.ones(len(pos)))


def vio_zero_info_cfg():
    return S.VioCfg(levels=3, max_iterations=5, exposure_estimate_en=False)


def expected_lio_iters(converged_pattern, m):
    """Iteration count of the LIO loop (voxel_map.cpp:482-499) for a sequence of per-iteration convergence decisions."""
    rematch = 0
    for it in range(m):
        if converged_pattern[it] or (rematch == 0 and it == m - 2):
            rematch += 1
        if rematch >= 2 or it == m - 1:
            return it + 1
    return m


# ----------------------------------------------------------------------------------------------- covariance families
def stress_covs():
    """Prior covariances at the edges of the gain: correlations up to 1 - 1e-8, variances down to 1e-12, and scalings that
    make the information dominate (A >> S^-1) or vanish (A << S^-1)."""
    base = S.random_prior_cov(np.random.default_rng(5))
    d = np.sqrt(np.diag(base))
    corr = base / np.outer(d, d)
    C = corr.copy()
    C[0:6, 0:6] = np.eye(6)
    for i in range(3):
        C[i, 3 + i] = C[3 + i, i] = 1 - 1e-8  # rotation axis i with position axis i
    C[0:6, 6:] = C[6:, 0:6] = 0.0
    hi_corr = C * np.outer(d, d)
    tiny = base.copy()
    tiny[10:, :] *= 1e-4
    tiny[:, 10:] *= 1e-4
    tiny[np.arange(10, 19), np.arange(10, 19)] = 1e-12  # bias and gravity variances
    return dict(base=base, corr_1m1e8=hi_corr, tiny_bias_grav=tiny, info_dominant=base * 1e4, info_negligible=base * 1e-9,
                propagated=propagated_cov())


def propagated_cov(ticks=300, seed=9):
    """Covariance of an IMU-propagated trajectory (IMU_Processing.cpp:380-400 with avia.yaml noise, 200 Hz IMU, a LIO-like
    and a VIO-like position/attitude update at 10 Hz): the conditioning a real run gives the gain."""
    rng = np.random.default_rng(seed)
    dt = 0.005
    cov_gyr, cov_acc, cov_bg, cov_ba = 0.1, 0.5, 1e-4, 1e-4  # avia.yaml: gyr_cov, acc_cov, b_gyr_cov, b_acc_cov
    P = np.eye(19) * 0.01
    P[6, 6] = 1e-5
    P[10:, 10:] = np.eye(9) * 1e-5
    R = np.eye(3)
    for k in range(ticks):
        w = rng.normal(0, 0.3, 3)
        a = rng.normal(0, 1.0, 3) + np.array([0, 0, 9.81])
        F = np.eye(19)
        F[0:3, 0:3] = S.so3_exp(-w * dt)
        F[0:3, 10:13] = -np.eye(3) * dt
        F[3:6, 7:10] = np.eye(3) * dt
        F[7:10, 0:3] = -R @ S.skew(a) * dt
        F[7:10, 13:16] = -R * dt
        F[7:10, 16:19] = np.eye(3) * dt
        Q = np.zeros((19, 19))
        Q[0:3, 0:3] = np.eye(3) * cov_gyr * dt * dt
        Q[7:10, 7:10] = R @ (np.eye(3) * cov_acc) @ R.T * dt * dt
        Q[10:13, 10:13] = np.eye(3) * cov_bg * dt * dt
        Q[13:16, 13:16] = np.eye(3) * cov_ba * dt * dt
        P = F @ P @ F.T + Q
        R = R @ S.so3_exp(w * dt)
        if k % 20 == 19:  # 10 Hz: an update observing pose (LIO-like, 6 rows) then pose + exposure (VIO-like)
            for m, r in ((6, 1e-4), (7, 1e-3)):
                H = np.zeros((m, 19))
                H[:, :m] = np.eye(m)
                K = P @ H.T @ np.linalg.inv(H @ P @ H.T + r * np.eye(m))
                P = (np.eye(19) - K @ H) @ P
        P = 0.5 * (P + P.T)
    return P


# ----------------------------------------------------------------------------------------------- high-precision references
def _mp(a):
    return mpmath.matrix(np.asarray(a, float).tolist())


def mp_gain(P, A, pscale, m):
    """K_1[:, :m] of the literal formula (H^T H + (P pscale)^-1)^-1 at MP_DPS digits, from the exact double inputs."""
    with mpmath.workdps(MP_DPS):
        Pm = _mp(P) * mpmath.mpf(pscale)
        H = mpmath.zeros(19, 19)
        for i in range(m):
            for j in range(m):
                H[i, j] = mpmath.mpf(float(A[i, j]))
        K = (H + Pm ** -1) ** -1
        return K[:, 0:m]


def mp_solution(P, A, HTz, vec, pscale, m, sign):
    """solution = sign K_1 H^T z + vec - G vec[:m] (LIO sign +, VIO sign -) and G = K_1 A, as mpmath matrices."""
    with mpmath.workdps(MP_DPS):
        K = mp_gain(P, A, pscale, m)
        Am = _mp(np.asarray(A)[:m, :m])
        G = K * Am
        z = _mp(np.asarray(HTz, float).reshape(m, 1))
        v = _mp(np.asarray(vec, float).reshape(19, 1))
        sol = K * z * sign + v - G * v[0:m, 0]
        return sol, G


def mp_cov_lio(P, G):
    """(I - G) P with G padded to 19 x 19."""
    with mpmath.workdps(MP_DPS):
        Pm = _mp(P)
        Gf = mpmath.zeros(19, 19)
        for i in range(19):
            for j in range(G.cols):
                Gf[i, j] = G[i, j]
        return (mpmath.eye(19) - Gf) * Pm


def mp_cov_vio(P, G):
    """P - G P[:m, :] (vio.cpp:800 with G's zero columns dropped)."""
    with mpmath.workdps(MP_DPS):
        Pm = _mp(P)
        return Pm - G * Pm[0:G.cols, :]


def mp_exp(v):
    with mpmath.workdps(MP_DPS):
        v = [mpmath.mpf(float(x)) for x in v]
        n = mpmath.sqrt(v[0] ** 2 + v[1] ** 2 + v[2] ** 2)
        E = mpmath.eye(3)
        if n > mpmath.mpf(1e-5):
            r = [x / n for x in v]
            K = mpmath.matrix([[0, -r[2], r[1]], [r[2], 0, -r[0]], [-r[1], r[0], 0]])
            E = E + mpmath.sin(n) * K + (1 - mpmath.cos(n)) * (K * K)
        return E


def mp_boxplus_chain(state, sols):
    """R Exp(s_0) Exp(s_1) ... and p + s_0[3:6] + s_1[3:6] + ...: the state the reported solutions lead to."""
    with mpmath.workdps(MP_DPS):
        R = _mp(np.asarray(state[0:9]).reshape(3, 3))
        p = _mp(np.asarray(state[9:12]).reshape(3, 1))
        for s in sols:
            R = R * mp_exp(s[0:3])
            p = p + _mp(np.asarray(s[3:6]).reshape(3, 1))
        return R, p


def to_np(M):
    return np.array([[float(M[i, j]) for j in range(M.cols)] for i in range(M.rows)])


def rel_err(x, truth):
    x, truth = np.asarray(x, float), np.asarray(truth, float)
    return float(np.abs(x - truth).max() / max(np.abs(truth).max(), 1e-300))


# ----------------------------------------------------------------------------------------------- the device gain, emulated
def _rcp(x):
    return float(Fraction(1) / Fraction(x))


def _spd_sweep(cols, m):
    """spd_sweep<m> of esikf_solve.cu on a list of columns (one per lane): pivot reciprocal correctly rounded, the pivot
    row scaled by one rounded product, every other row updated by one fused multiply-add."""
    for k in range(m):
        piv = list(cols[k])
        r = _rcp(piv[k])
        for col in cols:
            vk = col[k] * r
            for i in range(m):
                if i != k:
                    col[i] = fma(-piv[i], vk, col[i])
            col[k] = vk
    return cols


def emulate_device_solution(P, A, HTz, vec, pscale, m, sign):
    """gain_setup / gain_rows / G / solution of solve_mode 0 in the device's operation order with exact FMA."""
    P, A = np.asarray(P, float), np.asarray(A, float)
    cols = [[float(P[l, i] * pscale) for i in range(m)] for l in range(19)] + [[1.0 if i == j else 0.0 for i in range(m)] for j in range(m)]
    cols = _spd_sweep(cols, m)
    B = [[1.0 if i == r else 0.0 for i in range(m)] if r < m else cols[r] for r in range(19)]
    Sinv = [cols[19 + j] for j in range(m)]  # row j of S^-1
    C = [[Sinv[i][c] + float(A[i, c]) for i in range(m)] for c in range(m)]  # lane c: column c of S^-1 + A
    cols = _spd_sweep(C + [list(B[r]) for r in range(19)], m)
    sol = np.zeros(19)
    G = np.zeros((19, m))
    for r in range(19):
        x = cols[m + r]
        for j in range(m):
            s = 0.0
            for k in range(m):
                s = fma(x[k], float(A[k, j]), s)
            G[r, j] = s
        s1, s2 = 0.0, 0.0
        for k in range(m):
            s1 = fma(x[k], float(HTz[k]), s1)
            s2 = fma(G[r, k], float(vec[k]), s2)
        sol[r] = ((s1 if sign > 0 else -s1) + float(vec[r])) - s2
    return sol, G


# ----------------------------------------------------------------------------------------------- the cases on the oracle
LIO_CASES = lio_zero_info_cases()
VIO_CASES = vio_zero_info_cases()
EMPTY_MAP = dict(keys=np.zeros((0, 3), np.int64), first=np.zeros(0, np.int32), count=np.zeros(0, np.int32), planes=np.zeros(0, S.PLANE_DTYPE))


def lio_cfg(case):
    return S.LioCfg(max_iterations=case["max_iterations"])


def oracle_lio_zero(case):
    lio = O.OracleLIO(lio_cfg(case), S.avia_extrinsics())
    lio.set_map(EMPTY_MAP)
    return lio.state_estimation(lio_zero_info_scan(), case["state_in"], case["state_prop"])


def oracle_vio_zero(case):
    cam, vcfg, ext = S.CamCfg(), vio_zero_info_cfg(), S.avia_extrinsics()
    d = vio_zero_info_inputs(cam, ext, vcfg.levels)
    vio = O.OracleVIO(cam, ext, vcfg)
    return vio.update(d["img"], d["pos"], d["warp_patch"], d["search_levels"], d["inv_expo"], case["state_in"], case["state_prop"])


def check_lio_rule(r, m):
    """converged[it] is the rule on solution[it], and the iteration count follows the rematch / stop rule."""
    for it in range(r["iters"]):
        assert bool(r["converged"][it]) == lio_converged(r["solution"][it]), f"iteration {it}"
    assert r["iters"] == expected_lio_iters([bool(c) for c in r["converged"]], m)


def check_vio_rule(r, levels):
    """Each level ends after its first accepted iteration whose solution meets the rule (or at max_iterations); with the
    zero-information tie every iteration is accepted."""
    for lvl in range(levels):
        n_it, n_acc = int(r["iters_per_level"][lvl]), int(r["accepted_per_level"][lvl])
        assert n_acc == n_it
        ends = [vio_end(r["solution"][lvl][it]) for it in range(n_acc)]
        assert not any(ends[:-1])
        assert ends[-1] or n_it == vio_zero_info_cfg().max_iterations


def gain_frames():
    return dict(small=dict(seed=1, n_pts=4000, n_map=150_000, scene_scale=0.5),
                corridor=dict(seed=5, n_pts=6000, n_map=400_000, lio=S.LioCfg(voxel_size=0.4, min_eigen_value=1e-4, max_points_num=100),
                              ext=S.hilti_extrinsics(), scene="corridor", scene_scale=0.25),
                vio=dict(seed=2, n_pts=2000, n_map=120_000, n_patches=150, scene_scale=0.5),
                vio_expo_off=dict(seed=8, n_pts=1000, n_map=100_000, n_patches=120, scene_scale=0.5, vio=S.VioCfg(levels=3, exposure_estimate_en=False)))


def gain_inputs(frame_name, cov_name):
    """(frame, state_in, state_prop): the frame's prior with the family's covariance, the iterate displaced from it so that
    state_propagat (-) state is not zero."""
    fr = get_frame(**gain_frames()[frame_name])
    P = stress_covs()[cov_name]
    prop = fr["state_prior"].copy()
    prop[25:] = P.reshape(-1)
    st = prop.copy()
    st[0:9] = (prop[0:9].reshape(3, 3) @ S.so3_exp(np.array([2e-4, -1e-4, 3e-4]))).reshape(9)
    st[9:12] += np.array([3e-3, -2e-3, 1e-3])
    return fr, st, prop


def oracle_vio_warp(fr, state):
    w = O.oracle_warp_patches(fr, state)
    return w["warp_patch"], w["search_levels"]


def gain_truth(kind, P, HTH, HTz, vec, img_point_cov=None):
    """(mpmath solution, mpmath G, emulated device solution) of one iteration."""
    m, sign, ps = (6, 1, 1.0) if kind == "lio" else (7, -1, 1.0 / img_point_cov)
    sol, G = mp_solution(P, HTH, HTz, vec, ps, m, sign)
    emu, _ = emulate_device_solution(P, HTH, HTz, vec, ps, m, sign)
    return to_np(sol).reshape(19), G, emu


def boxminus(prop, st):
    v = np.zeros(19)
    O.load().orc_boxminus(O.dptr(O.c64(prop)), O.dptr(O.c64(st)), O.dptr(v))
    return v


def oracle_gain_run(frame_name, cov_name):
    fr, st, prop = gain_inputs(frame_name, cov_name)
    if frame_name.startswith("vio"):
        wp, sl = oracle_vio_warp(fr, prop)
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
    e_orc, e_emu = rel_err(sol0, truth), rel_err(emu, truth)
    return dict(oracle=e_orc, emulation=e_emu, bound=4 * max(e_orc, e_emu) + 1e-14, run=r)
