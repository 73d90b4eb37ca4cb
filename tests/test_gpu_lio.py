"""GPU parity: the CUDA LIO update (through the C ABI) against the CPU oracle on the same seeded inputs."""
import numpy as np
import pytest

import oracle_bind as O
from conftest import get_frame
from fast_livo2_b200 import synthetic as S
from harness import compare_lio, lio_gpu, lio_oracle, sweep, variant
from parity_util import assert_state_close, rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed,n_pts", [(1, 4000), (3, 5000), (4, 20000)])
def test_lio_matches_oracle(gpu_ctx, seed, n_pts):
    fr = get_frame(seed=seed, n_pts=n_pts, n_map=150_000, scene_scale=0.5)
    compare_lio(lio_gpu(gpu_ctx, fr), lio_oracle(fr))


def test_lio_literal_solve_mode_matches_oracle_and_woodbury(gpu_ctx, small_frame):
    fr = small_frame
    o = lio_oracle(fr)
    with variant(gpu_ctx, solve_mode=1):
        g1 = lio_gpu(gpu_ctx, fr)
    g0 = lio_gpu(gpu_ctx, fr)
    compare_lio(g1, o)
    assert_state_close(g0["state"], g1["state"], cov_tol=1e-7)


def test_config1_three_iterations(gpu_ctx):
    """BASELINE config 1: 5k points, LIO only, max_iterations = 3."""
    fr = get_frame(seed=0, n_pts=5000, n_map=150_000, scene_scale=0.5)
    cfg = S.LioCfg(**{**fr["lio_cfg"].__dict__, "max_iterations": 3})
    g, o = lio_gpu(gpu_ctx, fr, cfg), lio_oracle(fr, cfg)
    assert g["iters"] == 3
    compare_lio(g, o)


def test_early_stop_on_double_convergence(gpu_ctx, small_frame):
    fr = small_frame
    o = lio_oracle(fr)
    st = o["state"].copy()
    st[25:] = (np.eye(19) * 1e-12).reshape(-1)
    fr2 = dict(fr, state_prior=st)
    g, o2 = lio_gpu(gpu_ctx, fr2), lio_oracle(fr2)
    assert o2["iters"] == 2 and g["iters"] == 2
    compare_lio(g, o2)


def test_hilti_like_config_non_identity_extrinsics_and_voxel_04(gpu_ctx):
    """config 3 flavour: voxel 0.4 (not exactly representable: float vs double voxel size differ), non-identity extR,
    degenerate corridor scene."""
    cfg = S.LioCfg(voxel_size=0.4, min_eigen_value=1e-4, max_points_num=100)
    fr = get_frame(seed=5, n_pts=6000, n_map=400_000, lio=cfg, ext=S.hilti_extrinsics(), scene="corridor", scene_scale=0.25)
    g, o = lio_gpu(gpu_ctx, fr), lio_oracle(fr)
    assert o["M"][0] > 1000
    compare_lio(g, o)


def test_edge_cases(gpu_ctx, small_frame):
    fr = small_frame
    cfg = fr["lio_cfg"]
    # (a) zero-z and exactly-on-voxel-boundary / negative-coordinate points mixed into the scan
    pts = fr["pts"].copy()
    pts[:50, 2] = 0.0
    pts[50:60] = 0.0
    pts[50:60, 0] = np.arange(10) * 0.5 + 1.0
    fr_a = dict(fr, pts=pts)
    compare_lio(lio_gpu(gpu_ctx, fr_a), lio_oracle(fr_a))
    # (b) every point far outside the map: nothing matches, M = 0, the update falls back to the prior
    far = fr["pts"] + np.float32(500.0)
    fr_b = dict(fr, pts=far)
    g, o = lio_gpu(gpu_ctx, fr_b), lio_oracle(fr_b)
    assert g["M"].tolist() == [0] * g["iters"] and np.all(g["match_plane"] == -1)
    compare_lio(g, o)
    # (c) a single point, and an empty scan
    fr_c = dict(fr, pts=fr["pts"][:1])
    compare_lio(lio_gpu(gpu_ctx, fr_c), lio_oracle(fr_c))
    g = lio_gpu(gpu_ctx, dict(fr, pts=np.zeros((0, 3), np.float32)))
    assert g["iters"] == cfg.max_iterations or g["iters"] >= 2
    # (d) empty map
    empty = dict(keys=np.zeros((0, 3), np.int64), first=np.zeros(0, np.int32), count=np.zeros(0, np.int32), planes=np.zeros(0, S.PLANE_DTYPE))
    fr_d = dict(fr, map=empty)
    g, o = lio_gpu(gpu_ctx, fr_d), lio_oracle(fr_d)
    assert np.all(g["match_plane"] == -1)
    compare_lio(g, o)


def test_argument_errors(gpu_ctx, small_frame):
    from fast_livo2_b200 import api

    fr = small_frame
    bad = dict(fr["map"], keys=fr["map"]["keys"].copy())
    bad["keys"][0, 0] = 1 << 40
    with pytest.raises(api.EsikfError):
        gpu_ctx.map_upload(bad, 0.5)
    cfg = S.LioCfg(**{**fr["lio_cfg"].__dict__, "max_iterations": 9})
    gpu_ctx.map_upload(fr["map"], 0.5)
    with pytest.raises(api.EsikfError):
        gpu_ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], cfg)


def test_point_cov_outputs_match_oracle_lists(gpu_ctx, small_frame):
    """body_cov_list_ / cross_mat_list_ consumed by LIVMapper.cpp:418-419."""
    import ctypes as C

    fr = small_frame
    lio_gpu(gpu_ctx, fr)
    bc, cm = gpu_ctx.lio_fetch_point_cov()
    lib = O.load()
    for i in range(0, 400, 7):
        p = fr["pts"][i].astype(np.float64)
        cov = np.zeros(9)
        lib.orc_calc_body_cov(O.dptr(p), C.c_float(fr["lio_cfg"].dept_err), C.c_float(fr["lio_cfg"].beam_err), O.dptr(cov), None)
        np.testing.assert_allclose(bc[i], cov.reshape(3, 3), rtol=1e-11, atol=1e-18)
        np.testing.assert_allclose(cm[i], S.skew(fr["ext"].extR @ p + fr["ext"].extT), rtol=1e-14)


def test_full_size_properties(gpu_ctx):
    """BASELINE config 2 LiDAR size (100 k points): run-to-run bit reproducibility, symmetric PSD information matrix,
    and agreement with the oracle on the whole update."""
    fr = get_frame(seed=0, n_pts=100_000, n_map=1_000_000)
    a = lio_gpu(gpu_ctx, fr)
    b = lio_gpu(gpu_ctx, fr)
    assert np.array_equal(a["state"], b["state"]) and np.array_equal(a["HTH"], b["HTH"])  # fixed-order reductions
    assert np.array_equal(a["match_plane"], b["match_plane"])
    for H in a["HTH"]:
        assert rel(H, H.T) < 1e-12
        assert np.linalg.eigvalsh(0.5 * (H + H.T)).min() > 0
    assert a["M"][0] > 0.85 * 100_000
    compare_lio(a, lio_oracle(fr))


def test_persistent_and_per_iteration_loops_are_bit_identical(gpu_ctx, small_frame):
    """loop_mode 2 / 1 (one cooperative kernel for the whole update, solve in every CTA / on CTA 0) vs loop_mode 0
    (residual + solve launch per iteration)."""
    fr = get_frame(seed=4, n_pts=20000, n_map=150_000, scene_scale=0.5)
    a2, a, b = sweep(gpu_ctx, lambda: lio_gpu(gpu_ctx, fr), [dict(loop_mode=2), dict(loop_mode=1), dict(loop_mode=0)])
    for x in (a, a2):
        assert x["iters"] == b["iters"]
        assert np.array_equal(x["state"], b["state"]) and np.array_equal(x["HTH"], b["HTH"]) and np.array_equal(x["match_plane"], b["match_plane"])
    compare_lio(b, lio_oracle(fr))


def test_config4_260k_points_several_tiles_per_cta(gpu_ctx):
    """BASELINE config 4 size (NTU_VIRAL: 260 k points, LIO only, beam_err 0.01): more points than one round of 132 x 704
    lanes, so every CTA walks several tiles and nothing stays resident in its slots."""
    cfg = S.LioCfg(beam_err=0.01)
    fr = get_frame(seed=12, n_pts=260_000, n_map=1_000_000, lio=cfg)
    g, o = lio_gpu(gpu_ctx, fr), lio_oracle(fr)
    assert o["M"][0] > 200_000
    compare_lio(g, o)
    with variant(gpu_ctx, loop_mode=0):
        g0 = lio_gpu(gpu_ctx, fr)
    assert np.array_equal(g0["state"], g["state"]) and np.array_equal(g0["match_plane"], g["match_plane"])


@pytest.mark.parametrize("name", ["small", "hilti_voxel_04_non_identity_extrinsics"])
def test_lio_matches_reference_source_golden(gpu_ctx, name):
    """The CUDA path against the committed outputs of the REFERENCE SOURCE (src/voxel_map.cpp compiled against stand-in
    headers, tests/golden/ref_lio_golden.npz): iteration count, effective feature number per iteration, matched planes and
    signed distances bit-exact, posterior within the north-star tolerance (held to 1e-9 / 1e-6 like the oracle checks)."""
    from ref_pin_cases import LIO_GOLDEN, lio_case

    g = np.load(LIO_GOLDEN)
    fr, cfg = lio_case(name)
    r = lio_gpu(gpu_ctx, fr, cfg)
    planes = fr["map"]["planes"]
    assert r["iters"] == int(g[f"{name}_iters"]) and np.array_equal(r["M"], g[f"{name}_M"])
    mk = r["match_plane"] >= 0
    assert np.array_equal(planes["center"][r["match_plane"][mk]], g[f"{name}_ptpl_center"])
    assert np.array_equal(r["dis_to_plane"][mk], g[f"{name}_ptpl_dis"])
    want = np.where(r["normal_plane"][:, None] >= 0, planes["normal"][np.maximum(r["normal_plane"], 0)], 0.0)
    assert np.array_equal(want, g[f"{name}_normals"])
    assert_state_close(r["state"], g[f"{name}_state"])
