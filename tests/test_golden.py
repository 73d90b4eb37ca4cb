"""Golden vectors (tests/golden/esikf_golden.npz, made by tests/golden/make_golden.py): the oracle must keep reproducing
them bit-for-bit (CPU), and the CUDA path must match them through the C ABI without the oracle in the loop (GPU)."""
import os

import numpy as np
import pytest

from fast_livo2_b200 import synthetic as S
from parity_util import GOLDEN_DIR, load_golden

def test_oracle_reproduces_golden_vectors():
    import oracle_bind as O

    g, lio_cfg, vio_cfg, cam, ext, vmap = load_golden()
    lio = O.OracleLIO(lio_cfg, ext)
    lio.set_map(vmap)
    o = lio.state_estimation(g["pts"], g["state_prior"], g["state_prior"])
    assert o["iters"] == int(g["lio_iters"]) and np.array_equal(o["M"], g["lio_M"])
    assert np.array_equal(o["match_plane"], g["lio_match"]) and np.array_equal(o["normal_plane"], g["lio_normal"])
    assert np.array_equal(o["dis_to_plane"], g["lio_dis"])
    assert np.array_equal(o["state"], g["lio_state"])
    vio = O.OracleVIO(cam, ext, vio_cfg)
    v = vio.update(g["img"], g["vis_pos"], g["warp_patch"], g["search_levels"], g["inv_ref_expo"], g["lio_state"], g["lio_state"])
    assert v["total_iters"] == int(g["vio_total_iters"]) and np.array_equal(v["iters_per_level"], g["vio_iters_per_level"])
    assert np.array_equal(v["state"], g["vio_state"]) and np.array_equal(v["errors"], g["vio_errors"])


def test_oracle_reproduces_inverse_variant_golden_vectors():
    """Same inputs, vio/inverse_composition_en on (tests/golden/esikf_golden_inverse.npz)."""
    import oracle_bind as O

    g, lio_cfg, vio_cfg, cam, ext, vmap = load_golden()
    gi = np.load(os.path.join(GOLDEN_DIR, "esikf_golden_inverse.npz"))
    vio = O.OracleVIO(cam, ext, vio_cfg)
    vio.set_inverse_refs([g["img_ref"]], gi["ref_img_index"], gi["ref_px"], gi["ref_f"], gi["ref_R"], gi["ref_pos"])
    vio.set_inverse(True)
    n = len(g["vis_pos"])
    v = vio.update(g["img"], g["vis_pos"], g["warp_patch"], g["search_levels"], np.ones(n), g["lio_state"], g["lio_state"])
    assert v["total_iters"] == int(gi["vio_total_iters"]) and np.array_equal(v["iters_per_level"], gi["vio_iters_per_level"])
    assert np.array_equal(v["accepted_per_level"], gi["vio_accepted_per_level"])
    assert np.array_equal(v["state"], gi["vio_state"]) and np.array_equal(v["errors"], gi["vio_errors"])
    assert np.array_equal(v["error_trace"], gi["vio_error_trace"])
    assert np.array_equal(vio.precompute_reference_patches(g["vis_pos"], 1)[:8], gi["H_sub_inv_level1"])


@pytest.mark.gpu
def test_cuda_path_matches_golden_vectors(gpu_ctx):
    from fast_livo2_b200 import api
    from parity_util import assert_state_close

    g, lio_cfg, vio_cfg, cam, ext, vmap = load_golden()
    ctx = gpu_ctx
    ctx.set_extrinsics(ext)
    ctx.map_upload(vmap, lio_cfg.voxel_size)
    r = ctx.lio_update(g["pts"], g["state_prior"], g["state_prior"], lio_cfg)
    assert r["iters"] == int(g["lio_iters"]) and np.array_equal(r["M"], g["lio_M"])
    assert np.array_equal(r["match_plane"], g["lio_match"]) and np.array_equal(r["normal_plane"], g["lio_normal"])
    assert np.array_equal(r["dis_to_plane"], g["lio_dis"])
    assert_state_close(r["state"], g["lio_state"])
    ctx.vio_set_camera(cam, vio_cfg)
    ctx.vio_set_image(g["img"])
    ctx.vio_set_ref_images([g["img_ref"]])
    st = S.unpack_state(g["lio_state"])
    n = len(g["vis_pos"])
    T_ref = np.tile(api.pack_T(g["T_ref_R"], g["T_ref_t"]), (n, 1))
    w = ctx.vio_warp_patches(np.zeros(n, np.int32), g["px_ref"], g["vis_pos"], g["vis_normal"], T_ref, api.pack_T(*S.camera_pose(ext, st["R"], st["p"])))
    np.testing.assert_allclose(w["A_cur_ref"], g["A_cur_ref"], rtol=1e-10, atol=1e-12)
    assert np.array_equal(w["search_levels"], g["search_levels"])
    np.testing.assert_allclose(w["warp_patch"], g["warp_patch"], atol=2e-3)
    v = ctx.vio_update(g["img"], g["vis_pos"], g["warp_patch"], g["search_levels"], g["inv_ref_expo"], g["lio_state"], g["lio_state"])
    assert v["total_iters"] == int(g["vio_total_iters"]) and np.array_equal(v["iters_per_level"], g["vio_iters_per_level"])
    assert_state_close(v["state"], g["vio_state"], rot_tol=1e-8, pos_tol=1e-8, cov_tol=1e-6, rest_tol=1e-8)
    np.testing.assert_allclose(v["errors"], g["vio_errors"], rtol=2e-6, atol=1e-3)
