"""The cases on which the oracle is pinned against the reference source (tests/test_oracle_ref_pin.py, _vio.py) and which
other tests and tests/golden/make_ref_golden.py run too: the frames, where the reference's committed outputs lie, the VIO pin
store and the border inputs.

The reference's stored outputs (tests/golden/ref_*_golden.npz, tests/golden/ref_pin/*.npz) are keyed to exactly these
inputs: a change here that moves one input bit invalidates them."""
import os

import numpy as np
import pytest

import oracle_bind as O
from conftest import get_frame
from fast_livo2_b200 import synthetic as S

HERE = os.path.dirname(os.path.abspath(__file__))

# ----------------------------------------------------------------------------------------------------- LIO
LIO_GOLDEN = os.path.join(HERE, "golden", "ref_lio_golden.npz")

LIO_CASES = {
    "small": dict(frame=dict(seed=1, n_pts=4000, n_map=150_000, scene_scale=0.5)),
    "seed3": dict(frame=dict(seed=3, n_pts=5000, n_map=150_000, scene_scale=0.5)),
    "20k": dict(frame=dict(seed=4, n_pts=20000, n_map=150_000, scene_scale=0.5)),
    "three_iterations": dict(frame=dict(seed=0, n_pts=5000, n_map=150_000, scene_scale=0.5), cfg=dict(max_iterations=3)),
    "hilti_voxel_04_non_identity_extrinsics": dict(frame=dict(seed=5, n_pts=6000, n_map=400_000, lio=S.LioCfg(voxel_size=0.4, min_eigen_value=1e-4, max_points_num=100),
                                                            ext=S.hilti_extrinsics(), scene="corridor", scene_scale=0.25)),
    "voxel_2m": dict(frame=dict(seed=7, n_pts=6000, n_map=300_000, lio=S.LioCfg(voxel_size=2.0, min_eigen_value=0.005), scene_scale=2.0)),
}

EDGE_FRAMES = {
    "voxel_0.5": dict(seed=1, n_pts=4000, n_map=150_000, scene_scale=0.5),
    "voxel_0.4": dict(seed=5, n_pts=6000, n_map=400_000, lio=S.LioCfg(voxel_size=0.4, min_eigen_value=1e-4, max_points_num=100), ext=S.hilti_extrinsics(), scene="corridor",
                      scene_scale=0.25),
    "voxel_2.0": dict(seed=7, n_pts=6000, n_map=300_000, lio=S.LioCfg(voxel_size=2.0, min_eigen_value=0.005), scene_scale=2.0),
}


def lio_case(name):
    """(frame, LIO config) of LIO_CASES[name]."""
    c = LIO_CASES[name]
    fr = get_frame(**c["frame"])
    cfg = fr["lio_cfg"]
    if "cfg" in c:
        cfg = S.LioCfg(**{**cfg.__dict__, **c["cfg"]})
    return fr, cfg


# ----------------------------------------------------------------------------------------------------- VIO
VIO_GOLDEN = os.path.join(HERE, "golden", "ref_vio_golden.npz")
VIO_PIN = O.RefPin("vio")  # one store: recording (FL2_RECORD_REF_PIN=1) merges every VIO test's outputs into one file
vio_needs_ref = pytest.mark.skipif(not O.RefPin.available("vio"), reason="neither oracle/_ref/libfl2_ref_vio.so nor tests/golden/ref_pin/vio.npz")

VIO_CASES = {
    "small": dict(seed=2, n_pts=2000, n_map=120_000, n_patches=150, scene_scale=0.5),
    "exposure": dict(seed=6, n_pts=1000, n_map=120_000, n_patches=200, scene_scale=0.5, vio=S.VioCfg(exposure_estimate_en=True)),
    "three_levels": dict(seed=8, n_pts=1000, n_map=120_000, n_patches=300, scene_scale=0.5, vio=S.VioCfg(levels=3, img_point_cov=400.0)),
    "distorted_pinhole": dict(seed=9, n_pts=1000, n_map=120_000, n_patches=200, scene_scale=0.5,
                              cam=S.CamCfg(d=(-0.05, 0.02, 0.001, -0.0005, 0.0))),
    # config 3's camera (HILTI22 fisheye, vk::EquidistantCamera) behind the same abstract interface
    "fisheye": dict(seed=10, n_pts=1000, n_map=120_000, n_patches=200, scene_scale=0.5, vio=S.VioCfg(img_point_cov=1000.0),
                    cam=S.CamCfg(model=1, width=720, height=540, fx=351.31400364193297, fy=351.4911744656785, cx=367.8522793375995, cy=253.8402144980996,
                                 d=(-0.03696737352869157, -0.008917880497032812, 0.008912969593422046, -0.0037685977496087313, 0.0))),
}


def vio_pin_prior(fr, seed=3):
    """The prior of the pinned VIO cases. It draws the rotation before the covariance, unlike harness.vio_prior: the two give
    different states, and the stored reference outputs belong to this one."""
    rng = np.random.default_rng(seed)
    t = S.unpack_state(fr["state_true"])
    return S.pack_state(t["R"] @ S.so3_exp(rng.normal(0, np.deg2rad(0.15), 3)), t["p"] + rng.normal(0, 0.01, 3), 1.0 + rng.normal(0, 0.01), t["v"], g=t["g"],
                        cov=S.random_prior_cov(rng, scale=0.2))


def vio_inputs(name):
    """(frame, prior, the oracle's warp patches at the prior) of VIO_CASES[name]."""
    fr = get_frame(**VIO_CASES[name])
    prior = vio_pin_prior(fr)
    w = O.oracle_warp_patches(fr, prior)
    return fr, prior, w


# The border rule (DESIGN §4): taps use the reference's linear addressing and read 0 outside [0, w·h). Where the reference is
# well defined — a footprint that wraps to the neighbouring row but stays inside the buffer, and warpAffine's explicit
# in-frame test — the oracle must reproduce it bit for bit. Beyond the buffer the reference reads outside img.data
# (undefined), so those cases are checked against the oracle only (tests/test_oracle_numpy_crosscheck.py, tests/test_gpu_vio_border.py).
BORDER_FRAME = dict(seed=2, n_pts=2000, n_map=120_000, n_patches=250, scene_scale=0.5)


def warp_affine_border_cases(cols, rows):
    """(A_cur_ref, px_ref, search_level) whose warpAffine samples fall on both sides of 0 / cols-1 / rows-1 and exactly on
    them: dyadic matrices (exact inverses and determinants, so the sample positions are exact) around reference pixels at
    integer and half-integer distances from the edges, plus a zero matrix (NaN inverse: the patch is left untouched)."""
    mats = [np.eye(2), 2.0 * np.eye(2), 0.5 * np.eye(2), np.array([[1.25, -0.5], [0.5, 1.25]]), np.array([[1.0, 0.5], [0.25, 1.0]])]
    pxs = [(cols - 4.0, 200.0), (cols - 3.5, 300.5), (cols - 1.0, 250.25), (cols - 1.5, 260.0), (0.0, 220.0), (3.0, 230.5), (0.5, 240.0),
           (320.0, rows - 4.0), (321.5, rows - 2.5), (300.25, rows - 1.0), (310.0, 0.0), (305.5, 2.0), (cols - 3.0, rows - 3.0), (2.0, 1.0),
           (cols - 1.0, rows - 1.0), (0.0, 0.0)]
    cases = [(A, np.array(px), sl) for sl in range(3) for A in mats for px in pxs]
    cases.append((np.zeros((2, 2)), np.array([cols - 4.0, 200.0]), 0))
    return cases
