"""Visual sub-maps drawn from many keyframes, as FAST-LIVO2 builds them: every sub-map entry carries its own reference
Feature — its own keyframe image, pose T_f_w_, bearing f_ / pixel px_ and inverse exposure time (vio.cpp:770, 1592, 1621;
1345-1353 for the inverse-compositional variant).

build(name) renders K keyframes of a synthetic frame's own scene from poses around the truth, each with its own exposure
gain, optionally re-renders the current image with a gain != 1 (so the true inverse exposure is 1 / g_cur while the prior
stays near 1), assigns the frame's visual points to keyframes in one of three orders (interleaved, sorted by keyframe, a
seeded shuffle), optionally replicates them beyond the frame's point count (every replica of a point from another keyframe)
and returns every input of the forward update, the inverse-compositional reference data, the oracle's warp patches at the
prior and the esikf_vio_select_patches candidates of the same points.

The reference's stored outputs (tests/golden/ref_pin/keyframes.npz) are keyed to exactly these inputs: a change here that
moves one input bit invalidates them (re-record with FL2_RECORD_REF_PIN=1 where oracle/_ref is built)."""
import dataclasses

import numpy as np

import oracle_bind as O
from conftest import get_frame
from fast_livo2_b200 import synthetic as S
from ref_pin_cases import VIO_CASES, vio_pin_prior

PINHOLE = dict(seed=2, n_pts=1000, n_map=120_000, n_patches=300, scene_scale=0.5)  # config 2's camera (S.CamCfg())
DISTORTED = VIO_CASES["distorted_pinhole"]
THREE_LEVELS = VIO_CASES["three_levels"]
CONFIG5_CAM = S.CamCfg(width=612, height=512, fx=612.0 * 0.72, fy=612.0 * 0.72, cx=306.0, cy=256.0)
CONFIG5 = dict(seed=13, n_pts=1000, n_map=300_000, n_patches=4000, scene_scale=0.7, cam=CONFIG5_CAM, vio=S.VioCfg(levels=5, img_point_cov=1000.0))
FISHEYE_CAM = VIO_CASES["fisheye"]["cam"]
FISHEYE = dict(seed=9, n_pts=1000, n_map=100_000, n_patches=200, scene_scale=0.5, cam=FISHEYE_CAM, vio=S.VioCfg(img_point_cov=1000.0), ext=S.hilti_extrinsics())

# name -> (frame, keyword arguments of make_case)
CASES = {
    "pinhole": (PINHOLE, dict()),
    "pinhole_gain": (PINHOLE, dict(g_cur=1.25)),
    "pinhole_expo_off": (PINHOLE, dict(exposure_en=False)),
    "pinhole_gain_expo_off": (PINHOLE, dict(g_cur=1.25, exposure_en=False)),
    "pinhole_sorted": (PINHOLE, dict(g_cur=1.25, order="sorted")),
    "pinhole_shuffled": (PINHOLE, dict(g_cur=1.25, order="shuffled")),
    "distorted_gain": (DISTORTED, dict(g_cur=1.25)),
    "three_levels_mixed": (THREE_LEVELS, dict(g_cur=0.8, mixed_search=True)),
    "config5_4k": (CONFIG5, dict(g_cur=1.25, mixed_search=True)),
    "config5_6k": (CONFIG5, dict(g_cur=1.25, mixed_search=True, n=6000)),
    # above 4 224 = 2 x 16 warps x 132 SMs: more than 32 patches per CTA of the persistent update
    "pinhole_5k": (PINHOLE, dict(g_cur=1.25, n=5000)),
    "fisheye_gain": (FISHEYE, dict(g_cur=1.25)),
}
ORDERS = ("interleaved", "sorted", "shuffled")

_cache = {}


def border(levels):
    """make_frame's margin: every tap of a patch at the coarsest level lies inside the image."""
    return (4 + 1) * (1 << levels) + 8


def _once(key, make):
    if key not in _cache:
        _cache[key] = make()
    return _cache[key]


def keyframes(fr, K, seed, rot_deg=3.0, pos=0.15, gains=(0.6, 1.5)):
    """K keyframe camera poses (Rcw, Pcw) around the frame's true IMU pose, their exposure gains (spread over `gains` in a
    seeded order) and their images rendered from the frame's scene."""
    return _once(("keyframes", id(fr), K, seed, rot_deg, pos, gains), lambda: _keyframes(fr, K, seed, rot_deg, pos, gains))


def _keyframes(fr, K, seed, rot_deg, pos, gains):
    rng = np.random.default_rng(seed)
    t = S.unpack_state(fr["state_true"])
    cam, ext = fr["cam_cfg"], fr["ext"]
    poses = []
    for _ in range(K):
        R = t["R"] @ S.so3_exp(rng.normal(0, 1, 3) / np.sqrt(3) * np.deg2rad(rot_deg))
        p = t["p"] + rng.normal(0, 1, 3) / np.sqrt(3) * pos
        poses.append(S.camera_pose(ext, R, p))
    g = rng.permutation(np.linspace(gains[0], gains[1], K))
    imgs = [S.render(fr["rects"], cam, Rcw, Pcw, expo_gain=gk) for (Rcw, Pcw), gk in zip(poses, g)]
    return poses, g, imgs


def make_case(frame, K=12, g_cur=1.0, exposure_en=True, order="interleaved", n=None, mixed_search=False, seed=0):
    fr = get_frame(**frame)
    cam, L = fr["cam_cfg"], fr["vio_cfg"].levels
    vio_cfg = dataclasses.replace(fr["vio_cfg"], exposure_estimate_en=exposure_en)
    poses, gains, ref_imgs = keyframes(fr, K, seed)
    img = fr["img"] if g_cur == 1.0 else _once(("img", id(fr), g_cur), lambda: S.render(fr["rects"], cam, *fr["T_cur_true"], expo_gain=g_cur))

    # where each keyframe sees each point; a keyframe that sees it outside the border (or behind) is not its reference
    b = border(L)
    pos_all = fr["vis_pos"]
    n0 = len(pos_all)
    pc_k = np.stack([pos_all @ R.T + P for R, P in poses])  # (K, n0, 3)
    px_k = np.stack([S.cam_project(cam, pc) for pc in pc_k])
    ok = (pc_k[..., 2] > 0.1) & (px_k[..., 0] > b) & (px_k[..., 0] < cam.width - b) & (px_k[..., 1] > b) & (px_k[..., 1] < cam.height - b)

    # entry j is replica r = j // n0 of point p = j % n0, from keyframe (p + r) % K: neighbouring entries (one warp's patches,
    # the two cache slots of a warp) and the replicas of one point come from different keyframes. A keyframe that does not
    # see the point passes it on to the next one; a point no keyframe sees is dropped.
    N = n0 if n is None else n
    rep = np.arange(N) % n0
    want = (rep + np.arange(N) // n0) % K
    ref_idx = np.full(N, -1)
    for s in range(K):
        k = (want + s) % K
        free = (ref_idx < 0) & ok[k, rep]
        ref_idx[free] = k[free]
    keep = np.nonzero(ref_idx >= 0)[0]
    rep, ref_idx = rep[keep], ref_idx[keep]
    if order == "sorted":
        o = np.argsort(ref_idx, kind="stable")
    elif order == "shuffled":
        o = np.random.default_rng(seed + 1).permutation(len(rep))
    else:
        assert order == "interleaved", order
        o = np.arange(len(rep))
    rep, ref_idx = rep[o], ref_idx[o].astype(np.int32)
    m = len(rep)

    R_ref = np.stack([poses[k][0] for k in ref_idx])
    t_ref = np.stack([poses[k][1] for k in ref_idx])
    pc_ref = pc_k[ref_idx, rep]
    px_ref = np.ascontiguousarray(px_k[ref_idx, rep])
    f_ref = pc_ref / np.linalg.norm(pc_ref, axis=1, keepdims=True)
    vis_pos, vis_normal = np.ascontiguousarray(pos_all[rep]), np.ascontiguousarray(fr["vis_normal"][rep])
    inv_ref_expo = 1.0 / gains[ref_idx]
    T_ref = np.concatenate([R_ref.reshape(m, 9), t_ref], 1)
    refs = dict(ref_imgs=ref_imgs, ref_img_index=ref_idx, ref_px=px_ref, ref_f=np.ascontiguousarray(f_ref), ref_R=np.ascontiguousarray(R_ref.reshape(m, 9)),
                ref_pos=np.ascontiguousarray(-np.einsum("nji,nj->ni", R_ref, t_ref)), ref_t=np.ascontiguousarray(t_ref))

    prior = vio_pin_prior(fr)
    st = S.unpack_state(prior)
    T_cur = S.camera_pose(fr["ext"], st["R"], st["p"])

    # the oracle's warp patches at the prior, each from its own keyframe's pose and image
    orc = O.OracleVIO(cam, fr["ext"], vio_cfg)
    A = np.zeros((m, 2, 2))
    sl = np.zeros(m, np.int32)
    for i in range(m):
        A[i], sl[i] = orc.warp_matrix(px_ref[i], vis_pos[i], vis_normal[i], (R_ref[i], t_ref[i]), T_cur)
    if mixed_search:
        sl[::3] = np.where(sl[::3] == 0, 1, 0)  # a third of the patches one search level off the matrix's choice
    wp = np.stack([orc.warp_affine(ref_imgs[ref_idx[i]], A[i], px_ref[i], sl[i]) for i in range(m)])

    pc_cur = S.cam_project(cam, vis_pos @ T_cur[0].T + T_cur[1])
    select = dict(camcfg=cam, img=img, ref_imgs=ref_imgs, ref_idx=ref_idx, px_ref=px_ref, ref_level=np.zeros(m, np.int32), ref_f=refs["ref_f"],
                  ref_pos=refs["ref_pos"], pos_w=vis_pos, normal_w=vis_normal, T_ref=T_ref, ref_inv_expo=inv_ref_expo,
                  ref_key=(1000 + 7 * ref_idx).astype(np.int32), pc=pc_cur, T_cur=np.concatenate([T_cur[0].reshape(9), T_cur[1]]), inv_expo=float(st["inv_expo"]))
    return dict(frame=fr, cam_cfg=cam, ext=fr["ext"], vio_cfg=vio_cfg, K=K, gains=gains, g_cur=g_cur, img=img, ref_imgs=ref_imgs, vis_pos=vis_pos,
                vis_normal=vis_normal, rep=rep, ref_idx=ref_idx, px_ref=px_ref, T_ref=T_ref, inv_ref_expo=inv_ref_expo, refs=refs, prior=prior,
                T_cur=T_cur, warp_patch=wp, search_levels=sl, A_cur_ref=A, select=select)


def build(name):
    """make_case of CASES[name], built once per session (rendering costs about 0.5 s per keyframe)."""
    frame, kw = CASES[name]
    return _once(name, lambda: make_case(frame, **kw))


def update_args(c, inv_ref_expo=None):
    """The positional arguments of OracleVIO.update / RefVIO.update / Context.vio_update."""
    ie = c["inv_ref_expo"] if inv_ref_expo is None else inv_ref_expo
    return (c["img"], c["vis_pos"], c["warp_patch"], c["search_levels"], ie, c["prior"], c["prior"])


def oracle(c, inverse=False, refs=None):
    """OracleVIO on the case's camera / config, set up for the inverse-compositional variant with `refs` (default: the case's)."""
    vio = O.OracleVIO(c["cam_cfg"], c["ext"], dataclasses.replace(c["vio_cfg"], inverse_composition_en=inverse))
    if inverse:
        vio.set_inverse_refs(**(c["refs"] if refs is None else refs))
        vio.set_inverse(True)
    return vio


def pack_T(R, t):
    return np.concatenate([np.asarray(R).reshape(9), np.asarray(t).reshape(3)])
