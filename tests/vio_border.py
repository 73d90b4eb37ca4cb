"""Visual patches whose tap footprints reach the image border.

make_frame keeps every visual point well inside the image, but in the reference border-crossing footprints are normal:
retrieval checks (4+1)·2^L px once, on the level-0 projection, and updateState then reads an 11 x 11 strided footprint of
radius 5·2^(level+search_level) with no in-frame check (vio.cpp:1564-1597). These helpers place visual points so that their
PRIOR projection lands on chosen pixels at the edges, corners and just outside the image, and count in plain numpy how many
footprints actually leave it, so that tests can assert that the border cases are really there."""
import numpy as np

import oracle_bind as O
from fast_livo2_b200 import synthetic as S

HALF = 5  # updateState's taps reach 5 strides around the anchor pixel (patch pixels -4..3 plus the gradient neighbours)


def place_points(fr, state, px):
    """Scene points seen at pixels `px` (N, 2) from the camera pose of `state`: back-projected with cam_rays, cast onto the
    scene, with the hit rectangle's normal and the projection into the reference view (as make_frame builds them)."""
    cam = fr["cam_cfg"]
    st = S.unpack_state(state)
    Rcw, Pcw = S.camera_pose(fr["ext"], st["R"], st["p"])
    f = S.cam_rays(cam, np.asarray(px, np.float64))
    _, idx, hit = S.raycast(fr["rects"], -Rcw.T @ Pcw, f @ Rcw)
    assert (idx >= 0).all(), "every border ray must hit the scene"
    normals = np.stack([r.n for r in fr["rects"]])[idx]
    Rr, Pr = fr["T_ref"]
    return np.ascontiguousarray(hit), np.ascontiguousarray(normals), np.ascontiguousarray(S.cam_project(cam, hit @ Rr.T + Pr))


def footprint_box(px, stride):
    """Tap range [lo, hi] (pixels, both axes) of updateState's footprint at tap stride `stride`: anchor floor(u/s)*s, taps
    -5s .. +5s. Returns (x_lo, x_hi, y_lo, y_hi)."""
    s = np.asarray(stride, np.float64)
    ui = np.floor((px[:, 0] / s).astype(np.float32)) * s
    vi = np.floor((px[:, 1] / s).astype(np.float32)) * s
    return ui - HALF * s, ui + HALF * s, vi - HALF * s, vi + HALF * s


def leaves_image(px, search_levels, levels, width, height):
    """Per patch: does its footprint leave [0, width) x [0, height) at some pyramid level (evaluated at `px`)?"""
    out = np.zeros(len(px), bool)
    for lvl in range(levels):
        x0, x1, y0, y1 = footprint_box(px, 1 << (lvl + np.asarray(search_levels)))
        out |= (x0 < 0) | (x1 > width - 1) | (y0 < 0) | (y1 > height - 1)
    return out


def border_targets(width, height, levels, rng, max_search_level=2):
    """Target pixels and forced search levels of border patches.

    For every tap stride s = 2^p used (p = level + search_level, up to levels-1+max_search_level) and every edge, the
    footprint (radius 5s) is placed just inside, exactly at, and partly beyond the edge; plus the four corners and points
    slightly outside the image (updateState does not reject them). Left / right edge targets sit on rows far enough from
    the top and bottom that the reference's linear row wrap stays inside the buffer (`in_buffer`)."""
    p_max = levels - 1 + max_search_level
    reach = HALF << p_max  # vertical reach of the coarsest footprint
    mid_lo, mid_hi = reach + 40, height - 1 - reach - 40
    assert mid_lo < mid_hi, "image too small for an in-buffer band"
    px, sl, inb = [], [], []
    k = 0
    for p in range(p_max + 1):
        s = 1 << p
        valid = [q for q in range(max_search_level + 1) if 0 <= p - q <= levels - 1]  # search levels that reach stride s
        for off in (s + 0.37, 0.37, -0.5 * s + 0.37):  # anchor 1 stride inside / exactly at / half a radius past the edge
            a = HALF * s + off
            lvl_sl = valid[k % len(valid)]
            k += 1
            for edge in range(4):
                if edge < 2:
                    v = rng.uniform(mid_lo, mid_hi)
                    u = a if edge == 0 else width - 1 - a + 0.26
                    inb.append(True)
                else:
                    u = rng.uniform(0.3 * width, 0.7 * width)
                    v = a if edge == 2 else height - 1 - a + 0.26
                    inb.append(False)
                px.append((u, v))
                sl.append(lvl_sl)
    for u in (-0.3, 0.4, width - 0.6, width - 1.4):  # slightly outside / on the outermost pixel column
        px.append((u, rng.uniform(mid_lo, mid_hi)))
        sl.append(len(px) % (max_search_level + 1))
        inb.append(True)
    for v in (-0.3, height - 0.6):
        px.append((rng.uniform(0.3 * width, 0.7 * width), v))
        sl.append(len(px) % (max_search_level + 1))
        inb.append(False)
    for u, v in ((3.3, 2.7), (width - 3.6, 4.1), (2.2, height - 3.3), (width - 2.9, height - 2.4)):  # corners
        px.append((u, v))
        sl.append(len(px) % (max_search_level + 1))
        inb.append(False)
    return np.array(px), np.array(sl, np.int32), np.array(inb)


def patches_at(fr, state, px, search_levels):
    """Visual patches at prior projection `px` with forced `search_levels`: scene points (place_points) and their warp
    patches (getWarpMatrixAffineHomography + warpAffine of the oracle, all of the frame's pyramid levels)."""
    pos, nrm, pref = place_points(fr, state, px)
    vio = O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"])
    st = S.unpack_state(state)
    T_cur = S.camera_pose(fr["ext"], st["R"], st["p"])
    wp = np.zeros((len(px), 64 * fr["vio_cfg"].levels), np.float32)
    for j in range(len(px)):
        A, _ = vio.warp_matrix(pref[j], pos[j], nrm[j], fr["T_ref"], T_cur)
        wp[j] = vio.warp_affine(fr["img_ref"], A, pref[j], int(search_levels[j]))
    return dict(vis_pos=pos, vis_normal=nrm, px_ref=pref, search_levels=np.asarray(search_levels, np.int32), warp_patch=wp)


def with_interior(fr, state, extra):
    """The frame's interior patches (search levels as getBestSearchLevel picks them) followed by the patches `extra`."""
    w = O.oracle_warp_patches(fr, state)
    out = {k: np.ascontiguousarray(np.concatenate([a, extra[k]])) for k, a in
           (("vis_pos", fr["vis_pos"]), ("vis_normal", fr["vis_normal"]), ("px_ref", fr["px_ref"]), ("search_levels", w["search_levels"]),
            ("warp_patch", w["warp_patch"]))}
    out["inv_ref_expo"] = np.ones(len(out["vis_pos"]))
    return out


def border_patch_set(fr, state, seed=0, in_buffer_only=False, every=1, max_search_level=2):
    """The frame's interior patches plus border patches placed at the prior `state`'s projection (every `every`-th target
    of border_targets). Returns vis_pos / vis_normal / px_ref / search_levels / warp_patch / inv_ref_expo, `px` (prior
    projection targets, NaN for interior patches), `border` (mask), `in_buffer` (mask of border patches whose reads stay
    inside the image buffer) and `n_leave` (patches whose footprint leaves the image at some level at the prior, counted
    here in numpy)."""
    cam, L = fr["cam_cfg"], fr["vio_cfg"].levels
    tpx, tsl, tin = border_targets(cam.width, cam.height, L, np.random.default_rng(seed), max_search_level)
    keep = tin if in_buffer_only else np.ones(len(tpx), bool)
    tpx, tsl, tin = tpx[keep][::every], tsl[keep][::every], tin[keep][::every]
    out = with_interior(fr, state, patches_at(fr, state, tpx, tsl))
    n_int = len(fr["vis_pos"])
    out.update(px=np.concatenate([np.full((n_int, 2), np.nan), tpx]), border=np.concatenate([np.zeros(n_int, bool), np.ones(len(tpx), bool)]),
               in_buffer=np.concatenate([np.zeros(n_int, bool), tin]), n_leave=int(leaves_image(tpx, tsl, L, cam.width, cam.height).sum()))
    return out


def edge_pixels(width, height, levels, rng, n_mid=2):
    """getImagePatch query pixels at the edges for levels 0..levels-1: the 8 x 8 patch (+1 tap for the bilinear weights)
    reaches 4s left / up and 4s + s right / down of the anchor floor(u/s)*s. Returns (in_buffer (N, 2), outside (N, 2)):
    left / right edge pixels on rows whose reads stay inside the buffer, and top / bottom / corner pixels whose linear
    indices leave it."""
    reach = 5 << (levels - 1)
    ins, outs = [], []
    for lvl in range(levels):
        s = 1 << lvl
        for off in (-0.3, 0.21, 0.5 * s + 0.13, 4 * s - 0.6, 4 * s + 0.4, 5 * s + 0.4):
            for _ in range(n_mid):
                v = rng.uniform(reach + 8, height - 1 - reach - 8)
                ins.append((off, v))
                ins.append((width - 1 - off + 0.02, v))
                u = rng.uniform(reach + 8, width - 1 - reach - 8)
                outs.append((u, off))
                outs.append((u, height - 1 - off + 0.02))
    outs += [(0.3, 0.6), (width - 0.7, 1.2), (1.6, height - 0.4), (width - 1.3, height - 1.8)]
    return np.array(ins), np.array(outs)
