"""GPU: the front-end entry points share one per-call scratch block and one pinned host block in the context. A call's
answers must not depend on what ran on the context before it, and what a call leaves for a later one (the depth image of
retrieve_scan, the world cloud of rgb_set_cloud, the sub-map of warp_patches(keep_on_device)) must survive the calls in
between.

1. Size order: on one context every entry point runs at a large size, a small one and the large one again, in the order
   of a VIO tick; each answer equals, bit for bit, the same call on a fresh context. On a fresh context the observation
   store is filled a few points per call, so that vmap_score's rows outgrow both its inputs and the pinned block the
   earlier calls left.
2. State that outlives a call: retrieve_scan -> depth_check, rgb_set_cloud -> rgb_colorize and warp_patches(keep_on_device)
   -> vio_run, with larger front-end calls in between, equal the same pairs on a fresh context."""
import numpy as np
import pytest

import color_cases as CC
import generate_cases as GC
import map_find as MF
import map_mirror as MM
import observe_cases as OC
import refpatch_cases as RFC
import retrieve_cases as RC
import select_cases as SC
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S

pytestmark = pytest.mark.gpu
CAMERA = "pinhole"
EXT = CC.CAMERAS[CAMERA][1]


@pytest.fixture(scope="module")
def ctx():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = api.Context(0)
    yield c
    c.close()


def on_fresh_context(run):
    c = api.Context(0)
    try:
        return run(c)
    finally:
        c.close()


def assert_same(got, want, label):
    if isinstance(want, dict):
        assert got.keys() == want.keys(), label
        for k in want:
            assert_same(got[k], want[k], f"{label}.{k}")
        return
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, label
    assert got.tobytes() == want.tobytes(), f"{label}: {int(np.sum(got != want))} of {want.size} differ"


# ------------------------------------------------------------------------------------------------------------- inputs
_inputs = {}


def inputs(name, large):
    """Seeded inputs of one entry point, built once so that every context sees the same arrays."""
    key = (name, large)
    if key not in _inputs:
        _inputs[key] = _make(name, large)
    return _inputs[key]


def _make(name, large):
    if name == "retrieve":
        sc = RC.scene(CAMERA, 120_000 if large else 800, seed=3 if large else 4, n_vis=6000 if large else 300)
        st = S.unpack_state(sc["state"])
        Rcw, Pcw = S.camera_pose(sc["ext"], st["R"], st["p"])
        pf = sc["pos"] @ Rcw.T + Pcw
        pc = S.cam_project(sc["cam"], pf)
        ok = (pf[:, 2] > 0.1) & (pc[:, 0] > 8) & (pc[:, 0] < sc["cam"].width - 8) & (pc[:, 1] > 8) & (pc[:, 1] < sc["cam"].height - 8)
        return dict(sc=sc, pos=np.ascontiguousarray(sc["pos"][ok]), pc=np.ascontiguousarray(pc[ok]))
    if name == "map":  # a device map and find_correspond queries near its points
        sc = GC.scene(CAMERA, 20_000, seed=5)
        rng = np.random.default_rng(6)
        n = 150_000 if large else 300
        q = sc["point_w"][rng.integers(0, len(sc["point_w"]), n)] + rng.normal(0, 0.3, (n, 3))
        if not large:
            q = np.concatenate([q, MF.boundary_points()])
        return dict(point_w=sc["point_w"], var=sc["var"].reshape(-1, 9), query=np.ascontiguousarray(q))
    if name == "select":
        return SC.candidates(CAMERA, 12_000 if large else 150, seed=7 if large else 8)
    if name == "color":
        return CC.scene(CAMERA, 300_000 if large else 1500, seed=9 if large else 10)
    if name == "generate":
        return GC.scene(CAMERA, 150_000 if large else 600, seed=11 if large else 12)
    if name == "observe":
        return OC.scene(CAMERA, 40_000 if large else 200, seed=13 if large else 14)
    if name == "refpatch":
        rng = np.random.default_rng(15 if large else 16)
        n = 6000 if large else 40
        return RFC.concat([RFC.point(rng, int(k), kind="zero" if k % 2 else "small") for k in rng.integers(1, 14, n)])
    if name == "lio":  # a scan to map and to run the LIO update on
        sc = CC.scene(CAMERA, 60_000 if large else 2000, seed=17 if large else 18)
        return dict(pts=sc["pts"], state=sc["lio_state"], ext=sc["ext"])
    if name == "patch":  # the lio scan's map in esikf_map_upload's form, and records to patch into it
        d = inputs("lio", large)
        m = on_fresh_context(lambda c: (_map_build(c, d), c.map_device_download())[1])
        rng = np.random.default_rng(19 if large else 20)
        ids = np.sort(rng.choice(len(m["planes"]), size=len(m["planes"]) // 3, replace=False)).astype(np.int32)
        return dict(map=m, ids=ids, planes=np.ascontiguousarray(m["planes"][rng.permutation(ids)]))
    if name == "vmap":  # an observation store of the retrieval scene's visual points, and the inputs of its calls
        sc = inputs("retrieve", large)["sc"]
        rng = np.random.default_rng(21 if large else 22)
        n_obs = np.asarray(sc["n_obs"], np.int32)
        first = np.concatenate([[0], np.cumsum(n_obs)]).astype(np.int32)
        m, n = int(first[-1]), len(n_obs)
        T = np.zeros((m, 12))
        T[:, [0, 4, 8]] = 1.0
        T[:, 9:] = rng.normal(0, 2.0, (m, 3))
        normal = rng.normal(size=(n, 3))
        return dict(sc=sc, first=first, px=rng.uniform(0, 600, (m, 2)), patch=rng.uniform(0, 255, (m, 64)).astype(np.float32), T=T,
                    id=rng.integers(0, 5, m).astype(np.int32), mean=rng.uniform(0, 200, m).astype(np.float32), score=rng.uniform(0, 1, m).astype(np.float32),
                    converged=(rng.random(n) < 0.3).astype(np.uint8), normal=normal / np.linalg.norm(normal, axis=1)[:, None])
    raise KeyError(name)


# ------------------------------------------------------------------------------------------------------- entry points
# Each step sets up what its call reads, makes the call(s) and returns the answers.
def _map_build(c, d):
    c.set_extrinsics(d["ext"])
    c.map_device_init(S.LioCfg(), root_capacity=1 << 16, grow=True)
    c.lio_set_scan(d["pts"])
    c.map_device_build(d["state"])


def step_lio_tick(c, large):
    d = inputs("lio", large)
    _map_build(c, d)
    c.lio_run(d["state"], d["state"], S.LioCfg())
    body_cov, cross = c.lio_fetch_point_cov()
    m, e = c.map_device_download(), c.map_device_export()
    order = np.lexsort(m["keys"].T[::-1])  # the download lists roots in no fixed order
    planes = np.concatenate([m["planes"][f:f + k] for f, k in zip(m["first"][order], m["count"][order])])
    return dict(normals=c.lio_fetch_normals(), body_cov=body_cov, cross=cross, keys=m["keys"][order], planes=planes, export=MM.export_dump(e))


def step_map_patch(c, large):
    d, p = inputs("lio", large), inputs("patch", large)
    cfg = S.LioCfg()
    c.set_extrinsics(d["ext"])
    c.map_upload(p["map"], cfg.voxel_size)
    c.map_patch(p["ids"], p["planes"])
    return c.lio_update(d["pts"], d["state"], d["state"], cfg)


def step_colorize(c, large):
    sc = inputs("color", large)
    c.set_extrinsics(sc["ext"])
    c.vio_set_camera(sc["cam"], S.VioCfg())
    c.rgb_set_cloud(sc["pts"], sc["lio_state"])
    return c.rgb_colorize(sc["img"], sc["blind"], state=sc["vio_state"])


def step_retrieve(c, large):
    d = inputs("retrieve", large)
    sc = d["sc"]
    c.set_extrinsics(sc["ext"])
    c.vio_set_camera(sc["cam"], RC.VIO_CFG)
    out = dict(scan=c.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"], depth=True))
    out["flags"] = c.vio_depth_check(d["pos"], d["pc"])
    return out


def step_find(c, large):
    d = inputs("map", large)
    c.map_device_init(S.LioCfg(), root_capacity=1 << 16, grow=True)
    c.map_device_update_points(d["point_w"], d["var"])
    return dict(patch=c.map_device_find(d["query"], api.FIND_RULE_PATCH), raycast=c.map_device_find(d["query"], api.FIND_RULE_RAYCAST))


def _select_setup(c, s):
    c.set_extrinsics(EXT)
    c.vio_set_camera(s["camcfg"], S.VioCfg())
    c.vio_set_image(s["img"])
    c.vio_set_ref_images(s["ref_imgs"])


def step_select(c, large):
    s = inputs("select", large)
    _select_setup(c, s)
    args = (s["ref_idx"], s["px_ref"], s["pos_w"], s["T_ref"], s["ref_inv_expo"], s["pc"], s["T_cur"], s["inv_expo"])
    out = dict(depth=c.vio_select_patches(*args, ref_level=s["ref_level"], ref_f=s["ref_f"], ref_pos=s["ref_pos"], ref_key=s["ref_key"], normal_en=False))
    out["homography"] = c.vio_select_patches(*args, normal_w=s["normal_w"], want_patches=True)
    return out


def step_warp(c, large):
    s = inputs("select", large)
    _select_setup(c, s)
    w = c.vio_warp_patches(s["ref_idx"], s["px_ref"], s["pos_w"], s["normal_w"], s["T_ref"], s["T_cur"])
    return dict(warp=w, affine=c.vio_warp_affine(s["ref_idx"], s["px_ref"], w["A_cur_ref"], w["search_levels"]),
                patch=c.vio_get_image_patch(s["pc"], 1))


def step_update_points(c, large):
    sc = inputs("observe", large)
    n = len(sc["pos"])
    c.set_extrinsics(sc["ext"])
    c.vio_set_camera(sc["cam"], S.VioCfg())
    c.vio_set_image(sc["img"])
    c.vio_set_patches(np.ascontiguousarray(sc["pos"]), np.zeros((n, 4 * 64), np.float32), np.ascontiguousarray(sc["search_levels"]), np.ones(n))
    return c.vio_update_points(sc["converged"], sc["last_T"], sc["last_px"], state=sc["state"])


def generate(c, large):
    """generate_points on the camera already set (vio_set_camera would void the depth image of retrieve_scan)."""
    sc = inputs("generate", large)
    c.vio_set_image(sc["img"])
    return c.vio_generate_points(sc["mask"], sc["grid_size"], sc["grid_n_width"], sc["grid_n_height"], sc["border"], pg=(sc["point_w"], sc["normal"], sc["var"]),
                                 add_from=(sc["add_pos"], sc["add_normal"]), state=sc["state"])


def step_generate(c, large):
    sc = inputs("generate", large)
    c.set_extrinsics(sc["ext"])
    c.vio_set_camera(sc["cam"], S.VioCfg())
    return generate(c, large)


def step_score(c, large):
    r = inputs("refpatch", large)
    return c.vio_score_ref_patches(r["first"], r["pos"], r["normal"], r["patch"], r["mean"], r["id"], r["T"])


def step_vmap(c, large):
    """The observation store through a tick: filled a few points per call, scored, edited by the update's new observations,
    read back, placed and walked."""
    v = inputs("vmap", large)
    sc = v["sc"]
    first, n = v["first"], len(v["first"]) - 1
    c.set_extrinsics(sc["ext"])
    c.vio_set_camera(sc["cam"], RC.VIO_CFG)
    c.vmap_init(1)
    ids = []
    for a in range(0, n, 4):
        f = first[a:a + 5]
        o = slice(int(f[0]), int(f[-1]))
        ids.append(c.vmap_add_points(f - f[0], v["px"][o], v["patch"][o], v["T"][o], v["id"][o], v["mean"][o], v["score"][o], np.full(len(f) - 1, -1, np.int32)))
    ids = np.concatenate(ids)
    pos, fp = sc["pos"], -(sc["pos"].mean(axis=0))
    out = dict(score=c.vmap_score(ids, pos, v["normal"]), choose=c.vmap_choose_ref(ids, False, pos=pos, frame_pos=fp))
    c.vio_set_image(sc["img"])
    c.vio_set_patches(pos, np.zeros((n, RC.VIO_CFG.levels * 64), np.float32), np.zeros(n, np.int32), np.ones(n))
    out["update"] = c.vmap_update_points(ids, v["converged"], 3, state=sc["state"])
    out["download"] = c.vmap_download(ids)
    c.vmap_place_points(ids, pos)
    keys = c.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"])["keys"]
    out["retrieve"] = c.vmap_retrieve(keys, *[int(sc[k]) for k in ("grid_size", "grid_n_width", "grid_n_height", "border")], False)
    return out


# the order of a VIO tick: the LIO tick's normals, point covariances and map mirror, a host map patched in place, the coloured
# scan, the retrieval, the sub-map, the update's new points, the reference patches and the observation store
TICK = [step_lio_tick, step_map_patch, step_colorize, step_retrieve, step_find, step_select, step_warp, step_update_points, step_generate, step_score, step_vmap]


def test_large_small_large_equals_fresh_contexts(ctx):
    want = {(f.__name__, large): on_fresh_context(lambda c: f(c, large)) for f in TICK for large in (True, False)}
    for rnd, large in enumerate((True, False, True)):
        for f in TICK:
            assert_same(f(ctx, large), want[(f.__name__, large)], f"round {rnd} {f.__name__} ({'large' if large else 'small'})")


# ------------------------------------------------------------------------------------------------- state that outlives a call
def _others(c):
    """Front-end calls larger than the call whose state has to survive them."""
    step_score(c, True)
    step_find(c, True)
    generate(c, True)


def test_depth_image_survives_later_calls(ctx):
    d = inputs("retrieve", False)
    sc = d["sc"]

    def scan(c):
        c.set_extrinsics(sc["ext"])
        c.vio_set_camera(sc["cam"], RC.VIO_CFG)
        return c.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"], depth=True)

    want = on_fresh_context(lambda c: (scan(c), c.vio_depth_check(d["pos"], d["pc"])))
    got_scan = scan(ctx)
    _others(ctx)
    assert_same(got_scan, want[0], "retrieve_scan")
    assert_same(ctx.vio_depth_check(d["pos"], d["pc"]), want[1], "depth_check after other calls")


def test_world_cloud_survives_later_calls(ctx):
    sc = inputs("color", False)

    def set_cloud(c):
        c.set_extrinsics(sc["ext"])
        c.vio_set_camera(sc["cam"], S.VioCfg())
        c.rgb_set_cloud(sc["pts"], sc["lio_state"])

    def colorize(c):
        return c.rgb_colorize(sc["img"], sc["blind"], state=sc["vio_state"])

    want = on_fresh_context(lambda c: (set_cloud(c), colorize(c))[1])
    set_cloud(ctx)
    step_score(ctx, True)
    assert_same(colorize(ctx), want, "colorize after a large score_ref_patches")


def test_installed_sub_map_survives_later_calls(ctx):
    s = inputs("select", False)
    state = S.pack_state(np.eye(3), np.zeros(3))

    def install(c):
        _select_setup(c, s)
        return c.vio_warp_patches(s["ref_idx"], s["px_ref"], s["pos_w"], s["normal_w"], s["T_ref"], s["T_cur"], keep_on_device=True)

    def update(c):
        c.vio_run(state, state)
        return c.vio_fetch()

    want = on_fresh_context(lambda c: (install(c), update(c)))
    assert_same(install(ctx), want[0], "warp_patches(keep_on_device)")
    big = inputs("select", True)
    ctx.vio_warp_affine(big["ref_idx"], big["px_ref"], np.tile(np.eye(2), (len(big["px_ref"]), 1, 1)), np.zeros(len(big["px_ref"]), np.int32))
    ctx.vio_get_image_patch(big["pc"], 0)
    step_score(ctx, True)
    step_find(ctx, True)
    assert_same(update(ctx), want[1], "vio_run after other front-end calls")
