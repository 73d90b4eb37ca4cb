"""GPU: the shim managers stage every call through one pinned block each. A method's answers must not depend on what ran on
the managers before it, and what a call leaves for a later one must survive the calls in between.

The managers run in tests/shim_staging_driver.cpp on seeded inputs from synthetic.make_frame and the *_cases modules; its
answers are compared bit for bit.
1. Against the C ABI: each method equals the plain esikf_* call on the same inputs (on the managers' context, right after
   the method; ScoreReferencePatches and GenerateVisualMapPoints also against api.Context on the refpatch / generate cases).
2. Size order: every method at a large size, a small one and the large one again on one manager pair equals the same
   calls on fresh managers (the coloured cloud outgrows its room on the first large call; the resident scan has more voxel
   keys than RetrieveScanVoxels first makes room for).
3. State that outlives a call: the association a lazy MaterializePointLists reads after UpdateVoxelMap(), FindCorrespond
   and SetWorldCloud, and the sub-map of SelectSubSparseMap after the other front-end calls.
4. A BuildVoxelMap that fails after uploading the scan leaves nothing that changes the next, larger calls."""
import functools
import os
import subprocess

import numpy as np
import pytest

import generate_cases as GC
import refpatch_cases as RFC
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "fast_livo2_b200")

# SubMapCandidate of fl2_shim.hpp
CAND = np.dtype([("ref_img_index", "<i4"), ("ref_level", "<i4"), ("ref_key", "<i4"), ("pad", "<i4"), ("px_ref", "<f8", 2), ("ref_f", "<f8", 3), ("ref_pos", "<f8", 3),
                 ("pos_w", "<f8", 3), ("normal_w", "<f8", 3), ("T_ref_w", "<f8", 12), ("ref_inv_expo", "<f8"), ("pc", "<f8", 2)])
# ScoredPoint and PatchObservation of fl2_shim.hpp
SCORED = np.dtype([("pos", "<f8", 3), ("normal", "<f8", 3)])
OBS = np.dtype([("T", "<f8", 12), ("patch", "<f4", 64), ("mean", "<f4"), ("id", "<i4")])
RESIDENT_ROOM = 1 << 16  # the keys RetrieveScanVoxels makes room for before it has seen a resident scan


@functools.cache
def gen_case():
    return GC.scene("pinhole", 20_000, seed=7)


@functools.cache
def score_cases():
    """A refpatch case, and observations without points (the call answers nothing)."""
    rng = np.random.default_rng(41)
    cases = RFC.concat([RFC.point(rng, int(k), kind="zero" if k % 2 else "small") for k in rng.integers(1, 14, 300)])
    none = dict(first=np.zeros(1, np.int32), pos=np.zeros((0, 3)), normal=np.zeros((0, 3)), patch=np.ones((5, 64), np.float32), mean=np.zeros(5, np.float32),
                id=np.arange(5, dtype=np.int32), T=np.zeros((5, 12)))
    return dict(cases=cases, none=none)


def put(d, name, a, dtype=None):
    np.ascontiguousarray(a, dtype=dtype).tofile(os.path.join(d, name + ".bin"))


def write_inputs(d):
    fr = S.make_frame(seed=31, n_pts=60_000, n_map=1000, n_patches=1500)
    cam, ext = fr["cam_cfg"], fr["ext"]
    st = S.unpack_state(fr["state_true"])
    Rcw, Pcw = S.camera_pose(ext, st["R"], st["p"])
    T_cur = np.concatenate([Rcw.reshape(9), Pcw])
    meta = np.concatenate([[cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height], ext.extR.reshape(9), ext.extT, ext.Rcl.reshape(9), ext.Pcl, T_cur])
    meta.astype(np.float64).tofile(os.path.join(d, "meta.bin"))
    img = np.ascontiguousarray(fr["img"], dtype=np.uint8)
    img.tofile(os.path.join(d, "img.bin"))
    np.ascontiguousarray(fr["img_ref"], dtype=np.uint8).tofile(os.path.join(d, "ref.bin"))
    np.ascontiguousarray(np.stack([img, 255 - img, img // 2], -1)).tofile(os.path.join(d, "bgr.bin"))
    Rr, Pr = fr["T_ref"]
    rng = np.random.default_rng(32)
    pts = fr["pts"].astype(np.float32)
    for key, step, n_cand in (("L", 1, len(fr["vis_pos"])), ("S", 20, 100)):
        c = np.zeros(n_cand, CAND)
        c["px_ref"], c["pos_w"], c["normal_w"] = fr["px_ref"][:n_cand], fr["vis_pos"][:n_cand], fr["vis_normal"][:n_cand]
        c["T_ref_w"] = np.concatenate([Rr.reshape(9), Pr])
        c["ref_inv_expo"] = 1.0
        c["pc"] = S.cam_project(cam, fr["vis_pos"][:n_cand] @ Rcw.T + Pcw)
        c.tofile(os.path.join(d, f"{key}_cands.bin"))
        np.ascontiguousarray(pts[::step]).tofile(os.path.join(d, f"{key}_pts.bin"))
        np.ascontiguousarray(np.concatenate([pts[::step], pts[::step] * 1.5])).tofile(os.path.join(d, f"{key}_dense.bin"))
        np.ascontiguousarray(fr["state_prior"]).tofile(os.path.join(d, f"{key}_state.bin"))
        q = np.concatenate([fr["vis_pos"][:n_cand], fr["vis_pos"][: n_cand // 3]]) + rng.normal(0, 0.2, (n_cand + n_cand // 3, 3))
        np.ascontiguousarray(q).tofile(os.path.join(d, f"{key}_query.bin"))
    # the wide scan: one point per 0.5 m voxel for most of its points, more than RESIDENT_ROOM of them
    put(d, "W_pts", rng.uniform(-40, 40, (100_000, 3)), np.float32)
    for name, c in score_cases().items():
        put(d, name + "_first", c["first"], np.int32)
        sp = np.zeros(len(c["pos"]), SCORED)
        sp["pos"], sp["normal"] = c["pos"], c["normal"]
        put(d, name + "_pts", sp)
        ob = np.zeros(len(c["patch"]), OBS)
        ob["T"], ob["patch"], ob["mean"], ob["id"] = c["T"], c["patch"], c["mean"], c["id"]
        put(d, name + "_obs", ob)
    g = gen_case()
    cam, ext = g["cam"], g["ext"]
    put(d, "gen_meta", np.concatenate([[cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height], cam.d, ext.extR.reshape(9), ext.extT, ext.Rcl.reshape(9), ext.Pcl,
                                       [g["grid_size"], g["grid_n_width"], g["grid_n_height"], g["border"]]]), np.float64)
    put(d, "gen_pw", g["point_w"], np.float64), put(d, "gen_normal", g["normal"], np.float64), put(d, "gen_var", g["var"], np.float64)
    put(d, "gen_add_pos", g["add_pos"], np.float64), put(d, "gen_add_normal", g["add_normal"], np.float64), put(d, "gen_state", g["state"], np.float64)
    put(d, "gen_img", g["img"], np.uint8), put(d, "gen_mask", g["mask"], np.uint8)


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    d = tmp_path_factory.mktemp("shim_staging")
    exe = str(d / "shim_staging_driver")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "shim_staging_driver.cpp"),
           "-L" + PKG, "-lfl2_shim", "-lesikf_b200", "-Wl,-rpath," + PKG, "-o", exe]
    build = subprocess.run(cmd, capture_output=True, text=True)
    assert build.returncode == 0, build.stderr
    inp = d / "in"
    inp.mkdir()
    write_inputs(str(inp))
    runs = [0]

    def run(*commands):
        runs[0] += 1
        out = d / f"out{runs[0]}"
        out.mkdir()
        r = subprocess.run([exe, str(inp), str(out), *commands], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        res = {}
        for f in os.listdir(out):
            tag, name = f[:-4].split(".", 1)
            res.setdefault(tag, {})[name] = (out / f).read_bytes()
        return res

    return run


def assert_same(got, want, label):
    assert sorted(got) == sorted(want), label
    for k in want:
        assert got[k] == want[k], f"{label}: {k} differs"


def assert_ok(answers, label):
    for k, v in answers.items():
        if k.endswith(".status"):
            assert np.frombuffer(v, np.int32)[0] == 0, f"{label}: {k}"


def assert_equals_c_abi(answers, label):
    """Every answer the driver also computed with the plain C-ABI call (<name>_abi) equals the method's."""
    pairs = [k for k in answers if k.endswith("_abi") and not k.endswith(".status")]
    assert pairs, label
    for k in pairs:
        assert answers[k] == answers[k[:-4]], f"{label}: {k[:-4]} differs from the C-ABI call"


def as_f64(answer):
    return np.frombuffer(answer, np.float64)


def test_methods_equal_the_c_abi(driver):
    got = driver("tick:L:L", "tick:S:S")
    for tag in ("L", "S"):
        assert_ok(got[tag], tag)
        assert_equals_c_abi(got[tag], tag)
    names = {k[:-4] for k in got["L"] if k.endswith("_abi") and not k.endswith(".status")}
    assert {"retrieve.keys", "depth.flags", "find.found", "find.planes", "select.errors", "select.levels", "select.index", "warp.patches", "colorize.cloud",
            "generate.points", "observe.flags", "observe.new", "patches.cur", "score.score", "score.mean", "score.ref", "affine.level"} <= names
    for k in ("retrieve.keys", "find.planes", "select.index", "warp.patches", "colorize.cloud", "observe.flags", "patches.cur", "score.score"):
        assert len(got["L"][k]) > 0, k


def test_score_reference_patches_equals_api_context(driver):
    got = driver("score:cases:cases", "score:none:none")
    c = score_cases()["cases"]
    ctx = api.Context(0)
    try:
        want = ctx.vio_score_ref_patches(c["first"], c["pos"], c["normal"], c["patch"], c["mean"], c["id"], c["T"])
    finally:
        ctx.close()
    assert_ok(got["cases"], "cases")
    for k in ("score", "mean", "ref"):
        assert got["cases"]["score." + k] == want[k].tobytes(), k
    # no points: the call answers nothing, and the method gives zero scores and means, one per observation
    assert_ok(got["none"], "none")
    assert got["none"]["score.score"] == got["none"]["score.mean"] == np.zeros(5, np.float32).tobytes() and got["none"]["score.ref"] == b""


def test_generate_visual_map_points_equals_api_context(driver):
    got = driver("generate:gen")["gen"]
    g = gen_case()
    ctx = api.Context(0)
    try:
        ctx.set_extrinsics(g["ext"])
        ctx.vio_set_camera(g["cam"], S.VioCfg())
        ctx.vio_set_image(g["img"])
        r = ctx.vio_generate_points(g["mask"], g["grid_size"], g["grid_n_width"], g["grid_n_height"], g["border"], pg=(g["point_w"], g["normal"], g["var"]),
                                    add_from=(g["add_pos"], g["add_normal"]), state=g["state"])
    finally:
        ctx.close()
    k = len(r["source"])
    assert k > 0
    want = np.concatenate([r["source"][:, None], r["cell"][:, None], r["pos"], r["pc"], r["normal"], r["var"].reshape(k, 9), r["score"][:, None], r["patch"]], 1)
    assert_ok(got, "generate")
    assert got["generate.points"] == want.astype(np.float64).tobytes()


def test_resident_scan_beyond_the_key_room(driver):
    """The first RetrieveScanVoxels of a resident scan with more keys than its first room calls again with more: after a
    large tick as on fresh managers, and as the C ABI. A second one (the room now fits) again as the C ABI; its map and
    pose differ from the first's, the wide scan having been added to the map."""
    got = driver("tick:L:t", "resident:first", "resident:again")
    want = driver("resident:fresh")["fresh"]
    assert_ok(want, "fresh")
    assert len(as_f64(want["resident.keys"])) // 3 > RESIDENT_ROOM
    assert want["resident.keys"] == want["resident.keys_abi"]
    assert_ok(got["first"], "first")
    assert_same(got["first"], want, "after a large tick")
    assert_ok(got["again"], "again")
    assert got["again"]["resident.keys"] == got["again"]["resident.keys_abi"]


def test_large_small_large_equals_fresh_managers(driver):
    got = driver("tick:L:r0", "tick:S:r1", "tick:L:r2")
    want = driver("tick:L:L", "new", "tick:S:S")
    for tag, size in (("r0", "L"), ("r1", "S"), ("r2", "L")):
        assert_ok(got[tag], tag)
        assert_same(got[tag], want[size], f"{tag} against a fresh pair")
    assert len(got["r0"]["colorize.cloud"]) > len(got["r1"]["colorize.cloud"]) > 0
    assert len(got["r0"]["select.index"]) > len(got["r1"]["select.index"]) > 0


def test_point_lists_survive_later_calls(driver):
    got = driver("lazy:S:lazy")
    want = driver("tick:S:now")
    assert_ok(got["lazy"], "lazy")
    lists = {k: v for k, v in want["now"].items() if k.startswith(("lio", "lists"))}
    assert_same(got["lazy"], lists, "lazy MaterializePointLists after UpdateVoxelMap, FindCorrespond and SetWorldCloud")


def test_selected_sub_map_survives_later_calls(driver):
    got = driver("select:S:later")
    want = driver("select_now:S:now")
    assert_ok(got["later"], "later")
    assert_ok(got["later_between"], "between")
    assert_same(got["later"], want["now"], "MaterializeWarpPatches and the update after the other front-end calls")


def test_failed_upload_then_larger_calls_equal_fresh_managers(driver):
    got = driver("tick:S:small", "failbuild:fail", "tick:L:large")
    want = driver("tick:L:L")
    assert np.frombuffer(got["fail"]["build.status"], np.int32)[0] != 0
    assert_same(got["large"], want["L"], "calls after a failed BuildVoxelMap")
