"""GPU: the visual map's observation store (esikf_vmap_*) against the oracle's host copy (tests/vmap_cases.OracleStore) on a
seeded sequence of VIO ticks and on hand-built states, bit for bit with a pinhole camera; the store's scoring and flags
against the packed entry points (esikf_vio_score_ref_patches, esikf_vio_update_points) on the same lists; growth; refusals."""
import numpy as np
import pytest

import shim_bind as SB
import vmap_cases as VC
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _install(ctx, cam, ext, img, pos):
    n = len(pos)
    ctx.set_extrinsics(ext)
    ctx.vio_set_camera(cam, S.VioCfg())
    ctx.vio_set_image(img)
    ctx.vio_set_patches(np.ascontiguousarray(pos), np.zeros((n, 4 * 64), np.float32), np.zeros(n, np.int32), np.ones(n))


def _same_update(got, want, label):
    for k in ("update_flag", "entry", "pc", "patch", "evicted", "count"):
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), f"{label}: {k}"


def _same_store(ctx, st, label):
    ids = np.arange(st.points, dtype=np.int32)
    bad = VC.same_lists(ctx.vmap_download(ids), st.download(ids))
    assert bad is None, f"{label}: {bad} differs"


def test_tick_sequence_matches_the_oracle(gpu_ctx):
    """44 ticks of generate -> sub-map -> update points -> score -> getCloseViewObs (the sequence tests/test_oracle_vmap.py
    holds the restatement to the reference source on): every point's list, count, order, px_, T_f_w_,
    id_, patch_, mean_, score_ and ref after every tick, and every call's outputs."""
    cam, ext, ticks = VC.sequence()
    st = VC.OracleStore(cam, ext)
    gpu_ctx.vmap_init(16)
    for tk in ticks:
        label = f"tick {tk['t']}"
        assert np.array_equal(gpu_ctx.vmap_add_points(**tk["add"]), st.add(**tk["add"]))
        _install(gpu_ctx, cam, ext, tk["img"], tk["pos"])
        got = gpu_ctx.vmap_update_points(tk["sub"], tk["converged"], tk["t"], T_f_w=tk["T_new"], state=tk["state"])
        want = st.update(tk["sub"], tk["converged"], tk, frame_id=tk["t"], T_new=tk["T_new"])
        _same_update(got, want, label)
        sel = VC.scored(want["update_flag"], tk["converged"], want["count"])
        pid = tk["sub"][sel]
        g, w = gpu_ctx.vmap_score(pid, tk["pos"][sel], tk["normal"][pid]), st.score_points(pid, tk["pos"][sel], tk["normal"][pid])
        for k in ("ref", "score", "mean"):
            assert g[k].tobytes() == w[k].tobytes(), f"{label}: score {k}"
        pos = tk["all_pos"][tk["ret"]]
        g = gpu_ctx.vmap_choose_ref(tk["ret"], False, pos=pos, frame_pos=tk["frame_pos"])
        assert np.array_equal(g, st.choose(tk["ret"], False, pos=pos, frame_pos=tk["frame_pos"])), f"{label}: choose"
        _same_store(gpu_ctx, st, label)
    counts = np.diff(gpu_ctx.vmap_download(np.arange(st.points, dtype=np.int32))["first"])
    assert counts.max() == 30 and (counts == 0).any() and gpu_ctx.vmap_stats()[1] >= st.points


def _hand(ctx):
    cam, ext = VC.OC.CAMERAS["pinhole"]
    R, p = S.so3_exp(np.array([0.01, -0.02, 0.03])), np.array([0.3, -0.2, 0.1])
    T_near, pts = VC.hand_lists(np.random.default_rng(3), cam, ext, R, p)
    sc = dict(img=VC.OC.grey_image(cam, 9), state=S.pack_state(R, p, 1.0), pos=np.array([q["pos"] for q in pts]))
    st = VC.OracleStore(cam, ext, capacity=64)
    ids = st.add(**VC.lists_of(pts))
    ctx.vmap_init(64)
    assert np.array_equal(ctx.vmap_add_points(**VC.lists_of(pts)), ids)
    _install(ctx, cam, ext, sc["img"], sc["pos"])
    return cam, ext, st, pts, ids, sc, T_near


def test_hand_built_edits_match_the_oracle(gpu_ctx):
    """Eviction under tied, NaN, FLT_MAX and inf scores, of the ref, of the oldest observation on the tick it decides the flag,
    and converged points with and without a ref."""
    cam, ext, st, pts, ids, sc, T_near = _hand(gpu_ctx)
    conv = np.array([q["conv"] for q in pts], np.uint8)
    got = gpu_ctx.vmap_update_points(ids, conv, 77, T_f_w=T_near, state=sc["state"])
    want = st.update(ids, conv, sc, frame_id=77, T_new=T_near)
    _same_update(got, want, "hand")
    _same_store(gpu_ctx, st, "hand")
    names = [q["name"] for q in pts]
    assert got["evicted"][names.index("tie")] == 3 and got["count"][names.index("conv_noref")] == 0
    assert got["update_flag"][names.index("oldest_decides")] == 1 and got["evicted"][names.index("oldest_decides")] == 29


def test_frame_pose_of_the_flags_is_the_default_new_pose(gpu_ctx):
    """T_f_w = NULL stores the frame pose the flags were computed with: the same lists as that pose passed explicitly."""
    cam, ext, st, pts, ids, sc, T_near = _hand(gpu_ctx)
    conv = np.zeros(len(ids), np.uint8)
    got = gpu_ctx.vmap_update_points(ids, conv, 5, state=sc["state"])
    a = gpu_ctx.vmap_download(ids)
    T0 = a["T_f_w"][a["first"][:-1][got["count"] == 30][0]]
    assert np.abs(T0 - T_near).max() < 1e-12  # the frame pose of the flags
    _, _, st2, _, ids2, _, _ = _hand(gpu_ctx)
    gpu_ctx.vmap_update_points(ids2, conv, 5, T_f_w=T0, state=sc["state"])
    assert VC.same_lists(gpu_ctx.vmap_download(ids2), a) is None


def test_store_flags_equal_the_packed_update_points(gpu_ctx):
    """esikf_vmap_update_points' flags, entries, pixels and patches are esikf_vio_update_points' with the oldest observations
    passed explicitly."""
    cam, ext, ticks = VC.sequence(ticks=12)
    gpu_ctx.vmap_init(4096)
    for tk in ticks[:-1]:
        gpu_ctx.vmap_add_points(**tk["add"])
    tk = ticks[-1]
    gpu_ctx.vmap_add_points(**tk["add"])
    sub = tk["sub"]
    d = gpu_ctx.vmap_download(sub)
    last = d["first"][1:] - 1
    _install(gpu_ctx, cam, ext, tk["img"], tk["pos"])
    want = gpu_ctx.vio_update_points(tk["converged"], d["T_f_w"][last], d["px"][last], state=tk["state"])
    got = gpu_ctx.vmap_update_points(sub, tk["converged"], tk["t"], T_f_w=tk["T_new"], state=tk["state"])
    for k in ("update_flag", "entry", "pc", "patch"):
        assert got[k].tobytes() == want[k].tobytes(), k


def test_store_scoring_equals_the_packed_scoring(gpu_ctx):
    """esikf_vmap_score on the store equals esikf_vio_score_ref_patches on the downloaded lists; a ref is kept where no score
    beats -1000 (every observation of one id_: NaN)."""
    cam, ext, ticks = VC.sequence(ticks=30)
    gpu_ctx.vmap_init(4096)
    for tk in ticks:
        gpu_ctx.vmap_add_points(**tk["add"])
        _install(gpu_ctx, cam, ext, tk["img"], tk["pos"])
        gpu_ctx.vmap_update_points(tk["sub"], tk["converged"], tk["t"], T_f_w=tk["T_new"], state=tk["state"])
    rng = np.random.default_rng(1)
    c = 6
    same = dict(first=np.array([0, c], np.int32), px=np.zeros((c, 2)), patch=rng.normal(100, 20, (c, 64)).astype(np.float32),
                T_f_w=np.tile(np.concatenate([np.eye(3).reshape(9), [0.0, 0.0, 0.0]]), (c, 1)), id=np.full(c, 3, np.int32),
                mean=np.zeros(c, np.float32), score=np.zeros(c, np.float32), ref=np.array([2], np.int32))
    sid = gpu_ctx.vmap_add_points(**same)[0]
    n = gpu_ctx.vmap_stats()[0]
    ids = np.arange(n, dtype=np.int32)
    d = gpu_ctx.vmap_download(ids)
    assert np.diff(d["first"]).max() >= 20
    pos = np.concatenate([ticks[-1]["all_pos"], [[0.0, 0.0, 10.0]]])
    normal = np.concatenate([ticks[-1]["normal"], [[0.0, 0.0, -1.0]]])
    want = gpu_ctx.vio_score_ref_patches(d["first"], pos, normal, d["patch"], d["mean"], d["id"], d["T_f_w"])
    got = gpu_ctx.vmap_score(ids, pos, normal)
    assert got["ref"].tobytes() == want["ref"].tobytes() and (want["ref"] >= 0).sum() > 100
    counts = np.diff(d["first"])
    assert np.concatenate([got["score"][i, :k] for i, k in enumerate(counts)]).tobytes() == want["score"].tobytes()
    assert np.concatenate([got["mean"][i, :k] for i, k in enumerate(counts)]).tobytes() == want["mean"].tobytes()
    after = gpu_ctx.vmap_download(ids)
    assert after["score"].tobytes() == want["score"].tobytes() and after["mean"].tobytes() == want["mean"].tobytes()
    assert got["ref"][sid] == -1 and after["ref"][sid] == 2  # the reference leaves ref_patch alone
    keep = want["ref"] >= 0
    assert np.array_equal(after["ref"][keep], want["ref"][keep]) and np.array_equal(after["ref"][~keep], d["ref"][~keep])


def test_reference_choice_matches_the_oracle(gpu_ctx):
    cam, ext = VC.OC.CAMERAS["pinhole"]
    pos, fp = np.array([1.0, -2.0, 14.0]), np.array([0.2, 0.1, -0.3])
    lists = VC.choose_lists(np.random.default_rng(4), pos, fp)
    st = VC.OracleStore(cam, ext, capacity=16)
    ids = st.add(**VC.lists_of(lists))
    gpu_ctx.vmap_init(16)
    gpu_ctx.vmap_add_points(**VC.lists_of(lists))
    P = np.tile(pos, (len(ids), 1))
    for normal_en in (False, True, False, True):
        g = gpu_ctx.vmap_choose_ref(ids, normal_en, pos=P, frame_pos=fp)
        assert np.array_equal(g, st.choose(ids, normal_en, pos=P, frame_pos=fp)), normal_en
        _same_store(gpu_ctx, st, f"choose {normal_en}")


def test_grown_store_downloads_as_a_large_one(gpu_ctx):
    """A store grown from capacity 1 (by doubling on every add that outgrows it) holds the bytes of one created large."""
    cam, ext, ticks = VC.sequence(ticks=14)
    small, large = gpu_ctx, api.Context(0)
    try:
        small.vmap_init(1)
        large.vmap_init(8192)
        for c in (small, large):
            for tk in ticks:
                c.vmap_add_points(**tk["add"])
                _install(c, cam, ext, tk["img"], tk["pos"])
                c.vmap_update_points(tk["sub"], tk["converged"], tk["t"], T_f_w=tk["T_new"], state=tk["state"])
        n, cap = small.vmap_stats()
        assert cap == 1 << (n - 1).bit_length() and large.vmap_stats() == (n, 8192)
        ids = np.arange(n, dtype=np.int32)
        assert VC.same_lists(small.vmap_download(ids), large.vmap_download(ids)) is None
    finally:
        large.close()


def test_refusals_write_nothing(gpu_ctx):
    cam, ext, st, pts, ids, sc, T_near = _hand(gpu_ctx)
    n = len(ids)
    before = gpu_ctx.vmap_download(ids)
    assert VC.same_lists(gpu_ctx.vmap_download(ids), before) is None  # a pure read
    sentinel = np.full(n, 12345, np.int32)
    conv = np.zeros(n, np.uint8)
    bad_ids = (np.array([0, 0] + list(range(2, n)), np.int32), np.array(list(range(n - 1)) + [n], np.int32), np.array([-1] + list(range(1, n)), np.int32))
    for b in bad_ids:
        for call in (lambda: gpu_ctx.vmap_update_points(b, conv, 1, state=sc["state"]), lambda: gpu_ctx.vmap_score(b, sc["pos"], sc["pos"]),
                     lambda: gpu_ctx.vmap_choose_ref(b, True), lambda: gpu_ctx.vmap_download(b)):
            with pytest.raises(api.EsikfError, match="status -3"):
                call()
    with pytest.raises(api.EsikfError, match="status -3"):  # n differs from the installed sub-map's count
        gpu_ctx.vmap_update_points(ids[:-1], conv[:-1], 1, state=sc["state"])
    with pytest.raises(api.EsikfError, match="status -3"):  # 31 observations
        gpu_ctx.vmap_add_points(np.array([0, 31], np.int32), np.zeros((31, 2)), np.zeros((31, 64)), np.zeros((31, 12)), np.zeros(31), np.zeros(31),
                                np.zeros(31), np.array([-1]))
    with pytest.raises(api.EsikfError, match="status -3"):  # cap below the new observations: the store is left as it was
        gpu_ctx.vmap_update_points(ids, conv, 1, state=sc["state"], cap=0)
    assert gpu_ctx.vmap_stats()[0] == n
    assert VC.same_lists(gpu_ctx.vmap_download(ids), before) is None
    # the C ABI leaves the caller's buffers alone on a refusal
    import ctypes as C
    dup = np.array([1, 1], np.int32)
    out = sentinel.copy()
    rc = gpu_ctx.lib.esikf_vmap_choose_ref(gpu_ctx.h, 2, dup.ctypes.data, None, None, 1, out.ctypes.data)
    assert rc == -3 and np.array_equal(out, sentinel)
    fresh = api.Context(0)
    try:
        pts_, cap_ = C.c_int64(0), C.c_int64(0)
        assert fresh.lib.esikf_vmap_stats(fresh.h, C.byref(pts_), C.byref(cap_)) == -4  # before esikf_vmap_init
        assert fresh.lib.esikf_vmap_choose_ref(fresh.h, 0, None, None, None, 1, None) == -4
    finally:
        fresh.close()


def test_shim_overloads_equal_the_c_abi(gpu_ctx):
    """VIOManager::EnableDeviceObservations / AddVisualPoints / UpdateVisualMapPoints / ScoreReferencePatches /
    ChooseReferenceFeatures on one context equal esikf_vmap_* on another over 12 ticks: every output and every list."""
    import ctypes as C

    shim = SB.load()
    cam, ext, ticks = VC.sequence(ticks=12)
    other = api.Context(0)
    try:
        gpu_ctx.vmap_init(4)
        assert shim.fl2_shim_vmap_enable(other.h, 4) == 0
        for tk in ticks:
            a = {k: np.ascontiguousarray(v) for k, v in tk["add"].items()}
            n_add = len(a["ref"])
            ids = np.zeros(n_add, np.int32)
            assert shim.fl2_shim_vmap_add(other.h, n_add, *[a[k].ctypes.data for k in ("first", "px", "patch", "T_f_w", "id", "mean", "score", "ref")],
                                          ids.ctypes.data) == 0
            assert np.array_equal(ids, gpu_ctx.vmap_add_points(**tk["add"]))
            for c in (gpu_ctx, other):
                _install(c, cam, ext, tk["img"], tk["pos"])
            sub, conv = np.ascontiguousarray(tk["sub"]), np.ascontiguousarray(tk["converged"], np.uint8)
            n = len(sub)
            want = gpu_ctx.vmap_update_points(sub, conv, tk["t"], state=tk["state"])
            cnt = C.c_int32(0)
            got = dict(update_flag=np.zeros(n, np.uint8), entry=np.zeros(n, np.int32), pc=np.zeros((n, 2)), patch=np.zeros((n, 64), np.float32),
                       evicted=np.zeros(n, np.int32), count=np.zeros(n, np.int32))
            st = np.ascontiguousarray(tk["state"])
            assert shim.fl2_shim_vmap_update(other.h, st.ctypes.data, n, sub.ctypes.data, conv.ctypes.data, tk["t"], C.byref(cnt),
                                             *[got[k].ctypes.data for k in ("update_flag", "entry", "pc", "patch", "evicted", "count")]) == 0
            k = cnt.value
            got.update(entry=got["entry"][:k], pc=got["pc"][:k], patch=got["patch"][:k])
            _same_update(got, want, f"shim tick {tk['t']}")
            sel = VC.scored(want["update_flag"], conv, want["count"])
            pid = np.ascontiguousarray(sub[sel])
            pos, normal = np.ascontiguousarray(tk["pos"][sel]), np.ascontiguousarray(tk["normal"][pid])
            ref = np.zeros(max(len(pid), 1), np.int32)
            assert shim.fl2_shim_vmap_score(other.h, len(pid), pid.ctypes.data, pos.ctypes.data, normal.ctypes.data, ref.ctypes.data) == 0
            assert np.array_equal(ref[:len(pid)], gpu_ctx.vmap_score(pid, pos, normal)["ref"])
            ret = np.ascontiguousarray(tk["ret"])
            rpos, fp = np.ascontiguousarray(tk["all_pos"][ret]), np.ascontiguousarray(tk["frame_pos"])
            for normal_en in (False, tk["t"] % 2 == 0):
                ref = np.zeros(len(ret), np.int32)
                assert shim.fl2_shim_vmap_choose(other.h, len(ret), ret.ctypes.data, rpos.ctypes.data, fp.ctypes.data, int(normal_en), ref.ctypes.data) == 0
                assert np.array_equal(ref, gpu_ctx.vmap_choose_ref(ret, normal_en, pos=rpos, frame_pos=fp))
            ids_all = np.arange(gpu_ctx.vmap_stats()[0], dtype=np.int32)
            assert VC.same_lists(other.vmap_download(ids_all), gpu_ctx.vmap_download(ids_all)) is None
    finally:
        other.close()
