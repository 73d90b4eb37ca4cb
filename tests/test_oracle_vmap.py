"""CPU: the oracle's restatement of the observation store's list edits and reference choice (oracle/orc_vmap.cpp, driven by
tests/vmap_cases.OracleStore) against the reference source's own VisualPoint / Feature objects (oracle/_ref/libfl2_ref_vmap.so,
live where it was built, else its stored outputs in tests/golden/ref_pin/vmap.npz) over the seeded tick sequence that
tests/test_gpu_vmap.py holds the device to, and on hand-built states; and on hand-built states whose outcome follows from the
reference's code."""
import os

import numpy as np
import pytest

import vmap_cases as VC
from fast_livo2_b200 import synthetic as S


def _hand():
    cam, ext = VC.OC.CAMERAS["pinhole"]
    R, p = S.so3_exp(np.array([0.01, -0.02, 0.03])), np.array([0.3, -0.2, 0.1])
    T_near, pts = VC.hand_lists(np.random.default_rng(3), cam, ext, R, p)
    st = VC.OracleStore(cam, ext, capacity=64)
    ids = st.add(**VC.lists_of(pts))
    sc = dict(img=VC.OC.grey_image(cam, 9), state=S.pack_state(R, p, 1.0), pos=np.array([q["pos"] for q in pts]))
    return st, pts, ids, sc, T_near


def test_hand_built_edits_follow_the_reference():
    """Eviction of the first strict minimum from FLT_MAX (ties, NaN, FLT_MAX, inf), of the ref, of the oldest observation on
    the tick it decides the flag, and deleteNonRefPatchFeatures with and without a ref."""
    st, pts, ids, sc, T_near = _hand()
    conv = np.array([q["conv"] for q in pts], np.uint8)
    before = {q["name"]: st.download([i]) for q, i in zip(pts, ids)}
    o = st.update(ids, conv, sc, frame_id=77, T_new=T_near)
    got = {q["name"]: (int(f), int(e), int(c), int(st.ref[i])) for q, i, f, e, c in zip(pts, ids, o["update_flag"], o["evicted"], o["count"])}
    assert got == {"tie": (0, 3, 29, 9), "nan": (0, 0, 29, 3), "flt_max": (0, 0, 29, -1), "inf": (0, 0, 29, 24), "evict_ref": (0, 15, 29, -1),
                   "oldest_decides": (1, 29, 30, 3), "far_29": (1, -1, 30, 2), "conv_ref": (0, -1, 1, 0), "conv_noref": (0, -1, 0, -1), "near": (0, -1, 5, -1)}
    # the lists: the survivors in order, the new observation in front with the frame's pose, id_, mean_ 0 and score_ 0
    d = st.download([ids[[q["name"] for q in pts].index("oldest_decides")]])
    b = before["oldest_decides"]
    assert d["T_f_w"][1:].tobytes() == b["T_f_w"][:29].tobytes() and d["patch"][1:].tobytes() == b["patch"][:29].tobytes()
    assert d["T_f_w"][0].tobytes() == T_near.tobytes() and d["id"][0] == 77 and d["mean"][0] == 0 and d["score"][0] == 0
    d = st.download([ids[[q["name"] for q in pts].index("tie")]])
    keep = [j for j in range(30) if j != 3]
    assert d["patch"].tobytes() == before["tie"]["patch"][keep].tobytes() and d["score"].tobytes() == before["tie"]["score"][keep].tobytes()
    d = st.download([ids[[q["name"] for q in pts].index("conv_ref")]])
    assert d["patch"].tobytes() == before["conv_ref"]["patch"][3:4].tobytes()


def test_reference_choice_follows_the_reference():
    cam, ext = VC.OC.CAMERAS["pinhole"]
    rng = np.random.default_rng(4)
    pos, fp = np.array([1.0, -2.0, 14.0]), np.array([0.2, 0.1, -0.3])
    lists = VC.choose_lists(rng, pos, fp)
    st = VC.OracleStore(cam, ext, capacity=16)
    ids = st.add(**VC.lists_of(lists))
    names = [q["name"] for q in lists]
    q = lists[names.index("noref")]
    errs = []
    for r in range(q["c"]):
        e, cnt = np.float32(0), 0
        for j in range(q["c"]):
            if q["id"][j] != q["id"][r]:
                e = _acc(e, q["patch"][r], q["patch"][j])
                cnt += 1
        errs.append(np.float32(e / np.float32(cnt)))
    want_noref = int(np.argmin(errs))
    ref = dict(zip(names, st.choose(ids, True).tolist()))
    assert {k: ref[k] for k in ("one", "noref", "ref", "same_ids")} == {"one": 0, "noref": want_noref, "ref": 1, "same_ids": -1}
    assert min(ref["wide"], ref["mixed"], ref["behind"]) >= 0
    assert st.ref[ids[names.index("one")]] == 0 and st.ref[ids[names.index("noref")]] == want_noref and st.ref[ids[names.index("same_ids")]] == -1
    # getCloseViewObs: the smallest angle wins where its cosine is at least 0.5 (60 degrees); 61 degrees and more: -1
    ref = st.choose(ids, False, pos=np.tile(pos, (len(ids), 1)), frame_pos=fp)
    assert dict(zip(names, ref.tolist())) == {"one": 0, "noref": 0, "ref": 2, "same_ids": 2, "wide": -1, "mixed": 2, "behind": -1}


def _acc(e, a, b):
    """the running float sum of the squared differences of one more observation"""
    for x, y in zip(a, b):
        d = np.float32(x - y)
        e = np.float32(e + np.float32(d * d))
    return e


needs_ref = pytest.mark.skipif(not VC.ref_available() and not os.path.exists(VC.GOLDEN), reason="needs oracle/_ref (reference source) or the stored pin")


def _split(a, n):
    return np.split(a, np.cumsum(n)[:-1])


def _reference_sequence():
    """The reference's per-tick outputs: live where oracle/_ref was built, else the stored ones (made on the same inputs)."""
    if VC.ref_available():
        return VC.reference_sequence()
    g = np.load(VC.GOLDEN)
    return dict(flag=_split(g["seq_flag"], g["seq_flag_n"]), T=list(g["seq_T"]), close=_split(g["seq_close"], g["seq_close_n"]), digest=list(g["seq_digest"]),
                has_ref_ok=[True])


@needs_ref
def test_tick_sequence_equals_the_reference_after_every_tick():
    """44 ticks of generate -> sub-map -> update points -> score -> getCloseViewObs: after every tick every point's list (count,
    order, px_, T_f_w_, id_, patch_, mean_, score_, ref_patch) is the reference's bit for bit; the run reaches 30 observations,
    evictions, converged points with and without a ref, and the re-scoring of points that already have a ref."""
    r = _reference_sequence()
    assert all(r["has_ref_ok"])  # has_ref_patch_ is set exactly where ref_patch is
    cam, ext, ticks = VC.sequence()
    st = VC.OracleStore(cam, ext)
    seen = dict(full=0, evicted=0, conv_ref=0, conv_noref=0, rescored=0, close=0)
    for i, tk in enumerate(ticks):
        st.add(**tk["add"])
        had_ref = st.ref[tk["sub"]] >= 0
        o = st.update(tk["sub"], tk["converged"], tk, frame_id=tk["t"], T_new=r["T"][i])
        assert np.array_equal(o["update_flag"], r["flag"][i]), f"tick {i}: flags"
        seen["full"] += int((st.count[:st.points] == 30).sum())
        seen["evicted"] += int((o["evicted"] >= 0).sum())
        seen["conv_ref"] += int(((tk["converged"] == 1) & (o["count"] == 1)).sum())
        seen["conv_noref"] += int(((tk["converged"] == 1) & (o["count"] == 0)).sum())
        sel = VC.scored(o["update_flag"], tk["converged"], o["count"])
        seen["rescored"] += int((sel & had_ref).sum())
        st.score_points(tk["sub"][sel], tk["pos"][sel], tk["normal"][tk["sub"][sel]])
        close = st.choose(tk["ret"], False, pos=tk["all_pos"][tk["ret"]], frame_pos=tk["frame_pos"])
        assert np.array_equal(close, r["close"][i]), f"tick {i}: getCloseViewObs"
        seen["close"] += int((close >= 0).sum())
        d = VC.list_digests(st.download(np.arange(st.points)))
        bad = [f for f, a, b in zip(VC.LIST_FIELDS, d, r["digest"][i]) if a != b]
        assert not bad, f"tick {i}: {bad} differ from the reference"
    assert len(ticks) >= 40 and all(v > 0 for v in seen.values()), seen


@needs_ref
def test_hand_built_states_equal_the_reference():
    """The hand-built evictions (ties, NaN, FLT_MAX, inf, the ref, the oldest observation on the tick it sets the flag),
    converged points with and without a ref, and getCloseViewObs on cosines on both sides of 0.5: the reference's lists."""
    if VC.ref_available():
        r = VC.reference_hand()
    else:
        g = np.load(VC.GOLDEN)
        r = {k[5:]: g[k] for k in g.files if k.startswith("hand_")}
    cam, ext, T_near, pts, sc, lists, cpos, fp = VC.hand_case()
    st = VC.OracleStore(cam, ext, capacity=64)
    ids = st.add(**VC.lists_of(pts))
    o = st.update(ids, [q["conv"] for q in pts], sc, frame_id=77, T_new=r["T"])
    assert np.array_equal(o["update_flag"], r["flag"])
    d = st.download(ids)
    assert VC.same_lists(d, {k: r[f"list_{k}"] for k in VC.LIST_FIELDS}) is None
    assert np.array_equal(r["list_has_ref"], (r["list_ref"] >= 0).astype(np.uint8))
    c = VC.OracleStore(cam, ext, capacity=16)
    cid = c.add(**VC.lists_of(lists))
    assert np.array_equal(c.choose(cid, False, pos=np.tile(cpos, (len(cid), 1)), frame_pos=fp), r["close"])
