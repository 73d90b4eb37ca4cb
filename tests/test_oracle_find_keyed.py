"""CPU: the oracle's keyed find_correspond (oracle/orc_find_keyed.cpp), the lookups of updateReferencePatch and of the
retrieval's ray casting, checked against a numpy spelling of both key rules, against orc_lio_find_correspond where the two
agree (rule A at voxel 0.5), and against the reference source's own find_correspond (oracle/_ref/libfl2_ref_find.so) at voxel
0.5, where the reference's map keys its roots the way updateReferencePatch looks them up."""
import os

import numpy as np
import pytest

import map_find as MF
import map_mirror as MM
import map_streams as MS
from fast_livo2_b200 import synthetic as S
from test_map_mirror_host import ROOM_CFGS, export_all, room_ticks


def _map(cfg, ticks):
    orc, hm = MS.OracleSide(cfg), MM.HarnessMap(cfg)
    for pw, var in ticks:
        orc.apply(pw, var), hm.apply_touched(pw, var)
    return orc, hm


def test_key_rules_match_their_numpy_spelling():
    q = MF.boundary_points()
    orc, _ = _map(S.LioCfg(), list(room_ticks(S.LioCfg(), 1)))
    for rule, fn in ((0, MF.key_patch_numpy), (1, MF.key_raycast_numpy)):
        out, _ = MF.oracle_find_keyed(orc, q, rule)
        want = np.stack([fn(q[:, j]) for j in range(3)], axis=1)
        want[np.any(want == MF.NONE_KEY, axis=1)] = MF.NONE_KEY
        assert np.array_equal(out[:, 1:4], want), f"rule {rule}: keys differ on {int(np.any(out[:, 1:4] != want, axis=1).sum())} points"
        assert (out[np.any(want == MF.NONE_KEY, axis=1), 0] == 0).all()


def test_key_rules_reach_their_edges():
    """The boundary points separate the rules from each other and from floor(p / 0.5): rule A's float rounding lifts a key
    that floor would not, both subtract one from a negative exact multiple, -0.0 keys to 0, and keys at 2^20 are refused."""
    q = MF.boundary_points()[:, 0]
    a, b = MF.key_patch_numpy(q), MF.key_raycast_numpy(q)
    with np.errstate(invalid="ignore"):
        fl = np.floor(q / 0.5)
    ok = (a != MF.NONE_KEY) & (b != MF.NONE_KEY)
    assert np.any(ok & (a > fl)), "no quotient rounds up in float"
    assert np.any(ok & (a != b)), "the two rules never differ"
    assert MF.key_patch_numpy(-1.0) == -3 and MF.key_raycast_numpy(-1.0) == -3
    assert MF.key_patch_numpy(-0.0) == 0 and MF.key_raycast_numpy(-0.0) == 0
    assert MF.key_patch_numpy(2**20 * 0.5) == MF.NONE_KEY and MF.key_patch_numpy((2**20 - 0.25) * 0.5) == 2**20 - 1
    assert MF.key_patch_numpy(-(2**20) * 0.5) == MF.NONE_KEY and MF.key_patch_numpy(-(2**20 - 1) * 0.5) == -(2**20)
    assert MF.key_raycast_numpy(-(2**20 - 1) * 0.5) == -(2**20) and MF.key_raycast_numpy(-(2**20) * 0.5) == MF.NONE_KEY
    assert (MF.key_patch_numpy([np.nan, np.inf, -np.inf]) == MF.NONE_KEY).all() and (MF.key_raycast_numpy([np.nan, np.inf, -np.inf]) == MF.NONE_KEY).all()


@pytest.mark.parametrize("cfg", ROOM_CFGS, ids=["voxel0.5", "voxel0.4", "voxel2.0"])
def test_rule_a_at_voxel_half_is_orc_lio_find_correspond(cfg):
    """At voxel 0.5 updateReferencePatch's lookup is the map's own keying: the keyed restatement answers as
    orc_lio_find_correspond. At other voxel sizes the two key different roots and their answers differ somewhere."""
    orc, hm = _map(cfg, list(room_ticks(cfg, 3)))
    q = MM.query_points(export_all(hm, orc.flatten()["keys"])["nodes"], cfg, np.random.default_rng(4))
    out, _ = MF.oracle_find_keyed(orc, q, 0)
    old = MM.oracle_find(orc, q)
    mine = np.stack([out[:, 0] != 0, out[:, 4], out[:, 5], out[:, 0] == 2], axis=1).astype(np.int64)
    mine[out[:, 0] == 0, 1:] = 0
    if cfg.voxel_size == 0.5:
        assert np.array_equal(mine, old)
    else:
        assert not np.array_equal(mine, old)
    assert (out[:, 0] == 2).any() and (out[:, 0] == 0).any()


PIN_CFGS = {"voxel0.5": ROOM_CFGS[0], "voxel0.4": ROOM_CFGS[1], "voxel2.0": ROOM_CFGS[2]}
N_PATCH, N_CELLS, N_SAMPLES = 2500, 60, 24


def pin_inputs(name):
    """The pinned scene of one voxel size: three room ticks; rule A's query points (a sample of map_mirror.query_points on
    every node plus the finite key-rule edges); rule B's frame (a pose inside the room) and rays (one a cell, samples at depths
    0.5 to 12 m along a random camera-frame direction)."""
    cfg = PIN_CFGS[name]
    ticks = list(room_ticks(cfg, 3, seed=31))
    orc, hm = _map(cfg, ticks)
    rng = np.random.default_rng(6)
    q = MM.query_points(export_all(hm, orc.flatten()["keys"])["nodes"], cfg, rng)
    q = q[rng.choice(len(q), min(N_PATCH, len(q)), replace=False)]
    b = MF.boundary_points()
    q = np.concatenate([q, b[np.all(np.isfinite(b) & (np.abs(b) < 1e5), axis=1)]])
    state = S.pack_state(np.eye(3), np.array([-4.0, 0.3, 0.8]), cov=np.eye(19) * 1e-4, g=np.array([0, 0, -9.81]))
    depth = np.linspace(0.5, 12.0, N_SAMPLES)
    rays = []
    for _ in range(N_CELLS):
        d = np.array([rng.uniform(-0.7, 0.7), rng.uniform(-0.6, 0.6), 1.0])
        rays.append(depth[:, None] * d[None, :])
    return cfg, ticks, orc, q, state, rays


def ref_outputs(name, cfg, ticks, q, state, rays):
    """The reference's own updateReferencePatch and ray-casting retrieval on the reference's own map: live where oracle/_ref
    was built, else the stored outputs (checked to have been made on the same inputs)."""
    if MF.ref_available():
        ref = MF.RefKeyed(cfg, S.CamCfg(), S.avia_extrinsics(), S.VioCfg())
        for pw, var in ticks:
            ref.update(pw, var)
        normal = ref.update_reference_patch(q)
        samples_w, add = ref.raycast(state, rays)
        return dict(normal=normal, samples_w=samples_w, add=add)
    g = np.load(MF.GOLDEN)
    assert np.array_equal(g[f"{name}_points"], q), "the stored pin was made on other query points"
    return dict(normal=g[f"{name}_normal"], samples_w=g[f"{name}_samples_w"], add=g[f"{name}_add"])


needs_ref = pytest.mark.skipif(not MF.ref_available() and not os.path.exists(MF.GOLDEN), reason="needs oracle/_ref (reference source) or the stored pin")


@needs_ref
@pytest.mark.parametrize("name", list(PIN_CFGS))
def test_rule_a_is_pinned_to_update_reference_patch(name):
    """The reference's own updateReferencePatch, on stand-in visual points whose gates pass whenever a plane is found, sets
    normal_ to the normal of the plane the keyed restatement finds with rule A, and leaves it where the restatement finds no
    plane, at voxel 0.5 and at 0.4 and 2.0, where the literal 0.5 keys other roots than the map inserts."""
    cfg, ticks, orc, q, state, rays = pin_inputs(name)
    got = ref_outputs(name, cfg, ticks, q, state, rays)["normal"]
    out, f = MF.oracle_find_keyed(orc, q, 0)
    want, ambiguous = MF.expect_reference_patch(q, out, f)
    changed = np.any(got != 0, axis=1)
    assert not np.any(changed & (out[:, 0] != 2)), "the reference found a plane where the restatement finds none"
    np.testing.assert_allclose(got[changed], want[changed], rtol=0, atol=1e-12)
    assert np.all(changed | ~(out[:, 0] == 2) | ambiguous), "the restatement finds a plane the reference does not take"
    assert changed.sum() > (100 if cfg.voxel_size < 1 else 0) and (out[:, 0] == 0).any()  # at 2.0 the 0.5 m keys rarely name a root
    if cfg.voxel_size != 0.5:  # rule A differs from the map's own keying somewhere on these points
        mine = np.stack([out[:, 0] != 0, out[:, 4], out[:, 5], out[:, 0] == 2], axis=1).astype(np.int64)
        mine[out[:, 0] == 0, 1:] = 0
        assert not np.array_equal(mine, MM.oracle_find(orc, q))


@needs_ref
@pytest.mark.parametrize("name", list(PIN_CFGS))
def test_rule_b_is_pinned_to_the_ray_casting_retrieval(name):
    """The reference's own retrieveFromVisualSparseMap with raycast_en on, an empty scan and no visual points on the rays:
    add_from_voxel_map holds, cell by cell, the plane the keyed restatement finds with rule B for the first sample of the
    cell's ray that finds one."""
    cfg, ticks, orc, q, state, rays = pin_inputs(name)
    r = ref_outputs(name, cfg, ticks, q, state, rays)
    out, f = MF.oracle_find_keyed(orc, r["samples_w"], 1)
    want = MF.expect_raycast(r["samples_w"], [len(x) for x in rays], out, f)
    assert len(r["add"]) == len(want), (len(r["add"]), len(want))
    np.testing.assert_allclose(r["add"], want, rtol=0, atol=1e-12)
    assert 0 < len(want) < len(rays) or cfg.voxel_size != 0.5
    assert len(want) > 0
