"""CPU: capacity growth of the device voxel map (esikf_map_cfg.grow), on the state machine compiled for the host
(tests/map_growth_harness.cu, which is tests/map_host_harness.cu plus the growth entry points):

  * the demand bound (map_root_demand, esikf_map.cuh) is never below what a root's replay takes, for every root, every
    resource and every tick of the room ticks, the build form, every hand-built stream and the voxel-face key grid;
  * a map grown from minimal capacities by the demand -> grow -> apply policy equals the oracle's bit for bit, also around
    slides, and every resource did grow."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__
import map_bind as MB
import map_streams as MS
import oracle_bind as O
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from map_bind import oracle_map, oracle_update_map, tick_points

RESOURCES = ("nodes", "pool", "recs")
MAP_ERR = {"nodes": 1, "pool": 2, "recs": 4, "hash": 8}
TINY = dict(hash_cap=64, node_cap=16, pool_cap=64, rec_cap=4)


class GrowMap(MB.HostMap):
    """HostMap on tests/map_growth_harness.cu: the host harness itself plus its growth entry points."""

    def __init__(self, cfg, hash_cap=1 << 16, node_cap=1 << 16, pool_cap=1 << 19, rec_cap=1 << 16):
        MB.build()  # builds both host harnesses
        self.lib = L = C.CDLL(__graft_entry__.MAP_GROWTH_HARNESS_LIB)
        L.maph_create.restype = C.c_void_p
        L.maph_create.argtypes = [C.c_float, C.c_float, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_int]
        L.maph_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.maph_flatten.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.maph_usage.argtypes = [C.c_void_p, C.c_void_p]
        L.maph_destroy.argtypes = [C.c_void_p]
        L.maph_slide.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.maph_dump_nodes.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.maph_slots_used.argtypes = [C.c_void_p]
        L.maph_apply_roots.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.maph_demand.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.maph_grow.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_int]
        L.maph_capacity.argtypes = [C.c_void_p, C.c_void_p]
        L.maph_apply_grow.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        lin = O.layer_init_num8(cfg)
        self.h = L.maph_create(cfg.voxel_size, cfg.min_eigen_value, cfg.max_layer, cfg.max_points_num, lin.ctypes.data, hash_cap, node_cap, pool_cap, rec_cap)
        self.grew = 0  # MAP_ERR bits of every resource that grew so far

    @staticmethod
    def _pt(pw, var):
        return np.ascontiguousarray(np.concatenate([np.asarray(pw, np.float64).reshape(-1, 3), np.asarray(var, np.float64).reshape(-1, 9)], axis=1))

    def apply_roots(self, pw, var, build=False):
        """Apply a tick root by root: [roots][6] = demand bound (nodes, pool, recs) | what the replay took."""
        pt = self._pt(pw, var)
        out = np.zeros((max(len(pt), 1), 6), np.int64)
        err = C.c_int(0)
        r = self.lib.maph_apply_roots(self.h, pt.ctypes.data, len(pt), 1 if build else 0, out.ctypes.data, len(out), C.byref(err))
        assert err.value == 0, err.value
        return out[:r]

    def apply_grow(self, pw, var, build=False):
        pt = self._pt(pw, var)
        grew = C.c_int(0)
        e = self.lib.maph_apply_grow(self.h, pt.ctypes.data, len(pt), 1 if build else 0, C.byref(grew))
        self.grew |= grew.value
        return e

    def grow(self, hash_cap, node_cap, pool_cap, rec_cap):
        return self.lib.maph_grow(self.h, hash_cap, node_cap, pool_cap, rec_cap)

    def capacity(self):
        c = np.zeros(4, np.int64)
        self.lib.maph_capacity(self.h, c.ctypes.data)
        return dict(hash=int(c[0]), nodes=int(c[1]), pool=int(c[2]), recs=int(c[3]))


class Tally:
    """Per scenario: every root's bound against its actual use; the totals give the bound / actual ratio."""

    def __init__(self):
        self.bound, self.actual, self.roots = np.zeros(3, np.int64), np.zeros(3, np.int64), 0

    def add(self, rows, what):
        bad = np.nonzero(np.any(rows[:, :3] < rows[:, 3:], axis=1))[0]
        assert len(bad) == 0, f"{what}: {len(bad)} roots take more than their bound; first bound {rows[bad[0], :3]} actual {rows[bad[0], 3:]}"
        self.bound += rows[:, :3].sum(0)
        self.actual += rows[:, 3:].sum(0)
        self.roots += len(rows)

    def report(self, name):
        ratio = {r: (self.bound[i] / self.actual[i] if self.actual[i] else float("inf")) for i, r in enumerate(RESOURCES)}
        print(f"\n[demand bound] {name}: {self.roots} root replays, bound / actual " + ", ".join(f"{r} {ratio[r]:.2f}" for r in RESOURCES))
        return ratio


ROOM_CFGS = [S.LioCfg(), S.LioCfg(voxel_size=0.4, max_layer=3, max_points_num=20), S.LioCfg(voxel_size=2.0, max_layer=1, min_eigen_value=0.0005)]
ROOM_IDS = ["avia_defaults", "voxel0.4_layer3_max20", "voxel2.0_layer1"]


def _room_tick(rng, rects, tick):
    lo = np.array([-10.0 + 1.5 * tick, -8.0, -2.0])
    return tick_points(rng, rects, 6000, lo, lo + np.array([8.0, 16.0, 6.0]))


@pytest.mark.parametrize("cfg", ROOM_CFGS, ids=ROOM_IDS)
def test_demand_bound_covers_every_root_of_ten_room_ticks(cfg):
    rng, rects = np.random.default_rng(5), S.make_scene("room", 0.5)
    gm, t = GrowMap(cfg), Tally()
    for tick in range(10):
        pw, var = _room_tick(rng, rects, tick)
        t.add(gm.apply_roots(pw, var), f"tick {tick}")
    assert np.all(t.actual > 0)
    t.report(f"room {cfg.voxel_size} / layer {cfg.max_layer}")


def test_demand_bound_covers_the_build_form_and_the_ticks_after_it():
    cfg = S.LioCfg()
    rng, rects = np.random.default_rng(9), S.make_scene("room", 0.5)
    lo, hi = np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0])
    gm, t = GrowMap(cfg), Tally()
    pw, var = tick_points(rng, rects, 40000, lo, hi)
    t.add(gm.apply_roots(pw, var, build=True), "build")
    for tick in range(5):
        pw, var = tick_points(rng, rects, 5000, lo, hi)
        t.add(gm.apply_roots(pw, var), f"tick {tick}")
    assert np.all(t.actual > 0)
    t.report("build form + 5 ticks")


class _BoundSide:
    """replay()'s side interface over GrowMap.apply_roots, tallying every tick."""

    def __init__(self, cfg, tally, name):
        self.m, self.t, self.name = GrowMap(cfg), tally, name

    def apply(self, pw, var):
        self.t.add(self.m.apply_roots(pw, var), self.name)

    def slide(self, lo, hi):
        assert self.m.slide(lo, hi) == 0

    def flatten(self):
        return self.m.flatten()

    def dump_nodes(self):
        return self.m.dump_nodes()

    def usage(self):
        return self.m.usage()


@pytest.mark.parametrize("name", list(MS.CASES))
def test_demand_bound_covers_every_hand_built_stream(name):
    c, t = MS.case(name), Tally()
    h = MS.replay(c, {"b": _BoundSide(c["cfg"], t, name), "orc": MS.OracleSide(c["cfg"])})
    # the bound side is the state machine itself: it must still reach what the stream was built for and equal the oracle
    for what, f in c["reach"].items():
        assert f(h["b"]) > 0, f"{name}: does not reach '{what}'"
    MB.compare_flat_maps(h["b"][-1]["flat"], h["orc"][-1]["flat"], exact=True)
    t.report(f"stream {name}")


@pytest.mark.parametrize("voxel_size", [0.5, 0.4, 2.0])
def test_demand_bound_covers_the_voxel_face_key_grid(voxel_size):
    cfg = S.LioCfg(voxel_size=voxel_size)
    ks = np.arange(-6, 7, dtype=np.float64)
    face = (ks * np.float64(np.float32(voxel_size))).astype(np.float32)
    vals = np.concatenate([face, np.nextafter(face, np.float32(np.inf)), np.nextafter(face, np.float32(-np.inf)), np.float32([0.0, -0.0, 1e-30, -1e-30])])
    grid = np.stack(np.meshgrid(vals, vals[::5], vals[::7], indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    var = np.tile(np.eye(3) * 1e-4, (len(grid), 1, 1))
    t = Tally()
    t.add(GrowMap(cfg).apply_roots(grid, var), "key grid")
    assert t.roots > 50
    t.report(f"voxel-face key grid {voxel_size}")


def test_demand_bound_of_a_tick_is_the_sum_over_its_roots():
    """maph_demand (what map_demand_kernel sums) on a copy of the map equals the per-root bounds of the same tick."""
    cfg = S.LioCfg()
    rng, rects = np.random.default_rng(5), S.make_scene("room", 0.5)
    a, b = GrowMap(cfg), GrowMap(cfg)
    for tick in range(3):
        pw, var = _room_tick(rng, rects, tick)
        pt = GrowMap._pt(pw, var)
        d = np.zeros(3, np.int64)
        assert b.lib.maph_demand(b.h, pt.ctypes.data, len(pt), 0, d.ctypes.data) == 0
        assert b.apply(pw, var) == 0
        rows = a.apply_roots(pw, var)
        assert np.array_equal(d, rows[:, :3].sum(0))


# ---------------------------------------------------------------------------------------------------- growth policy


def _grown_all(gm):
    return all(gm.grew & MAP_ERR[r] for r in ("nodes", "pool", "recs", "hash"))


@pytest.mark.parametrize("cfg", ROOM_CFGS[:2], ids=ROOM_IDS[:2])
def test_map_grown_from_minimal_capacities_equals_the_oracle_bit_for_bit(cfg):
    rng, rects = np.random.default_rng(5), S.make_scene("room", 0.5)
    orc, gm = oracle_map(cfg), GrowMap(cfg, **TINY)
    caps = [gm.capacity()]
    for tick in range(10):
        pw, var = _room_tick(rng, rects, tick)
        oracle_update_map(orc, pw, var)
        assert gm.apply_grow(pw, var) == 0
        MB.compare_flat_maps(gm.flatten(), orc.flatten(), what=(f"grown map, tick {tick}", "oracle"), exact=True)
        caps.append(gm.capacity())
    assert _grown_all(gm), gm.grew
    # capacities only grow, and by at least a factor of two when they do
    for a, b in zip(caps, caps[1:]):
        assert all(b[k] == a[k] or b[k] >= 2 * a[k] for k in a)
    assert gm.usage()["roots"] == len(orc.flatten()["keys"])


def _slide_box():
    c, half = np.array([4, -2, 1]), 12
    return c - half, c + half


def _oracle_slide(orc, lo, hi):
    return orc.lib.orc_lio_clear_out_of_map(orc.h, *MS.key_box(lo, hi))


@pytest.mark.parametrize("order", ["slide_then_grow", "grow_then_slide"])
def test_growth_around_a_slide_equals_the_oracle(order):
    """slide_then_grow: a map that fits, slid, then ticks that make it grow. grow_then_slide: a map grown from minimal
    capacities, slid, then more ticks. The map equals the oracle's bit for bit after every step."""
    cfg = S.LioCfg()
    rng, rects = np.random.default_rng(17), S.make_scene("room", 0.5)
    lo_w, hi_w = np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0])
    orc = oracle_map(cfg)
    gm = GrowMap(cfg) if order == "slide_then_grow" else GrowMap(cfg, **TINY)
    for tick in range(4):
        pw, var = tick_points(rng, rects, 6000, lo_w, hi_w)
        oracle_update_map(orc, pw, var)
        assert gm.apply_grow(pw, var) == 0
    grew_before = gm.grew
    lo, hi = _slide_box()
    assert _oracle_slide(orc, lo, hi) > 0
    assert gm.slide(lo, hi) == 0
    MB.compare_flat_maps(gm.flatten(), orc.flatten(), exact=True)
    if order == "slide_then_grow":
        assert grew_before == 0
        # the slide kept the large capacities: shrink them to what the map holds now, so that the next ticks must grow
        u = gm.usage()
        assert gm.grow(1 << 16, u["nodes"], u["pool_points"], u["recs"]) == 0
        MB.compare_flat_maps(gm.flatten(), orc.flatten(), exact=True)
    else:
        assert _grown_all(gm), grew_before
    gm.grew = 0
    for tick in range(4):
        pw, var = tick_points(rng, rects, 6000, lo_w - 4, hi_w + 4)
        oracle_update_map(orc, pw, var)
        assert gm.apply_grow(pw, var) == 0
        MB.compare_flat_maps(gm.flatten(), orc.flatten(), what=(f"tick {tick} after the slide", "oracle"), exact=True)
    if order == "slide_then_grow":
        assert gm.grew & MAP_ERR["nodes"] and gm.grew & MAP_ERR["pool"], gm.grew


def test_build_form_grown_from_minimal_capacities_equals_the_fixed_capacity_build():
    cfg = S.LioCfg()
    rng, rects = np.random.default_rng(9), S.make_scene("room", 0.5)
    lo, hi = np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0])
    pw, var = tick_points(rng, rects, 40000, lo, hi)
    fixed, gm = GrowMap(cfg), GrowMap(cfg, **TINY)
    assert fixed.apply(pw, var, build=True) == 0
    assert gm.apply_grow(pw, var, build=True) == 0
    assert _grown_all(gm), gm.grew
    MB.compare_flat_maps(gm.flatten(), fixed.flatten(), exact=True)
    MB.compare_node_dumps(gm.dump_nodes(), fixed.dump_nodes())


def test_key_range_is_still_an_error_with_growth():
    """A key outside +-2^20 is not a capacity: growing cannot help, the tick fails (MAP_ERR_KEY)."""
    cfg = S.LioCfg()
    rng, rects = np.random.default_rng(2), S.make_scene("room", 0.5)
    pw, var = tick_points(rng, rects, 500, np.array([-12.0, -9.0, -3.0]), np.array([12.0, 9.0, 5.0]))
    far = pw.copy()
    far[0] = [3e6, 0, 0]
    assert GrowMap(cfg, **TINY).apply_grow(far, var) & 16


def test_map_cfg_keeps_its_layout():
    """esikf_map_cfg.pad became grow: same offset, same size."""
    assert C.sizeof(api.MapCfgC) == 112
    assert api.MapCfgC.grow.offset == 72 and api.MapCfgC.grow.size == 4 and api.MapCfgC.root_capacity.offset == 80
    assert [f for f, _ in api.MapCfgC._fields_].index("grow") == 7
