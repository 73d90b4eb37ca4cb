"""GPU: the persistent update kernels at every grid and slice geometry their launches can take.

How a launch deals its work (csrc/esikf_api_update.cu vio_grid / lio_grid, esikf_vio.cu vio_block_range, esikf_lio.cu
lio_block_range, esikf_fused.cu persist_exchange / reduce_entry), with PB = min(SMs, 160) partial columns:
  VIO  G = min(ceil(n / 16), PB) CTAs of per = ceil(n / G) patches; patch lo + warp + 16 k goes to (warp, k) and the
       per-warp patch cache holds a CTA's patches while per <= 32 (above it slot 0 is refilled for every patch); trailing
       CTAs are empty once (G - 1) per >= n. Entry e of the 37 mailbox entries is summed by warp (e / G) mod 16 of CTA
       e mod G (G <= 2: warps own two entries, G > 37: CTAs own none), lane l summing columns l, l + 32, ...
  LIO  G = min(ceil(n / 32), PB) CTAs of whole 32-point chunks, the first chunks % G CTAs one chunk more.
Every count below is derived from PB and asserts the geometry it was chosen for, recomputed here from those formulas.

Nothing in the inputs can hide a slicing error: every visual patch is distinct (copies of config 2's patches moved by a
few millimetres, each copy with its own reference exposure), the first and last patch of every CTA, warp 0's second slot
and the last patch are border footprints at search levels 1 / 2, and before every run the per-patch / per-point outputs
are overwritten by a full-width update on a different sub-map or scan, so a patch or point the kernel never visits keeps
a wrong value. Every case is held to the oracle and to itself, bit for bit, across the launch forms."""
import dataclasses

import numpy as np
import pytest

import lio_assoc as A
import oracle_bind as O
import vio_border as VB
from conftest import get_frame
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from harness import LIO_KEYS, VIO_KEYS, bits_equal, compare_lio, compare_vio, lio_gpu, lio_oracle, sm_count, sweep, vio_prior, vio_setup

pytestmark = pytest.mark.gpu

VIO_WARPS, VIO_KMAX, VIO_ENTRIES, LIO_CHUNK = 16, 2, 37, 32
DELTA = 0.002  # m: lateral world offset between copies of a patch (a sub-pixel to pixel move of its projection)
CONFIG2 = dict(seed=0, n_pts=1000, n_map=300_000, n_patches=2000, scene_scale=0.7)  # 640 x 512, 4 levels: TMA-eligible
CONFIG5_CAM = S.CamCfg(width=612, height=512, fx=612.0 * 0.72, fy=612.0 * 0.72, cx=306.0, cy=256.0)  # pitch not a multiple of 16
CONFIG5 = dict(seed=13, n_pts=1000, n_map=300_000, n_patches=4000, scene_scale=0.7, cam=CONFIG5_CAM, vio=S.VioCfg(levels=5, img_point_cov=1000.0))


def partial_blocks():
    """PB of the device the tests run on. Parameter ids depend on it, so it is read at collection; without a device the
    H100 SXM's 132 names the cases (they are skipped there)."""
    import torch

    return min(sm_count(), 160) if torch.cuda.is_available() else 132


# ----------------------------------------------------------------------------------------------------- geometry
def vio_geometry(n, PB):
    G = max(1, min(-(-n // VIO_WARPS), PB))
    per = -(-n // G)
    return dict(G=G, per=per, cached=per <= VIO_WARPS * VIO_KMAX, empty=G - (-(-n // per)) > 0, two_entry_warps=VIO_WARPS * G < VIO_ENTRIES,
                entryless_ctas=max(G - VIO_ENTRIES, 0), columns=-(-G // 32))


def vio_slices(n, PB):
    per = vio_geometry(n, PB)["per"]
    return [(min(b * per, n), min(b * per + per, n)) for b in range(vio_geometry(n, PB)["G"])]


def lio_geometry(n, PB):
    chunks = -(-n // LIO_CHUNK)
    G = max(1, min(chunks, PB))
    return dict(G=G, partial=n % LIO_CHUNK != 0, per=chunks // G, extra=chunks % G)


def dedup(rows):
    """Rows (name, n, want) with equal n merged into the first one; the id names every row it stands for."""
    out = {}
    for name, n, want in rows:
        if n in out:
            out[n][0].append(name)
        else:
            out[n] = ([name], n, want)
    return [pytest.param(n, want, id=f"n{n}-" + "=".join(names)) for names, n, want in out.values()]


def vio_rows(PB):
    """(name, count, the geometry it reaches); ordered so that wide and narrow grids alternate on the shared context."""
    g = lambda **kw: kw
    return [
        ("1", 1, g(G=1, per=1)),
        ("16PB", 16 * PB, g(G=PB, per=16, cached=True, empty=False)),
        ("15", 15, g(G=1, per=15)),  # idle warp
        ("32PB+1", 32 * PB + 1, g(G=PB, per=33, cached=False, empty=True)),
        ("16", 16, g(G=1, per=16, two_entry_warps=True)),
        ("16PB+1", 16 * PB + 1, g(G=PB, per=17, cached=True, empty=True)),
        ("17", 17, g(G=2, per=9, two_entry_warps=True)),
        ("96PB+5", 3 * 32 * PB + 5, g(G=PB, per=97, cached=False)),
        ("32", 32, g(G=2, per=16, two_entry_warps=True)),
        ("32PB", 32 * PB, g(G=PB, per=32, cached=True, empty=False)),
        ("33", 33, g(G=3, per=11, two_entry_warps=False)),
        ("16PB-1", 16 * PB - 1, g(G=PB, per=16, cached=True)),
        ("16x32", 16 * 32, g(G=32, per=16, columns=1)),
        ("16x64+1", 16 * 64 + 1, g(G=65, columns=3, entryless_ctas=65 - VIO_ENTRIES)),
        ("16x32+1", 16 * 32 + 1, g(G=33, columns=2)),
        ("16x37+1", 16 * 37 + 1, g(G=38, entryless_ctas=1)),
        ("16x36", 16 * 36, g(G=36, entryless_ctas=0)),
        ("16x37", 16 * 37, g(G=37, entryless_ctas=0)),
    ]


def lio_rows(PB):
    rows = []
    for G in (1, 2, 28, 29, 30, 32, 33, PB - 1, PB):
        rows += [(f"G{G}", LIO_CHUNK * G, dict(G=G, partial=False)), (f"G{G}-partial", LIO_CHUNK * (G - 1) + 1, dict(G=G, partial=True))]
    rows += [("PB+1-chunks", LIO_CHUNK * (PB + 1), dict(G=PB, partial=False, per=1, extra=1)),  # one CTA takes a second chunk
             ("2PB-1-chunks", LIO_CHUNK * (2 * PB - 2) + 1, dict(G=PB, partial=True, per=1, extra=PB - 1))]  # all CTAs but the last do
    return rows


PB0 = partial_blocks()


def check_geometry(got, want, n):
    for k, v in want.items():
        assert got[k] == v, (n, k, got[k], v)


def skip_if_grid_too_wide(want, PB):
    if want.get("G", 1) > PB:
        pytest.skip(f"needs {want['G']} CTAs, the device has {PB} partial columns")


# ----------------------------------------------------------------------------------------------------- VIO sub-maps
def lateral(rng, pos, centre):
    """Unit vectors perpendicular to the viewing ray of each point."""
    ray = pos - centre
    ray /= np.linalg.norm(ray, axis=1, keepdims=True)
    u = rng.normal(size=pos.shape)
    u -= (u * ray).sum(1, keepdims=True) * ray
    return u / np.linalg.norm(u, axis=1, keepdims=True)


class Source:
    """A frame's patches (the oracle's warp at the prior) and a pool of border patches at search levels 1..max_sl, from
    which sub-maps of any size are drawn."""

    def __init__(self, fr, prior_seed, max_sl, alternate_search_level=False):
        self.fr, self.prior = fr, vio_prior(fr, prior_seed)
        cam, L = fr["cam_cfg"], fr["vio_cfg"].levels
        w = O.oracle_warp_patches(fr, self.prior)
        n = len(fr["vis_pos"])
        # config 5: every other patch at search level 1, so that the coarsest level's taps are 32 pixels apart
        sl = (np.arange(n) % 2).astype(np.int32) if alternate_search_level else w["search_levels"]
        self.interior = dict(pos=fr["vis_pos"], warp=w["warp_patch"], sl=sl, ie=fr["inv_ref_expo"], px_ref=fr["px_ref"])
        px, _, _ = VB.border_targets(cam.width, cam.height, L, np.random.default_rng(prior_seed), max_sl)
        bsl = (1 + np.arange(len(px)) % max_sl).astype(np.int32)
        b = VB.patches_at(fr, self.prior, px, bsl)
        self.border = dict(pos=b["vis_pos"], warp=b["warp_patch"], sl=b["search_levels"], ie=np.ones(len(px)), px_ref=b["px_ref"])
        st = S.unpack_state(self.prior)
        Rcw, Pcw = S.camera_pose(fr["ext"], st["R"], st["p"])
        self.centre = -Rcw.T @ Pcw

    def copies(self, kind, n, seed, draw=0):
        """n patches of `kind`: copy j = k // N of source patch k % N, moved laterally by j * DELTA, with inverse reference
        exposure ie * (1 + 0.002 j) * (1 + 0.001 draw)."""
        src = getattr(self, kind)
        N = len(src["pos"])
        k = np.arange(n)
        j, s = k // N, k % N
        pos = src["pos"][s] + (j * DELTA)[:, None] * lateral(np.random.default_rng(seed), src["pos"][s], self.centre)
        return dict(pos=pos, warp=src["warp"][s], sl=src["sl"][s], ie=src["ie"][s] * (1.0 + 0.002 * j) * (1.0 + 0.001 * draw), px_ref=src["px_ref"][s])

    def sub_map(self, n, PB, draw=0):
        """n distinct patches; the designed indices (first and last of every CTA, lo + 16 of every CTA, the last patch)
        are border patches. `draw` picks the directions of the copies' offsets and scales every reference exposure."""
        out = self.copies("interior", n, (n, draw), draw)
        d = designed_indices(n, PB)
        b = self.copies("border", len(d), (n, draw, 1), draw)
        for key in out:
            out[key] = np.array(out[key])
            out[key][d] = b[key]
        out["designed"] = d
        return out

    def poison(self, n, PB):
        """The sub-map an update runs on before each case: at least n patches on every CTA of the grid, in reverse
        order and at other reference exposures, so that its per-patch errors differ from the case's at every index."""
        m = max(n, VIO_WARPS * PB)
        p = self.copies("interior", m, m + 7)
        return {k: v[::-1] for k, v in p.items()} | dict(ie=p["ie"][::-1] * 0.9)

    def args(self, p):
        c = lambda a: np.ascontiguousarray(a)
        return (self.fr["img"], c(p["pos"]), c(p["warp"]), c(p["sl"]), c(p["ie"]), self.prior, self.prior)


def designed_indices(n, PB):
    d = {n - 1}
    for lo, hi in vio_slices(n, PB):
        if hi > lo:
            d |= {lo, hi - 1}
        if hi - lo > VIO_WARPS:
            d.add(lo + VIO_WARPS)  # warp 0's second slot
    return np.array(sorted(d))


_sources = {}


def source(name):
    if name not in _sources:
        if name == "config2":
            _sources[name] = Source(get_frame(**CONFIG2), 0, max_sl=2)
        else:  # five levels: search level 2 would take the coarsest footprint beyond the in-buffer band of a 512-row image
            _sources[name] = Source(get_frame(**CONFIG5), 13, max_sl=1, alternate_search_level=True)
    return _sources[name]


# solve mode 0: every loop mode and the TMA footprints (a silent no-op on config 5's 612-byte rows) bit for bit; solve mode
# 1 (the reference's literal op order) in both loop modes. The first run of each group is held to the oracle.
VIO_GROUPS = ([dict(loop_mode=2), dict(loop_mode=0), dict(loop_mode=1), dict(loop_mode=2, tuning=api.TUNE_VIO_TMA)],
              [dict(loop_mode=2, solve_mode=1), dict(loop_mode=0, solve_mode=1)])


# The oracle sums each iteration's error in float, in the reference's order (compare_vio); the device sums it in fp64. An
# accept / rollback decision between two errors closer than this (relative) can go either way between the two.
DECISION_MARGIN = 3e-6


def decisions_clear(o, L):
    for lvl in range(L):
        tr = o["error_trace"][lvl][:o["iters_per_level"][lvl]]
        if (np.abs(np.diff(tr)) < DECISION_MARGIN * tr[1:]).any():
            return False
    return True


def clear_sub_map(src, n, PB, oracle):
    """The sub-map of the first draw whose every decision the oracle takes is clear of DECISION_MARGIN, and the oracle's
    result on it."""
    for draw in range(16):
        sub = src.sub_map(n, PB, draw)
        o = oracle(src.args(sub), sub)
        if decisions_clear(o, src.fr["vio_cfg"].levels):
            assert len({tuple(np.round(p, 9)) for p in sub["pos"]}) == n  # every patch distinct
            assert (sub["sl"][sub["designed"]] >= 1).all()
            assert o["total_iters"] >= src.fr["vio_cfg"].levels
            return sub, o
    pytest.fail(f"no draw of {n} patches keeps every decision clear of the error sum's rounding")


def check_vio_case(ctx, src, n, PB):
    fr = src.fr
    sub, o = clear_sub_map(src, n, PB, lambda args, _: O.OracleVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"], threads=1).update(*args))
    args, pargs = src.args(sub), src.args(src.poison(n, PB))

    def run():
        ctx.vio_update(*pargs)
        return ctx.vio_update(*args)

    vio_setup(ctx, fr)
    for group in VIO_GROUPS:
        runs = sweep(ctx, run, group)
        compare_vio(runs[0], o, fr["vio_cfg"].levels)
        for r in runs[1:]:
            bits_equal(runs[0], r, VIO_KEYS)


# ----------------------------------------------------------------------------------------------------- VIO tests
VIO_PARAMS = dedup(vio_rows(PB0))


@pytest.mark.parametrize("n,want", VIO_PARAMS)
def test_vio_patch_counts_at_the_grid_boundaries(gpu_ctx, n, want):
    """Config 2's frame (640 x 512, 4 levels): one CTA to every SM, one and two patches per warp, the patch-cache limit,
    empty trailing CTAs, warps that sum two mailbox entries, CTAs that sum none and a lane's second / third column."""
    PB = min(sm_count(), 160)
    assert PB == PB0
    skip_if_grid_too_wide(want, PB)
    check_geometry(vio_geometry(n, PB), want, n)
    check_vio_case(gpu_ctx, source("config2"), n, PB)


@pytest.mark.parametrize("n", [4000, 6000])
def test_vio_config5_two_and_more_patches_per_warp(gpu_ctx, n):
    """Config 5's frame (612 x 512, 5 levels, every other patch at search level 1: tap strides up to 32). 4 k patches: two
    per warp, both cached across iterations; 6 k: more than the cache holds, slot 0 refilled every time."""
    PB = min(sm_count(), 160)
    geo = vio_geometry(n, PB)
    check_geometry(geo, dict(G=PB, cached=n == 4000), n)
    assert geo["per"] > VIO_WARPS, geo  # warp 0 holds a second patch
    src = source("config5")
    assert src.fr["cam_cfg"].width % 16 != 0 and src.fr["vio_cfg"].levels == 5
    check_vio_case(gpu_ctx, src, n, PB)


def test_vio_inverse_variant_large_small_large(gpu_ctx):
    """inverse_composition_en with reference data per copy: 32 PB + 1 (uncached, empty CTAs), 7, 8, 9 (the per-iteration
    precompute's 8-patch blocks: short, exact, one over), 16 PB + 1 on one context, so H_sub_inv (sized by the largest
    count so far) is reused by smaller updates and then larger ones. Against the oracle; persistent against per-iteration."""
    PB = min(sm_count(), 160)
    src = source("config2")
    fr = src.fr
    cam, cfg = fr["cam_cfg"], fr["vio_cfg"]
    inv_cfg = dataclasses.replace(cfg, inverse_composition_en=True)
    refs_of = lambda p: O.inverse_refs_from_frame(dict(fr, vis_pos=p["pos"], px_ref=p["px_ref"]))

    def inverse_oracle(args, sub):
        vio = O.OracleVIO(cam, fr["ext"], cfg, threads=1)
        vio.set_inverse_refs(**refs_of(sub))
        vio.set_inverse(True)
        return vio.update(*args)

    counts = (32 * PB + 1, 7, 8, 9, 16 * PB + 1)
    check_geometry(vio_geometry(counts[0], PB), dict(per=33, cached=False), counts[0])
    check_geometry(vio_geometry(counts[-1], PB), dict(per=17, cached=True), counts[-1])
    try:
        vio_setup(gpu_ctx, fr)
        gpu_ctx.vio_set_camera(cam, inv_cfg)
        for n in counts:
            sub, o = clear_sub_map(src, n, PB, inverse_oracle)
            poison = src.poison(n, PB)
            args, pargs = src.args(sub), src.args(poison)
            refs, prefs = refs_of(sub), refs_of(poison)
            set_refs = lambda r: gpu_ctx.vio_set_inverse_refs(r["ref_img_index"], r["ref_px"], r["ref_f"], r["ref_R"], r["ref_pos"])

            def run():
                set_refs(prefs)
                gpu_ctx.vio_update(*pargs)
                set_refs(refs)
                return gpu_ctx.vio_update(*args)

            a, b = sweep(gpu_ctx, run, [dict(loop_mode=0), dict(loop_mode=2)])
            bits_equal(a, b, VIO_KEYS)
            compare_vio(b, o, cfg.levels)
    finally:
        gpu_ctx.vio_set_camera(cam, cfg)


# ----------------------------------------------------------------------------------------------------- LIO
LIO_VARIANTS = [dict(loop_mode=2), dict(loop_mode=0), dict(loop_mode=1), dict(loop_mode=2, tuning=api.TUNE_STAGE_LDG),
                dict(loop_mode=0, tuning=api.TUNE_STAGE_LDG)]


@pytest.mark.parametrize("n,want", dedup(lio_rows(PB0)))
@pytest.mark.parametrize("name", ["main", "zero_prob"])
def test_lio_grid_sizes(gpu_ctx, name, n, want):
    """The hand-built association cases of tests/lio_assoc.py at chunk counts that give G = 1, 2, 28-30 (around the 29
    information entries), 32, 33, PB - 1 and PB CTAs, with a full and a partial last chunk, and above 32 PB points, where
    lio_block_range deals the remainder chunks. The scan's own points while they last, then its warps repeated; before
    each run the per-point outputs hold another scan's (the same points shifted by one index)."""
    PB = min(sm_count(), 160)
    assert PB == PB0
    skip_if_grid_too_wide(want, PB)
    check_geometry(lio_geometry(n, PB), want, n)
    fr = A.case(name)
    case = A.tiled(fr, n)
    m = max(n, LIO_CHUNK * PB)
    poison = dict(fr, pts=np.ascontiguousarray(np.roll(A.tiled(fr, m + 1)["pts"], -1, axis=0)[:m]))

    def run():
        lio_gpu(gpu_ctx, poison)
        return lio_gpu(gpu_ctx, case)

    o = lio_oracle(case)
    runs = sweep(gpu_ctx, run, LIO_VARIANTS)
    compare_lio(runs[0], o)
    for r in runs[1:]:
        bits_equal(runs[0], r, LIO_KEYS)
