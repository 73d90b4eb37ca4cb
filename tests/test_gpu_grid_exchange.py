"""GPU: the persistent VIO kernel exchanges its per-iteration information through the context's grid mailbox (tagged words,
double-buffered by the exchange counter's parity), the persistent LIO kernel through a grid barrier whose counters alternate
between launches. Launches of different grid sizes, both kernels, both launch forms and levels that end early, interleaved on
one context, must each give what a fresh context gives on the per-iteration launch path (loop_mode 0), bit for bit; so must
two contexts used alternately on one device."""
import numpy as np
import pytest

from conftest import get_frame
from fast_livo2_b200 import api
from harness import LIO_KEYS, VIO_KEYS, bits_equal, variant, vio_prior, vio_setup, vio_warp

pytestmark = pytest.mark.gpu


def _jobs(ctx):
    """name -> run(ctx): LIO on 132 CTAs (100 k points) and on 7 (200 points), VIO on 125 CTAs (2 000 patches), 10 (150)
    and 2 (20). Warps are taken with `ctx`, which is left with the ref images of the last frame."""
    big = get_frame(seed=0, n_pts=100_000, n_map=1_000_000, n_patches=2000)
    small = get_frame(seed=2, n_pts=2000, n_map=120_000, n_patches=150, scene_scale=0.5)
    vio_args = {}
    for name, fr, n in (("vio_125", big, None), ("vio_10", small, None), ("vio_2", small, 20)):
        vio_setup(ctx, fr)
        prior = vio_prior(fr)
        w = vio_warp(ctx, fr, prior)
        k = slice(None, n)
        vio_args[name] = (fr, (fr["img"], fr["vis_pos"][k], w["warp_patch"][k], w["search_levels"][k], fr["inv_ref_expo"][k], prior, prior))

    def lio(pts):
        def run(c):
            c.set_extrinsics(big["ext"])
            return c.lio_update(pts, big["state_prior"], big["state_prior"], big["lio_cfg"])
        return run

    def vio(name):
        fr, args = vio_args[name]

        def run(c):
            vio_setup(c, fr)
            return c.vio_update(*args)
        return run

    return {"lio_132": lio(big["pts"]), "lio_7": lio(big["pts"][:200]), "vio_125": vio("vio_125"), "vio_10": vio("vio_10"), "vio_2": vio("vio_2")}, big


def _keys(name):
    return LIO_KEYS if name.startswith("lio") else VIO_KEYS


def _reference(jobs, big):
    """Every job once on a fresh context, per-iteration launches."""
    ref = api.Context(0)
    try:
        ref.set_extrinsics(big["ext"])
        ref.map_upload(big["map"], big["lio_cfg"].voxel_size)
        with variant(ref, loop_mode=0):
            return {name: run(ref) for name, run in jobs.items()}
    finally:
        ref.close()


def test_interleaved_launches_on_one_context_are_bit_identical_to_a_fresh_per_iteration_context(gpu_ctx):
    jobs, big = _jobs(gpu_ctx)
    ref = _reference(jobs, big)
    assert any(ref["vio_125"]["iters_per_level"][l] < big["vio_cfg"].max_iterations for l in range(big["vio_cfg"].levels)), "no VIO level ends early"
    assert ref["lio_132"]["iters"] >= 3
    gpu_ctx.set_extrinsics(big["ext"])
    gpu_ctx.map_upload(big["map"], big["lio_cfg"].voxel_size)
    rng = np.random.default_rng(7)
    names = list(jobs)
    plan = [(names[i % len(names)], 2) for i in range(2 * len(names))]  # every job persistent at least twice
    plan += [(names[i], 0) for i in range(len(names))]                    # and on the per-iteration path once
    plan += [(names[rng.integers(len(names))], int(rng.choice([0, 2, 2, 2]))) for _ in range(30)]
    order = rng.permutation(len(plan))
    assert len(plan) >= 40
    for k in order:
        name, mode = plan[k]
        with variant(gpu_ctx, loop_mode=mode):
            r = jobs[name](gpu_ctx)
        bits_equal(ref[name], r, _keys(name))


def test_two_contexts_alternating_on_one_device(gpu_ctx):
    jobs, big = _jobs(gpu_ctx)
    ref = _reference(jobs, big)
    other = api.Context(0)
    try:
        for c in (gpu_ctx, other):
            c.set_extrinsics(big["ext"])
            c.map_upload(big["map"], big["lio_cfg"].voxel_size)
        for name in ("lio_132", "vio_125", "vio_2", "lio_7", "vio_10", "vio_125", "lio_132"):
            for c in (gpu_ctx, other):
                bits_equal(ref[name], jobs[name](c), _keys(name))
    finally:
        other.close()
