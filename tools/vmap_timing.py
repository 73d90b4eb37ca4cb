"""Time the observation store's calls against the packed entry points they replace, on the GPU.

  esikf_vmap_score          vs esikf_vio_score_ref_patches : 2 k / 4 k points x 6 / 15 / 30 observations (DESIGN.md §8's K13 sizes)
  esikf_vmap_update_points  vs esikf_vio_update_points     : 2 k / 10 k sub-map entries, config 2's camera

Call times: CUDA events on the context's stream around the call (median of `reps`); the call enqueues its uploads, kernels
and readback there and synchronises before it returns. Kernel times:
torch.profiler with CUDA activities in a separate pass (sum of the call's kernels, averaged per call). The card's name,
power limit and maximum SM clock are read in the same run.

  python tools/vmap_timing.py [--reps 30] [--out results.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import timing as T  # noqa: E402

import observe_cases as OC  # noqa: E402
from fast_livo2_b200 import api  # noqa: E402
from fast_livo2_b200 import synthetic as S  # noqa: E402


def lists(rng, n, k):
    """n points with k observations each: random patches and views around a point 10 m ahead, ids 0 .. k-1."""
    m = n * k
    R = np.tile(np.eye(3).reshape(9), (m, 1))
    t = rng.normal(0, 0.5, (m, 3))
    return dict(first=(np.arange(n + 1) * k).astype(np.int32), px=rng.uniform(0, 600, (m, 2)), patch=rng.normal(100, 20, (m, 64)).astype(np.float32),
                T_f_w=np.concatenate([R, t], 1), id=np.tile(np.arange(k, dtype=np.int32), n), mean=np.zeros(m, np.float32), score=np.zeros(m, np.float32),
                ref=np.full(n, -1, np.int32))


def call_ms(ctx, f, reps):
    import torch

    f()
    return float(np.median(T.per_call_ms(torch.cuda.ExternalStream(ctx.stream), f, reps)[0]))


def kernel_ms(f, reps):
    import torch

    f()
    torch.cuda.synchronize()
    return sum(sum(us) for us in T.kernel_us(f, reps).values()) / reps / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    T.require_gpu("vmap_timing")
    ctx = api.Context(0)
    rng = np.random.default_rng(0)
    out = dict(card=T.card(), score=[], update=[])
    for n in (2000, 4000):
        for k in (6, 15, 30):
            L = lists(rng, n, k)
            ctx.vmap_init(n)
            ids = ctx.vmap_add_points(**L)
            pos = np.tile([0.0, 0.0, 10.0], (n, 1)) + rng.normal(0, 0.1, (n, 3))
            normal = np.tile([0.0, 0.0, -1.0], (n, 1))
            ref = np.zeros(n, np.int32)

            def packed():
                ctx.vio_score_ref_patches(L["first"], pos, normal, L["patch"], L["mean"], L["id"], L["T_f_w"])

            def store():
                ctx.lib.esikf_vmap_score(ctx.h, n, ids.ctypes.data, pos.ctypes.data, normal.ctypes.data, ref.ctypes.data, None, None)  # no rows

            row = dict(points=n, obs=k, packed_call_ms=call_ms(ctx, packed, a.reps), store_call_ms=call_ms(ctx, store, a.reps), packed_kernel_ms=kernel_ms(packed, a.reps),
                       store_kernel_ms=kernel_ms(store, a.reps))
            out["score"].append(row)
            print("score", row, flush=True)
    for n in (2000, 10000):
        sc = OC.scene("pinhole", n, seed=3)
        ctx.set_extrinsics(sc["ext"])
        ctx.vio_set_camera(sc["cam"], S.VioCfg())
        ctx.vio_set_image(sc["img"])
        ctx.vio_set_patches(np.ascontiguousarray(sc["pos"]), np.zeros((n, 4 * 64), np.float32), np.zeros(n, np.int32), np.ones(n))
        ctx.vmap_init(n)
        one = dict(first=np.arange(n + 1, dtype=np.int32), px=sc["last_px"], patch=np.zeros((n, 64), np.float32), T_f_w=sc["last_T"],
                   id=np.zeros(n, np.int32), mean=np.zeros(n, np.float32), score=np.zeros(n, np.float32), ref=np.full(n, -1, np.int32))
        ids = ctx.vmap_add_points(**one)
        conv = sc["converged"]

        def packed():
            ctx.vio_update_points(conv, sc["last_T"], sc["last_px"], state=sc["state"])

        def store():
            ctx.vmap_update_points(ids, conv, 1, state=sc["state"])

        for _ in range(40):  # the store's lists at their steady state: 30 observations, one evicted per added one
            store()
        row = dict(entries=n, packed_call_ms=call_ms(ctx, packed, a.reps), store_call_ms=call_ms(ctx, store, a.reps), packed_kernel_ms=kernel_ms(packed, a.reps),
                   store_kernel_ms=kernel_ms(store, a.reps))
        out["update"].append(row)
        print("update", row, flush=True)
    print(out["card"])
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
