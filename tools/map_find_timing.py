"""What the VIO front end's find_correspond lookups cost on the device map (esikf_map_device_find, K12) against the host mirror
they replace, on the cfg2 frame with bench.py's map-leg call sequence (BuildVoxelMap from the scan at the true pose, then per
tick a LIO update and UpdateVoxelMap), after --warmup such ticks.

  device : for 2 k, 5 k and 20 k query points (plane centres of the map moved by up to a voxel, the kind of point
           updateReferencePatch and the ray samples look up), on a C-ABI context: the kernel time from torch.profiler, and the
           call time through the C ABI (CUDA events on the context's stream around the call, which returns synchronised, and
           the host wall time of the call), medians over --reps calls;
  shim   : in the same run, two VoxelMapManager sessions, mirror on and off, tick by tick in turn: the host wall time of
           UpdateVoxelMap(); and for the same query points the host find_correspond on the mirror (fl2_shim_mirror_find) and
           FindCorrespond through the mirror-off session.

Prints one JSON line with the card's name, power limit and maximum SM clock read in the same run.

    python tools/map_find_timing.py [--warmup 10] [--ticks 20] [--reps 50] [--out result.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import timing as T  # noqa: E402

SIZES = (2000, 5000, 20000)


def _profiled_kernel_ms(ctx, q):
    us = T.kernel_us(lambda: ctx.map_device_find(q, 0), 10, ("map_find_kernel",))["map_find_kernel"]
    assert us, "no map_find_kernel in the trace"
    return statistics.median(us) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--ticks", type=int, default=20)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import ctypes as C

    T.require_gpu("map_find_timing")
    import torch
    from fast_livo2_b200 import api, workloads
    from fast_livo2_b200.synthetic import PLANE_DTYPE
    from map_mirror import MirrorView, session, shim_sessions, vp

    fr = workloads.frame("cfg2")
    cfg, ext, pts = fr["lio_cfg"], fr["ext"], np.ascontiguousarray(fr["pts"], np.float32)
    prior = np.ascontiguousarray(fr["state_prior"])
    dev = torch.device("cuda", 0)
    ctx = api.Context(0)
    lib = shim_sessions()
    lib.fl2_shim_session_find_correspond.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    hs = {"mirror": session(lib, cfg, ext, fr["map"]), "plain": session(lib, cfg, ext, fr["map"])}
    res = dict(what=f"cfg2 frame ({len(pts)} points), bench.py's map-leg sequence after {args.warmup} warm-up ticks; lookups with updateReferencePatch's key rule", **T.card(),
               voxel_size=cfg.voxel_size)
    try:
        ctx.set_extrinsics(ext)
        ctx.map_device_init(cfg, root_capacity=1 << 19)
        ctx.lio_set_scan(pts)
        ctx.map_device_build(fr["state_true"])
        for name, h in hs.items():
            rc = lib.fl2_shim_session_device_map_mirror(h, vp(pts), len(pts), vp(np.ascontiguousarray(fr["state_true"])), cfg.min_eigen_value, cfg.max_points_num, 1 << 19,
                                                       0, 1 if name == "mirror" else 0)
            assert rc == 0, (name, rc)
        upd = {"mirror": [], "plain": []}
        for k in range(args.warmup + args.ticks):
            ctx.lio_update(pts, prior, prior, cfg)
            ctx.map_device_update()
            for name, h in hs.items():  # mirror then plain, every tick
                assert lib.fl2_shim_session_step(h, vp(pts), len(pts), vp(prior), vp(prior), None, 0, None, None, None, None, vp(np.zeros(386)), vp(np.zeros(386)),
                                                 vp(np.zeros(2, np.int32))) == 0
                t0 = time.perf_counter()
                assert lib.fl2_shim_session_update_map(h) == 0
                if k >= args.warmup:
                    upd[name].append((time.perf_counter() - t0) * 1e3)
        res["update_voxel_map_ms"] = {name: statistics.median(v) for name, v in upd.items()}
        planes = ctx.map_device_download()["planes"]
        rng = np.random.default_rng(0)
        stream = torch.cuda.ExternalStream(ctx.stream, device=dev)
        view = MirrorView(hs["mirror"], lib)
        res["sizes"] = {}
        for n in SIZES:
            q = np.ascontiguousarray(planes["center"][rng.integers(0, len(planes), n)] + rng.uniform(-1, 1, (n, 3)) * cfg.voxel_size)
            got = ctx.map_device_find(q, 0)
            for _ in range(5):
                ctx.map_device_find(q, 0)
            ev_ms, wall_ms = T.per_call_ms(stream, lambda: ctx.map_device_find(q, 0), args.reps)
            mirror_ms, shim_ms = [], []
            st, rows = np.zeros(n, np.uint8), np.zeros(n, PLANE_DTYPE)
            for _ in range(max(5, args.reps // 5)):
                t0 = time.perf_counter()
                view.find(q)
                mirror_ms.append((time.perf_counter() - t0) * 1e3)
                t0 = time.perf_counter()
                assert lib.fl2_shim_session_find_correspond(hs["plain"], q.ctypes.data, n, 0, st.ctypes.data, rows.ctypes.data) == 0
                shim_ms.append((time.perf_counter() - t0) * 1e3)
            res["sizes"][n] = dict(planes_found=int((got["status"] == 2).sum()), kernel_ms=_profiled_kernel_ms(ctx, q), call_events_ms=statistics.median(ev_ms),
                                   call_wall_ms=statistics.median(wall_ms), mirror_host_find_ms=statistics.median(mirror_ms),
                                   shim_find_correspond_ms=statistics.median(shim_ms))
    finally:
        for h in hs.values():
            lib.fl2_shim_session_destroy(h)
        ctx.close()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
