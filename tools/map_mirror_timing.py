"""What the host mirror of the device voxel map costs per tick (VoxelMapConfig::device_map_mirror_), on the cfg2 frame with
bench.py's map-leg call sequence (BuildVoxelMap from the scan at the true pose, then per tick a LIO update and UpdateVoxelMap).

  export : on a context of the C ABI, per tick the touched roots, exported nodes and bytes of esikf_map_device_export;
           the stream time of the whole call (CUDA events on the context's stream around it), and, from a torch.profiler
           pass over a second call on the same tick (the export is a pure read: same bytes), the device time of its kernels
           (the count / write kernels and the scan) and of its device-to-host copies;
  shim   : two fl2b200::VoxelMapManager sessions, mirror on and off, tick by tick in turn: the host wall time of
           UpdateVoxelMap() (it returns after the device synchronised; with the mirror, export + apply are inside).

Prints one JSON line with the card's name, power limit and maximum SM clock read in the same run.

    python tools/map_mirror_timing.py [--ticks 30] [--out result.json]
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


def _profiled_export(ctx):
    """Kernel and device-to-host copy time (ms) of one esikf_map_device_export call, from torch.profiler's CUDA activity."""
    us = T.kernel_us(ctx.map_device_export, 1, ("Memcpy DtoH", "map_export", "DeviceScan"))
    return (sum(us["map_export"]) + sum(us["DeviceScan"])) / 1e3, sum(us["Memcpy DtoH"]) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    T.require_gpu("map_mirror_timing")
    import torch
    from fast_livo2_b200 import api, workloads
    from map_mirror import session, shim_sessions, vp

    fr = workloads.frame("cfg2")
    cfg, ext, pts = fr["lio_cfg"], fr["ext"], np.ascontiguousarray(fr["pts"], np.float32)
    dev = torch.device("cuda", 0)
    ctx = api.Context(0)
    lib = shim_sessions()
    hs = {"mirror": session(lib, cfg, ext, fr["map"]), "plain": session(lib, cfg, ext, fr["map"])}
    rows = []
    try:
        ctx.set_extrinsics(ext)
        ctx.map_device_init(cfg, root_capacity=1 << 19)
        ctx.lio_set_scan(pts)
        ctx.map_device_build(fr["state_true"])
        for name, h in hs.items():
            rc = lib.fl2_shim_session_device_map_mirror(h, vp(pts), len(pts), vp(np.ascontiguousarray(fr["state_true"])), cfg.min_eigen_value, cfg.max_points_num, 1 << 19,
                                                       0, 1 if name == "mirror" else 0)
            assert rc == 0, (name, rc)
        stream = torch.cuda.ExternalStream(ctx.stream, device=dev)
        prior = np.ascontiguousarray(fr["state_prior"])
        for k in range(args.ticks):
            ctx.lio_update(pts, prior, prior, cfg)
            ctx.map_device_update()
            got = []
            (export_ms,), _ = T.per_call_ms(stream, lambda: got.append(ctx.map_device_export()), 1)
            exp = got[0]
            kern_ms, d2h_ms = _profiled_export(ctx)
            row = dict(tick=k, touched_roots=int(len(exp["keys"])), nodes=int(len(exp["nodes"])),
                       bytes=int(exp["nodes"].nbytes + exp["keys"].nbytes + exp["first"].nbytes + exp["count"].nbytes), export_call_ms=export_ms,
                       export_kernels_ms=kern_ms, export_d2h_ms=d2h_ms)
            for name, h in hs.items():  # mirror then plain, every tick
                lio_out, vio_out, iters = np.zeros(386), np.zeros(386), np.zeros(2, np.int32)
                assert lib.fl2_shim_session_step(h, vp(pts), len(pts), vp(prior), vp(prior), None, 0, None, None, None, None, vp(lio_out), vp(vio_out), vp(iters)) == 0
                t0 = time.perf_counter()
                assert lib.fl2_shim_session_update_map(h) == 0
                row[f"update_voxel_map_{name}_ms"] = (time.perf_counter() - t0) * 1e3
            rows.append(row)
    finally:
        for h in hs.values():
            lib.fl2_shim_session_destroy(h)
        ctx.close()
    steady = rows[3:] if len(rows) > 6 else rows
    med = lambda key: statistics.median(r[key] for r in steady)
    res = dict(what="cfg2 frame (100k points), bench.py's map-leg sequence; export on a C-ABI context, UpdateVoxelMap() through two shim sessions "
                    "(mirror on / off) alternating tick by tick; medians over ticks 3..",
               **T.card(), ticks=args.ticks, n_pts=int(len(pts)),
               median={k: med(k) for k in ("touched_roots", "nodes", "bytes", "export_call_ms", "export_kernels_ms", "export_d2h_ms", "update_voxel_map_mirror_ms",
                                           "update_voxel_map_plain_ms")},
               per_tick=rows)
    print(json.dumps({k: v for k, v in res.items() if k != "per_tick"}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
