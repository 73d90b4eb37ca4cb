"""What capacity growth of the device voxel map costs (esikf_map_cfg.grow): the call sequence of bench.py's map leg on the
cfg2 frame (BuildVoxelMap from the scan at the true pose, then per tick esikf_lio_update + esikf_map_device_update) on two
contexts, tick by tick in turn:

  A: fixed capacities, 2^19 roots, growth off (bench.py's sizing);
  B: growth on, starting from 2^12 roots.

CUDA events on each context's stream around esikf_map_device_update. Reports the steady-state tick time of both (B's extra
cost there is the demand kernel), the time of every tick on which B grew, both final capacities and the bytes they take
(computed from the capacities and the struct sizes, without the allocator's headroom), and the card's name, power limit and maximum SM clock
read in the same run. The two maps are compared bit for bit at the end.

    python tools/map_growth_timing.py [--ticks 30] [--out result.json]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import timing as T  # noqa: E402

# bytes per unit of each capacity: a hash slot (HashSlot + slot_root + slot_cap), a MapNode, a stored point (12 doubles),
# a record (PlaneRec + esikf_plane + rec_node)
BYTES = dict(root_capacity=2 * 24, node_capacity=312, point_capacity=96, record_capacity=144 + 256 + 4)
CAPS = ("root_capacity", "node_capacity", "record_capacity", "point_capacity")


def footprint(cap):
    return int(sum(cap[k] * BYTES[k] for k in CAPS))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    T.require_gpu("map_growth_timing")
    import map_bind as MB
    import torch
    from fast_livo2_b200 import api, workloads

    fr = workloads.frame("cfg2")
    cfg, ext, pts = fr["lio_cfg"], fr["ext"], np.ascontiguousarray(fr["pts"])
    dev = torch.device("cuda", 0)
    ctxs = {"A": api.Context(0), "B": api.Context(0)}
    try:
        init = {"A": dict(root_capacity=1 << 19), "B": dict(root_capacity=1 << 12, grow=True)}
        start = {}
        for name, c in ctxs.items():
            c.set_extrinsics(ext)
            c.map_device_init(cfg, **init[name])
            start[name] = c.map_device_capacity()
            c.lio_set_scan(pts)
            c.map_device_build(fr["state_true"])
        after_build = ctxs["B"].map_device_capacity()
        streams = {name: torch.cuda.ExternalStream(c.stream, device=dev) for name, c in ctxs.items()}
        ms = {"A": [], "B": []}
        grew = []
        for k in range(args.ticks):
            for name, c in ctxs.items():  # A then B, every tick
                c.lio_update(pts, fr["state_prior"], fr["state_prior"], cfg)
                before = c.map_device_capacity()
                ms[name] += T.per_call_ms(streams[name], c.map_device_update, 1)[0]
                now = c.map_device_capacity()
                if name == "B" and any(now[q] != before[q] for q in CAPS):
                    grew.append(dict(tick=k, ms=ms["B"][-1], grown={q: [before[q], now[q]] for q in CAPS if now[q] != before[q]}))
        steady = [k for k in range(args.ticks) if k not in {g["tick"] for g in grew}]
        MB.compare_flat_maps(ctxs["B"].map_device_download(), ctxs["A"].map_device_download(), what=("growing map", "fixed map"), exact=True)
        final = {name: c.map_device_capacity() for name, c in ctxs.items()}
        stats = {name: c.map_device_stats() for name, c in ctxs.items()}
        res = dict(
            what="esikf_map_device_update on the cfg2 frame (100k points, bench.py's map-leg sequence), A fixed at 2^19 roots, B growing from 2^12 roots, "
                 "alternating tick by tick; CUDA events on each context's stream",
            **T.card(), ticks=args.ticks, n_pts=int(len(pts)),
            steady_ms_median={name: statistics.median([ms[name][k] for k in steady]) for name in ms} if steady else "not measured",
            steady_ms_min={name: min(ms[name][k] for k in steady) for name in ms} if steady else "not measured",
            steady_ticks=len(steady), growth_ticks=grew, b_grew_at_build={q: [start["B"][q], after_build[q]] for q in CAPS if after_build[q] != start["B"][q]},
            final_capacity=final, final_bytes_from_capacities={name: footprint(final[name]) for name in final},
            roots=stats["A"]["roots"], nodes=stats["A"]["nodes"], pool_points=stats["A"]["pool_points"], maps_bit_identical=True, ms_per_tick=ms)
    finally:
        for c in ctxs.values():
            c.close()
    line = json.dumps({k: v for k, v in res.items() if k != "ms_per_tick"})
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
