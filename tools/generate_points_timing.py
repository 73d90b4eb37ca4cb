"""Time the new visual map points of a VIO tick (esikf_vio_generate_points) on config-2-shaped frames (pinhole 640 x 512, avia
extrinsics, 30-pixel cells, border 80) of 100 k and 300 k scan points with 300 add_from points, against the single-threaded
host loop of the oracle's restatement (oracle/orc_generate.cpp, the reference's arithmetic) on the same frames:

  api       : the call with the scan from the host (its upload is 120 bytes a point: 12 / 36 MB), the mask and the download
              of the winners (CUDA events on the context's stream around a call that ends in a device synchronise; host clock
              alongside). The resident form skips the scan's upload.
  kernels   : the device time of the kernels alone (gen_score, gen_cells, select_scan, gen_scatter, image_patch), from a
              torch.profiler run of its own, per tick
  host loop : orc_generate_points, one thread

The winners of the device and the oracle are checked to be equal. The card's name, power limit and maximum SM clock are printed in the same
run. Writes nothing; needs a GPU.

  python tools/generate_points_timing.py [--reps 30]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import timing as T  # noqa: E402
import torch  # noqa: E402

import generate_cases as GC  # noqa: E402
from fast_livo2_b200 import api  # noqa: E402
from fast_livo2_b200 import synthetic as S  # noqa: E402

KERNELS = ("gen_score_kernel", "gen_cells_kernel", "select_scan_kernel", "gen_scatter_kernel", "image_patch_kernel")
GEOM = ("grid_size", "grid_n_width", "grid_n_height", "border")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    T.require_gpu("generate_points_timing")
    print(f"device: {json.dumps(T.card())}")
    ctx = api.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    for n in (100_000, 300_000):
        sc = GC.scene("pinhole", n, seed=7)
        ctx.set_extrinsics(sc["ext"])
        ctx.vio_set_camera(sc["cam"], S.VioCfg())
        ctx.vio_set_image(sc["img"])

        def once():
            return ctx.vio_generate_points(sc["mask"], *[sc[k] for k in GEOM], pg=(sc["point_w"], sc["normal"], sc["var"]),
                                           add_from=(sc["add_pos"], sc["add_normal"]), state=sc["state"])

        for _ in range(5):
            got = once()
        ctx.synchronize()
        ev, wall = T.window_ms(stream, once, args.reps)
        print(f"n={n} api (H2D scan + mask, D2H winners)  events {ev:.3f} ms/tick  host {wall:.3f} ms/tick  "
              f"new points={len(got['cell'])}")

        us = {k: float(np.sum(v)) / args.reps if v else float("nan") for k, v in T.kernel_us(once, args.reps, KERNELS).items()}  # per tick
        print(f"n={n} kernels {sum(us.values()) / 1e3:.3f} ms/tick: " + ", ".join(f"{k} {v:.1f} us" for k, v in us.items()))

        o = GC.OracleGenerate(sc)
        t0 = time.perf_counter()
        for _ in range(3):
            want = o.run(sc)
        host = (time.perf_counter() - t0) / 3 * 1e3
        print(f"n={n} host loop (oracle restatement, 1 thread) {host:.3f} ms/tick")
        for k in GC.FIELDS:
            assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(want[k]).tobytes(), f"device and oracle differ in {k}"
    ctx.close()


if __name__ == "__main__":
    main()
