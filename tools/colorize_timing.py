"""Time the coloured scan (esikf_rgb_set_cloud + esikf_rgb_colorize) on config-2-shaped frames (pinhole 640 x 512, avia
extrinsics) of 100 k and 300 k LiDAR points, against the single-threaded host loop of the oracle's restatement
(oracle/orc_color.cpp, the reference's arithmetic) on the same frames:

  api       : both calls with the host cloud, the image upload and the download of the result (CUDA events on the context's
              stream around calls that end in a device synchronise; host clock alongside)
  kernels   : the device time of the kernels alone (rgb_world, rgb_color, the two of cub's device-wide scan, rgb_scatter),
              from a torch.profiler run of its own, per tick
  host loop : orc_color_world + orc_color_colorize, one thread

The kept sets of the device and the oracle are checked to be equal. The card's name, power limit and maximum SM clock are printed in the same
run. Writes nothing; needs a GPU.

  python tools/colorize_timing.py [--reps 30]"""
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

import color_cases as CC  # noqa: E402
from fast_livo2_b200 import api  # noqa: E402
from fast_livo2_b200 import synthetic as S  # noqa: E402

KERNELS = ("rgb_world_kernel", "rgb_color_kernel", "DeviceScan", "rgb_scatter_kernel")  # DeviceScan: cub's init + scan kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    T.require_gpu("colorize_timing")
    print(f"device: {json.dumps(T.card())}")
    ctx = api.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    for n in (100_000, 300_000):
        sc = CC.scene("pinhole", n, seed=7)
        ctx.set_extrinsics(sc["ext"])
        ctx.vio_set_camera(sc["cam"], S.VioCfg())

        def once():
            ctx.rgb_set_cloud(sc["pts"], sc["lio_state"])
            return ctx.rgb_colorize(sc["img"], sc["blind"], state=sc["vio_state"])

        for _ in range(5):
            got = once()
        ctx.synchronize()
        ev, wall = T.window_ms(stream, once, args.reps)
        print(f"n={n} api (H2D cloud + image, D2H result)  events {ev:.3f} ms/tick  host {wall:.3f} ms/tick  kept={len(got['index'])}")

        us = {k: float(np.sum(v)) / args.reps if v else float("nan") for k, v in T.kernel_us(once, args.reps, KERNELS).items()}  # per tick
        print(f"n={n} kernels {sum(us.values()) / 1e3:.3f} ms/tick: " + ", ".join(f"{k} {v:.1f} us" for k, v in us.items()))

        o = CC.OracleColor(sc)
        t0 = time.perf_counter()
        for _ in range(3):
            want = o.publish(sc)
        host = (time.perf_counter() - t0) / 3 * 1e3
        print(f"n={n} host loop (oracle restatement, 1 thread) {host:.3f} ms/tick")
        assert np.array_equal(got["index"], want["index"]) and got["bgr"].tobytes() == want["bgr"].tobytes(), "device and oracle differ"
    ctx.close()


if __name__ == "__main__":
    main()
