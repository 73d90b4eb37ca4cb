"""Time the coloured scan (esikf_rgb_set_cloud + esikf_rgb_colorize) on config-2-shaped frames (pinhole 640 x 512, avia
extrinsics) of 100 k and 300 k LiDAR points, against the single-threaded host loop of the oracle's restatement
(oracle/orc_color.cpp, the reference's arithmetic) on the same frames:

  api       : both calls with the host cloud, the image upload and the download of the result (CUDA events on the context's
              stream around calls that end in a device synchronise; host clock alongside)
  kernels   : the device time of the kernels alone (rgb_world, rgb_color, the two of cub's device-wide scan, rgb_scatter),
              from a torch.profiler run of its own, per tick
  host loop : orc_color_world + orc_color_colorize, one thread

The kept sets of the device and the oracle are checked to be equal. The card's name and power limit are printed in the same
run. Writes nothing; needs a GPU.

  python tools/colorize_timing.py [--reps 30]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402

import color_cases as CC  # noqa: E402
from fast_livo2_b200 import api  # noqa: E402
from fast_livo2_b200 import synthetic as S  # noqa: E402

KERNELS = ("rgb_world_kernel", "rgb_color_kernel", "DeviceScan", "rgb_scatter_kernel")  # DeviceScan: cub's init + scan kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"device: {q.splitlines()[0] if q else torch.cuda.get_device_name(0)}")
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
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        for _ in range(args.reps):
            once()
        e1.record(stream)
        ctx.synchronize()
        e1.synchronize()
        wall = (time.perf_counter() - t0) / args.reps * 1e3
        print(f"n={n} api (H2D cloud + image, D2H result)  events {e0.elapsed_time(e1) / args.reps:.3f} ms/tick  host {wall:.3f} ms/tick  kept={len(got['index'])}")

        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                once()
            ctx.synchronize()
        per = {k: [] for k in KERNELS}
        for ev in prof.events():
            for k in KERNELS:
                if k in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
                    per[k].append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)
        tot = 0.0
        parts = []
        for k in KERNELS:
            us = float(np.sum(per[k])) / args.reps if per[k] else float("nan")  # per tick
            tot += us
            parts.append(f"{k} {us:.1f} us")
        print(f"n={n} kernels {tot / 1e3:.3f} ms/tick: " + ", ".join(parts))

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
