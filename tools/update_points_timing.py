"""Time the new observations of the visual sub-map in a VIO tick (esikf_vio_update_points) on config 2's camera (pinhole
640 x 512, avia extrinsics) with sub-maps of 2 k and 10 k entries installed on the device, against the single-threaded host
loop of the oracle's restatement (oracle/orc_observe.cpp, the reference's arithmetic) on the same frames:

  api       : the call with the entries' converged flags and oldest observations from the host (113 bytes an entry), the
              flags and the added entries' pc and patches back (CUDA events on the context's stream around a call that ends
              in a device synchronise; host clock alongside)
  kernels   : the device time of the kernels alone (obs_flag, select_scan, obs_scatter, image_patch), from a torch.profiler
              run of its own, per tick
  host loop : orc_update_points, one thread

The outputs of the device and the oracle are checked to be equal. The card's name, power limit and maximum SM clock are printed in the same
run. Writes nothing; needs a GPU.

  python tools/update_points_timing.py [--reps 50]"""
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

import observe_cases as OC  # noqa: E402
from fast_livo2_b200 import api  # noqa: E402
from fast_livo2_b200 import synthetic as S  # noqa: E402

KERNELS = ("obs_flag_kernel", "select_scan_kernel", "obs_scatter_kernel", "image_patch_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    T.require_gpu("update_points_timing")
    print(f"device: {json.dumps(T.card())}")
    ctx = api.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    for n in (2000, 10_000):
        sc = OC.scene("pinhole", n, seed=9)
        ctx.set_extrinsics(sc["ext"])
        ctx.vio_set_camera(sc["cam"], S.VioCfg())
        ctx.vio_set_image(sc["img"])
        ctx.vio_set_patches(np.ascontiguousarray(sc["pos"]), np.zeros((n, 4 * 64), np.float32), np.ascontiguousarray(sc["search_levels"]), np.ones(n))

        def once():
            return ctx.vio_update_points(sc["converged"], sc["last_T"], sc["last_px"], state=sc["state"])

        for _ in range(5):
            got = once()
        ctx.synchronize()
        ev, wall = T.window_ms(stream, once, args.reps)
        print(f"n={n} api (H2D entries, D2H flags + added entries)  events {ev:.3f} ms/tick  host {wall:.3f} ms/tick  "
              f"added={len(got['entry'])}")

        us = {k: float(np.sum(v)) / args.reps if v else float("nan") for k, v in T.kernel_us(once, args.reps, KERNELS).items()}  # per tick
        print(f"n={n} kernels {sum(us.values()) / 1e3:.4f} ms/tick: " + ", ".join(f"{k} {v:.1f} us" for k, v in us.items()))

        o = OC.OracleObserve(sc)
        reps = 20
        t0 = time.perf_counter()
        for _ in range(reps):
            want = o.run(sc)
        host = (time.perf_counter() - t0) / reps * 1e3
        print(f"n={n} host loop (oracle restatement, 1 thread) {host:.3f} ms/tick")
        for k in OC.FIELDS:
            assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(want[k]).tobytes(), f"device and oracle differ in {k}"
    ctx.close()


if __name__ == "__main__":
    main()
