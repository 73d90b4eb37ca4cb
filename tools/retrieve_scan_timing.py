"""Time the scan side of the visual sub-map retrieval (esikf_vio_retrieve_scan + esikf_vio_depth_check) on config 2's camera
(pinhole 640 x 512, avia extrinsics) at 100 k and 300 k scan points, against the single-threaded host loop of the oracle's
restatement of vio.cpp:386-428 + 605-640 (oracle/orc_retrieve.cpp, the reference's arithmetic) on the same frames:

  api host     : both calls with the scan from host buffers (CUDA events on the context's stream around calls that end in a
                 device synchronise; host clock alongside)
  api resident : both calls on the pv list a map_device_update left on the device (pg = NULL)
  kernels      : the device time of the kernels alone, from a torch.profiler run of its own, per tick
  host loop    : orc_retrieve_scan + orc_depth_check, one thread

The device's keys, depth image and flags are checked against the oracle's. The card's name, power limit and maximum SM clock are printed in the
same run. Writes nothing; needs a GPU.

  python tools/retrieve_scan_timing.py [--reps 30]"""
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

import retrieve_cases as RC  # noqa: E402
from fast_livo2_b200 import api  # noqa: E402
from fast_livo2_b200 import synthetic as S  # noqa: E402

KERNELS = ("ret_scan_kernel", "ret_depth_kernel", "DeviceRadixSort", "ret_head_kernel", "DeviceScan", "ret_keys_kernel", "ret_depth_check_kernel")


def timed(ctx, stream, fn, reps):
    for _ in range(3):
        fn()
    ctx.synchronize()
    return T.window_ms(stream, fn, reps)


def resident_scan(ctx, sc):
    """The scene's scan as the resident pv list: body points = world points under an identity LIO posterior."""
    cfg = S.LioCfg()
    st = S.pack_state(np.eye(3), np.zeros(3))
    ext = S.Extrinsics(extR=np.eye(3), extT=np.zeros(3), Rcl=sc["ext"].Rcl, Pcl=sc["ext"].Pcl)
    ctx.set_extrinsics(ext)
    ctx.map_device_init(cfg, root_capacity=1 << 20, grow=True)
    pts = np.ascontiguousarray(sc["pg"], np.float32)
    ctx.lio_set_scan(pts)
    ctx.map_device_build(st)
    ctx.lio_update(pts, st, st, cfg)
    ctx.map_device_update(st)
    return ext


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    T.require_gpu("retrieve_scan_timing")
    print(f"device: {json.dumps(T.card())}")
    ctx = api.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    for n in (100_000, 300_000):
        sc = RC.scene("pinhole", n, seed=31, n_vis=6000)
        ctx.set_extrinsics(sc["ext"])
        ctx.vio_set_camera(sc["cam"], RC.VIO_CFG)
        orc = RC.OracleRetrieve(sc)
        want = orc.retrieve(sc)
        pos, pc = sc["pos"][want["cell_pt"][want["cells"]]], want["cell_pc"][want["cells"]]
        pg, st = np.ascontiguousarray(sc["pg"]), np.ascontiguousarray(sc["state"])

        def host_call():
            r = ctx.vio_retrieve_scan(sc["border"], pg=pg, state=st, cap=len(pg))
            return r, ctx.vio_depth_check(pos, pc)

        got, flags = host_call()
        assert np.array_equal(got["keys"].astype(np.int64), want["keys"]) and flags.tobytes() == want["flag"].tobytes()
        assert ctx.vio_retrieve_scan(sc["border"], pg=pg, state=st, depth=True)["depth"].tobytes() == want["depth"].tobytes()
        ev, wall = timed(ctx, stream, host_call, args.reps)
        print(f"n={n} api host buffers (retrieve_scan + depth_check of {len(pos)} points)  events {ev:.3f} ms/tick  host {wall:.3f} ms/tick  keys={len(want['keys'])}")

        per = {k: sum(v) for k, v in T.kernel_us(host_call, args.reps, KERNELS).items()}
        tot = sum(per.values()) / args.reps
        print(f"n={n} kernels {tot / 1e3:.4f} ms/tick: " + ", ".join(f"{k} {v / args.reps:.1f} us" for k, v in per.items()))

        try:
            rctx = api.Context(0)
            ext = resident_scan(rctx, sc)
            rctx.vio_set_camera(sc["cam"], RC.VIO_CFG)
            k_res = len(rctx.vio_retrieve_scan(sc["border"], state=st)["keys"])

            def res_call():
                rctx.vio_retrieve_scan(sc["border"], state=st, cap=k_res)
                return rctx.vio_depth_check(pos, pc)

            rstream = torch.cuda.ExternalStream(rctx.stream)
            ev, wall = timed(rctx, rstream, res_call, args.reps)
            print(f"n={n} api resident pv list (retrieve_scan(NULL) + depth_check)  events {ev:.3f} ms/tick  host {wall:.3f} ms/tick  keys={k_res}")
            rctx.close()
        except Exception as e:  # noqa: BLE001
            print(f"n={n} api resident pv list: not measured ({e})")

        reps = 5
        t0 = time.perf_counter()
        for _ in range(reps):
            s = orc.scan(sc)
            orc.depth_check(sc, s["depth"], pos, pc)
        print(f"n={n} host loop (oracle restatement of :386-428 + :605-640, 1 thread) {(time.perf_counter() - t0) / reps * 1e3:.3f} ms/tick")
    ctx.close()


if __name__ == "__main__":
    main()
