"""Time the map side of the visual sub-map retrieval (esikf_vmap_retrieve: walk, grid argmin, depth check, skip and reference
choice) on config 2's camera (pinhole 640 x 512, avia extrinsics) with visual maps of about 20 k, 100 k and 400 k placed points
and the scan keys of one frame, against host walks on the same frames:

  call        : esikf_vmap_retrieve (CUDA events on the context's stream around calls that end in a device synchronise;
                host clock alongside), normal_en on
  kernels     : the device time of its kernels alone, from a torch.profiler run of its own, per call
  host walk   : the restatement's orc_retrieve_walk (oracle/orc_retrieve.cpp, one thread): the walk and grid argmin only
  reference   : the reference source's own retrieveFromVisualSparseMap (oracle/_ref/libfl2_ref_vretrieve.so, where it was
                built), the whole retrieval with its scan side and the per-point warps after the choice

The device's cells are checked against the restatement first. The card's name, power limit and maximum SM clock are printed in the same run.
Writes nothing; needs a GPU.

  python tools/vmap_retrieve_timing.py [--reps 30]"""
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
import vmap_retrieve_cases as VR  # noqa: E402
from fast_livo2_b200 import api  # noqa: E402

KERNELS = ("vrt_hash_kernel", "vrt_init_kernel", "vrt_walk_kernel", "ret_depth_check_kernel", "vrt_cells_kernel", "select_scan_kernel",
           "vmap_choose_kernel", "vrt_refs_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    T.require_gpu("vmap_retrieve_timing")
    print("card:", json.dumps(T.card()))
    for n_vis in (20_000, 100_000, 400_000):
        sc = RC.scene("pinhole", max(n_vis, 100_000), seed=11, n_vis=n_vis)
        n = len(sc["pos"])
        order = np.random.default_rng(1).permutation(n).astype(np.int32)
        ctx = api.Context(0)
        try:
            ctx.set_extrinsics(sc["ext"])
            ctx.vio_set_camera(sc["cam"], RC.VIO_CFG)
            ctx.vmap_init(n)
            first = np.concatenate([[0], np.cumsum(sc["n_obs"])]).astype(np.int32)
            m = int(first[-1])
            T_f_w = np.zeros((m, 12))
            T_f_w[:, [0, 4, 8]] = 1.0
            rng = np.random.default_rng(2)
            ctx.vmap_add_points(first, np.zeros((m, 2)), rng.uniform(0, 255, (m, 64)).astype(np.float32), T_f_w, (np.arange(m) % 3).astype(np.int32),
                                np.zeros(m, np.float32), np.zeros(m, np.float32), np.full(n, -1, np.int32))
            ctx.vmap_place_points(order, sc["pos"][order])
            dev = ctx.vio_retrieve_scan(sc["border"], pg=sc["pg"], state=sc["state"], depth=True)
            orc = RC.OracleRetrieve(sc)
            s = orc.scan(sc)
            vis = VR.placed_visual_map(sc["pos"], sc["n_obs"], order)
            walk, want = VR.composed(orc, sc, vis, s["keys"], dev["depth"], np.ones(n, np.uint8))
            g = [int(sc[k]) for k in ("grid_size", "grid_n_width", "grid_n_height", "border")]
            got = ctx.vmap_retrieve(walk, *g, True)
            assert np.array_equal(got["cell"], want["cell"]) and np.array_equal(got["point_id"], want["point_id"])
            call = lambda: ctx.vmap_retrieve(walk, *g, True)  # noqa: E731
            stream = torch.cuda.ExternalStream(ctx.stream)
            for _ in range(3):
                call()
            ev, wall = T.window_ms(stream, call, args.reps)
            print(f"points={n} keys={len(walk)} cells={len(got['cell'])}  call: events {ev:.3f} ms  host {wall:.3f} ms")
            per = {k: sum(v) for k, v in T.kernel_us(call, args.reps, KERNELS).items()}
            print(f"points={n} kernels {sum(per.values()) / args.reps / 1e3:.4f} ms/call: " + ", ".join(f"{k} {v / args.reps:.1f} us" for k, v in per.items()))
            s2 = dict(sc, **vis)
            t0 = time.perf_counter()
            for _ in range(args.reps):
                orc.walk(s2, s["keys"])
            print(f"points={n} host walk (restatement, one thread) {(time.perf_counter() - t0) / args.reps * 1e3:.3f} ms")
            if VR.ref_vretrieve_available():
                ref = VR.RefVretrieve(sc)
                tk = dict(order=order, ids=np.arange(n, dtype=np.int32), first=first, pos=sc["pos"], normal=sc["normal"], ninit=np.ones(n, np.uint8),
                          patch=np.zeros((m, 64), np.float32), fid=(np.arange(m) % 3).astype(np.int32), T=T_f_w)
                ref.place(tk)
                ref.retrieve(sc, True)
                t0 = time.perf_counter()
                for _ in range(max(args.reps // 10, 3)):
                    ref.retrieve(sc, True)
                print(f"points={n} reference retrieveFromVisualSparseMap (whole) {(time.perf_counter() - t0) / max(args.reps // 10, 3) * 1e3:.3f} ms")
            else:
                print(f"points={n} reference: not measured (oracle/_ref not built)")
        finally:
            ctx.close()


if __name__ == "__main__":
    main()
