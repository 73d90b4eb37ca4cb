"""What the patch scoring of updateReferencePatch costs on the device (esikf_vio_score_ref_patches, K13) against the host loops
it replaces, on realistic observation sets (tests/refpatch_cases.realistic_case: the visual points of a keyframe frame, each
observed in exactly k of 30 keyframe images, patches cut by the device's image_patch_kernel, half the means cached).

For 2 k and 4 k points with k = 6, 15 and 30 observations:
  kernel  : refpatch_score_kernel's time from torch.profiler (median over --reps calls);
  call    : the call through the C ABI (uploads, kernel, one copy back; it returns synchronised): CUDA events on the context's
            stream around it, and the host wall time (medians over --reps calls);
  host    : the reference source's own updateReferencePatch with an empty plane map (oracle/_ref/libfl2_ref_refpatch.so, where
            it was built: only the scoring runs) and the oracle's restatement (oracle/liborc_refpatch.so), single-threaded on
            the same points (medians over --host-reps runs);
  upload  : the bytes the call copies to the device.

Prints one JSON line with the card's name, power limit and maximum SM clock read in the same run.

    python tools/refpatch_timing.py [--reps 50] [--host-reps 5] [--out result.json]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import timing as T  # noqa: E402

SIZES = (2000, 4000)
OBS = (6, 15, 30)


def _call(ctx, c):
    return ctx.vio_score_ref_patches(c["first"], c["pos"], c["normal"], c["patch"], c["mean"], c["id"], c["T"])


def _kernel_ms(ctx, c, reps):
    us = T.kernel_us(lambda: _call(ctx, c), reps, ("refpatch_score_kernel",))["refpatch_score_kernel"]
    assert us, "no refpatch_score_kernel in the trace"
    return statistics.median(us) / 1e3


def _orc_ms(c):
    import refpatch_cases as RC

    L = C.CDLL(RC.ORC_SO)
    L.orc_score_ref_patches.argtypes = [C.c_int] + [C.c_void_p] * 10
    n, m = len(c["first"]) - 1, len(c["patch"])
    outs = [np.zeros(m, np.float32), np.zeros(m, np.float32), np.zeros(n, np.int32)]
    ins = [np.ascontiguousarray(c[k]) for k in ("first", "pos", "normal", "patch", "mean", "id", "T")]
    t0 = time.perf_counter()
    L.orc_score_ref_patches(n, *[x.ctypes.data for x in ins], *[o.ctypes.data for o in outs])
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    T.require_gpu("refpatch_timing")
    import refpatch_cases as RC
    import torch
    from fast_livo2_b200 import api
    from fast_livo2_b200 import synthetic as S

    ctx = api.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    res = dict(what="realistic observation sets (tests/refpatch_cases.realistic_case), k observations per point", **T.card(), rows=[])
    for n in SIZES:
        for k in OBS:
            c = RC.realistic_case(ctx, n, seed=n + k, lo=k, hi=k)
            m = len(c["patch"])
            for _ in range(5):
                _call(ctx, c)
            ev_ms, wall_ms = T.per_call_ms(stream, lambda: _call(ctx, c), args.reps)
            row = dict(points=n, obs_per_point=k, observations=m, kernel_ms=round(_kernel_ms(ctx, c, args.reps), 4),
                       call_event_ms=round(statistics.median(ev_ms), 4), call_wall_ms=round(statistics.median(wall_ms), 4),
                       upload_bytes=int(m * (64 * 4 + 4 + 4 + 12 * 8) + n * (6 * 8 + 4) + 4),
                       orc_host_ms=round(statistics.median(_orc_ms(c) for _ in range(args.host_reps)), 3))
            if RC.ref_available():
                secs = [RC.reference(c, S.CamCfg(), S.avia_extrinsics(), S.VioCfg(), timed=True)[1] for _ in range(args.host_reps)]
                row["ref_host_ms"] = round(statistics.median(secs) * 1e3, 3)
            else:
                row["ref_host_ms"] = "not measured (oracle/_ref not built)"
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
