"""Where one iteration of the persistent VIO update goes, and what a change to it is worth, on the GPU.

For every library given with --lib NAME=PATH (ESIKF_LIB; the first is the one the others are compared against):

  breakdown: of the --stamped-lib NAME=PATH libraries (default: the --lib ones): the same sources built with
             -DESIKF_VIO_CHAIN_STAMPS, which the finer stamps need (they cost the kernel registers, so the libraries that
             are timed leave them out). Config 2, LIO + VIO update as bench.py's step, with phase stamps on (a separate,
             untimed pass). Per
             (level, iteration) slot, CTA 0's %globaltimer stamps split the iteration into
               consts      iteration start -> Rcw / Pcw / inv_expo in place
               projection  -> warp 0's first patch: projection and tap geometry done
               jacobian    -> its Jacobian constants (the 2 x 3 maps WR / WT) done
               grid        -> its bilinear value grid done (includes re-staging the tap footprint)
               rows_dmma   -> its 64 rows staged and contracted
               warp_exit   -> warp 0 left the slice
               cta_partial -> the CTA's 16 warps done and their partials summed (CTA 0's slice end)
               exchange    -> every CTA's contribution summed (all-gather complete)
               unpack      -> information vector in place
               gain, boxplus, solve_rest -> the replicated solve
             in us, averaged over the slots of --stamp-steps updates: all slots, level-entry slots (iteration 0, where
             the footprint and reference values are staged) and the rest. Also the spread of the CTAs' slice ends (each
             CTA's partial summed), in us after CTA 0's "consts" stamp. A library without the finer stamps reports only
             the coarse phases. "gain" and "boxplus" average the accepted iterations only.
  timing:    bench.py --no-cpu-baseline --no-shim, alternating the libraries: config 2 --cfg2-runs times each, the
             --configs --other-runs times each. Per library and config: bench's value and the LIO / VIO update durations
             in the timed region (min / median / max). The first run of every config writes bench.py --dump-outputs
             files, compared byte for byte with the first library's.

The card's name, power limit and maximum SM clock, and the SM clock bench.py sampled during each timed region, are read
in the same call.

    python tools/vio_chain_timing.py --lib parent=PATH --lib pr=PATH [--stamped-lib parent=PATH --stamped-lib pr=PATH]
                                     [--cfg2-runs 6] [--configs cfg3 cfg5] [--other-runs 2] [--out result.json]
"""
import argparse
import ctypes as C
import filecmp
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from lio_residency_timing import card, spread  # noqa: E402

SEGMENTS = ("consts", "projection", "jacobian", "grid", "rows_dmma", "warp_exit", "cta_partial", "exchange", "unpack", "gain", "boxplus", "solve_rest")
CHAIN_WORDS = 8 * 64 + 160 * 64  # ESIKF_VIO_CHAIN_STAMP_WORDS


def stamped_pass(steps):
    """In a child with ESIKF_LIB set: bench.py's config-2 step with phase stamps on; prints one JSON line."""
    import numpy as np
    import torch

    from fast_livo2_b200 import api, workloads
    from fast_livo2_b200 import synthetic as S

    fr = workloads.frame("cfg2")
    ctx = api.Context(0)
    ctx.set_extrinsics(fr["ext"])
    ctx.map_upload(fr["map"], fr["lio_cfg"].voxel_size)
    ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    pts_h, prior_h = pin(fr["pts"]), pin(fr["state_prior"])
    ctx.lio_set_scan(pts_h)
    ctx.lio_run(prior_h, prior_h, fr["lio_cfg"])
    post_h = pin(ctx.lio_fetch()["state"].copy())
    npatch, L, max_it = len(fr["vis_pos"]), fr["vio_cfg"].levels, fr["vio_cfg"].max_iterations
    ctx.vio_set_image(pin(fr["img"]))
    ctx.vio_set_ref_images([fr["img_ref"]])
    post = S.unpack_state(post_h.numpy())
    T_cur = api.pack_T(*S.camera_pose(fr["ext"], post["R"], post["p"]))
    w = ctx.vio_warp_patches(np.zeros(npatch, np.int32), fr["px_ref"], fr["vis_pos"], fr["vis_normal"], np.tile(api.pack_T(*fr["T_ref"]), (npatch, 1)), T_cur)
    keep = [pin(fr["vis_pos"]), pin(w["warp_patch"]), pin(w["search_levels"]), pin(fr["inv_ref_expo"])]
    ctx.vio_set_patches(*keep)
    lib = ctx.lib
    chain_ok = hasattr(lib, "esikf_get_vio_chain_stamps")
    if chain_ok:
        lib.esikf_get_vio_chain_stamps.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    ext_stream = torch.cuda.ExternalStream(ctx.stream)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def step():
        with torch.cuda.stream(ext_stream):
            flush.zero_()
        ctx.lio_run(prior_h, prior_h, fr["lio_cfg"])
        ctx.vio_run(post_h, post_h)

    for _ in range(3):
        step()
    ctx.set_phase_stamps(True)
    rows = {k: [] for k in ("all", "level_entry", "steady")}
    ends = []
    for _ in range(steps):
        step()
        ctx.synchronize()
        st = ctx.get_phase_stamps().astype(np.int64)
        ch = np.zeros(CHAIN_WORDS, np.uint64)
        if chain_ok:
            ctx._ck(lib.esikf_get_vio_chain_stamps(ctx.h, ch.ctypes.data_as(C.POINTER(C.c_uint64))))
        ch = ch.astype(np.int64)
        for slot in range(L * max_it):
            s = st[8 + slot]
            if s[0] <= 0 or s[5] <= 0:
                continue
            f = ch[8 * slot: 8 * slot + 4]
            cta = ch[512 + 160 * slot: 512 + 160 * (slot + 1)]
            cta = cta[cta > 0]
            fine = chain_ok and (f > 0).all() and len(cta) > 0
            t = [s[0], s[1], *(f if fine else [None] * 4), s[2], cta[0] if fine else None, s[3], s[4], s[6], s[7], s[5]]
            seg = {}
            for name, a, b in zip(SEGMENTS, t[:-1], t[1:]):
                seg[name] = (b - a) / 1e3 if a is not None and b is not None else None
            if not fine:  # coarse phases only: slice = consts in place -> warp 0 left the slice, exchange from there
                seg["exchange"] = (s[3] - s[2]) / 1e3
            if s[6] <= 0 or s[7] <= 0:  # rolled back: no gain, no boxplus
                seg["gain"] = seg["boxplus"] = None
                seg["solve_rest"] = (s[5] - s[4]) / 1e3
            seg["iteration"] = (s[5] - s[0]) / 1e3
            rows["all"].append(seg)
            rows["level_entry" if slot % max_it == 0 else "steady"].append(seg)
            if fine:
                ends.append((cta - s[1]) / 1e3)
    ctx.set_phase_stamps(False)
    ctx.close()
    mean = lambda rs, k: (float(np.mean([r[k] for r in rs if r[k] is not None])) if any(r[k] is not None for r in rs) else None)
    out = dict(fine_stamps=bool(ends), steps=steps,
               us_per_iteration={name: dict(slots=len(rs), **{k: mean(rs, k) for k in (*SEGMENTS, "iteration")}) for name, rs in rows.items()})
    if ends:
        e = np.concatenate(ends)
        last = np.array([x.max() for x in ends])
        out["cta_slice_end_us_after_consts"] = dict(ctas=int(len(ends[0])), min=float(e.min()), median=float(np.median(e)), max=float(e.max()),
                                                    slowest_cta_per_iteration_median=float(np.median(last)))
    print(json.dumps(out))


def bench(lib, config, steps, warmup, dump=None):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup), "--config", config, "--no-cpu-baseline", "--no-shim"]
    if dump:
        cmd += ["--dump-outputs", dump]
    r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, ESIKF_LIB=lib), capture_output=True, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        raise SystemExit(f"bench.py --config {config} with {lib} failed ({r.returncode}):\n{r.stderr[-3000:]}")
    out = json.loads(lines[-1])
    rl = out["roofline"]
    return dict(value=out["value"], lio_update_ms=rl["avg_launch_ms_in_timed_region"], vio_update_ms=rl.get("vio_update_ms_in_timed_region"),
                sm_mhz=out["clocks"].get("sm_mhz"), lio_iters=out["config"]["lio_iters"], vio_iters=out["config"]["vio_iters"], gpu_launches=out["gpu_launches"],
                parity_ok=out["parity_vs_oracle"]["ok"], repeatable=out["parity_vs_oracle"]["last_update_bit_identical_to_first"])


def same_dumps(a, b):
    fa, fb = set(os.listdir(a)), set(os.listdir(b))
    differ = sorted(fa ^ fb) + sorted(f for f in fa & fb if not filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False))
    return dict(files=len(fa & fb), differ=differ)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH")
    ap.add_argument("--stamped-lib", action="append", default=[], metavar="NAME=PATH")
    ap.add_argument("--cfg2-runs", type=int, default=6)
    ap.add_argument("--configs", nargs="*", default=["cfg3", "cfg5"])
    ap.add_argument("--other-runs", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--stamp-steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--stamped-pass", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.stamped_pass:
        stamped_pass(args.stamp_steps)
        return
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("vio_chain_timing: no CUDA device (the numbers are GPU timings; there is no CPU fallback)")
    libs = dict(kv.split("=", 1) for kv in args.lib) or {"tree": os.path.join(ROOT, "fast_livo2_b200", "libesikf_b200.so")}
    libs = {k: os.path.abspath(v) for k, v in libs.items()}
    stamped = {k: os.path.abspath(v) for k, v in (kv.split("=", 1) for kv in args.stamped_lib)} or libs
    res = dict(card=card(), libs=libs, stamped_libs=stamped, breakdown={}, runs={})
    for name, lib in stamped.items():
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--stamped-pass", "--stamp-steps", str(args.stamp_steps)], cwd=ROOT,
                           env=dict(os.environ, ESIKF_LIB=lib), capture_output=True, text=True)
        lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
        res["breakdown"][name] = json.loads(lines[-1]) if r.returncode == 0 and lines else dict(error=r.stderr[-3000:])
        print(f"breakdown {name}: {json.dumps(res['breakdown'][name].get('us_per_iteration', res['breakdown'][name]).get('all'))}", flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        plan = [("cfg2", args.cfg2_runs)] + [(c, args.other_runs) for c in args.configs]
        for config, runs in plan:
            for k in range(runs):
                for name, lib in libs.items():
                    dump = os.path.join(tmp, name, config) if k == 0 else None
                    r = bench(lib, config, args.steps, args.warmup, dump)
                    res["runs"].setdefault(config, {}).setdefault(name, []).append(r)
                    print(f"{config} {name} run {k}: value={r['value']:.1f} lio_update_ms={r['lio_update_ms']:.4f} vio_update_ms={r['vio_update_ms']}", flush=True)
        first = next(iter(libs))
        res["dumps_identical_to_" + first] = {config: {name: same_dumps(os.path.join(tmp, first, config), os.path.join(tmp, name, config)) for name in libs if name != first}
                                             for config, _ in plan}
    res["summary"] = {config: {name: {k: spread([r[k] for r in rs]) for k in ("value", "lio_update_ms", "vio_update_ms", "sm_mhz")}
                               | {k: sorted({r[k] for r in rs}) for k in ("gpu_launches", "lio_iters", "vio_iters")}
                               | dict(parity_ok=all(r["parity_ok"] for r in rs), repeatable=all(r["repeatable"] for r in rs))
                               for name, rs in per.items()}
                      for config, per in res["runs"].items()}
    print(json.dumps({k: res[k] for k in res if k != "runs"}, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
