"""What a change to the library is worth on the GPU: bench.py against whole library builds of the persistent update kernels,
alternating between them, with the per-iteration stamps of each build.

For every library given with --lib NAME=PATH (ESIKF_LIB; the first is the one the others are compared against; default:
the tree's library):

  timing:  bench.py --no-cpu-baseline --no-shim, alternating the libraries: config 2 (bench.py's metric) --cfg2-runs times
           each, the --configs --other-runs times each. Per library and config: bench's value, the LIO / VIO update
           durations in the timed region (roofline.avg_launch_ms_in_timed_region, vio_update_ms_in_timed_region), the
           residual-build phase stamps (roofline.residual_build_phase) and the SM clock bench.py sampled (min / median / max
           over the runs); iteration, matched-point and launch counts; parity with the oracle and repeatability. The first
           run of every config writes bench.py --dump-outputs files, compared byte for byte with the first library's.
  stamped: for each --stamped-lib NAME=PATH (default: the --lib ones), in a child process with phase stamps on (untimed):
    lio_slice_ends: config 2's LIO update, when each CTA finished its slice of iteration 3 (stamps[640 + b]), in us after
                    CTA 0's "constants in place" stamp of that iteration, and the all-arrived stamp; over 5 updates.
    vio_chain:      config 2's LIO + VIO update as bench.py's step. Per (level, iteration) slot, CTA 0's %globaltimer
                    stamps split the iteration into
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
                    in us, averaged over the slots of --stamp-steps updates: all slots, level-entry slots (iteration 0,
                    where the footprint and reference values are staged) and the rest. Also the spread of the CTAs' slice
                    ends, in us after CTA 0's "consts" stamp. The finer stamps need a library built with
                    -DESIKF_VIO_CHAIN_STAMPS (build() makes one: variants/chain_stamps); they cost the kernel registers, so
                    the libraries that are timed leave them out, and a library without them reports only the coarse phases.
                    "gain" and "boxplus" average the accepted iterations only.

The card's name, power limit and maximum SM clock are read in the same call. The script builds nothing; build() has made
the tree's library and its variants. The comparisons recorded in DESIGN.md section 8:

  L2 residency (768-lane CTAs against the 704-lane build of the same sources):
    python tools/ab_timing.py --lib l2w2=fast_livo2_b200/libesikf_b200.so --lib l2w0=fast_livo2_b200/variants/l2w0/libesikf_b200.so \\
                              --configs cfg4 cfg5 --other-runs 3
  grid exchange (a parent revision's library, built with the same flags, against this tree's):
    python tools/ab_timing.py --lib parent=PATH --lib new=fast_livo2_b200/libesikf_b200.so --configs cfg3 cfg4 cfg5
  VIO chain (the parent's and this tree's libraries, each with its chain-stamps build for the breakdown):
    python tools/ab_timing.py --lib parent=PATH --lib pr=fast_livo2_b200/libesikf_b200.so \\
                              --stamped-lib parent=PATH --stamped-lib pr=fast_livo2_b200/variants/chain_stamps/libesikf_b200.so
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
import timing as T  # noqa: E402

SEGMENTS = ("consts", "projection", "jacobian", "grid", "rows_dmma", "warp_exit", "cta_partial", "exchange", "unpack", "gain", "boxplus", "solve_rest")
CHAIN_WORDS = 8 * 64 + 160 * 64  # ESIKF_VIO_CHAIN_STAMP_WORDS
SUMMARY_SPREADS = ("value", "lio_update_ms", "vio_update_ms", *T.PHASE_KEYS, "sm_mhz")
SUMMARY_SETS = ("gpu_launches", "lio_iters", "vio_iters", "matched_points")


def lio_slice_ends():
    """Config 2's LIO update with phase stamps: per-CTA slice ends of iteration 3 (us after CTA 0's 'constants in place'
    stamp of that iteration) and the all-arrived stamp."""
    import numpy as np
    import torch

    from fast_livo2_b200 import api, workloads

    fr = workloads.frame("cfg2")
    ctx = api.Context(0)
    ctx.set_extrinsics(fr["ext"])
    ctx.map_upload(fr["map"], fr["lio_cfg"].voxel_size)
    ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], fr["lio_cfg"])
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ctx.set_phase_stamps(True)
    ends, arrived = [], []
    for _ in range(5):
        flush.zero_()
        torch.cuda.synchronize()
        ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], fr["lio_cfg"])
        st = ctx.get_phase_stamps().astype(np.int64)
        t0 = st[3, 1]
        cta = ctx.cta_stamps.astype(np.int64)
        cta = cta[cta > 0]
        if t0 > 0 and len(cta):
            ends.append((cta - t0) / 1e3)
            arrived.append((st[3, 3] - t0) / 1e3)
    ctx.set_phase_stamps(False)
    ctx.close()
    e = np.concatenate(ends)
    per_run = [dict(min=float(x.min()), median=float(np.median(x)), max=float(x.max())) for x in ends]
    return dict(ctas=int(len(ends[0])), slice_end_us_min=float(e.min()), slice_end_us_median=float(np.median(e)), slice_end_us_max=float(e.max()),
                all_arrived_us=float(np.median(arrived)), per_run=per_run)


def vio_chain(steps):
    """bench.py's config-2 step with phase stamps on: the per-segment breakdown of the VIO iteration."""
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
    return out


def main():
    ap = argparse.ArgumentParser(description="bench.py against whole library builds, alternating, with each build's stamped passes")
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
        print(json.dumps(dict(lio_slice_ends=lio_slice_ends(), vio_chain=vio_chain(args.stamp_steps))))
        return
    T.require_gpu("ab_timing")
    libs = {k: os.path.abspath(v) for k, v in (kv.split("=", 1) for kv in args.lib)} or {"tree": T.TREE_LIB}
    stamped = {k: os.path.abspath(v) for k, v in (kv.split("=", 1) for kv in args.stamped_lib)} or libs
    res = dict(card=T.card(), libs=libs, stamped_libs=stamped, stamped={}, runs={})
    for name, lib in stamped.items():
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--stamped-pass", "--stamp-steps", str(args.stamp_steps)], cwd=ROOT,
                           env=dict(os.environ, ESIKF_LIB=lib), capture_output=True, text=True)
        lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
        s = res["stamped"][name] = json.loads(lines[-1]) if r.returncode == 0 and lines else dict(error=r.stderr[-3000:])
        print(f"stamped {name}: " + (s["error"][-500:] if "error" in s else json.dumps(s["vio_chain"]["us_per_iteration"]["all"])), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        plan = [("cfg2", args.cfg2_runs)] + [(c, args.other_runs) for c in args.configs]
        for config, runs in plan:
            for k in range(runs):
                for name, lib in libs.items():
                    dump = os.path.join(tmp, name, config) if k == 0 else None
                    r = T.bench_run(lib, config, args.steps, args.warmup, dump)
                    res["runs"].setdefault(config, {}).setdefault(name, []).append(r)
                    print(f"{config} {name} run {k}: value={r['value']:.1f} lio_update_ms={r['lio_update_ms']:.4f} vio_update_ms={r['vio_update_ms']}", flush=True)
        first = next(iter(libs))
        res["dumps_identical_to_" + first] = {config: {name: T.same_dumps(os.path.join(tmp, first, config), os.path.join(tmp, name, config)) for name in libs if name != first}
                                             for config, _ in plan}
    res["summary"] = {config: {name: {k: T.spread([r[k] for r in rs]) for k in SUMMARY_SPREADS}
                               | {k: sorted({r[k] for r in rs}) for k in SUMMARY_SETS}
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
