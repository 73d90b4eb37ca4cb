"""What keeping the 100 k-point LIO slice resident is worth on the GPU: the library built twice from the same sources,

  l2w2: LIO_L2_WARPS=2 (768-lane CTAs, lanes 704-767 keep their slots in an L2-resident global block, the default);
  l2w0: LIO_L2_WARPS=0 (704-lane CTAs, all slots in shared memory: the 132 x 704 = 92.9 k geometry),

and bench.py run against each (ESIKF_LIB), alternating between the two: cfg2 (bench.py's metric) --cfg2-runs times per
build, then cfg4 and cfg5 --other-runs times per build. Per build and config it reports bench's `value`, the persistent
LIO update's duration in the timed region (roofline.avg_launch_ms_in_timed_region) and the residual-build phase stamps
(roofline.residual_build_phase), as min / median / max over the runs. A separate pass per build runs cfg2's LIO update
with phase stamps on and reports when each CTA finished its slice of iteration 3 (stamps[640 + b]), counted from CTA 0's
"constants in place" stamp of that iteration: the spread over the CTAs. The card's name and power limit are read in the
same run. --dump DIR additionally writes each build's `bench.py --dump-outputs` files of its first run of every config to
DIR/<build>/<config>.

    python tools/lio_residency_timing.py [--cfg2-runs 6] [--other-runs 3] [--out result.json] [--dump DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BUILDS = {"l2w2": 2, "l2w0": 0}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
    return q.stdout.strip() or "not available"


def build_all(out_dir):
    """Both libraries, compiled with the flags of __graft_entry__.build()."""
    import __graft_entry__ as G

    libs = {}
    for name, w in BUILDS.items():
        os.makedirs(os.path.join(out_dir, name), exist_ok=True)
        libs[name] = os.path.join(out_dir, name, "libesikf_b200.so")
        G.build_library(libs[name], [f"-DLIO_L2_WARPS={w}"], force=True)
    return libs


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
    ph = rl.get("residual_build_phase") or {}
    return dict(value=out["value"], lio_update_ms=rl["avg_launch_ms_in_timed_region"], lio_build_us_per_iteration=ph.get("lio_build_us_per_iteration"),
                lio_iteration_us=ph.get("lio_iteration_us"), lio_iters=out["config"]["lio_iters"], matched_points=out["config"]["matched_points"],
                parity_ok=out["parity_vs_oracle"]["ok"], repeatable=out["parity_vs_oracle"]["last_update_bit_identical_to_first"])


def cta_stamps():
    """Run in a child with ESIKF_LIB set: cfg2's LIO update with phase stamps, per-CTA slice ends of iteration 3 (us after
    CTA 0's 'constants in place' stamp of that iteration) and the all-arrived stamp."""
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
    print(json.dumps(dict(ctas=int(len(ends[0])), slice_end_us_min=float(e.min()), slice_end_us_median=float(np.median(e)), slice_end_us_max=float(e.max()),
                          all_arrived_us=float(np.median(arrived)), per_run=per_run)))


def spread(xs):
    xs = [x for x in xs if x is not None]
    return dict(min=min(xs), median=statistics.median(xs), max=max(xs), n=len(xs)) if xs else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg2-runs", type=int, default=6)
    ap.add_argument("--other-runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dump", default=None)
    ap.add_argument("--cta-stamps", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.cta_stamps:
        return cta_stamps()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("lio_residency_timing: no CUDA device (the numbers are GPU timings; there is no CPU fallback)")
    res = dict(card=card(), runs={})
    with tempfile.TemporaryDirectory() as tmp:
        libs = build_all(tmp)
        plan = [("cfg2", args.cfg2_runs), ("cfg4", args.other_runs), ("cfg5", args.other_runs)]
        for config, runs in plan:
            for k in range(runs):
                for name, lib in libs.items():
                    dump = os.path.join(args.dump, name, config) if args.dump and k == 0 else None
                    r = bench(lib, config, args.steps, args.warmup, dump)
                    res["runs"].setdefault(config, {}).setdefault(name, []).append(r)
                    print(f"{config} {name} run {k}: value={r['value']:.0f} lio_update_ms={r['lio_update_ms']:.4f} build_us={r['lio_build_us_per_iteration']}", flush=True)
        res["cta_stamps"] = {}
        for name, lib in libs.items():
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--cta-stamps"], cwd=ROOT, env=dict(os.environ, ESIKF_LIB=lib), capture_output=True, text=True)
            lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
            res["cta_stamps"][name] = json.loads(lines[-1]) if r.returncode == 0 and lines else dict(error=r.stderr[-2000:])
    res["summary"] = {config: {name: {k: spread([r[k] for r in rs]) for k in ("value", "lio_update_ms", "lio_build_us_per_iteration", "lio_iteration_us")}
                               | dict(lio_iters=sorted({r["lio_iters"] for r in rs}), matched_points=sorted({r["matched_points"] for r in rs}),
                                      parity_ok=all(r["parity_ok"] for r in rs), repeatable=all(r["repeatable"] for r in rs))
                               for name, rs in per.items()}
                      for config, per in res["runs"].items()}
    res["what"] = ("bench.py --gpus 1 --no-cpu-baseline --no-shim, alternating LIO_L2_WARPS=2 / 0 builds of the same sources; "
                   "lio_update_ms = roofline.avg_launch_ms_in_timed_region; cta_stamps: cfg2, iteration 3, us after CTA 0's constants-in-place stamp")
    print(json.dumps(dict(card=res["card"], summary=res["summary"], cta_stamps=res["cta_stamps"]), indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
