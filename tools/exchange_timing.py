"""What the grid-mailbox exchange of the persistent ESIKF kernels is worth on the GPU: bench.py run against two builds of
the library (ESIKF_LIB), alternating between them,

  new:    this tree, compiled with the flags of __graft_entry__.build();
  parent: an earlier revision's library, built beforehand with the same flags (for example from a git worktree of the
          parent commit) and passed as --parent-lib: the grid barrier and the every-CTA-reads-every-column sum.

cfg2 (bench.py's metric) --cfg2-runs times per build, then cfg3, cfg4 and cfg5 --other-runs times per build. Per build and
config it reports bench's `value`, the persistent LIO and VIO update durations in the timed region
(roofline.avg_launch_ms_in_timed_region, roofline.vio_update_ms_in_timed_region) and the phase stamps
(roofline.residual_build_phase), as min / median / max over the runs. A separate pass per build runs cfg2's LIO update with
phase stamps on and reports when each CTA finished its slice of iteration 3 (stamps[640 + b]), counted from CTA 0's
"constants in place" stamp of that iteration. The first run of every config per build writes bench.py --dump-outputs files,
and the two builds' files are compared byte for byte. The card's name and power limit are read in the same run.

    python tools/exchange_timing.py --parent-lib PATH [--cfg2-runs 6] [--other-runs 3] [--out result.json]
"""
import argparse
import filecmp
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from lio_residency_timing import card, spread  # noqa: E402

PHASE_KEYS = ("lio_build_us_per_iteration", "lio_iteration_us", "lio_tail_us_all_arrived_to_solved", "vio_build_us_per_iteration", "vio_iteration_us",
              "vio_tail_us_all_arrived_to_solved")


def build_new(out_dir):
    import __graft_entry__ as G

    lib = os.path.join(out_dir, "libesikf_b200.so")
    G.build_library(lib, force=True)
    return lib


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
    return dict(value=out["value"], lio_update_ms=rl["avg_launch_ms_in_timed_region"], vio_update_ms=rl.get("vio_update_ms_in_timed_region"),
                **{k: ph.get(k) for k in PHASE_KEYS}, gpu_launches=out["gpu_launches"], lio_iters=out["config"]["lio_iters"], vio_iters=out["config"]["vio_iters"],
                parity_ok=out["parity_vs_oracle"]["ok"], repeatable=out["parity_vs_oracle"]["last_update_bit_identical_to_first"])


def same_dumps(a, b):
    """Every file under a and b, byte for byte: the list of files that differ or exist on one side only."""
    fa = {os.path.relpath(os.path.join(d, f), a) for d, _, fs in os.walk(a) for f in fs}
    fb = {os.path.relpath(os.path.join(d, f), b) for d, _, fs in os.walk(b) for f in fs}
    differ = sorted(fa ^ fb) + sorted(f for f in fa & fb if not filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False))
    return dict(files=len(fa & fb), differ=differ)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", required=True)
    ap.add_argument("--cfg2-runs", type=int, default=6)
    ap.add_argument("--other-runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("exchange_timing: no CUDA device (the numbers are GPU timings; there is no CPU fallback)")
    res = dict(card=card(), runs={})
    with tempfile.TemporaryDirectory() as tmp:
        libs = {"new": build_new(tmp), "parent": os.path.abspath(args.parent_lib)}
        dumps = os.path.join(tmp, "dumps")
        plan = [("cfg2", args.cfg2_runs), ("cfg3", args.other_runs), ("cfg4", args.other_runs), ("cfg5", args.other_runs)]
        for config, runs in plan:
            for k in range(runs):
                for name, lib in libs.items():
                    dump = os.path.join(dumps, name, config) if k == 0 else None
                    r = bench(lib, config, args.steps, args.warmup, dump)
                    res["runs"].setdefault(config, {}).setdefault(name, []).append(r)
                    print(f"{config} {name} run {k}: value={r['value']:.1f} lio_update_ms={r['lio_update_ms']:.4f} vio_update_ms={r['vio_update_ms']}", flush=True)
        res["dumps_identical"] = {config: same_dumps(os.path.join(dumps, "new", config), os.path.join(dumps, "parent", config)) for config, _ in plan}
        res["cta_stamps"] = {}
        for name, lib in libs.items():
            r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "lio_residency_timing.py"), "--cta-stamps"], cwd=ROOT, env=dict(os.environ, ESIKF_LIB=lib),
                               capture_output=True, text=True)
            lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
            res["cta_stamps"][name] = json.loads(lines[-1]) if r.returncode == 0 and lines else dict(error=r.stderr[-2000:])
    res["summary"] = {config: {name: {k: spread([r[k] for r in rs]) for k in ("value", "lio_update_ms", "vio_update_ms", *PHASE_KEYS)}
                               | {k: sorted({r[k] for r in rs}) for k in ("gpu_launches", "lio_iters", "vio_iters")}
                               | dict(parity_ok=all(r["parity_ok"] for r in rs), repeatable=all(r["repeatable"] for r in rs))
                               for name, rs in per.items()}
                      for config, per in res["runs"].items()}
    res["what"] = ("bench.py --gpus 1 --no-cpu-baseline --no-shim, alternating the grid-mailbox build (new) and the grid-barrier build (parent); "
                   "lio/vio_update_ms = roofline.avg_launch_ms_in_timed_region / vio_update_ms_in_timed_region; cta_stamps: cfg2, iteration 3, "
                   "us after CTA 0's constants-in-place stamp")
    print(json.dumps(dict(card=res["card"], summary=res["summary"], dumps_identical=res["dumps_identical"], cta_stamps=res["cta_stamps"]), indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
