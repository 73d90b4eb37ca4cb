"""The measurement decisions the timing tools share: which card ran them, call time from CUDA events, kernel time from
torch.profiler, and A/B runs of bench.py against whole library builds. Nothing here sets a clock, power or mode of the card.

A tool imports it with `sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]`."""
import filecmp
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TREE_LIB = os.path.join(ROOT, "fast_livo2_b200", "libesikf_b200.so")
PHASE_KEYS = ("lio_build_us_per_iteration", "lio_iteration_us", "lio_tail_us_all_arrived_to_solved", "vio_build_us_per_iteration", "vio_iteration_us",
              "vio_tail_us_all_arrived_to_solved")


def require_gpu(tool):
    import torch

    if not torch.cuda.is_available():
        raise SystemExit(f"{tool}: no CUDA device (the numbers are GPU timings; there is no CPU fallback)")


def card():
    """Name, power limit and maximum SM clock of device 0 (a read-only nvidia-smi query); the name from torch where the query
    fails. A time is only worth something with the card and power limit it was measured at."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        fields = [f.strip() for f in q.stdout.strip().rsplit(",", 2)] if q.returncode == 0 else []
    except (OSError, subprocess.SubprocessError):
        fields = []
    if len(fields) == 3:
        return dict(gpu=fields[0], power_limit=fields[1], max_sm_clock=fields[2])
    import torch

    return dict(gpu=torch.cuda.get_device_name(0), power_limit="not available", max_sm_clock="not available")


def window_ms(stream, fn, reps):
    """fn() `reps` times between one pair of CUDA events on `stream`: the mean ms per call, and the host wall time alongside."""
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record(stream)
    for _ in range(reps):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / reps, (time.perf_counter() - t0) / reps * 1e3


def per_call_ms(stream, fn, reps):
    """fn() `reps` times, each between its own pair of CUDA events on `stream`: the lists of per-call event ms and host wall ms."""
    import torch

    ev, wall = [], []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t0 = time.perf_counter()
        fn()
        wall.append((time.perf_counter() - t0) * 1e3)
        e1.record(stream)
        e1.synchronize()
        ev.append(e0.elapsed_time(e1))
    return ev, wall


def kernel_us(fn, reps, names=None):
    """fn() `reps` times under torch.profiler with CUDA activities: the device time (us) of every launch, grouped by kernel
    name. names: only the device activities whose name contains one of these, grouped by the first it contains (every name
    gets a list, empty where nothing matched); None: every kernel except the Memcpy / Memset activities, by full name."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    per = {k: [] for k in names or ()}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if names is None:
            if "Memcpy" not in e.name and "Memset" not in e.name:
                per.setdefault(e.name, []).append(e.device_time)
            continue
        k = next((k for k in names if k in e.name), None)
        if k is not None:
            per[k].append(e.device_time)
    return per


def spread(xs):
    xs = [x for x in xs if x is not None]
    return dict(min=min(xs), median=statistics.median(xs), max=max(xs), n=len(xs)) if xs else None


def same_dumps(a, b):
    """Every file under a and b, byte for byte: the number present on both sides, and the files that differ or exist on one
    side only."""
    fa = {os.path.relpath(os.path.join(d, f), a) for d, _, fs in os.walk(a) for f in fs}
    fb = {os.path.relpath(os.path.join(d, f), b) for d, _, fs in os.walk(b) for f in fs}
    differ = sorted(fa ^ fb) + sorted(f for f in fa & fb if not filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False))
    return dict(files=len(fa & fb), differ=differ)


def bench_run(lib, config, steps, warmup, dump=None):
    """bench.py --gpus 1 --no-cpu-baseline --no-shim on `config` with ESIKF_LIB=lib (dump: also --dump-outputs there): its
    value, the LIO / VIO update durations in the timed region, the residual-build phase stamps, the SM clock it sampled,
    iteration, match and launch counts, and its parity verdicts."""
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
                **{k: ph.get(k) for k in PHASE_KEYS}, sm_mhz=out["clocks"].get("sm_mhz"), lio_iters=out["config"]["lio_iters"],
                vio_iters=out["config"]["vio_iters"], matched_points=out["config"]["matched_points"], gpu_launches=out["gpu_launches"],
                parity_ok=out["parity_vs_oracle"]["ok"], repeatable=out["parity_vs_oracle"]["last_update_bit_identical_to_first"])
