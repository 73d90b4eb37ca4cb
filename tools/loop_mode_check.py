"""Checks the loop modes of the update against each other (bit-identical states / associations / diagnostics) on a
small frame and on the BASELINE config-2 frame, and times the resident LIO + VIO update per mode (CUDA events, L2 flushed
between steps). Run on the GPU box:  timeout 170 python tools/loop_mode_check.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from fast_livo2_b200 import api, synthetic as S  # noqa: E402

MODES = [int(m) for m in os.environ.get("MODES", "2,0").split(",")]
STEPS = int(os.environ.get("STEPS", 30))


def run_once(ctx, fr, w):
    r = ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], fr["lio_cfg"])
    v = ctx.vio_update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], r["state"], r["state"])
    return r, v


def same(a, b):
    bad = []
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        if x.dtype.kind == "f":
            ok = np.array_equal(x.view(np.uint8), y.view(np.uint8))
        else:
            ok = np.array_equal(x, y)
        if not ok:
            bad.append(k)
    return bad


def check(fr, label, time_it):
    ctx = api.Context(0)
    ctx.set_extrinsics(fr["ext"])
    ctx.map_upload(fr["map"], fr["lio_cfg"].voxel_size)
    ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])
    r = ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], fr["lio_cfg"])
    st = S.unpack_state(r["state"])
    ctx.vio_set_image(fr["img"])
    ctx.vio_set_ref_images([fr["img_ref"]])
    n = len(fr["vis_pos"])
    w = ctx.vio_warp_patches(np.zeros(n, np.int32), fr["px_ref"], fr["vis_pos"], fr["vis_normal"], np.tile(api.pack_T(*fr["T_ref"]), (n, 1)),
                             api.pack_T(*S.camera_pose(fr["ext"], st["R"], st["p"])))
    ref = None
    ok = True
    for mode in MODES:
        ctx.set_loop_mode(mode)
        for rep in range(2):  # twice: the second launch uses the other barrier counter and continues the exchange counter
            r, v = run_once(ctx, fr, w)
        if ref is None:
            ref = (r, v)
            print(f"[{label}] mode {mode}: LIO iters {r['iters']} M {np.asarray(r['M'])[:r['iters']].tolist()}  VIO iters {v['total_iters']}", flush=True)
        else:
            bl, bv = same(ref[0], r), same(ref[1], v)
            ok = ok and not bl and not bv
            print(f"[{label}] mode {mode} vs mode {MODES[0]}: LIO differing keys {bl}  VIO differing keys {bv}", flush=True)
    for solve_mode in (1,):  # literal double-inversion solve through the replicated kernels
        ctx.set_solve_mode(solve_mode)
        outs = []
        for mode in MODES:
            ctx.set_loop_mode(mode)
            outs.append(run_once(ctx, fr, w))
        for mode, o in zip(MODES[1:], outs[1:]):
            bl, bv = same(outs[0][0], o[0]), same(outs[0][1], o[1])
            ok = ok and not bl and not bv
            print(f"[{label}] literal solve, mode {mode} vs mode {MODES[0]}: LIO {bl} VIO {bv}", flush=True)
        ctx.set_solve_mode(0)
    if time_it:
        dev = torch.device("cuda", 0)
        ext_stream = torch.cuda.ExternalStream(ctx.stream, device=dev)
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
        prior_h, post_h = pin(fr["state_prior"]), pin(ref[0]["state"])
        ctx.lio_set_scan(pin(fr["pts"]))
        ctx.vio_set_patches(pin(fr["vis_pos"]), pin(w["warp_patch"]), pin(w["search_levels"]), pin(fr["inv_ref_expo"]))
        iters = int(ref[0]["iters"] + ref[1]["total_iters"])
        runs = [(m, 0) for m in MODES] + [(2, int(f)) for f in os.environ.get("TUNING", "").split(",") if f]  # (loop mode, esikf_set_tuning flags)
        for mode, sched in runs:
            ctx.set_loop_mode(mode)
            ctx.set_tuning(sched)
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
            for k in range(-3, STEPS):
                with torch.cuda.stream(ext_stream):
                    flush.zero_()
                    if k >= 0:
                        evs[k][0].record(ext_stream)
                ctx.lio_run(prior_h, prior_h, fr["lio_cfg"])
                if k >= 0:
                    with torch.cuda.stream(ext_stream):
                        evs[k][1].record(ext_stream)
                ctx.vio_run(post_h, post_h)
                if k >= 0:
                    with torch.cuda.stream(ext_stream):
                        evs[k][2].record(ext_stream)
            torch.cuda.synchronize()
            lio = np.mean([a.elapsed_time(b) for a, b, _ in evs]) * 1e3
            vio = np.mean([b.elapsed_time(c) for _, b, c in evs]) * 1e3
            print(f"[{label}] mode {mode} tuning {sched}: LIO {lio:.1f} us  VIO {vio:.1f} us  step {lio + vio:.1f} us  -> {iters / ((lio + vio) * 1e-6):.0f} it/s resident", flush=True)
        if os.environ.get("INVERSE"):  # the inverse-compositional variant (f4): persistent kernel vs per-iteration launches
            import dataclasses
            R, t = fr["T_ref"]
            pc = fr["vis_pos"] @ R.T + t
            f = pc / np.linalg.norm(pc, axis=1, keepdims=True)
            ctx.vio_set_camera(fr["cam_cfg"], dataclasses.replace(fr["vio_cfg"], inverse_composition_en=True))
            ctx.vio_set_inverse_refs(np.zeros(n, np.int32), np.ascontiguousarray(fr["px_ref"], dtype=np.float64), np.ascontiguousarray(f), np.tile(R.reshape(1, 9), (n, 1)),
                                     np.tile(-R.T @ t, (n, 1)))
            res = {}
            for mode in (2, 0):
                ctx.set_loop_mode(mode)
                ctx.set_tuning(0)
                evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
                for k in range(-3, STEPS):
                    with torch.cuda.stream(ext_stream):
                        flush.zero_()
                        if k >= 0:
                            evs[k][0].record(ext_stream)
                    ctx.vio_run(post_h, post_h)
                    if k >= 0:
                        with torch.cuda.stream(ext_stream):
                            evs[k][1].record(ext_stream)
                torch.cuda.synchronize()
                res[mode] = ctx.vio_fetch()
                vio = np.mean([a.elapsed_time(b) for a, b in evs]) * 1e3
                print(f"[{label}] inverse-compositional VIO, mode {mode}: {vio:.1f} us for {res[mode]['total_iters']} iterations (per level {res[mode]['iters_per_level'][:fr['vio_cfg'].levels].tolist()})"
                      f" -> {vio / max(1, res[mode]['total_iters']):.2f} us / iteration", flush=True)
            bv = same({k: res[2][k] for k in ("state", "errors", "iters_per_level", "HTH", "HTz", "solution")}, {k: res[0][k] for k in ("state", "errors", "iters_per_level", "HTH", "HTz", "solution")})
            ok = ok and not bv
            print(f"[{label}] inverse-compositional VIO, mode 0 vs mode 2: differing keys {bv}", flush=True)
            ctx.vio_set_camera(fr["cam_cfg"], fr["vio_cfg"])
        if os.environ.get("STAMPS"):
            ctx.set_loop_mode(runs[-1][0])
            ctx.set_tuning(runs[-1][1])
            print(f"[{label}] phase stamps of mode {runs[-1][0]} tuning {runs[-1][1]}", flush=True)
            ctx.set_phase_stamps(True)
            for rep in range(2):
                ctx.lio_run(prior_h, prior_h, fr["lio_cfg"])
                ctx.vio_run(post_h, post_h)
            ctx.synchronize()
            s = ctx.get_phase_stamps().astype(np.int64)
            names = ["consts", "slice", "exchange", "sum+peer", "solve"]
            rows = [k for k in range(72) if s[k, 0] != 0]
            for j, slot in enumerate(rows):
                d = np.diff(s[slot, :6])
                nxt = s[rows[j + 1], 0] if j + 1 < len(rows) and (rows[j + 1] < 8) == (slot < 8) else s[slot, 5]
                fine = f" [gain={(s[slot, 6] - s[slot, 4]) / 1000:.2f} boxplus={(s[slot, 7] - s[slot, 6]) / 1000:.2f} rest={(s[slot, 5] - s[slot, 7]) / 1000:.2f}]" if s[slot, 6] else ""
                print(("LIO" if slot < 8 else "VIO"), slot if slot < 8 else slot - 8, " ".join(f"{n}={x / 1000:.2f}us" for n, x in zip(names, d)) + fine,
                      f"to-next={(nxt - s[slot, 5]) / 1000:.2f}us total={(nxt - s[slot, 0]) / 1000:.2f}us", flush=True)
            c = ctx.cta_stamps.astype(np.int64)
            c = c[c > 0]
            if len(c) and s[3, 0]:
                print(f"per-CTA slice end of LIO iteration 3 relative to CTA 0's iteration start (us): n={len(c)} min={(c.min() - s[3, 0]) / 1e3:.2f} "
                      f"p50={(np.median(c) - s[3, 0]) / 1e3:.2f} p90={(np.percentile(c, 90) - s[3, 0]) / 1e3:.2f} max={(c.max() - s[3, 0]) / 1e3:.2f}", flush=True)
        ctx.set_tuning(0)
    ctx.close()
    return ok


if __name__ == "__main__":
    small = S.make_frame(seed=11, n_pts=3000, n_map=100_000, n_patches=120, scene_scale=0.4)
    ok = check(small, "small", False)
    big = S.cached_frame(seed=0, n_pts=int(os.environ.get("N_PTS", 100000)), n_map=int(os.environ.get("N_MAP", 1000000)), n_patches=int(os.environ.get("N_PATCH", 2000)))
    ok = check(big, "cfg2", True) and ok
    print("LOOP MODES BIT-IDENTICAL" if ok else "LOOP MODES DIFFER")
    sys.exit(0 if ok else 1)
