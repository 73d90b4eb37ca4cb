"""Time esikf_vio_select_patches against the path it replaces, on config-2-shaped candidate sets (pinhole-radtan 640 x 512,
4 pyramid levels, 2 k and 4 k candidates, about half surviving the outlier gate):

  select   : esikf_vio_select_patches (warps, current patches, error, gates and the sub-map install on the device; the kept
             indices and errors come back)
  replaced : esikf_vio_warp_patches with the patches downloaded, getImagePatch through esikf_vio_get_image_patch, the error
             and gate loop on the host (numpy, the reference's per-candidate arithmetic) and esikf_vio_set_patches of the survivors

Both are timed with CUDA events on the context's stream and with the host clock, around calls that end in a device
synchronise, and the kept sets of the two paths are checked to be equal. The card's name, power limit and maximum SM clock are printed in the same run. Writes nothing; needs a GPU.

  python tools/select_patches_timing.py [--reps 50]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import timing as T  # noqa: E402
import torch  # noqa: E402

import select_cases as SC  # noqa: E402
from fast_livo2_b200 import api  # noqa: E402
from fast_livo2_b200 import synthetic as S  # noqa: E402


def host_gate(c, wp, cur, thr):
    """The reference's error (vio.cpp:746-751: double terms, float accumulator, index order), vectorised over candidates."""
    d = c["ref_inv_expo"][:, None] * wp[:, :64].astype(np.float64) - c["inv_expo"] * cur.astype(np.float64)
    t = d * d
    err = np.zeros(len(t), np.float32)
    for ind in range(64):
        err = (err.astype(np.float64) + t[:, ind]).astype(np.float32)
    return np.nonzero(~(err > thr * 64))[0], err


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    T.require_gpu("select_patches_timing")
    print(f"device: {json.dumps(T.card())}")
    ctx = api.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    for n in (2000, 4000):
        c = SC.candidates("radtan", n, n_frames=80, seed=21)
        ctx.set_extrinsics(S.avia_extrinsics())
        ctx.vio_set_camera(c["camcfg"], S.VioCfg(levels=4))
        ctx.vio_set_image(c["img"])
        ctx.vio_set_ref_images(c["ref_imgs"])
        sel = lambda thr: ctx.vio_select_patches(c["ref_idx"], c["px_ref"], c["pos_w"], c["T_ref"], c["ref_inv_expo"], c["pc"], c["T_cur"], c["inv_expo"],
                                                 normal_w=c["normal_w"], outlier_threshold=thr)
        all_ = ctx.vio_select_patches(c["ref_idx"], c["px_ref"], c["pos_w"], c["T_ref"], c["ref_inv_expo"], c["pc"], c["T_cur"], c["inv_expo"],
                                      normal_w=c["normal_w"], outlier_threshold=1e30)
        thr = float(np.median(all_["errors"])) / 64

        def replaced():
            w = ctx.vio_warp_patches(c["ref_idx"], c["px_ref"], c["pos_w"], c["normal_w"], c["T_ref"], c["T_cur"])
            cur = ctx.vio_get_image_patch(c["pc"], 0)
            k, err = host_gate(c, w["warp_patch"], cur, thr)
            ctx.vio_set_patches(c["pos_w"][k], w["warp_patch"][k], w["search_levels"][k], c["ref_inv_expo"][k])
            return k

        for name, fn in (("select", lambda: sel(thr)), ("replaced", replaced)):
            for _ in range(5):
                r = fn()
            ctx.synchronize()
            ev, wall = T.window_ms(stream, fn, args.reps)
            kept = len(r["kept"]) if isinstance(r, dict) else len(r)
            print(f"n={n} {name:8s} kept={kept:5d}  events {ev:.3f} ms/call  host {wall:.3f} ms/call")
        # both paths select the same sub-map (same warps, same current patches, the reference's error arithmetic)
        assert np.array_equal(sel(thr)["kept"], replaced()), "the two timed paths kept different candidates"
    ctx.close()


if __name__ == "__main__":
    main()
