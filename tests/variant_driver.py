"""The update cases that hold the compile-time variants of the update kernels (__graft_entry__.VARIANTS) to the default
build, and a driver that runs them on one library.

api.LIB_PATH is read when fast_livo2_b200.api is imported (ESIKF_LIB), so every library runs in a process of its own:

    ESIKF_LIB=<library> python tests/variant_driver.py OUT.npz CASE [CASE ...]

runs the named cases in every launch form, asserts that the forms are bit-identical, and writes the first form's outputs
to OUT.npz as "<case>/<key>" (tests/test_gpu_build_variants.py compares the files of two libraries and the oracle's
outputs on the same inputs). LIO forms: loop modes 2 and 0, each with the bulk-copy and the __ldg record staging. VIO
forms: loop modes 2 and 0, each with and without TMA tap staging, each with phase stamps off and on; a VIO case also
keeps "<case>/chain", the chain stamps after its persistent update with phase stamps on."""
import dataclasses
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import keyframe_cases as KC  # noqa: E402
import lio_assoc as A  # noqa: E402
import oracle_bind as O  # noqa: E402
from conftest import get_frame  # noqa: E402
from fast_livo2_b200 import api  # noqa: E402
from fast_livo2_b200 import synthetic as S  # noqa: E402
from harness import LIO_KEYS, VIO_KEYS, bits_equal, lio_gpu, sweep, vio_prior  # noqa: E402

LIO_FORMS = [dict(loop_mode=2), dict(loop_mode=0), dict(loop_mode=2, tuning=api.TUNE_STAGE_LDG), dict(loop_mode=0, tuning=api.TUNE_STAGE_LDG)]
VIO_FORMS = [dict(loop_mode=2), dict(loop_mode=0), dict(loop_mode=2, tuning=api.TUNE_VIO_TMA), dict(loop_mode=0, tuning=api.TUNE_VIO_TMA)]
CONFIG5 = dict(seed=13, n_pts=1000, n_map=300_000, n_patches=4000, scene_scale=0.7, cam=KC.CONFIG5_CAM, vio=S.VioCfg(levels=5, img_point_cov=1000.0))


# ---------------------------------------------------------------------------------------------------------------- LIO
def lio_sizes(G):
    """test_gpu_lio_assoc.py::test_resident_and_tiled_slices' sizes and test_gpu_lio_l2_slots.py's: one chunk per CTA and
    around it, both sides of the 704- and 768-lane residency, and 2.5 rounds of tiles of each."""
    R, R2 = G * A.SMEM_LANES, G * A.LANES
    return sorted({1, 31, 33, 32 * G - 1, 32 * G, 32 * G + 1, R - 1, R, R + 1, int(2.5 * R), R2 - 1, R2, R2 + 1, int(2.5 * R2)})


def lio_cases(G):
    """name -> frame maker: the hand-built association cases of lio_assoc.py at every size of lio_sizes and with every designed
    warp in lanes 704-767 (l2_lane_layout), config 2's 100 k-point frame (the 768-lane kernel) and config 4's 260 k (tiled)."""
    out = {}
    for name in A.CASES:
        for n in lio_sizes(G):
            out[f"{name}_n{n}"] = lambda name=name, n=n: A.tiled(A.case(name), n)
        W = len(A.case(name)["pts"]) // 32
        for start in range(0, W, 2 * G):
            out[f"{name}_l2_{start}"] = lambda name=name, start=start: A.l2_lane_layout(A.case(name), G, start)
    out["cfg2"] = lambda: get_frame(seed=0, n_pts=100_000, n_map=1_000_000)
    out["cfg4"] = lambda: get_frame(seed=12, n_pts=260_000, n_map=1_000_000, lio=S.LioCfg(beam_err=0.01))
    return out


def uses_l2_slots(n, G):
    """Whether the default build runs the 768-lane kernel on n points (lio_use_l2_slots, csrc/esikf_api_update.cu)."""
    chunks = (n + 31) // 32
    per_cta = -(-chunks // min(chunks, G))
    return A.SMEM_LANES // 32 < per_cta <= A.LANES // 32


# ---------------------------------------------------------------------------------------------------------------- VIO
def _frame_case(fr, prior_seed, inverse):
    """A synthetic frame's sub-map warped by the oracle at a perturbed prior (the same inputs for every library)."""
    prior = vio_prior(fr, prior_seed)
    w = O.oracle_warp_patches(fr, prior)
    n = len(fr["vis_pos"])
    return dict(cam_cfg=fr["cam_cfg"], ext=fr["ext"], vio_cfg=dataclasses.replace(fr["vio_cfg"], inverse_composition_en=inverse), ref_imgs=[fr["img_ref"]],
                refs=O.inverse_refs_from_frame(fr) if inverse else None,
                args=(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], np.ones(n) if inverse else fr["inv_ref_expo"], prior, prior))


def _keyframe_case(name, inverse):
    c = KC.build(name)
    return dict(cam_cfg=c["cam_cfg"], ext=c["ext"], vio_cfg=dataclasses.replace(c["vio_cfg"], inverse_composition_en=inverse), ref_imgs=c["ref_imgs"],
                refs=c["refs"] if inverse else None, args=KC.update_args(c))


VIO_CASES = {
    "vio_small": lambda: _frame_case(get_frame(seed=2, n_pts=2000, n_map=120_000, n_patches=150, scene_scale=0.5), 3, False),
    "vio_small_inverse": lambda: _frame_case(get_frame(seed=2, n_pts=2000, n_map=120_000, n_patches=150, scene_scale=0.5), 3, True),
    "vio_config5": lambda: _frame_case(get_frame(**CONFIG5), 13, False),  # 4 k patches: two per warp
    "vio_keyframes": lambda: _keyframe_case("pinhole_gain", False),
    "vio_keyframes_inverse": lambda: _keyframe_case("pinhole_gain", True),
}


def vio_oracle(c):
    vio = O.OracleVIO(c["cam_cfg"], c["ext"], c["vio_cfg"])
    if c["refs"] is not None:
        vio.set_inverse_refs(**c["refs"])
        vio.set_inverse(True)
    return vio.update(*c["args"])


# ---------------------------------------------------------------------------------------------------------------- runs
def run_lio(ctx, fr):
    runs = sweep(ctx, lambda: lio_gpu(ctx, fr), LIO_FORMS)
    for v, r in zip(LIO_FORMS[1:], runs[1:]):
        try:
            bits_equal(runs[0], r, LIO_KEYS)
        except AssertionError as e:
            raise AssertionError(f"launch form {v} differs from {LIO_FORMS[0]} in {e}") from None
    return runs[0]


def run_vio(ctx, c):
    ctx.set_extrinsics(c["ext"])
    ctx.vio_set_camera(c["cam_cfg"], c["vio_cfg"])
    ctx.vio_set_image(c["args"][0])
    ctx.vio_set_ref_images(c["ref_imgs"])
    if c["refs"] is not None:
        r = c["refs"]
        ctx.vio_set_inverse_refs(r["ref_img_index"], r["ref_px"], r["ref_f"], r["ref_R"], r["ref_pos"])
    runs, chain = [], None
    for stamps in (False, True):
        ctx.set_phase_stamps(stamps)
        try:
            for v in VIO_FORMS:
                runs.append((dict(v, stamps=stamps), sweep(ctx, lambda: ctx.vio_update(*c["args"]), [v])[0]))
                if chain is None and stamps and v == VIO_FORMS[0]:
                    chain = ctx.get_vio_chain_stamps()
        finally:
            ctx.set_phase_stamps(False)
    for v, r in runs[1:]:
        try:
            bits_equal(runs[0][1], r, VIO_KEYS + ("total_iters",))
        except AssertionError as e:
            raise AssertionError(f"launch form {v} differs from {runs[0][0]} in {e}") from None
    return dict(runs[0][1], chain=chain)


def main(out_path, names):
    from harness import sm_count

    G = min(sm_count(), 160)
    lio = lio_cases(G)
    ctx = api.Context(0)
    out = {}
    for name in names:
        try:
            if name in VIO_CASES:
                r = run_vio(ctx, VIO_CASES[name]())
                keys = VIO_KEYS + ("total_iters", "chain")
            else:
                r = run_lio(ctx, lio[name]())
                keys = LIO_KEYS + ("iters",)
        except AssertionError as e:
            raise AssertionError(f"{name}: {e}") from None
        out.update({f"{name}/{k}": np.asarray(r[k]) for k in keys})
    ctx.close()
    np.savez(out_path, **out)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2:])
