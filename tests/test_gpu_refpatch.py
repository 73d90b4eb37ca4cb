"""GPU: esikf_vio_score_ref_patches (refpatch_score_kernel, K13), the patch scoring of updateReferencePatch, against the
oracle's restatement (oracle/orc_refpatch.cpp) bit for bit: on the hand-built cases of tests/refpatch_cases.py, on
realistic observation sets (the visual points of a keyframe_cases frame, each observed in 6 to 30 keyframe images through
image_patch_kernel with those keyframes' poses), with cached means the patches do not have, twice in a row, through the
shim's VIOManager::ScoreReferencePatches, and on the refusals, which write nothing."""

import numpy as np
import pytest

import refpatch_cases as RC
import shim_bind as SB
from fast_livo2_b200 import api

pytestmark = pytest.mark.gpu
ERR_ARG = -3  # ESIKF_ERR_ARG


@pytest.fixture(scope="module")
def ctx():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = api.Context(0)
    yield c
    c.close()


def assert_oracle(got, c):
    """Bit for bit with the oracle; a NaN score equals any NaN (the host and the device encode 0 / 0 differently)."""
    want = RC.oracle(c)
    for k in ("score", "mean", "ref"):
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert RC.same_bits_but_nan(a, b), f"{k}: {int(np.sum((a.view(np.int32) != b.view(np.int32)) & ~(np.isnan(a) & np.isnan(b))))} of {len(a)} differ"


def run(ctx, c):
    return ctx.vio_score_ref_patches(c["first"], c["pos"], c["normal"], c["patch"], c["mean"], c["id"], c["T"])


@pytest.mark.parametrize("name", ["pin", "mean", "gpu_only"])
def test_hand_built_cases_are_the_oracle_bit_for_bit(ctx, name):
    """Zero and sub-1e-6 means, 1 to 200 observations (shared memory up to 32, global memory above), shared ids and count 0,
    flat and underflowing patches (NaN, inf), exact ties, nothing chosen, cached means on both sides of 1e-6."""
    c = {"pin": RC.pin_case, "mean": RC.mean_case, "gpu_only": RC.gpu_only_case}[name]()
    got = run(ctx, c)
    assert_oracle(got, c)
    if name == "pin":
        assert np.isnan(got["score"]).any() and np.isinf(got["score"]).any() and (got["ref"] == -1).any()


@pytest.mark.parametrize("n_points", [2000, 4000])
def test_realistic_observation_sets_are_the_oracle_bit_for_bit(ctx, n_points):
    c = RC.realistic_case(ctx, n_points, seed=n_points)
    counts = np.diff(c["first"])
    assert counts.min() >= 6 and counts.max() <= 30 and counts.max() > 20
    cached = np.abs(c["mean"]) >= 1e-6
    assert cached.any() and (~cached).any()
    got = run(ctx, c)
    assert_oracle(got, c)
    assert (got["ref"] >= 0).mean() > 0.99 and np.isfinite(got["score"]).mean() > 0.99  # flat patches give NaN
    assert (np.abs(got["mean"]) > 1).all()  # real intensities


def test_a_cached_mean_is_the_one_used(ctx):
    """mean_ above 1e-6 that is not the patch's own mean: it comes back unchanged and the scores use it (they differ from the
    scores on the patches' own means)."""
    c = RC.realistic_case(ctx, 300, seed=3)
    own = (c["patch"].astype(np.float64).sum(1).astype(np.float32) / np.float32(64)).astype(np.float32)
    c["mean"] = (own + np.float32(3.5)).astype(np.float32)
    got = run(ctx, c)
    assert RC.same_bits(got["mean"], c["mean"])
    assert_oracle(got, c)
    c2 = dict(c, mean=own)
    assert not RC.same_bits(run(ctx, c2)["score"], got["score"])


def test_a_repeated_call_is_byte_identical(ctx):
    c = RC.realistic_case(ctx, 2000, seed=11)
    a = run(ctx, c)
    run(ctx, RC.gpu_only_case())  # other sizes in between
    b = run(ctx, c)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def _raw(ctx, n, first, m, outs, c):
    vp = lambda x: None if x is None else x.ctypes.data  # noqa: E731
    return ctx.lib.esikf_vio_score_ref_patches(ctx.h, n, vp(first), m, vp(c["pos"]), vp(c["normal"]), vp(c["patch"]), vp(c["mean"]), vp(c["id"]),
                                              vp(c["T"]), *[vp(o) for o in outs])


def test_refusals_write_nothing_and_empty_calls_succeed(ctx):
    c = RC.pin_case()
    n, m = len(c["first"]) - 1, len(c["patch"])
    outs = [np.full(m, 7.0, np.float32), np.full(m, 7.0, np.float32), np.full(n, 7, np.int32)]
    keep = [o.copy() for o in outs]
    bad = []
    f = c["first"].copy()
    f[0] = 1
    bad.append((n, f, m))
    f = c["first"].copy()
    f[3], f[4] = f[4], f[3]
    bad.append((n, f, m))
    bad.append((n, c["first"], m - 1))
    bad.append((-1, c["first"], m))
    bad.append((n, c["first"], -1))
    for nn, ff, mm in bad:
        assert _raw(ctx, nn, ff, mm, outs, c) == ERR_ARG
        for o, k in zip(outs, keep):
            assert o.tobytes() == k.tobytes()
    assert _raw(ctx, n, None, m, outs, c) == ERR_ARG
    assert _raw(ctx, n, c["first"], m, [None] + outs[1:], c) == ERR_ARG
    for o, k in zip(outs, keep):
        assert o.tobytes() == k.tobytes()
    assert _raw(ctx, 0, None, 0, [None, None, None], dict(pos=None, normal=None, patch=None, mean=None, id=None, T=None)) == 0
    z = np.zeros(1, np.int32)
    assert _raw(ctx, 0, z, 0, [None, None, None], dict(pos=None, normal=None, patch=None, mean=None, id=None, T=None)) == 0
    # a point with no observations: nothing to score, nothing chosen
    e = RC.concat([])
    e["first"] = np.zeros(2, np.int32)
    e["pos"], e["normal"] = np.zeros((1, 3)), np.zeros((1, 3))
    got = run(ctx, e)
    assert got["ref"].tolist() == [-1] and len(got["score"]) == 0
    assert_oracle(run(ctx, c), c)  # the context works after the refusals


def test_shim_score_reference_patches_is_the_c_abi(ctx):
    shim = SB.load()
    for c in (RC.pin_case(), RC.realistic_case(ctx, 2000, seed=5)):
        n, m = len(c["first"]) - 1, len(c["patch"])
        out = dict(score=np.zeros(m, np.float32), mean=np.zeros(m, np.float32), ref=np.zeros(n, np.int32))
        ins = [np.ascontiguousarray(c[k]) for k in ("pos", "normal", "patch", "mean", "id", "T")]
        rc = shim.fl2_shim_score_ref_patches(n, c["first"].ctypes.data, m, *[x.ctypes.data for x in ins], *[out[k].ctypes.data for k in ("score", "mean", "ref")])
        assert rc == 0
        want = run(ctx, c)
        for k in out:
            assert out[k].tobytes() == want[k].tobytes(), k
