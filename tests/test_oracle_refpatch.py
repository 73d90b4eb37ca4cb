"""CPU: the oracle's restatement of updateReferencePatch's patch scoring (oracle/orc_refpatch.cpp) against the reference
source's own updateReferencePatch (oracle/_ref/libfl2_ref_refpatch.so, live where it was built, else its stored outputs in
tests/golden/ref_pin/refpatch.npz) and against a numpy spelling of the same arithmetic.

The reference's scores are compared where the reference is defined: every mean_ below 1e-6 that recomputes below 1e-6, so
ref_mean and other_mean are assigned at every read (pin_case). mean_ is compared everywhere (mean_case too)."""
import os

import numpy as np
import pytest

import refpatch_cases as RC
from fast_livo2_b200 import synthetic as S

needs_ref = pytest.mark.skipif(not RC.ref_available() and not os.path.exists(RC.GOLDEN), reason="needs oracle/_ref (reference source) or the stored pin")
CASES = {"pin": RC.pin_case, "mean": RC.mean_case}


def ref_outputs(name):
    """The reference's outputs on CASES[name]: live where oracle/_ref was built, else the stored ones (made on the same inputs)."""
    c = CASES[name]()
    if RC.ref_available():
        return c, RC.reference(c, S.CamCfg(), S.avia_extrinsics(), S.VioCfg())
    g = np.load(RC.GOLDEN)
    for k in RC.INPUTS:
        assert RC.same_bits(g[f"{name}_{k}"], c[k]), f"the stored pin was made on other {k}"
    return c, {k: g[f"{name}_{k}_out"] for k in ("score", "mean", "ref", "has_ref")}


@needs_ref
def test_scores_means_and_choice_are_the_reference_bit_for_bit():
    c, r = ref_outputs("pin")
    o = RC.oracle(c)
    for k in ("score", "mean", "ref"):
        assert RC.same_bits(o[k], r[k]), f"{k}: {int(np.sum(np.asarray(o[k]).view(np.int32) != np.asarray(r[k]).view(np.int32)))} differ"
    assert np.array_equal(r["has_ref"], (r["ref"] >= 0).astype(np.uint8))


@needs_ref
def test_means_are_the_reference_on_real_intensity_patches_and_at_the_threshold():
    c, r = ref_outputs("mean")
    o = RC.oracle(c)
    assert RC.same_bits(o["mean"], r["mean"])
    cached = np.abs(c["mean"].astype(np.float64)) >= 1e-6
    assert cached.any() and (~cached).any()
    assert RC.same_bits(o["mean"][cached], c["mean"][cached])  # a cached mean_ is kept as it is
    assert (np.abs(o["mean"][~cached]) > 1).any()  # recomputed from real intensities


def test_pin_inputs_reach_every_edge():
    """The pin holds what the comparison is meant to separate: NaN (0 / 0 and count 0) and infinite scores, a point with
    nothing chosen, 6 / 7 / 30 / 64 observations, shared ids, exact ties won by the first, nonzero sub-1e-6 means, and scores
    that a double sqrt, a per-pair restart of the sums or a double NCC accumulation would change."""
    c = RC.pin_case()
    o = RC.oracle(c)
    counts = np.diff(c["first"])
    assert {6, 7, 30, 64} <= set(counts.tolist())
    assert np.isnan(o["score"]).any() and np.isposinf(o["score"]).any() and (o["ref"] == -1).any()
    m = o["mean"]
    assert ((m != 0) & (np.abs(m) < 1e-6)).any() and (m == 0).all() == False  # noqa: E712
    ties = 0
    for i in range(len(counts)):
        s = o["score"][c["first"][i]:c["first"][i + 1]]
        r = o["ref"][i]
        if r >= 0 and np.sum(s == s[r]) > 1:
            assert np.nonzero(s == s[r])[0][0] == r
            ties += 1
    assert ties >= 2
    for kw in (dict(sqrt_in_double=True), dict(reset_per_pair=True)):
        v = RC.numpy_score(c, **kw)
        assert not RC.same_bits(v["score"], o["score"]), kw


@pytest.mark.parametrize("name", list(CASES) + ["gpu_only"])
def test_oracle_is_its_numpy_spelling(name):
    c = RC.gpu_only_case() if name == "gpu_only" else CASES[name]()
    o, v = RC.oracle(c), RC.numpy_score(c)
    for k in ("score", "mean", "ref"):
        assert RC.same_bits(o[k], v[k]), k


def test_cached_mean_is_used_and_a_recomputed_one_differs():
    """A caller-supplied mean_ above 1e-6 that is not the patch's own mean is the one the scores use."""
    rng = np.random.default_rng(5)
    p = RC.point(rng, 8, "zero")
    p["patch"] = rng.integers(0, 256, (8, 64)).astype(np.float32)
    p["mean"] = np.float32(100.0) + np.arange(8, dtype=np.float32)
    c = RC.concat([p])
    o = RC.oracle(c)
    assert RC.same_bits(o["mean"], p["mean"])
    assert not RC.same_bits(o["score"], RC.numpy_score(c, mean_recompute=True)["score"])
    assert RC.same_bits(o["score"], RC.numpy_score(c)["score"])
