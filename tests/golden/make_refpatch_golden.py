"""Regenerates tests/golden/ref_pin/refpatch.npz: the score_, mean_, chosen reference patch and has_ref_patch_ of the
REFERENCE SOURCE's own updateReferencePatch (oracle/_ref/libfl2_ref_refpatch.so, built by oracle/refpatch.mk from
/root/reference/src/vio.cpp) on the inputs of tests/refpatch_cases.py (pin_case, mean_case), stored with those inputs.
The scores and the choice of pin_case and every mean are checked against the oracle's restatement before anything is
written. Run in the build container (needs /root/reference):   python tests/golden/make_refpatch_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import refpatch_cases as RC  # noqa: E402
from fast_livo2_b200 import synthetic as S  # noqa: E402

assert RC.ref_available(), "build oracle/_ref first (make -C oracle -f refpatch.mk)"
out = {}
for name, make in (("pin", RC.pin_case), ("mean", RC.mean_case)):
    c = make()
    r = RC.reference(c, S.CamCfg(), S.avia_extrinsics(), S.VioCfg())
    o = RC.oracle(c)
    assert RC.same_bits(r["mean"], o["mean"]), f"{name}: the oracle's means differ from the reference source"
    if name == "pin":
        for k in ("score", "ref"):
            assert RC.same_bits(r[k], o[k]), f"{name}: the oracle's {k} differs from the reference source"
    for k in RC.INPUTS:
        out[f"{name}_{k}"] = c[k]
    for k, v in r.items():
        out[f"{name}_{k}_out"] = v
np.savez_compressed(RC.GOLDEN, **out)
print("wrote", RC.GOLDEN, os.path.getsize(RC.GOLDEN), "bytes")
