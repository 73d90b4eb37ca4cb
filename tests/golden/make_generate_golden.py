"""Regenerates tests/golden/ref_pin/generate.npz: the new visual map points of the REFERENCE SOURCE's own
generateVisualMapPoints (oracle/_ref/libfl2_ref_generate.so, built by oracle/generate.mk from /root/reference/src/vio.cpp) on
the pin scenes of tests/generate_cases.py, checked against the oracle's restatement before it is written. Run in the build
container (needs /root/reference):   python tests/golden/make_generate_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import generate_cases as GC  # noqa: E402
from test_oracle_generate import oracle_pins, reference_pins  # noqa: E402

assert GC.ref_generate_available(), "build oracle/_ref first (make -C oracle -f generate.mk)"
ref, orc = reference_pins(), oracle_pins()
for k in ref:
    assert ref[k].tobytes() == orc[k].tobytes(), f"the oracle differs from the reference source on {k}"
np.savez_compressed(GC.GOLDEN, **ref)
print("wrote", GC.GOLDEN, {k: v.shape for k, v in ref.items()})
