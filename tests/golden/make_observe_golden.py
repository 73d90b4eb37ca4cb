"""Regenerates tests/golden/ref_pin/observe.npz: the update flags and new observations of the REFERENCE SOURCE's own
updateVisualMapPoints (oracle/_ref/libfl2_ref_observe.so, built by oracle/observe.mk from /root/reference/src/vio.cpp) on the
pin scenes of tests/observe_cases.py, checked against the oracle's restatement before it is written. Run in the build
container (needs /root/reference):   python tests/golden/make_observe_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import observe_cases as OC  # noqa: E402
from test_oracle_observe import oracle_pins, reference_pins  # noqa: E402

assert OC.ref_observe_available(), "build oracle/_ref first (make -C oracle -f observe.mk)"
ref, orc = reference_pins(), oracle_pins()
for k in orc:
    assert ref[k].tobytes() == orc[k].tobytes(), f"the oracle differs from the reference source on {k}"
np.savez_compressed(OC.GOLDEN, **ref)
print("wrote", OC.GOLDEN, {k: v.shape for k, v in ref.items()})
