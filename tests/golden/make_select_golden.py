"""Regenerates tests/golden/ref_pin/select.npz: the REFERENCE SOURCE's getWarpMatrixAffine + getBestSearchLevel and
calculateNCC (oracle/_ref/libfl2_ref_select.so, built by oracle/select.mk from /root/reference/src/vio.cpp) on the pin cases
of tests/select_cases.py, checked against the oracle's restatement before it is written. Run in the build container (needs
/root/reference):   python tests/golden/make_select_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import select_cases as SC  # noqa: E402
from test_oracle_select import _oracle_pins, reference_pins  # noqa: E402

assert SC.ref_select_available(), "build oracle/_ref first (make -C oracle -f select.mk)"
ref, orc = reference_pins(), _oracle_pins()
for k in ref:
    assert np.array_equal(ref[k].view(np.uint8), orc[k].view(np.uint8)), f"the oracle differs from the reference source on {k}"
np.savez_compressed(SC.GOLDEN, **ref)
print("wrote", SC.GOLDEN, {k: v.shape for k, v in ref.items()})
