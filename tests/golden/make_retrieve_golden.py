"""Regenerates tests/golden/ref_pin/retrieve.npz: sub_feat_map, grid_num, retrieve_voxel_points and the points past the depth
check of the REFERENCE SOURCE's own retrieveFromVisualSparseMap (oracle/_ref/libfl2_ref_retrieve.so, built by
oracle/retrieve.mk from /root/reference/src/vio.cpp) on the pin scenes of tests/retrieve_cases.py, checked against the
oracle's restatement before it is written. Run in the build container (needs /root/reference):
    python tests/golden/make_retrieve_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import retrieve_cases as RC  # noqa: E402
from test_oracle_retrieve import oracle_pins, reference_pins  # noqa: E402

assert RC.ref_retrieve_available(), "build oracle/_ref first (make -C oracle -f retrieve.mk)"
ref, orc = reference_pins(), oracle_pins()
for k in orc:
    assert ref[k].tobytes() == orc[k].tobytes(), f"the oracle differs from the reference source on {k}"
np.savez_compressed(RC.GOLDEN, **ref)
print("wrote", RC.GOLDEN, {k: v.shape for k, v in ref.items()})
