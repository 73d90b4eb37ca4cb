"""Regenerates tests/golden/ref_pin/vmap_retrieve.npz: feat_map after every tick, sub_feat_map, grid_num,
retrieve_voxel_points, the points reaching visual_submap and their ref_patch, of the REFERENCE SOURCE's own
insertPointIntoVoxelMap + retrieveFromVisualSparseMap (oracle/_ref/libfl2_ref_vretrieve.so, built by oracle/vmap_retrieve.mk
from /root/reference/src/vio.cpp) over the ticks of tests/vmap_retrieve_cases.py, checked against the restatement before it
is written. Run in the build container (needs /root/reference):
    python tests/golden/make_vmap_retrieve_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import vmap_retrieve_cases as VR  # noqa: E402
from test_oracle_vmap_retrieve import oracle_pins, reference_pins  # noqa: E402

assert VR.ref_vretrieve_available(), "build oracle/_ref first (make -C oracle -f vmap_retrieve.mk)"
ref, orc = reference_pins(), oracle_pins()
assert set(ref) == set(orc)
for k in orc:
    assert ref[k].tobytes() == orc[k].tobytes(), f"the restatement differs from the reference source on {k}"
np.savez_compressed(VR.GOLDEN, **ref)
print("wrote", VR.GOLDEN, {k: v.shape for k, v in ref.items()})
