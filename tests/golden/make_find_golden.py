"""Regenerates tests/golden/ref_pin/find_correspond.npz: the REFERENCE SOURCE's VoxelOctoTree::find_correspond
(oracle/_ref/libfl2_ref_find.so, built by oracle/find.mk from /root/reference/src/voxel_map.cpp) on the query points of
tests/test_map_mirror_host.py's pinned scene, checked against the oracle's restatement before it is written. Run in the build
container (needs /root/reference):   python tests/golden/make_find_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import map_mirror as MM  # noqa: E402
from test_map_mirror_host import pin_case, pin_queries  # noqa: E402

assert MM.ref_find_available(), "build oracle/_ref first (make -C oracle -f find.mk)"
cfg, ticks = pin_case()
ref = MM.RefFindMap(cfg)
orc, q = pin_queries(cfg, ticks, ref)
r = ref.find(q)
assert np.array_equal(r, MM.oracle_find(orc, q)), "the oracle's find_correspond differs from the reference source's"
np.savez_compressed(MM.GOLDEN, points=q, ref=r)
print("wrote", MM.GOLDEN, dict(points=q.shape, found=int(r[:, 0].sum()), planes=int(r[:, 3].sum())))
