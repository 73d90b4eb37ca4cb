"""Regenerates tests/golden/ref_pin/find_keyed.npz: the REFERENCE SOURCE's own VIOManager::updateReferencePatch (rule A) and
ray-casting retrieveFromVisualSparseMap (rule B) on the reference's own map (oracle/_ref/libfl2_ref_find_keyed.so, built by
oracle/find_keyed.mk from the reference's src/vio.cpp and src/voxel_map.cpp), on the inputs of tests/test_oracle_find_keyed.py's
pinned scenes at voxel 0.5, 0.4 and 2.0, checked against the oracle's keyed restatement before it is written. Needs the
reference source:   python tests/golden/make_find_keyed_golden.py"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import map_find as MF  # noqa: E402
import test_oracle_find_keyed as T  # noqa: E402

assert MF.ref_available(), "build oracle/_ref first (make -C oracle -f find_keyed.mk)"
out = {}
for name in T.PIN_CFGS:
    cfg, ticks, orc, q, state, rays = T.pin_inputs(name)
    r = T.ref_outputs(name, cfg, ticks, q, state, rays)
    out.update({f"{name}_points": q, f"{name}_normal": r["normal"], f"{name}_samples_w": r["samples_w"], f"{name}_add": r["add"]})
np.savez_compressed(MF.GOLDEN, **out)
# the stored outputs pass the pins
sys.exit(pytest.main(["-q", "-p", "no:cacheprovider", os.path.join(os.path.dirname(HERE), "test_oracle_find_keyed.py")]))
