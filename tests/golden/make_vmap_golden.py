"""Regenerates tests/golden/ref_pin/vmap.npz: what the REFERENCE SOURCE's own VisualPoint / Feature objects hold when its own
updateVisualMapPoints, updateReferencePatch and getCloseViewObs (oracle/_ref/libfl2_ref_vmap.so, built by oracle/vmap.mk from
/root/reference/src/vio.cpp and src/visual_point.cpp) run over the tick sequence of tests/vmap_cases.py, and on its
hand-built states. Per tick: the flags, the frame's T_f_w_, getCloseViewObs of the retrieved points and the digests of every
list. Run in the build container (needs /root/reference):   python tests/golden/make_vmap_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import vmap_cases as VC  # noqa: E402

assert VC.ref_available(), "build oracle/_ref first (make -C oracle -f vmap.mk)"
r = VC.reference_sequence()
assert all(r["has_ref_ok"])
out = dict(seq_flag=np.concatenate(r["flag"]), seq_flag_n=np.array([len(f) for f in r["flag"]]), seq_T=np.array(r["T"]), seq_close=np.concatenate(r["close"]), seq_close_n=np.array([len(c) for c in r["close"]]),
           seq_digest=np.array(r["digest"]))
for k, v in VC.reference_hand().items():
    out[f"hand_{k}"] = v
np.savez_compressed(VC.GOLDEN, **out)
print("wrote", VC.GOLDEN, os.path.getsize(VC.GOLDEN), "bytes")
