"""Regenerates tests/golden/ref_pin/color.npz: the coloured scan of publish_frame_world on the REFERENCE SOURCE's own
updateFrameState / w2f / w2c / isInFrame / getInterpolatedPixel (oracle/_ref/libfl2_ref_color.so, built by oracle/color.mk
from /root/reference/src/vio.cpp) on the pin scenes of tests/color_cases.py, checked against the oracle's restatement before
it is written. Run in the build container (needs /root/reference):   python tests/golden/make_color_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import color_cases as CC  # noqa: E402
from test_oracle_color import oracle_pins, reference_pins  # noqa: E402

assert CC.ref_color_available(), "build oracle/_ref first (make -C oracle -f color.mk)"
ref, orc = reference_pins(), oracle_pins()
for k in ref:
    assert ref[k].tobytes() == orc[k].tobytes(), f"the oracle differs from the reference source on {k}"
np.savez_compressed(CC.GOLDEN, **ref)
print("wrote", CC.GOLDEN, {k: v.shape for k, v in ref.items()})
