"""Regenerates tests/golden/ref_pin/keyframes.npz: the REFERENCE SOURCE's VIO update (oracle/_ref/libfl2_ref_vio.so, built by
`make -C oracle` from a FAST-LIVO2 source tree) on the many-keyframe sub-maps of tests/keyframe_cases.py, recorded by running
tests/test_oracle_ref_pin_keyframes.py live, which checks the oracle against every output before it is stored:
    python tests/golden/make_keyframes_golden.py"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_bind as O  # noqa: E402

assert O.ref_lio_available() and O.ref_vio_available(), "build oracle/_ref first (make -C oracle)"
sys.exit(subprocess.run([sys.executable, "-m", "pytest", "-q", os.path.join(ROOT, "tests", "test_oracle_ref_pin_keyframes.py")], cwd=ROOT,
                        env=dict(os.environ, FL2_RECORD_REF_PIN="1")).returncode)
