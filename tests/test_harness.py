"""The GPU tests' launch variants, on a stand-in context that records the mode setters: the defaults come back whatever the
body does, and a sweep runs its variants in the order given."""
import os
import subprocess
import sys

import pytest

from fast_livo2_b200 import api
from harness import sweep, variant

DEFAULTS = {"loop_mode": api.DEFAULT_LOOP_MODE, "solve_mode": 0, "tuning": 0}


class RecordingContext:
    def __init__(self):
        self.calls = []
        self.modes = dict(DEFAULTS)

    def _set(self, name, value):
        self.calls.append((name, value))
        self.modes[name] = value

    def set_loop_mode(self, mode):
        self._set("loop_mode", mode)

    def set_solve_mode(self, mode):
        self._set("solve_mode", mode)

    def set_tuning(self, flags):
        self._set("tuning", flags)


def test_variant_sets_the_modes_and_restores_the_defaults():
    ctx = RecordingContext()
    with variant(ctx, loop_mode=0, solve_mode=1, tuning=api.TUNE_VIO_TMA):
        assert ctx.modes == {"loop_mode": 0, "solve_mode": 1, "tuning": api.TUNE_VIO_TMA}
    assert ctx.modes == DEFAULTS
    assert ctx.calls[-3:] == [("loop_mode", api.DEFAULT_LOOP_MODE), ("solve_mode", 0), ("tuning", 0)]


def test_variant_restores_the_defaults_when_the_body_raises():
    ctx = RecordingContext()
    with pytest.raises(ZeroDivisionError):
        with variant(ctx, loop_mode=1, solve_mode=1, tuning=api.TUNE_STAGE_LDG):
            1 / 0
    assert ctx.modes == DEFAULTS


def test_variant_restores_the_defaults_when_a_setter_refuses():
    """A mode the library refuses (EsikfError) leaves the context in its defaults, not half set."""
    ctx = RecordingContext()
    set_tuning = ctx.set_tuning

    def checked(flags):
        if flags & ~(api.TUNE_STAGE_LDG | api.TUNE_VIO_TMA):
            raise api.EsikfError("esikf_set_tuning: status -3")
        set_tuning(flags)

    ctx.set_tuning = checked
    with pytest.raises(api.EsikfError):
        with variant(ctx, loop_mode=0, solve_mode=1, tuning=8):
            pass
    assert ctx.modes == DEFAULTS


def test_sweep_runs_the_variants_in_order():
    ctx = RecordingContext()
    variants = [dict(loop_mode=0), dict(loop_mode=2), dict(loop_mode=2), dict(loop_mode=0, solve_mode=1), dict(tuning=api.TUNE_VIO_TMA)]
    seen = sweep(ctx, lambda: dict(ctx.modes), variants)
    assert seen == [{**DEFAULTS, **v} for v in variants]
    assert ctx.modes == DEFAULTS


def test_sweep_stops_at_a_failing_run_and_restores_the_defaults():
    ctx = RecordingContext()
    runs = []

    def run():
        runs.append(ctx.modes["loop_mode"])
        if len(runs) == 2:
            raise AssertionError("bits differ")
        return runs[-1]

    with pytest.raises(AssertionError):
        sweep(ctx, run, [dict(loop_mode=0), dict(loop_mode=1), dict(loop_mode=0)])
    assert runs == [0, 1] and ctx.modes == DEFAULTS


def test_importing_the_harness_loads_no_torch():
    """CPU-only collection imports the harness: it must not pull in torch (or touch a device) on import."""
    tests = os.path.dirname(os.path.abspath(__file__))
    path = os.pathsep.join([tests, os.path.dirname(tests)] + [p for p in [os.environ.get("PYTHONPATH")] if p])
    r = subprocess.run([sys.executable, "-c", "import sys, harness; sys.exit('torch' in sys.modules)"], env=dict(os.environ, PYTHONPATH=path),
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
