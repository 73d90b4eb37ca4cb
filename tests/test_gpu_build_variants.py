"""The compile-time variants of the update kernels (__graft_entry__.VARIANTS, built by build() next to the default library)
against the default build and the oracle. They are kept so that they can be timed against the default (DESIGN §8), and a
variant that no longer computes what the default computes would make such a timing compare against a broken build:

  full_rec       cold LIO candidates read their whole 144-byte plane record in one trip, with their own copy of the record
                 unpacking and of sigma_plane: every LIO output byte-equal to the default's;
  cold_noinline  the LIO cold paths out of line: every LIO output byte-equal;
  l2w0           only the 704-lane LIO kernel: byte-equal where the default runs it too; where the default runs the 768-lane
                 kernel (23 or 24 chunks per CTA) the association, counts, iterations and distances are byte-equal and the
                 sums (state, information, solution, residual) within 1e-12 relative, since warp 0 of each CTA contracts one
                 more chunk there;
  chain_stamps   the VIO kernel writes its chain stamps: VIO and LIO outputs byte-equal, with phase stamps off and on, and
                 after a persistent update the stamps are in exactly the words the layout of csrc/esikf_fused.cu names.

Every library runs the cases of tests/variant_driver.py in a process of its own (ESIKF_LIB is read at import); the driver
asserts that the launch forms of one library are bit-identical. A variant library that is missing is a failure: build()
makes them."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import __graft_entry__ as GE
import variant_driver as D
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S
from harness import LIO_KEYS, VIO_KEYS, bits_equal, compare_lio, compare_vio, lio_oracle, sm_count
from parity_util import rel

DRIVER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "variant_driver.py")
# what the 704- and the 768-lane kernels decide alike (association first), then the sums over a CTA's warps
L2W0_EXACT = ("match_plane", "normal_plane", "dis_to_plane", "M", "converged", "iters")
L2W0_SUMS = ("state", "HTH", "HTz", "solution", "total_residual")
L2W0_RTOL = 1e-12
LIO_OUT = L2W0_EXACT + L2W0_SUMS
assert set(LIO_OUT) == set(LIO_KEYS + ("iters",))
VIO_OUT = VIO_KEYS + ("total_iters",)
VIO_WARPS = 16  # warps of a VIO CTA: one patch per warp while the patches last (vio_grid, csrc/esikf_api_update.cu)


def c_abi(lib):
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    return sorted(s for s in (line.split()[-1] for line in out.splitlines()) if s.startswith("esikf_"))


def test_variant_libraries_are_built_with_the_default_c_abi():
    """build() makes every variant library, each exporting the C ABI of the default one."""
    want = c_abi(GE.LIB)
    assert len(want) >= 30
    for name in GE.VARIANTS:
        lib = GE.variant_lib(name)
        assert os.path.exists(lib), f"{lib} is missing: __graft_entry__.build() makes it"
        assert c_abi(lib) == want, name


# ----------------------------------------------------------------------------------------------------------- GPU runs
def run_driver(lib, names, out):
    assert os.path.exists(lib), f"{lib} is missing: __graft_entry__.build() makes it"
    t0 = time.perf_counter()
    r = subprocess.run([sys.executable, DRIVER, str(out), *names], env=dict(os.environ, ESIKF_LIB=lib), capture_output=True, text=True)
    assert r.returncode == 0, f"{lib}:\n{r.stderr[-6000:]}"
    print(f"{os.path.relpath(lib, GE.ROOT)}: {len(names)} cases in {time.perf_counter() - t0:.1f} s")
    return np.load(out)


def case_of(npz, name, keys):
    return {k: npz[f"{name}/{k}"] for k in keys}


def same(name, a, b, keys):
    try:
        bits_equal(a, b, keys)
    except AssertionError as e:
        raise AssertionError(f"{name}: {e} differs from the default build") from None


def grid():
    return min(sm_count(), 160)


def chain_lio_cases(G):
    """LIO cases for the stamped build (csrc/esikf_fused.cu changes with it): the 768-lane kernel and the 704-lane one."""
    return ["cfg2", f"main_n{G * D.A.SMEM_LANES}"]


@pytest.fixture(scope="module")
def default_outputs(gpu_ctx, tmp_path_factory):
    G = grid()
    names = [*D.lio_cases(G), *D.VIO_CASES, *chain_lio_cases(G)]
    return run_driver(GE.LIB, list(dict.fromkeys(names)), tmp_path_factory.mktemp("variants") / "default.npz")


_oracle = {}


def oracle(name, make):
    if name not in _oracle:
        _oracle[name] = make()
    return _oracle[name]


def state_rel(a, b):
    """The largest relative difference over the blocks of the packed state (rotation, position, ..., covariance)."""
    ua, ub = S.unpack_state(a), S.unpack_state(b)
    return max(rel(ua[k], ub[k]) for k in ub)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["full_rec", "cold_noinline", "l2w0"])
def test_lio_variant_computes_what_the_default_computes(default_outputs, variant, tmp_path):
    """The hand-built association cases (main, displaced, zero_prob) at every slice size of the resident / tiled and 768-lane
    boundary tests and with every designed warp in lanes 704-767, config 2's 100 k points and config 4's 260 k, in loop modes
    2 and 0 with both record stagings: byte-equal to the default build (l2w0: see the module docstring) and bit for bit
    against the oracle's association."""
    G = grid()
    cases = D.lio_cases(G)
    got = run_driver(GE.variant_lib(variant), list(cases), tmp_path / f"{variant}.npz")
    worst = {}  # l2w0: sum -> (largest relative difference from the default build, case)
    for name, make in cases.items():
        g, d = case_of(got, name, LIO_OUT), case_of(default_outputs, name, LIO_OUT)
        if variant == "l2w0" and D.uses_l2_slots(len(d["match_plane"]), G):
            same(name, g, d, L2W0_EXACT)
            for k in L2W0_SUMS:
                diff = state_rel(g[k], d[k]) if k == "state" else rel(g[k], d[k])
                assert diff <= L2W0_RTOL, (name, k, diff)
                worst[k] = max(worst.get(k, (0.0, None)), (diff, name), key=lambda x: x[0])
        else:
            same(name, g, d, LIO_OUT)
        o = oracle(name, lambda: lio_oracle(make()))
        compare_lio(d, o)
        compare_lio(g, o)
    if variant == "l2w0":
        assert worst, "no case ran the 768-lane kernel in the default build"
        print("l2w0, largest relative difference from the default build:", ", ".join(f"{k} {v[0]:.3g} ({v[1]})" for k, v in worst.items()))


def check_chain(chain, r, c, G, stamped):
    """The chain stamps after a persistent update: in the stamped build warp 0's four segment stamps of every (level,
    iteration) slot that ran (non-decreasing; the forward update's patch build only) and one slice-end stamp per CTA and
    slot, nothing anywhere else; in any other build nothing at all."""
    L, max_it, n = c["vio_cfg"].levels, c["vio_cfg"].max_iterations, len(c["args"][1])
    ctas = min(-(-n // VIO_WARPS), G)
    want = np.zeros(api.VIO_CHAIN_STAMP_WORDS, bool)
    if stamped:
        for level in range(L):
            for it in range(int(r["iters_per_level"][level])):
                s = (L - 1 - level) * max_it + it
                if not c["vio_cfg"].inverse_composition_en:
                    want[8 * s: 8 * s + 4] = True
                    assert np.all(np.diff(chain[8 * s: 8 * s + 4].astype(np.int64)) >= 0), (s, chain[8 * s: 8 * s + 4])
                want[api.VIO_CHAIN_CTA + api.VIO_CHAIN_MAX_CTAS * s: api.VIO_CHAIN_CTA + api.VIO_CHAIN_MAX_CTAS * s + ctas] = True
        assert want.sum() > 0
    assert np.array_equal(chain != 0, want), np.nonzero((chain != 0) != want)[0][:16]


@pytest.mark.gpu
def test_chain_stamps_variant_computes_what_the_default_computes(default_outputs, tmp_path):
    """Forward and inverse updates on a synthetic frame, config 5's 4 k patches (two per warp) and a sub-map from 12
    keyframes, in loop modes 2 and 0 with and without TMA tap staging, with phase stamps off and on: byte-equal to the
    default build and against the oracle; the chain stamps where the layout puts them (check_chain). LIO updates on the
    768- and the 704-lane kernel byte-equal too."""
    G = grid()
    lio = chain_lio_cases(G)
    got = run_driver(GE.variant_lib("chain_stamps"), [*D.VIO_CASES, *lio], tmp_path / "chain_stamps.npz")
    for name, make in D.VIO_CASES.items():
        c = make()
        g, d = case_of(got, name, VIO_OUT), case_of(default_outputs, name, VIO_OUT)
        same(name, g, d, VIO_OUT)
        o = oracle(name, lambda: D.vio_oracle(c))
        assert o["total_iters"] >= 4
        compare_vio(g, o, c["vio_cfg"].levels)
        check_chain(got[f"{name}/chain"], g, c, G, stamped=True)
        check_chain(default_outputs[f"{name}/chain"], d, c, G, stamped=False)
    for name in lio:
        same(name, case_of(got, name, LIO_OUT), case_of(default_outputs, name, LIO_OUT), LIO_OUT)
