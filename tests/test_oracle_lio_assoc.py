"""CPU: the hand-built association maps of tests/lio_assoc.py are valid octrees, and they really contain the cases the
device's cold path must get right (counted in numpy from the map, the scan and the oracle's outputs), so that none of
them can silently disappear from tests/test_gpu_lio_assoc.py."""
import numpy as np
import pytest

import lio_assoc as A
import oracle_bind as O
from fast_livo2_b200 import synthetic as S


def _runs(fr):
    lio = O.OracleLIO(fr["lio_cfg"], fr["ext"])
    lio.set_map(fr["map"])
    first = lio.single_pass(fr["pts"], fr["state_prior"], fr["state_prior"])["plane"]
    return first, lio.state_estimation(fr["pts"], fr["state_prior"], fr["state_prior"])


def test_every_cold_path_case_is_present():
    tot = {}
    for name in ("main", "zero_prob"):  # placed at the identity prior: the numpy association applies
        fr = A.case(name)
        first, o = _runs(fr)
        for k, v in A.coverage(fr, first, o["match_plane"]).items():
            tot[k] = tot.get(k, 0) + v
    first, o = _runs(A.case("displaced"))
    tot["changed_match"] += int((first != o["match_plane"]).sum())
    assert tot.pop("range_boundary_wrong", 0) == 0, "a one-ulp radius point is on the wrong side of the range gate"
    tot.pop("nb_other", None)  # neighbour roots with 10-33 candidates: not a designed kind
    for k, v in tot.items():
        assert v > 0, f"no {k} in the hand-built cases: {tot}"
    assert tot["warp_pairs_over_256"] >= 2 and tot["ties"] >= 10 and tot["zero_prob_pass"] >= 10


@pytest.mark.parametrize("name", A.CASES)
def test_hand_built_maps_are_valid_octrees(name):
    fr = A.case(name)
    A.validate_map(fr["map"], fr["lio_cfg"].max_layer)
    planes = fr["map"]["planes"]
    assert (planes["layer"] == fr["lio_cfg"].max_layer).any()
    assert len(fr["pts"]) % 32 == 0


def test_validator_rejects_broken_maps():
    fr = A.case("main")
    vm = fr["map"]
    r = int(np.argmax(vm["count"]))
    f, c = int(vm["first"][r]), int(vm["count"][r])

    def broken(edit):
        planes = vm["planes"].copy()
        edit(planes)
        return dict(vm, planes=planes)

    def swap(p):
        p[[f, f + 1]] = p[[f + 1, f]]

    def dup(p):
        p["layer"][f + 1], p["path"][f + 1] = p["layer"][f], p["path"][f]

    def above(p):
        p["layer"][f], p["path"][f] = 1, int(p["path"][f + 1]) & 7  # the layer-1 ancestor of the next record

    for edit in (swap, dup, above):
        with pytest.raises(AssertionError):
            A.validate_map(broken(edit), fr["lio_cfg"].max_layer)
    with pytest.raises(AssertionError):
        A.validate_map(vm, fr["lio_cfg"].max_layer - 1)
    assert c > 64 and vm["planes"].dtype == S.PLANE_DTYPE
