"""GPU: the LIO plane association on hand-built maps (tests/lio_assoc.py) against the oracle, bit for bit. These maps reach
what the synthetic ones hardly do: the warp-cooperative cold path of csrc/esikf_lio.cu with pair ranges that span
several chunks of 32, exact probability ties between the hot-path candidate and cold duplicates and between extras in
one chunk or in different chunks, deep octrees, neighbour voxels with one to 130 candidates, ties, no plane or none, and
(sigma_num = 40) passing candidates whose this_prob underflows to 0: unmatched, and at home they block the neighbour
probe, as in the reference."""
import numpy as np
import pytest

import lio_assoc as A
import oracle_bind as O
from fast_livo2_b200 import api
from test_gpu_lio import _compare
from test_gpu_loop_modes import LIO_KEYS, _bits_equal

pytestmark = pytest.mark.gpu


def _oracle(fr):
    lio = O.OracleLIO(fr["lio_cfg"], fr["ext"])
    lio.set_map(fr["map"])
    return lio.state_estimation(fr["pts"], fr["state_prior"], fr["state_prior"])


def _gpu(ctx, fr, loop_mode=api.DEFAULT_LOOP_MODE, tuning=0):
    try:
        ctx.set_loop_mode(loop_mode)
        ctx.set_tuning(tuning)
        ctx.set_extrinsics(fr["ext"])
        ctx.map_upload(fr["map"], fr["lio_cfg"].voxel_size)
        return ctx.lio_update(fr["pts"], fr["state_prior"], fr["state_prior"], fr["lio_cfg"])
    finally:
        ctx.set_loop_mode(api.DEFAULT_LOOP_MODE)
        ctx.set_tuning(0)


def _sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("name", A.CASES)
def test_association_matches_oracle_in_every_loop_mode_and_staging(gpu_ctx, name):
    """loop_mode 2 / 1 (persistent) and 0 (per-iteration launches), and ESIKF_TUNE_STAGE_LDG against the default bulk-copy
    staging: bit-identical to each other, and association / counts / distances bit for bit against the oracle."""
    fr = A.case(name)
    o = _oracle(fr)
    runs = [_gpu(gpu_ctx, fr, m) for m in (2, 1, 0)] + [_gpu(gpu_ctx, fr, 2, api.TUNE_STAGE_LDG)]
    for r in runs:
        _compare(r, o)
        _bits_equal(runs[0], r, LIO_KEYS)
    assert o["M"].min() > 50


def test_zero_probability_passes_are_unmatched_and_block_the_neighbour(gpu_ctx):
    """sigma_num = 40: the points placed 38.7-39.9 sigma off every plane of their home voxel pass the gate with
    this_prob == 0. None of them is matched, although a plane of their neighbour voxel runs right through each."""
    fr = A.case("zero_prob")
    g = _gpu(gpu_ctx, fr)
    o = _oracle(fr)
    lio = O.OracleLIO(fr["lio_cfg"], fr["ext"])
    lio.set_map(fr["map"])
    first = lio.single_pass(fr["pts"], fr["state_prior"], fr["state_prior"])["plane"]
    z = np.array([t.startswith("zero_prob") and "ok" not in t for t in fr["tags"]])
    assert z.sum() >= 10 and (first[z] == -1).all()
    _compare(g, o)


@pytest.mark.parametrize("name", A.CASES)
def test_resident_and_tiled_slices(gpu_ctx, name):
    """The designed warps repeated to sizes around the device's launch geometry (one CTA per SM, 704 lanes each, slices
    of whole 32-point chunks): 1, 31, 33 points; every CTA one chunk, the last partial, until one CTA gets a second;
    fully resident; one CTA tiling while the others stay resident; 2.5 rounds of tiles."""
    G = min(_sm_count(), 160)
    R = G * 704
    fr = A.case(name)
    for n in (1, 31, 33, 32 * G - 1, 32 * G, 32 * G + 1, R, R + 1, int(2.5 * R)):
        f = A.tiled(fr, n)
        g, o = _gpu(gpu_ctx, f), _oracle(f)
        _compare(g, o)
        if n >= R:
            _bits_equal(g, _gpu(gpu_ctx, f, 0), LIO_KEYS)
