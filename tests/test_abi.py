"""CPU checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/esikf_b200.h declares
(no compute calls without a GPU), struct layouts agree between the header and the ctypes binding, the context refuses
to exist without a device (no CPU fallback), and the C++ shim's map flattener round-trips."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import shim_bind as SB
from fast_livo2_b200 import api
from fast_livo2_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "esikf_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(esikf_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = api.load_library()
    names = _header_functions()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/esikf_b200.h but not exported by libesikf_b200.so"
    assert set(api.EXPORTED_SYMBOLS) <= set(names)


def test_struct_layouts_match_header():
    assert S.PLANE_DTYPE.itemsize == 256 and S.PLANE_DTYPE.fields["d"][1] == 216 and S.PLANE_DTYPE.fields["layer"][1] == 224
    assert C.sizeof(api.LioCfgC) == 40 and C.sizeof(api.ExtrinsicsC) == 192 and C.sizeof(api.CameraC) == 88 and C.sizeof(api.VioCfgC) == 24
    assert C.sizeof(api.LioStatsC) == 4 * 18 + 8 * (8 + 8 * 36 + 8 * 6 + 8 * 19)
    assert C.sizeof(api.VioStatsC) == 4 * 18 + 4 * 64 + 8 * 64 * (49 + 7 + 19)
    assert api.STATE_DOUBLES == 386 == S.STATE_PACK


def test_no_cpu_fallback_without_device():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(api.EsikfError):
        api.Context(0)


def test_shim_flattener_roundtrip(small_frame):
    """fl2_shim: flat arrays -> pointer octree (VoxelOctoTree mirrors) -> FlattenVoxelMap -> identical candidate lists."""
    if not os.path.exists(SB.PATH):
        pytest.skip("shim not built")
    api.load_library()
    shim = SB.load()
    m = small_frame["map"]
    k, f, c, p = (np.ascontiguousarray(m["keys"]), np.ascontiguousarray(m["first"]), np.ascontiguousarray(m["count"]), np.ascontiguousarray(m["planes"]))
    ko, fo, co, po = np.zeros_like(k), np.zeros_like(f), np.zeros_like(c), np.zeros_like(p)
    rc = shim.fl2_shim_flatten_roundtrip(k.ctypes.data_as(C.c_void_p), f.ctypes.data_as(C.c_void_p), c.ctypes.data_as(C.c_void_p), len(f),
                                         p.ctypes.data_as(C.c_void_p), len(p), C.c_double(0.5), 2, ko.ctypes.data_as(C.c_void_p),
                                         fo.ctypes.data_as(C.c_void_p), co.ctypes.data_as(C.c_void_p), po.ctypes.data_as(C.c_void_p))
    assert rc == 0
    src = {tuple(kk): (ff, cc) for kk, ff, cc in zip(k.tolist(), f, c)}
    assert len(src) == len(fo)
    for kk, ff, cc in zip(ko.tolist(), fo, co):
        f0, c0 = src[tuple(kk)]
        assert cc == c0
        for j in range(cc):
            a, b = p[f0 + j], po[ff + j]
            for name in ("center", "normal", "plane_var", "d", "radius", "layer", "path"):
                assert np.array_equal(a[name], b[name]), name


def test_shim_map_diff_finds_refitted_planes_and_structure_changes(small_frame):
    """fl2_shim DiffFlatVoxelMaps: what VoxelMapManager::SyncDeviceMap uses to choose between esikf_map_patch (same roots and
    candidate lists, some refitted plane records) and a full esikf_map_upload."""
    shim = SB.load()
    m = small_frame["map"]
    k, f, c = (np.ascontiguousarray(m["keys"], dtype=np.int64), np.ascontiguousarray(m["first"], dtype=np.int32), np.ascontiguousarray(m["count"], dtype=np.int32))
    pa = np.ascontiguousarray(m["planes"]).copy()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    ids = np.zeros(len(pa), np.int32)

    def diff(k2, f2, c2, pb):
        return shim.fl2_shim_diff(vp(k), vp(f), vp(c), len(f), vp(pa), len(pa), vp(k2), vp(f2), vp(c2), len(f2), vp(pb), len(pb), vp(ids))

    assert diff(k, f, c, pa.copy()) == 0
    pb = pa.copy()
    touched = [0, 7, len(pb) - 1]
    pb["d"][touched[0]] += np.float32(0.25)
    pb["normal"][touched[1]] = -pb["normal"][touched[1]]
    pb["plane_var"][touched[2], 3] *= 1.5
    assert diff(k, f, c, pb) == 3 and ids[:3].tolist() == touched
    # a candidate list that grew / a new root voxel / a missing root: structure change -> full upload
    c2 = c.copy()
    c2[0] += 1
    assert diff(k, f, c2, pa) == -1
    k2 = np.concatenate([k.reshape(-1, 3), [[9999, 9999, 9999]]]).astype(np.int64)
    assert diff(np.ascontiguousarray(k2), np.append(f, 0).astype(np.int32), np.append(c, 0).astype(np.int32), pa) == -1
    assert diff(np.ascontiguousarray(k.reshape(-1, 3)[:-1]), f[:-1].copy(), c[:-1].copy(), pa) == -1


def test_example_tick_loop_compiles_and_runs(tmp_path):
    """examples/tick_loop.cpp (the LIVMapper call sequence through the shim classes) builds with -Wall -Wextra against the
    in-tree libraries; without a device it reports the missing GPU and exits cleanly (no CPU fallback), with one it runs a tick pair."""
    import subprocess

    exe = str(tmp_path / "tick_loop")
    pkg = os.path.join(ROOT, "fast_livo2_b200")
    cmd = ["/usr/bin/g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "tick_loop.cpp"),
           "-L" + pkg, "-lfl2_shim", "-lesikf_b200", "-Wl,-rpath," + pkg, "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    run = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "no usable device" in run.stdout or ("BuildVoxelMap: status 0" in run.stdout and "tick 3 LIO: status 0" in run.stdout), run.stdout
