"""ctypes binding of the C++ shim's entry points (fast_livo2_b200/csrc/fl2_shim.cpp, libfl2_shim.so): the library is loaded
once, with the result and argument types of every fl2_shim_* hook declared here, for the tests and the timing tools."""
import ctypes as C

import __graft_entry__

PATH = __graft_entry__.SHIM_LIB

_vp, _i, _d, _ll = C.c_void_p, C.c_int, C.c_double, C.c_longlong
_FLAT = [_vp, _vp, _vp, _i, _vp, _i]  # keys, first, count, n_roots, planes, n_planes
# hook: (restype, argtypes)
HOOKS = {
    "fl2_shim_flatten_roundtrip": (_i, _FLAT + [_d, _i] + [_vp] * 4),
    "fl2_shim_diff": (_i, _FLAT + _FLAT + [_vp]),
    "fl2_shim_run": (_i, _FLAT + [_vp, _vp, _vp, _i] + [_vp] * 9 + [_i] + [_vp] * 6),
    "fl2_shim_resync_run": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "fl2_shim_select_run": (_i, [_vp] * 5 + [_i, _vp, _i] + [_vp] * 11),
    "fl2_shim_retrieve_run": (_i, [_vp] * 5 + [_i, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "fl2_shim_patch_helpers": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    "fl2_shim_score_ref_patches": (_i, [_i, _vp, _i] + [_vp] * 9),
    "fl2_shim_session_create": (_vp, _FLAT + [_vp] * 4 + [_i]),
    "fl2_shim_session_step": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i] + [_vp] * 7),
    "fl2_shim_session_point_lists": (None, [_vp, _i]),
    "fl2_shim_session_materialize": (_i, [_vp, _vp, _vp]),
    "fl2_shim_session_device_map": (_i, [_vp, _vp, _i, _vp, _d, _i, _ll]),
    "fl2_shim_session_device_map_mirror": (_i, [_vp, _vp, _i, _vp, _d, _i, _ll, _i, _i]),
    "fl2_shim_session_update_map": (_i, [_vp]),
    "fl2_shim_session_update_points": (_i, [_vp, _vp, _vp, _i]),
    "fl2_shim_session_map_sliding": (_i, [_vp, _vp, _i, _d]),
    "fl2_shim_session_find_correspond": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "fl2_shim_session_manager_ns": (_ll, [_vp]),
    "fl2_shim_session_context": (_vp, [_vp]),
    "fl2_shim_session_destroy": (None, [_vp]),
    "fl2_shim_mirror_create": (_vp, [_d, _i]),
    "fl2_shim_mirror_apply": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _i]),
    "fl2_shim_mirror_erase": (None, [_vp, _vp, _vp]),
    "fl2_shim_mirror_dump": (_i, [_vp, _vp, _i]),
    "fl2_shim_mirror_flatten": (_i, [_vp] * 7),
    "fl2_shim_mirror_find": (None, [_vp, _vp, _i, _vp]),
    "fl2_shim_vmap_enable": (_i, [_vp, C.c_int64]),
    "fl2_shim_vmap_add": (_i, [_vp, _i] + [_vp] * 9),
    "fl2_shim_vmap_update": (_i, [_vp, _vp, _i, _vp, _vp, C.c_int32] + [_vp] * 7),
    "fl2_shim_vmap_score": (_i, [_vp, _i] + [_vp] * 4),
    "fl2_shim_vmap_choose": (_i, [_vp, _i, _vp, _vp, _vp, _i, _vp]),
}

_lib = None


def load():
    """libfl2_shim.so with every hook of HOOKS declared (loaded on the first call)."""
    global _lib
    if _lib is None:
        lib = C.CDLL(PATH)
        for name, (res, args) in HOOKS.items():
            f = getattr(lib, name)
            f.restype, f.argtypes = res, args
        _lib = lib
    return _lib
