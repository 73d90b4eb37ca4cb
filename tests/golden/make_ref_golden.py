"""Regenerates tests/golden/ref_lio_golden.npz: the outputs of the REFERENCE SOURCE (oracle/_ref/libfl2_ref_lio.so =
/root/reference/src/voxel_map.cpp compiled against oracle/ref_shim/) on two seeded synthetic frames. Run in the build
container (needs /root/reference):   python tests/golden/make_ref_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import oracle_bind as O  # noqa: E402
from ref_pin_cases import lio_case, vio_inputs  # noqa: E402

assert O.ref_lio_available(), "build oracle/_ref first (make -C oracle)"
out = {}
for name in ("small", "hilti_voxel_04_non_identity_extrinsics"):
    fr, cfg = lio_case(name)
    r = O.ref_lio_state_estimation(fr, cfg=cfg)
    out[f"{name}_iters"] = np.int32(r["iters"])
    for k in ("M", "ptpl_center", "ptpl_dis", "normals", "state"):
        out[f"{name}_{k}"] = r[k]
np.savez_compressed(os.path.join(HERE, "ref_lio_golden.npz"), **out)
print("wrote", os.path.join(HERE, "ref_lio_golden.npz"), {k: np.asarray(v).shape for k, v in out.items()})

# ---- VIO half: oracle/_ref/libfl2_ref_vio.so = /root/reference/src/vio.cpp (+ frame.cpp, visual_point.cpp, voxel_map.cpp)
if O.ref_vio_available():
    vout = {}
    for name in ("small", "exposure"):
        fr, prior, w = vio_inputs(name)
        r = O.RefVIO(fr["cam_cfg"], fr["ext"], fr["vio_cfg"]).update(fr["img"], fr["vis_pos"], w["warp_patch"], w["search_levels"], fr["inv_ref_expo"], prior, prior)
        vout[f"{name}_state"], vout[f"{name}_errors"], vout[f"{name}_warp_patch"] = r["state"], r["errors"], w["warp_patch"]
        vout[f"{name}_search_levels"], vout[f"{name}_prior"] = w["search_levels"], prior
    np.savez_compressed(os.path.join(HERE, "ref_vio_golden.npz"), **vout)
    print("wrote", os.path.join(HERE, "ref_vio_golden.npz"), {k: np.asarray(v).shape for k, v in vout.items()})
