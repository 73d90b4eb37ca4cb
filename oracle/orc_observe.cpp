// ORACLE — TEST INFRASTRUCTURE ONLY. Restates VIOManager::updateVisualMapPoints (src/vio.cpp:908-967) up to the Feature objects
// it creates: the frame pose of updateFrameState (:1690-1697), per sub-map entry the converged skip, Frame::w2c, the pose of the
// entry's oldest observation against the frame (delta_pose = pose_ref * pose_cur.inverse(), delta_p, delta_theta with acos as
// the reference evaluates it), the pixel distance, the add rule, and for each added entry in entry order its pixel and
// getImagePatch(img, pc, patch, 0). Checks esikf_vio_update_points (tests/test_gpu_update_points.py); pinned to the reference
// source's own updateVisualMapPoints (oracle/ref_observe.cpp, tests/test_oracle_observe.py). Built by oracle/observe.mk together
// with the parity oracle's translation units (handles of orc_vio_create from the same library: the camera, Rci / Pci and
// getImagePatch).
#include <cmath>
#include <cstdint>
#include <vector>

#include "orc_vio.hpp"

using namespace orc;

extern "C" {

// updateVisualMapPoints on n sub-map entries (pos: n x 3; converged: n bytes; last_T: n x 12, obs_.back()->T_f_w_ as R
// row-major then t; last_px: n x 2, obs_.back()->px_) with the grey image `img` (the camera's size) and the frame pose of
// `state`. Outputs: update_flag (n bytes), and for the added entries in entry order, room for n each: entry, pc (2), patch (64).
// Returns their number.
int orc_update_points(void *h, const uint8_t *img, const double *state, const double *pos, const uint8_t *converged, const double *last_T,
                      const double *last_px, int n, uint8_t *update_flag, int32_t *entry, double *pc, float *patch) {
  VIOManager &v = *(VIOManager *)h;
  M3 Rwi;
  for (int k = 0; k < 9; k++) Rwi.a[k] = state[k];
  const M3 Rcw = v.Rci * T(Rwi);
  const V3 Pcw = -((v.Rci * T(Rwi)) * v3(state[9], state[10], state[11])) + v.Pci;
  const SE3 pose_cur(Rcw, Pcw);
  Image im;
  im.data = img, im.cols = v.width, im.rows = v.height;
  std::vector<float> patch_tmp((size_t)64 * v.patch_pyrimid_level);
  int add = 0;
  for (int i = 0; i < n; i++) {
    update_flag[i] = 0;
    if (converged[i]) continue;  // :918-922
    const V2 p = v.cam.world2cam(Rcw * v3(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]) + Pcw);  // :924
    const double *Tr = last_T + 12 * (size_t)i;
    M3 Rr;
    for (int k = 0; k < 9; k++) Rr.a[k] = Tr[k];
    const SE3 delta_pose = SE3(Rr, v3(Tr[9], Tr[10], Tr[11])) * pose_cur.inverse();  // :935-936
    const double delta_p = norm(delta_pose.t);
    const double trace = delta_pose.R(0, 0) + delta_pose.R(1, 1) + delta_pose.R(2, 2);
    const double delta_theta = (trace > 3.0 - 1e-6) ? 0.0 : std::acos(0.5 * (trace - 1));
    V2 d;
    d[0] = p[0] - last_px[2 * i], d[1] = p[1] - last_px[2 * i + 1];
    const double pixel_dist = norm(d);  // :942-943
    if (!(delta_p > 0.5 || delta_theta > 0.3 || pixel_dist > 40)) continue;
    update_flag[i] = 1;
    v.getImagePatch(im, p, patch_tmp.data(), 0);  // :927-928
    entry[add] = i;
    pc[2 * add] = p[0], pc[2 * add + 1] = p[1];
    for (int k = 0; k < 64; k++) patch[64 * add + k] = patch_tmp[k];
    add++;
  }
  return add;
}

}  // extern "C"
