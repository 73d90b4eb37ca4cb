// ORACLE — TEST INFRASTRUCTURE ONLY. Restates the coloured scan LIVMapper publishes after a VIO update: the world cloud of the
// LIO tick (src/LIVMapper.cpp:435-443 with RGBpointBodyToWorld, :682-690) and publish_frame_world (:1140-1173) with the frame
// pose of VIOManager::updateFrameState (src/vio.cpp:1690-1697), Frame::w2f / w2c, vk::AbstractCamera::isInFrame and
// VIOManager::getInterpolatedPixel (src/vio.cpp:1742-1760). Checks esikf_rgb_set_cloud / esikf_rgb_colorize
// (tests/test_gpu_color.py); pinned to the reference source's own pieces (oracle/ref_color.cpp, tests/test_oracle_color.py).
// Built by oracle/color.mk together with the parity oracle's translation units (handles of orc_vio_create from the same
// library: the camera and Rci / Pci).
#include <cmath>
#include <cstdint>

#include "orc_vio.hpp"

using namespace orc;

namespace {

// The frame pose (Rcw, Pcw) of a packed state: Rcw = Rci Rwi^T, Pcw = -Rci Rwi^T Pwi + Pci
void frame_pose(const VIOManager &v, const double *state, M3 &Rcw, V3 &Pcw) {
  M3 Rwi;
  for (int k = 0; k < 9; k++) Rwi.a[k] = state[k];
  const V3 Pwi = v3(state[9], state[10], state[11]);
  Rcw = v.Rci * T(Rwi);
  Pcw = -((v.Rci * T(Rwi)) * Pwi) + v.Pci;
}

// Bilinear B G R at the float position of pc: the four weights are rounded to float from double products of (1 - s), the
// last one is a float product; each channel is a float sum of the four weighted taps, left to right.
void interpolated_bgr(const uint8_t *img, int width, const V2 &pc, float out[3]) {
  const float fu = (float)pc[0], fv = (float)pc[1];
  const int iu = (int)floorf(fu), iv = (int)floorf(fv);
  const float du = fu - (float)iu, dv = fv - (float)iv;
  const float w[4] = {(float)((1.0 - du) * (1.0 - dv)), (float)(du * (1.0 - dv)), (float)((1.0 - du) * dv), du * dv};
  const uint8_t *tl = img + ((size_t)iv * width + iu) * 3, *bl = tl + (size_t)width * 3;
  for (int ch = 0; ch < 3; ch++) {
    float s = w[0] * tl[ch];
    s = s + w[1] * tl[ch + 3];
    s = s + w[2] * bl[ch];
    s = s + w[3] * bl[ch + 3];
    out[ch] = s;
  }
}

}  // namespace

extern "C" {

// The world cloud: rot_end (extR p + extT) + pos_end of every body point, in double, stored as float. world_out: n x 3.
void orc_color_world(const double *extR, const double *extT, const double *state, const float *pts, int n, float *world_out) {
  M3 eR, R;
  for (int k = 0; k < 9; k++) eR.a[k] = extR[k], R.a[k] = state[k];
  const V3 eT = v3(extT[0], extT[1], extT[2]), t = v3(state[9], state[10], state[11]);
  for (int i = 0; i < n; i++) {
    const V3 p = v3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
    const V3 w = R * (eR * p + eT) + t;
    for (int k = 0; k < 3; k++) world_out[3 * i + k] = (float)w[k];
  }
}

// The coloured points of the world cloud `cloud` (n x 3 float) in the BGR image `bgr` (the camera's width x height x 3) with
// the frame pose of `state`, in cloud order: xyz_out (n_kept x 3), bgr_out (n_kept x 3: B, G, R), index_out (n_kept, cloud
// indices). Room for n entries each. Returns n_kept.
int orc_color_colorize(void *h, const float *cloud, int n, const uint8_t *bgr, const double *state, double blind_rgb_points, float *xyz_out, uint8_t *bgr_out,
                       int32_t *index_out) {
  const VIOManager &v = *(const VIOManager *)h;
  const Camera &cam = v.cam;
  M3 Rcw;
  V3 Pcw;
  frame_pose(v, state, Rcw, Pcw);
  int kept = 0;
  for (int i = 0; i < n; i++) {
    const V3 p_w = v3(cloud[3 * i], cloud[3 * i + 1], cloud[3 * i + 2]);
    const V3 pf = Rcw * p_w + Pcw;
    if (pf[2] < 0) continue;
    const V2 pc = cam.world2cam(pf);
    const int ui = (int)pc[0], vi = (int)pc[1];  // truncation toward zero
    if (!(ui >= 3 && ui < cam.width - 3 && vi >= 3 && vi < cam.height - 3)) continue;
    float col[3];
    interpolated_bgr(bgr, cam.width, pc, col);
    if (!(norm(pf) > blind_rgb_points)) continue;
    for (int k = 0; k < 3; k++) xyz_out[3 * kept + k] = cloud[3 * i + k], bgr_out[3 * kept + k] = (uint8_t)col[k];
    index_out[kept++] = i;
  }
  return kept;
}

}  // extern "C"
