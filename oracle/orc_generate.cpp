// ORACLE — TEST INFRASTRUCTURE ONLY. Restates VIOManager::generateVisualMapPoints (src/vio.cpp:804-906) up to the records its
// VisualPoint / Feature objects are built from: the frame pose of updateFrameState (:1690-1697), Frame::w2c, the
// isInFrame(pc.cast<int>(), border) gate, the grid cell and TYPE_MAP test, vk::shiTomasiScore, the strict per-cell maximum
// over the scan then add_from_voxel_map, and per TYPE_POINTCLOUD cell in cell order the cos_theta sign of the normal and
// getImagePatch(img, pc, patch, 0). vk::shiTomasiScore is vikit's (unpinned): restated here as the vikit stand-in of
// oracle/ref_shim/vikit/vision.h restates it, like the camera model (DESIGN.md §5). Checks esikf_vio_generate_points
// (tests/test_gpu_generate_points.py); pinned to the reference source's own generateVisualMapPoints (oracle/ref_generate.cpp,
// tests/test_oracle_generate.py). Built by oracle/generate.mk together with the parity oracle's translation units (handles of
// orc_vio_create from the same library: the camera, Rci / Pci and getImagePatch).
#include <cmath>
#include <cstdint>
#include <vector>

#include "orc_vio.hpp"

using namespace orc;

namespace {

float shi_tomasi_score(const Image &img, int u, int v) {
  float dXX = 0.0, dYY = 0.0, dXY = 0.0;
  const int halfbox_size = 4, box_size = 2 * halfbox_size, box_area = box_size * box_size;
  const int x_min = u - halfbox_size, x_max = u + halfbox_size, y_min = v - halfbox_size, y_max = v + halfbox_size;
  if (x_min < 1 || x_max >= img.cols - 1 || y_min < 1 || y_max >= img.rows - 1) return 0.0;
  const int stride = img.cols;
  for (int y = y_min; y < y_max; ++y)
    for (int x = 0; x < box_size; ++x) {
      const uint8_t *p = img.data + stride * y + x_min + x;
      const float dx = p[1] - p[-1], dy = p[stride] - p[-stride];
      dXX += dx * dx, dYY += dy * dy, dXY += dx * dy;
    }
  dXX = dXX / (2.0 * box_area), dYY = dYY / (2.0 * box_area), dXY = dXY / (2.0 * box_area);
  return 0.5 * (dXX + dYY - std::sqrt((dXX + dYY) * (dXX + dYY) - 4 * (dXX * dYY - dXY * dXY)));
}

}  // namespace

extern "C" {

// generateVisualMapPoints on the pv list (point_w, normal, var: n x 3, n x 3, n x 9) and add_from (n_add x 3 positions and
// normals) with the grey image `img` (the camera's size), the frame pose of `state` and the TYPE_MAP mask (one byte per cell).
// Outputs in cell order, room for grid_n_width * grid_n_height entries each: source (scan index, or 0x40000000 | add_from
// index), cell, pos (3), pc (2), score, normal (3, sign-flipped), var (9), patch (64). Returns their number.
int orc_generate_points(void *h, const uint8_t *img, const double *state, const double *point_w, const double *normal, const double *var, int n,
                        const double *add_pos, const double *add_normal, int n_add, const uint8_t *type_map, int grid_size, int grid_n_width,
                        int grid_n_height, int border, int32_t *source, int32_t *cell, double *pos, double *pc, float *score, double *normal_out,
                        double *var_out, float *patch) {
  VIOManager &v = *(VIOManager *)h;
  const Camera &cam = v.cam;
  if (n <= 10) return 0;
  M3 Rwi;
  for (int k = 0; k < 9; k++) Rwi.a[k] = state[k];
  const M3 Rcw = v.Rci * T(Rwi);
  const V3 Pcw = -((v.Rci * T(Rwi)) * v3(state[9], state[10], state[11])) + v.Pci;
  const int length = grid_n_width * grid_n_height;
  std::vector<float> scan_value(length, 0.0f);
  std::vector<int> winner(length, -1);
  Image im;
  im.data = img, im.cols = v.width, im.rows = v.height;
  auto where = [&](int s) { return s < n ? v3(point_w[3 * s], point_w[3 * s + 1], point_w[3 * s + 2]) : v3(add_pos[3 * (s - n)], add_pos[3 * (s - n) + 1], add_pos[3 * (s - n) + 2]); };
  for (int s = 0; s < n + n_add; s++) {  // the scan (:809-832), then add_from (:834-854)
    if (s < n && normal[3 * s] == 0.0 && normal[3 * s + 1] == 0.0 && normal[3 * s + 2] == 0.0) continue;
    const V2 p = cam.world2cam(Rcw * where(s) + Pcw);
    const int ui = (int)p[0], vi = (int)p[1];
    if (!(ui >= border && ui < cam.width - border && vi >= border && vi < cam.height - border)) continue;
    const int index = (int)(p[1] / grid_size) * grid_n_width + (int)(p[0] / grid_size);
    if (index < 0 || index >= length || type_map[index]) continue;  // past the grid the reference indexes out of bounds
    const float cur_value = shi_tomasi_score(im, (int)p[0], (int)p[1]);
    if (cur_value > scan_value[index]) scan_value[index] = cur_value, winner[index] = s;
  }
  int add = 0;
  std::vector<float> patch_tmp((size_t)64 * v.patch_pyrimid_level);
  for (int i = 0; i < length; i++) {  // :860-898
    const int s = winner[i];
    if (s < 0) continue;
    const V3 pt = where(s);
    const double *nw = s < n ? normal + 3 * s : add_normal + 3 * (s - n);
    const V3 nv = v3(nw[0], nw[1], nw[2]);
    const V3 norm_vec = Rcw * nv;
    V3 dir = Rcw * pt + Pcw;
    dir = dir / norm(dir);
    const double cos_theta = dot(dir, norm_vec);
    const V2 p = cam.world2cam(Rcw * pt + Pcw);
    v.getImagePatch(im, p, patch_tmp.data(), 0);
    source[add] = s < n ? s : (0x40000000 | (s - n));
    cell[add] = i;
    score[add] = scan_value[i];
    for (int k = 0; k < 3; k++) pos[3 * add + k] = pt[k], normal_out[3 * add + k] = cos_theta < 0 ? -nv[k] : nv[k];
    pc[2 * add] = p[0], pc[2 * add + 1] = p[1];
    for (int k = 0; k < 9; k++) var_out[9 * add + k] = s < n ? var[9 * s + k] : 0.0;
    for (int k = 0; k < 64; k++) patch[64 * add + k] = patch_tmp[k];
    add++;
  }
  return add;
}

}  // extern "C"
