// ORACLE — TEST INFRASTRUCTURE ONLY. Restates the per-candidate tail of VIOManager::retrieveFromVisualSparseMap
// (src/vio.cpp:645-770) for candidates whose reference feature the caller has already chosen, in the caller's order: the warp
// matrix in both forms (getWarpMatrixAffineHomography when normal_en, getWarpMatrixAffine with the per-frame warp_map cache
// otherwise), warpAffine on every pyramid level, the current patch, the exposure-weighted photometric error, calculateNCC,
// the NCC and outlier gates and the append of the survivors. Checks esikf_vio_select_patches (tests/test_gpu_select_patches.py);
// getWarpMatrixAffine + getBestSearchLevel and calculateNCC are pinned to the reference source's own (oracle/ref_select.cpp,
// tests/test_oracle_select.py). Built by oracle/select.mk together with the parity oracle's translation units (handles of
// orc_vio_create from the same library).
#include <cmath>
#include <cstring>
#include <unordered_map>
#include <utility>

#include "orc_vio.hpp"

using namespace orc;

namespace {

// src/vio.cpp:275-290
void getWarpMatrixAffine(const Camera &cam, const V2 &px_ref, const V3 &f_ref, const double depth_ref, const SE3 &T_cur_ref, const int level_ref,
                         const int pyramid_level, const int halfpatch_size, M2 &A_cur_ref) {
  const V3 xyz_ref = f_ref * depth_ref;
  V2 du, dv;
  du[0] = px_ref[0] + (double)halfpatch_size * (1 << level_ref) * (1 << pyramid_level), du[1] = px_ref[1] + 0.0;
  dv[0] = px_ref[0] + 0.0, dv[1] = px_ref[1] + (double)halfpatch_size * (1 << level_ref) * (1 << pyramid_level);
  V3 xyz_du_ref = cam.cam2world(du);
  V3 xyz_dv_ref = cam.cam2world(dv);
  xyz_du_ref = xyz_du_ref * (xyz_ref[2] / xyz_du_ref[2]);
  xyz_dv_ref = xyz_dv_ref * (xyz_ref[2] / xyz_dv_ref[2]);
  const V2 px_cur = cam.world2cam(T_cur_ref * xyz_ref);
  const V2 px_du = cam.world2cam(T_cur_ref * xyz_du_ref);
  const V2 px_dv = cam.world2cam(T_cur_ref * xyz_dv_ref);
  A_cur_ref(0, 0) = (px_du[0] - px_cur[0]) / halfpatch_size;
  A_cur_ref(1, 0) = (px_du[1] - px_cur[1]) / halfpatch_size;
  A_cur_ref(0, 1) = (px_dv[0] - px_cur[0]) / halfpatch_size;
  A_cur_ref(1, 1) = (px_dv[1] - px_cur[1]) / halfpatch_size;
}

// src/vio.cpp:333-350
double calculateNCC(const float *ref_patch, const float *cur_patch, int patch_size) {
  double sum_ref = 0.0;
  for (int i = 0; i < patch_size; i++) sum_ref = sum_ref + ref_patch[i];  // std::accumulate(..., 0.0)
  const double mean_ref = sum_ref / patch_size;
  double sum_cur = 0.0;
  for (int i = 0; i < patch_size; i++) sum_cur = sum_cur + cur_patch[i];
  const double mean_curr = sum_cur / patch_size;
  double numerator = 0, demoniator1 = 0, demoniator2 = 0;
  for (int i = 0; i < patch_size; i++) {
    double n = (ref_patch[i] - mean_ref) * (cur_patch[i] - mean_curr);
    numerator += n;
    demoniator1 += (ref_patch[i] - mean_ref) * (ref_patch[i] - mean_ref);
    demoniator2 += (cur_patch[i] - mean_curr) * (cur_patch[i] - mean_curr);
  }
  return numerator / std::sqrt(demoniator1 * demoniator2 + 1e-10);
}

SE3 se3(const double *T12) {  // R(9) t(3)
  SE3 T;
  for (int i = 0; i < 9; i++) T.R.a[i] = T12[i];
  for (int i = 0; i < 3; i++) T.t[i] = T12[9 + i];
  return T;
}
V2 v2(const double *p) {
  V2 v;
  v[0] = p[0], v[1] = p[1];
  return v;
}
V3 v3p(const double *p) { return v3(p[0], p[1], p[2]); }

// getWarpMatrixAffine + getBestSearchLevel chained as at :726-729 (depth = |ref_pos - pos|, pyramid_level 0, halfpatch 4)
int depth_warp(VIOManager *v, const double *px_ref, const double *f_ref, const double *ref_pos, const double *pos_w, const double *T_ref,
               const double *T_cur, int level_ref, M2 &A) {
  const double depth = norm(v3p(ref_pos) - v3p(pos_w));
  getWarpMatrixAffine(v->cam, v2(px_ref), v3p(f_ref), depth, se3(T_cur) * se3(T_ref).inverse(), level_ref, 0, v->patch_size_half, A);
  return v->getBestSearchLevel(A, 2);
}

}  // namespace

extern "C" {

// The depth-form warp matrix and search level of one candidate (no cache): A_out row-major 2 x 2, returns the level.
int orc_select_warp_matrix_affine(void *h, const double *px_ref, const double *f_ref, const double *ref_pos, const double *pos_w, const double *T_ref,
                                  const double *T_cur, int level_ref, double *A_out) {
  M2 A;
  const int sl = depth_warp((VIOManager *)h, px_ref, f_ref, ref_pos, pos_w, T_ref, T_cur, level_ref, A);
  for (int i = 0; i < 4; i++) A_out[i] = A.a[i];
  return sl;
}

double orc_select_calculate_ncc(const float *ref_patch, const float *cur_patch) { return calculateNCC(ref_patch, cur_patch, 64); }

// The tail :645-770 over n candidates in order. Inputs as esikf_vio_select_patches (T_* as R(9) t(3)); ref_imgs of
// ref_cols x ref_rows, img of the camera's size. A_in / sl_in (nullable, n x 4 / n): use these warp matrices and levels
// instead of computing them (to check the later steps on a device's own matrices). Outputs per candidate: A_out (n x 4),
// sl_out, warp_out (n x levels*64), error_out, keep_out (1 = appended); kept_index (n_kept, candidate order). Returns n_kept.
int orc_select_patches(void *h, int n, const uint8_t *const *ref_imgs, int ref_cols, int ref_rows, const uint8_t *img, const int32_t *ref_img_index,
                       const double *px_ref, const int32_t *ref_level, const double *ref_f, const double *ref_pos, const double *pos_w,
                       const double *normal_w, const double *T_ref_w, const double *ref_inv_expo, const int32_t *ref_key, const double *pc,
                       const double *T_cur_w, double inv_expo_time, int normal_en, int ncc_en, double ncc_thre, double outlier_threshold,
                       const double *A_in, const int32_t *sl_in, double *A_out, int32_t *sl_out, float *warp_out, float *error_out, int32_t *keep_out,
                       int32_t *kept_index) {
  VIOManager *v = (VIOManager *)h;
  const int L = v->patch_pyrimid_level, pst = v->patch_size_total;
  Image im;
  im.data = img, im.cols = v->width, im.rows = v->height;
  std::unordered_map<int, std::pair<M2, int>> warp_map;  // cleared per frame (:369)
  std::vector<float> patch_buffer(pst * L);
  int n_kept = 0;
  for (int i = 0; i < n; i++) {
    std::vector<float> patch_wrap(pst * L);  // :646
    M2 A;
    int search_level;
    const double *Tr = T_ref_w + 12 * (size_t)i;
    if (A_in) {
      for (int k = 0; k < 4; k++) A.a[k] = A_in[4 * (size_t)i + k];
      search_level = sl_in[i];
    } else if (normal_en) {  // :699-715
      const SE3 Tref = se3(Tr);
      V3 norm_vec = Tref.R * v3p(normal_w + 3 * (size_t)i);
      norm_vec = norm_vec / norm(norm_vec);
      const V3 pf = Tref * v3p(pos_w + 3 * (size_t)i);
      const SE3 T_cur_ref = se3(T_cur_w) * Tref.inverse();
      v->getWarpMatrixAffineHomography(v->cam, v2(px_ref + 2 * (size_t)i), pf, norm_vec, T_cur_ref, 0, A);
      search_level = v->getBestSearchLevel(A, 2);
    } else {  // :716-734
      auto it = warp_map.find(ref_key[i]);
      if (it != warp_map.end()) {
        A = it->second.first;
        search_level = it->second.second;
      } else {
        search_level = depth_warp(v, px_ref + 2 * (size_t)i, ref_f + 3 * (size_t)i, ref_pos + 3 * (size_t)i, pos_w + 3 * (size_t)i, Tr, T_cur_w, ref_level[i], A);
        warp_map[ref_key[i]] = std::make_pair(A, search_level);
      }
    }
    Image ref;
    ref.data = ref_imgs[ref_img_index[i]], ref.cols = ref_cols, ref.rows = ref_rows;
    const int level_ref = ref_level ? ref_level[i] : 0;
    for (int pyramid_level = 0; pyramid_level <= L - 1; pyramid_level++)  // :739-742
      v->warpAffine(A, ref, v2(px_ref + 2 * (size_t)i), level_ref, search_level, pyramid_level, v->patch_size_half, patch_wrap.data());
    v->getImagePatch(im, v2(pc + 2 * (size_t)i), patch_buffer.data(), 0);  // :744
    const double ref_ie = ref_inv_expo[i];
    float error = 0.0;
    for (int ind = 0; ind < pst; ind++)  // :746-751
      error += (ref_ie * patch_wrap[ind] - inv_expo_time * patch_buffer[ind]) * (ref_ie * patch_wrap[ind] - inv_expo_time * patch_buffer[ind]);
    bool keep = true;
    if (ncc_en && calculateNCC(patch_wrap.data(), patch_buffer.data(), pst) < ncc_thre) keep = false;  // :753-761
    if (error > outlier_threshold * pst) keep = false;                                                   // :763
    for (int k = 0; k < 4; k++) A_out[4 * (size_t)i + k] = A.a[k];
    sl_out[i] = search_level;
    memcpy(warp_out + (size_t)i * pst * L, patch_wrap.data(), sizeof(float) * pst * L);
    error_out[i] = error;
    keep_out[i] = keep;
    if (keep) kept_index[n_kept++] = i;  // :765-770
  }
  return n_kept;
}

}  // extern "C"
