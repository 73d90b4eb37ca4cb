// ORACLE — TEST INFRASTRUCTURE ONLY. Restates the patch scoring of VIOManager::updateReferencePatch (src/vio.cpp:1036-1097)
// for visual points whose normal_ the plane half (:981-1034) has already left: per observation in obs_ order the cosine
// between its viewing ray and the normal, the cached or recomputed mean_, the NCC against every observation of another frame
// id (the three float sums running across the whole list, as the reference declares them once per reference observation),
// score_, and the first strict maximum above -1000. ref_mean / other_mean, which the reference leaves uninitialised when mean_
// is cached, are the observation's mean (DESIGN.md §4). The pinned reference build resolves abs, fabs and sqrt to their float
// overloads (using namespace std); so does this file. Checks esikf_vio_score_ref_patches (tests/test_gpu_refpatch.py); pinned
// to the reference source's own updateReferencePatch (oracle/ref_refpatch.cpp, tests/test_oracle_refpatch.py). Built by
// oracle/refpatch.mk with -ffp-contract=off.
#include <cmath>
#include <cstdint>
#include <vector>

#include "orc_math.hpp"

using namespace orc;

namespace {
// Feature::mean_ as the scoring reads it (:1055-1060): the cached value, else std::accumulate(patch, patch + 64, 0.0) narrowed
// to float and divided by patch_size_total (int) in float
float mean_of(const float *p, float cached) {
  if (std::abs(cached) < 1e-6) {
    double s = 0.0;
    for (int k = 0; k < 64; k++) s = s + p[k];
    const float sum = (float)s;
    return sum / 64;
  }
  return cached;
}
}  // namespace

extern "C" {

// n points, point i owning observations first[i] .. first[i + 1] - 1 in obs_ order; pos, normal [n][3]; per observation patch
// [m][64], mean [m], id [m], T_f_w [m][12] (R row-major, then t). Outputs score [m], mean_out [m], ref [n] (-1: none chosen).
void orc_score_ref_patches(int n, const int32_t *first, const double *pos, const double *normal, const float *patch, const float *mean, const int32_t *id,
                           const double *T_f_w, float *score_out, float *mean_out, int32_t *ref_out) {
  for (int i = 0; i < n; i++) {
    const int b = first[i], cnt = first[i + 1] - b;
    const V3 pw = v3(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]), nw = v3(normal[3 * i], normal[3 * i + 1], normal[3 * i + 2]);
    std::vector<float> mu(cnt);
    for (int j = 0; j < cnt; j++) mu[j] = mean_out[b + j] = mean_of(patch + 64 * (size_t)(b + j), mean[b + j]);
    float score_max = -1000.0f;
    int ref = -1;
    for (int r = 0; r < cnt; r++) {
      const double *T = T_f_w + 12 * (size_t)(b + r);
      M3 R;
      for (int k = 0; k < 9; k++) R.a[k] = T[k];
      V3 pf = R * pw + v3(T[9], T[10], T[11]);  // T_f_w_ * pos_
      const V3 norm_vec = R * nw;
      pf = pf / norm(pf);
      const double cos_angle = dot(pf, norm_vec);
      const float *a = patch + 64 * (size_t)(b + r);
      const float ref_mean = mu[r];
      float NCC_up = 0.0f, NCC_down1 = 0.0f, NCC_down2 = 0.0f, NCC = 0.0f;
      int count = 0;
      for (int j = 0; j < cnt; j++) {
        if (id[b + j] == id[b + r]) continue;
        const float *c = patch + 64 * (size_t)(b + j);
        const float other_mean = mu[j];
        for (int k = 0; k < 64; k++) {
          NCC_up += (a[k] - ref_mean) * (c[k] - other_mean);
          NCC_down1 += (a[k] - ref_mean) * (a[k] - ref_mean);
          NCC_down2 += (c[k] - other_mean) * (c[k] - other_mean);
        }
        NCC += std::fabs(NCC_up / std::sqrt(NCC_down1 * NCC_down2));
        count++;
      }
      NCC = NCC / count;
      const float score = NCC + cos_angle;
      score_out[b + r] = score;
      if (score > score_max) score_max = score, ref = r;
    }
    ref_out[i] = ref;
  }
}

}  // extern "C"
