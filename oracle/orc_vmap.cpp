// ORACLE — TEST INFRASTRUCTURE ONLY. Restates the list edits of VIOManager::updateVisualMapPoints (src/vio.cpp:914-964) and
// the reference-feature choice of retrieveFromVisualSparseMap (:651-697) on a host copy of the visual map's observation store
// (esikf_vmap_*): per point a count, the position of ref_patch (-1: none) and 30 observation slots in obs_ order, the newest
// first. The edits run on a list of slot indices with the operations the reference applies to obs_ (deleteNonRefPatchFeatures,
// findMinScoreFeature + deleteFeatureRef, addFrameRef), then the list is written back. The flags, pixels and patches of the new
// observations come from orc_update_points (orc_observe.cpp), the scores from orc_score_ref_patches (orc_refpatch.cpp).
// Checks esikf_vmap_* (tests/test_gpu_vmap.py). Built by oracle/vmap.mk with -ffp-contract=off.
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <list>
#include <vector>

namespace {
const int SLOTS = 30;

struct Store {
  int32_t *count, *ref;
  double *T, *px;
  float *patch, *mean, *score;
  int32_t *id;
};

struct Obs {
  double T[12], px[2];
  float patch[64], mean, score;
  int32_t id;
};

Obs get(const Store &s, size_t o) {
  Obs f;
  for (int k = 0; k < 12; k++) f.T[k] = s.T[12 * o + k];
  for (int k = 0; k < 2; k++) f.px[k] = s.px[2 * o + k];
  for (int k = 0; k < 64; k++) f.patch[k] = s.patch[64 * o + k];
  f.mean = s.mean[o], f.score = s.score[o], f.id = s.id[o];
  return f;
}
void put(const Store &s, size_t o, const Obs &f) {
  for (int k = 0; k < 12; k++) s.T[12 * o + k] = f.T[k];
  for (int k = 0; k < 2; k++) s.px[2 * o + k] = f.px[k];
  for (int k = 0; k < 64; k++) s.patch[64 * o + k] = f.patch[k];
  s.mean[o] = f.mean, s.score[o] = f.score, s.id[o] = f.id;
}
}  // namespace

extern "C" {

// The edits of n update entries (entry i = point pid[i]) after the flags: converged[i], flag[i] (update_flag), and for a flagged
// entry its new observation's pc (new_pc[i], 2) and patch (new_patch[i], 64), with T_new (12) and frame_id. Store arrays as
// esikf_vmap_download's per slot: count, ref [P]; T [P][30][12], px [P][30][2], patch [P][30][64], mean, score, id [P][30].
// Outputs evicted [n] (list position removed, -1) and count_out [n]. Slots past a point's count are left as they are.
void orc_vmap_edit(int n, const int32_t *pid, const uint8_t *converged, const uint8_t *flag, const double *new_pc, const float *new_patch,
                   const double *T_new, int32_t frame_id, int32_t *count, int32_t *ref, double *T, double *px, float *patch, float *mean, float *score,
                   int32_t *id, int32_t *evicted, int32_t *count_out) {
  const Store s{count, ref, T, px, patch, mean, score, id};
  for (int i = 0; i < n; i++) {
    const int p = pid[i];
    const size_t o = (size_t)p * SLOTS;
    std::list<Obs> obs;
    for (int j = 0; j < count[p]; j++) obs.push_back(get(s, o + j));
    auto ref_it = ref[p] >= 0 ? std::next(obs.begin(), ref[p]) : obs.end();  // obs.end(): ref_patch is nullptr
    evicted[i] = -1;
    if (converged[i]) {  // deleteNonRefPatchFeatures
      for (auto it = obs.begin(); it != obs.end();) it = it != ref_it ? obs.erase(it) : std::next(it);
    } else {
      if (obs.size() >= 30) {  // findMinScoreFeature, deleteFeatureRef
        auto min_it = obs.begin();
        float min_score = FLT_MAX;
        for (auto it = obs.begin(); it != obs.end(); ++it)
          if (it->score < min_score) min_score = it->score, min_it = it;
        evicted[i] = (int)std::distance(obs.begin(), min_it);
        if (ref_it == min_it) ref_it = obs.end();
        obs.erase(min_it);
      }
      if (flag[i]) {  // addFrameRef of the new Feature
        Obs f;
        for (int k = 0; k < 12; k++) f.T[k] = T_new[k];
        for (int k = 0; k < 2; k++) f.px[k] = new_pc[2 * i + k];
        for (int k = 0; k < 64; k++) f.patch[k] = new_patch[64 * i + k];
        f.mean = 0.0f, f.score = 0.0f, f.id = frame_id;
        obs.push_front(f);
      }
    }
    int j = 0, r = -1;
    for (auto it = obs.begin(); it != obs.end(); ++it, ++j) {
      if (it == ref_it) r = j;
      put(s, o + j, *it);
    }
    count[p] = count_out[i] = (int32_t)obs.size(), ref[p] = r;
  }
}

// The reference feature of n retrieved points (entry i = point pid[i]), as esikf_vmap_choose_ref: normal_en, or getCloseViewObs
// from frame_pos with pos [n][3]. Stores the choice of the first two normal_en cases in ref. Output ref_out [n].
void orc_vmap_choose_ref(int n, const int32_t *pid, const double *pos, const double *frame_pos, int normal_en, const int32_t *count, int32_t *ref,
                         const double *T, const float *patch, const int32_t *id, int32_t *ref_out) {
  for (int i = 0; i < n; i++) {
    const int p = pid[i], c = count[p];
    const size_t o = (size_t)p * SLOTS;
    int out = -1;
    if (normal_en) {
      if (c == 1) {
        out = ref[p] = 0;
      } else if (ref[p] < 0) {
        float errors_min = FLT_MAX;
        for (int r = 0; r < c; r++) {
          const float *a = patch + 64 * (o + r);
          float errors = 0.0;
          int cnt = 0;
          for (int j = 0; j < c; j++) {
            if (id[o + j] == id[o + r]) continue;
            const float *b = patch + 64 * (o + j);
            for (int k = 0; k < 64; k++) errors += (a[k] - b[k]) * (a[k] - b[k]);
            cnt++;
          }
          errors = errors / cnt;
          if (errors < errors_min) errors_min = errors, out = r;
        }
        ref[p] = out;  // -1 where the reference leaves ref_ftr unset
      } else {
        out = ref[p];
      }
    } else if (c > 0) {
      const double *pw = pos + 3 * i;
      double od[3] = {frame_pos[0] - pw[0], frame_pos[1] - pw[1], frame_pos[2] - pw[2]};
      const double on = std::sqrt(0.0 + od[0] * od[0] + od[1] * od[1] + od[2] * od[2]);
      for (int k = 0; k < 3; k++) od[k] /= on;
      double min_cos_angle = 0;
      int min_it = 0;
      for (int r = 0; r < c; r++) {
        const double *Tr = T + 12 * (o + r);
        double d[3];
        for (int k = 0; k < 3; k++) d[k] = (0.0 + Tr[k] * Tr[9] + Tr[3 + k] * Tr[10] + Tr[6 + k] * Tr[11]) * -1.0 - pw[k];
        const double dn = std::sqrt(0.0 + d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        for (int k = 0; k < 3; k++) d[k] /= dn;
        const double cos_angle = 0.0 + od[0] * d[0] + od[1] * d[1] + od[2] * d[2];
        if (cos_angle > min_cos_angle) min_cos_angle = cos_angle, min_it = r;
      }
      out = min_cos_angle < 0.5 ? -1 : min_it;
    }
    ref_out[i] = out;
  }
}

}  // extern "C"
