// oracle/_ref — the visual map's observations kept in the reference's own VisualPoint / Feature objects across calls, and
// changed only by the reference's own code: VIOManager::updateVisualMapPoints (src/vio.cpp:908-967, with deleteNonRefPatchFeatures,
// findMinScoreFeature, deleteFeatureRef and addFrameRef of src/visual_point.cpp), VisualPoint::getCloseViewObs, with the write-back of
// updateReferencePatch's scores (ref_vmap_set_scores), on the VIOManager the driver ref_vio.cpp
// (included as it is) creates. What is set up around the reference's code (not the reference's code): the points and their
// Features as the caller lists them (ref_vmap_add), the sub-map, update_flag, is_converged_, normal_ and
// is_normal_initialized_ of each call, new_frame_ (a Frame of the image with updateFrameState(state), its id_ set to the
// caller's frame id). Every list is read back in obs_ order. TEST INFRASTRUCTURE ONLY: pins the oracle's restatement
// (oracle/orc_vmap.cpp, tests/vmap_cases.py) in tests/test_oracle_vmap.py. Built by oracle/vmap.mk where the reference source
// exists.
#include "ref_vio.cpp"

namespace {
int position(const VisualPoint *pt, const Feature *f) {
  int j = 0;
  for (const Feature *g : pt->obs_) {
    if (g == f) return j;
    j++;
  }
  return -1;
}
}  // namespace

extern "C" {

// Appends n points (pos n x 3) with the observations first[i] .. first[i + 1] - 1 in obs_ order (px 2, patch 64, T_f_w 12: R
// row-major then t, id, mean, score) and ref (the position of ref_patch, -1: nullptr). The point ids continue from the last
// call, from 0 on a new handle of ref_vio_create.
void ref_vmap_add(void *h, int n, const double *pos, const int32_t *first, const double *px, const float *patch, const double *T_f_w, const int32_t *id,
                  const float *mean, const float *score, const int32_t *ref) {
  RefVio *r = (RefVio *)h;
  for (int i = 0; i < n; i++) {
    VisualPoint *pt = new VisualPoint(V3D(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]));
    pt->ref_patch = nullptr, pt->has_ref_patch_ = false;
    for (int j = first[i]; j < first[i + 1]; j++) {
      const double *T = T_f_w + 12 * (size_t)j;
      M3D R;
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) R(a, b) = T[3 * a + b];
      float *p = new float[64];
      for (int k = 0; k < 64; k++) p[k] = patch[64 * (size_t)j + k];
      Feature *f = new Feature(pt, p, V2D(px[2 * j], px[2 * j + 1]), V3D(0, 0, 1), SE3(R, V3D(T[9], T[10], T[11])), 0);
      f->id_ = id[j], f->mean_ = mean[j], f->score_ = score[j];
      pt->obs_.push_back(f);
      if (j - first[i] == ref[i]) pt->ref_patch = f, pt->has_ref_patch_ = true;
    }
    r->owned.push_back(pt);
  }
}

// updateVisualMapPoints on the sub-map of the points pid (n), with is_converged_ = converged, the image and the frame pose of
// state; new_frame_->id_ = frame_id. Outputs update_flag (n bytes) and the frame's T_f_w_ (12), which the new Features carry.
void ref_vmap_update(void *h, const uint8_t *img, const double *state, int frame_id, int n, const int32_t *pid, const uint8_t *converged,
                     uint8_t *update_flag, double *T_frame) {
  RefVio *r = (RefVio *)h;
  VIOManager &v = r->v;
  unpack_state(state, r->st);
  cv::Mat im = cv::Mat(v.height, v.width, CV_8UC1, (void *)img).clone();
  v.new_frame_.reset(new Frame(v.cam, im));
  v.updateFrameState(r->st);
  v.new_frame_->id_ = frame_id;
  SubSparseMap &sub = *v.visual_submap;
  sub.reset();
  for (int i = 0; i < n; i++) {
    VisualPoint *pt = r->owned[pid[i]];
    pt->is_converged_ = converged[i] != 0;
    sub.voxel_points.push_back(pt);
    sub.search_levels.push_back(0);
  }
  v.total_points = n;
  v.update_flag.assign(std::max(v.length, n), 0);  // resetGrid (:167)
  v.updateVisualMapPoints(im);
  for (int i = 0; i < n; i++) update_flag[i] = (uint8_t)v.update_flag[i];
  const M3D R = v.new_frame_->T_f_w_.rotation_matrix();
  const V3D t = v.new_frame_->T_f_w_.translation();
  for (int a = 0; a < 3; a++) {
    T_frame[9 + a] = t[a];
    for (int b = 0; b < 3; b++) T_frame[3 * a + b] = R(a, b);
  }
  sub.reset();
  v.total_points = 0;
}

// The write-back of updateReferencePatch's scoring (:1083-1096) on the points pid (n): each observation's score_ and mean_
// from the packed arrays (first, n + 1 offsets, in obs_ order) and, where ref[i] >= 0, ref_patch = that observation and
// has_ref_patch_ = true. The scores themselves come from the restatement of the scoring, which is pinned where the reference is
// defined (oracle/ref_refpatch.cpp): on real patches the reference reads an uninitialised ref_mean / other_mean once a mean
// is cached (DESIGN.md §4), so its own scores are not a fixed value to pin a sequence to.
void ref_vmap_set_scores(void *h, int n, const int32_t *pid, const int32_t *first, const float *score, const float *mean, const int32_t *ref) {
  RefVio *r = (RefVio *)h;
  for (int i = 0; i < n; i++) {
    VisualPoint *pt = r->owned[pid[i]];
    int j = first[i];
    for (Feature *f : pt->obs_) {
      f->score_ = score[j], f->mean_ = mean[j];
      if (j - first[i] == ref[i]) pt->ref_patch = f, pt->has_ref_patch_ = true;
      j++;
    }
  }
}

// getCloseViewObs(frame_pos) of the points pid (n): the position of the Feature it returns in obs_, or -1 when it returns false.
void ref_vmap_close_view(void *h, int n, const int32_t *pid, const double *frame_pos, int32_t *out) {
  RefVio *r = (RefVio *)h;
  for (int i = 0; i < n; i++) {
    const VisualPoint *pt = r->owned[pid[i]];
    Feature *f = nullptr;
    out[i] = pt->getCloseViewObs(V3D(frame_pos[0], frame_pos[1], frame_pos[2]), f, V2D(0, 0)) ? position(pt, f) : -1;
  }
}

// The lists of every point, as esikf_vmap_download: first (points + 1), then per observation px, patch, T_f_w, id, mean,
// score, and per point ref (position of ref_patch, -1: nullptr) and has_ref (has_ref_patch_). Returns the number of points;
// with first == NULL only that.
int ref_vmap_download(void *h, int32_t *first, double *px, float *patch, double *T_f_w, int32_t *id, float *mean, float *score, int32_t *ref,
                      uint8_t *has_ref) {
  RefVio *r = (RefVio *)h;
  const int n = (int)r->owned.size();
  if (!first) return n;
  int m = 0;
  first[0] = 0;
  for (int i = 0; i < n; i++) {
    const VisualPoint *pt = r->owned[i];
    for (const Feature *f : pt->obs_) {
      px[2 * m] = f->px_[0], px[2 * m + 1] = f->px_[1];
      for (int k = 0; k < 64; k++) patch[64 * (size_t)m + k] = f->patch_[k];
      const M3D R = f->T_f_w_.rotation_matrix();
      const V3D t = f->T_f_w_.translation();
      for (int a = 0; a < 3; a++) {
        T_f_w[12 * (size_t)m + 9 + a] = t[a];
        for (int b = 0; b < 3; b++) T_f_w[12 * (size_t)m + 3 * a + b] = R(a, b);
      }
      id[m] = f->id_, mean[m] = f->mean_, score[m] = f->score_;
      m++;
    }
    first[i + 1] = m;
    ref[i] = pt->ref_patch ? position(pt, pt->ref_patch) : -1;
    has_ref[i] = pt->has_ref_patch_ ? 1 : 0;
  }
  return n;
}
}
