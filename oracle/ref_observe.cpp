// oracle/_ref — VIOManager::updateVisualMapPoints (src/vio.cpp:908-967) run as it is, on the VIOManager the driver ref_vio.cpp
// (included as it is) creates: new_frame_ is a Frame of the image with updateFrameState(state), the visual sub-map holds one
// VisualPoint per entry with n_obs observations whose oldest (obs_.back()) has the given T_f_w_ and px_ (the others, and their
// scores for the eviction at 30, are filler), update_flag is reset as resetGrid leaves it, and the update_flag and each new
// obs_.front() (px_, patch_, level_) are read back. What is not the reference's code: vikit (the camera models of the
// stand-ins in ref_shim/vikit/, restatements of the published algorithm). TEST INFRASTRUCTURE ONLY: pins the oracle's
// restatement (oracle/orc_observe.cpp) in tests/test_oracle_observe.py. Built by oracle/observe.mk where the reference source
// exists.
#include <algorithm>

#include "ref_vio.cpp"

extern "C" {

// Inputs as orc_update_points, plus n_obs (observations of each entry, >= 1), has_ref (the entry's ref_patch is its newest
// filler observation) and search_levels. Outputs: update_flag (n bytes), and for the added entries in entry order: entry, pc
// (2, the new Feature's px_), patch (64, its patch_), level (its level_), and obs_left (n: obs_.size() after the call). Returns
// the number of added entries.
int ref_update_points(void *h, const uint8_t *img, const double *state, const double *pos, const uint8_t *converged, const double *last_T,
                      const double *last_px, const int32_t *n_obs, const uint8_t *has_ref, const int32_t *search_levels, int n, uint8_t *update_flag,
                      int32_t *entry, double *pc, float *patch, int32_t *level, int32_t *obs_left) {
  RefVio *r = (RefVio *)h;
  VIOManager &v = r->v;
  unpack_state(state, r->st);
  cv::Mat im = cv::Mat(v.height, v.width, CV_8UC1, (void *)img).clone();
  v.new_frame_.reset(new Frame(v.cam, im));
  v.updateFrameState(r->st);
  SubSparseMap &sub = *v.visual_submap;
  sub.reset();
  for (auto *p : r->owned) delete p;
  r->owned.clear();
  for (int i = 0; i < n; i++) {
    VisualPoint *pt = new VisualPoint(V3D(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]));
    r->owned.push_back(pt);
    pt->is_converged_ = converged[i] != 0;
    pt->ref_patch = nullptr;
    for (int k = 0; k + 1 < n_obs[i]; k++) {  // newer observations first (addFrameRef pushes at the front)
      Feature *f = new Feature(pt, new float[64](), V2D(10.0 + k, 20.0), V3D(0, 0, 1), SE3(), 0);
      f->score_ = (float)((i * 7 + k * 13) % 17);
      pt->obs_.push_back(f);
      if (has_ref[i] && k == 0) pt->ref_patch = f, pt->has_ref_patch_ = true;
    }
    const double *T = last_T + 12 * (size_t)i;
    M3D R;
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) R(a, b) = T[3 * a + b];
    Feature *last = new Feature(pt, new float[64](), V2D(last_px[2 * i], last_px[2 * i + 1]), V3D(0, 0, 1), SE3(R, V3D(T[9], T[10], T[11])), 0);
    last->score_ = (float)(i % 5);
    pt->obs_.push_back(last);
    sub.voxel_points.push_back(pt);
    sub.search_levels.push_back(search_levels[i]);
  }
  v.total_points = n;
  v.update_flag.assign(std::max(v.length, n), 0);  // resetGrid (:167); a retrieved sub-map has at most one entry per cell
  v.updateVisualMapPoints(im);
  int add = 0;
  for (int i = 0; i < n; i++) {
    const VisualPoint *pt = sub.voxel_points[i];
    update_flag[i] = (uint8_t)v.update_flag[i];
    obs_left[i] = (int32_t)pt->obs_.size();
    if (!v.update_flag[i]) continue;
    const Feature *f = pt->obs_.front();
    entry[add] = i, level[add] = f->level_;
    pc[2 * add] = f->px_[0], pc[2 * add + 1] = f->px_[1];
    for (int k = 0; k < 64; k++) patch[64 * add + k] = f->patch_[k];
    add++;
  }
  return add;
}
}
