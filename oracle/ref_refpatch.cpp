// oracle/_ref — the patch scoring of VIOManager::updateReferencePatch (src/vio.cpp:1036-1097) run as it is, on the VIOManager
// the driver ref_vio.cpp (included as it is) creates. The plane map handed to it is empty, so the plane half (:981-1034)
// finds no root and leaves every normal_ as set here, and only the scoring runs.
// What is set up around the reference's code (not the reference's code): one stand-in VisualPoint per point that passes the
// four skips of :977-980 (is_normal_initialized_, not converged, the caller's observations, update_flag 1), with pos_ and
// normal_ given, ref_patch = nullptr and has_ref_patch_ = false; its obs_ holds the caller's Features in list order, each with
// patch_, mean_, id_ and T_f_w_ given. Read back: every Feature's score_ and mean_, the position of ref_patch within obs_ (-1
// when it stays nullptr) and has_ref_patch_. The reference skips a point with five observations or fewer: its outputs stay
// as set up (score_ 0, mean_ unchanged, ref -1). TEST INFRASTRUCTURE ONLY: pins the oracle's restatement
// (oracle/orc_refpatch.cpp) in tests/test_oracle_refpatch.py. Built by oracle/refpatch.mk where the reference source exists.
#include <chrono>

#include "ref_vio.cpp"

extern "C" {

// Inputs as orc_score_ref_patches, on a handle of ref_vio_create. Outputs score_out, mean_out [m], ref_out [n], has_ref_out
// [n] bytes. Returns the seconds updateReferencePatch took (the call alone, not the set-up).
double ref_score_ref_patches(void *h, int n, const int32_t *first, const double *pos, const double *normal, const float *patch, const float *mean,
                             const int32_t *id, const double *T_f_w, float *score_out, float *mean_out, int32_t *ref_out, uint8_t *has_ref_out) {
  RefVio *r = (RefVio *)h;
  VIOManager &v = r->v;
  SubSparseMap &sub = *v.visual_submap;
  sub.reset();
  std::vector<VisualPoint *> pts;
  std::vector<std::vector<Feature *>> obs(n);
  for (int i = 0; i < n; i++) {
    VisualPoint *pt = new VisualPoint(V3D(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]));
    pt->normal_ = pt->previous_normal_ = V3D(normal[3 * i], normal[3 * i + 1], normal[3 * i + 2]);
    pt->is_normal_initialized_ = true, pt->is_converged_ = false;
    pt->ref_patch = nullptr, pt->has_ref_patch_ = false;
    for (int j = first[i]; j < first[i + 1]; j++) {
      const double *T = T_f_w + 12 * (size_t)j;
      M3D R;
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) R(a, b) = T[3 * a + b];
      float *p = new float[64];
      for (int k = 0; k < 64; k++) p[k] = patch[64 * (size_t)j + k];
      Feature *f = new Feature(pt, p, V2D(0, 0), V3D(0, 0, 1), SE3(R, V3D(T[9], T[10], T[11])), 0);
      f->mean_ = mean[j], f->id_ = id[j];
      pt->obs_.push_back(f);  // obs_ in the caller's order
      obs[i].push_back(f);
    }
    pts.push_back(pt);
    sub.voxel_points.push_back(pt);
  }
  v.total_points = n;
  v.update_flag.assign(n, 1);
  const std::unordered_map<VOXEL_LOCATION, VoxelOctoTree *> no_planes;
  const auto t0 = std::chrono::steady_clock::now();
  v.updateReferencePatch(no_planes);
  const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  for (int i = 0; i < n; i++) {
    ref_out[i] = -1;
    for (int j = 0; j < (int)obs[i].size(); j++) {
      score_out[first[i] + j] = obs[i][j]->score_, mean_out[first[i] + j] = obs[i][j]->mean_;
      if (pts[i]->ref_patch == obs[i][j]) ref_out[i] = j;
    }
    has_ref_out[i] = pts[i]->has_ref_patch_ ? 1 : 0;
  }
  sub.reset();
  for (auto *p : pts) delete p;  // ~VisualPoint deletes its observations and their patches
  v.total_points = 0;
  return sec;
}
}
