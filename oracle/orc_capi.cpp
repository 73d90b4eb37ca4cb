// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header). PARITY UNPINNED.
// Plain C entry points over the restatement so tests/ (ctypes) and bench.py's cpu_baseline
// leg can drive it. Nothing in fast_livo2_b200/ may load this library.
#include <chrono>
#include <cstdio>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "orc_lio.hpp"
#include "orc_vio.hpp"

using namespace orc;

extern "C" {

// ---------------------------------------------------------------- state algebra / math
void orc_boxplus(const double *state, const double *delta19, double *out) {
  StatesGroup x;
  unpack_state(state, x);
  V19 d;
  for (int i = 0; i < 19; i++) d[i] = delta19[i];
  x.boxplus(d);
  pack_state(x, out);
}
void orc_boxminus(const double *a, const double *b, double *out19) {
  StatesGroup xa, xb;
  unpack_state(a, xa);
  unpack_state(b, xb);
  V19 d = xa.boxminus(xb);
  for (int i = 0; i < 19; i++) out19[i] = d[i];
}
void orc_exp(const double *v, double *R9) {
  M3 R = Exp(v[0], v[1], v[2]);
  for (int i = 0; i < 9; i++) R9[i] = R.a[i];
}
void orc_log(const double *R9, double *v) {
  M3 R;
  for (int i = 0; i < 9; i++) R.a[i] = R9[i];
  V3 l = Log(R);
  for (int i = 0; i < 3; i++) v[i] = l[i];
}
void orc_inverse19(const double *A, double *Ainv) {
  M19 m;
  for (int i = 0; i < 361; i++) m.a[i] = A[i];
  M19 inv = inverse_pplu(m);
  for (int i = 0; i < 361; i++) Ainv[i] = inv.a[i];
}
void orc_calc_body_cov(const double *p, float range_inc, float degree_inc, double *cov9, double *p_out) {
  V3 pb = v3(p[0], p[1], p[2]);
  M3 cov;
  calcBodyCov(pb, range_inc, degree_inc, cov);
  for (int i = 0; i < 9; i++) cov9[i] = cov.a[i];
  if (p_out)
    for (int i = 0; i < 3; i++) p_out[i] = pb[i];
}
void orc_default_state(double *out) {
  StatesGroup x;
  pack_state(x, out);
}

// ---------------------------------------------------------------- LIO
// cfg = [voxel_size, max_layer, max_iterations, sigma_num, dept_err, beam_err, min_eigen_value, max_points_num]
static void apply_cfg(VoxelMapManager *m, const double *cfg) {
  m->config_setting_.max_voxel_size_ = cfg[0];
  m->config_setting_.max_layer_ = (int)cfg[1];
  m->config_setting_.max_iterations_ = (int)cfg[2];
  m->config_setting_.sigma_num_ = cfg[3];
  m->config_setting_.dept_err_ = cfg[4];
  m->config_setting_.beam_err_ = cfg[5];
  m->config_setting_.planner_threshold_ = cfg[6];
  m->config_setting_.max_points_num_ = (int)cfg[7];
}

void *orc_lio_create(const double *cfg, const double *extR, const double *extT, int omp_threads) {
  VoxelMapManager *m = new VoxelMapManager;
  apply_cfg(m, cfg);
  for (int i = 0; i < 9; i++) m->extR_.a[i] = extR[i];
  for (int i = 0; i < 3; i++) m->extT_[i] = extT[i];
  m->omp_threads_ = omp_threads;
  return m;
}
void orc_lio_destroy(void *h) { delete (VoxelMapManager *)h; }

void orc_lio_set_map_flat(void *h, const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots, const void *planes,
                          int n_planes) {
  ((VoxelMapManager *)h)->FromFlat(keys, first, count, n_roots, (const FlatPlane *)planes, n_planes);
}

// Oracle bookkeeping: a match needs the chosen plane's flat id (orc_lio.cpp: "require a chosen plane"), which Flatten assigns. Maps
// that grow natively (BuildVoxelMap / UpdateVoxelMap) get their ids refreshed after every change.
static void refresh_flat_ids(VoxelMapManager *m) {
  std::vector<int64_t> k;
  std::vector<int32_t> f, c;
  std::vector<FlatPlane> p;
  m->Flatten(k, f, c, p);
}

// BuildVoxelMap (src/voxel_map.cpp:532-591) from world/body points at `state`.
void orc_lio_build_map(void *h, const float *pts_world, const float *pts_body, int n, const double *state) {
  VoxelMapManager *m = (VoxelMapManager *)h;
  m->feats_down_world_.assign(pts_world, pts_world + 3 * (size_t)n);
  m->feats_down_body_.assign(pts_body, pts_body + 3 * (size_t)n);
  unpack_state(state, m->state_);
  m->BuildVoxelMap();
  refresh_flat_ids(m);
}
// UpdateVoxelMap (src/voxel_map.cpp:609-641) with caller-supplied world points + 3x3 vars.
void orc_lio_update_map(void *h, const double *pts_world, const double *var9, int n) {
  VoxelMapManager *m = (VoxelMapManager *)h;
  std::vector<pointWithVar> pts(n);
  for (int i = 0; i < n; i++) {
    pts[i].point_w = v3(pts_world[3 * i], pts_world[3 * i + 1], pts_world[3 * i + 2]);
    for (int k = 0; k < 9; k++) pts[i].var.a[k] = var9[9 * (size_t)i + k];
  }
  m->UpdateVoxelMap(pts);
  refresh_flat_ids(m);
}
// First LiDAR frame (LIVMapper.cpp:356-366): feats_down_world_ = transformLidar(state, feats_down_body_), BuildVoxelMap().
void orc_lio_tick_build_map(void *h, const float *pts_body, int n, const double *state) {
  VoxelMapManager *m = (VoxelMapManager *)h;
  m->feats_down_body_.assign(pts_body, pts_body + 3 * (size_t)n);
  m->feats_down_size_ = n;
  unpack_state(state, m->state_);
  m->TransformLidar(m->state_.rot_end, m->state_.pos_end, m->feats_down_body_, m->feats_down_world_);  // same expression as LIVMapper::transformLidar (:645)
  m->BuildVoxelMap();
  refresh_flat_ids(m);
}
// After StateEstimation (LIVMapper.cpp:413-424): world points with the posterior pose, var from body_cov_list_ / cross_mat_list_
// and the posterior covariance, then UpdateVoxelMap(pv_list_). Optionally returns the lists (n x 3, n x 9).
void orc_lio_tick_update_map(void *h, double *pts_world_out, double *var_out) {
  VoxelMapManager *m = (VoxelMapManager *)h;
  const StatesGroup &st = m->state_;
  std::vector<float> world;
  m->TransformLidar(st.rot_end, st.pos_end, m->feats_down_body_, world);
  const M3 RE = st.rot_end * m->extR_;
  M3 Prr, Ppp;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) Prr(r, c) = st.cov(r, c), Ppp(r, c) = st.cov(3 + r, 3 + c);
  for (size_t i = 0; i < m->pv_list_.size(); i++) {
    m->pv_list_[i].point_w = v3(world[3 * i], world[3 * i + 1], world[3 * i + 2]);
    const M3 point_crossmat = m->cross_mat_list_[i];
    M3 var = m->body_cov_list_[i];
    var = RE * var * T(RE) + (point_crossmat * -1.0) * Prr * T(point_crossmat * -1.0) + Ppp;
    m->pv_list_[i].var = var;
    if (pts_world_out)
      for (int k = 0; k < 3; k++) pts_world_out[3 * i + k] = m->pv_list_[i].point_w[k];
    if (var_out)
      for (int k = 0; k < 9; k++) var_out[9 * i + k] = var.a[k];
  }
  m->UpdateVoxelMap(m->pv_list_);
  refresh_flat_ids(m);
}
// clearMemOutOfMap (src/voxel_map.cpp:950-971): root voxels outside the box are deleted. Returns how many.
int orc_lio_clear_out_of_map(void *h, int x_max, int x_min, int y_max, int y_min, int z_max, int z_min) {
  VoxelMapManager *m = (VoxelMapManager *)h;
  int deleted = 0;
  for (auto it = m->voxel_map_.begin(); it != m->voxel_map_.end();) {
    const VOXEL_LOCATION &loc = it->first;
    const bool should_remove = loc.x > x_max || loc.x < x_min || loc.y > y_max || loc.y < y_min || loc.z > z_max || loc.z < z_min;
    if (should_remove) {
      delete it->second;
      it = m->voxel_map_.erase(it);
      deleted++;
    } else {
      ++it;
    }
  }
  refresh_flat_ids(m);  // StateEstimation on the pruned map reports flat ids of what is left
  return deleted;
}
// lio/layer_init_num (include/voxel_map.h:40): points a node of layer k collects before its first fit. n entries; a node of
// layer k reads entry k, so a map of max_layer L needs L + 1 of them.
void orc_lio_set_layer_init_num(void *h, const int32_t *lin, int n) {
  ((VoxelMapManager *)h)->config_setting_.layer_init_num_.assign(lin, lin + n);
}
// Every node of every root (DFS pre-order, leaves 0..7), 12 int64 a row: key x y z | layer path | init_octo octo_state
// update_enable is_plane | new_points temp_points_.size() points_size. Returns the number of nodes; rows beyond cap are not written.
static void dump_node(const VoxelOctoTree *nd, int64_t path, const VOXEL_LOCATION &key, int64_t *out, int cap, int *n) {
  if (*n < cap) {
    int64_t *r = out + (size_t)(*n) * 12;
    r[0] = key.x, r[1] = key.y, r[2] = key.z, r[3] = nd->layer_, r[4] = path;
    r[5] = nd->init_octo_, r[6] = nd->octo_state_, r[7] = nd->update_enable_, r[8] = nd->plane_ptr_->is_plane_;
    r[9] = nd->new_points_, r[10] = (int64_t)nd->temp_points_.size(), r[11] = nd->plane_ptr_->points_size_;
  }
  (*n)++;
  for (int l = 0; l < 8; l++)
    if (nd->leaves_[l]) dump_node(nd->leaves_[l], path | ((int64_t)l << (3 * nd->layer_)), key, out, cap, n);
}
int orc_lio_dump_nodes(void *h, int64_t *out, int cap) {
  VoxelMapManager *m = (VoxelMapManager *)h;
  int n = 0;
  for (auto &kv : m->voxel_map_) dump_node(kv.second, 0, kv.first, out, cap, &n);
  return n;
}
// Two-call flatten: sizes first (planes == NULL), then fill.
void orc_lio_flatten(void *h, int *n_roots, int *n_planes, int64_t *keys, int32_t *first, int32_t *count, void *planes) {
  VoxelMapManager *m = (VoxelMapManager *)h;
  std::vector<int64_t> k;
  std::vector<int32_t> f, c;
  std::vector<FlatPlane> p;
  m->Flatten(k, f, c, p);
  *n_roots = (int)f.size();
  *n_planes = (int)p.size();
  if (planes) {
    memcpy(keys, k.data(), k.size() * sizeof(int64_t));
    memcpy(first, f.data(), f.size() * sizeof(int32_t));
    memcpy(count, c.data(), c.size() * sizeof(int32_t));
    memcpy(planes, p.data(), p.size() * sizeof(FlatPlane));
  }
}

// StateEstimation (src/voxel_map.cpp:338-511). Returns wall seconds of the span the
// reference labels "ICP" (LIVMapper.cpp:368-374).
// stats_out (doubles): [0]=iters, then per iteration it<8: [1+it]=M, [9+it]=total_residual,
// [17+36*it..]=HTH, [305+6*it..]=HTz, [353+19*it..]=solution, [505+it]=converged
double orc_lio_state_estimation(void *h, const float *pts, int n, const double *state_in, const double *state_prop, double *state_out,
                                int32_t *match_plane, int32_t *normal_plane, float *dis_to_plane, double *stats_out,
                                double *H_rows /* n*6, rows of matched points of the last iteration, else 0 */,
                                double *R_inv /* n */) {
  VoxelMapManager *m = (VoxelMapManager *)h;
  m->feats_down_body_.assign(pts, pts + 3 * (size_t)n);
  m->feats_down_size_ = n;
  unpack_state(state_in, m->state_);
  StatesGroup prop;
  unpack_state(state_prop, prop);
  auto t0 = std::chrono::steady_clock::now();
  m->StateEstimation(prop);
  auto t1 = std::chrono::steady_clock::now();
  pack_state(m->state_, state_out);
  if (match_plane) {
    for (int i = 0; i < n; i++) match_plane[i] = -1;
    for (size_t k = 0; k < m->ptpl_list_.size(); k++) match_plane[m->ptpl_index_[k]] = m->ptpl_list_[k].plane_id_;
  }
  if (dis_to_plane) {
    for (int i = 0; i < n; i++) dis_to_plane[i] = 0.f;
    for (size_t k = 0; k < m->ptpl_list_.size(); k++) dis_to_plane[m->ptpl_index_[k]] = m->ptpl_list_[k].dis_to_plane_;
  }
  if (normal_plane)
    for (int i = 0; i < n; i++) normal_plane[i] = m->normal_plane_id_[i];
  if (stats_out) {
    const LioStats &s = m->stats_;
    for (int i = 0; i < 520; i++) stats_out[i] = 0;
    stats_out[0] = s.iters;
    for (int it = 0; it < 8; it++) {
      stats_out[1 + it] = s.effct_feat_num[it];
      stats_out[9 + it] = s.total_residual[it];
      for (int k = 0; k < 36; k++) stats_out[17 + 36 * it + k] = s.HTH[it][k];
      for (int k = 0; k < 6; k++) stats_out[305 + 6 * it + k] = s.HTz[it][k];
      for (int k = 0; k < 19; k++) stats_out[353 + 19 * it + k] = s.solution[it][k];
      stats_out[505 + it] = s.converged[it];
    }
  }
  (void)H_rows;
  (void)R_inv;
  return std::chrono::duration<double>(t1 - t0).count();
}

// The per-point residual pieces of ONE iteration at a given state, for finite-difference and
// invariant checks: signed distance and the Jacobian row [A, n] (src/voxel_map.cpp:453-457).
// Points whose association fails get plane -1.
void orc_lio_single_pass(void *h, const float *pts, int n, const double *state_cur, const double *state_prop, int32_t *plane_out,
                         float *dis_out, double *H_rows, double *R_inv_out, double *point_w_out, double *var_out) {
  VoxelMapManager *m = (VoxelMapManager *)h;
  StatesGroup cur, prop;
  unpack_state(state_cur, cur);
  unpack_state(state_prop, prop);
  m->feats_down_body_.assign(pts, pts + 3 * (size_t)n);
  m->feats_down_size_ = n;
  m->state_ = cur;
  std::vector<float> world;
  m->TransformLidar(cur.rot_end, cur.pos_end, m->feats_down_body_, world);
  std::vector<pointWithVar> pv(n);
  m->normal_plane_id_.assign(n, -1);
  M3 rot_var = block<3, 3>(cur.cov, 0, 0), t_var = block<3, 3>(cur.cov, 3, 3);
  for (int i = 0; i < n; i++) {
    V3 p = v3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
    pv[i].point_b = p;
    V3 pt = p;
    if (pt[2] == 0) pt[2] = 0.001;
    M3 bc;
    calcBodyCov(pt, m->config_setting_.dept_err_, m->config_setting_.beam_err_, bc);
    pt = m->extR_ * pt + m->extT_;
    M3 cm = skew(pt);
    pv[i].point_w = v3(world[3 * i], world[3 * i + 1], world[3 * i + 2]);
    pv[i].body_var = bc;
    pv[i].var = (cur.rot_end * bc) * T(cur.rot_end) + ((-cm) * rot_var) * (-T(cm)) + t_var;
    if (point_w_out)
      for (int k = 0; k < 3; k++) point_w_out[3 * i + k] = pv[i].point_w[k];
    if (var_out)
      for (int k = 0; k < 9; k++) var_out[9 * (size_t)i + k] = pv[i].var.a[k];
  }
  std::vector<PointToPlane> ptpl;
  m->BuildResidualListOMP(pv, ptpl);
  for (int i = 0; i < n; i++) {
    plane_out[i] = -1;
    if (dis_out) dis_out[i] = 0;
    if (R_inv_out) R_inv_out[i] = 0;
    if (H_rows)
      for (int k = 0; k < 6; k++) H_rows[6 * (size_t)i + k] = 0;
  }
  for (size_t k = 0; k < ptpl.size(); k++) {
    int i = m->ptpl_index_[k];
    const PointToPlane &q = ptpl[k];
    plane_out[i] = q.plane_id_;
    if (dis_out) dis_out[i] = q.dis_to_plane_;
    V3 point_this = m->extR_ * q.point_b_ + m->extT_;
    M3 cm = skew(point_this);
    V3 point_world = prop.rot_end * point_this + prop.pos_end;
    Mat<1, 6> J_nq;
    for (int c = 0; c < 3; c++) J_nq(0, c) = point_world[c] - q.center_[c], J_nq(0, 3 + c) = -q.normal_[c];
    M3 RE = prop.rot_end * m->extR_;
    M3 var = (RE * q.body_cov_) * T(RE);
    double sigma_l = ((J_nq * q.plane_var_) * T(J_nq))[0];
    double rinv = 1.0 / (0.001 + sigma_l + ((T(q.normal_) * var) * q.normal_)[0]);
    V3 A = (cm * T(cur.rot_end)) * q.normal_;
    if (R_inv_out) R_inv_out[i] = rinv;
    if (H_rows)
      for (int c = 0; c < 3; c++) H_rows[6 * (size_t)i + c] = A[c], H_rows[6 * (size_t)i + 3 + c] = q.normal_[c];
  }
}

// ---------------------------------------------------------------- VIO
// cam = [model, width, height, fx, fy, cx, cy, d0, d1, d2, d3, d4]
// cfg = [patch_pyrimid_level, max_iterations, img_point_cov, exposure_estimate_en]
void *orc_vio_create(const double *cam, const double *extR, const double *extT, const double *Rcl, const double *Pcl, const double *cfg,
                     int omp_threads) {
  VIOManager *v = new VIOManager;
  v->cam.model = (int)cam[0];
  v->cam.width = (int)cam[1];
  v->cam.height = (int)cam[2];
  v->cam.fx = cam[3], v->cam.fy = cam[4], v->cam.cx = cam[5], v->cam.cy = cam[6];
  for (int i = 0; i < 5; i++) v->cam.d[i] = cam[7 + i];
  M3 R, Rc;
  V3 t, Pc;
  for (int i = 0; i < 9; i++) R.a[i] = extR[i], Rc.a[i] = Rcl[i];
  for (int i = 0; i < 3; i++) t[i] = extT[i], Pc[i] = Pcl[i];
  v->setImuToLidarExtrinsic(t, R);      // LIVMapper.cpp:125-126 -> vio.cpp:29-33
  v->setLidarToCameraExtrinsic(Rc, Pc);  // vio.cpp:35-39
  v->patch_pyrimid_level = (int)cfg[0];
  v->max_iterations = (int)cfg[1];
  v->img_point_cov = cfg[2];
  v->exposure_estimate_en = cfg[3] != 0;
  v->omp_threads_ = omp_threads;
  v->initializeVIO();
  return v;
}
void orc_vio_destroy(void *h) { delete (VIOManager *)h; }

// stats_out (doubles): [0]=total_iters, [1+l]=iters at level l, [9+l]=accepted at level l,
// [17 + 8*l + it] = error trace, [81 + (8*l+it)*49..] HTH, [3217 + (8*l+it)*7..] HTz, [3665 + (8*l+it)*19] solution
double orc_vio_update(void *h, const uint8_t *img, int n_pts, const double *pos, const float *warp_patch, const int32_t *search_levels,
                      const double *inv_expo_list, const double *state_in, const double *state_prop, double *state_out, float *errors_out,
                      double *stats_out) {
  VIOManager *v = (VIOManager *)h;
  StatesGroup st, prop;
  unpack_state(state_in, st);
  unpack_state(state_prop, prop);
  v->state = &st;
  v->state_propagat = &prop;
  v->total_points = n_pts;
  v->pos.assign(pos, pos + 3 * (size_t)n_pts);
  v->warp_patch.assign(warp_patch, warp_patch + (size_t)n_pts * 64 * v->patch_pyrimid_level);
  v->search_levels.assign(search_levels, search_levels + n_pts);
  v->inv_expo_list.assign(inv_expo_list, inv_expo_list + n_pts);
  v->errors.assign(n_pts, 0.f);
  v->G = M19::Zero();
  Image im;
  im.data = img, im.cols = v->width, im.rows = v->height;
  auto t0 = std::chrono::steady_clock::now();
  v->computeJacobianAndUpdateEKF(im);
  auto t1 = std::chrono::steady_clock::now();
  pack_state(st, state_out);
  if (errors_out)
    for (int i = 0; i < n_pts; i++) errors_out[i] = v->errors[i];
  if (stats_out) {
    const VioStats &s = v->stats_;
    for (int i = 0; i < 4881; i++) stats_out[i] = 0;
    stats_out[0] = s.total_iters;
    for (int l = 0; l < 8; l++) {
      stats_out[1 + l] = s.iters_per_level[l];
      stats_out[9 + l] = s.accepted_per_level[l];
      for (int it = 0; it < 8; it++) {
        stats_out[17 + 8 * l + it] = s.error_trace[l][it];
        for (int k = 0; k < 49; k++) stats_out[81 + (8 * l + it) * 49 + k] = s.HTH[l][it][k];
        for (int k = 0; k < 7; k++) stats_out[3217 + (8 * l + it) * 7 + k] = s.HTz[l][it][k];
        for (int k = 0; k < 19; k++) stats_out[3665 + (8 * l + it) * 19 + k] = s.solution[l][it][k];
      }
    }
  }
  v->state = nullptr;
  v->state_propagat = nullptr;
  return std::chrono::duration<double>(t1 - t0).count();
}

// Inverse-compositional variant: per-point reference-feature data (kept by pointer for the images: the caller keeps them alive)
// and the switch the reference reads from vio/inverse_composition_en.
void orc_vio_set_inverse_refs(void *h, const uint8_t *const *imgs, int n_imgs, int n_pts, const int32_t *ref_img_index, const double *ref_px,
                              const double *ref_f, const double *ref_R, const double *ref_pos) {
  VIOManager *v = (VIOManager *)h;
  v->ref_imgs.resize(n_imgs);
  for (int k = 0; k < n_imgs; k++) v->ref_imgs[k].data = imgs[k], v->ref_imgs[k].cols = v->width, v->ref_imgs[k].rows = v->height;
  v->ref_img_index.assign(ref_img_index, ref_img_index + n_pts);
  v->ref_px.assign(ref_px, ref_px + 2 * (size_t)n_pts);
  v->ref_f.assign(ref_f, ref_f + 3 * (size_t)n_pts);
  v->ref_R.assign(ref_R, ref_R + 9 * (size_t)n_pts);
  v->ref_pos.assign(ref_pos, ref_pos + 3 * (size_t)n_pts);
}
void orc_vio_set_inverse(void *h, int enable) { ((VIOManager *)h)->inverse_composition_en = enable != 0; }
// H_sub_inv of the LAST level processed (level 0 after a full update): (n_pts*64) x 6
int orc_vio_get_h_sub_inv(void *h, double *out, int max_doubles) {
  VIOManager *v = (VIOManager *)h;
  int n = (int)v->H_sub_inv.size();
  if (out && n <= max_doubles) memcpy(out, v->H_sub_inv.data(), sizeof(double) * n);
  return n;
}
void orc_vio_precompute_reference_patches(void *h, int n_pts, const double *pos, int level) {
  VIOManager *v = (VIOManager *)h;
  v->total_points = n_pts;
  v->pos.assign(pos, pos + 3 * (size_t)n_pts);
  v->precomputeReferencePatches(level);
}

void orc_vio_get_image_patch(void *h, const uint8_t *img, const double *pc, int level, float *patch_out /* levels*64 */) {
  VIOManager *v = (VIOManager *)h;
  Image im;
  im.data = img, im.cols = v->width, im.rows = v->height;
  V2 p;
  p[0] = pc[0], p[1] = pc[1];
  v->getImagePatch(im, p, patch_out, level);
}
// warpAffine over all pyramid levels (src/vio.cpp:739-742).
void orc_vio_warp_affine(void *h, const uint8_t *img_ref, int cols, int rows, const double *A_cur_ref, const double *px_ref, int search_level,
                         float *patch_out /* levels*64 */) {
  VIOManager *v = (VIOManager *)h;
  Image im;
  im.data = img_ref, im.cols = cols, im.rows = rows;
  M2 A;
  for (int i = 0; i < 4; i++) A.a[i] = A_cur_ref[i];
  V2 p;
  p[0] = px_ref[0], p[1] = px_ref[1];
  for (int pyramid_level = 0; pyramid_level <= v->patch_pyrimid_level - 1; pyramid_level++)
    v->warpAffine(A, im, p, 0, search_level, pyramid_level, v->patch_size_half, patch_out);
}
// getWarpMatrixAffineHomography + getBestSearchLevel (src/vio.cpp:701-714).
// T_*_w given as R(9) + t(3) of the frame poses T_f_w_.
int orc_vio_warp_matrix(void *h, const double *px_ref, const double *pos_w, const double *normal_w, const double *R_ref_w,
                        const double *t_ref_w, const double *R_cur_w, const double *t_cur_w, double *A_out) {
  VIOManager *v = (VIOManager *)h;
  SE3 Tref, Tcur;
  for (int i = 0; i < 9; i++) Tref.R.a[i] = R_ref_w[i], Tcur.R.a[i] = R_cur_w[i];
  for (int i = 0; i < 3; i++) Tref.t[i] = t_ref_w[i], Tcur.t[i] = t_cur_w[i];
  V3 n = v3(normal_w[0], normal_w[1], normal_w[2]);
  V3 pw = v3(pos_w[0], pos_w[1], pos_w[2]);
  V3 norm_vec = Tref.R * n;
  norm_vec = norm_vec / norm(norm_vec);  // :701
  V3 pf = Tref * pw;                     // :703
  SE3 T_cur_ref = Tcur * Tref.inverse(); // :710
  V2 px;
  px[0] = px_ref[0], px[1] = px_ref[1];
  M2 A;
  v->getWarpMatrixAffineHomography(v->cam, px, pf, norm_vec, T_cur_ref, 0, A);
  for (int i = 0; i < 4; i++) A_out[i] = A.a[i];
  return v->getBestSearchLevel(A, 2);
}
void orc_cam_world2cam(void *h, const double *xyz, double *px) {
  V2 p = ((VIOManager *)h)->cam.world2cam(v3(xyz[0], xyz[1], xyz[2]));
  px[0] = p[0], px[1] = p[1];
}
void orc_cam_cam2world(void *h, const double *px, double *xyz) {
  V2 p;
  p[0] = px[0], p[1] = px[1];
  V3 f = ((VIOManager *)h)->cam.cam2world(p);
  for (int i = 0; i < 3; i++) xyz[i] = f[i];
}

int orc_max_threads() {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

}  // extern "C"
