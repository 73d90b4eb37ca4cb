// oracle/_ref — the reference's OWN LIO update, compiled from where it lies (/root/reference/src/voxel_map.cpp with
// include/voxel_map.h, common_lib.h, utils/*.h, unmodified) against the stand-in headers of oracle/ref_shim/ (Eigen, PCL,
// ROS message types: none of them is in this image). TEST INFRASTRUCTURE ONLY: used to pin the oracle restatement
// (oracle/orc_lio.cpp) against the reference's code — tests/test_oracle_ref_pin.py — and, optionally, as a CPU timing of the
// reference source. No reference source is copied into this repository; this file only #includes it and adds a C entry
// point that builds the octree the reference walks from the flat map arrays and runs VoxelMapManager::StateEstimation.
#define ROOT_DIR ""
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "/root/reference/src/voxel_map.cpp"

namespace {
// the 256-byte plane record of include/esikf_b200.h (restated here: the oracle side must not include product headers)
struct FlatPlane {
  double center[3];
  double normal[3];
  double plane_var[21];
  float d;
  float radius;
  int32_t layer;
  int32_t path;
  int32_t pad[6];
};
static_assert(sizeof(FlatPlane) == 256, "flat plane record");

void unpack_state(const double *s, StatesGroup &st) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) st.rot_end(i, j) = s[3 * i + j];
  for (int i = 0; i < 3; i++) st.pos_end(i) = s[9 + i], st.vel_end(i) = s[13 + i], st.bias_g(i) = s[16 + i], st.bias_a(i) = s[19 + i], st.gravity(i) = s[22 + i];
  st.inv_expo_time = s[12];
  for (int i = 0; i < 19; i++)
    for (int j = 0; j < 19; j++) st.cov(i, j) = s[25 + 19 * i + j];
}
void pack_state(const StatesGroup &st, double *s) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) s[3 * i + j] = st.rot_end(i, j);
  for (int i = 0; i < 3; i++) s[9 + i] = st.pos_end(i), s[13 + i] = st.vel_end(i), s[16 + i] = st.bias_g(i), s[19 + i] = st.bias_a(i), s[22 + i] = st.gravity(i);
  s[12] = st.inv_expo_time;
  for (int i = 0; i < 19; i++)
    for (int j = 0; j < 19; j++) s[25 + 19 * i + j] = st.cov(i, j);
}
}  // namespace

extern "C" {

// Version of this driver's C API. tests/oracle_bind.py uses the library live only at this version (an older build, whatever
// its timestamp, lacks entry points the tests call); the Makefile rebuilds a library that does not export it.
int ref_lio_driver_version_2(void) { return 2; }

// cfg: voxel_size, max_layer, max_iterations, sigma_num, dept_err, beam_err.
// Outputs: state_out (386), M_out[8] (effective feature num per iteration, parsed from the reference's own console line,
// voxel_map.cpp:404-405), iters_out, normals_out (n x 3: pv_list_[i].normal), and the final ptpl_list_ as
// ptpl_center (k x 3), ptpl_dis (k), ptpl_point_b (k x 3) with k = *n_ptpl (capacity n). Returns 0.
int ref_lio_state_estimation(const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots, const void *planes_v, int n_planes, const double *cfg,
                             const double *extR, const double *extT, const float *pts, int n, const double *state_in, const double *state_prop, double *state_out,
                             int32_t *M_out, int32_t *iters_out, double *normals_out, int32_t *n_ptpl, double *ptpl_center, float *ptpl_dis, float *ptpl_point_b,
                             double *seconds_out) {
  (void)n_planes;
  const FlatPlane *planes = static_cast<const FlatPlane *>(planes_v);
  VoxelMapConfig config;
  config.max_voxel_size_ = cfg[0], config.max_layer_ = (int)cfg[1], config.max_iterations_ = (int)cfg[2], config.sigma_num_ = cfg[3];
  config.dept_err_ = cfg[4], config.beam_err_ = cfg[5];
  config.layer_init_num_ = std::vector<int>{5, 5, 5, 5, 5};
  config.max_points_num_ = 50, config.planner_threshold_ = 0.01, config.is_pub_plane_map_ = false;
  config.sliding_thresh = 8, config.map_sliding_en = false, config.half_map_size = 100;
  std::unordered_map<VOXEL_LOCATION, VoxelOctoTree *> voxel_map;
  // the octree build_single_residual walks: roots positioned like BuildVoxelMap does (voxel_map.cpp:575-581), plane nodes at
  // (layer, path) carrying the fitted plane
  const float voxel_size = config.max_voxel_size_;
  for (int r = 0; r < n_roots; r++) {
    VOXEL_LOCATION position(keys[3 * r], keys[3 * r + 1], keys[3 * r + 2]);
    VoxelOctoTree *root = new VoxelOctoTree(config.max_layer_, 0, 5, config.max_points_num_, (float)config.planner_threshold_);
    root->quater_length_ = voxel_size / 4;
    root->voxel_center_[0] = (0.5 + position.x) * voxel_size;
    root->voxel_center_[1] = (0.5 + position.y) * voxel_size;
    root->voxel_center_[2] = (0.5 + position.z) * voxel_size;
    root->init_octo_ = true;
    voxel_map[position] = root;
    for (int c = 0; c < count[r]; c++) {
      const FlatPlane &f = planes[first[r] + c];
      VoxelOctoTree *node = root;
      for (int l = 0; l < f.layer; l++) {
        const int leaf = (f.path >> (3 * l)) & 7;
        if (node->leaves_[leaf] == nullptr) {
          VoxelOctoTree *ch = new VoxelOctoTree(config.max_layer_, l + 1, 5, config.max_points_num_, (float)config.planner_threshold_);
          const int xyz[3] = {(leaf >> 2) & 1, (leaf >> 1) & 1, leaf & 1};
          for (int k = 0; k < 3; k++) ch->voxel_center_[k] = node->voxel_center_[k] + (2 * xyz[k] - 1) * node->quater_length_;
          ch->quater_length_ = node->quater_length_ / 2;
          ch->init_octo_ = true;
          node->leaves_[leaf] = ch;
        }
        node = node->leaves_[leaf];
      }
      VoxelPlane &p = *node->plane_ptr_;
      for (int k = 0; k < 3; k++) p.center_(k) = f.center[k], p.normal_(k) = f.normal[k];
      int t = 0;
      for (int i = 0; i < 6; i++)
        for (int j = i; j < 6; j++) p.plane_var_(i, j) = p.plane_var_(j, i) = f.plane_var[t++];
      p.d_ = f.d, p.radius_ = f.radius, p.is_plane_ = true, p.is_init_ = true;
    }
  }
  int rc = 0;
  {
    VoxelMapManager mgr(config, voxel_map);
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) mgr.extR_(i, j) = extR[3 * i + j];
      mgr.extT_(i) = extT[i];
    }
    mgr.feats_down_body_->points.resize(n);
    for (int i = 0; i < n; i++) {
      PointType &p = mgr.feats_down_body_->points[i];
      p.x = pts[3 * i], p.y = pts[3 * i + 1], p.z = pts[3 * i + 2];
    }
    mgr.feats_down_size_ = n;
    unpack_state(state_in, mgr.state_);  // voxelmap_manager->state_ = _state (LIVMapper.cpp:257)
    StatesGroup prop;
    unpack_state(state_prop, prop);
    // the reference reports the per-iteration effective feature number on std::cout only: capture it
    std::ostringstream captured;
    std::streambuf *old = std::cout.rdbuf(captured.rdbuf());
    const double t0 = omp_get_wtime();
    mgr.StateEstimation(prop);  // LIVMapper.cpp:370
    const double t1 = omp_get_wtime();
    std::cout.rdbuf(old);
    if (seconds_out) *seconds_out = t1 - t0;
    int iters = 0;
    {
      const std::string txt = captured.str(), key = "effective feature num: ";
      size_t pos = 0;
      while ((pos = txt.find(key, pos)) != std::string::npos && iters < 8) {
        pos += key.size();
        M_out[iters++] = atoi(txt.c_str() + pos);
      }
    }
    *iters_out = iters;
    pack_state(mgr.state_, state_out);
    for (int i = 0; i < n; i++)
      for (int k = 0; k < 3; k++) normals_out[3 * i + k] = mgr.pv_list_[i].normal(k);
    const int k = (int)mgr.ptpl_list_.size();
    *n_ptpl = k;
    for (int i = 0; i < k && i < n; i++) {
      const PointToPlane &q = mgr.ptpl_list_[i];
      for (int c = 0; c < 3; c++) ptpl_center[3 * i + c] = q.center_(c), ptpl_point_b[3 * i + c] = (float)q.point_b_(c);
      ptpl_dis[i] = q.dis_to_plane_;
    }
  }
  for (auto &kv : voxel_map) delete kv.second;
  return rc;
}

// ---- the reference's own map construction (pins the oracle's BuildVoxelMap / UpdateVoxelMap / init_plane restatement, and through
// it what the device-resident map is held to): a persistent VoxelMapManager fed with caller-supplied (point_w, var) lists.
struct RefMap {
  VoxelMapConfig config;
  std::unordered_map<VOXEL_LOCATION, VoxelOctoTree *> map;
  VoxelMapManager *mgr = nullptr;
  ~RefMap() {
    if (mgr)
      for (auto &kv : mgr->voxel_map_) delete kv.second;  // the manager holds its own copy of the handle map (voxel_map.h:194, 221)
    delete mgr;
  }
};
// cfg: voxel_size, max_layer, min_eigen_value (planner_threshold_), max_points_num, layer_init_num[0..7] (a node of layer k
// reads entry k: max_layer up to 7)
void *ref_map_create(const double *cfg) {
  RefMap *r = new RefMap;
  VoxelMapConfig &c = r->config;
  c.max_voxel_size_ = cfg[0], c.max_layer_ = (int)cfg[1], c.planner_threshold_ = cfg[2], c.max_points_num_ = (int)cfg[3];
  c.layer_init_num_.clear();
  for (int k = 0; k < 8; k++) c.layer_init_num_.push_back((int)cfg[4 + k]);
  c.max_iterations_ = 5, c.sigma_num_ = 3, c.dept_err_ = 0.02, c.beam_err_ = 0.05, c.is_pub_plane_map_ = false;
  c.sliding_thresh = 8, c.map_sliding_en = false, c.half_map_size = 100;
  r->mgr = new VoxelMapManager(c, r->map);
  return r;
}
void ref_map_destroy(void *h) { delete static_cast<RefMap *>(h); }
// VoxelMapManager::UpdateVoxelMap (voxel_map.cpp:609-641) on the manager's own voxel_map_ (a by-value member, voxel_map.h:194).
void ref_map_update(void *h, const double *pts_world, const double *var9, int n) {
  RefMap *r = static_cast<RefMap *>(h);
  std::vector<pointWithVar> pts(n);
  for (int i = 0; i < n; i++) {
    pts[i].point_w << pts_world[3 * i], pts_world[3 * i + 1], pts_world[3 * i + 2];
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) pts[i].var(a, b) = var9[9 * (size_t)i + 3 * a + b];
  }
  r->mgr->UpdateVoxelMap(pts);
}
// First LiDAR frame (LIVMapper.cpp:356-366): feats_down_world_ = TransformLidar(state, feats_down_body_) (the manager's own
// TransformLidar, the same expression as LIVMapper::transformLidar :645), then VoxelMapManager::BuildVoxelMap (voxel_map.cpp:532-591).
void ref_map_build(void *h, const float *pts_body, int n, const double *state, const double *extR, const double *extT, double dept_err, double beam_err) {
  RefMap *r = static_cast<RefMap *>(h);
  VoxelMapManager &m = *r->mgr;
  m.config_setting_.dept_err_ = dept_err, m.config_setting_.beam_err_ = beam_err;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) m.extR_(i, j) = extR[3 * i + j];
    m.extT_(i) = extT[i];
  }
  m.feats_down_body_->points.resize(n);
  for (int i = 0; i < n; i++) {
    PointType &p = m.feats_down_body_->points[i];
    p.x = pts_body[3 * i], p.y = pts_body[3 * i + 1], p.z = pts_body[3 * i + 2];
  }
  m.feats_down_size_ = n;
  unpack_state(state, m.state_);
  pcl::PointCloud<pcl::PointXYZI>::Ptr world(new pcl::PointCloud<pcl::PointXYZI>());
  m.TransformLidar(m.state_.rot_end, m.state_.pos_end, m.feats_down_body_, world);
  m.feats_down_world_->points.resize(n);
  for (int i = 0; i < n; i++) {  // LIVMapper keeps the world cloud as PointXYZINormal: the float coordinates carry over unchanged
    PointType &p = m.feats_down_world_->points[i];
    p.x = world->points[i].x, p.y = world->points[i].y, p.z = world->points[i].z;
  }
  m.BuildVoxelMap();
}
// VoxelMapManager::clearMemOutOfMap (voxel_map.cpp:950-971); its console line is swallowed
void ref_map_clear_out_of_map(void *h, int x_max, int x_min, int y_max, int y_min, int z_max, int z_min) {
  RefMap *r = static_cast<RefMap *>(h);
  std::ostringstream captured;
  std::streambuf *old = std::cout.rdbuf(captured.rdbuf());
  r->mgr->clearMemOutOfMap(x_max, x_min, y_max, y_min, z_max, z_min);
  std::cout.rdbuf(old);
}
static void ref_flatten_node(const VoxelOctoTree *node, int layer, int max_layer, int path, std::vector<FlatPlane> *out, int *count) {
  if (node->plane_ptr_->is_plane_) {  // the order build_single_residual visits (voxel_map.cpp:721, 771-784)
    if (out) {
      const VoxelPlane &p = *node->plane_ptr_;
      FlatPlane f;
      memset(&f, 0, sizeof(f));
      for (int k = 0; k < 3; k++) f.center[k] = p.center_(k), f.normal[k] = p.normal_(k);
      int t = 0;
      for (int i = 0; i < 6; i++)
        for (int j = i; j < 6; j++) f.plane_var[t++] = p.plane_var_(i, j);
      f.d = p.d_, f.radius = p.radius_, f.layer = layer, f.path = path;
      out->push_back(f);
    }
    (*count)++;
    return;
  }
  if (layer < max_layer)
    for (int l = 0; l < 8; l++)
      if (node->leaves_[l] != nullptr) ref_flatten_node(node->leaves_[l], layer + 1, max_layer, path | (l << (3 * layer)), out, count);
}
// two-call: planes == NULL returns the sizes
void ref_map_flatten(void *h, int *n_roots, int *n_planes, int64_t *keys, int32_t *first, int32_t *count, void *planes_v) {
  RefMap *r = static_cast<RefMap *>(h);
  const auto &vm = r->mgr->voxel_map_;
  std::vector<FlatPlane> planes;
  int nr = 0, np = 0;
  for (const auto &kv : vm) {
    int c = 0;
    ref_flatten_node(kv.second, 0, r->config.max_layer_, 0, planes_v ? &planes : nullptr, &c);
    if (planes_v) keys[3 * nr] = kv.first.x, keys[3 * nr + 1] = kv.first.y, keys[3 * nr + 2] = kv.first.z, first[nr] = np, count[nr] = c;
    nr++, np += c;
  }
  *n_roots = nr, *n_planes = np;
  if (planes_v) memcpy(planes_v, planes.data(), planes.size() * sizeof(FlatPlane));
}

// Every node of every root (DFS pre-order, leaves 0..7), 12 int64 a row: key x y z | layer path | init_octo octo_state
// update_enable is_plane | new_points temp_points_.size() points_size. Returns the number of nodes; rows beyond cap are not written.
static void ref_dump_node(const VoxelOctoTree *nd, int64_t path, const VOXEL_LOCATION &key, int64_t *out, int cap, int *n) {
  if (*n < cap) {
    int64_t *r = out + (size_t)(*n) * 12;
    r[0] = key.x, r[1] = key.y, r[2] = key.z, r[3] = nd->layer_, r[4] = path;
    r[5] = nd->init_octo_, r[6] = nd->octo_state_, r[7] = nd->update_enable_, r[8] = nd->plane_ptr_->is_plane_;
    r[9] = nd->new_points_, r[10] = (int64_t)nd->temp_points_.size(), r[11] = nd->plane_ptr_->points_size_;
  }
  (*n)++;
  for (int l = 0; l < 8; l++)
    if (nd->leaves_[l]) ref_dump_node(nd->leaves_[l], path | ((int64_t)l << (3 * nd->layer_)), key, out, cap, n);
}
int ref_map_dump_nodes(void *h, int64_t *out, int cap) {
  RefMap *r = static_cast<RefMap *>(h);
  int n = 0;
  for (const auto &kv : r->mgr->voxel_map_) ref_dump_node(kv.second, 0, kv.first, out, cap, &n);
  return n;
}

// calcBodyCov of the reference (voxel_map.cpp:15-34) for one point.
void ref_calc_body_cov(const double *pb, float range_inc, float degree_inc, double *cov9) {
  Eigen::Vector3d p(pb[0], pb[1], pb[2]);
  Eigen::Matrix3d cov;
  calcBodyCov(p, range_inc, degree_inc, cov);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) cov9[3 * i + j] = cov(i, j);
}

}  // extern "C"
