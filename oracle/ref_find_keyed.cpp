// oracle/_ref — the reference's OWN two call sites of find_correspond in the VIO front end, run as they are on the reference's
// own map: VIOManager::updateReferencePatch (src/vio.cpp:969-1034, key rule A) and the ray-casting branch of
// VIOManager::retrieveFromVisualSparseMap (:484-596 with raycast_en on, key rule B). The VIOManager is the one the driver
// ref_vio.cpp (included as it is) creates; the map is a VoxelMapManager of the reference's voxel_map.cpp (which ref_vio.cpp
// includes) fed with (point_w, var) lists through its own UpdateVoxelMap, as the driver ref_voxel_map.cpp feeds it.
// What is set up around the reference's code (not the reference's code):
//   rule A: stand-in VisualPoints that pass the four skips (is_normal_initialized_, not converged, six observations,
//           update_flag 1) with normal_ = previous_normal_ = 0 and covariance_ = 1e12 I, and every plane's radius_ raised to
//           FLT_MAX for the call (restored after), so that the distance gates pass whenever a plane is found: normal_ then
//           becomes the found plane's normal_ (previous_normal_ . normal_ = 0 is not < 0), and stays 0 otherwise (the one
//           exception: range_dis is NaN when float rounding makes dis_to_center - dis_to_plane^2 negative);
//   rule B: one grid row of n cells, each with the caller's ray (camera-frame samples in rays_with_sample_points), an empty
//           scan, and a feat_map holding one empty voxel far from every ray (the retrieval returns at once on an empty one).
// Read back: the points' normal_ (rule A); the samples' world points f2w(it) and add_from_voxel_map (rule B).
// TEST INFRASTRUCTURE ONLY: pins the oracle's keyed restatement (oracle/orc_find_keyed.cpp) in tests/test_oracle_find_keyed.py.
// Built by oracle/find_keyed.mk where the reference source exists.
#include <cfloat>

#include "ref_vio.cpp"

namespace {
struct RefKeyed {
  VoxelMapConfig config;
  std::unordered_map<VOXEL_LOCATION, VoxelOctoTree *> map;
  VoxelMapManager *mgr = nullptr;
  RefVio *vio = nullptr;
  ~RefKeyed() {
    if (mgr)
      for (auto &kv : mgr->voxel_map_) delete kv.second;
    delete mgr;
    delete vio;
  }
};

void planes_of(VoxelOctoTree *t, std::vector<VoxelPlane *> &out) {
  if (t->plane_ptr_->is_plane_) out.push_back(t->plane_ptr_);
  for (int l = 0; l < 8; l++)
    if (t->leaves_[l]) planes_of(t->leaves_[l], out);
}
}  // namespace

extern "C" {

// map_cfg as ref_map_create's (voxel_size, max_layer, min_eigen_value, max_points_num, layer_init_num[8]); cam / extrinsics /
// vio_cfg as ref_vio_create's
void *ref_keyed_create(const double *map_cfg, const double *cam, const double *extR, const double *extT, const double *Rcl, const double *Pcl,
                       const double *vio_cfg) {
  RefKeyed *r = new RefKeyed;
  VoxelMapConfig &c = r->config;
  c.max_voxel_size_ = map_cfg[0], c.max_layer_ = (int)map_cfg[1], c.planner_threshold_ = map_cfg[2], c.max_points_num_ = (int)map_cfg[3];
  c.layer_init_num_.clear();
  for (int k = 0; k < 8; k++) c.layer_init_num_.push_back((int)map_cfg[4 + k]);
  c.max_iterations_ = 5, c.sigma_num_ = 3, c.dept_err_ = 0.02, c.beam_err_ = 0.05, c.is_pub_plane_map_ = false;
  c.sliding_thresh = 8, c.map_sliding_en = false, c.half_map_size = 100;
  r->mgr = new VoxelMapManager(c, r->map);
  r->vio = (RefVio *)ref_vio_create(cam, extR, extT, Rcl, Pcl, vio_cfg);
  if (!r->vio) {
    delete r;
    return nullptr;
  }
  return r;
}
void ref_keyed_destroy(void *h) { delete static_cast<RefKeyed *>(h); }

// VoxelMapManager::UpdateVoxelMap (voxel_map.cpp:609-641) with point_w [n][3], var [n][9]
void ref_keyed_update(void *h, const double *pts_world, const double *var9, int n) {
  RefKeyed *r = static_cast<RefKeyed *>(h);
  std::vector<pointWithVar> pts(n);
  for (int i = 0; i < n; i++) {
    pts[i].point_w << pts_world[3 * i], pts_world[3 * i + 1], pts_world[3 * i + 2];
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) pts[i].var(a, b) = var9[9 * (size_t)i + 3 * a + b];
  }
  r->mgr->UpdateVoxelMap(pts);
}

// Rule A: updateReferencePatch over n stand-in points at pos [n][3]; normal_out [n][3] = their normal_ afterwards.
void ref_keyed_update_reference_patch(void *h, const double *pos, int n, double *normal_out) {
  RefKeyed *r = static_cast<RefKeyed *>(h);
  VIOManager &v = r->vio->v;
  std::vector<VoxelPlane *> planes;
  for (auto &kv : r->mgr->voxel_map_) planes_of(kv.second, planes);
  std::vector<float> radius(planes.size());
  for (size_t k = 0; k < planes.size(); k++) radius[k] = planes[k]->radius_, planes[k]->radius_ = FLT_MAX;
  SubSparseMap &sub = *v.visual_submap;
  sub.reset();
  std::vector<VisualPoint *> pts;
  for (int i = 0; i < n; i++) {
    VisualPoint *pt = new VisualPoint(V3D(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]));
    pt->normal_ = V3D(0, 0, 0), pt->previous_normal_ = V3D(0, 0, 0);
    pt->is_normal_initialized_ = true, pt->is_converged_ = false;
    pt->covariance_ = M3D::Identity() * 1e12;
    for (int k = 0; k < 6; k++) {
      Feature *f = new Feature(pt, new float[64](), V2D(0, 0), V3D(0, 0, 1), SE3(), 0);
      f->id_ = k;
      pt->obs_.push_back(f);
    }
    pts.push_back(pt);
    sub.voxel_points.push_back(pt);
  }
  v.total_points = n;
  v.update_flag.assign(n, 1);
  v.updateReferencePatch(r->mgr->voxel_map_);
  for (int i = 0; i < n; i++)
    for (int k = 0; k < 3; k++) normal_out[3 * i + k] = pts[i]->normal_[k];
  sub.reset();
  for (auto *p : pts) delete p;  // ~VisualPoint deletes its observations and their patches
  v.total_points = 0;
  for (size_t k = 0; k < planes.size(); k++) planes[k]->radius_ = radius[k];
}

// Rule B: the ray-casting branch of retrieveFromVisualSparseMap with the frame at the packed state, one grid row of n_cells
// cells, cell c casting rays[ray_first[c] .. ray_first[c] + ray_count[c]) (camera frame, [m][3]). Out: samples_w [m][3] =
// new_frame_->f2w of every ray sample; add_out [cap][6] = add_from_voxel_map in order (point_w, normal); returns its size.
int ref_keyed_raycast(void *h, const double *state, int n_cells, const int32_t *ray_first, const int32_t *ray_count, const double *rays, int m,
                      double *samples_w, double *add_out, int cap) {
  RefKeyed *r = static_cast<RefKeyed *>(h);
  VIOManager &v = r->vio->v;
  for (auto &kv : v.feat_map) delete kv.second;
  v.feat_map.clear();
  v.feat_map[VOXEL_LOCATION(1000000000, 1000000000, 1000000000)] = new VOXEL_POINTS(0);  // non-empty, far from every ray
  v.grid_size = 8, v.grid_n_width = n_cells, v.grid_n_height = 1, v.length = n_cells;
  v.grid_num.resize(v.length), v.map_index.resize(v.length), v.map_dist.resize(v.length), v.update_flag.resize(v.length), v.scan_value.resize(v.length);
  v.border_flag.assign(v.length, 0);
  v.rays_with_sample_points.assign(v.length, std::vector<V3D>());
  for (int c = 0; c < n_cells; c++)
    for (int q = ray_first[c]; q < ray_first[c] + ray_count[c]; q++) v.rays_with_sample_points[c].push_back(V3D(rays[3 * q], rays[3 * q + 1], rays[3 * q + 2]));
  v.normal_en = true, v.ncc_en = false, v.raycast_en = true;
  unpack_state(state, r->vio->st);
  cv::Mat im = cv::Mat::zeros(v.height, v.width, CV_8UC1);
  v.new_frame_.reset(new Frame(v.cam, im));
  v.updateFrameState(r->vio->st);
  for (int q = 0; q < m; q++) {
    const V3D w = v.new_frame_->f2w(V3D(rays[3 * q], rays[3 * q + 1], rays[3 * q + 2]));
    for (int k = 0; k < 3; k++) samples_w[3 * q + k] = w[k];
  }
  vector<pointWithVar> pg;
  v.resetGrid();
  v.retrieveFromVisualSparseMap(im, pg, r->mgr->voxel_map_);
  const std::vector<pointWithVar> &add = v.visual_submap->add_from_voxel_map;
  for (int j = 0; j < (int)add.size() && j < cap; j++)
    for (int k = 0; k < 3; k++) add_out[6 * j + k] = add[j].point_w[k], add_out[6 * j + 3 + k] = add[j].normal[k];
  v.raycast_en = false;
  return (int)add.size();
}
}
