// oracle/_ref — VIOManager::resetGrid + retrieveFromVisualSparseMap (src/vio.cpp:162-177, 352-782) run as they are, on the
// VIOManager the driver ref_vio.cpp (included as it is) creates: new_frame_ is a Frame of the image with updateFrameState(state),
// feat_map holds stand-in VisualPoints (position, normal, is_normal_initialized_) with n_obs Features each whose img_ is the
// frame image, taken at the frame pose at the point's pixel (the first one its ref_patch); normal_en on, ncc_en and raycast_en off and an outlier threshold
// of infinity, so every point past the depth check reaches visual_submap. Read back: sub_feat_map in iteration order, grid_num and
// retrieve_voxel_points per cell, and the surviving visual_submap->voxel_points. The VIOManager (and so sub_feat_map) lives
// across calls, as the member does across frames. What is not the reference's code: vikit (the camera models of the
// stand-ins in ref_shim/vikit/). TEST INFRASTRUCTURE ONLY: pins the oracle's restatement (oracle/orc_retrieve.cpp) in
// tests/test_oracle_retrieve.py. Built by oracle/retrieve.mk where the reference source exists.
#include <limits>
#include <map>

#include "ref_vio.cpp"

extern "C" {

// Inputs: the grey image (the camera's size), the packed state, the scan (point_w n x 3), the flat visual map (n_vox voxels:
// vkeys n_vox x 3, vfirst / vcount into the points; points: pos P x 3, normal P x 3, n_obs P) and the grid geometry.
// Outputs: sub_keys (room for n x 3; returns their number), grid_type (length bytes, 1 = TYPE_MAP), cell_pt (length: the
// point index of retrieve_voxel_points, -1 none), survivors (room for length: point indices of visual_submap->voxel_points,
// *n_survivors of them).
int ref_retrieve(void *h, const uint8_t *img, const double *state, const double *point_w, int n, const int64_t *vkeys, const int32_t *vfirst,
                 const int32_t *vcount, int n_vox, const double *pos, const double *normal, const int32_t *n_obs, int grid_size, int grid_n_width,
                 int grid_n_height, int border, int64_t *sub_keys, uint8_t *grid_type, int32_t *cell_pt, int32_t *survivors, int32_t *n_survivors) {
  RefVio *r = (RefVio *)h;
  VIOManager &v = r->v;
  for (auto &kv : v.feat_map) delete kv.second;  // ~VOXEL_POINTS deletes its points and their features
  v.feat_map.clear();
  v.grid_size = grid_size, v.grid_n_width = grid_n_width, v.grid_n_height = grid_n_height, v.border = border;
  v.length = grid_n_width * grid_n_height;
  v.grid_num.resize(v.length), v.map_index.resize(v.length), v.map_dist.resize(v.length), v.update_flag.resize(v.length), v.scan_value.resize(v.length);
  v.border_flag.assign(v.length, 0);
  v.normal_en = true, v.ncc_en = false, v.raycast_en = false, v.outlier_threshold = std::numeric_limits<double>::infinity();
  unpack_state(state, r->st);
  cv::Mat im = cv::Mat(v.height, v.width, CV_8UC1, (void *)img).clone();
  v.new_frame_.reset(new Frame(v.cam, im));
  v.updateFrameState(r->st);
  std::map<const VisualPoint *, int> index;
  for (int j = 0; j < n_vox; j++) {
    VOXEL_POINTS *vox = new VOXEL_POINTS(0);
    for (int q = vfirst[j]; q < vfirst[j] + vcount[j]; q++) {
      VisualPoint *pt = new VisualPoint(V3D(pos[3 * q], pos[3 * q + 1], pos[3 * q + 2]));
      pt->normal_ = V3D(normal[3 * q], normal[3 * q + 1], normal[3 * q + 2]);
      pt->is_normal_initialized_ = true;
      const V2D px = v.new_frame_->w2c(pt->pos_);
      for (int k = 0; k < n_obs[q]; k++) {
        Feature *f = new Feature(pt, new float[64](), px, V3D(0, 0, 1), v.new_frame_->T_f_w_, 0);
        f->img_ = im;
        pt->obs_.push_back(f);
      }
      if (!pt->obs_.empty()) pt->ref_patch = pt->obs_.front(), pt->has_ref_patch_ = true;  // the reference feature is not under test here
      vox->voxel_points.push_back(pt);
      index[pt] = q;
    }
    v.feat_map[VOXEL_LOCATION(vkeys[3 * j], vkeys[3 * j + 1], vkeys[3 * j + 2])] = vox;
  }
  vector<pointWithVar> pg(n);
  for (int i = 0; i < n; i++)
    for (int k = 0; k < 3; k++) pg[i].point_w[k] = point_w[3 * i + k];
  unordered_map<VOXEL_LOCATION, VoxelOctoTree *> plane_map;
  v.resetGrid();
  v.retrieveFromVisualSparseMap(im, pg, plane_map);
  int k = 0;
  for (auto &kv : v.sub_feat_map) sub_keys[3 * k] = kv.first.x, sub_keys[3 * k + 1] = kv.first.y, sub_keys[3 * k + 2] = kv.first.z, k++;
  for (int c = 0; c < v.length; c++) {
    grid_type[c] = v.grid_num[c] == VIOManager::TYPE_MAP;
    cell_pt[c] = (v.grid_num[c] == VIOManager::TYPE_MAP && v.retrieve_voxel_points[c]) ? index[v.retrieve_voxel_points[c]] : -1;
  }
  const std::vector<VisualPoint *> &sv = v.visual_submap->voxel_points;
  for (size_t q = 0; q < sv.size(); q++) survivors[q] = index[sv[q]];
  *n_survivors = (int32_t)sv.size();
  return k;
}
}
