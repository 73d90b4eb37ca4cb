// oracle/_ref — VIOManager::generateVisualMapPoints (src/vio.cpp:804-906) run as it is, on the VIOManager the driver ref_vio.cpp
// (included as it is) creates: the grid geometry and grid_num (TYPE_MAP where the mask says so) are set as initializeVIO /
// resetGrid / the retrieval would leave them, new_frame_ is a Frame of the image with updateFrameState(state), pg and
// visual_submap->add_from_voxel_map are filled, and the VisualPoints the call inserts are read back out of feat_map. What is not
// the reference's code: vikit (vk::shiTomasiScore and the camera models of the stand-ins in ref_shim/vikit/, restatements of the
// published algorithm). TEST INFRASTRUCTURE ONLY: pins the oracle's restatement (oracle/orc_generate.cpp) in
// tests/test_oracle_generate.py. Built by oracle/generate.mk where the reference source exists.
#include <algorithm>

#include "ref_vio.cpp"

extern "C" {

// Inputs as orc_generate_points. Outputs in cell order, room for grid_n_width * grid_n_height entries each: cell, pos (3), pc (2,
// the Feature's px_), score (scan_value of the cell), normal (3, VisualPoint::normal_), var (9, covariance_), patch (64, the
// Feature's patch_). Returns their number.
int ref_generate_points(void *h, const uint8_t *img, const double *state, const double *point_w, const double *normal, const double *var, int n,
                        const double *add_pos, const double *add_normal, int n_add, const uint8_t *type_map, int grid_size, int grid_n_width,
                        int grid_n_height, int border, int32_t *cell, double *pos, double *pc, float *score, double *normal_out, double *var_out,
                        float *patch) {
  RefVio *r = (RefVio *)h;
  VIOManager &v = r->v;
  for (auto &kv : v.feat_map) delete kv.second;  // ~VOXEL_POINTS deletes its points and their features
  v.feat_map.clear();
  v.grid_size = grid_size, v.grid_n_width = grid_n_width, v.grid_n_height = grid_n_height, v.border = border;
  v.length = grid_n_width * grid_n_height;
  v.grid_num.resize(v.length), v.map_index.resize(v.length), v.map_dist.resize(v.length), v.update_flag.resize(v.length), v.scan_value.resize(v.length);
  v.resetGrid();
  for (int i = 0; i < v.length; i++)
    if (type_map[i]) v.grid_num[i] = VIOManager::TYPE_MAP;
  unpack_state(state, r->st);
  cv::Mat im = cv::Mat(v.height, v.width, CV_8UC1, (void *)img).clone();
  v.new_frame_.reset(new Frame(v.cam, im));
  v.updateFrameState(r->st);
  vector<pointWithVar> pg(n);
  for (int i = 0; i < n; i++) {
    for (int k = 0; k < 3; k++) pg[i].point_w[k] = point_w[3 * i + k], pg[i].normal[k] = normal[3 * i + k];
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) pg[i].var(a, b) = var[9 * i + 3 * a + b];
  }
  v.visual_submap->reset();
  for (int j = 0; j < n_add; j++) {
    pointWithVar p;
    for (int k = 0; k < 3; k++) p.point_w[k] = add_pos[3 * j + k], p.normal[k] = add_normal[3 * j + k];
    v.visual_submap->add_from_voxel_map.push_back(p);
  }
  v.generateVisualMapPoints(im, pg);
  std::vector<std::pair<int, VisualPoint *>> got;
  for (auto &kv : v.feat_map)
    for (VisualPoint *p : kv.second->voxel_points) {
      const V2D px = p->obs_.front()->px_;
      got.emplace_back(static_cast<int>(px[1] / grid_size) * grid_n_width + static_cast<int>(px[0] / grid_size), p);  // :818
    }
  std::sort(got.begin(), got.end(), [](const std::pair<int, VisualPoint *> &a, const std::pair<int, VisualPoint *> &b) { return a.first < b.first; });
  for (size_t q = 0; q < got.size(); q++) {
    const int c = got[q].first;
    const VisualPoint *p = got[q].second;
    const Feature *f = p->obs_.front();
    cell[q] = c, score[q] = v.scan_value[c];
    for (int k = 0; k < 3; k++) pos[3 * q + k] = p->pos_[k], normal_out[3 * q + k] = p->normal_[k];
    pc[2 * q] = f->px_[0], pc[2 * q + 1] = f->px_[1];
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) var_out[9 * q + 3 * a + b] = p->covariance_(a, b);
    for (int k = 0; k < 64; k++) patch[64 * q + k] = f->patch_[k];
  }
  return (int)got.size();
}
}
