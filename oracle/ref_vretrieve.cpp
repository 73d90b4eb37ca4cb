// oracle/_ref — the reference's own VIOManager::insertPointIntoVoxelMap (src/vio.cpp:227-250) and resetGrid +
// retrieveFromVisualSparseMap (:162-177, 352-782) on one VIOManager kept across ticks (the driver ref_vio.cpp, included as it
// is): ref_vrt_place builds stand-in VisualPoints (pos_, normal_, is_normal_initialized_, obs_ of Features with the given
// patch_, id_ and T_f_w_) and inserts each with the reference's function; ref_vrt_feat_map reads feat_map back (keys and
// voxel_points order); ref_vrt_retrieve runs the retrieval with normal_en as given, ncc_en and raycast_en off and an outlier
// threshold of infinity, so every point past the depth check and the reference choice reaches visual_submap. Read back:
// sub_feat_map in iteration order, grid_num and retrieve_voxel_points per cell, visual_submap->voxel_points and the position
// of each survivor's ref_patch in its obs_. What is not the reference's code: vikit (the stand-ins in ref_shim/vikit/).
// TEST INFRASTRUCTURE ONLY: pins tests/vmap_retrieve_cases.py's restatement (tests/test_oracle_vmap_retrieve.py). Built by
// oracle/vmap_retrieve.mk where the reference source exists.
#include <iterator>
#include <limits>
#include <map>

#include "ref_vio.cpp"

namespace {
struct RefVrt {
  RefVio *r = nullptr;
  cv::Mat im;  // every Feature's img_
  std::map<const VisualPoint *, int> id;
};
}  // namespace

extern "C" {

void *ref_vrt_create(const double *cam, const double *extR, const double *extT, const double *Rcl, const double *Pcl, const double *cfg, const uint8_t *img) {
  RefVio *r = (RefVio *)ref_vio_create(cam, extR, extT, Rcl, Pcl, cfg);
  if (!r) return nullptr;
  RefVrt *h = new RefVrt;
  h->r = r;
  h->im = cv::Mat(r->v.height, r->v.width, CV_8UC1, (void *)img).clone();
  return h;
}
void ref_vrt_destroy(void *h) {
  RefVrt *t = (RefVrt *)h;
  ref_vio_destroy(t->r);  // the points stay allocated: feat_map's VOXEL_POINTS are not freed by ~VIOManager either
  delete t;
}

// n new points, point i with id ids[i], pos / normal (3 each), ninit, and the observations first[i] .. first[i + 1] - 1:
// patch (64 floats), id_ and T_f_w_ (R row-major, then t) each, in obs_ order; px_ is the image centre, level_ 0.
void ref_vrt_place(void *h, int n, const int32_t *ids, const double *pos, const double *normal, const uint8_t *ninit, const int32_t *first, const float *patch,
                   const int32_t *fid, const double *T) {
  RefVrt *t = (RefVrt *)h;
  VIOManager &v = t->r->v;
  for (int i = 0; i < n; i++) {
    VisualPoint *pt = new VisualPoint(V3D(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]));
    pt->normal_ = V3D(normal[3 * i], normal[3 * i + 1], normal[3 * i + 2]);
    pt->is_normal_initialized_ = ninit[i] != 0;
    for (int q = first[i]; q < first[i + 1]; q++) {
      M3D R;
      for (int k = 0; k < 9; k++) R(k / 3, k % 3) = T[12 * q + k];
      float *p = new float[64];
      for (int k = 0; k < 64; k++) p[k] = patch[64 * q + k];
      Feature *f = new Feature(pt, p, V2D(v.width / 2, v.height / 2), V3D(0, 0, 1), SE3(R, V3D(T[12 * q + 9], T[12 * q + 10], T[12 * q + 11])), 0);
      f->id_ = fid[q];
      f->img_ = t->im;
      pt->obs_.push_back(f);
    }
    t->id[pt] = ids[i];
    v.insertPointIntoVoxelMap(pt);
  }
}

// feat_map in its iteration order: keys (n_vox x 3; returns n_vox), first (n_vox + 1) and the point ids of each voxel_points
int ref_vrt_feat_map(void *h, int64_t *keys, int32_t *first, int32_t *ids) {
  RefVrt *t = (RefVrt *)h;
  int j = 0, q = 0;
  first[0] = 0;
  for (auto &kv : t->r->v.feat_map) {
    keys[3 * j] = kv.first.x, keys[3 * j + 1] = kv.first.y, keys[3 * j + 2] = kv.first.z;
    for (VisualPoint *pt : kv.second->voxel_points) ids[q++] = t->id[pt];
    first[++j] = q;
  }
  return j;
}

// One tick: the scan (point_w n x 3) at the packed state. Outputs: sub_keys (room for n x 3; returns their number), grid_type
// (length bytes, 1 = TYPE_MAP), cell_pt (length: the id of retrieve_voxel_points, -1 none), survivors (room for length: ids of
// visual_submap->voxel_points, *n_survivors of them) and ref (the position of each survivor's ref_patch in obs_, -1 none).
int ref_vrt_retrieve(void *h, const double *state, const double *point_w, int n, int grid_size, int grid_n_width, int grid_n_height, int border,
                     int normal_en, int64_t *sub_keys, uint8_t *grid_type, int32_t *cell_pt, int32_t *survivors, int32_t *ref, int32_t *n_survivors) {
  RefVrt *t = (RefVrt *)h;
  VIOManager &v = t->r->v;
  v.grid_size = grid_size, v.grid_n_width = grid_n_width, v.grid_n_height = grid_n_height, v.border = border;
  v.length = grid_n_width * grid_n_height;
  v.grid_num.resize(v.length), v.map_index.resize(v.length), v.map_dist.resize(v.length), v.update_flag.resize(v.length), v.scan_value.resize(v.length);
  v.border_flag.assign(v.length, 0);
  v.normal_en = normal_en != 0, v.ncc_en = false, v.raycast_en = false, v.outlier_threshold = std::numeric_limits<double>::infinity();
  unpack_state(state, t->r->st);
  v.new_frame_.reset(new Frame(v.cam, t->im));
  v.updateFrameState(t->r->st);
  vector<pointWithVar> pg(n);
  for (int i = 0; i < n; i++)
    for (int k = 0; k < 3; k++) pg[i].point_w[k] = point_w[3 * i + k];
  unordered_map<VOXEL_LOCATION, VoxelOctoTree *> plane_map;
  v.resetGrid();
  v.retrieveFromVisualSparseMap(t->im, pg, plane_map);
  int k = 0;
  for (auto &kv : v.sub_feat_map) sub_keys[3 * k] = kv.first.x, sub_keys[3 * k + 1] = kv.first.y, sub_keys[3 * k + 2] = kv.first.z, k++;
  for (int c = 0; c < v.length; c++) {
    grid_type[c] = v.grid_num[c] == VIOManager::TYPE_MAP;
    cell_pt[c] = (v.grid_num[c] == VIOManager::TYPE_MAP && v.retrieve_voxel_points[c]) ? t->id[v.retrieve_voxel_points[c]] : -1;
  }
  const std::vector<VisualPoint *> &sv = v.visual_submap->voxel_points;
  for (size_t q = 0; q < sv.size(); q++) {
    survivors[q] = t->id[sv[q]];
    ref[q] = -1;
    int j = 0;
    if (sv[q]->has_ref_patch_)
      for (auto it = sv[q]->obs_.begin(); it != sv[q]->obs_.end(); ++it, ++j)
        if (*it == sv[q]->ref_patch) ref[q] = j;
  }
  *n_survivors = (int32_t)sv.size();
  return k;
}
}
