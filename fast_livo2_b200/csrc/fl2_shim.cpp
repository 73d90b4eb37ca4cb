// fl2_shim.cpp — see fl2_shim.hpp. Host C++ only (no CUDA here): fills the reference-shaped member fields from / into
// the packed buffers of the C ABI (libesikf_b200.so, resolved at load time through the dynamic linker).
#include "fl2_shim.hpp"
#include "scratch_layout.hpp"

#include <omp.h>

#include <chrono>
#include <memory>

#include <cmath>
#include <cstring>

namespace fl2b200 {

// Host-side packing of the per-tick inputs into the page-locked staging buffers runs on a few threads (a num_threads clause, so
// nothing leaks into the process like the reference's omp_set_num_threads calls do): at 100 k points + 2 k patches the
// single-threaded copies were 0.29 ms of a 0.82 ms tick pair; 4 threads (the reference's MP_PROC_NUM) brought the pair to
// 0.71 ms, 8 are used since the copies are memory-bound and the GPU hosts have the cores.
#define FL2_PACK_THREADS 8
static void par_memcpy(void *dst, const void *src, size_t bytes) {
  const size_t chunk = 64 * 1024;
  const long n_chunks = (long)((bytes + chunk - 1) / chunk);
  if (n_chunks <= 2) {
    memcpy(dst, src, bytes);
    return;
  }
#pragma omp parallel for num_threads(FL2_PACK_THREADS) schedule(static)
  for (long c = 0; c < n_chunks; c++) {
    const size_t off = (size_t)c * chunk;
    memcpy(static_cast<char *>(dst) + off, static_cast<const char *>(src) + off, bytes - off < chunk ? bytes - off : chunk);
  }
}

// A manager's calls stage their inputs and answers in its one pinned block (scratch_layout.hpp), so no method may return with
// a copy from it queued. On success each ends in a synchronising call: the fetch of esikf_lio_update / esikf_vio_update /
// esikf_vio_run, the error check of the map updates, esikf_rgb_set_cloud, the export, or the front-end call itself. The
// exceptions are the early successful returns of the calls that upload a packed state (state_or_posterior in esikf_api_ctx.cu):
// GenerateVisualMapPoints at 10 points or fewer and ColorizeFrameWorld of an empty cloud (UpdateVisualMapPoints returns
// before update_points at no entries). They leave that upload queued into a device copy that every reader rewrites in stream
// order first, so what the block then holds is never read. esikf_lio_set_scan, esikf_vio_set_image and
// esikf_vio_set_patches return with their copies queued and a call failing part-way may skip its synchronisation, so Record
// drains the stream on every error; the first attempt of a grow-and-call-again loop fails only after its call synchronised.
template <typename F> static bool lay_out_staging(PinnedBuf<uint8_t> &block, F &&lay) {
  ScratchLayout s;
  lay(s);
  uint8_t *p = block.get(s.bytes);
  if (!p && s.bytes) return false;
  s = ScratchLayout{(uintptr_t)p};
  lay(s);
  return true;
}

// The guards of the managers' calls: false when the call has what it needs, else true with ESIKF_ERR_STATE and the call's
// message recorded. Every guarded call needs the device context; some also a state (VIOManager::state) or the device map.
static bool missing(CallStatus &c, const char *call, const esikf_ctx *ctx) {
  if (ctx) return false;
  c.last_status_ = ESIKF_ERR_STATE, c.last_error_ = std::string(call) + ": no device context";
  return true;
}
static bool missing(CallStatus &c, const char *call, const esikf_ctx *ctx, const StatesGroup *state) {
  if (ctx && state) return false;
  c.last_status_ = ESIKF_ERR_STATE, c.last_error_ = std::string(call) + ": no device context or state";
  return true;
}
static bool no_device_map(CallStatus &c, bool device_map, const char *error) {
  if (device_map) return false;
  c.last_status_ = ESIKF_ERR_STATE, c.last_error_ = error;
  return true;
}

StatesGroup::StatesGroup() {
  for (int i = 0; i < 361; i++) cov[i] = 0.0;
  for (int i = 0; i < 19; i++) cov[i * 19 + i] = 0.01;   // INIT_COV, include/common_lib.h:31,137
  cov[6 * 19 + 6] = 0.00001;                              // :138
  for (int i = 10; i < 19; i++) cov[i * 19 + i] = 0.00001;  // :139
}
void StatesGroup::pack(double *s) const {
  memcpy(s, rot_end.m, 9 * sizeof(double));
  memcpy(s + 9, pos_end.v, 3 * sizeof(double));
  s[12] = inv_expo_time;
  memcpy(s + 13, vel_end.v, 3 * sizeof(double));
  memcpy(s + 16, bias_g.v, 3 * sizeof(double));
  memcpy(s + 19, bias_a.v, 3 * sizeof(double));
  memcpy(s + 22, gravity.v, 3 * sizeof(double));
  memcpy(s + 25, cov, 361 * sizeof(double));
}
void StatesGroup::unpack(const double *s) {
  memcpy(rot_end.m, s, 9 * sizeof(double));
  memcpy(pos_end.v, s + 9, 3 * sizeof(double));
  inv_expo_time = s[12];
  memcpy(vel_end.v, s + 13, 3 * sizeof(double));
  memcpy(bias_g.v, s + 16, 3 * sizeof(double));
  memcpy(bias_a.v, s + 19, 3 * sizeof(double));
  memcpy(gravity.v, s + 22, 3 * sizeof(double));
  memcpy(cov, s + 25, 361 * sizeof(double));
}

pointWithVar::pointWithVar() {
  for (int i = 0; i < 9; i++) var_nostate.m[i] = body_var.m[i] = var.m[i] = point_crossmat.m[i] = 0.0;
}

// The plane fields a C ABI row (esikf_plane, esikf_map_node) shares with a VoxelPlane. The row holds plane_var_'s upper
// triangle, row by row (DESIGN.md §4): the layout the device map, its export and the oracle all read.
template <typename Row> static void plane_from_row(const Row &r, VoxelPlane &p) {
  for (int k = 0; k < 3; k++) p.center_[k] = r.center[k], p.normal_[k] = r.normal[k];
  for (int a = 0, t = 0; a < 6; a++)
    for (int b = a; b < 6; b++, t++) p.plane_var_[6 * a + b] = p.plane_var_[6 * b + a] = r.plane_var[t];
  p.d_ = r.d, p.radius_ = r.radius;
}
static void row_from_plane(const VoxelPlane &p, esikf_plane &r) {
  for (int k = 0; k < 3; k++) r.center[k] = p.center_[k], r.normal[k] = p.normal_[k];
  for (int a = 0, t = 0; a < 6; a++)
    for (int b = a; b < 6; b++, t++) r.plane_var[t] = p.plane_var_[6 * a + b];
  r.d = p.d_, r.radius = p.radius_;
}

VoxelOctoTree::~VoxelOctoTree() {
  for (int i = 0; i < 8; i++) delete leaves_[i];
  delete plane_ptr_;
}

// src/voxel_map.cpp:292-305
// The node a point falls into: descend while the node is a cut, non-plane node above the last layer and the point's leaf
// exists. The leaf is chosen by a strict comparison with the node's centre on each axis (x: 4, y: 2, z: 1).
VoxelOctoTree *VoxelOctoTree::find_correspond(V3D pw) {
  VoxelOctoTree *node = this;
  while (node->init_octo_ && !node->plane_ptr_->is_plane_ && node->layer_ < node->max_layer_) {
    const int leaf = (pw[0] > node->voxel_center_[0]) * 4 + (pw[1] > node->voxel_center_[1]) * 2 + (pw[2] > node->voxel_center_[2]);
    if (!node->leaves_[leaf]) break;
    node = node->leaves_[leaf];
  }
  return node;
}

bool ApplyMapExport(VoxelMap &map, const VoxelMapConfig &cfg, const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots, const esikf_map_node *nodes,
                    int n_nodes, std::string *err) {
  std::vector<VoxelOctoTree *> at;
  for (int r = 0; r < n_roots; r++) {
    const int f = first[r], c = count[r];
    if (f < 0 || c < 1 || f + c > n_nodes || nodes[f].parent != -1) {
      if (err) *err = "map export: root " + std::to_string(r) + " has no valid node range";
      return false;
    }
    const VOXEL_LOCATION key(keys[3 * r], keys[3 * r + 1], keys[3 * r + 2]);
    VoxelOctoTree *&root = map[key];
    if (!root) root = new VoxelOctoTree, root->plane_ptr_ = new VoxelPlane;
    at.assign(c, nullptr);
    for (int j = 0; j < c; j++) {
      const esikf_map_node &e = nodes[f + j];
      VoxelOctoTree *t = root;
      if (j > 0) {
        if (e.parent < 0 || e.parent >= j || e.leaf < 0 || e.leaf > 7) {
          if (err) *err = "map export: node " + std::to_string(f + j) + " does not follow its parent in DFS pre-order";
          return false;
        }
        VoxelOctoTree *&leaf = at[e.parent]->leaves_[e.leaf];
        if (!leaf) leaf = new VoxelOctoTree, leaf->plane_ptr_ = new VoxelPlane;
        t = leaf;
      }
      at[j] = t;
      t->layer_ = e.layer, t->max_layer_ = cfg.max_layer_;
      for (int k = 0; k < 3; k++) t->voxel_center_[k] = e.voxel_center[k];
      t->quater_length_ = e.quater_length;
      t->init_octo_ = e.init_octo != 0, t->octo_state_ = e.octo_state, t->update_enable_ = e.update_enable != 0;
      t->new_points_ = e.new_points, t->temp_points_size_ = e.temp_points;
      VoxelPlane &p = *t->plane_ptr_;
      plane_from_row(e, p);
      p.points_size_ = e.points_size;
      p.is_plane_ = e.is_plane != 0, p.is_init_ = e.points_size > 0;
    }
  }
  return true;
}

void EraseRootsOutside(VoxelMap &map, const int64_t lo[3], const int64_t hi[3]) {
  for (auto it = map.begin(); it != map.end();) {
    const VOXEL_LOCATION &loc = it->first;
    const bool should_remove = loc.x > hi[0] || loc.x < lo[0] || loc.y > hi[1] || loc.y < lo[1] || loc.z > hi[2] || loc.z < lo[2];
    if (should_remove) {
      delete it->second;
      it = map.erase(it);
    } else {
      ++it;
    }
  }
}

void ClearVoxelMap(VoxelMap &map) {
  for (auto &kv : map) delete kv.second;
  map.clear();
}

static void flatten_node(const VoxelOctoTree *node, int layer, int max_layer, int path, FlatVoxelMap &out) {
  if (node->plane_ptr_ && node->plane_ptr_->is_plane_) {
    const VoxelPlane &p = *node->plane_ptr_;
    esikf_plane f;
    memset(&f, 0, sizeof(f));
    row_from_plane(p, f);
    f.layer = layer;
    f.path = path;
    out.planes.push_back(f);
    out.plane_src.push_back(&p);
    return;
  }
  if (layer < max_layer)
    for (int l = 0; l < 8; l++)
      if (node->leaves_[l] != nullptr) flatten_node(node->leaves_[l], layer + 1, max_layer, path | (l << (3 * layer)), out);
}

bool FlattenVoxelMap(const VoxelMap &map, const VoxelMapConfig &cfg, FlatVoxelMap &out, std::string *err) {
  out.keys.clear(), out.first.clear(), out.count.clear(), out.planes.clear(), out.plane_src.clear();
  const float vs = (float)cfg.max_voxel_size_;
  for (const auto &kv : map) {
    const VoxelOctoTree *root = kv.second;
    if (!root) continue;
    // the device derives the root centre / quarter length from the key (src/voxel_map.cpp:578-581): check the host agrees
    const double c[3] = {(0.5 + kv.first.x) * vs, (0.5 + kv.first.y) * vs, (0.5 + kv.first.z) * vs};
    for (int k = 0; k < 3; k++)
      if (root->voxel_center_[k] != c[k] || root->quater_length_ != vs / 4) {
        if (err) *err = "root voxel centre / quarter length does not follow (0.5 + key) * voxel_size";
        return false;
      }
    out.keys.push_back(kv.first.x), out.keys.push_back(kv.first.y), out.keys.push_back(kv.first.z);
    out.first.push_back((int32_t)out.planes.size());
    flatten_node(root, 0, cfg.max_layer_, 0, out);
    out.count.push_back((int32_t)out.planes.size() - out.first.back());
  }
  return true;
}

bool DiffFlatVoxelMaps(const FlatVoxelMap &synced, const FlatVoxelMap &now, std::vector<int32_t> &changed_ids) {
  changed_ids.clear();
  if (synced.keys != now.keys || synced.first != now.first || synced.count != now.count || synced.planes.size() != now.planes.size()) return false;
  for (size_t i = 0; i < now.planes.size(); i++) {
    // layer / path are part of the record: a plane that moved inside its octree changes them and is patched like a refit
    if (memcmp(&synced.planes[i], &now.planes[i], sizeof(esikf_plane)) != 0) changed_ids.push_back((int32_t)i);
  }
  return true;
}

VoxelMapManager::VoxelMapManager(VoxelMapConfig &config_setting, VoxelMap &voxel_map, int device) : config_setting_(config_setting), voxel_map_(voxel_map) {
  last_status_ = esikf_create(&ctx_, device);
  if (last_status_ != 0) last_error_ = "esikf_create failed (no sm_90 CUDA device?) — there is no CPU fallback";
}
VoxelMapManager::~VoxelMapManager() { esikf_destroy(ctx_); }

void VoxelMapManager::SyncDeviceMap() {
  if (!ctx_) return;
  if (device_map_) {  // the device owns the map: nothing to mirror
    map_synced_ = true;
    return;
  }
  std::string err;
  FlatVoxelMap now;
  if (!FlattenVoxelMap(voxel_map_, config_setting_, now, &err)) {
    last_status_ = ESIKF_ERR_ARG, last_error_ = err;
    return;
  }
  std::vector<int32_t> ids;
  if (device_has_map_ && DiffFlatVoxelMaps(flat_, now, ids)) {
    // same roots and candidate lists as on the device: only the refitted records travel
    std::vector<esikf_plane> recs(ids.size());
    for (size_t k = 0; k < ids.size(); k++) recs[k] = now.planes[ids[k]];
    Record(ctx_, ids.empty() ? 0 : esikf_map_patch(ctx_, ids.data(), recs.data(), (int32_t)ids.size()));
    last_sync_patched_ = (int)ids.size();
  } else {
    Record(ctx_, esikf_map_upload(ctx_, now.keys.data(), now.first.data(), now.count.data(), (int32_t)now.first.size(), now.planes.data(),
                                  (int32_t)now.planes.size(), config_setting_.max_voxel_size_));
    last_sync_patched_ = -1;
  }
  if (last_status_) {
    device_has_map_ = false;  // unknown device state: the next sync uploads everything
  } else {
    flat_.keys.swap(now.keys), flat_.first.swap(now.first), flat_.count.swap(now.count), flat_.planes.swap(now.planes), flat_.plane_src.swap(now.plane_src);
    device_has_map_ = true;
  }
  map_synced_ = (last_status_ == 0);
}

void VoxelMapManager::EnableDeviceMap() {
  if (!ctx_) return;
  esikf_map_cfg m;
  memset(&m, 0, sizeof(m));
  m.voxel_size = config_setting_.max_voxel_size_, m.min_eigen_value = config_setting_.planner_threshold_;
  m.dept_err = config_setting_.dept_err_, m.beam_err = config_setting_.beam_err_;
  m.max_layer = config_setting_.max_layer_, m.max_points_num = config_setting_.max_points_num_;
  const std::vector<int> &lin = config_setting_.layer_init_num_;
  for (int k = 0; k < 8; k++) m.layer_init_num[k] = lin.empty() ? 5 : lin[k < (int)lin.size() ? k : (int)lin.size() - 1];
  m.root_capacity = config_setting_.device_root_capacity_;
  m.grow = config_setting_.device_map_grow_ ? 1 : 0;
  device_map_mirror_ = config_setting_.device_map_mirror_;
  if (device_map_mirror_) ClearVoxelMap(voxel_map_);  // the mirror starts as empty as the device map
  mirror_valid_ = false;
  if (Record(ctx_, esikf_map_device_init(ctx_, &m))) return;
  device_map_ = true, map_synced_ = true, device_has_map_ = true;
  mirror_valid_ = device_map_mirror_;
}

void VoxelMapManager::InvalidateMirror() {
  ClearVoxelMap(voxel_map_);
  mirror_valid_ = false;
}

// After a device build / update: apply its export to the mirror. An export holds only the roots of one tick, so once a tick
// is missing (a failed call, export or apply) no later export can complete the mirror: it stays empty and every later call
// reports so, until EnableDeviceMap() starts a new map that BuildVoxelMap() fills again.
void VoxelMapManager::UpdateMirror() {
  if (!device_map_mirror_) return;
  if (last_status_) return InvalidateMirror();
  if (!mirror_valid_) {
    last_status_ = ESIKF_ERR_STATE;
    last_error_ = "the host mirror of the device map is void since an earlier call failed: EnableDeviceMap() and BuildVoxelMap() rebuild it";
    return;
  }
  // one export call into room sized by the ticks before; a second one only when that is too small
  int32_t nr = 0, nn = 0;
  int64_t *keys; int32_t *first, *count; esikf_map_node *nodes;
  for (int attempt = 0; attempt < 2; attempt++) {
    auto lay = [&](ScratchLayout &s) {
      keys = s.take<int64_t>(3 * exp_roots_cap_), first = s.take<int32_t>(exp_roots_cap_), count = s.take<int32_t>(exp_roots_cap_), nodes = s.take<esikf_map_node>(exp_nodes_cap_);
    };
    if (!lay_out_staging(block_, lay)) {
      StagingFailed();
      return InvalidateMirror();
    }
    last_status_ = esikf_map_device_export(ctx_, keys, first, count, exp_roots_cap_, nodes, exp_nodes_cap_, &nr, &nn);
    if (last_status_ == 0 || (nr <= exp_roots_cap_ && nn <= exp_nodes_cap_)) break;
    exp_roots_cap_ = nr + nr / 4 + 64, exp_nodes_cap_ = nn + nn / 4 + 64;  // too small: grow and export again
  }
  if (Record(ctx_, last_status_)) return InvalidateMirror();
  if (!ApplyMapExport(voxel_map_, config_setting_, keys, first, count, nr, nodes, nn, &last_error_)) {
    last_status_ = ESIKF_ERR_STATE;
    return InvalidateMirror();
  }
}

// include/voxel_map.h:231 / src/voxel_map.cpp:532-591 with feats_down_world_ = transformLidar(state_) (LIVMapper.cpp:360)
void VoxelMapManager::BuildVoxelMap() {
  if (no_device_map(*this, ctx_ && device_map_, "BuildVoxelMap: EnableDeviceMap first (a host-owned voxel_map_ is built by the reference's own code)")) return;
  const int n = feats_down_size_;
  float *pts; double *sbuf;
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { pts = s.take<float>((size_t)n * 3 + 4), sbuf = s.take<double>(ESIKF_STATE_DOUBLES); })) return StagingFailed();
  if (n) par_memcpy(pts, &feats_down_body_[0].x, (size_t)n * 12);
  state_.pack(sbuf);
  if ((last_status_ = esikf_set_lidar_extrinsics(ctx_, extR_.m, extT_.v)) == 0 && (last_status_ = esikf_lio_set_scan(ctx_, pts, n)) == 0)
    last_status_ = esikf_map_device_build(ctx_, sbuf);
  Record(ctx_, last_status_);
  UpdateMirror();
}

// LIVMapper.cpp:413-424: pv_list_[i].point_w / .var with the posterior, then UpdateVoxelMap(pv_list_) — on the device
void VoxelMapManager::UpdateVoxelMap() {
  if (no_device_map(*this, ctx_ && device_map_, "UpdateVoxelMap(): EnableDeviceMap first")) return;
  double *sbuf;
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { sbuf = s.take<double>(ESIKF_STATE_DOUBLES); })) return StagingFailed();
  state_.pack(sbuf);  // _state == voxelmap_manager->state_ at this point of the tick (LIVMapper.cpp:371); 3 kB
  Record(ctx_, esikf_map_device_update(ctx_, sbuf));
  UpdateMirror();
}

void VoxelMapManager::SetWorldCloud(const std::vector<PointXYZ> *dense_scan) {
  if (missing(*this, "SetWorldCloud", ctx_)) return;
  const int n = dense_scan ? (int)dense_scan->size() : 0;
  double *sbuf; float *pts;
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { sbuf = s.take<double>(ESIKF_STATE_DOUBLES), pts = dense_scan ? s.take<float>((size_t)n * 3 + 3) : nullptr; }))
    return StagingFailed();
  state_.pack(sbuf);  // _state == state_ after StateEstimation (LIVMapper.cpp:371)
  for (int i = 0; i < n; i++) pts[3 * i] = (*dense_scan)[i].x, pts[3 * i + 1] = (*dense_scan)[i].y, pts[3 * i + 2] = (*dense_scan)[i].z;
  Record(ctx_, esikf_rgb_set_cloud(ctx_, pts, n, sbuf));
}

void VoxelMapManager::FindCorrespond(int n, const V3D *pts, int rule, uint8_t *status, VoxelPlane *planes) {
  if (no_device_map(*this, ctx_ && device_map_, "FindCorrespond: EnableDeviceMap first (a host-owned voxel_map_ is read by the reference's own code)")) return;
  if (n < 0 || (n > 0 && (!pts || !status || !planes))) {
    last_status_ = ESIKF_ERR_ARG, last_error_ = "FindCorrespond: bad argument";
    return;
  }
  double *p; int64_t *keys; uint8_t *st; esikf_plane *rows;
  auto lay = [&](ScratchLayout &s) { p = s.take<double>(3 * n + 3), st = s.take<uint8_t>(n + 1), keys = s.take<int64_t>(3 * n + 3), rows = s.take<esikf_plane>(n + 1); };
  if (!lay_out_staging(block_, lay)) return StagingFailed();
  for (int i = 0; i < n; i++)
    for (int k = 0; k < 3; k++) p[3 * i + k] = pts[i][k];
  if (Record(ctx_, esikf_map_device_find(ctx_, p, n, rule, st, keys, rows))) return;
  for (int i = 0; i < n; i++) {
    status[i] = st[i];
    VoxelPlane &o = planes[i];
    o = VoxelPlane();
    if (st[i] == ESIKF_FIND_NO_ROOT) continue;
    plane_from_row(rows[i], o);
    o.is_plane_ = st[i] == ESIKF_FIND_PLANE;
  }
}

// src/voxel_map.cpp:924-948: nothing until the sensor moved sliding_thresh, then roots further than half_map_size voxels go
void VoxelMapManager::mapSliding() {
  if (no_device_map(*this, ctx_ && device_map_, "mapSliding: EnableDeviceMap first (a host-owned voxel_map_ slides in the reference's own code)")) return;
  double d2 = 0;
  for (int k = 0; k < 3; k++) d2 += (position_last_[k] - last_slide_position[k]) * (position_last_[k] - last_slide_position[k]);
  if (sqrt(d2) < config_setting_.sliding_thresh) return;
  last_slide_position = position_last_;
  int64_t lo[3], hi[3];
  for (int j = 0; j < 3; j++) {
    float loc = (float)(position_last_[j] / config_setting_.max_voxel_size_);  // :938 (double quotient narrowed to float)
    if (loc < 0) loc -= 1.0;
    lo[j] = (int64_t)loc - config_setting_.half_map_size, hi[j] = (int64_t)loc + config_setting_.half_map_size;
  }
  Record(ctx_, esikf_map_device_slide(ctx_, lo, hi));
  if (device_map_mirror_) {
    if (last_status_) {
      InvalidateMirror();
    } else if (!mirror_valid_) {
      last_status_ = ESIKF_ERR_STATE;
      last_error_ = "the host mirror of the device map is void since an earlier call failed: EnableDeviceMap() and BuildVoxelMap() rebuild it";
    } else {
      EraseRootsOutside(voxel_map_, lo, hi);
    }
  }
}

// include/voxel_map.h:232 / src/voxel_map.cpp:609-641
void VoxelMapManager::UpdateVoxelMap(const std::vector<pointWithVar> &input_points) {
  if (no_device_map(*this, ctx_ && device_map_, "UpdateVoxelMap: EnableDeviceMap first")) return;
  const size_t n = input_points.size();
  double *pw, *var;
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { pw = s.take<double>(n * 3 + 1), var = s.take<double>(n * 9 + 1); })) return StagingFailed();
  for (size_t i = 0; i < n; i++) {
    for (int k = 0; k < 3; k++) pw[3 * i + k] = input_points[i].point_w[k];
    memcpy(var + 9 * i, input_points[i].var.m, 72);
  }
  Record(ctx_, esikf_map_device_update_points(ctx_, pw, var, (int32_t)n));
  UpdateMirror();
}

// include/voxel_map.h:229 / src/voxel_map.cpp:338-511
void VoxelMapManager::StateEstimation(StatesGroup &state_propagat) {
  if (!ctx_) return;
  if (!map_synced_) SyncDeviceMap();
  if (!map_synced_) return;
  // lidar -> imu extrinsics only: the camera part belongs to the VIOManager sharing this context (it must survive the LIO tick)
  if (Record(ctx_, esikf_set_lidar_extrinsics(ctx_, extR_.m, extT_.v))) return;
  const int n = feats_down_size_;
  esikf_lio_cfg cfg;
  cfg.voxel_size = config_setting_.max_voxel_size_, cfg.sigma_num = config_setting_.sigma_num_;
  cfg.dept_err = config_setting_.dept_err_, cfg.beam_err = config_setting_.beam_err_;
  cfg.max_layer = config_setting_.max_layer_, cfg.max_iterations = config_setting_.max_iterations_;
  double *sbuf;
  float *pts, *dis = st_dis_.get((size_t)n + 1);
  int32_t *match = st_match_.get((size_t)n + 1), *normal = st_normal_.get((size_t)n + 1);
  auto lay = [&](ScratchLayout &s) { sbuf = s.take<double>(3 * ESIKF_STATE_DOUBLES), pts = s.take<float>((size_t)n * 3 + 4); };
  if (!dis || !match || !normal || !lay_out_staging(block_, lay)) return StagingFailed();
  double *sin = sbuf, *sprop = sbuf + ESIKF_STATE_DOUBLES, *sout = sbuf + 2 * ESIKF_STATE_DOUBLES;
  state_.pack(sin);
  state_propagat.pack(sprop);
  esikf_lio_stats stats;
  static_assert(sizeof(PointXYZ) == 12, "xyz float32");
  if (n) par_memcpy(pts, &feats_down_body_[0].x, (size_t)n * 12);
  if (Record(ctx_, esikf_lio_update(ctx_, n ? pts : nullptr, n, sin, sprop, &cfg, sout, &stats, match, normal, dis))) return;
  state_.unpack(sout);                 // _state = voxelmap_manager->state_  (LIVMapper.cpp:371)
  position_last_ = state_.pos_end;     // src/voxel_map.cpp:492
  effct_feat_num_ = stats.iters > 0 ? stats.effct_feat_num[stats.iters - 1] : 0;
  last_iters_ = stats.iters;
  lists_pending_ = fill_point_lists_;
  if (fill_point_lists_ && !lazy_point_lists_) MaterializePointLists();
}

// body_cov_list_ / cross_mat_list_ (LIVMapper.cpp:418-419), pv_list_ (:372) and ptpl_list_ (:446) of the last StateEstimation
void VoxelMapManager::MaterializePointLists() {
  if (!ctx_ || !lists_pending_) return;
  lists_pending_ = false;
  const int n = feats_down_size_;
  const int32_t *match = st_match_.data(), *normal = st_normal_.data();
  const float *dis = st_dis_.data();
  double *bc, *cm, *dev_normals = nullptr;
  // with the device map no host VoxelPlane exists: pv.normal comes from the device records
  auto lay = [&](ScratchLayout &s) { bc = s.take<double>(9 * n + 1), cm = s.take<double>(9 * n + 1), dev_normals = device_map_ ? s.take<double>(3 * n + 2) : nullptr; };
  if (!lay_out_staging(block_, lay)) return StagingFailed();
  if (Record(ctx_, esikf_lio_fetch_point_cov(ctx_, bc, cm))) return;
  body_cov_list_.resize(n), cross_mat_list_.resize(n);
  pv_list_.resize(n);
  ptpl_list_.clear();
  if (device_map_ && Record(ctx_, esikf_lio_fetch_normals(ctx_, dev_normals))) return;
  const double *R = state_.rot_end.m;
  for (int i = 0; i < n; i++) {
    memcpy(body_cov_list_[i].m, &bc[(size_t)i * 9], 72);
    memcpy(cross_mat_list_[i].m, &cm[(size_t)i * 9], 72);
    pointWithVar &pv = pv_list_[i];
    pv = pointWithVar();  // the reference rebuilds pv_list_ from default-constructed elements every call (voxel_map.cpp:362-363)
    pv.point_b[0] = feats_down_body_[i].x, pv.point_b[1] = feats_down_body_[i].y, pv.point_b[2] = feats_down_body_[i].z;
    pv.body_var = body_cov_list_[i];
    // point_w / var are recomputed by the caller with the posterior state right after the call (LIVMapper.cpp:413-423);
    // point_w is provided here with the posterior pose for convenience.
    double pi[3], pw[3];
    for (int r = 0; r < 3; r++) pi[r] = extR_.m[3 * r] * pv.point_b[0] + extR_.m[3 * r + 1] * pv.point_b[1] + extR_.m[3 * r + 2] * pv.point_b[2] + extT_[r];
    for (int r = 0; r < 3; r++) pw[r] = R[3 * r] * pi[0] + R[3 * r + 1] * pi[1] + R[3 * r + 2] * pi[2] + state_.pos_end[r];
    for (int r = 0; r < 3; r++) pv.point_w[r] = (double)(float)pw[r];
    if (dev_normals) {
      for (int k = 0; k < 3; k++) pv.normal[k] = dev_normals[3 * (size_t)i + k];
      if (match[i] >= 0) {  // the plane's own fields stay on the device (esikf_map_device_download); what the tick produced is filled
        PointToPlane q;
        memset(q.plane_var_, 0, sizeof(q.plane_var_));
        q.point_b_ = pv.point_b, q.point_w_ = pv.point_w, q.normal_ = pv.normal, q.body_cov_ = pv.body_var;
        q.is_valid_ = true, q.dis_to_plane_ = dis[i];
        ptpl_list_.push_back(q);
      }
      continue;
    }
    if (normal[i] >= 0) pv.normal = flat_.plane_src[normal[i]]->normal_;  // pv.normal (voxel_map.cpp:744), zero if never matched
    if (match[i] >= 0) {
      const VoxelPlane &pl = *flat_.plane_src[match[i]];
      PointToPlane q;
      q.point_b_ = pv.point_b, q.point_w_ = pv.point_w, q.normal_ = pl.normal_, q.center_ = pl.center_;
      memcpy(q.plane_var_, pl.plane_var_, sizeof(q.plane_var_));
      q.body_cov_ = pv.body_var;
      q.layer_ = flat_.planes[match[i]].layer, q.d_ = pl.d_, q.is_valid_ = true, q.dis_to_plane_ = dis[i];
      ptpl_list_.push_back(q);
    }
  }
}

VIOManager::VIOManager(esikf_ctx *shared_ctx) : ctx_(shared_ctx) {}

void VIOManager::GenerateVisualMapPoints(const std::vector<uint8_t> &type_map, int grid_size, int grid_n_width, int grid_n_height, int border,
                                         const std::vector<pointWithVar> *pg, const std::vector<pointWithVar> *add_from_voxel_map,
                                         std::vector<NewVisualPoint> &new_points) {
  new_points.clear();
  if (missing(*this, "GenerateVisualMapPoints", ctx_, state)) return;
  const size_t n = pg ? pg->size() : 0, m = add_from_voxel_map ? add_from_voxel_map->size() : 0;
  const int cap = (int)type_map.size();  // at most one point per cell
  double *sbuf, *pw, *nv, *var, *ap, *an, *pos, *pc, *normal, *pvar;
  int32_t *src, *cell; float *score, *patch; uint8_t *cells;
  auto lay = [&](ScratchLayout &s) {
    sbuf = s.take<double>(ESIKF_STATE_DOUBLES), cells = s.take<uint8_t>(cap + 1);
    pw = s.take<double>(3 * n + 1), nv = s.take<double>(3 * n + 1), var = s.take<double>(9 * n + 1), ap = s.take<double>(3 * m + 1), an = s.take<double>(3 * m + 1);
    src = s.take<int32_t>(cap + 1), cell = s.take<int32_t>(cap + 1), pos = s.take<double>(3 * cap + 3), pc = s.take<double>(2 * cap + 2);
    normal = s.take<double>(3 * cap + 3), pvar = s.take<double>(9 * cap + 9), score = s.take<float>(cap + 1), patch = s.take<float>(64 * cap + 64);
  };
  if (!lay_out_staging(block_, lay)) return StagingFailed();
  state->pack(sbuf);
  memcpy(cells, type_map.data(), cap);
  for (size_t i = 0; i < n; i++) {
    const pointWithVar &p = (*pg)[i];
    for (int k = 0; k < 3; k++) pw[3 * i + k] = p.point_w[k], nv[3 * i + k] = p.normal[k];
    memcpy(var + 9 * i, p.var.m, 72);
  }
  for (size_t j = 0; j < m; j++)
    for (int k = 0; k < 3; k++) ap[3 * j + k] = (*add_from_voxel_map)[j].point_w[k], an[3 * j + k] = (*add_from_voxel_map)[j].normal[k];
  int32_t k = 0;
  if (Record(ctx_, esikf_vio_generate_points(ctx_, pg ? pw : nullptr, nv, var, (int32_t)n, ap, an, (int32_t)m, cells, cap, grid_size, grid_n_width, grid_n_height, border,
                                             sbuf, cap, &k, src, cell, pos, pc, score, normal, pvar, patch)))
    return;
  new_points.resize(k);
  for (int i = 0; i < k; i++) {
    NewVisualPoint &q = new_points[i];
    q.source = src[i], q.cell = cell[i], q.score = score[i];
    memcpy(q.pos, pos + 3 * i, sizeof(q.pos)), memcpy(q.pc, pc + 2 * i, sizeof(q.pc)), memcpy(q.normal, normal + 3 * i, sizeof(q.normal));
    memcpy(q.var, pvar + 9 * i, sizeof(q.var)), memcpy(q.patch, patch + 64 * i, sizeof(q.patch));
  }
}

void VIOManager::UpdateVisualMapPoints(const std::vector<uint8_t> &converged, const std::vector<LastObservation> &last_obs, std::vector<uint8_t> &update_flag,
                                       std::vector<NewObservation> &new_obs) {
  new_obs.clear();
  if (missing(*this, "UpdateVisualMapPoints", ctx_, state)) return;
  update_flag.assign(total_points > 0 ? total_points : 0, 0);
  if (total_points <= 0) {  // src/vio.cpp:910
    last_status_ = ESIKF_OK;
    return;
  }
  if (converged.size() != (size_t)total_points || last_obs.size() != (size_t)total_points) {
    last_status_ = ESIKF_ERR_ARG, last_error_ = "UpdateVisualMapPoints: converged / last_obs must have total_points entries";
    return;
  }
  const size_t n = last_obs.size();
  double *sbuf, *T, *px, *pc; uint8_t *conv, *flag; int32_t *entry; float *patch;
  auto lay = [&](ScratchLayout &s) {
    sbuf = s.take<double>(ESIKF_STATE_DOUBLES), conv = s.take<uint8_t>(n), T = s.take<double>(12 * n), px = s.take<double>(2 * n);
    flag = s.take<uint8_t>(n), entry = s.take<int32_t>(n + 1), pc = s.take<double>(2 * n + 2), patch = s.take<float>(64 * n + 64);
  };
  if (!lay_out_staging(block_, lay)) return StagingFailed();
  state->pack(sbuf);
  memcpy(conv, converged.data(), n);
  for (size_t i = 0; i < n; i++) memcpy(T + 12 * i, last_obs[i].T_f_w, sizeof(last_obs[i].T_f_w)), memcpy(px + 2 * i, last_obs[i].px, sizeof(last_obs[i].px));
  int32_t k = 0;
  if (Record(ctx_, esikf_vio_update_points(ctx_, (int32_t)n, conv, T, px, sbuf, (int32_t)n, &k, flag, entry, pc, patch))) return;
  memcpy(update_flag.data(), flag, n);
  new_obs.resize(k);
  for (int i = 0; i < k; i++) {
    NewObservation &q = new_obs[i];
    q.entry = entry[i];
    memcpy(q.pc, pc + 2 * i, sizeof(q.pc)), memcpy(q.patch, patch + 64 * i, sizeof(q.patch));
  }
}

void VIOManager::RetrieveScanVoxels(int border, const std::vector<pointWithVar> *pg, std::vector<VOXEL_LOCATION> &keys) {
  keys.clear();
  if (missing(*this, "RetrieveScanVoxels", ctx_, state)) return;
  const size_t n = pg ? pg->size() : 0;
  // room for one key per point of a host scan; for the resident scan a first call reports the count when the room is short
  int32_t cap = pg ? (int32_t)n : (int32_t)(keys_cap_ > 0 ? keys_cap_ : 1 << 16), k = -1;
  double *sbuf, *pw; int32_t *kb;
  auto lay = [&](ScratchLayout &s) { sbuf = s.take<double>(ESIKF_STATE_DOUBLES), pw = s.take<double>(3 * n + 3), kb = s.take<int32_t>(3 * (size_t)cap + 3); };
  if (!lay_out_staging(block_, lay)) return StagingFailed();
  state->pack(sbuf);
  for (size_t i = 0; i < n; i++)
    for (int k = 0; k < 3; k++) pw[3 * i + k] = (*pg)[i].point_w[k];
  last_status_ = esikf_vio_retrieve_scan(ctx_, pg ? pw : nullptr, (int32_t)n, border, sbuf, cap, &k, kb, nullptr);
  if (last_status_ == ESIKF_ERR_ARG && !pg && k > cap) {
    cap = k, keys_cap_ = k;
    if (!lay_out_staging(block_, lay)) return StagingFailed();
    state->pack(sbuf);
    last_status_ = esikf_vio_retrieve_scan(ctx_, nullptr, 0, border, sbuf, cap, &k, kb, nullptr);
  }
  if (Record(ctx_, last_status_)) return;
  keys.resize(k);
  for (int i = 0; i < k; i++) keys[i] = VOXEL_LOCATION(kb[3 * i], kb[3 * i + 1], kb[3 * i + 2]);
}

void VIOManager::CheckDepthContinuity(int n, const double *pos, const double *pc, std::vector<uint8_t> &discontinuous) {
  discontinuous.assign(n > 0 ? n : 0, 0);
  if (missing(*this, "CheckDepthContinuity", ctx_)) return;
  if (n <= 0) {
    last_status_ = n < 0 ? ESIKF_ERR_ARG : ESIKF_OK;
    return;
  }
  double *cb; uint8_t *fb;
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { cb = s.take<double>(5 * (size_t)n), fb = s.take<uint8_t>(n); })) return StagingFailed();
  memcpy(cb, pos, 3 * (size_t)n * sizeof(double)), memcpy(cb + 3 * (size_t)n, pc, 2 * (size_t)n * sizeof(double));
  if (Record(ctx_, esikf_vio_depth_check(ctx_, n, cb, cb + 3 * (size_t)n, fb))) return;
  memcpy(discontinuous.data(), fb, (size_t)n);
}

void VIOManager::ScoreReferencePatches(const std::vector<int32_t> &first, const std::vector<ScoredPoint> &pts, const std::vector<PatchObservation> &obs,
                                       std::vector<float> &score, std::vector<float> &mean, std::vector<int32_t> &ref) {
  if (missing(*this, "ScoreReferencePatches", ctx_)) return;
  if (first.size() != pts.size() + 1) {
    last_status_ = ESIKF_ERR_ARG, last_error_ = "ScoreReferencePatches: first must have pts.size() + 1 entries";
    return;
  }
  const size_t n = pts.size(), m = obs.size();
  double *d;  // pos 3n | normal 3n | T_f_w 12m, then by element type patch 64m | mean m | score m | mean_out m and first n + 1 | id m | ref n
  float *f; int32_t *k;
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { d = s.take<double>(6 * n + 12 * m), f = s.take<float>(67 * m), k = s.take<int32_t>(2 * n + 1 + m); }))
    return StagingFailed();
  float *sc = f + 65 * m, *mu = f + 66 * m;
  int32_t *rf = k + n + 1 + m;
  if (n == 0) memset(sc, 0, 2 * m * sizeof(float));  // the call answers nothing: zero scores and means, as many as observations
  memcpy(k, first.data(), (n + 1) * sizeof(int32_t));
  for (size_t i = 0; i < n; i++) memcpy(d + 3 * i, pts[i].pos, sizeof(pts[i].pos)), memcpy(d + 3 * n + 3 * i, pts[i].normal, sizeof(pts[i].normal));
  for (size_t j = 0; j < m; j++) {
    memcpy(d + 6 * n + 12 * j, obs[j].T_f_w, sizeof(obs[j].T_f_w)), memcpy(f + 64 * j, obs[j].patch, sizeof(obs[j].patch));
    f[64 * m + j] = obs[j].mean, k[n + 1 + j] = obs[j].id;
  }
  if (Record(ctx_, esikf_vio_score_ref_patches(ctx_, (int32_t)n, k, (int32_t)m, d, d + 3 * n, f, f + 64 * m, k + n + 1, d + 6 * n, sc, mu, rf))) return;
  score.assign(sc, sc + m), mean.assign(mu, mu + m), ref.assign(rf, rf + n);
}

void VIOManager::EnableDeviceObservations(int64_t capacity) {
  if (missing(*this, "EnableDeviceObservations", ctx_)) return;
  Record(ctx_, esikf_vmap_init(ctx_, capacity));
}

void VIOManager::AddVisualPoints(const std::vector<int32_t> &first, const std::vector<StoredObservation> &obs, const std::vector<int32_t> &ref,
                                 std::vector<int32_t> &point_ids) {
  point_ids.clear();
  if (missing(*this, "AddVisualPoints", ctx_)) return;
  if (first.size() != ref.size() + 1) {
    last_status_ = ESIKF_ERR_ARG, last_error_ = "AddVisualPoints: first must have ref.size() + 1 entries";
    return;
  }
  const size_t n = ref.size(), m = obs.size();
  double *d;  // px 2m | T_f_w 12m, then patch 64m | mean m | score m, then first n + 1 | id m | ref n | ids n
  float *f; int32_t *k;
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { d = s.take<double>(14 * m), f = s.take<float>(66 * m), k = s.take<int32_t>(3 * n + 1 + m); }))
    return StagingFailed();
  int32_t *id = k + n + 1, *rf = id + m, *ids = rf + n;
  memcpy(k, first.data(), (n + 1) * sizeof(int32_t)), memcpy(rf, ref.data(), n * sizeof(int32_t));
  for (size_t j = 0; j < m; j++) {
    memcpy(d + 2 * j, obs[j].px, sizeof(obs[j].px)), memcpy(d + 2 * m + 12 * j, obs[j].T_f_w, sizeof(obs[j].T_f_w));
    memcpy(f + 64 * j, obs[j].patch, sizeof(obs[j].patch));
    f[64 * m + j] = obs[j].mean, f[65 * m + j] = obs[j].score, id[j] = obs[j].id;
  }
  if (Record(ctx_, esikf_vmap_add_points(ctx_, (int32_t)n, k, (int32_t)m, d, f, d + 2 * m, id, f + 64 * m, f + 65 * m, rf, ids))) return;
  point_ids.assign(ids, ids + n);
}

void VIOManager::UpdateVisualMapPoints(const std::vector<int32_t> &point_ids, const std::vector<uint8_t> &converged, int32_t frame_id,
                                       std::vector<uint8_t> &update_flag, std::vector<NewObservation> &new_obs, std::vector<int32_t> &evicted,
                                       std::vector<int32_t> &count) {
  new_obs.clear();
  if (missing(*this, "UpdateVisualMapPoints", ctx_, state)) return;
  const int n = total_points > 0 ? total_points : 0;
  update_flag.assign(n, 0), evicted.assign(n, -1), count.assign(n, 0);
  if (point_ids.size() != (size_t)n || converged.size() != (size_t)n) {
    last_status_ = ESIKF_ERR_ARG, last_error_ = "UpdateVisualMapPoints: point_ids / converged must have total_points entries";
    return;
  }
  if (n == 0) {  // src/vio.cpp:910
    last_status_ = ESIKF_OK;
    return;
  }
  const size_t N = (size_t)n;
  double *sbuf, *pc; uint8_t *conv, *flag; int32_t *pid, *entry, *ev, *cnt; float *patch;
  auto lay = [&](ScratchLayout &s) {
    sbuf = s.take<double>(ESIKF_STATE_DOUBLES), pid = s.take<int32_t>(N), conv = s.take<uint8_t>(N), flag = s.take<uint8_t>(N);
    entry = s.take<int32_t>(N), ev = s.take<int32_t>(N), cnt = s.take<int32_t>(N), pc = s.take<double>(2 * N), patch = s.take<float>(64 * N);
  };
  if (!lay_out_staging(block_, lay)) return StagingFailed();
  state->pack(sbuf);
  memcpy(pid, point_ids.data(), N * sizeof(int32_t)), memcpy(conv, converged.data(), N);
  int32_t k = 0;
  if (Record(ctx_, esikf_vmap_update_points(ctx_, n, pid, conv, nullptr, frame_id, sbuf, n, &k, flag, entry, pc, patch, ev, cnt))) return;
  memcpy(update_flag.data(), flag, N), memcpy(evicted.data(), ev, N * sizeof(int32_t)), memcpy(count.data(), cnt, N * sizeof(int32_t));
  new_obs.resize(k);
  for (int i = 0; i < k; i++) {
    NewObservation &q = new_obs[i];
    q.entry = entry[i];
    memcpy(q.pc, pc + 2 * i, sizeof(q.pc)), memcpy(q.patch, patch + 64 * i, sizeof(q.patch));
  }
}

void VIOManager::ScoreReferencePatches(const std::vector<int32_t> &point_ids, const std::vector<ScoredPoint> &pts, std::vector<int32_t> &ref) {
  ref.clear();
  if (missing(*this, "ScoreReferencePatches", ctx_)) return;
  if (point_ids.size() != pts.size()) {
    last_status_ = ESIKF_ERR_ARG, last_error_ = "ScoreReferencePatches: point_ids and pts differ in size";
    return;
  }
  const size_t n = pts.size();
  double *d; int32_t *k;  // pos 3n | normal 3n, then point_ids n | ref n
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { d = s.take<double>(6 * n), k = s.take<int32_t>(2 * n); })) return StagingFailed();
  memcpy(k, point_ids.data(), n * sizeof(int32_t));
  for (size_t i = 0; i < n; i++) memcpy(d + 3 * i, pts[i].pos, sizeof(pts[i].pos)), memcpy(d + 3 * n + 3 * i, pts[i].normal, sizeof(pts[i].normal));
  if (Record(ctx_, esikf_vmap_score(ctx_, (int32_t)n, k, d, d + 3 * n, k + n, nullptr, nullptr))) return;
  ref.assign(k + n, k + 2 * n);
}

void VIOManager::ChooseReferenceFeatures(const std::vector<int32_t> &point_ids, const double *pos, const double frame_pos[3], bool normal_en,
                                         std::vector<int32_t> &ref) {
  ref.clear();
  if (missing(*this, "ChooseReferenceFeatures", ctx_)) return;
  const size_t n = point_ids.size();
  double *d; int32_t *k;  // pos 3n | frame_pos 3, then point_ids n | ref n
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { d = s.take<double>(3 * n + 3), k = s.take<int32_t>(2 * n); })) return StagingFailed();
  memcpy(k, point_ids.data(), n * sizeof(int32_t));
  if (pos) memcpy(d, pos, 3 * n * sizeof(double));
  if (frame_pos) memcpy(d + 3 * n, frame_pos, 3 * sizeof(double));
  if (Record(ctx_, esikf_vmap_choose_ref(ctx_, (int32_t)n, k, pos ? d : nullptr, frame_pos ? d + 3 * n : nullptr, normal_en ? 1 : 0, k + n))) return;
  ref.assign(k + n, k + 2 * n);
}

void VIOManager::initializeVIO() {
  if (!ctx_) return;
  esikf_extrinsics ext;
  memcpy(ext.extR, extR.m, sizeof(ext.extR));
  memcpy(ext.extT, extT.v, sizeof(ext.extT));
  memcpy(ext.Rcl, Rcl.m, sizeof(ext.Rcl));
  memcpy(ext.Pcl, Pcl.v, sizeof(ext.Pcl));
  last_status_ = esikf_set_extrinsics(ctx_, &ext);
  esikf_vio_cfg cfg;
  cfg.img_point_cov = img_point_cov, cfg.patch_pyrimid_level = patch_pyrimid_level, cfg.max_iterations = max_iterations;
  cfg.exposure_estimate_en = exposure_estimate_en ? 1 : 0, cfg.inverse_composition_en = 0;
  if (!last_status_) last_status_ = esikf_vio_set_camera(ctx_, &cam, &cfg);
  Record(ctx_, last_status_);
}

// include/vio.h:153 / src/vio.cpp:784-802
void VIOManager::computeJacobianAndUpdateEKF(const GrayImage &img) {
  if (!ctx_ || !state || !state_propagat || !visual_submap) return;
  if (total_points == 0) return;  // src/vio.cpp:786
  const int n = total_points, L = patch_pyrimid_level;
  if (visual_submap == selected_submap_ && n == selected_count_) {
    // the sub-map SelectSubSparseMap installed is still on the device: image and states only
    double *sbuf; float *err;
    if (!lay_out_staging(block_, [&](ScratchLayout &s) { sbuf = s.take<double>(3 * ESIKF_STATE_DOUBLES), err = s.take<float>(n); })) return StagingFailed();
    double *sin = sbuf, *sprop = sbuf + ESIKF_STATE_DOUBLES, *sout = sbuf + 2 * ESIKF_STATE_DOUBLES;
    state->pack(sin);
    state_propagat->pack(sprop);
    esikf_vio_stats stats;
    last_status_ = esikf_vio_set_image(ctx_, img.data, img.cols, img.rows);
    patch_img_ = nullptr;
    if (!last_status_) last_status_ = esikf_vio_run(ctx_, sin, sprop);
    if (!last_status_) last_status_ = esikf_vio_fetch(ctx_, sout, &stats, err);
    if (Record(ctx_, last_status_)) return;
    visual_submap->errors.assign(err, err + n);
    state->unpack(sout);
    last_total_iters_ = stats.total_iters;
    return;
  }
  double *pos, *ie, *sbuf; float *wp, *err; int32_t *sl; uint8_t *im;
  auto lay = [&](ScratchLayout &s) {
    pos = s.take<double>((size_t)n * 3), ie = s.take<double>(n), sbuf = s.take<double>(3 * ESIKF_STATE_DOUBLES), wp = s.take<float>((size_t)n * 64 * L);
    err = s.take<float>(n), sl = s.take<int32_t>(n), im = s.take<uint8_t>((size_t)img.cols * img.rows);
  };
  if (!lay_out_staging(block_, lay)) return StagingFailed();
  const SubSparseMap &sub = *visual_submap;
#pragma omp parallel for num_threads(FL2_PACK_THREADS) schedule(static) if (n > 256)
  for (int i = 0; i < n; i++) {
    for (int k = 0; k < 3; k++) pos[(size_t)3 * i + k] = sub.voxel_points_pos[i][k];
    memcpy(&wp[(size_t)i * 64 * L], sub.warp_patch[i].data(), sizeof(float) * 64 * L);
    sl[i] = visual_submap->search_levels[i];
    ie[i] = visual_submap->inv_expo_list[i];
  }
  par_memcpy(im, img.data, (size_t)img.cols * img.rows);
  double *sin = sbuf, *sprop = sbuf + ESIKF_STATE_DOUBLES, *sout = sbuf + 2 * ESIKF_STATE_DOUBLES;
  state->pack(sin);
  state_propagat->pack(sprop);
  esikf_vio_stats stats;
  patch_img_ = nullptr;  // the update installs its own current image
  last_status_ = esikf_vio_update(ctx_, im, img.cols, img.rows, pos, wp, sl, ie, n, sin, sprop, sout, &stats, err);
  selected_submap_ = nullptr, selected_count_ = -1;  // the device now holds this upload
  submap_uploads_++;
  if (Record(ctx_, last_status_)) return;
  visual_submap->errors.assign(err, err + n);
  state->unpack(sout);
  last_total_iters_ = stats.total_iters;
}

// include/vio.h:151 / src/vio.cpp:203-225: writes patch_tmp[patch_size_total * level + row * patch_size + col]
void VIOManager::getImagePatch(const GrayImage &img, const double pc[2], float *patch_tmp, int level) {
  if (!ctx_ || !img.data || !pc || !patch_tmp) return;
  last_status_ = 0;
  if (img.data != patch_img_ || img.cols != patch_img_w_ || img.rows != patch_img_h_) {
    last_status_ = esikf_vio_set_image(ctx_, img.data, img.cols, img.rows);
    patch_img_ = last_status_ ? nullptr : img.data, patch_img_w_ = img.cols, patch_img_h_ = img.rows;
  }
  float out[64];
  if (!last_status_) last_status_ = esikf_vio_get_image_patch(ctx_, pc, 1, level, out);
  if (Record(ctx_, last_status_)) return;
  memcpy(patch_tmp + 64 * level, out, sizeof(out));
}

// include/vio.h:161-162 / src/vio.cpp:292-318: writes patch[patch_size_total * pyramid_level + y * patch_size + x].
// level_ref is unused by the reference as well; halfpatch_size must be 4 (patch_size 8).
void VIOManager::warpAffine(const double A_cur_ref[4], const GrayImage &img_ref, const double px_ref[2], int level_ref, int search_level, int pyramid_level,
                            int halfpatch_size, float *patch) {
  (void)level_ref;
  if (!ctx_ || !img_ref.data || !A_cur_ref || !px_ref || !patch) return;
  if (halfpatch_size != 4 || pyramid_level < 0 || pyramid_level >= patch_pyrimid_level) {
    last_status_ = ESIKF_ERR_ARG;
    last_error_ = "warpAffine: halfpatch_size must be 4 and pyramid_level inside the pyramid";
    return;
  }
  last_status_ = 0;
  if (img_ref.data != patch_ref_img_ || img_ref.cols != patch_ref_w_ || img_ref.rows != patch_ref_h_) {
    const uint8_t *imgs[1] = {img_ref.data};
    last_status_ = esikf_vio_set_ref_images(ctx_, imgs, 1, img_ref.cols, img_ref.rows);
    patch_ref_img_ = last_status_ ? nullptr : img_ref.data, patch_ref_w_ = img_ref.cols, patch_ref_h_ = img_ref.rows;
    ref_imgs_current_ = false;
  }
  float *all;
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { all = s.take<float>(64 * patch_pyrimid_level); })) return StagingFailed();
  const int32_t idx = 0, sl = search_level;
  if (!last_status_) last_status_ = esikf_vio_warp_affine(ctx_, 1, &idx, px_ref, A_cur_ref, &sl, all);
  if (Record(ctx_, last_status_)) return;
  // a singular A leaves the patch untouched in the reference (vio.cpp:297-301); the kernel writes zeros into its own
  // scratch in that case, so only copy when A is invertible
  const double det = A_cur_ref[0] * A_cur_ref[3] - A_cur_ref[1] * A_cur_ref[2];
  const double inv_det = 1.0 / det;
  const float inv00 = (float)(A_cur_ref[3] * inv_det);  // same expression as the kernel's A_ref_cur(0, 0)
  if (inv00 != inv00) return;
  memcpy(patch + 64 * pyramid_level, all + 64 * pyramid_level, sizeof(float) * 64);
}

void VIOManager::SetReferenceImages(const GrayImage *imgs, int n) {
  if (!ctx_) return;
  std::vector<const uint8_t *> ptrs;
  for (int k = 0; k < n; k++) ptrs.push_back(imgs[k].data);
  last_status_ = n > 0 ? esikf_vio_set_ref_images(ctx_, ptrs.data(), n, imgs[0].cols, imgs[0].rows) : ESIKF_ERR_ARG;
  ref_imgs_.assign(imgs, imgs + (n > 0 ? n : 0));
  ref_imgs_current_ = last_status_ == 0;
  patch_ref_img_ = nullptr;  // the per-patch warpAffine uploads its own image again
  if (last_status_) last_error_ = n > 0 ? esikf_last_error(ctx_) : "SetReferenceImages: no image";
}

void VIOManager::ColorizeFrameWorld(const BgrImage &img_rgb, double blind_rgb_points, std::vector<PointXYZRGB> &laserCloudWorldRGB) {
  laserCloudWorldRGB.clear();
  if (missing(*this, "ColorizeFrameWorld", ctx_, state)) return;
  int32_t kept = 0;
  double *sbuf; float *xyz; uint8_t *bgr;
  // room for the largest coloured scan seen so far; a larger one is computed again with more room
  for (int attempt = 0; attempt < 2; attempt++) {
    auto lay = [&](ScratchLayout &s) { sbuf = s.take<double>(ESIKF_STATE_DOUBLES), xyz = s.take<float>((size_t)rgb_cap_ * 3 + 3), bgr = s.take<uint8_t>((size_t)rgb_cap_ * 3 + 3); };
    if (!lay_out_staging(block_, lay)) return StagingFailed();
    state->pack(sbuf);
    last_status_ = esikf_rgb_colorize(ctx_, img_rgb.data, img_rgb.cols, img_rgb.rows, sbuf, blind_rgb_points, rgb_cap_, &kept, xyz, bgr, nullptr);
    if (last_status_ == ESIKF_ERR_ARG && kept > rgb_cap_) {
      rgb_cap_ = kept;
      continue;
    }
    if (Record(ctx_, last_status_)) return;
    laserCloudWorldRGB.resize(kept);
    for (int i = 0; i < kept; i++) {
      PointXYZRGB &p = laserCloudWorldRGB[i];
      p.x = xyz[3 * i], p.y = xyz[3 * i + 1], p.z = xyz[3 * i + 2];
      p.b = bgr[3 * i], p.g = bgr[3 * i + 1], p.r = bgr[3 * i + 2];
    }
    return;
  }
}

void VIOManager::SelectSubSparseMap(const SubMapCandidate *c, int n, const GrayImage &img, const double T_cur_w[12]) {
  if (!ctx_ || !state || !visual_submap || n < 0 || (n > 0 && !c) || !T_cur_w) return;
  selected_submap_ = nullptr, selected_count_ = -1;
  last_status_ = ref_imgs_current_ ? 0 : ESIKF_ERR_STATE;
  if (last_status_) {
    last_error_ = "SelectSubSparseMap before SetReferenceImages";
    return;
  }
  last_status_ = esikf_vio_set_image(ctx_, img.data, img.cols, img.rows);
  patch_img_ = last_status_ ? nullptr : img.data, patch_img_w_ = img.cols, patch_img_h_ = img.rows;
  const size_t N = (size_t)n;
  int32_t *idx, *lvl, *key, *kept, *sl;
  double *px, *f, *rp, *pw, *nw, *T, *ie, *pc, *A; float *err;
  auto lay = [&](ScratchLayout &s) {
    idx = s.take<int32_t>(N), lvl = s.take<int32_t>(N), key = s.take<int32_t>(N), kept = s.take<int32_t>(N), sl = s.take<int32_t>(N);
    px = s.take<double>(2 * N), f = s.take<double>(3 * N), rp = s.take<double>(3 * N), pw = s.take<double>(3 * N), nw = s.take<double>(3 * N);
    T = s.take<double>(12 * N), ie = s.take<double>(N), pc = s.take<double>(2 * N), A = s.take<double>(4 * N), err = s.take<float>(N);
  };
  if (!lay_out_staging(block_, lay)) return StagingFailed();
  for (size_t i = 0; i < N; i++) {
    idx[i] = c[i].ref_img_index, lvl[i] = c[i].ref_level, key[i] = c[i].ref_key, ie[i] = c[i].ref_inv_expo;
    memcpy(px + 2 * i, c[i].px_ref, 16), memcpy(pc + 2 * i, c[i].pc, 16), memcpy(T + 12 * i, c[i].T_ref_w, 96);
    memcpy(f + 3 * i, c[i].ref_f, 24), memcpy(rp + 3 * i, c[i].ref_pos, 24), memcpy(pw + 3 * i, c[i].pos_w, 24), memcpy(nw + 3 * i, c[i].normal_w, 24);
  }
  esikf_vio_select_cfg cfg;
  cfg.normal_en = normal_en ? 1 : 0, cfg.ncc_en = ncc_en ? 1 : 0, cfg.ncc_thre = ncc_thre, cfg.outlier_threshold = outlier_threshold;
  int32_t nk = 0;
  if (!last_status_)
    last_status_ = esikf_vio_select_patches(ctx_, n, idx, px, lvl, f, rp, pw, nw, T, ie, key, pc, T_cur_w, state->inv_expo_time, &cfg, &nk, kept, err, sl, A, nullptr);
  if (Record(ctx_, last_status_)) return;
  SubSparseMap &sub = *visual_submap;  // :765-770, in candidate order
  sub.voxel_points_pos.resize(nk), sub.search_levels.assign(sl, sl + nk), sub.errors.assign(err, err + nk);
  sub.inv_expo_list.resize(nk), sub.candidate_index.assign(kept, kept + nk), sub.warp_patch.clear();
  sel_ref_idx_.resize(nk), sel_sl_.assign(sl, sl + nk), sel_px_.resize(2 * (size_t)nk), sel_A_.assign(A, A + 4 * (size_t)nk);
  for (int j = 0; j < nk; j++) {
    const SubMapCandidate &k = c[kept[j]];
    for (int a = 0; a < 3; a++) sub.voxel_points_pos[j][a] = k.pos_w[a];
    sub.inv_expo_list[j] = k.ref_inv_expo;
    sel_ref_idx_[j] = k.ref_img_index, sel_px_[2 * j] = k.px_ref[0], sel_px_[2 * j + 1] = k.px_ref[1];
  }
  total_points = nk;
  selected_submap_ = visual_submap, selected_count_ = nk;
}

void VIOManager::MaterializeWarpPatches() {
  if (!ctx_ || !selected_submap_ || selected_submap_ != visual_submap) return;
  const int nk = selected_count_, L = patch_pyrimid_level;
  if ((int)visual_submap->warp_patch.size() == nk) return;
  last_status_ = 0;
  if (!ref_imgs_current_ && !ref_imgs_.empty()) {  // the per-patch warpAffine replaced them since
    std::vector<GrayImage> imgs = ref_imgs_;
    SetReferenceImages(imgs.data(), (int)imgs.size());
  }
  // the same kernel on the same matrices, levels and reference pixels as the selection: the patches the device holds
  float *wp;
  if (!lay_out_staging(block_, [&](ScratchLayout &s) { wp = s.take<float>((size_t)nk * 64 * L); })) return StagingFailed();
  if (!last_status_) last_status_ = esikf_vio_warp_affine(ctx_, nk, sel_ref_idx_.data(), sel_px_.data(), sel_A_.data(), sel_sl_.data(), wp);
  if (Record(ctx_, last_status_)) return;
  visual_submap->warp_patch.resize(nk);
  for (int j = 0; j < nk; j++) visual_submap->warp_patch[j].assign(wp + (size_t)j * 64 * L, wp + (size_t)(j + 1) * 64 * L);
}

}  // namespace fl2b200

// ---------------------------------------------------------------------------------------------------------------------
// C entry points for the parity tests (Python / ctypes): rebuild a pointer octree from flat arrays, run the shim on it.
using namespace fl2b200;

static void build_tree(VoxelMap &map, const VoxelMapConfig &cfg, const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots,
                       const esikf_plane *planes) {
  const float vs = (float)cfg.max_voxel_size_;
  for (int r = 0; r < n_roots; r++) {
    VOXEL_LOCATION loc(keys[3 * r], keys[3 * r + 1], keys[3 * r + 2]);
    VoxelOctoTree *root = new VoxelOctoTree;
    root->plane_ptr_ = new VoxelPlane;
    root->quater_length_ = vs / 4;
    root->voxel_center_[0] = (0.5 + loc.x) * vs, root->voxel_center_[1] = (0.5 + loc.y) * vs, root->voxel_center_[2] = (0.5 + loc.z) * vs;
    root->init_octo_ = true;
    map[loc] = root;
    for (int c = 0; c < count[r]; c++) {
      const esikf_plane &f = planes[first[r] + c];
      VoxelOctoTree *node = root;
      for (int l = 0; l < f.layer; l++) {
        const int leaf = (f.path >> (3 * l)) & 7;
        if (!node->leaves_[leaf]) {
          VoxelOctoTree *ch = new VoxelOctoTree;
          ch->plane_ptr_ = new VoxelPlane;
          ch->layer_ = l + 1;
          const int xyz[3] = {(leaf >> 2) & 1, (leaf >> 1) & 1, leaf & 1};
          for (int k = 0; k < 3; k++) ch->voxel_center_[k] = node->voxel_center_[k] + (2 * xyz[k] - 1) * node->quater_length_;
          ch->quater_length_ = node->quater_length_ / 2;
          ch->init_octo_ = true;
          node->leaves_[leaf] = ch;
        }
        node = node->leaves_[leaf];
      }
      VoxelPlane &p = *node->plane_ptr_;
      plane_from_row(f, p);
      p.is_plane_ = true, p.is_init_ = true;
    }
  }
}

// VoxelMapConfig from the C ABI's LIO settings; the map-building part keeps its defaults
static VoxelMapConfig map_config(const esikf_lio_cfg &l) {
  VoxelMapConfig cfg;
  cfg.max_voxel_size_ = l.voxel_size, cfg.max_layer_ = l.max_layer, cfg.max_iterations_ = l.max_iterations;
  cfg.beam_err_ = l.beam_err, cfg.dept_err_ = l.dept_err, cfg.sigma_num_ = l.sigma_num;
  return cfg;
}

// A VIOManager set up from the C ABI's camera and VIO settings, then initializeVIO. A null ext keeps the manager's default
// extrinsics.
static void configure_vio(VIOManager &vio, const esikf_camera &cam, const esikf_vio_cfg &vcfg, const esikf_extrinsics *ext) {
  vio.cam = cam;
  vio.patch_pyrimid_level = vcfg.patch_pyrimid_level, vio.max_iterations = vcfg.max_iterations, vio.img_point_cov = vcfg.img_point_cov;
  vio.exposure_estimate_en = vcfg.exposure_estimate_en != 0;
  if (ext) memcpy(vio.Rcl.m, ext->Rcl, 72), memcpy(vio.Pcl.v, ext->Pcl, 24), memcpy(vio.extR.m, ext->extR, 72), memcpy(vio.extT.v, ext->extT, 24);
  vio.initializeVIO();
}

namespace {
// The managers a hook runs on, held as LIVMapper holds them: the host octree, the VoxelMapManager on it (whose constructor
// creates the device context) and a VIOManager sharing that context, on the session's states and visual sub-map. The
// session hooks keep one across ticks (bench.py e2e_shim); the one-shot GPU hooks open one per call. A mirror handle
// (fl2_shim_mirror_create) is a session without managers.
struct ShimSession {
  VoxelMapConfig cfg;
  VoxelMap map;
  std::unique_ptr<VoxelMapManager> mgr;
  std::unique_ptr<VIOManager> vio;
  SubSparseMap sub;
  StatesGroup st, stp;
  bool has_vio = false;
  esikf_camera cam{};
  esikf_vio_cfg vcfg{};
  long long manager_ns = 0;
  ~ShimSession() {
    vio.reset(), mgr.reset();
    ClearVoxelMap(map);
  }
  // A VoxelMapManager on the session's map and a new device context: all the hooks that need no map open. Returns its status.
  int open(int device = 0) {
    mgr.reset(new VoxelMapManager(cfg, map, device));
    return mgr->last_status_;
  }
  // The LIO half: the octree of the flat map, its manager set up from lcfg and the LiDAR extrinsics of ext, and the map's
  // first upload. Returns the first failing esikf_status.
  int open_map(const esikf_lio_cfg &lcfg, const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots, const esikf_plane *planes,
               const esikf_extrinsics &ext, int device) {
    cfg = map_config(lcfg);
    build_tree(map, cfg, keys, first, count, n_roots, planes);
    if (int rc = open(device)) return rc;
    memcpy(mgr->extR_.m, ext.extR, 72), memcpy(mgr->extT_.v, ext.extT, 24);
    mgr->SyncDeviceMap();
    return mgr->last_status_;
  }
  // The VIO half: a VIOManager on the context, st, stp and sub; with cam (and vcfg) configured by configure_vio, without left
  // as constructed. Returns its status.
  int open_vio(const esikf_camera *c, const esikf_vio_cfg *v, const esikf_extrinsics *ext) {
    vio.reset(new VIOManager(mgr->context()));
    vio->state = &st, vio->state_propagat = &stp, vio->visual_submap = &sub;
    if (c) has_vio = true, cam = *c, vcfg = *v, configure_vio(*vio, *c, *v, ext);
    return vio->last_status_;
  }
};
}  // namespace

static ShimSession *session_of(void *h) { return static_cast<ShimSession *>(h); }

extern "C" {

// CPU-only: flat arrays -> pointer octree -> FlattenVoxelMap -> flat arrays (sizes returned; buffers sized like the input).
int fl2_shim_flatten_roundtrip(const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots, const esikf_plane *planes, int n_planes,
                               double voxel_size, int max_layer, int64_t *keys_out, int32_t *first_out, int32_t *count_out, esikf_plane *planes_out) {
  VoxelMapConfig cfg;
  cfg.max_voxel_size_ = voxel_size, cfg.max_layer_ = max_layer;
  VoxelMap map;
  build_tree(map, cfg, keys, first, count, n_roots, planes);
  FlatVoxelMap out;
  std::string err;
  const bool ok = FlattenVoxelMap(map, cfg, out, &err);
  for (auto &kv : map) delete kv.second;
  if (!ok || (int)out.first.size() != n_roots || (int)out.planes.size() != n_planes) return -1;
  memcpy(keys_out, out.keys.data(), out.keys.size() * sizeof(int64_t));
  memcpy(first_out, out.first.data(), out.first.size() * sizeof(int32_t));
  memcpy(count_out, out.count.data(), out.count.size() * sizeof(int32_t));
  memcpy(planes_out, out.planes.data(), out.planes.size() * sizeof(esikf_plane));
  return 0;
}

// GPU: VoxelMapManager::StateEstimation + VIOManager::computeJacobianAndUpdateEKF through the shim classes.
// vio arrays may be null (LIO only). Returns 0 or the first failing esikf_status.
int fl2_shim_run(const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots, const esikf_plane *planes, int n_planes,
                 const esikf_lio_cfg *lcfg, const esikf_extrinsics *ext, const float *pts, int n, const double *state_in, const double *state_prop,
                 double *lio_state_out, int32_t *n_effective, int32_t *n_ptpl, double *normals_out /* n x 3 */, const esikf_camera *cam,
                 const esikf_vio_cfg *vcfg, const uint8_t *img, int n_patches, const double *pos, const float *warp_patch, const int32_t *search_levels,
                 const double *inv_expo, double *vio_state_out, float *errors_out) {
  (void)n_planes;
  ShimSession s;
  int rc = s.open_map(*lcfg, keys, first, count, n_roots, planes, *ext, 0);
  VoxelMapManager &mgr = *s.mgr;
  mgr.feats_down_body_.resize(n);
  memcpy(mgr.feats_down_body_.data(), pts, (size_t)n * 12);
  mgr.feats_down_size_ = n;
  mgr.state_.unpack(state_in);              // voxelmap_manager->state_ = _state  (LIVMapper.cpp:257)
  StatesGroup prop;
  prop.unpack(state_prop);
  if (!rc) {
    mgr.StateEstimation(prop);              // LIVMapper.cpp:370
    rc = mgr.last_status_;
  }
  if (!rc) {
    mgr.state_.pack(lio_state_out);
    *n_effective = mgr.effct_feat_num_;
    *n_ptpl = (int32_t)mgr.ptpl_list_.size();
    for (int i = 0; i < n; i++)
      for (int k = 0; k < 3; k++) normals_out[3 * i + k] = mgr.pv_list_[i].normal[k];
  }
  if (!rc && cam && n_patches > 0) {
    s.st = mgr.state_, s.stp = mgr.state_;
    SubSparseMap &sub = s.sub;
    const int L = vcfg->patch_pyrimid_level;
    for (int i = 0; i < n_patches; i++) {
      V3D p;
      for (int k = 0; k < 3; k++) p[k] = pos[3 * i + k];
      sub.voxel_points_pos.push_back(p);
      sub.warp_patch.emplace_back(warp_patch + (size_t)i * 64 * L, warp_patch + (size_t)(i + 1) * 64 * L);
      sub.search_levels.push_back(search_levels[i]);
      sub.inv_expo_list.push_back(inv_expo[i]);
    }
    rc = s.open_vio(cam, vcfg, ext);
    s.vio->total_points = n_patches;
    GrayImage im;
    im.data = img, im.cols = cam->width, im.rows = cam->height;
    if (!rc) s.vio->computeJacobianAndUpdateEKF(im);
    rc = s.vio->last_status_;
    if (!rc) {
      s.st.pack(vio_state_out);
      for (int i = 0; i < n_patches; i++) errors_out[i] = sub.errors[i];
    }
  }
  return rc;
}

// CPU-only: DiffFlatVoxelMaps on two flat maps given as arrays (same root arrays for both unless keys_b is non-null).
// Returns -1 if the structure differs, else the number of changed plane ids written to ids_out (capacity n_planes_a).
int fl2_shim_diff(const int64_t *keys_a, const int32_t *first_a, const int32_t *count_a, int n_roots_a, const esikf_plane *planes_a, int n_planes_a,
                  const int64_t *keys_b, const int32_t *first_b, const int32_t *count_b, int n_roots_b, const esikf_plane *planes_b, int n_planes_b,
                  int32_t *ids_out) {
  FlatVoxelMap a, b;
  a.keys.assign(keys_a, keys_a + 3 * (size_t)n_roots_a), a.first.assign(first_a, first_a + n_roots_a), a.count.assign(count_a, count_a + n_roots_a);
  a.planes.assign(planes_a, planes_a + n_planes_a);
  b.keys.assign(keys_b, keys_b + 3 * (size_t)n_roots_b), b.first.assign(first_b, first_b + n_roots_b), b.count.assign(count_b, count_b + n_roots_b);
  b.planes.assign(planes_b, planes_b + n_planes_b);
  std::vector<int32_t> ids;
  if (!DiffFlatVoxelMaps(a, b, ids)) return -1;
  for (size_t k = 0; k < ids.size(); k++) ids_out[k] = ids[k];
  return (int)ids.size();
}

// GPU: map refresh through the shim. Builds the octree of map A, syncs (full upload), overwrites the plane fits with map B's
// (same structure: an UpdateVoxelMap that only refitted planes), syncs again (incremental: esikf_map_patch of the changed
// records) and runs StateEstimation. The caller compares with a run on a fresh manager holding map B.
int fl2_shim_resync_run(const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots, const esikf_plane *planes_a, const esikf_plane *planes_b,
                        int n_planes, const esikf_lio_cfg *lcfg, const esikf_extrinsics *ext, const float *pts, int n, const double *state_in,
                        double *state_out, int32_t *n_patched) {
  (void)n_planes;
  ShimSession s;
  int rc = s.open_map(*lcfg, keys, first, count, n_roots, planes_a, *ext, 0);
  VoxelMapManager &mgr = *s.mgr;
  if (!rc) {
    // the host map changes under the manager: same octree, new plane fits
    for (int r = 0; r < n_roots; r++) {
      VOXEL_LOCATION loc(keys[3 * r], keys[3 * r + 1], keys[3 * r + 2]);
      for (int c = 0; c < count[r]; c++) {
        const esikf_plane &f = planes_b[first[r] + c];
        VoxelOctoTree *node = s.map[loc];
        for (int l = 0; l < f.layer; l++) node = node->leaves_[(f.path >> (3 * l)) & 7];
        plane_from_row(f, *node->plane_ptr_);
      }
    }
    mgr.MarkMapDirty();
    mgr.SyncDeviceMap();
    rc = mgr.last_status_;
    *n_patched = mgr.last_sync_patched_;
  }
  if (!rc) {
    mgr.feats_down_body_.resize(n);
    memcpy(mgr.feats_down_body_.data(), pts, (size_t)n * 12);
    mgr.feats_down_size_ = n;
    mgr.fill_point_lists_ = false;
    mgr.state_.unpack(state_in);
    StatesGroup prop;
    prop.unpack(state_in);
    mgr.StateEstimation(prop);
    rc = mgr.last_status_;
    if (!rc) mgr.state_.pack(state_out);
  }
  return rc;
}

// GPU: VIOManager::SelectSubSparseMap + computeJacobianAndUpdateEKF (sub-map left on the device), then the same update from
// the host-assembled sub-map (MaterializeWarpPatches, a copy of visual_submap, the set_patches path). gate = [normal_en, ncc_en,
// ncc_thre, outlier_threshold]. counts = [launches of the first update, sub-map uploads after it, launches of the second
// update, sub-map uploads after it]. Returns 0 or the first failing esikf_status.
int fl2_shim_select_run(const esikf_camera *cam, const esikf_vio_cfg *vcfg, const esikf_extrinsics *ext, const uint8_t *img, const uint8_t *const *ref_imgs,
                        int n_imgs, const SubMapCandidate *cands, int n, const double *T_cur_w, const double *state_in, const double *gate, int32_t *n_kept,
                        int32_t *kept, double *state_sel, float *errors_sel, double *state_host, float *errors_host, float *warp_out, int64_t *counts) {
  ShimSession s;
  int rc = s.open();
  if (rc) return rc;
  esikf_ctx *ctx = s.mgr->context();
  StatesGroup &st = s.st;
  SubSparseMap &sub = s.sub;
  st.unpack(state_in), s.stp.unpack(state_in);
  s.open_vio(cam, vcfg, ext);
  VIOManager &vio = *s.vio;
  vio.normal_en = gate[0] != 0, vio.ncc_en = gate[1] != 0, vio.ncc_thre = gate[2], vio.outlier_threshold = gate[3];
  GrayImage im;
  im.data = img, im.cols = cam->width, im.rows = cam->height;
  std::vector<GrayImage> refs(n_imgs);
  for (int k = 0; k < n_imgs; k++) refs[k].data = ref_imgs[k], refs[k].cols = cam->width, refs[k].rows = cam->height;
  if (!vio.last_status_) vio.SetReferenceImages(refs.data(), n_imgs);
  if (!vio.last_status_) vio.SelectSubSparseMap(cands, n, im, T_cur_w);
  rc = vio.last_status_;
  if (!rc) {
    *n_kept = vio.total_points;
    for (int j = 0; j < vio.total_points; j++) kept[j] = sub.candidate_index[j];
    int64_t l0 = esikf_launch_count(ctx);
    vio.computeJacobianAndUpdateEKF(im);
    counts[0] = esikf_launch_count(ctx) - l0, counts[1] = vio.submap_uploads_;
    rc = vio.last_status_;
  }
  if (!rc) {
    st.pack(state_sel);
    for (int j = 0; j < vio.total_points; j++) errors_sel[j] = sub.errors[j];
    vio.MaterializeWarpPatches();
    rc = vio.last_status_;
  }
  if (!rc) {
    const int L = vio.patch_pyrimid_level;
    for (int j = 0; j < vio.total_points; j++) memcpy(warp_out + (size_t)j * 64 * L, sub.warp_patch[j].data(), sizeof(float) * 64 * L);
    SubSparseMap host = sub;  // the sub-map as a host-side retrieval would have assembled it
    vio.visual_submap = &host;
    st.unpack(state_in);
    int64_t l0 = esikf_launch_count(ctx);
    vio.computeJacobianAndUpdateEKF(im);
    counts[2] = esikf_launch_count(ctx) - l0, counts[3] = vio.submap_uploads_;
    rc = vio.last_status_;
    if (!rc) {
      st.pack(state_host);
      for (int j = 0; j < vio.total_points; j++) errors_host[j] = host.errors[j];
    }
  }
  return rc;
}

// GPU: VIOManager::RetrieveScanVoxels on n host points (pg: n x 3) with the frame pose of `state`, then
// VIOManager::CheckDepthContinuity on n_cand points (cand_pos: n_cand x 3, cand_pc: n_cand x 2). Outputs: *n_keys, keys (room
// for n x 3) and flags (n_cand). Returns 0 or the first failing esikf_status.
int fl2_shim_retrieve_run(const esikf_camera *cam, const esikf_vio_cfg *vcfg, const esikf_extrinsics *ext, const double *state, const double *pg, int n, int border,
                          const double *cand_pos, const double *cand_pc, int n_cand, int32_t *n_keys, int64_t *keys, uint8_t *flags) {
  ShimSession s;
  int rc = s.open();
  if (rc) return rc;
  s.st.unpack(state), s.stp.unpack(state);
  s.open_vio(cam, vcfg, ext);
  VIOManager &vio = *s.vio;
  std::vector<pointWithVar> scan(n);
  for (int i = 0; i < n; i++)
    for (int k = 0; k < 3; k++) scan[i].point_w[k] = pg[3 * i + k];
  std::vector<VOXEL_LOCATION> kv;
  std::vector<uint8_t> fl;
  if (!vio.last_status_) vio.RetrieveScanVoxels(border, &scan, kv);
  if (!vio.last_status_) vio.CheckDepthContinuity(n_cand, cand_pos, cand_pc, fl);
  rc = vio.last_status_;
  if (!rc) {
    *n_keys = (int32_t)kv.size();
    for (size_t i = 0; i < kv.size(); i++) keys[3 * i] = kv[i].x, keys[3 * i + 1] = kv[i].y, keys[3 * i + 2] = kv[i].z;
    memcpy(flags, fl.data(), fl.size());
  }
  return rc;
}

// GPU: VIOManager::getImagePatch / VIOManager::warpAffine through the shim class (one patch each).
int fl2_shim_patch_helpers(const esikf_camera *cam, const esikf_vio_cfg *vcfg, const uint8_t *img, int cols, int rows, const double *pc, int level,
                           float *patch_tmp /* levels*64, only `level` written */, const double *A_cur_ref, const uint8_t *img_ref, const double *px_ref,
                           int search_level, int pyramid_level, float *warp_patch /* levels*64, only `pyramid_level` written */) {
  ShimSession s;
  int rc = s.open();
  if (rc) return rc;
  // no extrinsics: both helpers sample images at the pixel coordinates they are given
  rc = s.open_vio(cam, vcfg, nullptr);
  VIOManager &vio = *s.vio;
  GrayImage g{img, cols, rows}, gr{img_ref, cols, rows};
  if (!rc) {
    vio.getImagePatch(g, pc, patch_tmp, level);
    rc = vio.last_status_;
  }
  if (!rc) {
    vio.warpAffine(A_cur_ref, gr, px_ref, 0, search_level, pyramid_level, 4, warp_patch);
    rc = vio.last_status_;
  }
  return rc;
}

// ---- persistent session for the end-to-end measurement through the drop-in classes (bench.py e2e_shim): the managers,
// the host octree and the visual sub-map live across ticks like they do inside LIVMapper.
void *fl2_shim_session_create(const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots, const esikf_plane *planes, int n_planes,
                              const esikf_lio_cfg *lcfg, const esikf_extrinsics *ext, const esikf_camera *cam, const esikf_vio_cfg *vcfg, int device) {
  (void)n_planes;
  ShimSession *s = new ShimSession;
  if (s->open_map(*lcfg, keys, first, count, n_roots, planes, *ext, device) || (cam && vcfg && s->open_vio(cam, vcfg, ext))) {
    delete s;
    return nullptr;
  }
  return s;
}

// One LIVMapper tick pair: LIO (LIVMapper.cpp:356-372) then VIO on the LIO posterior (:305, vio.cpp:1810). iters_out[0] = LIO
// iterations, [1] = VIO iterations.
int fl2_shim_session_step(void *h, const float *pts, int n, const double *state_in, const double *state_prop, const uint8_t *img, int n_patches, const double *pos,
                          const float *warp_patch, const int32_t *search_levels, const double *inv_expo, double *lio_state_out, double *vio_state_out, int32_t *iters_out) {
  ShimSession *s = session_of(h);
  if (!s) return ESIKF_ERR_ARG;
  VoxelMapManager &mgr = *s->mgr;
  mgr.feats_down_body_.resize(n);
  if (n) memcpy(mgr.feats_down_body_.data(), pts, (size_t)n * 12);
  mgr.feats_down_size_ = n;
  mgr.state_.unpack(state_in);  // voxelmap_manager->state_ = _state  (LIVMapper.cpp:257)
  StatesGroup prop;
  prop.unpack(state_prop);
  const auto t_lio0 = std::chrono::steady_clock::now();
  mgr.StateEstimation(prop);    // LIVMapper.cpp:370
  s->manager_ns = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t_lio0).count();
  if (mgr.last_status_) return mgr.last_status_;
  mgr.state_.pack(lio_state_out);
  iters_out[0] = mgr.last_iters_, iters_out[1] = 0;
  if (s->has_vio && n_patches > 0) {
    VIOManager &vio = *s->vio;
    s->st = mgr.state_, s->stp = mgr.state_;
    SubSparseMap &sub = s->sub;
    const int L = s->vcfg.patch_pyrimid_level;
    if ((int)sub.voxel_points_pos.size() != n_patches) {  // the visual sub-map of the tick (retrieveFromVisualSparseMap's output)
      sub.voxel_points_pos.resize(n_patches), sub.warp_patch.resize(n_patches), sub.search_levels.resize(n_patches), sub.inv_expo_list.resize(n_patches);
    }
    for (int i = 0; i < n_patches; i++) {
      for (int k = 0; k < 3; k++) sub.voxel_points_pos[i][k] = pos[3 * i + k];
      sub.warp_patch[i].assign(warp_patch + (size_t)i * 64 * L, warp_patch + (size_t)(i + 1) * 64 * L);
      sub.search_levels[i] = search_levels[i];
      sub.inv_expo_list[i] = inv_expo[i];
    }
    vio.total_points = n_patches;
    GrayImage im;
    im.data = img, im.cols = s->cam.width, im.rows = s->cam.height;
    const auto t_vio0 = std::chrono::steady_clock::now();
    vio.computeJacobianAndUpdateEKF(im);
    s->manager_ns += std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t_vio0).count();
    if (vio.last_status_) return vio.last_status_;
    s->st.pack(vio_state_out);
    iters_out[1] = vio.last_total_iters_;
  }
  return 0;
}

// mode 0: pv_list_ / ptpl_list_ / body_cov_list_ / cross_mat_list_ filled inside every StateEstimation (the reference's member
// contract); 1: filled lazily (MaterializePointLists — never, in the timed loop of a caller that does not read them); 2: off.
void fl2_shim_session_point_lists(void *h, int mode) {
  ShimSession *s = session_of(h);
  if (!s) return;
  s->mgr->fill_point_lists_ = (mode != 2);
  s->mgr->lazy_point_lists_ = (mode == 1);
}
// number of entries the lists hold after materialising them (checks the lazy path in the tests)
int fl2_shim_session_materialize(void *h, int32_t *n_pv, int32_t *n_ptpl) {
  ShimSession *s = session_of(h);
  if (!s) return ESIKF_ERR_ARG;
  s->mgr->MaterializePointLists();
  if (n_pv) *n_pv = (int32_t)s->mgr->pv_list_.size();
  if (n_ptpl) *n_ptpl = (int32_t)s->mgr->ptpl_list_.size();
  return s->mgr->last_status_;
}

// Device-resident map for the session: the map the session was created with is dropped, an empty device map takes its place and
// absorbs `pts` at `state` through BuildVoxelMap (first LiDAR frame, LIVMapper.cpp:356-366).
int fl2_shim_session_device_map(void *h, const float *pts, int n, const double *state, double min_eigen_value, int max_points_num, long long root_capacity) {
  ShimSession *s = session_of(h);
  if (!s) return ESIKF_ERR_ARG;
  VoxelMapManager &mgr = *s->mgr;
  mgr.config_setting_.planner_threshold_ = min_eigen_value, mgr.config_setting_.max_points_num_ = max_points_num;
  mgr.config_setting_.device_root_capacity_ = root_capacity;
  mgr.EnableDeviceMap();
  if (mgr.last_status_) return mgr.last_status_;
  mgr.feats_down_body_.resize(n);
  if (n) memcpy(mgr.feats_down_body_.data(), pts, (size_t)n * 12);
  mgr.feats_down_size_ = n;
  mgr.state_.unpack(state);
  mgr.BuildVoxelMap();
  return mgr.last_status_;
}
// LIVMapper.cpp:413-424 after the LIO half of a tick: the device map absorbs the scan with the LIO posterior.
int fl2_shim_session_update_map(void *h) {
  ShimSession *s = session_of(h);
  if (!s) return ESIKF_ERR_ARG;
  s->mgr->UpdateVoxelMap();
  return s->mgr->last_status_;
}

// nanoseconds the last step spent inside StateEstimation + computeJacobianAndUpdateEKF (the two calls LIVMapper makes; filling
// the managers' members from the harness' flat buffers — which LIVMapper already holds in that shape — is outside)
long long fl2_shim_session_manager_ns(void *h) {
  ShimSession *s = session_of(h);
  return s ? s->manager_ns : 0;
}

void fl2_shim_session_destroy(void *h) { delete session_of(h); }

// ---- the host mirror of a device map (VoxelMapConfig::device_map_mirror_). A mirror handle is a session without managers:
// the apply code runs on the CPU there. The dump / flatten / find hooks take either kind of handle.
void *fl2_shim_mirror_create(double voxel_size, int max_layer) {
  ShimSession *s = new ShimSession;
  s->cfg.max_voxel_size_ = voxel_size, s->cfg.max_layer_ = max_layer;
  return s;
}
int fl2_shim_mirror_apply(void *h, const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots, const esikf_map_node *nodes, int n_nodes) {
  ShimSession *s = session_of(h);
  if (!s) return ESIKF_ERR_ARG;
  return ApplyMapExport(s->map, s->cfg, keys, first, count, n_roots, nodes, n_nodes, nullptr) ? 0 : ESIKF_ERR_ARG;
}
void fl2_shim_mirror_erase(void *h, const int64_t *lo, const int64_t *hi) { EraseRootsOutside(session_of(h)->map, lo, hi); }
// The mirror's nodes as oracle_bind.NODE_COLS rows (DFS pre-order, leaves 0..7, roots in map order). Returns the number of
// nodes; rows beyond cap are counted, not written.
static void mirror_dump_node(const VoxelOctoTree *t, int64_t path, const VOXEL_LOCATION &key, int64_t *out, int cap, int *n) {
  if (*n < cap) {
    int64_t *r = out + (size_t)(*n) * 12;
    r[0] = key.x, r[1] = key.y, r[2] = key.z, r[3] = t->layer_, r[4] = path;
    r[5] = t->init_octo_, r[6] = t->octo_state_, r[7] = t->update_enable_, r[8] = t->plane_ptr_->is_plane_;
    r[9] = t->new_points_, r[10] = t->temp_points_size_, r[11] = t->plane_ptr_->points_size_;
  }
  (*n)++;
  for (int l = 0; l < 8; l++)
    if (t->leaves_[l]) mirror_dump_node(t->leaves_[l], path | ((int64_t)l << (3 * t->layer_)), key, out, cap, n);
}
int fl2_shim_mirror_dump(void *h, int64_t *out, int cap) {
  int n = 0;
  for (const auto &kv : session_of(h)->map) mirror_dump_node(kv.second, 0, kv.first, out, cap, &n);
  return n;
}
// FlattenVoxelMap of the mirror, two calls: planes == NULL returns the sizes
int fl2_shim_mirror_flatten(void *h, int *n_roots, int *n_planes, int64_t *keys, int32_t *first, int32_t *count, esikf_plane *planes) {
  ShimSession *s = session_of(h);
  FlatVoxelMap flat;
  std::string err;
  if (!FlattenVoxelMap(s->map, s->cfg, flat, &err)) return ESIKF_ERR_ARG;
  *n_roots = (int)flat.first.size(), *n_planes = (int)flat.planes.size();
  if (planes) {
    memcpy(keys, flat.keys.data(), flat.keys.size() * sizeof(int64_t));
    memcpy(first, flat.first.data(), flat.first.size() * sizeof(int32_t));
    memcpy(count, flat.count.data(), flat.count.size() * sizeof(int32_t));
    memcpy(planes, flat.planes.data(), flat.planes.size() * sizeof(esikf_plane));
  }
  return 0;
}
// updateReferencePatch's lookup (src/vio.cpp:983-993) per point: the root voxel by the float quotient (with the map's voxel
// size), then find_correspond. out: n x 4 = found, layer, path, is_plane of the node it returns.
void fl2_shim_mirror_find(void *h, const double *pts, int n, int64_t *out) {
  ShimSession *s = session_of(h);
  for (int i = 0; i < n; i++) {
    const double *p = pts + 3 * (size_t)i;
    float loc_xyz[3];
    for (int j = 0; j < 3; j++) {
      loc_xyz[j] = p[j] / s->cfg.max_voxel_size_;
      if (loc_xyz[j] < 0) loc_xyz[j] -= 1.0;
    }
    int64_t *o = out + 4 * (size_t)i;
    o[0] = o[1] = o[2] = o[3] = 0;
    auto it = s->map.find(VOXEL_LOCATION((int64_t)loc_xyz[0], (int64_t)loc_xyz[1], (int64_t)loc_xyz[2]));
    if (it == s->map.end()) continue;
    V3D pw;
    for (int k = 0; k < 3; k++) pw[k] = p[k];
    const VoxelOctoTree *t = it->second->find_correspond(pw);
    int64_t path = 0;  // the leaves find_correspond took (it follows them again)
    for (const VoxelOctoTree *u = it->second; u != t;) {
      const int l = 4 * (pw[0] > u->voxel_center_[0]) + 2 * (pw[1] > u->voxel_center_[1]) + (pw[2] > u->voxel_center_[2]);
      path |= (int64_t)l << (3 * u->layer_);
      u = u->leaves_[l];
    }
    o[0] = 1, o[1] = t->layer_, o[2] = path, o[3] = t->plane_ptr_->is_plane_;
  }
}
// fl2_shim_session_device_map with the growth and mirror switches of VoxelMapConfig
int fl2_shim_session_device_map_mirror(void *h, const float *pts, int n, const double *state, double min_eigen_value, int max_points_num, long long root_capacity, int grow,
                                       int mirror) {
  ShimSession *s = session_of(h);
  if (!s) return ESIKF_ERR_ARG;
  s->mgr->config_setting_.device_map_grow_ = grow != 0, s->mgr->config_setting_.device_map_mirror_ = mirror != 0;
  return fl2_shim_session_device_map(h, pts, n, state, min_eigen_value, max_points_num, root_capacity);
}
// UpdateVoxelMap(input_points) (include/voxel_map.h:232) with point_w [n][3] and var [n][9]
int fl2_shim_session_update_points(void *h, const double *pw, const double *var, int n) {
  ShimSession *s = session_of(h);
  if (!s) return ESIKF_ERR_ARG;
  std::vector<pointWithVar> pts(n);
  for (int i = 0; i < n; i++) {
    for (int k = 0; k < 3; k++) pts[i].point_w[k] = pw[3 * i + k];
    memcpy(pts[i].var.m, var + 9 * (size_t)i, 72);
  }
  s->mgr->UpdateVoxelMap(pts);
  return s->mgr->last_status_;
}
// mapSliding (src/voxel_map.cpp:924-948) with the sensor at `position`
int fl2_shim_session_map_sliding(void *h, const double *position, int half_map_size, double sliding_thresh) {
  ShimSession *s = session_of(h);
  if (!s) return ESIKF_ERR_ARG;
  VoxelMapManager &mgr = *s->mgr;
  mgr.config_setting_.half_map_size = half_map_size, mgr.config_setting_.sliding_thresh = sliding_thresh;
  for (int k = 0; k < 3; k++) mgr.position_last_[k] = position[k];
  mgr.mapSliding();
  return mgr.last_status_;
}
// VoxelMapManager::FindCorrespond through a session; the answers in esikf_plane rows (plane_var_'s upper triangle; layer and
// path are not part of a VoxelPlane and stay 0)
int fl2_shim_session_find_correspond(void *h, const double *pts, int n, int rule, uint8_t *status, esikf_plane *rows) {
  ShimSession *s = session_of(h);
  if (!s || n < 0) return ESIKF_ERR_ARG;
  std::vector<V3D> p(n);
  for (int i = 0; i < n; i++)
    for (int k = 0; k < 3; k++) p[i][k] = pts[3 * (size_t)i + k];
  std::vector<VoxelPlane> planes(n);
  s->mgr->FindCorrespond(n, p.data(), rule, status, planes.data());
  if (s->mgr->last_status_) return s->mgr->last_status_;
  for (int i = 0; i < n; i++) {
    memset(&rows[i], 0, sizeof(rows[i]));
    row_from_plane(planes[i], rows[i]);
  }
  return 0;
}
// GPU: VIOManager::ScoreReferencePatches on its own context, with the arrays of esikf_vio_score_ref_patches packed into the
// shim's records. Returns 0 or the failing esikf_status (the outputs untouched).
int fl2_shim_score_ref_patches(int n, const int32_t *first, int m, const double *pos, const double *normal, const float *patch, const float *mean,
                               const int32_t *id, const double *T_f_w, float *score_out, float *mean_out, int32_t *ref_out) {
  if (n < 0 || m < 0 || !first) return ESIKF_ERR_ARG;
  ShimSession s;
  int rc = s.open();
  if (rc) return rc;
  s.open_vio(nullptr, nullptr, nullptr);  // the scoring reads no camera, VIO settings or extrinsics
  VIOManager &vio = *s.vio;
  std::vector<int32_t> fi(first, first + n + 1);
  std::vector<ScoredPoint> pts(n);
  for (int i = 0; i < n; i++) memcpy(pts[i].pos, pos + 3 * i, sizeof(pts[i].pos)), memcpy(pts[i].normal, normal + 3 * i, sizeof(pts[i].normal));
  std::vector<PatchObservation> obs(m);
  for (int j = 0; j < m; j++) {
    memcpy(obs[j].T_f_w, T_f_w + 12 * (size_t)j, sizeof(obs[j].T_f_w)), memcpy(obs[j].patch, patch + 64 * (size_t)j, sizeof(obs[j].patch));
    obs[j].mean = mean[j], obs[j].id = id[j];
  }
  std::vector<float> sc, mu;
  std::vector<int32_t> rf;
  vio.ScoreReferencePatches(fi, pts, obs, sc, mu, rf);
  rc = vio.last_status_;
  if (!rc) {
    memcpy(score_out, sc.data(), sc.size() * sizeof(float)), memcpy(mean_out, mu.data(), mu.size() * sizeof(float));
    memcpy(ref_out, rf.data(), rf.size() * sizeof(int32_t));
  }
  return rc;
}
// GPU: the observation-store overloads of VIOManager on the caller's context (a VIOManager shares it, as LIVMapper's does),
// one per C ABI call; the same arguments as esikf_vmap_*. Each returns 0 or the failing esikf_status.
int fl2_shim_vmap_enable(void *ctx, int64_t capacity) {
  VIOManager vio((esikf_ctx *)ctx);
  vio.EnableDeviceObservations(capacity);
  return vio.last_status_;
}
int fl2_shim_vmap_add(void *ctx, int n, const int32_t *first, const double *px, const float *patch, const double *T_f_w, const int32_t *id,
                      const float *mean, const float *score, const int32_t *ref, int32_t *ids_out) {
  VIOManager vio((esikf_ctx *)ctx);
  std::vector<int32_t> fi(first, first + n + 1), rf(ref, ref + n), ids;
  std::vector<StoredObservation> obs(fi[n]);
  for (int j = 0; j < fi[n]; j++) {
    memcpy(obs[j].px, px + 2 * j, sizeof(obs[j].px)), memcpy(obs[j].T_f_w, T_f_w + 12 * (size_t)j, sizeof(obs[j].T_f_w));
    memcpy(obs[j].patch, patch + 64 * (size_t)j, sizeof(obs[j].patch));
    obs[j].id = id[j], obs[j].mean = mean[j], obs[j].score = score[j];
  }
  vio.AddVisualPoints(fi, obs, rf, ids);
  if (!vio.last_status_) memcpy(ids_out, ids.data(), ids.size() * sizeof(int32_t));
  return vio.last_status_;
}
int fl2_shim_vmap_update(void *ctx, const double *state, int n, const int32_t *point_id, const uint8_t *converged, int32_t frame_id, int32_t *n_out,
                         uint8_t *flag_out, int32_t *entry_out, double *pc_out, float *patch_out, int32_t *evicted_out, int32_t *count_out) {
  VIOManager vio((esikf_ctx *)ctx);
  StatesGroup st;
  st.unpack(state);
  vio.state = &st, vio.total_points = n;
  std::vector<int32_t> pid(point_id, point_id + n), ev, cnt;
  std::vector<uint8_t> conv(converged, converged + n), flag;
  std::vector<NewObservation> obs;
  vio.UpdateVisualMapPoints(pid, conv, frame_id, flag, obs, ev, cnt);
  if (vio.last_status_) return vio.last_status_;
  *n_out = (int32_t)obs.size();
  memcpy(flag_out, flag.data(), n), memcpy(evicted_out, ev.data(), n * sizeof(int32_t)), memcpy(count_out, cnt.data(), n * sizeof(int32_t));
  for (size_t i = 0; i < obs.size(); i++) {
    entry_out[i] = obs[i].entry;
    memcpy(pc_out + 2 * i, obs[i].pc, sizeof(obs[i].pc)), memcpy(patch_out + 64 * i, obs[i].patch, sizeof(obs[i].patch));
  }
  return 0;
}
int fl2_shim_vmap_score(void *ctx, int n, const int32_t *point_id, const double *pos, const double *normal, int32_t *ref_out) {
  VIOManager vio((esikf_ctx *)ctx);
  std::vector<ScoredPoint> pts(n);
  for (int i = 0; i < n; i++) memcpy(pts[i].pos, pos + 3 * i, sizeof(pts[i].pos)), memcpy(pts[i].normal, normal + 3 * i, sizeof(pts[i].normal));
  std::vector<int32_t> ref;
  vio.ScoreReferencePatches(std::vector<int32_t>(point_id, point_id + n), pts, ref);
  if (!vio.last_status_) memcpy(ref_out, ref.data(), ref.size() * sizeof(int32_t));
  return vio.last_status_;
}
int fl2_shim_vmap_choose(void *ctx, int n, const int32_t *point_id, const double *pos, const double *frame_pos, int normal_en, int32_t *ref_out) {
  VIOManager vio((esikf_ctx *)ctx);
  std::vector<int32_t> ref;
  vio.ChooseReferenceFeatures(std::vector<int32_t>(point_id, point_id + n), pos, frame_pos, normal_en != 0, ref);
  if (!vio.last_status_) memcpy(ref_out, ref.data(), ref.size() * sizeof(int32_t));
  return vio.last_status_;
}
void *fl2_shim_session_context(void *h) { return session_of(h)->mgr->context(); }

}  // extern "C"
