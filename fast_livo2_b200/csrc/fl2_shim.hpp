// fl2_shim.hpp — C++ host side of the drop-in boundary: mirrors of the reference's VoxelMapManager / VIOManager call
// surface (same member names, same call order, same "void return + public member fields" convention) on top of the C ABI
// of include/esikf_b200.h. The reference's own headers need Eigen / PCL / ROS / OpenCV / vikit (absent from this image),
// so the boundary types are restated here as layout-compatible PODs; INTEGRATION.md shows the two-line adaptation from the
// real Eigen types (Eigen fixed-size matrices are plain arrays of doubles).
//
// Reference interface being replaced (hku-mars/FAST-LIVO2 @ 0d2c034):
//   VoxelMapManager::StateEstimation(StatesGroup &)                    include/voxel_map.h:229   src/voxel_map.cpp:338-511
//   VoxelMapManager::{state_, feats_down_body_, feats_down_size_, pv_list_, ptpl_list_, effct_feat_num_, position_last_,
//                     cross_mat_list_, body_cov_list_, extR_, extT_, config_setting_, voxel_map_}   include/voxel_map.h:187-218
//   VIOManager::computeJacobianAndUpdateEKF(cv::Mat)                   include/vio.h:153         src/vio.cpp:784-802
//   VIOManager::{state, state_propagat, visual_submap, total_points, G, H_T_H, ...}                  include/vio.h
#pragma once
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/esikf_b200.h"

namespace fl2b200 {

struct V3D { double v[3] = {0, 0, 0}; double &operator[](int i) { return v[i]; } const double &operator[](int i) const { return v[i]; } };
struct M3D { double m[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}; double &operator()(int r, int c) { return m[3 * r + c]; } const double &operator()(int r, int c) const { return m[3 * r + c]; } };  // row-major

// include/common_lib.h:126-223
struct StatesGroup {
  M3D rot_end;
  V3D pos_end, vel_end;
  double inv_expo_time = 1.0;
  V3D bias_g, bias_a, gravity;
  double cov[19 * 19];  // row-major
  StatesGroup();
  void pack(double *out386) const;
  void unpack(const double *in386);
};

// include/common_lib.h:102-123 (fields the hot path reads / writes)
struct pointWithVar {
  V3D point_b, point_i, point_w;
  M3D var_nostate, body_var, var, point_crossmat;
  V3D normal;
  pointWithVar();
};

// include/voxel_map.h:54-67
struct PointToPlane {
  V3D point_b_, point_w_, normal_, center_;
  double plane_var_[36];
  M3D body_cov_;
  int layer_ = 0;
  double d_ = 0, eigen_value_ = 0;
  bool is_valid_ = false;
  float dis_to_plane_ = 0;
};

// include/voxel_map.h:69-94
struct VoxelPlane {
  V3D center_, normal_, y_normal_, x_normal_;
  M3D covariance_;
  double plane_var_[36] = {0};  // row-major 6x6
  float radius_ = 0, min_eigen_value_ = 1, mid_eigen_value_ = 1, max_eigen_value_ = 1, d_ = 0;
  int points_size_ = 0;
  bool is_plane_ = false, is_init_ = false;
  int id_ = 0;
  bool is_update_ = false;
};

// include/voxel_map.h:96-118
struct VOXEL_LOCATION {
  int64_t x, y, z;
  VOXEL_LOCATION(int64_t vx = 0, int64_t vy = 0, int64_t vz = 0) : x(vx), y(vy), z(vz) {}
  bool operator==(const VOXEL_LOCATION &o) const { return x == o.x && y == o.y && z == o.z; }
};
struct VoxelLocationHash {
  int64_t operator()(const VOXEL_LOCATION &s) const {
    const int64_t P = 116101, N = 10000000000LL;
    return ((((s.z) * P) % N + (s.y)) * P) % N + (s.x);
  }
};

// include/voxel_map.h:129-183 (structure only; the map bookkeeping stays with the reference's own code). The state members below
// the plane are what the host mirror of a device-resident map carries (VoxelMapConfig::device_map_mirror_).
struct VoxelOctoTree {
  VoxelPlane *plane_ptr_ = nullptr;
  int layer_ = 0;
  VoxelOctoTree *leaves_[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  double voxel_center_[3] = {0, 0, 0};
  float quater_length_ = 0;
  bool init_octo_ = false;
  int max_layer_ = 0, octo_state_ = 0, new_points_ = 0;
  bool update_enable_ = true;
  int temp_points_size_ = 0;  // temp_points_.size() of the device node; the point list itself is not mirrored
  ~VoxelOctoTree();
  VoxelOctoTree *find_correspond(V3D pw);  // include/voxel_map.h:181, src/voxel_map.cpp:292-305
};
typedef std::unordered_map<VOXEL_LOCATION, VoxelOctoTree *, VoxelLocationHash> VoxelMap;

// include/voxel_map.h:35-52
struct VoxelMapConfig {
  double max_voxel_size_ = 0.5;
  int max_layer_ = 2;
  int max_iterations_ = 5;
  double beam_err_ = 0.05, dept_err_ = 0.02, sigma_num_ = 3.0;
  // map-building part (read by the device-resident map only; a host-owned map is built by the reference's own code)
  double planner_threshold_ = 0.0025;  // lio/min_eigen_value
  int max_points_num_ = 50;            // lio/max_points_num
  std::vector<int> layer_init_num_{5, 5, 5, 5, 5};
  long long device_root_capacity_ = 0;  // 0: esikf_map_device_init's default (2^20 root voxels); the starting size when growing
  bool device_map_grow_ = false;        // the device map grows when a tick would exceed its capacities (esikf_map_cfg.grow)
  // device map: keep voxel_map_ as a read-only host mirror of it (the roots every build / update changed are exported and
  // applied after the call; mapSliding erases what the slide dropped), for the host code that reads the octree, such as
  // VIOManager::updateReferencePatch's find_correspond. The point lists are not mirrored: the reference's own UpdateVoxelMap
  // must not run on it. Read by EnableDeviceMap.
  bool device_map_mirror_ = false;
  bool map_sliding_en = false;          // local_map/map_sliding_en
  int half_map_size = 100;              // local_map/half_map_size
  double sliding_thresh = 8.0;          // local_map/sliding_thresh
};

struct PointXYZ { float x, y, z; };  // pcl::PointXYZINormal's xyz as consumed at src/voxel_map.cpp:351,520-521

// The flattened map handed to esikf_map_upload: root keys + DFS-ordered candidate planes.
struct FlatVoxelMap {
  std::vector<int64_t> keys;
  std::vector<int32_t> first, count;
  std::vector<esikf_plane> planes;
  std::vector<const VoxelPlane *> plane_src;  // flat plane id -> the VoxelPlane it mirrors (for map_patch / pv.normal)
};
// DFS of every root in leaf order 0..7, plane nodes terminate their branch: exactly what build_single_residual visits
// (src/voxel_map.cpp:721, 771-784). Throws nothing; returns false with `err` set on inconsistent roots.
bool FlattenVoxelMap(const VoxelMap &map, const VoxelMapConfig &cfg, FlatVoxelMap &out, std::string *err);
// What changed between two flattenings of the same map: false if the structure differs (roots added / removed, a candidate
// list grew or shrank or moved — needs a full upload), true with the ids of the plane records whose content changed
// (refitted planes: what esikf_map_patch takes). is_update_ is not used: the reference sets it on every fit and never clears it.
bool DiffFlatVoxelMaps(const FlatVoxelMap &synced, const FlatVoxelMap &now, std::vector<int32_t> &changed_ids);
// The host mirror of a device map (VoxelMapConfig::device_map_mirror_). ApplyMapExport walks every exported root's rows
// (esikf_map_device_export) alongside the root's subtree in `map`: nodes that exist are overwritten field by field, missing
// ones are allocated (between slides a root only grows). False with `err` set on a malformed export. EraseRootsOutside is
// clearMemOutOfMap's predicate (src/voxel_map.cpp:958) with the bounds the slide was given; ClearVoxelMap deletes every root.
bool ApplyMapExport(VoxelMap &map, const VoxelMapConfig &cfg, const int64_t *keys, const int32_t *first, const int32_t *count, int n_roots, const esikf_map_node *nodes,
                    int n_nodes, std::string *err);
void EraseRootsOutside(VoxelMap &map, const int64_t lo[3], const int64_t hi[3]);
void ClearVoxelMap(VoxelMap &map);

// Grow-only page-locked host buffer (esikf_host_alloc): what the shim hands to the C ABI, so that every per-tick copy is a
// DMA from / into pinned memory instead of a driver-staged pageable copy. Growing discards the contents.
template <typename T> class PinnedBuf {
 public:
  PinnedBuf() = default;
  PinnedBuf(const PinnedBuf &) = delete;
  PinnedBuf &operator=(const PinnedBuf &) = delete;
  ~PinnedBuf() { esikf_host_free(p_); }
  T *get(size_t n) {
    if (n > cap_) {
      esikf_host_free(p_);
      cap_ = n + n / 4 + 16;
      p_ = static_cast<T *>(esikf_host_alloc(cap_ * sizeof(T)));
      if (!p_) cap_ = 0;
    }
    return p_;
  }
  T *data() { return p_; }

 private:
  T *p_ = nullptr;
  size_t cap_ = 0;
};

// The outcome of a manager's last call (the reference's calls return void): an esikf_status, and the message when it failed;
// and the pinned block the manager's calls stage through.
struct CallStatus {
  int last_status_ = 0;
  std::string last_error_;

 protected:
  // records the esikf_* return code of a call on ctx, with the context's message when it is an error; returns the code. A
  // failed call may leave a copy from the manager's pinned block queued, so an error also drains the stream (fl2_shim.cpp).
  int Record(esikf_ctx *ctx, int status) {
    last_status_ = status;
    if (status) last_error_ = esikf_last_error(ctx), esikf_synchronize(ctx);
    return status;
  }
  void StagingFailed() { last_status_ = ESIKF_ERR_CUDA, last_error_ = "pinned staging allocation failed"; }
  PinnedBuf<uint8_t> block_;  // every call's inputs and answers, laid out per call (lay_out_staging); nothing is kept across calls
};

class VoxelMapManager : public CallStatus {
 public:
  VoxelMapConfig config_setting_;
  VoxelMap &voxel_map_;
  std::vector<PointXYZ> feats_down_body_;
  int feats_down_size_ = 0;
  int effct_feat_num_ = 0;
  M3D extR_;
  V3D extT_;
  StatesGroup state_;
  V3D position_last_;
  std::vector<M3D> cross_mat_list_, body_cov_list_;
  std::vector<pointWithVar> pv_list_;
  std::vector<PointToPlane> ptpl_list_;
  bool fill_point_lists_ = true;   // pv_list_ / ptpl_list_ / cross_mat_list_ / body_cov_list_ filled by StateEstimation (off: state_ only)
  bool lazy_point_lists_ = false;  // with fill_point_lists_: fill them on MaterializePointLists() instead of inside StateEstimation —
                                   // the 14 MB device->host copy of the per-point covariances and the host loops over the scan
                                   // only happen for callers that read the lists (LIVMapper's host-side UpdateVoxelMap does)
  int last_iters_ = 0;             // iterations executed by the last StateEstimation

  VoxelMapManager(VoxelMapConfig &config_setting, VoxelMap &voxel_map, int device = 0);
  ~VoxelMapManager();
  // call after BuildVoxelMap / UpdateVoxelMap / mapSliding changed voxel_map_: re-flatten, then patch the refitted plane
  // records in place (esikf_map_patch) when the candidate lists kept their shape, full upload (esikf_map_upload) otherwise
  void SyncDeviceMap();
  void MarkMapDirty() { map_synced_ = false; }
  int last_sync_patched_ = -1;     // planes patched by the last SyncDeviceMap, -1 = it was a full upload
  void StateEstimation(StatesGroup &state_propagat);  // include/voxel_map.h:229
  // ---- device-resident map: the octrees, point lists and refits live on the GPU (esikf_map_device_*); voxel_map_ is not used
  // unless config_setting_.device_map_mirror_ makes it a read-only host mirror of the device map
  // and SyncDeviceMap is never needed. EnableDeviceMap once after construction, then the reference's own call sequence:
  //   BuildVoxelMap()              first LiDAR frame, from feats_down_body_ and state_      (include/voxel_map.h:231, LIVMapper.cpp:356-366)
  //   UpdateVoxelMap()             LIVMapper.cpp:413-424 in ONE call: world points + covariances with the posterior and the
  //                                update, all on the device (nothing but a status crosses PCIe)
  //   UpdateVoxelMap(input_points) the reference's signature (include/voxel_map.h:232) with host lists
  void EnableDeviceMap();
  bool device_map_ = false;
  bool device_map_mirror_ = false;  // voxel_map_ mirrors the device map (config_setting_.device_map_mirror_ at EnableDeviceMap)
  // false once a build / update / slide, or the export or apply after it, failed: the mirror is then empty and every later
  // call reports ESIKF_ERR_STATE until EnableDeviceMap() starts a new map (an export holds one tick's roots only)
  bool mirror_valid_ = false;
  void BuildVoxelMap();
  void UpdateVoxelMap();
  void UpdateVoxelMap(const std::vector<pointWithVar> &input_points);
  void mapSliding();  // include/voxel_map.h:247 / src/voxel_map.cpp:924-948 (device-resident map); uses position_last_, sliding_thresh, half_map_size
  V3D last_slide_position;
  void MaterializePointLists();                       // fills the four lists from the last StateEstimation (idempotent per call of it)
  // The world cloud of this LIO tick for the coloured scan VIOManager::ColorizeFrameWorld publishes (LIVMapper.cpp:435-443):
  // every point of `dense_scan` (feats_undistort, dense_map_en = true) or, with nullptr, of feats_down_body_ as the last
  // StateEstimation left it on the device (dense_map_en = false), moved to the world frame with state_. Call after
  // StateEstimation, once per LIO tick.
  void SetWorldCloud(const std::vector<PointXYZ> *dense_scan = nullptr);
  // The VIO front end's find_correspond lookups on the device map, mirror or no mirror (esikf_map_device_find): for the n points
  // pts, the root voxel by the call site's key rule (ESIKF_FIND_RULE_PATCH: updateReferencePatch, ESIKF_FIND_RULE_RAYCAST: the
  // retrieval's ray casting), then find_correspond. status[i] = ESIKF_FIND_*; planes[i] = the found node's plane_ptr_ as the
  // callers read it (center_, normal_, plane_var_ as 6 x 6, d_, radius_, is_plane_), a default VoxelPlane where no root exists.
  void FindCorrespond(int n, const V3D *pts, int rule, uint8_t *status, VoxelPlane *planes);
  esikf_ctx *context() { return ctx_; }

 private:
  esikf_ctx *ctx_ = nullptr;
  FlatVoxelMap flat_;  // the host map as the device holds it: SyncDeviceMap diffs against it, MaterializePointLists reads its planes
  bool map_synced_ = false, device_has_map_ = false;
  // the association of the last StateEstimation, which a lazy MaterializePointLists reads after the calls in between
  PinnedBuf<int32_t> st_match_, st_normal_;
  PinnedBuf<float> st_dis_;
  bool lists_pending_ = false;
  // the host mirror: export of the last device build / update applied to voxel_map_ (cleared when either fails)
  void UpdateMirror();
  void InvalidateMirror();
  int32_t exp_roots_cap_ = 1024, exp_nodes_cap_ = 4096;  // what the export is requested with (grown from the ticks seen)
};

// include/vio.h:26-57 restated over flat storage
struct SubSparseMap {
  std::vector<float> errors;
  std::vector<std::vector<float>> warp_patch;  // [i][level*64 + row*8 + col]
  std::vector<int> search_levels;
  std::vector<V3D> voxel_points_pos;           // voxel_points[i]->pos_
  std::vector<double> inv_expo_list;
  std::vector<int> candidate_index;            // VIOManager::SelectSubSparseMap: the candidate each entry came from
};

// One candidate of VIOManager::SelectSubSparseMap: a visual point that passed the retrieval's depth-continuity check
// (src/vio.cpp:614-640) and the reference feature chosen for it (:645-697). Inputs as esikf_vio_select_patches.
struct SubMapCandidate {
  int32_t ref_img_index;  // into VIOManager::SetReferenceImages
  int32_t ref_level;      // Feature::level_ (depth form)
  int32_t ref_key;        // Feature::id_, the warp_map key (depth form)
  int32_t pad_;
  double px_ref[2];       // Feature::px_
  double ref_f[3];        // Feature::f_ (depth form)
  double ref_pos[3];      // Feature::pos() (depth form)
  double pos_w[3];        // VisualPoint::pos_
  double normal_w[3];     // VisualPoint::normal_ (homography form)
  double T_ref_w[12];     // Feature::T_f_w_ as R (row-major) and t
  double ref_inv_expo;    // Feature::inv_expo_time_
  double pc[2];           // new_frame_->w2c(pos_), computed by the retrieval at :614
};

struct GrayImage { const uint8_t *data = nullptr; int cols = 0, rows = 0; };  // cv::Mat CV_8UC1 continuous
struct BgrImage { const uint8_t *data = nullptr; int cols = 0, rows = 0; };   // cv::Mat CV_8UC3 continuous (img_rgb)
struct PointXYZRGB { float x, y, z; uint8_t r, g, b; };                          // pcl::PointXYZRGB's fields as published
// One new visual map point of VIOManager::GenerateVisualMapPoints: what generateVisualMapPoints (src/vio.cpp:864-890) builds
// its VisualPoint and Feature from. INTEGRATION.md §2 shows the objects made from it.
struct NewVisualPoint {
  int32_t source;    // index into pg, or ESIKF_GEN_ADD_FROM | index into add_from_voxel_map
  int32_t cell;      // grid cell
  double pos[3];     // VisualPoint::pos_ (pt_var.point_w)
  double pc[2];      // new_frame_->w2c(pos_): Feature::px_
  double normal[3];  // VisualPoint::normal_ (pt_var.normal, negated when cos_theta < 0)
  double var[9];     // VisualPoint::covariance_ (pt_var.var, row-major)
  float score;       // scan_value of the cell (vk::shiTomasiScore)
  float patch[64];   // getImagePatch(img, pc, patch, 0): Feature::patch_
};
// The oldest observation of a visual sub-map entry, pt->obs_.back() (addFrameRef pushes at the front): what
// VIOManager::UpdateVisualMapPoints compares the current frame with.
struct LastObservation {
  double T_f_w[12];  // Feature::T_f_w_: R row-major, then t
  double px[2];      // Feature::px_
};
// One new observation of VIOManager::UpdateVisualMapPoints: what updateVisualMapPoints (src/vio.cpp:954-964) builds its
// Feature from. INTEGRATION.md §2 shows the Feature made from it.
struct NewObservation {
  int32_t entry;     // index into visual_submap (voxel_points, search_levels)
  double pc[2];      // new_frame_->w2c(pt->pos_): Feature::px_
  float patch[64];   // getImagePatch(img, pc, patch, 0): Feature::patch_
};

// One observation (Feature) of a visual point as updateReferencePatch scores it: VIOManager::ScoreReferencePatches' input.
struct PatchObservation {
  double T_f_w[12];  // Feature::T_f_w_: R row-major, then t
  float patch[64];   // Feature::patch_
  float mean;        // Feature::mean_
  int32_t id;        // Feature::id_
};
// One visual point whose patches updateReferencePatch scores: pos_ and the normal_ the plane half left.
struct ScoredPoint {
  double pos[3];
  double normal[3];
};
// One observation (Feature) of a visual point as the device's observation store keeps it: VIOManager::AddVisualPoints' input.
struct StoredObservation {
  double px[2];      // Feature::px_
  double T_f_w[12];  // Feature::T_f_w_: R row-major, then t
  float patch[64];   // Feature::patch_
  int32_t id;        // Feature::id_
  float mean;        // Feature::mean_
  float score;       // Feature::score_
};

class VIOManager : public CallStatus {
 public:
  StatesGroup *state = nullptr, *state_propagat = nullptr;  // raw pointers into LIVMapper (LIVMapper.cpp:135-136)
  SubSparseMap *visual_submap = nullptr;
  int total_points = 0;
  int patch_size = 8, patch_pyrimid_level = 4, max_iterations = 5;
  double img_point_cov = 100;
  bool exposure_estimate_en = true;
  esikf_camera cam{};
  M3D Rcl;
  V3D Pcl;
  M3D extR;  // setImuToLidarExtrinsic / setLidarToCameraExtrinsic (src/vio.cpp:29-39)
  V3D extT;
  // retrieval gate (LIVMapper.cpp:59,70; include/vio.h:101,109). ncc_thre has no default in the reference (the node never
  // reads it and ncc_en stays false); 0 here, which rejects only anti-correlated patches when ncc_en is set.
  bool normal_en = true, ncc_en = false;
  double outlier_threshold = 1000, ncc_thre = 0;
  int last_total_iters_ = 0;  // iterations executed by the last computeJacobianAndUpdateEKF
  int64_t submap_uploads_ = 0;  // sub-map uploads (esikf_vio_set_patches) made by computeJacobianAndUpdateEKF
  // The per-patch mirrors below are called once per point and level by the reference's retrieval code: the image they are
  // handed is uploaded only when it is not the one of the previous call (same pixel pointer and size). A caller that rewrites
  // the pixels in place calls InvalidatePatchImages().
  void InvalidatePatchImages() { patch_img_ = patch_ref_img_ = nullptr; }

  explicit VIOManager(esikf_ctx *shared_ctx);  // shares the device context (and stream) of the VoxelMapManager
  void initializeVIO();                         // src/vio.cpp:41-160 (the parts the update needs)
  void computeJacobianAndUpdateEKF(const GrayImage &img);  // include/vio.h:153
  // Feature::img_ of the reference frames the candidates of SelectSubSparseMap address by ref_img_index.
  void SetReferenceImages(const GrayImage *imgs, int n);
  // The per-candidate tail of retrieveFromVisualSparseMap (src/vio.cpp:699-770) on the device for n candidates in grid-cell
  // order, against the current frame `img` at pose T_cur_w (new_frame_->T_f_w_, R row-major then t) and state->inv_expo_time:
  // warp form by normal_en, gates by outlier_threshold / ncc_en / ncc_thre. Fills visual_submap (voxel_points_pos,
  // search_levels, inv_expo_list, errors, candidate_index; warp_patch stays empty, see MaterializeWarpPatches) and
  // total_points. The warp patches stay on the device: the next computeJacobianAndUpdateEKF on the same visual_submap with
  // the same total_points uploads only the image and the states.
  void SelectSubSparseMap(const SubMapCandidate *candidates, int n, const GrayImage &img, const double T_cur_w[12]);
  // Fills visual_submap->warp_patch of the last SelectSubSparseMap (the same patches the device holds), for callers that read
  // them on the host. Idempotent per selection.
  void MaterializeWarpPatches();
  // Per-patch helpers with the reference's signatures (include/vio.h:151, 161-162; V2D / Matrix2d as plain arrays). One
  // launch and one small read-back per call: the frame path should use the batched esikf_vio_get_image_patch /
  // esikf_vio_warp_patches.
  void getImagePatch(const GrayImage &img, const double pc[2], float *patch_tmp, int level);
  void warpAffine(const double A_cur_ref[4] /* row-major 2x2 */, const GrayImage &img_ref, const double px_ref[2], int level_ref, int search_level,
                  int pyramid_level, int halfpatch_size, float *patch);
  // LIVMapper::publish_frame_world (src/LIVMapper.cpp:1140-1173) on the device: the world cloud of the last
  // VoxelMapManager::SetWorldCloud, coloured from img_rgb (the camera's size) with the frame pose of *state (the VIO
  // posterior after computeJacobianAndUpdateEKF), the points closer than blind_rgb_points dropped. Fills laserCloudWorldRGB
  // in the reference's order. Call once per VIO tick, after computeJacobianAndUpdateEKF.
  void ColorizeFrameWorld(const BgrImage &img_rgb, double blind_rgb_points, std::vector<PointXYZRGB> &laserCloudWorldRGB);
  // generateVisualMapPoints (src/vio.cpp:804-906) on the device, up to the object creation: the new visual map points of this
  // frame, at most one per grid cell, in cell order. type_map: grid_num after the retrieval, one entry per cell, nonzero
  // where it is TYPE_MAP; grid_size .. border as initializeVIO left them (vio.cpp:66-80, 154). pg == nullptr: the pv list
  // the last VoxelMapManager::UpdateVoxelMap() left on the device (_pv_list), else those points (point_w, normal, var).
  // add_from_voxel_map: visual_submap->add_from_voxel_map (point_w, normal), or nullptr. The frame pose is that of *state
  // and the image the one of the last computeJacobianAndUpdateEKF. Call once per VIO tick, after it.
  void GenerateVisualMapPoints(const std::vector<uint8_t> &type_map, int grid_size, int grid_n_width, int grid_n_height, int border,
                               const std::vector<pointWithVar> *pg, const std::vector<pointWithVar> *add_from_voxel_map,
                               std::vector<NewVisualPoint> &new_points);
  // updateVisualMapPoints (src/vio.cpp:908-967) on the device, up to the Feature objects and the eviction at 30 observations:
  // which entries of the visual sub-map on the device (the last SelectSubSparseMap or computeJacobianAndUpdateEKF, total_points
  // entries) this frame becomes a new observation of. converged: pt->is_converged_ and last_obs: pt->obs_.back() of every
  // entry, indexed like visual_submap. Fills update_flag (one per entry, as updateReferencePatch reads it) and new_obs (the
  // added entries in entry order). The frame pose is that of *state and the image the one of the last
  // computeJacobianAndUpdateEKF. Call once per VIO tick, after it.
  void UpdateVisualMapPoints(const std::vector<uint8_t> &converged, const std::vector<LastObservation> &last_obs, std::vector<uint8_t> &update_flag,
                             std::vector<NewObservation> &new_obs);
  // The scan side of retrieveFromVisualSparseMap (src/vio.cpp:386-428) on the device: keys receives the scan's distinct 0.5 m
  // voxel keys in first-occurrence order (insert them into sub_feat_map in this order: it then iterates as the reference's),
  // and the device keeps the depth image for CheckDepthContinuity. pg == nullptr: the pv list the last
  // VoxelMapManager::UpdateVoxelMap() left on the device (_pv_list), else those points. border as initializeVIO left it; the
  // frame pose is that of *state (the VIO prior). Call at the start of the VIO tick.
  void RetrieveScanVoxels(int border, const std::vector<pointWithVar> *pg, std::vector<VOXEL_LOCATION> &keys);
  // The depth-continuity check of :614-640 for n retrieved points (pos: VisualPoint::pos_, pc: the w2c(pos_) the map-side walk
  // computed, 3 and 2 doubles each) against the depth image of the last RetrieveScanVoxels: discontinuous[i] = depth_continous.
  void CheckDepthContinuity(int n, const double *pos, const double *pc, std::vector<uint8_t> &discontinuous);
  // The patch scoring of updateReferencePatch (src/vio.cpp:1036-1097) on the device (esikf_vio_score_ref_patches), after the
  // plane half: point i of pts owns obs[first[i] .. first[i + 1]), in obs_ order. Fills score (Feature::score_) and mean
  // (Feature::mean_ afterwards) per observation, and ref per point: the position of the new ref_patch within its list, or -1
  // when ref_patch and has_ref_patch_ stay as they were. first has pts.size() + 1 entries, first[0] = 0 and the last obs.size().
  void ScoreReferencePatches(const std::vector<int32_t> &first, const std::vector<ScoredPoint> &pts, const std::vector<PatchObservation> &obs,
                             std::vector<float> &score, std::vector<float> &mean, std::vector<int32_t> &ref);

  // The visual map's observations kept on the device (esikf_vmap_*, DESIGN.md §3 K14); the host's VisualPoint / Feature objects
  // mirror them from what these calls return (INTEGRATION.md §3) and need no patch_. EnableDeviceObservations creates an
  // empty store with room for `capacity` points (it grows by doubling), replacing any store the context held.
  void EnableDeviceObservations(int64_t capacity);
  // New points (generateVisualMapPoints' winners, or an existing host map): point i owns obs[first[i] .. first[i + 1]) in obs_
  // order and ref[i], the position of ref_patch or -1. point_ids receives their store ids.
  void AddVisualPoints(const std::vector<int32_t> &first, const std::vector<StoredObservation> &obs, const std::vector<int32_t> &ref,
                       std::vector<int32_t> &point_ids);
  // updateVisualMapPoints (src/vio.cpp:914-964) on the store: entry i of visual_submap is store point point_ids[i], with
  // is_converged_ converged[i]; the frame pose is *state's and the new Features' id_ is frame_id. update_flag and new_obs as the
  // overload above; per entry evicted (the list position deleteFeatureRef removed, -1 none) and count (the count afterwards).
  void UpdateVisualMapPoints(const std::vector<int32_t> &point_ids, const std::vector<uint8_t> &converged, int32_t frame_id,
                             std::vector<uint8_t> &update_flag, std::vector<NewObservation> &new_obs, std::vector<int32_t> &evicted,
                             std::vector<int32_t> &count);
  // The patch scoring of updateReferencePatch on the store (esikf_vmap_score): score_ and mean_ stay on the device; ref[i] is
  // the new ref_patch's position, or -1 when ref_patch and has_ref_patch_ stay as they were.
  void ScoreReferencePatches(const std::vector<int32_t> &point_ids, const std::vector<ScoredPoint> &pts, std::vector<int32_t> &ref);
  // The reference feature of retrieveFromVisualSparseMap (:651-697) for n retrieved points (pos: pos_, 3 doubles each) seen
  // from frame_pos (new_frame_->pos()): ref[i] is its position in obs_, -1 where the point is skipped (getCloseViewObs false)
  // or the reference leaves ref_ftr unset. With normal_en the first two cases of :655-689 set the point's ref on the device.
  void ChooseReferenceFeatures(const std::vector<int32_t> &point_ids, const double *pos, const double frame_pos[3], bool normal_en,
                               std::vector<int32_t> &ref);

 private:
  const uint8_t *patch_img_ = nullptr, *patch_ref_img_ = nullptr;  // what the per-patch helpers uploaded last
  int patch_img_w_ = 0, patch_img_h_ = 0, patch_ref_w_ = 0, patch_ref_h_ = 0;
  esikf_ctx *ctx_ = nullptr;
  // the sub-map SelectSubSparseMap left on the device, and what MaterializeWarpPatches needs to rebuild its patches
  const SubSparseMap *selected_submap_ = nullptr;
  int selected_count_ = -1;
  std::vector<int32_t> sel_ref_idx_, sel_sl_;
  std::vector<double> sel_px_, sel_A_;
  std::vector<GrayImage> ref_imgs_;  // SetReferenceImages (the caller keeps the pixels, as Feature::img_ does)
  int32_t rgb_cap_ = 0;              // ColorizeFrameWorld's answers are requested with room for the largest coloured scan seen
  int32_t keys_cap_ = 0;             // the resident scan's largest key count seen
  bool ref_imgs_current_ = false;    // false once the per-patch warpAffine replaced the device's reference images
};

}  // namespace fl2b200
