// The call sequence of LIVMapper's LIO + VIO ticks (src/LIVMapper.cpp:351-428, 300-320) through the shim classes of
// fast_livo2_b200/csrc/fl2_shim.hpp — a compile-checked companion to INTEGRATION.md. The voxel map is DEVICE-RESIDENT here:
// BuildVoxelMap on the first frame, StateEstimation + UpdateVoxelMap() every tick; no plane, point list or key crosses PCIe
// and no host-side flatten / diff / patch runs between ticks (the host-owned form — SyncDeviceMap() after the reference's own
// UpdateVoxelMap — stays available, INTEGRATION.md §3). The scene is a floor patch and a trivial image: it shows WHICH calls
// happen WHEN and who owns what, not a meaningful estimate. Needs an H100 to run; without one the managers report an error.
//   g++ -std=c++17 -Iinclude examples/tick_loop.cpp -Lfast_livo2_b200 -lfl2_shim -lesikf_b200 -Wl,-rpath,$PWD/fast_livo2_b200 -o tick_loop
#include <cstdio>
#include <cstring>
#include <vector>

#include "../fast_livo2_b200/csrc/fl2_shim.hpp"

using namespace fl2b200;

static std::vector<PointXYZ> floor_scan(int n, float jitter) {
  std::vector<PointXYZ> pts(n);
  for (int i = 0; i < n; i++) {
    const float u = (float)(i % 40) * 0.05f, v = (float)(i / 40) * 0.05f;
    pts[i] = {u - 1.0f, v - 1.0f, -1.0f + jitter * (float)((i * 37) % 11 - 5) * 0.001f};
  }
  return pts;
}

int main() {
  // ---- node start-up (LIVMapper::initializeComponents): configuration; voxel_map stays empty — the device owns the map
  VoxelMapConfig cfg;
  cfg.max_voxel_size_ = 0.5, cfg.max_layer_ = 2, cfg.max_iterations_ = 5, cfg.sigma_num_ = 3.0, cfg.dept_err_ = 0.02, cfg.beam_err_ = 0.05;
  cfg.planner_threshold_ = 0.0025, cfg.max_points_num_ = 50, cfg.layer_init_num_ = {5, 5, 5, 5, 5};
  cfg.device_root_capacity_ = 1 << 16;
  VoxelMap voxel_map;
  VoxelMapManager voxelmap_manager(cfg, voxel_map, /*device*/ 0);
  if (voxelmap_manager.last_status_) {
    std::printf("no usable device (%s) — the managers never fall back to the CPU\n", voxelmap_manager.last_error_.c_str());
    return 0;
  }
  voxelmap_manager.EnableDeviceMap();
  voxelmap_manager.lazy_point_lists_ = true;             // pv_list_ & co. only when somebody reads them (MaterializePointLists)
  VIOManager vio_manager(voxelmap_manager.context());    // shares the device context and stream
  StatesGroup _state, state_propagat;                    // LIVMapper members; the managers hold pointers / copies like the reference
  vio_manager.state = &_state, vio_manager.state_propagat = &state_propagat;
  vio_manager.cam.model = 0, vio_manager.cam.width = 64, vio_manager.cam.height = 48;
  vio_manager.cam.fx = vio_manager.cam.fy = 60.0, vio_manager.cam.cx = 32.0, vio_manager.cam.cy = 24.0;
  vio_manager.patch_pyrimid_level = 2;
  vio_manager.initializeVIO();
  // the visual map's observations on the device (INTEGRATION.md §3): the sub-map's one entry is store point 0, observed once
  // from the identity pose at its reference pixel; the host's VisualPoint / Feature objects mirror the store without patch_
  vio_manager.EnableDeviceObservations(1 << 10);
  std::vector<int32_t> store_ids;
  vio_manager.AddVisualPoints({0, 1}, {StoredObservation{{32.0, 24.0}, {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0}, {}, 0, 0.0f, 0.0f}}, {-1}, store_ids);
  std::printf("observation store: status %d, %zu points\n", vio_manager.last_status_, store_ids.size());

  // ---- first LiDAR frame (LIVMapper.cpp:356-366): the map is built from the scan at the initial pose
  voxelmap_manager.feats_down_body_ = floor_scan(1600, 1.0f);
  voxelmap_manager.feats_down_size_ = (int)voxelmap_manager.feats_down_body_.size();
  voxelmap_manager.state_ = _state;                      // :257
  voxelmap_manager.BuildVoxelMap();                      // :364  (on the device)
  std::printf("BuildVoxelMap: status %d\n", voxelmap_manager.last_status_);

  for (int tick = 1; tick <= 3; tick++) {
    // ---- LIO tick (LIVMapper::handleLIO) after IMU propagation and down-sampling
    voxelmap_manager.feats_down_body_ = floor_scan(1600, 1.0f + 0.1f * tick);
    voxelmap_manager.feats_down_size_ = (int)voxelmap_manager.feats_down_body_.size();
    voxelmap_manager.state_ = _state;                    // :257
    voxelmap_manager.StateEstimation(state_propagat);    // :370
    _state = voxelmap_manager.state_;                    // :371
    voxelmap_manager.UpdateVoxelMap();                   // :413-424 in one call: world points, covariances, octree update, refits
    // :435-443, the world cloud of the coloured scan with the LIO posterior: dense_map_en = true hands over feats_undistort
    // (here a wall 3 m in front of the camera); dense_map_en = false would be SetWorldCloud() on the scan itself
    std::vector<PointXYZ> feats_undistort = floor_scan(1600, 0.0f);
    for (PointXYZ &p : feats_undistort) p.z = 3.0f;
    voxelmap_manager.SetWorldCloud(&feats_undistort);
    std::printf("tick %d LIO: status %d, effective points %d\n", tick, voxelmap_manager.last_status_, voxelmap_manager.effct_feat_num_);

    // ---- VIO tick (LIVMapper::handleVIO -> processFrame -> computeJacobianAndUpdateEKF, vio.cpp:1810)
    std::vector<uint8_t> pixels(64 * 48, 128);
    GrayImage img{pixels.data(), 64, 48};
    // retrieveFromVisualSparseMap (vio.cpp:352-782). The scan side runs on the device, from the pv list UpdateVoxelMap left
    // there: the scan's voxel keys (inserted into the persistent sub_feat_map in the returned order) and the depth image, with
    // the frame pose of *state; border (patch_size_half + 1) << patch_pyrimid_level as initializeVIO leaves it. The walk over
    // feat_map, ray casting and the choice of each point's reference feature stay on the host (INTEGRATION.md §2); the depth
    // check of the retrieved points runs on the device; the per-candidate tail runs in SelectSubSparseMap.
    std::vector<VOXEL_LOCATION> scan_voxels;
    vio_manager.RetrieveScanVoxels(5 << 2, nullptr, scan_voxels);
    std::printf("tick %d scan voxels: status %d, %zu keys\n", tick, vio_manager.last_status_, scan_voxels.size());
    std::vector<uint8_t> ref_pixels(64 * 48, 128);
    GrayImage ref_img{ref_pixels.data(), 64, 48};        // Feature::img_ of the one reference frame
    vio_manager.SetReferenceImages(&ref_img, 1);
    SubMapCandidate cand{};                              // one visual point 2 m ahead, seen from the same pose
    cand.ref_img_index = 0, cand.ref_level = 0, cand.ref_key = 7;
    cand.px_ref[0] = 32.0, cand.px_ref[1] = 24.0, cand.ref_f[2] = 1.0, cand.pos_w[2] = 2.0, cand.normal_w[2] = -1.0;
    cand.T_ref_w[0] = cand.T_ref_w[4] = cand.T_ref_w[8] = 1.0, cand.ref_inv_expo = 1.0;
    cand.pc[0] = 32.0, cand.pc[1] = 24.0;                // new_frame_->w2c(pos_), :614
    std::vector<uint8_t> depth_discontinuous;            // :614-640 for the one retrieved point: 1 drops it
    vio_manager.CheckDepthContinuity(1, cand.pos_w, cand.pc, depth_discontinuous);
    std::printf("tick %d depth check: status %d, discontinuous %d\n", tick, vio_manager.last_status_, depth_discontinuous.empty() ? -1 : (int)depth_discontinuous[0]);
    const double T_cur_w[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};  // new_frame_->T_f_w_
    SubSparseMap submap;
    vio_manager.visual_submap = &submap;
    vio_manager.SelectSubSparseMap(&cand, 1, img, T_cur_w);  // fills submap and total_points; patches stay on the device
    std::printf("tick %d retrieval: status %d, %d of 1 candidates kept\n", tick, vio_manager.last_status_, vio_manager.total_points);
    state_propagat = _state;
    vio_manager.computeJacobianAndUpdateEKF(img);
    std::printf("tick %d VIO: status %d, patch error %.3f\n", tick, vio_manager.last_status_, submap.errors.empty() ? -1.0f : submap.errors[0]);
    // publish_frame_world (LIVMapper.cpp:1140-1173): the LIO tick's world cloud coloured from img_rgb at the VIO posterior
    std::vector<uint8_t> bgr(64 * 48 * 3);
    for (size_t i = 0; i < bgr.size(); i++) bgr[i] = (uint8_t)(i % 3 == 0 ? 40 : i % 3 == 1 ? 120 : 200);
    std::vector<PointXYZRGB> laserCloudWorldRGB;
    vio_manager.ColorizeFrameWorld(BgrImage{bgr.data(), 64, 48}, /*blind_rgb_points*/ 0.01, laserCloudWorldRGB);
    std::printf("tick %d coloured scan: status %d, %zu points\n", tick, vio_manager.last_status_, laserCloudWorldRGB.size());
    // generateVisualMapPoints (vio.cpp:804-906) on the scan the device holds: grid of initializeVIO (vio/grid_size 5,
    // grid_n_height 17 on a 64 x 48 image: 2-pixel cells, 32 x 24) and border (patch_size_half + 1) << patch_pyrimid_level;
    // the retrieval marked the candidate's cell TYPE_MAP. The VisualPoint / Feature objects are the caller's (INTEGRATION.md §2).
    std::vector<uint8_t> grid_num(32 * 24, 0);
    grid_num[12 * 32 + 16] = 1;
    std::vector<NewVisualPoint> new_points;
    vio_manager.GenerateVisualMapPoints(grid_num, 2, 32, 24, 5 << 2, nullptr, nullptr, new_points);
    std::printf("tick %d new visual map points: status %d, %zu points\n", tick, vio_manager.last_status_, new_points.size());
    // updateVisualMapPoints (vio.cpp:908-967): the sub-map's one entry was last observed from the identity pose at its
    // reference pixel; whether this frame becomes a new observation of it. The Feature objects and the eviction at 30
    // observations are the caller's (INTEGRATION.md §2).
    std::vector<uint8_t> converged(vio_manager.total_points, 0), update_flag;
    std::vector<LastObservation> last_obs(vio_manager.total_points, LastObservation{{1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0}, {32.0, 24.0}});
    std::vector<NewObservation> new_obs;
    vio_manager.UpdateVisualMapPoints(converged, last_obs, update_flag, new_obs);
    std::printf("tick %d new observations: status %d, %zu of %d entries\n", tick, vio_manager.last_status_, new_obs.size(), vio_manager.total_points);
    // updateReferencePatch (vio.cpp:969-1034): the plane under each sub-map entry that passes the four skips, in one lookup
    // on the device map (no host mirror); the normal refinement stays the caller's (INTEGRATION.md §3).
    std::vector<V3D> ref_pos(1);
    ref_pos[0][0] = 0.3, ref_pos[0][1] = 0.2, ref_pos[0][2] = 0.0;  // the candidate's pos_, on the floor
    uint8_t found[1];
    VoxelPlane plane[1];
    voxelmap_manager.FindCorrespond(1, ref_pos.data(), ESIKF_FIND_RULE_PATCH, found, plane);
    std::printf("tick %d reference-patch lookup: status %d, answer %d\n", tick, voxelmap_manager.last_status_, (int)found[0]);
    // ... and the patch scoring (vio.cpp:1036-1097) of the same entry in one call: its six observations, seen from the
    // identity pose and from five poses stepped along x, with the floor's normal; the caller writes score_, mean_ and the
    // chosen ref_patch back into its Feature / VisualPoint objects (INTEGRATION.md §3).
    std::vector<ScoredPoint> scored(1, ScoredPoint{{0.3, 0.2, 0.0}, {0.0, 0.0, 1.0}});
    std::vector<PatchObservation> obs(6);
    for (int k = 0; k < 6; k++) {
      PatchObservation &o = obs[k];
      const double T[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0.1 * k, 0, 2.0};
      memcpy(o.T_f_w, T, sizeof(T));
      for (int t = 0; t < 64; t++) o.patch[t] = (float)(100 + (t * (k + 3)) % 17);
      o.mean = 0.0f, o.id = tick * 10 + k;
    }
    std::vector<float> score, mean;
    std::vector<int32_t> ref;
    vio_manager.ScoreReferencePatches(std::vector<int32_t>{0, 6}, scored, obs, score, mean, ref);
    std::printf("tick %d reference patch: status %d, observation %d\n", tick, vio_manager.last_status_, ref.empty() ? -1 : ref[0]);
    // the same three steps on the device's observation store: the new points join it, the sub-map entry's oldest observation
    // is read and its list edited where it lies, and its patches are scored in place; the retrieval's reference feature of
    // the entry (getCloseViewObs from the frame's position) is read from it too
    std::vector<int32_t> first(new_points.size() + 1, 0), none(new_points.size(), -1), ids;
    std::vector<StoredObservation> born(new_points.size());
    for (size_t i = 0; i < new_points.size(); i++) {
      StoredObservation &o = born[i];
      memcpy(o.px, new_points[i].pc, sizeof(o.px)), memcpy(o.patch, new_points[i].patch, sizeof(o.patch));
      const double T[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
      memcpy(o.T_f_w, T, sizeof(T));
      o.id = tick, o.mean = 0.0f, o.score = 0.0f;
      first[i + 1] = (int32_t)i + 1;
    }
    vio_manager.AddVisualPoints(first, born, none, ids);
    std::printf("tick %d store add: status %d, %zu points\n", tick, vio_manager.last_status_, ids.size());
    std::vector<int32_t> sub_ids(vio_manager.total_points, store_ids.empty() ? 0 : store_ids[0]), evicted, count;
    vio_manager.UpdateVisualMapPoints(sub_ids, converged, tick, update_flag, new_obs, evicted, count);
    std::printf("tick %d store update: status %d, %zu new, count %d\n", tick, vio_manager.last_status_, new_obs.size(), count.empty() ? -1 : count[0]);
    vio_manager.ScoreReferencePatches(std::vector<int32_t>(1, sub_ids.empty() ? 0 : sub_ids[0]), scored, ref);
    std::printf("tick %d store reference patch: status %d, observation %d\n", tick, vio_manager.last_status_, ref.empty() ? -1 : ref[0]);
    const double frame_pos[3] = {0.0, 0.0, 0.0};
    vio_manager.ChooseReferenceFeatures(std::vector<int32_t>(1, 0), scored[0].pos, frame_pos, false, ref);
    std::printf("tick %d store reference feature: status %d, observation %d\n", tick, vio_manager.last_status_, ref.empty() ? -1 : ref[0]);
  }
  // somebody wants the warp patches of the last selection on the host after all
  vio_manager.MaterializeWarpPatches();
  std::printf("warp_patch %zu entries\n", vio_manager.visual_submap->warp_patch.size());
  // somebody wants the per-point lists of the last tick after all (e.g. publishing the effective points)
  voxelmap_manager.MaterializePointLists();
  std::printf("pv_list_ %zu entries, ptpl_list_ %zu\n", voxelmap_manager.pv_list_.size(), voxelmap_manager.ptpl_list_.size());
  return 0;
}
