/*
 * esikf_b200.h — C ABI of the CUDA ESIKF measurement update for FAST-LIVO2 (H100, sm_90a).
 *
 * Drop-in boundary for the two calls LIVMapper makes per tick (reference @ 0d2c034):
 *   VoxelMapManager::StateEstimation(StatesGroup&)        include/voxel_map.h:229, called at src/LIVMapper.cpp:370
 *   VIOManager::computeJacobianAndUpdateEKF(cv::Mat img)  include/vio.h:153,      called at src/vio.cpp:1810
 * plus the per-frame producers of the VIO inputs named by the north star:
 *   VIOManager::getImagePatch                              include/vio.h:151  (src/vio.cpp:203-225)
 *   VIOManager::warpAffine / getWarpMatrixAffineHomography include/vio.h:161-162 (src/vio.cpp:252-318)
 *
 * Plain pointers and sizes only; every function returns 0 on success or a negative
 * esikf_status; nothing throws across this boundary. All `double*` state arguments use the
 * packed POD below (fp64, row-major). The library is CUDA-only: there is no CPU fallback, and
 * esikf_create fails with ESIKF_ERR_NO_DEVICE when no sm_90 (H100) device is usable.
 */
#ifndef ESIKF_B200_H_
#define ESIKF_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct esikf_ctx esikf_ctx;

enum esikf_status {
  ESIKF_OK = 0,
  ESIKF_ERR_NO_DEVICE = -1,   /* no CUDA device / wrong architecture */
  ESIKF_ERR_CUDA = -2,        /* a CUDA runtime call failed; see esikf_last_error */
  ESIKF_ERR_ARG = -3,         /* bad argument (null pointer, negative size, key out of range ...) */
  ESIKF_ERR_STATE = -4,       /* call order (e.g. lio_run before map_upload / set_scan) */
  ESIKF_ERR_COMM = -5         /* NCCL / peer-memory set-up failed, or a bounded in-kernel wait (grid barrier, grid mailbox, peer mailbox)
                                 expired: the update that reported it is invalid (returned by the fetch calls) */
};

/* StatesGroup (include/common_lib.h:126-223) as a packed POD, 386 doubles:
 *   [0:9) rot_end row-major | [9:12) pos_end | [12] inv_expo_time | [13:16) vel_end |
 *   [16:19) bias_g | [19:22) bias_a | [22:25) gravity | [25:386) cov 19x19 row-major
 * Error-state order (common_lib.h:167-206): dtheta(0:3) dp(3:6) dinv_expo(6) dv(7:10) dbg(10:13) dba(13:16) dg(16:19). */
#define ESIKF_STATE_DOUBLES 386

/* One plane of the adaptive voxel map: VoxelPlane (include/voxel_map.h:69-94) reduced to what
 * build_single_residual / the Jacobian loop read (src/voxel_map.cpp:721-754, 425-449).
 * plane_var holds the upper triangle (row-major, i<=j) of the 6x6 plane_var_. 256 bytes. */
typedef struct esikf_plane {
  double center[3];
  double normal[3];
  double plane_var[21];
  float d;       /* VoxelPlane::d_ */
  float radius;  /* VoxelPlane::radius_ */
  int32_t layer; /* depth of the node inside its root voxel (PointToPlane::layer_) */
  int32_t path;  /* 3 bits per layer: leaf index at layer 1 | leaf index at layer 2 << 3 | ... */
  int32_t pad[6];
} esikf_plane;

/* VoxelMapConfig (include/voxel_map.h:35-52), hot-path subset; loadVoxelConfig src/voxel_map.cpp:36-53 */
typedef struct esikf_lio_cfg {
  double voxel_size;      /* lio/voxel_size      max_voxel_size_ */
  double sigma_num;       /* lio/sigma_num */
  double dept_err;        /* lio/dept_err */
  double beam_err;        /* lio/beam_err */
  int32_t max_layer;      /* lio/max_layer */
  int32_t max_iterations; /* lio/max_iterations (<= 8) */
} esikf_lio_cfg;

/* extrinsics: LIVMapper.cpp:125-126 (extR_/extT_), vio.cpp:29-39,57-65 (Rcl/Pcl) */
typedef struct esikf_extrinsics {
  double extR[9]; /* lidar -> imu rotation, row-major */
  double extT[3];
  double Rcl[9]; /* lidar -> camera */
  double Pcl[3];
} esikf_extrinsics;

/* vk::AbstractCamera as used by the path (cam->world2cam at vio.cpp:1574, fx()/fy() at :45-46).
 * model 0 = Pinhole + radtan d[0..4] (config/camera_pinhole.yaml), 1 = EquidistantCamera k1..k4 in d[0..3]
 * (config/camera_fisheye_HILTI22.yaml). Intrinsics are already multiplied by the camera `scale`. */
typedef struct esikf_camera {
  int32_t model, width, height, pad_;
  double fx, fy, cx, cy;
  double d[5];
} esikf_camera;

/* vio/ parameters (LIVMapper.cpp:50-117): patch_size is fixed at 8 (every shipped config). */
typedef struct esikf_vio_cfg {
  double img_point_cov;
  int32_t patch_pyrimid_level; /* <= 8 */
  int32_t max_iterations;      /* <= 8 */
  int32_t exposure_estimate_en;
  int32_t inverse_composition_en; /* vio/inverse_composition_en (LIVMapper.cpp:60): updateStateInverse instead of updateState;
                                     needs esikf_vio_set_inverse_refs. 0 in every shipped config. */
} esikf_vio_cfg;

/* Per-call diagnostics (what the reference prints at src/voxel_map.cpp:404-405). */
typedef struct esikf_lio_stats {
  int32_t iters;                /* iterations executed */
  int32_t effct_feat_num[8];    /* matched points per iteration (global over all ranks) */
  int32_t converged[8];
  int32_t pad_;
  double total_residual[8];     /* sum |dis_to_plane| per iteration */
  double HTH[8][36];            /* 6x6 H^T R^-1 H per iteration */
  double HTz[8][6];
  double solution[8][19];
} esikf_lio_stats;

typedef struct esikf_vio_stats {
  int32_t total_iters;
  int32_t iters_per_level[8];
  int32_t accepted_per_level[8];
  int32_t pad_;
  float error_trace[8][8];      /* [level][iteration] mean squared photometric error */
  double HTH[8][8][49];         /* [level][iteration] 7x7 H^T H (accepted iterations) */
  double HTz[8][8][7];
  double solution[8][8][19];
} esikf_vio_stats;

/* ---------------------------------------------------------------- context */
int esikf_create(esikf_ctx **out, int device);
void esikf_destroy(esikf_ctx *ctx);
const char *esikf_last_error(const esikf_ctx *ctx);
/* The CUDA stream (cudaStream_t) every kernel of this context is launched on. */
void *esikf_stream(esikf_ctx *ctx);
int esikf_synchronize(esikf_ctx *ctx);
/* Page-locked host memory for callers that stage the per-tick buffers themselves (the C++ shim does): copies from / into
 * it are DMA transfers instead of driver-staged pageable copies. NULL on failure; free(NULL) is a no-op. */
void *esikf_host_alloc(size_t bytes);
void esikf_host_free(void *p);
/* Number of launches this context has enqueued since creation (bench.py "gpu_launches"). Each kernel launch counts one,
 * the persistent update kernel's single cooperative launch included, and each CUB device-wide call (a sort or a scan)
 * counts one, however many kernels it runs. A launch that fails to enqueue is not counted. */
int64_t esikf_launch_count(const esikf_ctx *ctx);
/* solve_mode: 0 = Woodbury 6x6/7x7 form of (H^T H + P^-1)^-1 (default), 1 = literal two 19x19
 * partial-pivot inversions as at src/voxel_map.cpp:468 / src/vio.cpp:1661. */
int esikf_set_solve_mode(esikf_ctx *ctx, int mode);
/* loop_mode: how the iteration loop of an update is driven. Results of all modes are bit-identical.
 *   2 (default; 1 is accepted as an alias) = one persistent cooperative kernel per update: every CTA keeps the state on
 *       chip, sums the per-CTA partial vectors after ONE grid exchange per iteration (LIO: a grid barrier, VIO: a tagged-word mailbox) and runs the gain solve itself. With
 *       peer GPUs attached (esikf_peer_attach) the same kernel also carries the NVLink exchange of the information vector.
 *   0 = one residual + one solve launch per iteration (also used with an NCCL communicator or kernel timing on). */
int esikf_set_loop_mode(esikf_ctx *ctx, int mode);
/* Measurement variants, OR-ed flags; 0 = none (default). Same results bit for bit.
 *   ESIKF_TUNE_STAGE_LDG : LIO plane records are brought into shared memory by coalesced half-warp __ldg copies instead of
 *                          one cp.async.bulk (TMA engine) per lane — the round-1 staging, kept to measure against.
 *   ESIKF_TUNE_VIO_TMA   : VIO tap footprints (the 11 x 11 strided taps of a patch, vio.cpp:1595-1631) are brought in by ONE
 *                          tiled TMA load per patch (cp.async.bulk.tensor.2d of 11 image rows, elementStrides {1, s}) instead
 *                          of four byte loads per lane. Needs an image row pitch that is a multiple of 16 bytes; otherwise,
 *                          for tap strides 16 / 32 and for footprints leaving the image the per-lane loads are used. */
#define ESIKF_TUNE_STAGE_LDG 1u
#define ESIKF_TUNE_VIO_TMA 2u
int esikf_set_tuning(esikf_ctx *ctx, uint32_t flags);
int esikf_set_extrinsics(esikf_ctx *ctx, const esikf_extrinsics *ext);
/* Only the lidar -> imu part (extR_, extT_ of VoxelMapManager, LIVMapper.cpp:125-126); the camera part set before is kept.
 * Cheap when nothing changed (no copy, no synchronisation): the LIO shim calls it every tick. */
int esikf_set_lidar_extrinsics(esikf_ctx *ctx, const double extR[9], const double extT[3]);

/* ---------------------------------------------------------------- voxel map mirror
 * Device mirror of `std::unordered_map<VOXEL_LOCATION, VoxelOctoTree*> voxel_map_`
 * (include/voxel_map.h:194). `keys` are n_roots x 3 int64 VOXEL_LOCATIONs; root r owns the
 * ordered candidate planes [first[r], first[r]+count[r]) — the DFS order in which
 * build_single_residual (src/voxel_map.cpp:771-784) visits the octree. */
int esikf_map_upload(esikf_ctx *ctx, const int64_t *keys, const int32_t *first, const int32_t *count, int32_t n_roots,
                     const esikf_plane *planes, int32_t n_planes, double voxel_size);
/* Overwrite planes whose VoxelPlane::is_update_ flag was set by UpdateVoxelMap (voxel_map.h:86). */
int esikf_map_patch(esikf_ctx *ctx, const int32_t *plane_ids, const esikf_plane *planes, int32_t n);

/* ---------------------------------------------------------------- device-resident voxel map
 * VoxelMapManager::BuildVoxelMap / UpdateVoxelMap (src/voxel_map.cpp:532-591, 609-641) with the octrees, the nodes' point
 * lists (temp_points_) and the plane refits (init_plane, :55-135) kept on the GPU: after a LIO update the map absorbs the
 * scan without any plane, point list or key crossing PCIe, and the next esikf_lio_run reads the refitted records in place.
 * Replaces the per-tick host refit + flatten + esikf_map_patch of a host-owned map (esikf_map_upload stays available; the
 * two forms are exclusive: whichever was set up last owns the context's map). */
typedef struct esikf_map_cfg {
  double voxel_size;          /* lio/voxel_size       max_voxel_size_ */
  double min_eigen_value;     /* lio/min_eigen_value  planner_threshold_ */
  double dept_err, beam_err;  /* lio/dept_err, lio/beam_err (BuildVoxelMap's own calcBodyCov, :546) */
  int32_t max_layer;          /* lio/max_layer (<= 7) */
  int32_t max_points_num;     /* lio/max_points_num */
  int32_t layer_init_num[8];  /* lio/layer_init_num, entries 0..max_layer are used */
  /* 0: the capacities below are fixed. 1: they are starting sizes, and a build / update that would exceed one grows the map
   * instead (the arena is copied into a larger one, then the tick is applied; the map is the same as with large fixed
   * capacities). A failed allocation there returns ESIKF_ERR_CUDA and invalidates the map. */
  int32_t grow;
  /* capacities; 0 = default derived from root_capacity (default 2^20): nodes 4 x, plane records 4 x, stored points 64 x the
   * roots. With grow == 0 they are fixed at init (nothing is allocated per tick), and exceeding one is reported by the
   * update call (ESIKF_ERR_STATE, flags in esikf_map_stats.errors) and invalidates the map. With grow == 1 they are where
   * the map starts; esikf_map_device_capacity reports where it is. Key-range and octree-depth errors are errors either way. */
  int64_t root_capacity, node_capacity, record_capacity, point_capacity;
} esikf_map_cfg;
typedef struct esikf_map_stats {
  int32_t roots, nodes, records; /* root voxels, octree nodes, record slots handed out (incl. dead blocks of relocated lists) */
  int32_t touched_roots;         /* roots the last build / update replayed */
  int32_t errors;                /* 1 nodes | 2 point pool | 4 records | 8 hash | 16 key outside +-2^20 | 32 octree depth */
  int32_t pad;
  int64_t pool_points;           /* point slots handed out */
} esikf_map_stats;
/* Empty device map with the given configuration (drops any map the context held). */
int esikf_map_device_init(esikf_ctx *ctx, const esikf_map_cfg *cfg);
/* BuildVoxelMap on the resident scan (esikf_lio_set_scan) at pose `state` (packed, host): LIVMapper.cpp:356-366. Needs an
 * empty map. */
int esikf_map_device_build(esikf_ctx *ctx, const double *state);
/* LIVMapper.cpp:413-424: world points / covariances of the resident scan with the posterior of the update that just ran
 * (state == NULL: the one resident on the device; else a packed host state), then UpdateVoxelMap(pv_list_). Call after
 * esikf_lio_run / esikf_lio_update of this scan and before the VIO update overwrites the resident state. */
int esikf_map_device_update(esikf_ctx *ctx, const double *state);
/* UpdateVoxelMap(input_points) with the caller's own lists: point_w [n][3], var [n][9] row-major (host). */
int esikf_map_device_update_points(esikf_ctx *ctx, const double *point_w, const double *var, int32_t n);
/* mapSliding / clearMemOutOfMap (src/voxel_map.cpp:924-971): root voxels whose key lies outside [key_min, key_max]
 * (component-wise, inclusive) are dropped; the survivors are copied into a second arena of the same capacities, which also
 * reclaims dead record blocks and point-list slack (NULL bounds: compaction only). The per-point plane ids of the last
 * update are void afterwards (esikf_lio_fetch normals / ids refer to the old records): call it between ticks. */
int esikf_map_device_slide(esikf_ctx *ctx, const int64_t key_min[3], const int64_t key_max[3]);
int esikf_map_device_stats(esikf_ctx *ctx, esikf_map_stats *out);
/* The current capacities and grow flag of the device map in esikf_map_cfg's terms (root_capacity = hash slots / 2, the
 * inverse of init's sizing); the other fields of `out` are left as they are. */
int esikf_map_device_capacity(esikf_ctx *ctx, esikf_map_cfg *out);
/* The map in esikf_map_upload's flat form (roots in no particular order). keys == NULL: sizes only. */
int esikf_map_device_download(esikf_ctx *ctx, int64_t *keys, int32_t *first, int32_t *count, int32_t roots_cap, esikf_plane *planes, int32_t planes_cap,
                              int32_t *n_roots, int32_t *n_planes);
/* One octree node of the device map: VoxelOctoTree (include/voxel_map.h:129-183) with its VoxelPlane, everything the device
 * keeps of a node except its point list. 312 bytes. */
typedef struct esikf_map_node {
  int64_t key[3];          /* VOXEL_LOCATION of the root voxel */
  int32_t layer;           /* layer_ */
  int32_t path;            /* 3 bits per layer, as esikf_plane.path */
  int32_t parent;          /* index of the parent node inside its root's range (0 = the root itself), -1 for the root */
  int32_t leaf;            /* slot of the node in its parent's leaves_, -1 for the root */
  double voxel_center[3];  /* voxel_center_ */
  float quater_length;     /* quater_length_ */
  uint8_t init_octo, octo_state, update_enable, is_plane;  /* init_octo_, octo_state_, update_enable_, plane_ptr_->is_plane_ */
  int32_t new_points;      /* new_points_ */
  int32_t points_size;     /* plane_ptr_->points_size_ */
  int32_t temp_points;     /* temp_points_.size() on the device (a cut node's list is released there, see DESIGN.md K6) */
  int32_t pad_;
  double center[3], normal[3];  /* plane_ptr_->center_, normal_ */
  double plane_var[21];         /* upper triangle (row-major, i <= j) of plane_ptr_->plane_var_ */
  float d, radius;              /* plane_ptr_->d_, radius_ */
} esikf_map_node;
/* The subtrees of the roots the last esikf_map_device_build / _update / _update_points replayed (in the order of their hash
 * slots), for a host mirror of the map: root r owns nodes [first[r], first[r] + count[r]) in DFS pre-order, leaves 0..7.
 * A pure read: calling it twice gives the same bytes. keys == NULL: sizes only. ESIKF_ERR_STATE after esikf_map_device_init,
 * esikf_map_device_slide or a failed build / update (there is no tick to export: the caller drops the roots the slide
 * removed with the slide's own bounds). */
int esikf_map_device_export(esikf_ctx *ctx, int64_t *keys, int32_t *first, int32_t *count, int32_t roots_cap, esikf_map_node *nodes, int32_t nodes_cap,
                            int32_t *n_roots, int32_t *n_nodes);
/* The VIO front end's octree lookups on the device map, without a host mirror: for each of n world points (host, n x 3), the
 * root voxel the reference looks up, then VoxelOctoTree::find_correspond (src/voxel_map.cpp:292-305) from that root. The key
 * rule is the reference's own at the call site, and both divide by the literal 0.5 (not the map's voxel size):
 *   ESIKF_FIND_RULE_PATCH   updateReferencePatch (src/vio.cpp:983-989): float loc = p / 0.5, loc -= 1.0 when negative, (int64_t)loc
 *   ESIKF_FIND_RULE_RAYCAST the retrieval's ray casting (:508-514): int loc = floor(p / 0.5), loc -= 1.0 when negative
 * Outputs per point: status (ESIKF_FIND_*), keys (n x 3, the root looked up; INT64_MIN on every axis when the key leaves
 * [-2^20, 2^20), NaN and infinities included, which answers ESIKF_FIND_NO_ROOT), and rows (n): for a found node its layer and
 * path (as esikf_plane.path) and its plane_ptr_ fields center, normal, plane_var, d, radius (the bytes esikf_map_device_export
 * gives for the node; meaningful for ESIKF_FIND_PLANE); all zero for ESIKF_FIND_NO_ROOT.
 * A pure read of the map, enqueued on the context's stream after the calls before it; returns when the answers are in. Every
 * rank answers every point. ESIKF_ERR_STATE when no device map is live (never set up, invalidated by a failed call, or
 * replaced by esikf_map_upload); ESIKF_ERR_ARG for n < 0, an unknown rule or a NULL buffer with n > 0. A failed call writes
 * nothing. */
#define ESIKF_FIND_RULE_PATCH 0
#define ESIKF_FIND_RULE_RAYCAST 1
#define ESIKF_FIND_NO_ROOT 0
#define ESIKF_FIND_NODE 1  /* a node that is not a plane */
#define ESIKF_FIND_PLANE 2
int esikf_map_device_find(esikf_ctx *ctx, const double *points, int32_t n, int32_t rule, uint8_t *status, int64_t *keys, esikf_plane *rows);

/* ---------------------------------------------------------------- LIO update (StateEstimation)
 * Staged form (device-resident between calls):
 *   set_scan : feats_down_body_ (xyz float32, n points) -> device + per-frame calcBodyCov/crossmat
 *              (src/voxel_map.cpp:349-360). shard_begin/shard_count select this rank's slice.
 *   run      : the iteration loop (src/voxel_map.cpp:372-500) asynchronously on esikf_stream.
 *   fetch    : state_ / stats / per-point results back to host (synchronises the stream).
 * The per-point calcBodyCov / crossmat precompute is made by the first run after set_scan, and redone by a later run on the
 * same scan whose lidar extrinsics (extR, extT) or dept_err / beam_err differ from the ones it was made with. */
int esikf_lio_set_scan(esikf_ctx *ctx, const float *pts_xyz, int32_t n);
int esikf_lio_run(esikf_ctx *ctx, const double *state_in, const double *state_prop, const esikf_lio_cfg *cfg);
int esikf_lio_fetch(esikf_ctx *ctx, double *state_out, esikf_lio_stats *stats /* nullable */,
                    int32_t *match_plane /* n, plane id matched in the last iteration or -1: ptpl_list_ */,
                    int32_t *normal_plane /* n, plane id behind pv.normal (sticky across iterations) or -1 */,
                    float *dis_to_plane /* n, PointToPlane::dis_to_plane_ of the last iteration */);
/* One-shot form with host buffers = set_scan + run + fetch (what the C++ shim calls). */
int esikf_lio_update(esikf_ctx *ctx, const float *pts_xyz, int32_t n, const double *state_in, const double *state_prop,
                     const esikf_lio_cfg *cfg, double *state_out, esikf_lio_stats *stats, int32_t *match_plane,
                     int32_t *normal_plane, float *dis_to_plane);
/* body_cov_list_ / cross_mat_list_ (include/voxel_map.h:215-216) of the current scan: n x 9 doubles each. */
/* pv_list_[i].normal of the last update (src/voxel_map.cpp:744; zero for an unmatched point): [n][3] doubles. Valid after the
 * map absorbed the scan too (esikf_map_device_update snapshots the normals before plane records may move). */
int esikf_lio_fetch_normals(esikf_ctx *ctx, double *normals);
int esikf_lio_fetch_point_cov(esikf_ctx *ctx, double *body_cov9 /* nullable */, double *cross_mat9 /* nullable */);

/* ---------------------------------------------------------------- VIO update (computeJacobianAndUpdateEKF)
 * set_camera    : vk camera + vio/ parameters. It voids the retrieval (esikf_vio_retrieve_scan); a new width or height voids
 *                 the current image, and a new patch_pyrimid_level the installed sub-map and its inverse-compositional refs.
 *                 Calls that read a voided input return ESIKF_ERR_STATE until it is set again. Re-setting an identical
 *                 camera voids only the retrieval.
 * set_image     : the current 8-bit grey image, width x height of the camera.
 * set_patches   : visual_submap (include/vio.h:26-57): voxel_points[i]->pos_ (n x 3 f64), warp_patch
 *                 (n x levels*64 f32, [level][row][col]), search_levels (n), inv_expo_list (n).
 * run / fetch   : the coarse-to-fine loop (src/vio.cpp:784-802, 1520-1688). */
int esikf_vio_set_camera(esikf_ctx *ctx, const esikf_camera *cam, const esikf_vio_cfg *cfg);
int esikf_vio_set_image(esikf_ctx *ctx, const uint8_t *img, int32_t width, int32_t height);
int esikf_vio_set_patches(esikf_ctx *ctx, const double *pos, const float *warp_patch, const int32_t *search_levels,
                          const double *inv_expo_list, int32_t n);
int esikf_vio_run(esikf_ctx *ctx, const double *state_in, const double *state_prop);
int esikf_vio_fetch(esikf_ctx *ctx, double *state_out, esikf_vio_stats *stats /* nullable */, float *errors /* n, nullable */);
int esikf_vio_update(esikf_ctx *ctx, const uint8_t *img, int32_t width, int32_t height, const double *pos,
                     const float *warp_patch, const int32_t *search_levels, const double *inv_expo_list, int32_t n,
                     const double *state_in, const double *state_prop, double *state_out, esikf_vio_stats *stats,
                     float *errors);

/* ---------------------------------------------------------------- per-frame patch producers
 * get_image_patch: batched getImagePatch (src/vio.cpp:203-225) on the image set by set_image:
 *                  pc n x 2 f64 -> patch n x 64 f32 at `level`.
 * warp_patches   : batched getWarpMatrixAffineHomography + getBestSearchLevel + warpAffine over all
 *                  pyramid levels (src/vio.cpp:701-714, 739-742). Reference images are registered
 *                  once (Feature::img_, include/feature.h) and addressed by index. keep_on_device installs every warped
 *                  patch with inv_expo 1 and gates nothing: callers that need the reference features' exposure times,
 *                  the depth-form warp or the photometric / NCC gate use esikf_vio_select_patches instead. */
int esikf_vio_get_image_patch(esikf_ctx *ctx, const double *pc, int32_t n, int32_t level, float *patch_out);
int esikf_vio_set_ref_images(esikf_ctx *ctx, const uint8_t *const *imgs, int32_t n_imgs, int32_t width, int32_t height);
int esikf_vio_warp_patches(esikf_ctx *ctx, int32_t n, const int32_t *ref_img_index, const double *px_ref /* n x 2 */,
                           const double *pos_w /* n x 3 */, const double *normal_w /* n x 3 */,
                           const double *T_ref_w /* n x 12: R(9) t(3) of Feature::T_f_w_ */,
                           const double *T_cur_w /* 12: new_frame_->T_f_w_ */, double *A_cur_ref_out /* n x 4, nullable */,
                           int32_t *search_level_out /* n */, float *warp_patch_out /* n x levels*64 */,
                           int32_t keep_on_device /* 1: also install as the patches of set_patches */);
/* Gate settings of the sub-map selection (vio/ parameters, LIVMapper.cpp:59,70; include/vio.h:101,109). */
typedef struct esikf_vio_select_cfg {
  int32_t normal_en;         /* 1: homography warp (getWarpMatrixAffineHomography); 0: depth warp (getWarpMatrixAffine) */
  int32_t ncc_en;            /* 1: reject candidates whose calculateNCC is below ncc_thre */
  double ncc_thre;
  double outlier_threshold;  /* reject candidates whose photometric error exceeds outlier_threshold * 64 */
} esikf_vio_select_cfg;
/* select_patches : the per-candidate tail of retrieveFromVisualSparseMap (src/vio.cpp:699-770) for n candidates in the
 *                  caller's (grid-cell) order, whose reference feature the caller has chosen (:645-697): the warp matrix and
 *                  search level (normal_en: homography form from pos_w / normal_w; else the depth form from ref_f /
 *                  ref_pos / ref_level, cached per ref_key = Feature::id_ like warp_map: a candidate takes the matrix of
 *                  the first candidate with its key), warpAffine on every pyramid level, the current patch at pc (level 0
 *                  of the set_image image), the exposure-weighted error, the NCC gate and the outlier gate. The survivors,
 *                  in candidate order, become the visual sub-map of the next esikf_vio_run (pos_w, warp patch, search level,
 *                  inv_expo = ref_inv_expo, errors = the gate error); n_kept == 0 installs an empty sub-map.
 *                  Per candidate: ref_img_index (into set_ref_images), px_ref (2) = Feature::px_, ref_level = Feature::level_,
 *                  ref_f (3) = Feature::f_, ref_pos (3) = Feature::pos(), pos_w (3), normal_w (3), T_ref_w (12, R(9) t(3) of
 *                  Feature::T_f_w_), ref_inv_expo = Feature::inv_expo_time_, ref_key, pc (2) = new_frame_->w2c(pos_w).
 *                  ref_f / ref_pos / ref_level / ref_key may be null when normal_en is set, normal_w when it is not.
 *                  Outputs hold room for n entries; only the first *n_kept are written: kept_index (candidate indices),
 *                  error_out, search_level_out, A_cur_ref_out (4 each, row-major) and warp_patch_out (levels*64 each) are
 *                  nullable. On an error return the installed sub-map is left as it was. */
int esikf_vio_select_patches(esikf_ctx *ctx, int32_t n, const int32_t *ref_img_index, const double *px_ref, const int32_t *ref_level,
                             const double *ref_f, const double *ref_pos, const double *pos_w, const double *normal_w,
                             const double *T_ref_w, const double *ref_inv_expo, const int32_t *ref_key, const double *pc,
                             const double *T_cur_w /* 12 */, double inv_expo_time /* the current frame's, state->inv_expo_time */,
                             const esikf_vio_select_cfg *cfg, int32_t *n_kept, int32_t *kept_index, float *error_out /* nullable */,
                             int32_t *search_level_out /* nullable */, double *A_cur_ref_out /* nullable */,
                             float *warp_patch_out /* nullable */);
/* set_inverse_refs: what the inverse-compositional variant (src/vio.cpp:1327-1518) reads of every visual point's reference
 *                  feature (include/feature.h): image (index into set_ref_images), px_, f_ (unit bearing), the rotation
 *                  of T_f_w_ (row-major) and pos() = T_f_w_.inverse().translation(). n must equal the n of set_patches. */
int esikf_vio_set_inverse_refs(esikf_ctx *ctx, int32_t n, const int32_t *ref_img_index, const double *ref_px /* n x 2 */,
                               const double *ref_f /* n x 3 */, const double *ref_R /* n x 9 */, const double *ref_pos /* n x 3 */);
/* warp_affine    : batched warpAffine alone (src/vio.cpp:292-318, include/vio.h:161-162) with caller-provided affine
 *                  matrices A_cur_ref (n x 4, row-major [a00 a01 a10 a11]) and search levels; writes all pyramid levels,
 *                  patch i level l at warp_patch_out[(i*levels + l)*64 ...] like visual_submap->warp_patch[i]. */
int esikf_vio_warp_affine(esikf_ctx *ctx, int32_t n, const int32_t *ref_img_index, const double *px_ref /* n x 2 */,
                          const double *A_cur_ref /* n x 4 */, const int32_t *search_level /* n */,
                          float *warp_patch_out /* n x levels*64 */);

/* ---------------------------------------------------------------- coloured scan (publish_frame_world)
 * The coloured point cloud LIVMapper publishes after each VIO update (src/LIVMapper.cpp:1140-1173), computed on the device.
 * One call per tick of each kind:
 *   LIO tick : esikf_lio_run, then esikf_rgb_set_cloud (before the VIO update overwrites the resident LIO posterior)
 *   VIO tick : esikf_vio_run, then esikf_rgb_colorize
 * With several ranks, both calls cover the whole cloud on every rank (the poses are identical on every rank).
 * The context owns the cloud and image buffers; esikf_destroy frees them. */
/* The world cloud of this LIO tick (LIVMapper.cpp:435-443, RGBpointBodyToWorld at :682-690):
 * p_w = rot_end * (extR * p_body + extT) + pos_end in double, stored as float.
 * pts_xyz == NULL: the resident scan of esikf_lio_set_scan, n ignored (dense_map_en = false); else n body points, host float
 * xyz (feats_undistort, dense_map_en = true). state == NULL: the posterior the last esikf_lio_run left on the device
 * (ESIKF_ERR_STATE when no LIO update ran or a VIO update ran since); else a packed host state. The host buffers may be
 * reused as soon as the call returns. */
int esikf_rgb_set_cloud(esikf_ctx *ctx, const float *pts_xyz, int32_t n, const double *state);
/* publish_frame_world on the cloud of esikf_rgb_set_cloud with the image `bgr` (8-bit B G R interleaved, width x height of
 * the camera, row-major): a point is kept when pf[2] >= 0, isInFrame(pc.cast<int>(), 3) holds and pf.norm() > blind_rgb_points,
 * with pf = new_frame_->w2f(p_w), pc = w2c(p_w) and the frame pose of updateFrameState (vio.cpp:1690-1697) of `state`
 * (NULL: the posterior resident after esikf_vio_run; else a packed host state). Its colour is getInterpolatedPixel
 * (vio.cpp:1742-1760), each channel converted to uint8 as the assignment to PointXYZRGB does (truncation).
 * The survivors come out in cloud order: xyz_out (3 floats each), bgr_out (B, G, R each), index_out (their cloud index,
 * nullable). *n_out = the number kept; if it exceeds cap, nothing else is written and the call returns ESIKF_ERR_ARG. */
int esikf_rgb_colorize(esikf_ctx *ctx, const uint8_t *bgr, int32_t width, int32_t height, const double *state, double blind_rgb_points,
                       int32_t cap, int32_t *n_out, float *xyz_out, uint8_t *bgr_out, int32_t *index_out);

/* ---------------------------------------------------------------- new visual map points (generateVisualMapPoints)
 * VIOManager::generateVisualMapPoints (src/vio.cpp:804-906) on the device, minus the host-side object creation: the points of
 * the scan pg, then of add_from_voxel_map, that become new visual map points, at most one per grid cell. Called in the VIO
 * tick after esikf_vio_run; the image is the one of esikf_vio_set_image (or esikf_vio_update).
 *   pg      : point_w == NULL: the pv list the last esikf_map_device_update left on the device (pv_list_ after
 *             LIVMapper.cpp:413-424: the float-narrowed posterior world point, the recomputed var and the LIO normal), n
 *             ignored; ESIKF_ERR_STATE when there is none (no update yet, or esikf_map_device_build / _update_points since).
 *             Else n host points: point_w (3 doubles each), normal (3), var (9, row-major).
 *   add_from: n_add points (position and normal, 3 doubles each; their var is zero), scored after the scan (:834-854).
 *   type_map: one byte per grid cell (n_cells = grid_n_width * grid_n_height, else ESIKF_ERR_ARG), nonzero where the retrieval
 *             set grid_num[cell] = TYPE_MAP; those cells get no new point.
 *   grid_size, grid_n_width, grid_n_height, border: as initializeVIO left them (vio.cpp:66-80, 154).
 *   state   : NULL: the posterior resident after esikf_vio_run; else a packed host state (the frame pose is updateFrameState's).
 * A point is scored when its normal is not zero (scan points only), isInFrame(pc.cast<int>(), border) holds and its cell
 * (int)(pc[1] / grid_size) * grid_n_width + (int)(pc[0] / grid_size) is not TYPE_MAP; the score is vk::shiTomasiScore(img,
 * (int)pc[0], (int)pc[1]). A cell's winner is the first point with the cell's largest score > 0 (cur_value > scan_value[index],
 * scan_value reset to 0). Nothing is produced when the scan has 10 points or fewer (:806).
 * The winners come out in cell order, *n_out of them: source_out (scan index, or ESIKF_GEN_ADD_FROM | add_from index),
 * cell_out, pos_out (point_w, 3 doubles), pc_out (w2c, 2 doubles), score_out, normal_out (the point's normal, negated when
 * cos_theta < 0, :867-890), var_out (9 doubles), patch_out (getImagePatch(img, pc, patch, 0), 64 floats). Each output may be
 * NULL. If *n_out exceeds cap, nothing else is written and the call returns ESIKF_ERR_ARG. */
#define ESIKF_GEN_ADD_FROM 0x40000000
int esikf_vio_generate_points(esikf_ctx *ctx, const double *point_w, const double *normal, const double *var, int32_t n, const double *add_pos,
                              const double *add_normal, int32_t n_add, const uint8_t *type_map, int32_t n_cells, int32_t grid_size, int32_t grid_n_width,
                              int32_t grid_n_height, int32_t border, const double *state, int32_t cap, int32_t *n_out, int32_t *source_out,
                              int32_t *cell_out, double *pos_out, double *pc_out, float *score_out, double *normal_out, double *var_out, float *patch_out);

/* ---------------------------------------------------------------- new observations of the visual sub-map (updateVisualMapPoints)
 * VIOManager::updateVisualMapPoints (src/vio.cpp:908-967) on the device, minus the host-side object management: which entries
 * of the visual sub-map the current frame becomes a new observation (Feature) of, with that Feature's pixel and patch. Called
 * in the VIO tick after esikf_vio_run (and esikf_vio_generate_points); the image is the one of esikf_vio_set_image (or
 * esikf_vio_update).
 *   sub-map  : the one the last esikf_vio_select_patches, esikf_vio_set_patches, esikf_vio_update or esikf_vio_warp_patches
 *              (keep_on_device) installed; its pos is read on the device. ESIKF_ERR_STATE when none was installed;
 *              n must equal its count, else ESIKF_ERR_ARG.
 *   converged: n bytes, VisualPoint::is_converged_ of each entry.
 *   last_T_f_w: n x 12 doubles, obs_.back()->T_f_w_ (the oldest observation: addFrameRef pushes at the front) as R
 *              (row-major) then t.
 *   last_px  : n x 2 doubles, obs_.back()->px_.
 *   state    : NULL: the posterior resident after esikf_vio_run; else a packed host state (the frame pose is updateFrameState's).
 * A converged entry gets flag 0. Any other entry i gets pc = new_frame_->w2c(pos_), delta_pose = pose_ref *
 * pose_cur.inverse(), delta_p = |t|, delta_theta = 0 when the rotation's trace > 3 - 1e-6, else acos(0.5 * (trace - 1));
 * it is added (update_flag[i] = 1) when delta_p > 0.5 || delta_theta > 0.3 || |pc - last_px| > 40. The flags do not depend
 * on the eviction at 30 observations, which stays with the caller.
 * Outputs: update_flag_out (n bytes), and for the added entries in entry order, *n_out of them: entry_out (sub-map index),
 * pc_out (2 doubles: the new Feature's px_) and patch_out (getImagePatch(img, pc, patch, 0), 64 floats); the new Feature's
 * level is search_levels[entry] of the selection. Each output may be NULL. If *n_out exceeds cap, nothing else is written and
 * the call returns ESIKF_ERR_ARG; a call that fails its argument checks writes nothing. With several ranks every rank
 * evaluates all n entries. */
int esikf_vio_update_points(esikf_ctx *ctx, int32_t n, const uint8_t *converged, const double *last_T_f_w, const double *last_px, const double *state,
                            int32_t cap, int32_t *n_out, uint8_t *update_flag_out, int32_t *entry_out, double *pc_out, float *patch_out);

/* ---------------------------------------------------------------- scan side of the visual sub-map retrieval (retrieveFromVisualSparseMap)
 * The parts of VIOManager::retrieveFromVisualSparseMap that read the LiDAR scan pg, on the device: the scan's voxel keys and its
 * depth image (src/vio.cpp:386-428), and the depth-continuity check of the retrieved points (:614-640). The walk over the
 * host's feat_map, ray casting and the choice of the reference feature stay with the caller (INTEGRATION.md §2). Call
 * esikf_vio_retrieve_scan at the start of the VIO tick, then esikf_vio_depth_check on the retrieved points, before
 * esikf_vio_select_patches.
 *
 * esikf_vio_retrieve_scan:
 *   pg      : point_w == NULL: the pv list the last esikf_map_device_update left on the device (the source of
 *             esikf_vio_generate_points(point_w = NULL)), n ignored; ESIKF_ERR_STATE when there is none. Else n host points
 *             (point_w, 3 doubles each).
 *   border  : as initializeVIO left it (vio.cpp:154).
 *   state   : a packed host state whose frame pose (updateFrameState's) is the frame's: *state at the start of processFrame, the
 *             VIO prior. NULL: the LIO posterior resident on the device after esikf_lio_run (ESIKF_ERR_STATE when the device
 *             holds another one); a caller that propagates the state between the LIO and the VIO tick passes it explicitly.
 * Keys: every scan point's voxel key, loc = floor(c / 0.5) in double, then loc -= 1.0 when negative (the retrieval's own
 * formula, :392-396, not the map's), including points behind the camera or outside the image. The distinct keys come out in
 * first-occurrence order (the scan index of each key's first point), *n_keys of them, 3 int32 each: inserted into
 * sub_feat_map in this order they give the reference's insertion sequence. If *n_keys exceeds cap, nothing else is written and
 * the call returns ESIKF_ERR_ARG. A key outside [-2^20, 2^20) (the device map's key range): ESIKF_ERR_ARG, nothing written.
 * Depth image (width x height floats, kept on the device for esikf_vio_depth_check, copied to depth_out when not NULL): a
 * point with pt_c[2] > 0 and isInFrame(px.cast<int>(), border) writes float(pt_c[2]) at width * int(px[1]) + int(px[0]);
 * the last such point in scan order wins a pixel; an untouched pixel is 0.
 *
 * esikf_vio_depth_check: for n retrieved points (the retrieve_voxel_points[i] of the TYPE_MAP cells, in cell order), pos_w
 * (VisualPoint::pos_, 3 doubles each) and pc (the caller's w2c(pos_), 2 doubles each, as it computed the cell index at
 * :466-471), discontinuous_out[i] = 1 when a tap (int(pc[0]) + u, int(pc[1]) + v), u, v in [-4, 4], (u, v) != (0, 0), of the
 * depth image holds a nonzero depth with |pt_cam[2] - depth| > 0.5 in double, pt_cam = w2f(pos_) with the frame pose of the
 * last esikf_vio_retrieve_scan; such a point is dropped (:640). A tap outside the image is empty. ESIKF_ERR_STATE when no
 * esikf_vio_retrieve_scan succeeded since the last esikf_vio_set_camera.
 * With several ranks every rank evaluates the whole scan and all points. */
int esikf_vio_retrieve_scan(esikf_ctx *ctx, const double *point_w, int32_t n, int32_t border, const double *state, int32_t cap, int32_t *n_keys,
                            int32_t *keys_out, float *depth_out);
int esikf_vio_depth_check(esikf_ctx *ctx, int32_t n, const double *pos_w, const double *pc, uint8_t *discontinuous_out);

/* ---------------------------------------------------------------- reference patches (updateReferencePatch)
 * The patch scoring of VIOManager::updateReferencePatch (src/vio.cpp:1036-1097) on the device, for the n visual points that
 * pass the four skips of :977-980, after the plane half (:981-1034, the caller's, on esikf_map_device_find's answers) has left
 * their normal_. Point i owns the observations first[i] .. first[i + 1] - 1, in obs_ order (the newest first, as addFrameRef
 * pushes them); first has n + 1 entries, first[0] = 0 and first[n] = m. Per point (host, 3 doubles each): pos (pos_) and
 * normal (normal_). Per observation: patch (patch_, 64 floats), mean (mean_), id (id_) and T_f_w (T_f_w_: R row-major, then
 * t; 12 doubles).
 * For each observation r of a point, in list order:
 *   cos_angle = pf.dot(R normal_) with pf = T_f_w_ * pos_ normalised, in double;
 *   the mean of an observation is its mean_, or when abs(mean_) < 1e-6 the double sum of its 64 taps narrowed to float and
 *   divided by 64 in float (mean_out: what the reference leaves in mean_);
 *   over every other observation j with id_ != r's id_, in list order, the float sums up += (a - mean_r)(b - mean_j),
 *   d1 += (a - mean_r)^2 and d2 += (b - mean_j)^2 over the 64 taps in order, running across all j (they are not reset per j),
 *   and after each j, ncc += fabs(up / sqrt(d1 * d2)) in float; ncc / count (NaN when no observation has another id_);
 *   score_out[r] = ncc + cos_angle in double, narrowed to float (the reference's score_).
 * ref_out[i] = the position within the point's list of the first observation whose score beats the running maximum, which
 * starts at -1000 (strict >: a tie keeps the earlier one, NaN never wins), or -1 when none does; the caller then sets
 * ref_patch to it and has_ref_patch_ = true, and leaves both as they were for -1.
 * The reference declares ref_mean and other_mean (:1054, :1067) without a value and assigns them only when mean_ is below
 * 1e-6, so a cached mean_ is read as an uninitialised float. Here both are the observation's mean as defined above: the cached
 * mean_ the code means to use. On inputs where every mean is recomputed at each read the results are the reference's.
 * One host-to-device copy per input array, one kernel, one copy of the answers into pinned staging; the caller's outputs are
 * written only after both copies succeeded. ESIKF_ERR_ARG for n < 0, m < 0, a NULL buffer that is needed, first[0] != 0,
 * first[n] != m or decreasing offsets: a failed call writes nothing. n = 0 succeeds and does nothing. Every observation count
 * is accepted, 1 included. With several ranks every rank evaluates all points. */
int esikf_vio_score_ref_patches(esikf_ctx *ctx, int32_t n, const int32_t *first, int32_t m, const double *pos, const double *normal, const float *patch,
                                const float *mean, const int32_t *id, const double *T_f_w, float *score_out, float *mean_out, int32_t *ref_out);

/* ---------------------------------------------------------------- the visual map's observations on the device (K14)
 * A store of every visual point's obs_ list (VisualPoint::obs_), kept on the device so that the per-tick passes over the
 * observations read and change them in place instead of receiving them from the host. A point id is the slot add_points
 * handed out, in order from 0. Per point: its observations in obs_ order (the newest first, as addFrameRef pushes them), at
 * most 30, and ref, the position of ref_patch in the list or -1 (has_ref_patch_ false). Per observation: px_ (2 doubles),
 * T_f_w_ (12 doubles: R row-major, then t), patch_ (64 floats), id_, mean_ and score_. level_, inv_expo_time_, f_ and img_,
 * which no device pass reads, stay on the caller's Feature objects, which mirror the store from what each call returns
 * (INTEGRATION.md §3). A point takes 11,408 bytes of device memory whatever its count: 0.75 GB at 2^16 points.
 *
 * esikf_vmap_init      : an empty store with room for point_capacity points (1 .. 2^26), replacing any store the context
 *                        held. esikf_destroy frees it.
 * esikf_vmap_add_points: appends n points; point i owns the observations first[i] .. first[i + 1] - 1 of the packed arrays
 *                        (first[0] = 0, first[n] = m, 0 .. 30 each) and ref[i] (-1 .. count - 1). Its id goes to
 *                        point_id_out[i]. A new point of generateVisualMapPoints (src/vio.cpp:874-895, esikf_vio_generate_points'
 *                        winners) has one observation: px_ = pc, the level-0 patch, the frame's T_f_w_ and id_, mean_ 0,
 *                        score_ 0, ref -1. When the store is full its capacity doubles until the points fit; the old records
 *                        are copied, and if the larger allocation fails the call returns ESIKF_ERR_CUDA with the store as it
 *                        was. The capacity never shrinks.
 * esikf_vmap_update_points: VIOManager::updateVisualMapPoints (:914-964) for the installed sub-map (n must equal its count),
 *                        entry i being point point_id[i]. The flags, *n_out and the added entries' entry_out, pc_out and
 *                        patch_out are esikf_vio_update_points' (same rule, same kernels), with each entry's oldest observation
 *                        (obs_.back(), read before any eviction, as :931 precedes :947) taken from the store. Then per entry:
 *                          converged: deleteNonRefPatchFeatures, only the ref observation stays (none when ref is -1: the
 *                                     reference compares with a null or unset ref_patch); evicted_out -1;
 *                          else, with 30 observations, the first strict minimum of score_ from FLT_MAX goes (the newest when
 *                                     every score is NaN or >= FLT_MAX; evicted_out = its position, and ref becomes -1 if it was
 *                                     the ref); then a flagged entry gets the new observation at the front: px_ = pc, the patch,
 *                                     T_f_w_ = T_f_w (NULL: the frame pose of the flags, updateFrameState's), id_ = frame_id,
 *                                     mean_ 0, score_ 0.
 *                        count_out[i] = the count afterwards. With evicted_out and count_out the caller applies the same
 *                        deleteNonRefPatchFeatures / deleteFeatureRef / addFrameRef to its own objects. An entry without
 *                        observations (the reference would read obs_.back() of an empty list) is not flagged (DESIGN.md §4).
 *                        If *n_out exceeds cap, only *n_out is written, the store is left as it was, and the call returns
 *                        ESIKF_ERR_ARG. Every output but n_out may be NULL.
 * esikf_vmap_score     : esikf_vio_score_ref_patches (K13, same kernel and arithmetic) on the store for n points that pass the
 *                        caller's four skips of updateReferencePatch (:977-980); pos and normal (3 doubles each) per entry. The
 *                        scores and means are written back to the store; a point's ref is set where ref_out[i] >= 0 and left
 *                        as it was otherwise. score_out and mean_out (NULL or [n][30] floats, 0 past a point's count) receive
 *                        the store's rows afterwards.
 * esikf_vmap_choose_ref: the reference feature of retrieveFromVisualSparseMap (:651-697) for retrieved points that passed the
 *                        depth check and the caller's is_normal_initialized_ skip. normal_en != 0: a point with one observation
 *                        -> 0; without a ref -> the first strict minimum, from FLT_MAX, of the float sum of the squared patch
 *                        differences against every observation of another id_, in list order, divided by their count; else
 *                        its ref. The first two are stored as the point's ref. normal_en == 0: getCloseViewObs(frame_pos),
 *                        the first strict maximum, from 0, of the cosine between (frame_pos - pos_) and (the observation's
 *                        camera centre - pos_), both normalised; -1 below 0.5 (the point is skipped). pos (3 doubles per
 *                        entry) and frame_pos (new_frame_->pos()) are read only then. ref_out[i] = -1 also where the
 *                        reference leaves ref_ftr unset: no error beats FLT_MAX (every observation has the same id_, 0/0).
 * esikf_vmap_download  : the inverse of add_points for n points: first_out (n + 1), then the packed observations (cap of them)
 *                        and ref (n). If there are more than cap, only first_out is written and the call returns ESIKF_ERR_ARG.
 * esikf_vmap_stats     : points added and capacity.
 * ESIKF_ERR_ARG, with nothing written, for a point id outside [0, points), an id twice in one call, a count above 30 (add)
 * or n different from the installed sub-map's count (update_points). ESIKF_ERR_STATE before esikf_vmap_init. With several
 * ranks every rank holds the whole store and applies every call. */
int esikf_vmap_init(esikf_ctx *ctx, int64_t point_capacity);
int esikf_vmap_add_points(esikf_ctx *ctx, int32_t n, const int32_t *first, int32_t m, const double *px, const float *patch, const double *T_f_w,
                          const int32_t *id, const float *mean, const float *score, const int32_t *ref, int32_t *point_id_out);
int esikf_vmap_update_points(esikf_ctx *ctx, int32_t n, const int32_t *point_id, const uint8_t *converged, const double *T_f_w, int32_t frame_id,
                             const double *state, int32_t cap, int32_t *n_out, uint8_t *update_flag_out, int32_t *entry_out, double *pc_out,
                             float *patch_out, int32_t *evicted_out, int32_t *count_out);
int esikf_vmap_score(esikf_ctx *ctx, int32_t n, const int32_t *point_id, const double *pos, const double *normal, int32_t *ref_out, float *score_out,
                     float *mean_out);
int esikf_vmap_choose_ref(esikf_ctx *ctx, int32_t n, const int32_t *point_id, const double *pos, const double *frame_pos, int32_t normal_en,
                          int32_t *ref_out);
int esikf_vmap_download(esikf_ctx *ctx, int32_t n, const int32_t *point_id, int32_t cap, int32_t *first_out, double *px, float *patch, double *T_f_w,
                        int32_t *id, float *mean, float *score, int32_t *ref);
int esikf_vmap_stats(esikf_ctx *ctx, int64_t *points, int64_t *capacity);

/* ---------------------------------------------------------------- the map side of the visual sub-map retrieval (K15)
 * retrieveFromVisualSparseMap's walk over feat_map (src/vio.cpp:438-484, raycast_en off) on a device feat_map of the store's
 * points, with the depth check (:614-640), the is_normal_initialized_ skip (:651) and the reference-feature choice (:653-697)
 * chained after it on the device.
 * esikf_vmap_place_points: places n store points in their visual voxels, as insertPointIntoVoxelMap (:227-250) does: pos
 *                        (3 doubles per point) is the point's pos_, normal_init its is_normal_initialized_ (NULL: all true).
 *                        The key of a coordinate c is the insertion rule: float(c / 0.5), minus 1.0 in double and narrowed
 *                        again when negative, truncated; it is not the scan's floor rule (x = -0.3: insertion key -1, scan
 *                        key -2), and the walk looks scan keys up in this map, as the reference does. Within a voxel the
 *                        points keep their placement order (call order, later calls after earlier ones). Positions never
 *                        change and points are never removed. The point arrays grow by doubling; if that allocation fails the
 *                        call returns ESIKF_ERR_CUDA with everything as it was.
 * esikf_vmap_retrieve  : the walk for the frame pose and depth image of the last esikf_vio_retrieve_scan. keys: n_keys scan
 *                        voxel keys (3 int32 each) in the caller's sub_feat_map iteration order. For each placed point with
 *                        obs_ count > 0 whose voxel is among them, dir[2] >= 0 and isInFrame(pc.cast<int>(), border): its
 *                        cell int(pc[1] / grid_size) * grid_n_width + int(pc[0] / grid_size) is TYPE_MAP, and the cell's
 *                        point is the one of least float distance |new_frame_->pos() - pos_| (<= 10000.0f); of equal
 *                        distances the one latest in the walk: the later key, then the later place in the voxel's list.
 *                        The TYPE_MAP cells come out in cell order (at most cap): cell_out, point_id_out (-1: no winner,
 *                        every point of the cell being beyond 10000 m or NaN; the reference would read a null pointer),
 *                        pc_out (2 doubles, the winner's w2c(pos_)), status_out (ESIKF_RETRIEVE_*) and ref_out: the
 *                        position in obs_ of the reference feature esikf_vmap_choose_ref would give the kept point (with
 *                        normal_en it is stored as the point's ref), -1 for the other statuses. *n_cells = their count.
 *                        With no placed point, or no key, the call returns 0 cells (the reference returns at :354 when
 *                        feat_map is empty: the caller then inserts no keys into its sub_feat_map either).
 * ESIKF_ERR_ARG, with nothing written and the store untouched: an id outside the store or placed before (or twice in one
 * call), a voxel key outside [-2^20, 2^20) (NaN and inf included), a walk key twice or outside that range, a grid with
 * grid_n_width * grid_size < width - border (or the same for the height), and more cells than cap (*n_cells is then
 * written, so that the caller can retry). ESIKF_ERR_STATE before esikf_vmap_init, and for esikf_vmap_retrieve without an
 * esikf_vio_retrieve_scan since the last esikf_vio_set_camera. esikf_vmap_init forgets every placement. With several ranks
 * every rank holds the whole visual map and applies every call. */
#define ESIKF_RETRIEVE_KEPT 0       /* passed every test; ref_out is its reference feature */
#define ESIKF_RETRIEVE_DEPTH 1      /* depth-discontinuous (:640) */
#define ESIKF_RETRIEVE_NOT_INIT 2   /* !is_normal_initialized_ (:651) */
#define ESIKF_RETRIEVE_NO_REF 3     /* no reference feature: getCloseViewObs false, or (normal_en) none below FLT_MAX */
#define ESIKF_RETRIEVE_NO_WINNER 4  /* a TYPE_MAP cell without a point */
int esikf_vmap_place_points(esikf_ctx *ctx, int32_t n, const int32_t *point_id, const double *pos, const uint8_t *normal_init);
int esikf_vmap_retrieve(esikf_ctx *ctx, int32_t n_keys, const int32_t *keys, int32_t grid_size, int32_t grid_n_width, int32_t grid_n_height, int32_t border,
                        int32_t normal_en, int32_t cap, int32_t *n_cells, int32_t *cell_out, int32_t *point_id_out, double *pc_out, int32_t *status_out,
                        int32_t *ref_out);

/* ---------------------------------------------------------------- multi-GPU (one process per GPU)
 * The residual point / patch set is sharded by contiguous blocks; each iteration all-reduces the
 * packed information buffer [HTH upper | HTz | M | sum|d| ...] and every rank solves redundantly.
 * esikf_comm_unique_id: rank 0 creates the NCCL id, the host side broadcasts it (torch.distributed).
 * esikf_comm_init     : ncclCommInitRank on this context. shard = [begin, begin+count) of the scan /
 *                       patch arrays given to set_scan / set_patches (all ranks pass the full arrays).
 * With more than one rank the per-point / per-patch outputs of a rank (match_plane, normal_plane, dis_to_plane,
 * errors) are valid on that rank's esikf_shard_range slice only; the state and the stats are identical on every rank. */
int esikf_comm_unique_id(char out[128]);
int esikf_comm_init(esikf_ctx *ctx, int32_t rank, int32_t nranks, const char unique_id[128]);
int esikf_comm_rank(const esikf_ctx *ctx, int32_t *rank, int32_t *nranks);
/* NVLink peer-memory path (no NCCL in the loop): every rank exports a CUDA-IPC handle of its 72-double mailbox, the host
 * side all-gathers the 64-byte handles, esikf_peer_attach maps the peers' mailboxes. The persistent update kernels then
 * all-reduce the information buffer themselves (stores into every peer's mailbox + flag spin) and stay one launch per
 * update. <= 8 ranks of one NVSwitch box; every rank must issue the same sequence of updates. */
int esikf_peer_export(esikf_ctx *ctx, char out[64]);
int esikf_peer_attach(esikf_ctx *ctx, int32_t rank, int32_t nranks, const char *handles /* nranks x 64 bytes */);
/* The contiguous slice [begin, begin+count) of n units owned by `rank` (host-only helper, no device needed). */
int esikf_shard_range(int32_t n, int32_t rank, int32_t nranks, int32_t *begin, int32_t *count);

/* ---------------------------------------------------------------- measurement hooks (bench.py)
 * Average device time (ms, CUDA events on esikf_stream) of `reps` back-to-back launches of one
 * kernel on the resident inputs: which = 0 LIO residual kernel, 1 solve kernel, 2 VIO patch kernel
 * (level given by `arg`, in [0, patch_pyrimid_level)), 3 per-frame LIO precompute. flush_l2 != 0 writes a >L2 buffer between launches
 * (excluded from the timing). */
int esikf_profile_kernel(esikf_ctx *ctx, int32_t which, int32_t arg, int32_t reps, int32_t flush_l2, float *avg_ms);

/* Per-launch device times of the update loops. enable != 0 brackets every residual / patch / solve launch of the
 * following lio_run / vio_run calls with CUDA events on esikf_stream (adds sub-microsecond gaps: use a separate,
 * untimed pass). get: ms of the launches of the LAST run, in launch order; LIO: residual[8], solve[8];
 * VIO: patch[64], solve[64] indexed (levels-1-level)*max_iterations + iteration. Unlaunched slots are 0. */
int esikf_set_kernel_timing(esikf_ctx *ctx, int32_t enable);
int esikf_get_kernel_timing(esikf_ctx *ctx, float *lio_residual_ms /* 8 */, float *lio_solve_ms /* 8 */,
                            float *vio_patch_ms /* 64 */, float *vio_solve_ms /* 64 */);

/* Phase timestamps of the persistent update kernels (ns, %globaltimer, written by CTA 0): 8 per iteration slot
 * [start, consts loaded, slice done, all CTAs arrived, partials summed, solved, state published, spare];
 * slots 0..7 = LIO iterations, 8..71 = VIO (levels-1-level)*max_iterations + iteration. 0 = slot not executed. */
int esikf_set_phase_stamps(esikf_ctx *ctx, int32_t enable);
int esikf_get_phase_stamps(esikf_ctx *ctx, uint64_t *out /* 800: 576 phase stamps + 64 fine-grained debug stamps + 160 per-CTA slice-end stamps of LIO iteration 3 */);
// The persistent VIO update's finer stamps of the last stamped update (ns, %globaltimer; 0 = not written: a library built
// without ESIKF_VIO_CHAIN_STAMPS writes none), per (level,
// iteration) slot s in the order of the phase stamps: [8 s + 0..3] CTA 0's warp 0, its first patch: projection and tap
// geometry done, Jacobian constants done, bilinear grid done, rows contracted; [512 + 160 s + b] CTA b's partial summed.
#define ESIKF_VIO_CHAIN_STAMP_WORDS (8 * 64 + 160 * 64)
int esikf_get_vio_chain_stamps(esikf_ctx *ctx, uint64_t *out /* ESIKF_VIO_CHAIN_STAMP_WORDS */);

#ifdef __cplusplus
}
#endif
#endif /* ESIKF_B200_H_ */
