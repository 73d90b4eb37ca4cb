// The VIO front end on the device: the coloured scan, new visual map points and new observations, the scan and map sides of
// the sub-map retrieval, reference-patch scoring, and the visual map's observation store.
#include <math.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "esikf_api.cuh"

#include "esikf_color.cu"
#include "esikf_generate.cu"
#include "esikf_observe.cu"
#include "esikf_retrieve.cu"
#include "esikf_refpatch.cu"
#include "esikf_vmap.cu"
#include "esikf_vretrieve.cu"

extern "C" {

// ---------------------------------------------------------------------------------------------------------------- coloured scan
int esikf_rgb_set_cloud(esikf_ctx *ctx, const float *pts_xyz, int32_t n, const double *state) {
  if (!ctx || (pts_xyz && n < 0)) return fail(ctx, ESIKF_ERR_ARG, "rgb_set_cloud: bad argument");
  if (int rc = need(ctx, "rgb_set_cloud", IN_EXT | (pts_xyz ? 0 : IN_SCAN | (state ? 0 : IN_RUN_SCAN)))) return rc;
  CK(cudaSetDevice(ctx->device));
  const double *dev_state = nullptr;
  if (int rc = state_or_posterior(ctx, state, esikf_ctx::RESIDENT_LIO, "rgb_set_cloud", &dev_state)) return rc;
  if (!pts_xyz) n = ctx->n_pts;
  void_inputs(ctx, IN_CLOUD);  // until the new cloud is in place
  CK(ctx->rgb_cloud.reserve((size_t)n * 3 + 4));
  cudaStream_t st = ctx->stream;
  if (pts_xyz && n > 0) CK(cudaMemcpyAsync(ctx->rgb_cloud.p, pts_xyz, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
  if (pts_xyz || state) CK(cudaStreamSynchronize(st));  // the caller may reuse its buffers on return, pinned ones included
  if (n > 0) {
    RgbWorldArgs a;
    a.body = pts_xyz ? ctx->rgb_cloud.p : ctx->pts.p, a.world = ctx->rgb_cloud.p, a.n = n, a.state = dev_state;
    memcpy(a.extR, ctx->ext.extR, sizeof(a.extR)), memcpy(a.extT, ctx->ext.extT, sizeof(a.extT));
    CK(launch(ctx, rgb_world_kernel, (n + 255) / 256, 256, 0, a));
  }
  ctx->rgb_n = n;
  return ESIKF_OK;
}

int esikf_rgb_colorize(esikf_ctx *ctx, const uint8_t *bgr, int32_t width, int32_t height, const double *state, double blind_rgb_points, int32_t cap,
                       int32_t *n_out, float *xyz_out, uint8_t *bgr_out, int32_t *index_out) {
  if (!ctx || !bgr || !n_out || cap < 0 || (cap > 0 && (!xyz_out || !bgr_out))) return fail(ctx, ESIKF_ERR_ARG, "rgb_colorize: bad argument");
  if (int rc = need(ctx, "rgb_colorize", IN_CLOUD | IN_CAMERA)) return rc;
  if (width != ctx->cam.width || height != ctx->cam.height)
    return fail(ctx, ESIKF_ERR_ARG, "rgb_colorize: image is %dx%d, camera %dx%d", width, height, ctx->cam.width, ctx->cam.height);
  CK(cudaSetDevice(ctx->device));
  const double *dev_state = nullptr;
  if (int rc = state_or_posterior(ctx, state, esikf_ctx::RESIDENT_VIO, "rgb_colorize", &dev_state)) return rc;
  const int n = ctx->rgb_n;
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)n, img_bytes = (size_t)width * height * 3;
  // device-wide scan: select_scan_kernel's single CTA took 90 % of the pass at 300 k points (DESIGN.md §8)
  size_t tmp_bytes = 0;
  if (n > 0) CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, (int32_t *)nullptr, (int32_t *)nullptr, n + 1, st));
  uint8_t *img, *color, *bgr_kept, *tmp;
  int32_t *keep, *dst, *index;
  float *xyz;
  auto lay = [&](CallLayout &s) {
    img = s.take<uint8_t>(img_bytes), s.end_inputs();
    keep = s.take<int32_t>(N + 1), color = s.take<uint8_t>(N * 3 + 4), tmp = s.take<uint8_t>(tmp_bytes);
    s.begin_answers();  // keep[n] = 0: dst[n] is the number kept
    dst = s.take<int32_t>(N + 1), xyz = s.take<float>(N * 3 + 4), bgr_kept = s.take<uint8_t>(N * 3 + 4), index = s.take<int32_t>(N + 1);
  };
  CK(lay_out_scratch(ctx, lay));
  int32_t kept = 0;
  if (n > 0) {
    CK(upload(ctx, {{img, bgr, img_bytes}}));
    RgbColorArgs a;
    a.cloud = ctx->rgb_cloud.p, a.n = n, a.bgr = img, a.state = dev_state, a.blind = blind_rgb_points;
    frame_consts(ctx, a.cam, a.Rci, a.Pci);
    a.keep = keep, a.color = color;
    CK(launch(ctx, rgb_color_kernel, (n + 1 + 255) / 256, 256, 0, a));
    CK(counted(ctx, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, keep, dst, n + 1, st)));
    CK(launch(ctx, rgb_scatter_kernel, (n + 255) / 256, 256, 0, keep, dst, n, ctx->rgb_cloud.p, color, xyz, bgr_kept, index));
    CK(read_back_to(ctx, dst + n, &kept));
  }
  *n_out = kept;
  if (kept > cap) return fail(ctx, ESIKF_ERR_ARG, "rgb_colorize: %d points kept, room for %d", kept, cap);
  if (kept > 0) {
    const size_t K = (size_t)kept;
    CK(read_back(ctx, xyz, index_out ? (const void *)(index + K) : (const void *)(bgr_kept + K * 3)));
    copy_out(ctx, xyz_out, xyz, xyz, K * 3 * sizeof(float)), copy_out(ctx, bgr_out, xyz, bgr_kept, K * 3);
    if (index_out) copy_out(ctx, index_out, xyz, index, K * sizeof(int32_t));
  }
  return ESIKF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- new visual map points
int esikf_vio_generate_points(esikf_ctx *ctx, const double *point_w, const double *normal, const double *var, int32_t n, const double *add_pos,
                              const double *add_normal, int32_t n_add, const uint8_t *type_map, int32_t n_cells, int32_t grid_size, int32_t grid_n_width,
                              int32_t grid_n_height, int32_t border, const double *state, int32_t cap, int32_t *n_out, int32_t *source_out,
                              int32_t *cell_out, double *pos_out, double *pc_out, float *score_out, double *normal_out, double *var_out, float *patch_out) {
  if (!ctx || !n_out || !type_map || cap < 0 || n_add < 0 || (n_add > 0 && (!add_pos || !add_normal)) || (point_w && (n < 0 || !normal || !var)))
    return fail(ctx, ESIKF_ERR_ARG, "vio_generate_points: bad argument");
  if (grid_size <= 0 || grid_n_width <= 0 || grid_n_height <= 0 || border < 0)
    return fail(ctx, ESIKF_ERR_ARG, "vio_generate_points: grid %d px, %d x %d cells, border %d", grid_size, grid_n_width, grid_n_height, border);
  if ((long long)grid_n_width * grid_n_height != n_cells)
    return fail(ctx, ESIKF_ERR_ARG, "vio_generate_points: the TYPE_MAP mask has %d cells, the grid %d x %d", n_cells, grid_n_width, grid_n_height);
  if (int rc = need(ctx, "vio_generate_points", IN_CAMERA | IN_IMAGE | (point_w ? 0 : IN_PV_LIST))) return rc;
  if ((long long)(point_w ? n : ctx->pv_n) + n_add >= ESIKF_GEN_ADD_FROM) return fail(ctx, ESIKF_ERR_ARG, "vio_generate_points: too many points");
  CK(cudaSetDevice(ctx->device));
  *n_out = 0;
  const double *dev_state = nullptr;
  if (int rc = state_or_posterior(ctx, state, esikf_ctx::RESIDENT_VIO, "vio_generate_points", &dev_state)) return rc;
  if (!point_w) n = ctx->pv_n;
  if (n <= 10) return ESIKF_OK;  // :806, add_from included
  cudaStream_t st = ctx->stream;
  const int L = n_cells;
  const size_t N = (size_t)n;
  GenArgs a;
  a.img = ctx->img.p;
  frame_consts(ctx, a.cam, a.Rci, a.Pci);
  a.state = dev_state, a.n = n, a.n_add = n_add, a.pt_stride = MAP_PT_D;
  a.grid_size = grid_size, a.grid_n_width = grid_n_width, a.length = L, a.border = border;
  const size_t M = (size_t)n_add, C = (size_t)L;
  double *pt = nullptr, *pt_normal = nullptr, *add_pos_d, *add_normal_d;
  uint8_t *mask;
  int32_t *d_keep, *d_dst, *d_nk;
  GenOut o;
  float *d_patch;
  // direct copies: staged through the pinned block, a 300 k-point call took 8.2-9.6 ms against 5.8-7.4 ms (H100, 700 W)
  auto lay = [&](ScratchLayout &s) {
    if (point_w) pt = s.take<double>(N * MAP_PT_D + 4), pt_normal = s.take<double>(N * 3 + 4);  // pv_list_ from the host
    add_pos_d = s.take<double>(3 * M + 4), add_normal_d = s.take<double>(3 * M);
    mask = s.take<uint8_t>(C + 16), a.key = s.take<unsigned long long>(C + 1);
    d_keep = s.take<int32_t>(C), d_dst = s.take<int32_t>(C), d_nk = s.take<int32_t>(1), o.source = s.take<int32_t>(C), o.cell = s.take<int32_t>(C);
    o.pos = s.take<double>(3 * C), o.pc = s.take<double>(2 * C), o.normal = s.take<double>(3 * C), o.var = s.take<double>(9 * C);
    o.score = s.take<float>(C), d_patch = s.take<float>(64 * C);
  };
  CK(lay_out_scratch(ctx, lay));
  if (point_w) {  // point_w | var rows as map_pt holds them
    CK(cudaMemcpy2DAsync(pt, MAP_PT_D * sizeof(double), point_w, 3 * sizeof(double), 3 * sizeof(double), N, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpy2DAsync(pt + 3, MAP_PT_D * sizeof(double), var, 9 * sizeof(double), 9 * sizeof(double), N, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(pt_normal, normal, N * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    a.pt = pt, a.normal = pt_normal;
  } else {
    a.pt = ctx->map_pt.p, a.normal = ctx->map_pt_normal.p;
  }
  if (n_add > 0) {
    CK(cudaMemcpyAsync(add_pos_d, add_pos, M * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(add_normal_d, add_normal, M * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  a.add_pos = add_pos_d, a.add_normal = add_normal_d;
  CK(cudaMemcpyAsync(mask, type_map, L, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(a.key, 0, C * sizeof(unsigned long long), st));
  a.type_map = mask;
  CK(launch(ctx, gen_score_kernel, (n + n_add + GEN_THREADS - 1) / GEN_THREADS, GEN_THREADS, 0, a));
  CK(launch(ctx, gen_cells_kernel, (L + 255) / 256, 256, 0, a.key, L, d_keep));
  CK(launch(ctx, select_scan_kernel, 1, SELECT_SCAN_THREADS, 0, d_keep, L, d_dst, d_nk));
  CK(launch(ctx, gen_scatter_kernel, (L + GEN_THREADS - 1) / GEN_THREADS, GEN_THREADS, 0, a, d_keep, d_dst, o));
  int32_t nk = 0;
  CK(cudaMemcpyAsync(&nk, d_nk, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));  // also: the caller may reuse its buffers on return
  *n_out = nk;
  if (nk > cap) return fail(ctx, ESIKF_ERR_ARG, "vio_generate_points: %d new points, room for %d", nk, cap);
  if (nk == 0) return ESIKF_OK;
  if (patch_out) {
    CK(launch(ctx, image_patch_kernel, (nk * 64 + 255) / 256, 256, 0, ctx->img.p, ctx->img_w, ctx->img_h, o.pc, nk, 0, d_patch));
    CK(cudaMemcpyAsync(patch_out, d_patch, (size_t)nk * 64 * sizeof(float), cudaMemcpyDeviceToHost, st));
  }
  const size_t K = (size_t)nk;
  if (source_out) CK(cudaMemcpyAsync(source_out, o.source, K * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (cell_out) CK(cudaMemcpyAsync(cell_out, o.cell, K * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (pos_out) CK(cudaMemcpyAsync(pos_out, o.pos, K * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (pc_out) CK(cudaMemcpyAsync(pc_out, o.pc, K * 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (score_out) CK(cudaMemcpyAsync(score_out, o.score, K * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (normal_out) CK(cudaMemcpyAsync(normal_out, o.normal, K * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (var_out) CK(cudaMemcpyAsync(var_out, o.var, K * 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ESIKF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- new observations of the sub-map
// The largest double x with acos(x) > 0.3 under the host's acos, by bisection over the bit patterns of [0.5, 1] (positive
// doubles order as their bits; acos(0.5) > 0.3 >= acos(1)). acos is decreasing, so delta_theta > 0.3 (vio.cpp:938-939) holds
// exactly when -1 <= 0.5 * (trace - 1) <= this bound.
static double acos_03_bound() {
  uint64_t lo, hi;
  const double a = 0.5, b = 1.0;
  memcpy(&lo, &a, 8), memcpy(&hi, &b, 8);
  while (hi - lo > 1) {
    const uint64_t mid = lo + (hi - lo) / 2;
    double x;
    memcpy(&x, &mid, 8);
    (acos(x) > 0.3 ? lo : hi) = mid;
  }
  double x;
  memcpy(&x, &lo, 8);
  return x;
}

int esikf_vio_update_points(esikf_ctx *ctx, int32_t n, const uint8_t *converged, const double *last_T_f_w, const double *last_px, const double *state,
                            int32_t cap, int32_t *n_out, uint8_t *update_flag_out, int32_t *entry_out, double *pc_out, float *patch_out) {
  if (!ctx || n < 0 || !n_out || cap < 0 || (n > 0 && (!converged || !last_T_f_w || !last_px)))
    return fail(ctx, ESIKF_ERR_ARG, "vio_update_points: bad argument");
  if (int rc = need(ctx, "vio_update_points", IN_CAMERA | IN_EXT | IN_IMAGE | IN_SUBMAP)) return rc;
  if (n != ctx->n_patches) return fail(ctx, ESIKF_ERR_ARG, "vio_update_points: %d entries, the installed sub-map has %d", n, ctx->n_patches);
  CK(cudaSetDevice(ctx->device));
  const double *dev_state = nullptr;
  if (int rc = state_or_posterior(ctx, state, esikf_ctx::RESIDENT_VIO, "vio_update_points", &dev_state)) return rc;
  static const double cos_max = acos_03_bound();
  *n_out = 0;
  if (n == 0) return ESIKF_OK;  // total_points == 0 (:910)
  const size_t N = (size_t)n;
  ObsArgs a;
  double *last_T, *last_px_d, *out_pc;
  uint8_t *conv;
  int32_t *d_keep, *d_dst, *d_nk, *d_entry;
  float *patch;
  auto lay = [&](CallLayout &s) {
    last_T = s.take<double>(12 * N), last_px_d = s.take<double>(2 * N), conv = s.take<uint8_t>(N), s.end_inputs();
    a.pc = s.take<double>(2 * N), d_keep = s.take<int32_t>(N), d_dst = s.take<int32_t>(N);
    s.begin_answers();
    d_nk = s.take<int32_t>(1), a.flag = s.take<uint8_t>(N), d_entry = s.take<int32_t>(N), out_pc = s.take<double>(2 * N), patch = s.take<float>(64 * N);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{last_T, last_T_f_w, N * 12 * sizeof(double)}, {last_px_d, last_px, N * 2 * sizeof(double)}, {conv, converged, N}}));
  frame_consts(ctx, a.cam, a.Rci, a.Pci);
  a.state = dev_state, a.pos = ctx->vis_pos.p, a.converged = conv, a.last_T = last_T, a.last_px = last_px_d;
  a.n = n, a.cos_max = cos_max, a.keep = d_keep;
  CK(launch(ctx, obs_flag_kernel, (n + OBS_THREADS - 1) / OBS_THREADS, OBS_THREADS, 0, a));
  CK(launch(ctx, select_scan_kernel, 1, SELECT_SCAN_THREADS, 0, d_keep, n, d_dst, d_nk));
  CK(launch(ctx, obs_scatter_kernel, (n + 255) / 256, 256, 0, d_keep, d_dst, a.pc, n, d_entry, out_pc));
  int32_t nk;
  CK(read_back_to(ctx, d_nk, &nk));
  *n_out = nk;
  if (nk > cap) return fail(ctx, ESIKF_ERR_ARG, "vio_update_points: %d new observations, room for %d", nk, cap);
  const size_t K = (size_t)nk;
  if (nk > 0 && patch_out) CK(launch(ctx, image_patch_kernel, (nk * 64 + 255) / 256, 256, 0, ctx->img.p, ctx->img_w, ctx->img_h, out_pc, nk, 0, patch));
  const void *f0 = a.flag;
  CK(read_back(ctx, f0, patch_out ? (const void *)(patch + 64 * K) : (const void *)(out_pc + 2 * K)));
  if (update_flag_out) copy_out(ctx, update_flag_out, f0, a.flag, N);
  if (entry_out) copy_out(ctx, entry_out, f0, d_entry, K * sizeof(int32_t));
  if (pc_out) copy_out(ctx, pc_out, f0, out_pc, K * 2 * sizeof(double));
  if (patch_out) copy_out(ctx, patch_out, f0, patch, K * 64 * sizeof(float));
  return ESIKF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- scan side of the retrieval
int esikf_vio_retrieve_scan(esikf_ctx *ctx, const double *point_w, int32_t n, int32_t border, const double *state, int32_t cap, int32_t *n_keys,
                            int32_t *keys_out, float *depth_out) {
  if (!ctx || !n_keys || cap < 0 || border < 0 || (point_w && n < 0) || (cap > 0 && !keys_out)) return fail(ctx, ESIKF_ERR_ARG, "vio_retrieve_scan: bad argument");
  if (int rc = need(ctx, "vio_retrieve_scan", IN_CAMERA | IN_EXT | (point_w ? 0 : IN_PV_LIST))) return rc;
  CK(cudaSetDevice(ctx->device));
  const double *dev_state = nullptr;
  if (int rc = state_or_posterior(ctx, state, esikf_ctx::RESIDENT_LIO, "vio_retrieve_scan", &dev_state)) return rc;
  void_inputs(ctx, IN_RETRIEVAL);
  if (!point_w) n = ctx->pv_n;
  cudaStream_t st = ctx->stream;
  const int W = ctx->cam.width, H = ctx->cam.height;
  const size_t N = (size_t)n, npix = (size_t)W * H;
  size_t sort_bytes = 0, scan_bytes = 0;
  CK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, n, 0, 63,
                                     st));
  CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int32_t *)nullptr, (int32_t *)nullptr, n + 1, st));
  double *pt = nullptr;
  unsigned long long *k_out;
  uint32_t *i_out;
  int32_t *d_head, *d_dst, *d_keys;
  uint8_t *tmp;
  float *depth;
  RetArgs a;
  auto lay = [&](CallLayout &s) {
    if (point_w) pt = s.take<double>(3 * N + 3);  // a host scan
    s.end_inputs();
    a.key = s.take<unsigned long long>(N + 1), k_out = s.take<unsigned long long>(N + 1), a.idx = s.take<uint32_t>(N + 1), i_out = s.take<uint32_t>(N + 1);
    d_head = s.take<int32_t>(N + 1), a.depth_pt = s.take<float>(N + 1), a.win = s.take<int32_t>(npix), tmp = s.take<uint8_t>(std::max(sort_bytes, scan_bytes));
    s.begin_answers();  // dst[n] and bad: the counts
    d_dst = s.take<int32_t>(N + 1), a.bad = s.take<int32_t>(1), d_keys = s.take<int32_t>(3 * N), depth = s.take<float>(npix);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(ctx->ret_state.reserve(S_N));
  CK(ctx->ret_depth.reserve(npix));
  // the frame pose stays with the depth image for esikf_vio_depth_check, whatever a later update writes to `state`
  CK(cudaMemcpyAsync(ctx->ret_state.p, dev_state, S_N * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CK(cudaMemsetAsync(a.win, 0xff, npix * sizeof(int32_t), st));
  CK(cudaMemsetAsync(a.bad, 0, sizeof(int32_t), st));
  frame_consts(ctx, a.cam, a.Rci, a.Pci);
  a.state = ctx->ret_state.p, a.n = n, a.border = border;
  if (point_w) {
    if (n > 0) CK(upload(ctx, {{pt, point_w, 3 * N * sizeof(double)}}));
    a.pt = pt, a.pt_stride = 3;
  } else {
    a.pt = ctx->map_pt.p, a.pt_stride = MAP_PT_D;
  }
  if (n > 0) CK(launch(ctx, ret_scan_kernel, (n + RET_THREADS - 1) / RET_THREADS, RET_THREADS, 0, a));
  CK(launch(ctx, ret_depth_kernel, (int)((npix + 255) / 256), 256, 0, a.win, a.depth_pt, (int)npix, ctx->ret_depth.p));
  int32_t counts[2] = {0, 0};  // distinct keys, bad
  if (n > 0) {
    CK(counted(ctx, cub::DeviceRadixSort::SortPairs(tmp, sort_bytes, a.key, k_out, a.idx, i_out, n, 0, 63, st)));
    CK(launch(ctx, ret_head_kernel, (n + 1 + 255) / 256, 256, 0, k_out, i_out, n, d_head));
    CK(counted(ctx, cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, d_head, d_dst, n + 1, st)));
    CK(launch(ctx, ret_keys_kernel, (n + 255) / 256, 256, 0, d_head, d_dst, a.key, n, d_keys));
  }
  CK(read_back(ctx, d_dst + n, a.bad + 1));  // also: the caller may reuse its buffers on return
  if (n > 0) copy_out(ctx, &counts[0], d_dst + n, d_dst + n, sizeof(int32_t)), copy_out(ctx, &counts[1], d_dst + n, a.bad, sizeof(int32_t));
  if (counts[1]) return fail(ctx, ESIKF_ERR_ARG, "vio_retrieve_scan: a voxel key leaves [-2^20, 2^20)");
  *n_keys = counts[0];
  if (counts[0] > cap) return fail(ctx, ESIKF_ERR_ARG, "vio_retrieve_scan: %d voxel keys, room for %d", counts[0], cap);
  const size_t K = (size_t)counts[0];
  if (depth_out) CK(cudaMemcpyAsync(depth, ctx->ret_depth.p, npix * sizeof(float), cudaMemcpyDeviceToDevice, st));
  CK(read_back(ctx, d_keys, depth_out ? (const void *)(depth + npix) : (const void *)(d_keys + 3 * K)));
  if (K > 0) copy_out(ctx, keys_out, d_keys, d_keys, K * 3 * sizeof(int32_t));
  if (depth_out) copy_out(ctx, depth_out, d_keys, depth, npix * sizeof(float));
  memcpy(ctx->ret_Rci, a.Rci, sizeof(a.Rci)), memcpy(ctx->ret_Pci, a.Pci, sizeof(a.Pci));
  ctx->ret_w = W, ctx->ret_h = H;
  return ESIKF_OK;
}

int esikf_vio_depth_check(esikf_ctx *ctx, int32_t n, const double *pos_w, const double *pc, uint8_t *discontinuous_out) {
  if (!ctx || n < 0 || (n > 0 && (!pos_w || !pc || !discontinuous_out))) return fail(ctx, ESIKF_ERR_ARG, "vio_depth_check: bad argument");
  if (int rc = need(ctx, "vio_depth_check", IN_RETRIEVAL)) return rc;
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  const size_t N = (size_t)n;
  double *pos, *pc_d;
  uint8_t *flag;
  auto lay = [&](CallLayout &s) { pos = s.take<double>(3 * N), pc_d = s.take<double>(2 * N), s.end_inputs(), s.begin_answers(), flag = s.take<uint8_t>(N); };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{pos, pos_w, 3 * N * sizeof(double)}, {pc_d, pc, 2 * N * sizeof(double)}}));
  DepthCheckArgs a;
  memcpy(a.Rci, ctx->ret_Rci, sizeof(a.Rci)), memcpy(a.Pci, ctx->ret_Pci, sizeof(a.Pci));
  a.state = ctx->ret_state.p, a.pos = pos, a.pc = pc_d, a.n = n, a.width = ctx->ret_w, a.height = ctx->ret_h;
  a.depth = ctx->ret_depth.p, a.flag = flag;
  CK(launch(ctx, ret_depth_check_kernel, (n + RET_THREADS - 1) / RET_THREADS, RET_THREADS, 0, a));
  CK(read_back_to(ctx, flag, discontinuous_out, N));
  return ESIKF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- reference patches
int esikf_vio_score_ref_patches(esikf_ctx *ctx, int32_t n, const int32_t *first, int32_t m, const double *pos, const double *normal, const float *patch,
                                const float *mean, const int32_t *id, const double *T_f_w, float *score_out, float *mean_out, int32_t *ref_out) {
  if (!ctx || n < 0 || m < 0 || (n > 0 && (!first || !pos || !normal || !ref_out)) || (m > 0 && (!patch || !mean || !id || !T_f_w || !score_out || !mean_out)))
    return fail(ctx, ESIKF_ERR_ARG, "vio_score_ref_patches: bad argument");
  if (n == 0) return ESIKF_OK;
  if (first[0] != 0 || first[n] != m) return fail(ctx, ESIKF_ERR_ARG, "vio_score_ref_patches: first[0] = %d, first[n] = %d for %d observations", first[0], first[n], m);
  for (int32_t i = 0; i < n; i++)
    if (first[i + 1] < first[i]) return fail(ctx, ESIKF_ERR_ARG, "vio_score_ref_patches: first[%d] > first[%d]", i, i + 1);
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)n, M = (size_t)m;
  double *d_pos, *d_normal, *d_T;
  float *d_patch, *d_mean;
  int32_t *d_first, *d_id;
  RefPatchArgs a;
  a.n = n;
  auto lay = [&](CallLayout &s) {
    d_pos = s.take<double>(3 * N), d_normal = s.take<double>(3 * N), d_T = s.take<double>(12 * M), d_patch = s.take<float>(64 * M), d_mean = s.take<float>(M);
    d_first = s.take<int32_t>(N + 1), d_id = s.take<int32_t>(M);
    s.begin_answers(), a.score = s.take<float>(M), a.mean_out = s.take<float>(M), a.ref = s.take<int32_t>(N);
  };
  CK(lay_out_scratch(ctx, lay));
  // direct copies: staged through the pinned block, 120 k observations took 7.8-11.5 ms a call against 5.0-5.1 ms (H100, 700 W)
  CK(cudaMemcpyAsync(d_pos, pos, 3 * N * sizeof(double), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_normal, normal, 3 * N * sizeof(double), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_first, first, (N + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (m > 0) {
    CK(cudaMemcpyAsync(d_T, T_f_w, 12 * M * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_patch, patch, 64 * M * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_mean, mean, M * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_id, id, M * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  }
  a.pos = d_pos, a.normal = d_normal, a.T = d_T, a.patch = d_patch, a.mean = d_mean, a.id = d_id;
  CK(launch(ctx, refpatch_score_kernel<RpPacked>, (n + RP_WARPS - 1) / RP_WARPS, RP_WARPS * 32, 0, a, RpPacked{d_first}));
  CK(read_back(ctx, a.score, a.ref + N));
  copy_out(ctx, score_out, a.score, a.score, 4 * M);
  copy_out(ctx, mean_out, a.score, a.mean_out, 4 * M);
  copy_out(ctx, ref_out, a.score, a.ref, 4 * N);
  return ESIKF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- visual map observation store
static const int64_t VMAP_MAX_POINTS = (int64_t)1 << 26;  // every slot index p * 30 stays below 2^31

static VmapView vmap_of(esikf_ctx *ctx) { return vmap_view(ctx->vmap.p, (size_t)ctx->vmap_cap); }

// exactly `cap` point records into the empty b
static cudaError_t vmap_alloc(DevBuf<uint8_t> &b, int64_t cap) {
  uint8_t *p = nullptr;
  const size_t bytes = vmap_bytes((size_t)cap);
  const cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return e;
  }
  b.p = p, b.cap = bytes;
  return cudaSuccess;
}

// the point ids of one call: each in [0, points), none twice
static int vmap_check_ids(esikf_ctx *ctx, int32_t n, const int32_t *point_id, const char *what) {
  std::vector<uint32_t> &seen = ctx->vmap_seen;
  if (seen.size() < (size_t)ctx->vmap_points) seen.resize((size_t)ctx->vmap_points, 0);
  if (++ctx->vmap_epoch == 0) std::fill(seen.begin(), seen.end(), 0), ctx->vmap_epoch = 1;  // the epoch wrapped
  const uint32_t e = ctx->vmap_epoch;
  for (int32_t i = 0; i < n; i++) {
    const int32_t p = point_id[i];
    if (p < 0 || p >= ctx->vmap_points) return fail(ctx, ESIKF_ERR_ARG, "%s: point id %d outside [0, %lld)", what, p, (long long)ctx->vmap_points);
    if (seen[p] == e) return fail(ctx, ESIKF_ERR_ARG, "%s: point id %d appears twice", what, p);
    seen[p] = e;
  }
  return ESIKF_OK;
}

int esikf_vmap_init(esikf_ctx *ctx, int64_t point_capacity) {
  if (!ctx || point_capacity < 1 || point_capacity > VMAP_MAX_POINTS) return fail(ctx, ESIKF_ERR_ARG, "vmap_init: capacity %lld outside [1, 2^26]", (long long)point_capacity);
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->vmap = DevBuf<uint8_t>();
  ctx->vmap_cap = ctx->vmap_points = 0;
  ctx->vmap_seen.clear(), ctx->vmap_epoch = 0;
  ctx->vpl = DevBuf<uint8_t>();
  ctx->vpl_cap = ctx->vpl_hi = ctx->vpl_placed = 0;
  ctx->vpl_done.clear();
  CK(vmap_alloc(ctx->vmap, point_capacity));
  ctx->vmap_cap = point_capacity;
  return ESIKF_OK;
}

int esikf_vmap_stats(esikf_ctx *ctx, int64_t *points, int64_t *capacity) {
  if (!ctx || !points || !capacity) return fail(ctx, ESIKF_ERR_ARG, "vmap_stats: bad argument");
  if (int rc = need(ctx, "vmap_stats", IN_STORE)) return rc;
  *points = ctx->vmap_points, *capacity = ctx->vmap_cap;
  return ESIKF_OK;
}

int esikf_vmap_add_points(esikf_ctx *ctx, int32_t n, const int32_t *first, int32_t m, const double *px, const float *patch, const double *T_f_w,
                          const int32_t *id, const float *mean, const float *score, const int32_t *ref, int32_t *point_id_out) {
  if (!ctx) return ESIKF_ERR_ARG;
  if (int rc = need(ctx, "vmap_add_points", IN_STORE)) return rc;
  if (n < 0 || m < 0 || (n > 0 && (!first || !ref || !point_id_out)) || (m > 0 && (!px || !patch || !T_f_w || !id || !mean || !score)))
    return fail(ctx, ESIKF_ERR_ARG, "vmap_add_points: bad argument");
  if (n == 0) return m == 0 ? ESIKF_OK : fail(ctx, ESIKF_ERR_ARG, "vmap_add_points: %d observations for no point", m);
  if (first[0] != 0 || first[n] != m) return fail(ctx, ESIKF_ERR_ARG, "vmap_add_points: first[0] = %d, first[n] = %d for %d observations", first[0], first[n], m);
  for (int32_t i = 0; i < n; i++) {
    const int32_t c = first[i + 1] - first[i];
    if (c < 0 || c > VMAP_SLOTS) return fail(ctx, ESIKF_ERR_ARG, "vmap_add_points: point %d has %d observations (0 .. 30)", i, c);
    if (ref[i] < -1 || ref[i] >= c) return fail(ctx, ESIKF_ERR_ARG, "vmap_add_points: point %d: ref %d of %d observations", i, ref[i], c);
  }
  const int64_t base = ctx->vmap_points, need = base + n;
  if (need > VMAP_MAX_POINTS) return fail(ctx, ESIKF_ERR_ARG, "vmap_add_points: %lld points exceed 2^26", (long long)need);
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  if (need > ctx->vmap_cap) {  // double until the points fit; the old records move over, a failed allocation leaves the store as it was
    int64_t cap = ctx->vmap_cap;
    while (cap < need) cap = std::min(2 * cap, VMAP_MAX_POINTS);
    DevBuf<uint8_t> grown;
    if (vmap_alloc(grown, cap) != cudaSuccess) return fail(ctx, ESIKF_ERR_CUDA, "vmap_add_points: growing the store to %lld points failed", (long long)cap);
    const VmapView o = vmap_of(ctx), v = vmap_view(grown.p, (size_t)cap);
    const size_t P = (size_t)base, S = P * VMAP_SLOTS;
    CK(cudaMemcpyAsync(v.T, o.T, 12 * S * sizeof(double), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(v.px, o.px, 2 * S * sizeof(double), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(v.patch, o.patch, 64 * S * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(v.mean, o.mean, S * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(v.score, o.score, S * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(v.id, o.id, S * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(v.count, o.count, P * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(v.ref, o.ref, P * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    CK(cudaStreamSynchronize(st));
    ctx->vmap = std::move(grown);  // the old records leave with `grown`
    ctx->vmap_cap = cap;
  }
  const size_t N = (size_t)n, M = (size_t)m;
  VmapPackArgs a;
  int32_t *d_pid, *d_first;
  auto lay = [&](CallLayout &s) {
    a.T = s.take<double>(12 * M), a.px = s.take<double>(2 * M), a.patch = s.take<float>(64 * M), a.mean = s.take<float>(M), a.score = s.take<float>(M);
    a.id = s.take<int32_t>(M), a.ref = s.take<int32_t>(N), d_pid = s.take<int32_t>(N), d_first = s.take<int32_t>(N + 1);
    s.end_inputs();
  };
  CK(lay_out_scratch(ctx, lay));
  std::vector<int32_t> pid(N);
  for (size_t i = 0; i < N; i++) pid[i] = (int32_t)(base + (int64_t)i);
  CK(upload(ctx, {{a.T, T_f_w, 12 * M * sizeof(double)}, {a.px, px, 2 * M * sizeof(double)}, {a.patch, patch, 64 * M * sizeof(float)},
                  {a.mean, mean, M * sizeof(float)}, {a.score, score, M * sizeof(float)}, {a.id, id, M * sizeof(int32_t)},
                  {a.ref, ref, N * sizeof(int32_t)}, {d_pid, pid.data(), N * sizeof(int32_t)}, {d_first, first, (N + 1) * sizeof(int32_t)}}));
  a.s = vmap_of(ctx), a.pid = d_pid, a.first = d_first, a.n = n, a.to_store = 1;
  CK(launch(ctx, vmap_pack_kernel, (n + VMAP_WARPS - 1) / VMAP_WARPS, VMAP_WARPS * 32, 0, a));
  CK(cudaStreamSynchronize(st));
  ctx->vmap_points = need;
  memcpy(point_id_out, pid.data(), N * sizeof(int32_t));
  return ESIKF_OK;
}

int esikf_vmap_update_points(esikf_ctx *ctx, int32_t n, const int32_t *point_id, const uint8_t *converged, const double *T_f_w, int32_t frame_id,
                             const double *state, int32_t cap, int32_t *n_out, uint8_t *update_flag_out, int32_t *entry_out, double *pc_out,
                             float *patch_out, int32_t *evicted_out, int32_t *count_out) {
  if (!ctx) return ESIKF_ERR_ARG;
  if (int rc = need(ctx, "vmap_update_points", IN_STORE)) return rc;
  if (n < 0 || !n_out || cap < 0 || (n > 0 && (!point_id || !converged))) return fail(ctx, ESIKF_ERR_ARG, "vmap_update_points: bad argument");
  if (int rc = need(ctx, "vmap_update_points", IN_CAMERA | IN_EXT | IN_IMAGE | IN_SUBMAP)) return rc;
  if (n != ctx->n_patches) return fail(ctx, ESIKF_ERR_ARG, "vmap_update_points: %d entries, the installed sub-map has %d", n, ctx->n_patches);
  if (int rc = vmap_check_ids(ctx, n, point_id, "vmap_update_points")) return rc;
  CK(cudaSetDevice(ctx->device));
  const double *dev_state = nullptr;
  if (int rc = state_or_posterior(ctx, state, esikf_ctx::RESIDENT_VIO, "vmap_update_points", &dev_state)) return rc;
  static const double cos_max = acos_03_bound();
  *n_out = 0;
  if (n == 0) return ESIKF_OK;  // total_points == 0 (:910)
  const size_t N = (size_t)n;
  VmapEditArgs e;
  ObsArgs &a = e.obs;
  int32_t *d_pid, *d_keep, *d_dst, *d_nk, *d_entry, *d_evicted, *d_count;
  uint8_t *conv;
  double *last_T, *last_px, *out_pc, *d_Tnew;
  float *patch;
  auto lay = [&](CallLayout &s) {
    d_pid = s.take<int32_t>(N), conv = s.take<uint8_t>(N), d_Tnew = s.take<double>(12);
    s.end_inputs();
    last_T = s.take<double>(12 * N), last_px = s.take<double>(2 * N), a.pc = s.take<double>(2 * N), d_keep = s.take<int32_t>(N), d_dst = s.take<int32_t>(N);
    s.begin_answers();  // the count, then the rest read back as one span ending with the k patches
    d_nk = s.take<int32_t>(1), a.flag = s.take<uint8_t>(N), d_entry = s.take<int32_t>(N), d_evicted = s.take<int32_t>(N), d_count = s.take<int32_t>(N);
    out_pc = s.take<double>(2 * N), patch = s.take<float>(64 * N);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{d_pid, point_id, N * sizeof(int32_t)}, {conv, converged, N}, {d_Tnew, T_f_w, 12 * sizeof(double)}}));
  e.s = vmap_of(ctx);
  CK(launch(ctx, vmap_last_kernel, (n + 255) / 256, 256, 0, e.s, d_pid, n, last_T, last_px));
  frame_consts(ctx, a.cam, a.Rci, a.Pci);
  a.state = dev_state, a.pos = ctx->vis_pos.p, a.converged = conv, a.last_T = last_T, a.last_px = last_px;
  a.n = n, a.cos_max = cos_max, a.keep = d_keep;
  CK(launch(ctx, obs_flag_kernel, (n + OBS_THREADS - 1) / OBS_THREADS, OBS_THREADS, 0, a));
  CK(launch(ctx, select_scan_kernel, 1, SELECT_SCAN_THREADS, 0, d_keep, n, d_dst, d_nk));
  CK(launch(ctx, obs_scatter_kernel, (n + 255) / 256, 256, 0, d_keep, d_dst, a.pc, n, d_entry, out_pc));
  int32_t nk;
  CK(read_back_to(ctx, d_nk, &nk));
  *n_out = nk;
  // the store is edited only once the answers fit: a call refused here can be repeated with a larger cap
  if (nk > cap) return fail(ctx, ESIKF_ERR_ARG, "vmap_update_points: %d new observations, room for %d", nk, cap);
  if (nk > 0) CK(launch(ctx, image_patch_kernel, (nk * 64 + 255) / 256, 256, 0, ctx->img.p, ctx->img_w, ctx->img_h, out_pc, nk, 0, patch));
  e.pid = d_pid, e.dst = d_dst, e.new_pc = out_pc, e.new_patch = patch, e.T_f_w = T_f_w ? d_Tnew : nullptr, e.frame_id = frame_id;
  e.evicted = d_evicted, e.count = d_count;
  CK(launch(ctx, vmap_edit_kernel, (n + VMAP_WARPS - 1) / VMAP_WARPS, VMAP_WARPS * 32, 0, e));
  CK(read_back(ctx, a.flag, patch + 64 * (size_t)nk));
  const void *f0 = a.flag;
  if (update_flag_out) copy_out(ctx, update_flag_out, f0, a.flag, N);
  if (evicted_out) copy_out(ctx, evicted_out, f0, d_evicted, N * sizeof(int32_t));
  if (count_out) copy_out(ctx, count_out, f0, d_count, N * sizeof(int32_t));
  if (entry_out) copy_out(ctx, entry_out, f0, d_entry, (size_t)nk * sizeof(int32_t));
  if (pc_out) copy_out(ctx, pc_out, f0, out_pc, (size_t)nk * 2 * sizeof(double));
  if (patch_out) copy_out(ctx, patch_out, f0, patch, (size_t)nk * 64 * sizeof(float));
  return ESIKF_OK;
}

int esikf_vmap_score(esikf_ctx *ctx, int32_t n, const int32_t *point_id, const double *pos, const double *normal, int32_t *ref_out, float *score_out,
                     float *mean_out) {
  if (!ctx) return ESIKF_ERR_ARG;
  if (int rc = need(ctx, "vmap_score", IN_STORE)) return rc;
  if (n < 0 || (n > 0 && (!point_id || !pos || !normal || !ref_out))) return fail(ctx, ESIKF_ERR_ARG, "vmap_score: bad argument");
  if (int rc = vmap_check_ids(ctx, n, point_id, "vmap_score")) return rc;
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  const size_t N = (size_t)n;
  int32_t *d_pid;
  double *d_pos, *d_normal;
  float *d_score = nullptr, *d_mean = nullptr;
  RefPatchArgs a;
  auto lay = [&](CallLayout &s) {
    d_pid = s.take<int32_t>(N), d_pos = s.take<double>(3 * N), d_normal = s.take<double>(3 * N);
    s.end_inputs(), s.begin_answers();
    a.ref = s.take<int32_t>(N);
    if (score_out) d_score = s.take<float>(VMAP_SLOTS * N);
    if (mean_out) d_mean = s.take<float>(VMAP_SLOTS * N);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{d_pid, point_id, N * sizeof(int32_t)}, {d_pos, pos, 3 * N * sizeof(double)}, {d_normal, normal, 3 * N * sizeof(double)}}));
  const VmapView v = vmap_of(ctx);
  a.pos = d_pos, a.normal = d_normal, a.T = v.T, a.patch = v.patch, a.mean = v.mean, a.id = v.id, a.n = n;
  a.score = v.score, a.mean_out = v.mean;  // in place
  CK(launch(ctx, refpatch_score_kernel<RpStore>, (n + RP_WARPS - 1) / RP_WARPS, RP_WARPS * 32, 0, a, RpStore{d_pid, v.count, v.ref}));
  if (score_out || mean_out) CK(launch(ctx, vmap_rows_kernel, (n * VMAP_SLOTS + 255) / 256, 256, 0, v, d_pid, n, nullptr, d_score, d_mean));
  const float *end = d_mean ? d_mean + VMAP_SLOTS * N : d_score ? d_score + VMAP_SLOTS * N : nullptr;
  CK(read_back(ctx, a.ref, end ? (const void *)end : (const void *)(a.ref + N)));
  copy_out(ctx, ref_out, a.ref, a.ref, N * sizeof(int32_t));
  if (score_out) copy_out(ctx, score_out, a.ref, d_score, VMAP_SLOTS * N * sizeof(float));
  if (mean_out) copy_out(ctx, mean_out, a.ref, d_mean, VMAP_SLOTS * N * sizeof(float));
  return ESIKF_OK;
}

int esikf_vmap_choose_ref(esikf_ctx *ctx, int32_t n, const int32_t *point_id, const double *pos, const double *frame_pos, int32_t normal_en,
                          int32_t *ref_out) {
  if (!ctx) return ESIKF_ERR_ARG;
  if (int rc = need(ctx, "vmap_choose_ref", IN_STORE)) return rc;
  if (n < 0 || (n > 0 && (!point_id || !ref_out || (!normal_en && (!pos || !frame_pos))))) return fail(ctx, ESIKF_ERR_ARG, "vmap_choose_ref: bad argument");
  if (int rc = vmap_check_ids(ctx, n, point_id, "vmap_choose_ref")) return rc;
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  const size_t N = (size_t)n;
  VmapChooseArgs a;
  int32_t *d_pid;
  double *d_pos;
  auto lay = [&](CallLayout &s) { d_pid = s.take<int32_t>(N), d_pos = s.take<double>(3 * N), s.end_inputs(), s.begin_answers(), a.ref = s.take<int32_t>(N); };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{d_pid, point_id, N * sizeof(int32_t)}, {d_pos, pos, 3 * N * sizeof(double)}}));
  a.s = vmap_of(ctx), a.pid = d_pid, a.pos = d_pos, a.n = n, a.normal_en = normal_en != 0;
  for (int k = 0; k < 3; k++) a.frame_pos[k] = frame_pos ? frame_pos[k] : 0.0;
  CK(launch(ctx, vmap_choose_kernel, (n + VMAP_WARPS - 1) / VMAP_WARPS, VMAP_WARPS * 32, 0, a));
  CK(read_back_to(ctx, a.ref, ref_out, N));
  return ESIKF_OK;
}

int esikf_vmap_download(esikf_ctx *ctx, int32_t n, const int32_t *point_id, int32_t cap, int32_t *first_out, double *px, float *patch, double *T_f_w,
                        int32_t *id, float *mean, float *score, int32_t *ref) {
  if (!ctx) return ESIKF_ERR_ARG;
  if (int rc = need(ctx, "vmap_download", IN_STORE)) return rc;
  if (n < 0 || cap < 0 || !first_out || (n > 0 && (!point_id || !ref)) || (cap > 0 && (!px || !patch || !T_f_w || !id || !mean || !score)))
    return fail(ctx, ESIKF_ERR_ARG, "vmap_download: bad argument");
  if (int rc = vmap_check_ids(ctx, n, point_id, "vmap_download")) return rc;
  if (n == 0) {
    first_out[0] = 0;
    return ESIKF_OK;
  }
  CK(cudaSetDevice(ctx->device));
  const size_t N = (size_t)n;
  int32_t *d_pid, *d_count;
  auto lay1 = [&](CallLayout &s) { d_pid = s.take<int32_t>(N), s.end_inputs(), s.begin_answers(), d_count = s.take<int32_t>(N); };
  CK(lay_out_scratch(ctx, lay1));
  CK(upload(ctx, {{d_pid, point_id, N * sizeof(int32_t)}}));
  const VmapView v = vmap_of(ctx);
  CK(launch(ctx, vmap_rows_kernel, (n * VMAP_SLOTS + 255) / 256, 256, 0, v, d_pid, n, d_count, nullptr, nullptr));
  CK(read_back(ctx, d_count, d_count + N));
  std::vector<int32_t> first(N + 1, 0);
  copy_out(ctx, first.data() + 1, d_count, d_count, N * sizeof(int32_t));
  for (size_t i = 0; i < N; i++) first[i + 1] += first[i];
  const int32_t m = first[N];
  if (m > cap) {
    memcpy(first_out, first.data(), (N + 1) * sizeof(int32_t));
    return fail(ctx, ESIKF_ERR_ARG, "vmap_download: %d observations, room for %d", m, cap);
  }
  const size_t M = (size_t)m;
  VmapPackArgs a;
  int32_t *d_first;
  auto lay2 = [&](CallLayout &s) {
    d_pid = s.take<int32_t>(N), d_first = s.take<int32_t>(N + 1), s.end_inputs(), s.begin_answers();
    a.T = s.take<double>(12 * M), a.px = s.take<double>(2 * M), a.patch = s.take<float>(64 * M), a.mean = s.take<float>(M), a.score = s.take<float>(M);
    a.id = s.take<int32_t>(M), a.ref = s.take<int32_t>(N);
  };
  // the count is known only now, after the readback's synchronisation: the pinned block may be reserved again
  CK(lay_out_scratch(ctx, lay2));
  CK(upload(ctx, {{d_pid, point_id, N * sizeof(int32_t)}, {d_first, first.data(), (N + 1) * sizeof(int32_t)}}));
  a.s = v, a.pid = d_pid, a.first = d_first, a.n = n, a.to_store = 0;
  CK(launch(ctx, vmap_pack_kernel, (n + VMAP_WARPS - 1) / VMAP_WARPS, VMAP_WARPS * 32, 0, a));
  CK(read_back(ctx, a.T, a.ref + N));
  const void *f0 = a.T;
  memcpy(first_out, first.data(), (N + 1) * sizeof(int32_t));
  if (m > 0) {
    copy_out(ctx, T_f_w, f0, a.T, 12 * M * sizeof(double)), copy_out(ctx, px, f0, a.px, 2 * M * sizeof(double));
    copy_out(ctx, patch, f0, a.patch, 64 * M * sizeof(float)), copy_out(ctx, mean, f0, a.mean, M * sizeof(float));
    copy_out(ctx, score, f0, a.score, M * sizeof(float)), copy_out(ctx, id, f0, a.id, M * sizeof(int32_t));
  }
  copy_out(ctx, ref, f0, a.ref, N * sizeof(int32_t));
  return ESIKF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- the map side of the retrieval
int esikf_vmap_place_points(esikf_ctx *ctx, int32_t n, const int32_t *point_id, const double *pos, const uint8_t *normal_init) {
  if (!ctx) return ESIKF_ERR_ARG;
  if (int rc = need(ctx, "vmap_place_points", IN_STORE)) return rc;
  if (n < 0 || (n > 0 && (!point_id || !pos))) return fail(ctx, ESIKF_ERR_ARG, "vmap_place_points: bad argument");
  if (int rc = vmap_check_ids(ctx, n, point_id, "vmap_place_points")) return rc;
  int64_t hi = ctx->vpl_hi;
  for (int32_t i = 0; i < n; i++) {
    const int32_t p = point_id[i];
    if ((size_t)p < ctx->vpl_done.size() && ctx->vpl_done[p]) return fail(ctx, ESIKF_ERR_ARG, "vmap_place_points: point id %d was placed before", p);
    hi = std::max(hi, (int64_t)p + 1);
  }
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  if (hi > ctx->vpl_cap) {  // double until the ids fit; a failed allocation leaves everything as it was
    int64_t cap = std::max<int64_t>(ctx->vpl_cap, 1);
    while (cap < hi) cap = std::min(2 * cap, VMAP_MAX_POINTS);
    uint8_t *p = nullptr;
    if (cudaMalloc(&p, vpl_bytes((size_t)cap)) != cudaSuccess) {
      cudaGetLastError();
      return fail(ctx, ESIKF_ERR_CUDA, "vmap_place_points: growing the point arrays to %lld points failed", (long long)cap);
    }
    DevBuf<uint8_t> grown;
    grown.p = p, grown.cap = vpl_bytes((size_t)cap);
    const VplView v = vpl_view(grown.p, (size_t)cap);
    CK(cudaMemsetAsync(v.key, 0xff, (size_t)cap * sizeof(unsigned long long), st));  // not placed
    if (ctx->vpl_hi > 0) {
      const VplView o = vpl_view(ctx->vpl.p, (size_t)ctx->vpl_cap);
      const size_t P = (size_t)ctx->vpl_hi;
      CK(cudaMemcpyAsync(v.pos, o.pos, 3 * P * sizeof(double), cudaMemcpyDeviceToDevice, st));
      CK(cudaMemcpyAsync(v.key, o.key, P * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
      CK(cudaMemcpyAsync(v.seq, o.seq, P * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
      CK(cudaMemcpyAsync(v.ninit, o.ninit, P, cudaMemcpyDeviceToDevice, st));
    }
    CK(cudaStreamSynchronize(st));
    ctx->vpl = std::move(grown);  // the old arrays leave with `grown`
    ctx->vpl_cap = cap;
  }
  const size_t N = (size_t)n;
  VplArgs a;
  int32_t *d_pid;
  double *d_pos;
  uint8_t *d_ninit = nullptr;
  auto lay = [&](CallLayout &s) {
    d_pid = s.take<int32_t>(N), d_pos = s.take<double>(3 * N);
    if (normal_init) d_ninit = s.take<uint8_t>(N);
    s.end_inputs();
    a.key = s.take<unsigned long long>(N), s.begin_answers(), a.bad = s.take<int32_t>(1);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{d_pid, point_id, N * sizeof(int32_t)}, {d_pos, pos, 3 * N * sizeof(double)}, {d_ninit, normal_init, normal_init ? N : 0}}));
  CK(cudaMemsetAsync(a.bad, 0, sizeof(int32_t), st));
  a.v = vpl_view(ctx->vpl.p, (size_t)ctx->vpl_cap), a.pid = d_pid, a.pos = d_pos, a.ninit = d_ninit, a.n = n, a.seq0 = (int32_t)ctx->vpl_placed;
  CK(launch(ctx, vpl_key_kernel, (n + 255) / 256, 256, 0, a));
  CK(launch(ctx, vpl_commit_kernel, (n + 255) / 256, 256, 0, a));  // writes nothing when a key was out of range
  int32_t bad;
  CK(read_back_to(ctx, a.bad, &bad));
  if (bad) return fail(ctx, ESIKF_ERR_ARG, "vmap_place_points: a voxel key leaves [-2^20, 2^20)");
  ctx->vpl_hi = hi, ctx->vpl_placed += n;
  if (ctx->vpl_done.size() < (size_t)hi) ctx->vpl_done.resize((size_t)hi, 0);
  for (int32_t i = 0; i < n; i++) ctx->vpl_done[point_id[i]] = 1;
  return ESIKF_OK;
}

int esikf_vmap_retrieve(esikf_ctx *ctx, int32_t n_keys, const int32_t *keys, int32_t grid_size, int32_t grid_n_width, int32_t grid_n_height, int32_t border,
                        int32_t normal_en, int32_t cap, int32_t *n_cells, int32_t *cell_out, int32_t *point_id_out, double *pc_out, int32_t *status_out,
                        int32_t *ref_out) {
  if (!ctx) return ESIKF_ERR_ARG;
  if (int rc = need(ctx, "vmap_retrieve", IN_STORE)) return rc;
  if (n_keys < 0 || (n_keys > 0 && !keys) || !n_cells || cap < 0 || border < 0 || (cap > 0 && (!cell_out || !point_id_out || !pc_out || !status_out || !ref_out)))
    return fail(ctx, ESIKF_ERR_ARG, "vmap_retrieve: bad argument");
  if (int rc = need(ctx, "vmap_retrieve", IN_RETRIEVAL)) return rc;
  const int W = ctx->ret_w, H = ctx->ret_h;
  if (grid_size <= 0 || grid_n_width <= 0 || grid_n_height <= 0 || (int64_t)grid_n_width * grid_n_height > (1 << 24) ||
      (int64_t)grid_n_width * grid_size < W - border || (int64_t)grid_n_height * grid_size < H - border)
    return fail(ctx, ESIKF_ERR_ARG, "vmap_retrieve: a %d x %d grid of %d px does not cover the %d x %d image inside a border of %d", grid_n_width, grid_n_height,
                grid_size, W, H, border);
  {  // the walk keys: in the key range, each once
    std::vector<unsigned long long> packed((size_t)n_keys);
    for (int32_t i = 0; i < n_keys; i++) {
      const int32_t *k = keys + 3 * (size_t)i;
      if (!key_in_range(k[0], k[1], k[2])) return fail(ctx, ESIKF_ERR_ARG, "vmap_retrieve: walk key %d leaves [-2^20, 2^20)", i);
      packed[i] = pack_key(k[0], k[1], k[2]);
    }
    std::sort(packed.begin(), packed.end());
    if (std::adjacent_find(packed.begin(), packed.end()) != packed.end()) return fail(ctx, ESIKF_ERR_ARG, "vmap_retrieve: a walk key appears twice");
  }
  if (ctx->vpl_placed == 0 || n_keys == 0) {  // feat_map empty (the reference returns at :354), or nothing to walk
    *n_cells = 0;
    return ESIKF_OK;
  }
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int L = grid_n_width * grid_n_height;
  const size_t K = (size_t)n_keys, NL = (size_t)L;
  uint32_t T = 64;
  while (T < 2 * K) T <<= 1;
  VrtArgs a;
  VrtCellArgs c;
  int32_t *d_keys, *cnt, *ref_tmp;
  unsigned long long *table;
  uint8_t *disc;
  double *fpos;
  auto lay = [&](CallLayout &s) {
    d_keys = s.take<int32_t>(3 * K);
    s.end_inputs();
    table = s.take<unsigned long long>(T), a.wrank = s.take<int32_t>(T);
    a.type = s.take<uint8_t>(NL), a.dist = s.take<uint32_t>(NL), a.tie = s.take<unsigned long long>(NL), a.win = s.take<int32_t>(NL);
    a.pc = s.take<double>(2 * NL), a.wpos = s.take<double>(3 * NL), disc = s.take<uint8_t>(NL);
    c.keep = s.take<int32_t>(NL), c.dst = s.take<int32_t>(NL), c.skeep = s.take<int32_t>(NL), c.sdst = s.take<int32_t>(NL);
    c.spid = s.take<int32_t>(NL), c.sat = s.take<int32_t>(NL), c.spos = s.take<double>(3 * NL), ref_tmp = s.take<int32_t>(NL);
    s.begin_answers();
    fpos = s.take<double>(3), cnt = s.take<int32_t>(2);  // read back first: frame_pos, cells, survivors
    c.pc_out = s.take<double>(2 * NL), c.cell_out = s.take<int32_t>(NL), c.id_out = s.take<int32_t>(NL), c.status_out = s.take<int32_t>(NL);
    c.ref_out = s.take<int32_t>(NL);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{d_keys, keys, 3 * K * sizeof(int32_t)}}));
  CK(cudaMemsetAsync(table, 0xff, T * sizeof(unsigned long long), st));
  CK(launch(ctx, vrt_hash_kernel, (n_keys + 255) / 256, 256, 0, d_keys, n_keys, table, (int32_t *)a.wrank, T - 1));
  CamDev cam;
  frame_consts(ctx, cam, a.Rci, a.Pci);
  memcpy(a.Rci, ctx->ret_Rci, sizeof(a.Rci)), memcpy(a.Pci, ctx->ret_Pci, sizeof(a.Pci));  // the scan call's
  a.cam = cam, a.state = ctx->ret_state.p, a.v = vpl_view(ctx->vpl.p, (size_t)ctx->vpl_cap), a.count = vmap_of(ctx).count, a.n_pts = (int)ctx->vpl_hi;
  a.wkey = table, a.wmask = T - 1, a.grid_size = grid_size, a.grid_n_width = grid_n_width, a.length = L, a.border = border, a.frame_pos = fpos;
  CK(launch(ctx, vrt_init_kernel, (L + 255) / 256, 256, 0, a));
  const int pb = (a.n_pts + VRT_THREADS - 1) / VRT_THREADS;
  CK(launch(ctx, vrt_walk_kernel<0>, pb, VRT_THREADS, 0, a));
  CK(launch(ctx, vrt_walk_kernel<1>, pb, VRT_THREADS, 0, a));
  CK(launch(ctx, vrt_walk_kernel<2>, pb, VRT_THREADS, 0, a));
  DepthCheckArgs dc;  // K11's check on every cell's winner (a cell without one is not read)
  memcpy(dc.Rci, ctx->ret_Rci, sizeof(dc.Rci)), memcpy(dc.Pci, ctx->ret_Pci, sizeof(dc.Pci));
  dc.state = ctx->ret_state.p, dc.pos = a.wpos, dc.pc = a.pc, dc.n = L, dc.width = W, dc.height = H, dc.depth = ctx->ret_depth.p, dc.flag = disc;
  CK(launch(ctx, ret_depth_check_kernel, (L + RET_THREADS - 1) / RET_THREADS, RET_THREADS, 0, dc));
  c.length = L, c.type = a.type, c.disc = disc, c.ninit = a.v.ninit, c.win = a.win, c.pc = a.pc, c.wpos = a.wpos;
  CK(launch(ctx, vrt_cells_kernel<true>, (L + 255) / 256, 256, 0, c));
  CK(launch(ctx, select_scan_kernel, 1, SELECT_SCAN_THREADS, 0, c.keep, L, c.dst, cnt));
  CK(launch(ctx, select_scan_kernel, 1, SELECT_SCAN_THREADS, 0, c.skeep, L, c.sdst, cnt + 1));
  CK(launch(ctx, vrt_cells_kernel<false>, (L + 255) / 256, 256, 0, c));
  // vmap_choose_kernel takes its count and new_frame_->pos() by value: both come back before it runs, and a call refused for
  // its cap has not touched the store
  CK(read_back(ctx, fpos, cnt + 2));
  double fp[3];
  int32_t counts[2];
  copy_out(ctx, fp, fpos, fpos, sizeof(fp)), copy_out(ctx, counts, fpos, cnt, sizeof(counts));
  *n_cells = counts[0];
  if (counts[0] > cap) return fail(ctx, ESIKF_ERR_ARG, "vmap_retrieve: %d cells, room for %d", counts[0], cap);
  const int ns = counts[1];
  if (ns > 0) {
    VmapChooseArgs ca;
    ca.s = vmap_of(ctx), ca.pid = c.spid, ca.pos = c.spos, ca.n = ns, ca.normal_en = normal_en != 0, ca.ref = ref_tmp;
    for (int k = 0; k < 3; k++) ca.frame_pos[k] = fp[k];
    CK(launch(ctx, vmap_choose_kernel, (ns + VMAP_WARPS - 1) / VMAP_WARPS, VMAP_WARPS * 32, 0, ca));
    CK(launch(ctx, vrt_refs_kernel, (ns + 255) / 256, 256, 0, ref_tmp, c.sat, ns, c.ref_out, c.status_out));
  }
  const size_t M = (size_t)counts[0];
  CK(read_back(ctx, c.pc_out, c.ref_out + M));
  const void *f0 = c.pc_out;
  if (M > 0) {
    copy_out(ctx, pc_out, f0, c.pc_out, 2 * M * sizeof(double)), copy_out(ctx, cell_out, f0, c.cell_out, M * sizeof(int32_t));
    copy_out(ctx, point_id_out, f0, c.id_out, M * sizeof(int32_t)), copy_out(ctx, status_out, f0, c.status_out, M * sizeof(int32_t));
    copy_out(ctx, ref_out, f0, c.ref_out, M * sizeof(int32_t));
  }
  return ESIKF_OK;
}

}  // extern "C"
