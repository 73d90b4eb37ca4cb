// The ESIKF updates: LIO / VIO set, run and fetch (one persistent cooperative kernel per update, or one residual + one solve
// launch per iteration), the patch producers that install the visual sub-map, and esikf_profile_kernel.
#include <cuda.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include "esikf_api.cuh"

#include "esikf_lio.cu"
#include "esikf_solve.cu"
#include "esikf_vio.cu"
#include "esikf_fused.cu"

#define VIO_PERSIST_SMEM (sizeof(VioSmem) + sizeof(FusedSolveSmem))

static cudaEvent_t *timing_events(esikf_ctx *ctx, int base, int slot) {
  size_t need = (size_t)(base + slot + 1) * 3;
  while (ctx->ev.size() < need) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return cudaGetLastError(), nullptr;  // the run goes on untimed; no later launch reports this
    ctx->ev.push_back(e);
  }
  return &ctx->ev[(size_t)(base + slot) * 3];
}

// Dynamic shared memory and occupancy of the LIO kernels of one CTA geometry (L2W L2-slot warps), with their resources
// under ESIKF_DEBUG. Returns the co-resident CTAs per SM of its persistent kernels.
template <int L2W> static int lio_kernels_setup(bool debug) {
  const int smem = (int)sizeof(LioSmem<L2W>), threads = LioSmem<L2W>::THREADS;
  cudaFuncSetAttribute(lio_residual_kernel<L2W>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaFuncSetAttribute(lio_update_kernel<false, L2W>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaFuncSetAttribute(lio_update_kernel<true, L2W>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  int occ_l = 0, occ_lp = 0, occ_r = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_l, lio_update_kernel<false, L2W>, threads, smem);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_lp, lio_update_kernel<true, L2W>, threads, smem);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_r, lio_residual_kernel<L2W>, threads, smem);
  if (debug) {
    cudaFuncAttributes fr, fu;
    cudaFuncGetAttributes(&fr, lio_residual_kernel<L2W>);
    cudaFuncGetAttributes(&fu, lio_update_kernel<false, L2W>);
    fprintf(stderr, "[esikf] LIO %d lanes: smem=%d occupancy lio_update=%d/%d lio_residual=%d; lio_residual regs=%d local=%zu; lio_update regs=%d local=%zu\n", threads,
            smem, occ_l, occ_lp, occ_r, fr.numRegs, fr.localSizeBytes, fu.numRegs, fu.localSizeBytes);
  }
  return occ_l < occ_lp ? occ_l : occ_lp;
}

// The 768-lane kernel (LIO_L2_WARPS L2-slot warps) runs where its lanes hold every CTA's slice and the 704 lanes of the other
// one would not: 23 or 24 chunks of 32 points per CTA (config 2's 100 k points on 132 SMs). Smaller slices are resident in
// 704 lanes too. A larger slice is tiled either way, and the 704-lane kernel tiles faster: its lanes all have shared-memory
// slots, while the L2-slot lanes would be cold in every tile.
static bool lio_use_l2_slots(int count, int grid) {
  const int chunks = (count + 31) / 32, per_cta = (chunks + grid - 1) / grid;
  return LIO_L2_WARPS > 0 && per_cta > LIO_SMEM_WARPS && per_cta <= LIO_SMEM_WARPS + LIO_L2_WARPS;
}
static cudaError_t launch_lio_residual(esikf_ctx *ctx, bool l2_slots, int grid, const LioKernelArgs &ka) {
  if (l2_slots) return launch(ctx, lio_residual_kernel<LIO_L2_WARPS>, grid, LioSmem<LIO_L2_WARPS>::THREADS, sizeof(LioSmem<LIO_L2_WARPS>), ka);
  return launch(ctx, lio_residual_kernel<0>, grid, LioSmem<0>::THREADS, sizeof(LioSmem<0>), ka);
}

cudaError_t update_kernels_setup(esikf_ctx *ctx) {
  cudaError_t e;
  if ((e = ctx->grid_mbox.reserve(grid_mbox_words(ctx->partial_blocks) + 1)) ||
      (e = ctx->lio_slot_block.reserve((size_t)ctx->partial_blocks * LIO_L2_WARPS * 32 * SLOT_D)))
    return e;
  cudaMemsetAsync(ctx->grid_mbox.p, 0, ctx->grid_mbox.cap * sizeof(unsigned long long), ctx->stream);  // tag 0 is never sent
  ctx->exchange_seq = reinterpret_cast<unsigned int *>(ctx->grid_mbox.p + grid_mbox_words(ctx->partial_blocks));
  cudaFuncSetAttribute(vio_patch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(VioSmem));
  cudaFuncSetAttribute(vio_inverse_patch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(VioSmem));
  cudaError_t eb = cudaFuncSetAttribute(vio_update_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)VIO_PERSIST_SMEM);
  cudaFuncSetAttribute(vio_update_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)VIO_PERSIST_SMEM);
  cudaFuncSetAttribute(vio_update_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)VIO_PERSIST_SMEM);
  cudaFuncSetAttribute(vio_update_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)VIO_PERSIST_SMEM);
  // the persistent kernels need every CTA co-resident: check what the device can hold
  const bool debug = getenv("ESIKF_DEBUG") != nullptr;
  const int occ_l0 = lio_kernels_setup<0>(debug), occ_l2 = lio_kernels_setup<LIO_L2_WARPS>(debug);
  int occ_v = 0, occ_vp = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_v, vio_update_kernel<false, false>, VIO_THREADS, VIO_PERSIST_SMEM);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_vp, vio_update_kernel<true, true>, VIO_THREADS, VIO_PERSIST_SMEM);
  ctx->coop_lio = occ_l0 < occ_l2 ? occ_l0 : occ_l2, ctx->coop_vio = occ_v < occ_vp ? occ_v : occ_vp;
  if (debug) {
    fprintf(stderr, "[esikf] SMs=%d smem VIO=%zu attr=%d occupancy: vio_update=%d coop=%d\n", ctx->sm_count, VIO_PERSIST_SMEM, (int)eb, occ_v, ctx->coop_ok);
    cudaFuncAttributes fa;
    cudaFuncGetAttributes(&fa, vio_update_kernel<false, false>);
    fprintf(stderr, "[esikf] vio_update: regs=%d local=%zu\n", fa.numRegs, fa.localSizeBytes);
  }
  return cudaSuccess;
}

extern "C" {

// ---------------------------------------------------------------------------------------------------------------- LIO
int esikf_lio_set_scan(esikf_ctx *ctx, const float *pts_xyz, int32_t n) {
  if (!ctx || n < 0 || (n > 0 && !pts_xyz)) return fail(ctx, ESIKF_ERR_ARG, "lio_set_scan: bad argument");
  CK(cudaSetDevice(ctx->device));
  CK(ctx->pts.reserve((size_t)n * 3 + 4));
  ctx->pre_stride = (n + 31) & ~31;
  CK(ctx->pre.reserve((size_t)ctx->pre_stride * 9 + 16));
  CK(ctx->match_plane.reserve(n + 1));
  CK(ctx->normal_plane.reserve(n + 1));
  CK(ctx->dis.reserve(n + 1));
  if (n) CK(cudaMemcpyAsync(ctx->pts.p, pts_xyz, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  ctx->n_pts = n;
  ctx->scan = esikf_ctx::SCAN_SET;
  return ESIKF_OK;
}

// calcBodyCov and the cross-matrix vector of every point of the resident scan (voxel_map.cpp:349-360). StateEstimation
// recomputes both every call; here they are kept with what they were made from and redone only when the scan, the lidar
// extrinsics or the noise model changed.
static cudaError_t lio_precompute(esikf_ctx *ctx, float dept_err, float beam_err) {
  const cudaError_t e = launch(ctx, lio_precompute_kernel, (ctx->n_pts + 255) / 256, 256, 0, ctx->pts.p, ctx->n_pts, ctx->pre.p, ctx->pre_stride, ctx->ext_dev.p,
                               dept_err, beam_err);
  if (e) return e;
  memcpy(ctx->pre_ext, ctx->ext_host, sizeof(ctx->pre_ext));
  ctx->pre_dept_err = dept_err, ctx->pre_beam_err = beam_err;
  return cudaSuccess;
}
static bool lio_precompute_current(const esikf_ctx *ctx, float dept_err, float beam_err) {
  return ctx->scan != esikf_ctx::SCAN_SET && memcmp(ctx->pre_ext, ctx->ext_host, sizeof(ctx->pre_ext)) == 0 && ctx->pre_dept_err == dept_err && ctx->pre_beam_err == beam_err;
}

static int lio_fill_args(esikf_ctx *ctx, LioKernelArgs &ka, double *state_ptr) {
  memset(&ka, 0, sizeof(ka));
  ka.pts = ctx->pts.p, ka.pre = ctx->pre.p;
  ka.pre_stride = ctx->pre_stride;
  ka.partial_stride = ctx->partial_blocks;
  shard_of(ctx->n_pts, ctx->rank, ctx->nranks, ka.begin, ka.count);
  ka.state = state_ptr, ka.prop = ctx->prop;
  ka.slots = ctx->map.slots.p, ka.hash_mask = ctx->hash_mask, ka.recs = ctx->map.recs.p;
  ka.stage_mode = (ctx->tuning & ESIKF_TUNE_STAGE_LDG) ? 1 : 0;
  memcpy(ka.extR, ctx->ext.extR, sizeof(ka.extR));
  memcpy(ka.extT, ctx->ext.extT, sizeof(ka.extT));
  ka.voxel_size = ctx->lio_cfg.voxel_size;
  ka.inv_voxel_size = 1.0 / ctx->lio_cfg.voxel_size;
  {
    int ex = 0;
    ka.inv_voxel_exact = (frexp(ctx->lio_cfg.voxel_size, &ex) == 0.5) ? 1 : 0;  // power of two: the reciprocal is exact
  }
  ka.voxel_size_f = (float)ctx->lio_cfg.voxel_size;
  ka.sigma_num = ctx->lio_cfg.sigma_num;
  ka.prob_sure_sigma = prob_sure_sigma_of(ka.sigma_num);
  ka.match_plane = ctx->match_plane.p, ka.normal_plane = ctx->normal_plane.p, ka.dis_to_plane = ctx->dis.p;
  ka.partials = ctx->partials.p, ka.info = ctx->info.p, ka.ctrl = ctx->ctrl;
  ka.slot_block = ctx->lio_slot_block.p;
  return 0;
}
static int lio_grid(const esikf_ctx *ctx, int count) {
  int chunks = (count + 31) / 32;  // whole warps are dealt to the CTAs: every SM takes part as soon as there is a warp for it
  int g = chunks < ctx->partial_blocks ? chunks : ctx->partial_blocks;
  return g < 1 ? 1 : g;
}
// Stage the two packed states of an update in pinned memory and upload them with ONE copy ([state | prop] is contiguous).
static int upload_states(esikf_ctx *ctx, const double *state_in, const double *state_prop) {
  void_inputs(ctx, IN_POSTERIOR);  // until the update's launch has succeeded
  const unsigned slot = ctx->stage_idx++ % esikf_ctx::STAGE_SLOTS;
  CK(cudaEventSynchronize(ctx->stage_ev[slot]));  // the copy that last used this slot has been consumed
  double *h = ctx->stage + (size_t)slot * 2 * S_N;
  memcpy(h, state_in, S_N * sizeof(double));
  memcpy(h + S_N, state_prop, S_N * sizeof(double));
  CK(cudaMemcpyAsync(ctx->state_prop.p, h, 2 * S_N * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaEventRecord(ctx->stage_ev[slot], ctx->stream));
  return ESIKF_OK;
}
static int allreduce_info(esikf_ctx *ctx) {
  if (ctx->nranks <= 1) return ESIKF_OK;
  if (!ctx->comm) return fail(ctx, ESIKF_ERR_STATE, "per-iteration launches with %d ranks need esikf_comm_init (NCCL)", ctx->nranks);
  int r = g_nccl.AllReduce(ctx->info.p, ctx->info.p, NE_MAX, NCCL_FLOAT64, NCCL_SUM, ctx->comm, ctx->stream);
  if (r != 0) return fail(ctx, ESIKF_ERR_COMM, "ncclAllReduce failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
  return ESIKF_OK;
}

// The SolveArgs fields every solve reads; the LIO / VIO callers add their own.
static SolveArgs solve_args(const esikf_ctx *ctx, double *state, int max_iterations) {
  SolveArgs sa;
  memset(&sa, 0, sizeof(sa));
  sa.state = state, sa.prop = ctx->prop, sa.info = ctx->info.p, sa.ctrl = ctx->ctrl;
  sa.max_iterations = max_iterations, sa.solve_mode = ctx->solve_mode;
  return sa;
}

// One persistent cooperative kernel per update (coop_blocks: co-resident CTAs per SM of that kernel); otherwise one
// residual + one solve launch per iteration.
static bool persistent_update(const esikf_ctx *ctx, int coop_blocks) {
  return ctx->loop_mode >= 1 && (ctx->nranks == 1 || ctx->p2p) && ctx->coop_ok && coop_blocks > 0 && !ctx->timing;
}

// Cooperative launch of lio_update_kernel<PEER, L2W> / vio_update_kernel<PEER, INVERSE>. Their arguments are
// (ka, sa, grid sync, stamps, peer, tail...): `ka` is the kernel's LioKernelArgs /
// VioKernelArgs, `tail` the VIO-only arguments. Both instantiations get the same argument list, so the single-GPU
// launch passes exactly what the peer launch does. `stamp_off` / `stamp_words`: this kernel's slice of the phase stamps.
static int launch_persistent(esikf_ctx *ctx, const void *fn, const void *fn_peer, const char *name, int grid, int threads, size_t smem, void *ka, SolveArgs &sa,
                             size_t stamp_off, size_t stamp_words, bool &timed, std::initializer_list<void *> tail, esikf_ctx::Resident posterior) {
  const unsigned par = ctx->launch_parity & 1;
  GridSync gs;
  gs.barrier = ctx->barrier.p + 64 * par, gs.barrier_next = ctx->barrier.p + 64 * (par ^ 1);  // this launch's barrier / the next launch's (zeroed by the kernel)
  gs.mbox = ctx->grid_mbox.p;
  unsigned long long *stamps = ctx->want_stamps ? ctx->stamps.p + stamp_off : nullptr;
  if (stamps) CK(cudaMemsetAsync(stamps, 0, stamp_words * sizeof(unsigned long long), ctx->stream));
  PeerArgs peer;
  peer.mbox = ctx->p2p ? ctx->peer_ptrs_dev.p : nullptr, peer.seq = ctx->exchange_seq;
  peer.rank = ctx->rank, peer.nranks = ctx->p2p ? ctx->nranks : 1;
  void *kargs[7] = {ka, (void *)&sa, (void *)&gs, (void *)&stamps, (void *)&peer};
  std::copy(tail.begin(), tail.end(), kargs + 5);
  cudaError_t le = cudaLaunchCooperativeKernel(ctx->p2p && ctx->nranks > 1 ? fn_peer : fn, dim3(grid), dim3(threads), kargs, smem, ctx->stream);
  if (le != cudaSuccess) return fail(ctx, ESIKF_ERR_CUDA, "cooperative launch of %s failed: %s", name, cudaGetErrorString(le));
  ctx->launch_parity++;  // only a launch that happened consumes its barrier counter (the kernel zeroes the other one)
  ctx->launches += 1;
  ctx->resident = posterior;  // what `state` holds once the launch has happened
  timed = false;
  return ESIKF_OK;
}

int esikf_lio_run(esikf_ctx *ctx, const double *state_in, const double *state_prop, const esikf_lio_cfg *cfg) {
  if (!ctx || !state_in || !state_prop || !cfg) return fail(ctx, ESIKF_ERR_ARG, "lio_run: null argument");
  if (int rc = need(ctx, "lio_run", IN_MAP | IN_EXT)) return rc;
  void_inputs(ctx, IN_NORMALS);  // a snapshot of pv.normal belongs to the update it was taken after
  if (cfg->max_iterations < 1 || cfg->max_iterations > 8) return fail(ctx, ESIKF_ERR_ARG, "lio_run: max_iterations must be in [1,8]");
  CK(cudaSetDevice(ctx->device));
  ctx->lio_cfg = *cfg;
  cudaStream_t st = ctx->stream;
  if (int rc = upload_states(ctx, state_in, state_prop)) return rc;
  const bool fused_lio = persistent_update(ctx, ctx->coop_lio);
  // the persistent kernel initialises its own loop control / stats / barrier; the per-iteration path needs them zeroed
  if (!fused_lio) CK(cudaMemsetAsync(ctx->lio_stats, 0, sizeof(esikf_lio_stats) + sizeof(Ctrl) + 64, st));
  const int n = ctx->n_pts;
  const float dept_err = (float)cfg->dept_err, beam_err = (float)cfg->beam_err;
  if (!lio_precompute_current(ctx, dept_err, beam_err)) {
    if (n > 0) CK(lio_precompute(ctx, dept_err, beam_err));
    if (ctx->scan == esikf_ctx::SCAN_SET) ctx->scan = esikf_ctx::SCAN_RUN;
  }
  LioKernelArgs ka;
  lio_fill_args(ctx, ka, ctx->state);
  SolveArgs sa = solve_args(ctx, ctx->state, cfg->max_iterations);
  sa.lio_stats = ctx->lio_stats;
  const int grid = lio_grid(ctx, ka.count);
  const bool l2_slots = lio_use_l2_slots(ka.count, grid);
  if (fused_lio && l2_slots)
    return launch_persistent(ctx, (const void *)lio_update_kernel<false, LIO_L2_WARPS>, (const void *)lio_update_kernel<true, LIO_L2_WARPS>, "lio_update_kernel", grid,
                             LioSmem<LIO_L2_WARPS>::THREADS, sizeof(LioSmem<LIO_L2_WARPS>), &ka, sa, 0, 64, ctx->lio_timed, {}, esikf_ctx::RESIDENT_LIO);
  if (fused_lio)
    return launch_persistent(ctx, (const void *)lio_update_kernel<false, 0>, (const void *)lio_update_kernel<true, 0>, "lio_update_kernel", grid, LioSmem<0>::THREADS,
                             sizeof(LioSmem<0>), &ka, sa, 0, 64, ctx->lio_timed, {}, esikf_ctx::RESIDENT_LIO);
  ctx->lio_timed = ctx->timing;
  ctx->lio_slots = cfg->max_iterations;
  for (int it = 0; it < cfg->max_iterations; it++) {
    cudaEvent_t *e = ctx->timing ? timing_events(ctx, EV_LIO_BASE, it) : nullptr;
    if (e) CK(cudaEventRecord(e[0], st));
    ka.init_normal = (it == 0);
    CK(launch_lio_residual(ctx, l2_slots, grid, ka));
    if (e) CK(cudaEventRecord(e[1], st));
    int rc = allreduce_info(ctx);
    if (rc) return rc;
    CK(launch(ctx, lio_solve_kernel, 1, SOLVE_THREADS, 0, sa));
    if (e) CK(cudaEventRecord(e[2], st));
  }
  ctx->resident = esikf_ctx::RESIDENT_LIO;
  return ESIKF_OK;
}

// Common tail of the fetch calls: bring the loop-control block along, synchronise, and turn an expired in-kernel wait
// (Ctrl::comm_error, sticky on the device) into ESIKF_ERR_COMM once.
static int finish_fetch(esikf_ctx *ctx) {
  Ctrl *h = reinterpret_cast<Ctrl *>(ctx->stage_ctrl);
  CK(cudaMemcpyAsync(h, ctx->ctrl, sizeof(Ctrl), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (h->comm_error) {
    CK(cudaMemsetAsync(&ctx->ctrl->comm_error, 0, sizeof(int), ctx->stream));
    return fail(ctx, ESIKF_ERR_COMM, "a bounded in-kernel wait expired (grid barrier, grid or peer mailbox): a rank did not take part in the update");
  }
  return ESIKF_OK;
}

int esikf_lio_fetch(esikf_ctx *ctx, double *state_out, esikf_lio_stats *stats, int32_t *match_plane, int32_t *normal_plane, float *dis_to_plane) {
  if (!ctx) return ESIKF_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t n = (size_t)ctx->n_pts;
  if (state_out) CK(cudaMemcpyAsync(state_out, ctx->state, S_N * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (stats) CK(cudaMemcpyAsync(stats, ctx->lio_stats, sizeof(esikf_lio_stats), cudaMemcpyDeviceToHost, st));
  if (match_plane && n) CK(cudaMemcpyAsync(match_plane, ctx->match_plane.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (normal_plane && n) CK(cudaMemcpyAsync(normal_plane, ctx->normal_plane.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (dis_to_plane && n) CK(cudaMemcpyAsync(dis_to_plane, ctx->dis.p, n * sizeof(float), cudaMemcpyDeviceToHost, st));
  return finish_fetch(ctx);
}

int esikf_lio_update(esikf_ctx *ctx, const float *pts_xyz, int32_t n, const double *state_in, const double *state_prop, const esikf_lio_cfg *cfg,
                     double *state_out, esikf_lio_stats *stats, int32_t *match_plane, int32_t *normal_plane, float *dis_to_plane) {
  int rc = esikf_lio_set_scan(ctx, pts_xyz, n);
  if (rc) return rc;
  rc = esikf_lio_run(ctx, state_in, state_prop, cfg);
  if (rc) return rc;
  return esikf_lio_fetch(ctx, state_out, stats, match_plane, normal_plane, dis_to_plane);
}

__global__ void expand_point_cov_kernel(const double *__restrict__ pre, int pre_stride, int n, double *__restrict__ body_cov9, double *__restrict__ cross9) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double p[9];
  for (int k = 0; k < 9; k++) p[k] = pre[(size_t)k * pre_stride + i];
  if (body_cov9) {
    double *o = body_cov9 + 9 * (size_t)i;
    o[0] = p[3], o[1] = p[4], o[2] = p[5], o[3] = p[4], o[4] = p[6], o[5] = p[7], o[6] = p[5], o[7] = p[7], o[8] = p[8];
  }
  if (cross9) {
    double *o = cross9 + 9 * (size_t)i;
    o[0] = 0, o[1] = -p[2], o[2] = p[1], o[3] = p[2], o[4] = 0, o[5] = -p[0], o[6] = -p[1], o[7] = p[0], o[8] = 0;
  }
}

int esikf_lio_fetch_point_cov(esikf_ctx *ctx, double *body_cov9, double *cross_mat9) {
  if (!ctx) return ESIKF_ERR_ARG;
  if (int rc = need(ctx, "fetch_point_cov", IN_RUN_SCAN)) return rc;
  CK(cudaSetDevice(ctx->device));
  const int n = ctx->n_pts;
  if (n == 0) return ESIKF_OK;
  const size_t N9 = (size_t)n * 9;
  double *body, *cross;
  auto lay = [&](CallLayout &s) { s.begin_answers(), body = s.take<double>(N9), cross = s.take<double>(N9); };
  CK(lay_out_scratch(ctx, lay));
  CK(launch(ctx, expand_point_cov_kernel, (n + 255) / 256, 256, 0, ctx->pre.p, ctx->pre_stride, n, body_cov9 ? body : nullptr, cross_mat9 ? cross : nullptr));
  const double *f0 = body_cov9 ? body : cross;
  CK(read_back(ctx, f0, cross_mat9 ? cross + N9 : body_cov9 ? body + N9 : f0));
  if (body_cov9) copy_out(ctx, body_cov9, f0, body, N9 * sizeof(double));
  if (cross_mat9) copy_out(ctx, cross_mat9, f0, cross, N9 * sizeof(double));
  return ESIKF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- VIO
// The installed sub-map's buffers, reserved for n patches of L levels (growing discards their contents), and the record of
// what they hold once they are filled. set_patches, warp_patches(keep_on_device) and select_patches install one.
static int install_submap(esikf_ctx *ctx, int n, int L) {
  CK(ctx->vis_pos.reserve((size_t)n * 3 + 4));
  CK(ctx->warp_patch.reserve((size_t)n * 64 * L + 64));
  CK(ctx->search_levels.reserve(n + 1));
  CK(ctx->inv_expo.reserve(n + 1));
  CK(ctx->errors.reserve(n + 1));
  return ESIKF_OK;
}
static void commit_submap(esikf_ctx *ctx, int n, int L) { ctx->n_patches = n, ctx->submap_levels = L; }

// ESIKF_ERR_ARG naming `call` when `index` names none of the reference images.
static int check_ref_image(esikf_ctx *ctx, const char *call, int32_t index) {
  if (index < 0 || index >= (int)ctx->ref_imgs.size()) return fail(ctx, ESIKF_ERR_ARG, "%s: ref image index %d", call, index);
  return ESIKF_OK;
}

int esikf_vio_set_camera(esikf_ctx *ctx, const esikf_camera *cam, const esikf_vio_cfg *cfg) {
  if (!ctx || !cam || !cfg) return fail(ctx, ESIKF_ERR_ARG, "vio_set_camera: null argument");
  if (cam->model < 0 || cam->model > 1 || cam->width <= 0 || cam->height <= 0) return fail(ctx, ESIKF_ERR_ARG, "vio_set_camera: bad camera");
  if (cfg->patch_pyrimid_level < 1 || cfg->patch_pyrimid_level > 8 || cfg->max_iterations < 1 || cfg->max_iterations > 8 || !(cfg->img_point_cov > 0))
    return fail(ctx, ESIKF_ERR_ARG, "vio_set_camera: bad vio cfg");
  const bool resized = cam->width != ctx->cam.width || cam->height != ctx->cam.height;  // a first camera voids no sub-map
  void_inputs(ctx, IN_RETRIEVAL | (resized ? IN_IMAGE : 0) | (ctx->cam.width && cfg->patch_pyrimid_level != ctx->vio_cfg.patch_pyrimid_level ? IN_SUBMAP : 0));
  ctx->cam = *cam;
  ctx->vio_cfg = *cfg;
  return ESIKF_OK;
}

int esikf_vio_set_image(esikf_ctx *ctx, const uint8_t *img, int32_t width, int32_t height) {
  if (!ctx || !img || width <= 0 || height <= 0) return fail(ctx, ESIKF_ERR_ARG, "vio_set_image: bad argument");
  if (int rc = need(ctx, "vio_set_image", IN_CAMERA)) return rc;
  if (width != ctx->cam.width || height != ctx->cam.height) return fail(ctx, ESIKF_ERR_ARG, "vio_set_image: image is %dx%d, camera %dx%d", width, height, ctx->cam.width, ctx->cam.height);
  CK(cudaSetDevice(ctx->device));
  CK(ctx->img.reserve((size_t)width * height + 64));
  CK(cudaMemcpyAsync(ctx->img.p, img, (size_t)width * height, cudaMemcpyHostToDevice, ctx->stream));
  ctx->img_w = width, ctx->img_h = height;
  return ESIKF_OK;
}

int esikf_vio_set_patches(esikf_ctx *ctx, const double *pos, const float *warp_patch, const int32_t *search_levels, const double *inv_expo_list, int32_t n) {
  if (!ctx || n < 0 || (n > 0 && (!pos || !warp_patch || !search_levels || !inv_expo_list))) return fail(ctx, ESIKF_ERR_ARG, "vio_set_patches: bad argument");
  if (int rc = need(ctx, "vio_set_patches", IN_CAMERA)) return rc;
  CK(cudaSetDevice(ctx->device));
  const int L = ctx->vio_cfg.patch_pyrimid_level;
  if (int rc = install_submap(ctx, n, L)) return rc;
  cudaStream_t st = ctx->stream;
  if (n) {
    CK(cudaMemcpyAsync(ctx->vis_pos.p, pos, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->warp_patch.p, warp_patch, (size_t)n * 64 * L * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->search_levels.p, search_levels, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->inv_expo.p, inv_expo_list, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  commit_submap(ctx, n, L);
  return ESIKF_OK;
}

static void vio_fill_args(esikf_ctx *ctx, VioKernelArgs &ka, double *state_ptr) {
  memset(&ka, 0, sizeof(ka));
  ka.img = ctx->img.p;
  cam_dev(ctx, ka.cam);
  ka.pos = ctx->vis_pos.p, ka.warp_patch = ctx->warp_patch.p, ka.search_levels = ctx->search_levels.p, ka.inv_expo_list = ctx->inv_expo.p;
  shard_of(ctx->n_patches, ctx->rank, ctx->nranks, ka.begin, ka.count);
  ka.levels = ctx->vio_cfg.patch_pyrimid_level;
  ka.exposure_en = ctx->vio_cfg.exposure_estimate_en;
  ka.state = state_ptr;
  vio_consts(ctx, ka.Rci, ka.Pci, ka.Jdp_dR);
  ka.errors = ctx->errors.p, ka.partials = ctx->partials.p, ka.info = ctx->info.p, ka.ctrl = ctx->ctrl;
  ka.partial_stride = ctx->partial_blocks;
}
static int vio_grid(const esikf_ctx *ctx, int count) {
  int g = (count + VIO_WARPS - 1) / VIO_WARPS;  // one patch per warp while the patches last
  if (g > ctx->partial_blocks) g = ctx->partial_blocks;
  return g < 1 ? 1 : g;
}

// Tiled tensor maps of the level-0 u8 image, one per tap stride 1 << l (see VioTma). Encoded through the driver entry
// point (no link-time dependency on libcuda). Images whose row pitch is not a multiple of 16 bytes cannot be described:
// the variant then stays on the per-lane loads (enabled = 0).
static int vio_encode_tma(esikf_ctx *ctx) {
  if (ctx->tma_img == ctx->img.p && ctx->tma_w == ctx->img_w && ctx->tma_h == ctx->img_h) return ESIKF_OK;
  memset(&ctx->tma, 0, sizeof(ctx->tma));
  ctx->tma_img = ctx->img.p, ctx->tma_w = ctx->img_w, ctx->tma_h = ctx->img_h;
  if (ctx->img_w % 16 != 0 || ((uintptr_t)ctx->img.p & 15)) return ESIKF_OK;
  typedef CUresult (*encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  void *fn = nullptr;
  cudaDriverEntryPointQueryResult qr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || qr != cudaDriverEntryPointSuccess || !fn)
    return fail(ctx, ESIKF_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
  static_assert(sizeof(CUtensorMap) == 128, "descriptor size");
  for (int l = 0; l <= VIO_TMA_MAXLVL; l++) {
    const cuuint64_t dims[2] = {(cuuint64_t)ctx->img_w, (cuuint64_t)ctx->img_h};
    const cuuint64_t strides[1] = {(cuuint64_t)ctx->img_w};  // bytes between rows
    const cuuint32_t box[2] = {VIO_TMA_INNER(l), 11u << l};
    const cuuint32_t estr[2] = {1u, 1u << l};
    CUresult r = ((encode_fn)fn)(reinterpret_cast<CUtensorMap *>(ctx->tma.map[l]), CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void *)ctx->img.p, dims, strides, box, estr,
                                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(ctx, ESIKF_ERR_CUDA, "cuTensorMapEncodeTiled (tap stride %d) failed: %d", 1 << l, (int)r);
  }
  ctx->tma.enabled = 1;
  return ESIKF_OK;
}

int esikf_vio_run(esikf_ctx *ctx, const double *state_in, const double *state_prop) {
  if (!ctx || !state_in || !state_prop) return fail(ctx, ESIKF_ERR_ARG, "vio_run: null argument");
  const bool inverse = ctx->vio_cfg.inverse_composition_en != 0;
  if (int rc = need(ctx, "vio_run", IN_CAMERA | IN_EXT | IN_IMAGE | (ctx->n_patches > 0 ? IN_SUBMAP | (inverse ? IN_INV_REFS : 0) : 0))) return rc;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  if (int rc = upload_states(ctx, state_in, state_prop)) return rc;
  const bool fused_vio = ctx->n_patches > 0 && persistent_update(ctx, ctx->coop_vio);
  if (!fused_vio) {
    CK(cudaMemsetAsync(ctx->ctrl, 0, sizeof(Ctrl), st));
    CK(cudaMemsetAsync(ctx->vio_stats, 0, sizeof(esikf_vio_stats), st));
  }
  if (ctx->n_patches == 0) return ctx->resident = esikf_ctx::RESIDENT_VIO, ESIKF_OK;  // total_points == 0: early return (vio.cpp:786)
  VioKernelArgs ka;
  vio_fill_args(ctx, ka, ctx->state);
  SolveArgs sa = solve_args(ctx, ctx->state, ctx->vio_cfg.max_iterations);
  sa.vio_stats = ctx->vio_stats, sa.old_state = ctx->old_state.p, sa.G = ctx->G.p, sa.img_point_cov = ctx->vio_cfg.img_point_cov;
  const int grid = vio_grid(ctx, ka.count);
  VioInvArgs iv;
  memset(&iv, 0, sizeof(iv));
  if (inverse) {
    CK(ctx->H_sub_inv.reserve((size_t)ka.count * 64 * 6 + 8));
    iv.ref_imgs = ctx->ref_img_ptrs.p, iv.ref_idx = ctx->inv_ref_idx.p, iv.ref_px = ctx->inv_ref_px.p, iv.ref_f = ctx->inv_ref_f.p;
    iv.ref_R = ctx->inv_ref_R.p, iv.ref_pos = ctx->inv_ref_pos.p, iv.H_sub_inv = ctx->H_sub_inv.p;
    iv.ref_w = ctx->ref_w, iv.ref_h = ctx->ref_h, iv.fx = ctx->cam.fx, iv.fy = ctx->cam.fy;
  }
  if (fused_vio) {
    VioTma tma_off;
    tma_off.enabled = 0;
    VioTma *tma = &tma_off;
    if (ctx->tuning & ESIKF_TUNE_VIO_TMA) {
      int rc = vio_encode_tma(ctx);
      if (rc) return rc;
      tma = &ctx->tma;
    }
    const void *fn = inverse ? (const void *)vio_update_kernel<false, true> : (const void *)vio_update_kernel<false, false>;
    const void *fn_peer = inverse ? (const void *)vio_update_kernel<true, true> : (const void *)vio_update_kernel<true, false>;
    static_assert(VIO_CHAIN_CTA + VIO_CHAIN_MAX_CTAS * 64 == ESIKF_VIO_CHAIN_STAMP_WORDS, "VIO chain stamp layout");
    if (ctx->want_stamps) {
      ka.chain = ctx->stamps.p + 800;
      CK(cudaMemsetAsync(ka.chain, 0, ESIKF_VIO_CHAIN_STAMP_WORDS * sizeof(unsigned long long), ctx->stream));
    }
    return launch_persistent(ctx, fn, fn_peer, "vio_update_kernel", grid, VIO_THREADS, VIO_PERSIST_SMEM, &ka, sa, 64, 512, ctx->vio_timed, {&iv, tma}, esikf_ctx::RESIDENT_VIO);
  }
  ctx->vio_timed = ctx->timing;
  ctx->vio_slots = ctx->vio_cfg.patch_pyrimid_level * ctx->vio_cfg.max_iterations;
  int slot = 0;
  for (int level = ctx->vio_cfg.patch_pyrimid_level - 1; level >= 0; level--) {
    if (inverse)  // has_ref_patch_cache = false at every level (vio.cpp:794): H_sub_inv of this level's tap stride
      CK(launch(ctx, vio_inverse_precompute_kernel, (ka.count + 7) / 8, 256, 0, ka, iv, level));
    for (int it = 0; it < ctx->vio_cfg.max_iterations; it++, slot++) {
      ka.level = level, ka.slot_iter = it;
      cudaEvent_t *e = ctx->timing ? timing_events(ctx, EV_VIO_BASE, slot) : nullptr;
      if (e) CK(cudaEventRecord(e[0], st));
      if (inverse)
        CK(launch(ctx, vio_inverse_patch_kernel, grid, VIO_THREADS, sizeof(VioSmem), ka, iv));
      else
        CK(launch(ctx, vio_patch_kernel, grid, VIO_THREADS, sizeof(VioSmem), ka));
      if (e) CK(cudaEventRecord(e[1], st));
      int rc = allreduce_info(ctx);
      if (rc) return rc;
      sa.level = level, sa.slot_iter = it, sa.last_slot = (level == 0 && it == ctx->vio_cfg.max_iterations - 1);
      CK(launch(ctx, vio_solve_kernel, 1, SOLVE_THREADS, 0, sa));
      if (e) CK(cudaEventRecord(e[2], st));
    }
  }
  ctx->resident = esikf_ctx::RESIDENT_VIO;
  return ESIKF_OK;
}

int esikf_vio_fetch(esikf_ctx *ctx, double *state_out, esikf_vio_stats *stats, float *errors) {
  if (!ctx) return ESIKF_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  if (state_out) CK(cudaMemcpyAsync(state_out, ctx->state, S_N * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (stats) CK(cudaMemcpyAsync(stats, ctx->vio_stats, sizeof(esikf_vio_stats), cudaMemcpyDeviceToHost, st));
  if (errors && ctx->n_patches) CK(cudaMemcpyAsync(errors, ctx->errors.p, (size_t)ctx->n_patches * sizeof(float), cudaMemcpyDeviceToHost, st));
  return finish_fetch(ctx);
}

int esikf_vio_update(esikf_ctx *ctx, const uint8_t *img, int32_t width, int32_t height, const double *pos, const float *warp_patch,
                     const int32_t *search_levels, const double *inv_expo_list, int32_t n, const double *state_in, const double *state_prop,
                     double *state_out, esikf_vio_stats *stats, float *errors) {
  int rc = esikf_vio_set_image(ctx, img, width, height);
  if (rc) return rc;
  rc = esikf_vio_set_patches(ctx, pos, warp_patch, search_levels, inv_expo_list, n);
  if (rc) return rc;
  rc = esikf_vio_run(ctx, state_in, state_prop);
  if (rc) return rc;
  return esikf_vio_fetch(ctx, state_out, stats, errors);
}

// ---------------------------------------------------------------------------------------------------------------- patch producers
int esikf_vio_get_image_patch(esikf_ctx *ctx, const double *pc, int32_t n, int32_t level, float *patch_out) {
  if (!ctx || n < 0 || level < 0 || level > 12 || (n > 0 && (!pc || !patch_out))) return fail(ctx, ESIKF_ERR_ARG, "get_image_patch: bad argument");
  if (int rc = need(ctx, "get_image_patch", IN_IMAGE)) return rc;
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  const size_t N = (size_t)n;
  double *pc_d;
  float *patch;
  auto lay = [&](CallLayout &s) { pc_d = s.take<double>(N * 2), s.end_inputs(), s.begin_answers(), patch = s.take<float>(N * 64); };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{pc_d, pc, N * 2 * sizeof(double)}}));
  CK(launch(ctx, image_patch_kernel, (n * 64 + 255) / 256, 256, 0, ctx->img.p, ctx->img_w, ctx->img_h, pc_d, n, level, patch));
  CK(read_back_to(ctx, patch, patch_out, N * 64));
  return ESIKF_OK;
}

int esikf_vio_set_ref_images(esikf_ctx *ctx, const uint8_t *const *imgs, int32_t n_imgs, int32_t width, int32_t height) {
  if (!ctx || n_imgs < 0 || width <= 0 || height <= 0 || (n_imgs > 0 && !imgs)) return fail(ctx, ESIKF_ERR_ARG, "set_ref_images: bad argument");
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->ref_imgs.clear();
  void_inputs(ctx, IN_INV_REFS);  // their indices pointed into the images just released
  std::vector<const uint8_t *> ptrs;
  for (int i = 0; i < n_imgs; i++) {
    DevBuf<uint8_t> d;
    CK(cudaMalloc(&d.p, (size_t)width * height + 64));  // exact size: the images are replaced as a whole, never grown
    d.cap = (size_t)width * height + 64;
    ptrs.push_back(d.p);
    ctx->ref_imgs.push_back(std::move(d));
    CK(cudaMemcpyAsync(ctx->ref_imgs.back().p, imgs[i], (size_t)width * height, cudaMemcpyHostToDevice, ctx->stream));
  }
  CK(ctx->ref_img_ptrs.reserve(n_imgs + 1));
  if (n_imgs) CK(cudaMemcpyAsync(ctx->ref_img_ptrs.p, ptrs.data(), n_imgs * sizeof(uint8_t *), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->ref_w = width, ctx->ref_h = height;
  return ESIKF_OK;
}

int esikf_vio_warp_patches(esikf_ctx *ctx, int32_t n, const int32_t *ref_img_index, const double *px_ref, const double *pos_w, const double *normal_w,
                           const double *T_ref_w, const double *T_cur_w, double *A_cur_ref_out, int32_t *search_level_out, float *warp_patch_out,
                           int32_t keep_on_device) {
  if (!ctx || n < 0 || (n > 0 && (!ref_img_index || !px_ref || !pos_w || !normal_w || !T_ref_w || !T_cur_w)))
    return fail(ctx, ESIKF_ERR_ARG, "warp_patches: bad argument");
  if (int rc = need(ctx, "warp_patches", IN_CAMERA | IN_REF_IMAGES)) return rc;
  for (int i = 0; i < n; i++)
    if (int rc = check_ref_image(ctx, "warp_patches", ref_img_index[i])) return rc;
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  const int L = ctx->vio_cfg.patch_pyrimid_level;
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)n;
  int32_t *ref_idx, *levels;
  double *px, *pos, *normal, *T_ref, *T_cur, *ones = nullptr, *A;
  float *warp;
  auto lay = [&](CallLayout &s) {
    if (keep_on_device) ones = s.take<double>(N);  // the installed sub-map's inv_expo
    ref_idx = s.take<int32_t>(N), px = s.take<double>(2 * N), pos = s.take<double>(3 * N), normal = s.take<double>(3 * N);
    T_ref = s.take<double>(12 * N), T_cur = s.take<double>(12), s.end_inputs(), s.begin_answers();
    A = s.take<double>(4 * N), levels = s.take<int32_t>(N), warp = s.take<float>(N * 64 * L);
  };
  CK(lay_out_scratch(ctx, lay));
  if (keep_on_device) {
    if (int rc = install_submap(ctx, n, L)) return rc;
  } else {  // the sub-map's search levels and patches are the warp's work arrays
    CK(ctx->search_levels.reserve(n + 1));
    CK(ctx->warp_patch.reserve(N * 64 * L + 64));
  }
  const std::vector<double> one(keep_on_device ? N : 0, 1.0);
  CK(upload(ctx, {{ones, one.data(), one.size() * sizeof(double)}, {ref_idx, ref_img_index, N * sizeof(int32_t)}, {px, px_ref, N * 2 * sizeof(double)},
                  {pos, pos_w, N * 3 * sizeof(double)}, {normal, normal_w, N * 3 * sizeof(double)}, {T_ref, T_ref_w, N * 12 * sizeof(double)},
                  {T_cur, T_cur_w, 12 * sizeof(double)}}));
  CamDev cam;
  cam_dev(ctx, cam);
  CK(launch(ctx, warp_matrix_kernel, (n + 127) / 128, 128, 0, cam, n, px, pos, normal, T_ref, T_cur, A, ctx->search_levels.p));
  CK(cudaMemsetAsync(ctx->warp_patch.p, 0, N * 64 * L * sizeof(float), st));
  CK(launch(ctx, warp_affine_kernel, (n * L * 64 + 255) / 256, 256, 0, ctx->ref_img_ptrs.p, ref_idx, ctx->ref_w, ctx->ref_h, n, L, A, px, ctx->search_levels.p,
            ctx->warp_patch.p));
  if (search_level_out) CK(cudaMemcpyAsync(levels, ctx->search_levels.p, N * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  if (warp_patch_out) CK(cudaMemcpyAsync(warp, ctx->warp_patch.p, N * 64 * L * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (keep_on_device) {
    // install as the visual sub-map of the coming update: pos = pos_w, inv_expo filled by the caller through set_patches otherwise
    CK(cudaMemcpyAsync(ctx->vis_pos.p, pos, N * 3 * sizeof(double), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(ctx->inv_expo.p, ones, N * sizeof(double), cudaMemcpyDeviceToDevice, st));
  }
  CK(read_back(ctx, A, warp_patch_out ? (const void *)(warp + N * 64 * L) : search_level_out ? (const void *)(levels + N) : (const void *)(A + 4 * N)));
  if (keep_on_device) commit_submap(ctx, n, L);
  if (A_cur_ref_out) copy_out(ctx, A_cur_ref_out, A, A, N * 4 * sizeof(double));
  if (search_level_out) copy_out(ctx, search_level_out, A, levels, N * sizeof(int32_t));
  if (warp_patch_out) copy_out(ctx, warp_patch_out, A, warp, N * 64 * L * sizeof(float));
  return ESIKF_OK;
}

int esikf_vio_select_patches(esikf_ctx *ctx, int32_t n, const int32_t *ref_img_index, const double *px_ref, const int32_t *ref_level,
                             const double *ref_f, const double *ref_pos, const double *pos_w, const double *normal_w,
                             const double *T_ref_w, const double *ref_inv_expo, const int32_t *ref_key, const double *pc,
                             const double *T_cur_w, double inv_expo_time, const esikf_vio_select_cfg *cfg, int32_t *n_kept, int32_t *kept_index,
                             float *error_out, int32_t *search_level_out, double *A_cur_ref_out, float *warp_patch_out) {
  if (!ctx || n < 0 || !cfg || !n_kept) return fail(ctx, ESIKF_ERR_ARG, "select_patches: bad argument");
  const bool homography = cfg->normal_en != 0;
  if (n > 0 && (!ref_img_index || !px_ref || !pos_w || !T_ref_w || !ref_inv_expo || !pc || !T_cur_w || !kept_index ||
                (homography ? !normal_w : (!ref_f || !ref_pos || !ref_level || !ref_key))))
    return fail(ctx, ESIKF_ERR_ARG, "select_patches: null argument");
  if (int rc = need(ctx, "select_patches", IN_CAMERA | IN_IMAGE | (n > 0 ? IN_REF_IMAGES : 0))) return rc;
  for (int i = 0; i < n; i++) {
    if (int rc = check_ref_image(ctx, "select_patches", ref_img_index[i])) return rc;
    if (!homography && (ref_level[i] < 0 || ref_level[i] > 8)) return fail(ctx, ESIKF_ERR_ARG, "select_patches: ref level %d", ref_level[i]);
  }
  CK(cudaSetDevice(ctx->device));
  const int L = ctx->vio_cfg.patch_pyrimid_level;
  cudaStream_t st = ctx->stream;
  // every argument check is above: from here on the call replaces the installed sub-map
  if (int rc = install_submap(ctx, n, L)) return rc;
  *n_kept = 0;
  if (n == 0) return commit_submap(ctx, 0, L), ESIKF_OK;
  const size_t N = (size_t)n;
  double *d_px, *d_f, *d_rp, *d_pos, *d_nrm, *d_T, *d_ie, *d_pc, *d_Tc, *d_A, *d_Akept;
  int32_t *d_idx, *d_lvl, *d_key, *d_sl, *d_keep, *d_dst, *d_nk, *d_kept, *d_sl_out;
  float *d_warp, *d_err, *d_err_out, *d_warp_out;
  auto lay = [&](CallLayout &s) {
    d_px = s.take<double>(2 * N), d_f = s.take<double>(3 * N), d_rp = s.take<double>(3 * N), d_pos = s.take<double>(3 * N), d_nrm = s.take<double>(3 * N);
    d_T = s.take<double>(12 * N), d_ie = s.take<double>(N), d_pc = s.take<double>(2 * N), d_Tc = s.take<double>(12);
    d_idx = s.take<int32_t>(N), d_lvl = s.take<int32_t>(N), d_key = s.take<int32_t>(N);
    s.end_inputs();
    d_sl = s.take<int32_t>(N), d_keep = s.take<int32_t>(N), d_dst = s.take<int32_t>(N);
    d_A = s.take<double>(4 * N), d_warp = s.take<float>(N * 64 * L), d_err = s.take<float>(N);
    s.begin_answers();  // the count, then the kept candidates' rows (those of the installed sub-map copied here)
    d_nk = s.take<int32_t>(1), d_kept = s.take<int32_t>(N), d_Akept = s.take<double>(4 * N), d_err_out = s.take<float>(N), d_sl_out = s.take<int32_t>(N);
    d_warp_out = s.take<float>(N * 64 * L);
  };
  CK(lay_out_scratch(ctx, lay));
  // the inputs the chosen warp form does not read stay zero
  CK(upload(ctx, {{d_px, px_ref, 2 * N * sizeof(double)}, {d_f, ref_f, 3 * N * sizeof(double)}, {d_rp, ref_pos, 3 * N * sizeof(double)},
                  {d_pos, pos_w, 3 * N * sizeof(double)}, {d_nrm, normal_w, 3 * N * sizeof(double)}, {d_T, T_ref_w, 12 * N * sizeof(double)},
                  {d_ie, ref_inv_expo, N * sizeof(double)}, {d_pc, pc, 2 * N * sizeof(double)}, {d_Tc, T_cur_w, 12 * sizeof(double)},
                  {d_idx, ref_img_index, N * sizeof(int32_t)}, {d_lvl, homography ? nullptr : ref_level, N * sizeof(int32_t)},
                  {d_key, homography ? nullptr : ref_key, N * sizeof(int32_t)}}));
  CamDev cam;
  cam_dev(ctx, cam);
  if (homography)
    CK(launch(ctx, warp_matrix_kernel, (n + 127) / 128, 128, 0, cam, n, d_px, d_pos, d_nrm, d_T, d_Tc, d_A, d_sl));
  else
    CK(launch(ctx, warp_matrix_depth_kernel, (n + 127) / 128, 128, 0, cam, n, d_px, d_f, d_rp, d_pos, d_T, d_Tc, d_lvl, d_key, d_A, d_sl));
  // patch_wrap is a fresh zero vector per candidate (:646): a NaN inverse leaves it zero (:297-301)
  CK(cudaMemsetAsync(d_warp, 0, N * 64 * L * sizeof(float), st));
  CK(launch(ctx, warp_affine_kernel, (n * L * 64 + 255) / 256, 256, 0, ctx->ref_img_ptrs.p, d_idx, ctx->ref_w, ctx->ref_h, n, L, d_A, d_px, d_sl, d_warp));
  SelectGateArgs ga;
  ga.img = ctx->img.p, ga.width = ctx->img_w, ga.height = ctx->img_h, ga.n = n, ga.levels = L, ga.ncc_en = cfg->ncc_en != 0;
  ga.pc = d_pc, ga.warp = d_warp, ga.ref_inv_expo = d_ie;
  ga.cur_inv_expo = inv_expo_time, ga.ncc_thre = cfg->ncc_thre, ga.outlier_threshold = cfg->outlier_threshold;
  ga.error = d_err, ga.keep = d_keep;
  CK(launch(ctx, select_gate_kernel, (n + SELECT_GATE_WARPS - 1) / SELECT_GATE_WARPS, 32 * SELECT_GATE_WARPS, 0, ga));
  CK(launch(ctx, select_scan_kernel, 1, SELECT_SCAN_THREADS, 0, d_keep, n, d_dst, d_nk));
  SelectScatterArgs sa;
  sa.n = n, sa.levels = L, sa.keep = d_keep, sa.dst = d_dst, sa.search_level = d_sl, sa.pos_w = d_pos, sa.ref_inv_expo = d_ie, sa.A = d_A;
  sa.warp = d_warp, sa.error = d_err;
  sa.vis_pos = ctx->vis_pos.p, sa.inv_expo = ctx->inv_expo.p, sa.A_kept = d_Akept, sa.warp_patch = ctx->warp_patch.p, sa.errors = ctx->errors.p;
  sa.search_levels = ctx->search_levels.p, sa.kept_index = d_kept;
  CK(launch(ctx, select_scatter_kernel, (n + 7) / 8, 256, 0, sa));
  int32_t nk;
  CK(read_back_to(ctx, d_nk, &nk));
  commit_submap(ctx, nk, L);
  *n_kept = nk;
  if (nk > 0) {
    const size_t K = (size_t)nk;
    if (error_out) CK(cudaMemcpyAsync(d_err_out, ctx->errors.p, K * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (search_level_out) CK(cudaMemcpyAsync(d_sl_out, ctx->search_levels.p, K * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    if (warp_patch_out) CK(cudaMemcpyAsync(d_warp_out, ctx->warp_patch.p, K * 64 * L * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CK(read_back(ctx, d_kept, warp_patch_out ? (const void *)(d_warp_out + K * 64 * L) : (const void *)(d_sl_out + K)));
    copy_out(ctx, kept_index, d_kept, d_kept, K * sizeof(int32_t));
    if (error_out) copy_out(ctx, error_out, d_kept, d_err_out, K * sizeof(float));
    if (search_level_out) copy_out(ctx, search_level_out, d_kept, d_sl_out, K * sizeof(int32_t));
    if (A_cur_ref_out) copy_out(ctx, A_cur_ref_out, d_kept, d_Akept, K * 4 * sizeof(double));
    if (warp_patch_out) copy_out(ctx, warp_patch_out, d_kept, d_warp_out, K * 64 * L * sizeof(float));
  }
  return ESIKF_OK;
}

int esikf_vio_set_inverse_refs(esikf_ctx *ctx, int32_t n, const int32_t *ref_img_index, const double *ref_px, const double *ref_f, const double *ref_R,
                               const double *ref_pos) {
  if (!ctx || n < 0 || (n > 0 && (!ref_img_index || !ref_px || !ref_f || !ref_R || !ref_pos))) return fail(ctx, ESIKF_ERR_ARG, "set_inverse_refs: bad argument");
  if (int rc = need(ctx, "set_inverse_refs", n > 0 ? IN_REF_IMAGES : 0)) return rc;
  for (int i = 0; i < n; i++)
    if (int rc = check_ref_image(ctx, "set_inverse_refs", ref_img_index[i])) return rc;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  CK(ctx->inv_ref_idx.reserve(n + 1));
  CK(ctx->inv_ref_px.reserve((size_t)n * 2 + 2));
  CK(ctx->inv_ref_f.reserve((size_t)n * 3 + 3));
  CK(ctx->inv_ref_R.reserve((size_t)n * 9 + 9));
  CK(ctx->inv_ref_pos.reserve((size_t)n * 3 + 3));
  if (n > 0) {
    CK(cudaMemcpyAsync(ctx->inv_ref_idx.p, ref_img_index, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->inv_ref_px.p, ref_px, (size_t)n * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->inv_ref_f.p, ref_f, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->inv_ref_R.p, ref_R, (size_t)n * 9 * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->inv_ref_pos.p, ref_pos, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));  // the caller's arrays may go away
  }
  ctx->n_inv_refs = n;
  return ESIKF_OK;
}

int esikf_vio_warp_affine(esikf_ctx *ctx, int32_t n, const int32_t *ref_img_index, const double *px_ref, const double *A_cur_ref,
                          const int32_t *search_level, float *warp_patch_out) {
  if (!ctx || n < 0 || (n > 0 && (!ref_img_index || !px_ref || !A_cur_ref || !search_level || !warp_patch_out)))
    return fail(ctx, ESIKF_ERR_ARG, "warp_affine: bad argument");
  if (int rc = need(ctx, "warp_affine", IN_CAMERA | IN_REF_IMAGES)) return rc;
  for (int i = 0; i < n; i++) {
    if (int rc = check_ref_image(ctx, "warp_affine", ref_img_index[i])) return rc;
    if (search_level[i] < 0 || search_level[i] > 8) return fail(ctx, ESIKF_ERR_ARG, "warp_affine: search level %d", search_level[i]);
  }
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  const int L = ctx->vio_cfg.patch_pyrimid_level;
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)n;
  // all in scratch: the patches / search levels installed by set_patches (or warp_patches with keep_on_device) stay untouched
  int32_t *ref_idx, *levels;
  double *px, *A;
  float *out;
  auto lay = [&](CallLayout &s) {
    ref_idx = s.take<int32_t>(N), px = s.take<double>(2 * N), A = s.take<double>(4 * N), levels = s.take<int32_t>(N + 1), s.end_inputs();
    s.begin_answers(), out = s.take<float>(N * 64 * L + 64);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{ref_idx, ref_img_index, N * sizeof(int32_t)}, {px, px_ref, N * 2 * sizeof(double)}, {A, A_cur_ref, N * 4 * sizeof(double)},
                  {levels, search_level, N * sizeof(int32_t)}}));
  CK(cudaMemsetAsync(out, 0, N * 64 * L * sizeof(float), st));
  CK(launch(ctx, warp_affine_kernel, (n * L * 64 + 255) / 256, 256, 0, ctx->ref_img_ptrs.p, ref_idx, ctx->ref_w, ctx->ref_h, n, L, A, px, levels, out));
  CK(read_back_to(ctx, out, warp_patch_out, N * 64 * L));
  return ESIKF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- measurement
int esikf_profile_kernel(esikf_ctx *ctx, int32_t which, int32_t arg, int32_t reps, int32_t flush_l2, float *avg_ms) {
  if (!ctx || !avg_ms || reps < 1) return fail(ctx, ESIKF_ERR_ARG, "profile_kernel: bad argument");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t flush_bytes = 256u << 20;
  if (flush_l2) CK(ctx->flush.reserve(flush_bytes));
  // work on a scratch copy of the resident state so the measured launches never disturb an update in flight
  CK(cudaMemcpyAsync(ctx->scratch_state.p, ctx->state, S_N * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CK(cudaMemsetAsync(ctx->ctrl, 0, sizeof(Ctrl), st));
  LioKernelArgs la;
  VioKernelArgs va;
  SolveArgs sa;
  memset(&sa, 0, sizeof(sa));
  int grid = 1;
  if (which == 0 || which == 1 || which == 3) {
    if (int rc = need(ctx, "profile_kernel: no resident LIO frame", IN_MAP | IN_RUN_SCAN)) return rc;
    if (ctx->n_pts == 0) return fail(ctx, ESIKF_ERR_STATE, "profile_kernel: no resident LIO frame (run lio once)");
    lio_fill_args(ctx, la, ctx->scratch_state.p);
    grid = lio_grid(ctx, la.count);
    sa = solve_args(ctx, ctx->scratch_state.p, 1 << 20);
  } else if (which == 2) {
    if (int rc = need(ctx, "profile_kernel: no resident VIO frame", IN_IMAGE | IN_SUBMAP)) return rc;
    if (ctx->n_patches == 0) return fail(ctx, ESIKF_ERR_STATE, "profile_kernel: no resident VIO frame (an empty sub-map)");
    if (arg < 0 || arg >= ctx->vio_cfg.patch_pyrimid_level) return fail(ctx, ESIKF_ERR_ARG, "profile_kernel: level %d outside [0, %d)", arg, ctx->vio_cfg.patch_pyrimid_level);
    vio_fill_args(ctx, va, ctx->scratch_state.p);
    va.level = arg, va.slot_iter = 0;
    grid = vio_grid(ctx, va.count);
  } else {
    return fail(ctx, ESIKF_ERR_ARG, "profile_kernel: which=%d", which);
  }
  struct Events {  // destroyed on every return
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    ~Events() {
      if (e0) cudaEventDestroy(e0);
      if (e1) cudaEventDestroy(e1);
    }
  } ev;
  cudaEvent_t &e0 = ev.e0, &e1 = ev.e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  double total = 0.0;
  for (int r = 0; r < reps + 3; r++) {  // 3 warm-up launches
    if (flush_l2) CK(cudaMemsetAsync(ctx->flush.p, r & 0xff, flush_bytes, st));
    if (which == 1) {
      CK(cudaMemcpyAsync(ctx->scratch_state.p, ctx->state, S_N * sizeof(double), cudaMemcpyDeviceToDevice, st));
      CK(cudaMemsetAsync(ctx->ctrl, 0, sizeof(Ctrl), st));
    }
    CK(cudaEventRecord(e0, st));
    if (which == 0) CK(launch_lio_residual(ctx, lio_use_l2_slots(la.count, grid), grid, la));
    else if (which == 1) CK(launch(ctx, lio_solve_kernel, 1, SOLVE_THREADS, 0, sa));
    else if (which == 2) CK(launch(ctx, vio_patch_kernel, grid, VIO_THREADS, sizeof(VioSmem), va));
    else CK(lio_precompute(ctx, (float)ctx->lio_cfg.dept_err, (float)ctx->lio_cfg.beam_err));
    CK(cudaEventRecord(e1, st));
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (r >= 3) total += ms;
  }
  *avg_ms = (float)(total / reps);
  return ESIKF_OK;
}

}  // extern "C"
