// The context: create / destroy, setters, multi-GPU, phase stamps and kernel timing, and the helpers every host file of the
// C ABI shares (esikf_api.cuh).
#include <stdarg.h>
#include <stdio.h>

#include "esikf_api.cuh"

NcclApi g_nccl;

int fail(esikf_ctx *c, int code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (c) c->err = buf;
  return code;
}

int need(esikf_ctx *ctx, const char *call, unsigned inputs) {
  const esikf_ctx &c = *ctx;
  const struct { unsigned in; bool ok; const char *missing; } rules[] = {
      {IN_EXT, c.have_ext, "no extrinsics (set_extrinsics)"},
      {IN_CAMERA, c.cam.width != 0, "no camera (vio_set_camera)"},
      {IN_IMAGE, c.img_w != 0, "no image of the camera's size (vio_set_image)"},
      {IN_SUBMAP, c.submap_levels == c.vio_cfg.patch_pyrimid_level, "no visual sub-map laid out for the camera's level count"},
      {IN_INV_REFS, c.n_inv_refs == c.n_patches && c.ref_w == c.cam.width && c.ref_h == c.cam.height, "no inverse refs for every patch, or reference images of another size"},
      {IN_REF_IMAGES, !c.ref_imgs.empty(), "no reference images (set_ref_images)"},
      {IN_SCAN, c.scan != esikf_ctx::SCAN_NONE, "no resident scan (esikf_lio_set_scan)"},
      {IN_RUN_SCAN, c.scan != esikf_ctx::SCAN_SET, "the resident scan has not been through esikf_lio_run yet"},
      {IN_MAP, c.map_kind == esikf_ctx::MAP_HOST || c.map_kind == esikf_ctx::MAP_DEVICE, "no live map (map_upload, esikf_map_device_init)"},
      {IN_HOST_MAP, c.map_kind == esikf_ctx::MAP_HOST, "no host-uploaded map (map_upload); a device-resident map refits itself"},
      {IN_DEVICE_MAP, c.map_kind >= esikf_ctx::MAP_DEVICE, "no device-resident map (esikf_map_device_init)"},
      {IN_EXPORT, c.map_export_points >= 0, "no build / update to export (the map was initialised or slid since, or the last one failed)"},
      {IN_PV_LIST, c.pv_n >= 0, "no esikf_map_device_update of the resident scan left its points on the device"},
      {IN_CLOUD, c.rgb_n >= 0, "no cloud (rgb_set_cloud)"},
      {IN_RETRIEVAL, c.ret_w != 0, "no esikf_vio_retrieve_scan since the last vio_set_camera"},
      {IN_STORE, c.vmap_cap != 0, "no observation store (esikf_vmap_init)"},
  };
  for (const auto &r : rules)
    if ((inputs & r.in) && !r.ok) return fail(ctx, ESIKF_ERR_STATE, "%s: %s", call, r.missing);
  return ESIKF_OK;
}

void void_inputs(esikf_ctx *ctx, unsigned inputs) {
  if (inputs & IN_IMAGE) ctx->img_w = ctx->img_h = 0;
  if (inputs & IN_SUBMAP) ctx->submap_levels = 0;
  if (inputs & (IN_SUBMAP | IN_INV_REFS)) ctx->n_inv_refs = 0;
  if (inputs & IN_MAP) ctx->map_kind = esikf_ctx::MAP_DEVICE_VOID;
  if (inputs & IN_EXPORT) ctx->map_export_points = -1;
  if (inputs & IN_PV_LIST) ctx->pv_n = -1;
  if (inputs & IN_NORMALS) ctx->normals_n = -1;
  if (inputs & IN_CLOUD) ctx->rgb_n = -1;
  if (inputs & IN_RETRIEVAL) ctx->ret_w = ctx->ret_h = 0;
  if (inputs & IN_POSTERIOR) ctx->resident = esikf_ctx::RESIDENT_NONE;
}

cudaError_t upload(esikf_ctx *ctx, std::initializer_list<HostIn> in) {
  size_t bytes = 0;
  for (const HostIn &h : in) {
    if (!h.bytes) continue;
    const size_t at = (const uint8_t *)h.dst - ctx->scratch.p;
    bytes = std::max(bytes, at + h.bytes);
    if (bytes > ctx->host.cap) return cudaErrorInvalidValue;  // the layout did not mark its inputs
    if (h.src) memcpy(ctx->host.p + at, h.src, h.bytes);
    else memset(ctx->host.p + at, 0, h.bytes);
  }
  return cudaMemcpyAsync(ctx->scratch.p, ctx->host.p, bytes, cudaMemcpyHostToDevice, ctx->stream);
}

cudaError_t read_back(esikf_ctx *ctx, const void *first, const void *end) {
  const size_t bytes = (const uint8_t *)end - (const uint8_t *)first;
  if (bytes > ctx->host.cap) return cudaErrorInvalidValue;  // the layout did not mark these answers
  const cudaError_t e = cudaMemcpyAsync(ctx->host.p, first, bytes, cudaMemcpyDeviceToHost, ctx->stream);
  return e == cudaSuccess ? cudaStreamSynchronize(ctx->stream) : e;
}
void copy_out(const esikf_ctx *ctx, void *dst, const void *first, const void *src, size_t bytes) {
  memcpy(dst, ctx->host.p + ((const uint8_t *)src - (const uint8_t *)first), bytes);
}

void shard_of(int n, int rank, int nranks, int &begin, int &count) {
  // contiguous blocks, remainder spread over the first ranks
  int base = n / nranks, rem = n % nranks;
  begin = rank * base + (rank < rem ? rank : rem);
  count = base + (rank < rem ? 1 : 0);
}

void vio_consts(const esikf_ctx *ctx, double Rci[9], double Pci[3], double Jdp_dR[9]) {
  // vio.cpp:29-33, 57-65: Rli = extR^T, Pli = -extR^T extT, Rci = Rcl Rli, Pci = Rcl Pli + Pcl, Pic = -Rci^T Pci, Jdp_dR = -Rci [Pic]x
  const esikf_extrinsics &e = ctx->ext;
  double Rli[9], Pli[3];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) Rli[3 * r + c] = e.extR[3 * c + r];
  for (int r = 0; r < 3; r++) Pli[r] = -(Rli[3 * r] * e.extT[0] + Rli[3 * r + 1] * e.extT[1] + Rli[3 * r + 2] * e.extT[2]);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) Rci[3 * r + c] = e.Rcl[3 * r] * Rli[c] + e.Rcl[3 * r + 1] * Rli[3 + c] + e.Rcl[3 * r + 2] * Rli[6 + c];
  for (int r = 0; r < 3; r++) Pci[r] = e.Rcl[3 * r] * Pli[0] + e.Rcl[3 * r + 1] * Pli[1] + e.Rcl[3 * r + 2] * Pli[2] + e.Pcl[r];
  double Pic[3];
  for (int r = 0; r < 3; r++) Pic[r] = -(Rci[r] * Pci[0] + Rci[3 + r] * Pci[1] + Rci[6 + r] * Pci[2]);
  const double tmp[9] = {0.0, -Pic[2], Pic[1], Pic[2], 0.0, -Pic[0], -Pic[1], Pic[0], 0.0};
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) Jdp_dR[3 * r + c] = -(Rci[3 * r] * tmp[c] + Rci[3 * r + 1] * tmp[3 + c] + Rci[3 * r + 2] * tmp[6 + c]);
}
void cam_dev(const esikf_ctx *ctx, CamDev &c) {
  c.model = ctx->cam.model, c.width = ctx->cam.width, c.height = ctx->cam.height;
  c.fx = ctx->cam.fx, c.fy = ctx->cam.fy, c.cx = ctx->cam.cx, c.cy = ctx->cam.cy;
  for (int i = 0; i < 5; i++) c.d[i] = ctx->cam.d[i];
}
void frame_consts(const esikf_ctx *ctx, CamDev &cam, double Rci[9], double Pci[3]) {
  cam_dev(ctx, cam);
  double Jdp_dR[9];
  vio_consts(ctx, Rci, Pci, Jdp_dR);
}

int state_or_posterior(esikf_ctx *ctx, const double *state, esikf_ctx::Resident want, const char *what, const double **out) {
  if (!state && ctx->resident != want)
    return fail(ctx, ESIKF_ERR_STATE, "%s(state = NULL): the device holds no %s posterior", what, want == esikf_ctx::RESIDENT_LIO ? "LIO" : "VIO");
  if (!state) return *out = ctx->state, ESIKF_OK;
  CK(ctx->scratch_state.reserve(S_N));
  CK(cudaMemcpyAsync(ctx->scratch_state.p, state, S_N * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  *out = ctx->scratch_state.p;
  return ESIKF_OK;
}

extern "C" {

int esikf_create(esikf_ctx **out, int device) {
  if (!out) return ESIKF_ERR_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return ESIKF_ERR_NO_DEVICE;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return ESIKF_ERR_NO_DEVICE;
  if (prop.major != 9) return ESIKF_ERR_NO_DEVICE;  // sm_90a binary only
  esikf_ctx *ctx = new esikf_ctx;
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete ctx;
    return ESIKF_ERR_CUDA;
  }
  bool ok = ctx->state_prop.reserve(2 * S_N) == cudaSuccess && ctx->info.reserve(NE_MAX) == cudaSuccess &&
            cudaMallocHost(&ctx->stage, (size_t)esikf_ctx::STAGE_SLOTS * 2 * S_N * sizeof(double)) == cudaSuccess &&
            cudaMallocHost(&ctx->stage_ctrl, 256) == cudaSuccess &&
            ctx->old_state.reserve(32) == cudaSuccess && ctx->G.reserve(19 * 7) == cudaSuccess &&
            ctx->ctl_block.reserve(sizeof(esikf_lio_stats) + sizeof(Ctrl) + 64 + sizeof(esikf_vio_stats)) == cudaSuccess && ctx->ext_dev.reserve(12) == cudaSuccess &&
            ctx->scratch_state.reserve(S_N) == cudaSuccess;
  ctx->partial_blocks = ctx->sm_count < 160 ? ctx->sm_count : 160;  // persistent residual kernels: one CTA per SM
  ok = ok && ctx->partials.reserve((size_t)2 * ctx->partial_blocks * NE_MAX) == cudaSuccess && ctx->stamps.reserve(800 + ESIKF_VIO_CHAIN_STAMP_WORDS) == cudaSuccess &&
       ctx->barrier.reserve(128) == cudaSuccess;
  if (ok) cudaMemsetAsync(ctx->barrier.p, 0, 128 * sizeof(unsigned int), ctx->stream);
  if (ok) {
    ctx->state = ctx->state_prop.p, ctx->prop = ctx->state_prop.p + S_N;
    for (int i = 0; i < esikf_ctx::STAGE_SLOTS; i++) ok = ok && cudaEventCreateWithFlags(&ctx->stage_ev[i], cudaEventDisableTiming) == cudaSuccess;
  }
  if (ok) {
    unsigned char *b = ctx->ctl_block.p;
    ctx->lio_stats = reinterpret_cast<esikf_lio_stats *>(b);
    ctx->ctrl = reinterpret_cast<Ctrl *>(b + sizeof(esikf_lio_stats));
    ctx->vio_stats = reinterpret_cast<esikf_vio_stats *>(b + sizeof(esikf_lio_stats) + sizeof(Ctrl) + 64);
    cudaMemsetAsync(b, 0, ctx->ctl_block.cap, ctx->stream);
  }
  cudaDeviceGetAttribute(&ctx->coop_ok, cudaDevAttrCooperativeLaunch, device);
  if (!ok || update_kernels_setup(ctx) != cudaSuccess) {
    delete ctx;
    return ESIKF_ERR_CUDA;
  }
  cudaGetLastError();
  *out = ctx;
  return ESIKF_OK;
}

void esikf_destroy(esikf_ctx *ctx) { delete ctx; }

const char *esikf_last_error(const esikf_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }
void *esikf_stream(esikf_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }
int64_t esikf_launch_count(const esikf_ctx *ctx) { return ctx ? ctx->launches : 0; }

void *esikf_host_alloc(size_t bytes) {
  void *p = nullptr;
  if (bytes == 0 || cudaMallocHost(&p, bytes) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}
void esikf_host_free(void *p) {
  if (p) cudaFreeHost(p);
}

int esikf_synchronize(esikf_ctx *ctx) {
  if (!ctx) return ESIKF_ERR_ARG;
  CK(cudaStreamSynchronize(ctx->stream));
  return ESIKF_OK;
}
int esikf_set_solve_mode(esikf_ctx *ctx, int mode) {
  if (!ctx || mode < 0 || mode > 1) return ESIKF_ERR_ARG;
  ctx->solve_mode = mode;
  return ESIKF_OK;
}
int esikf_set_loop_mode(esikf_ctx *ctx, int mode) {
  if (!ctx || mode < 0 || mode > 2) return ESIKF_ERR_ARG;  // 1 and 2 both select the persistent kernels
  ctx->loop_mode = mode;
  return ESIKF_OK;
}
int esikf_set_tuning(esikf_ctx *ctx, uint32_t flags) {
  if (!ctx || (flags & ~(uint32_t)(ESIKF_TUNE_STAGE_LDG | ESIKF_TUNE_VIO_TMA))) return ESIKF_ERR_ARG;
  ctx->tuning = flags;
  return ESIKF_OK;
}
int esikf_set_extrinsics(esikf_ctx *ctx, const esikf_extrinsics *ext) {
  if (!ctx || !ext) return ESIKF_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  double h[12];
  memcpy(h, ext->extR, 9 * sizeof(double));
  memcpy(h + 9, ext->extT, 3 * sizeof(double));
  if (!ctx->have_ext || memcmp(h, ctx->ext_host, sizeof(h)) != 0) {  // unchanged (the shim sets it every tick): nothing to upload
    CK(cudaMemcpyAsync(ctx->ext_dev.p, h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));  // `h` is a stack buffer
    memcpy(ctx->ext_host, h, sizeof(h));
  }
  ctx->ext = *ext;
  ctx->have_ext = true;
  return ESIKF_OK;
}

int esikf_set_lidar_extrinsics(esikf_ctx *ctx, const double extR[9], const double extT[3]) {
  if (!ctx || !extR || !extT) return ESIKF_ERR_ARG;
  esikf_extrinsics e = ctx->ext;
  if (!ctx->have_ext) {
    memset(&e, 0, sizeof(e));
    e.Rcl[0] = e.Rcl[4] = e.Rcl[8] = 1.0;
  }
  memcpy(e.extR, extR, sizeof(e.extR));
  memcpy(e.extT, extT, sizeof(e.extT));
  return esikf_set_extrinsics(ctx, &e);
}

// ---------------------------------------------------------------------------------------------------------------- multi-GPU
int esikf_comm_unique_id(char out[128]) {
  if (!out) return ESIKF_ERR_ARG;
  if (!g_nccl.load()) return ESIKF_ERR_COMM;
  ncclUniqueId id;
  if (g_nccl.GetUniqueId(&id) != 0) return ESIKF_ERR_COMM;
  memcpy(out, id.internal, 128);
  return ESIKF_OK;
}
int esikf_comm_init(esikf_ctx *ctx, int32_t rank, int32_t nranks, const char unique_id[128]) {
  if (!ctx || nranks < 1 || rank < 0 || rank >= nranks || !unique_id) return fail(ctx, ESIKF_ERR_ARG, "comm_init: bad argument");
  if (nranks == 1) {
    ctx->rank = 0, ctx->nranks = 1;
    return ESIKF_OK;
  }
  if (!g_nccl.load()) return fail(ctx, ESIKF_ERR_COMM, "libnccl.so.2 not found");
  CK(cudaSetDevice(ctx->device));
  ncclUniqueId id;
  memcpy(id.internal, unique_id, 128);
  int r = g_nccl.CommInitRank(&ctx->comm, nranks, id, rank);
  if (r != 0) return fail(ctx, ESIKF_ERR_COMM, "ncclCommInitRank failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
  ctx->rank = rank, ctx->nranks = nranks;
  return ESIKF_OK;
}
int esikf_peer_export(esikf_ctx *ctx, char out[64]) {
  if (!ctx || !out) return ESIKF_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  if (!ctx->mailbox) {
    const size_t words = (size_t)2 * PEER_MAX_RANKS * PEER_SLOT_WORDS;
    CK(cudaMalloc(&ctx->mailbox, words * sizeof(unsigned long long)));
    CK(cudaMemset(ctx->mailbox, 0, words * sizeof(unsigned long long)));  // tag 0 is never sent
  }
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, ctx->mailbox));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(out, &h, 64);
  return ESIKF_OK;
}
int esikf_peer_attach(esikf_ctx *ctx, int32_t rank, int32_t nranks, const char *handles) {
  if (!ctx || !handles || nranks < 1 || nranks > PEER_MAX_RANKS || rank < 0 || rank >= nranks) return fail(ctx, ESIKF_ERR_ARG, "peer_attach: bad argument (1..8 ranks)");
  if (!ctx->mailbox) return fail(ctx, ESIKF_ERR_STATE, "peer_attach before peer_export");
  CK(cudaSetDevice(ctx->device));
  ctx->peer_ptrs.assign(nranks, nullptr);
  for (int r = 0; r < nranks; r++) {
    if (r == rank) {
      ctx->peer_ptrs[r] = ctx->mailbox;
      continue;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + 64 * (size_t)r, 64);
    void *p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return fail(ctx, ESIKF_ERR_COMM, "cudaIpcOpenMemHandle(rank %d) failed: %s", r, cudaGetErrorString(e));
    ctx->peer_ptrs[r] = (unsigned long long *)p;
  }
  CK(ctx->peer_ptrs_dev.reserve(nranks));
  CK(cudaMemcpy(ctx->peer_ptrs_dev.p, ctx->peer_ptrs.data(), nranks * sizeof(unsigned long long *), cudaMemcpyHostToDevice));
  // the peer mailbox was zeroed at export time (before the host-side all-gather): a peer may already be writing into it. The
  // exchange counter has to start equal on every rank, so it restarts from 0 when the peers first attach, after this
  // context's earlier updates; the grid mailbox restarts with it (a word left from before could carry a tag again).
  if (!ctx->p2p) {
    CK(cudaMemsetAsync(ctx->grid_mbox.p, 0, ctx->grid_mbox.cap * sizeof(unsigned long long), ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  ctx->rank = rank, ctx->nranks = nranks, ctx->p2p = true;
  return ESIKF_OK;
}
int esikf_shard_range(int32_t n, int32_t rank, int32_t nranks, int32_t *begin, int32_t *count) {
  if (n < 0 || nranks < 1 || rank < 0 || rank >= nranks || !begin || !count) return ESIKF_ERR_ARG;
  int b, c;
  shard_of(n, rank, nranks, b, c);
  *begin = b, *count = c;
  return ESIKF_OK;
}
int esikf_comm_rank(const esikf_ctx *ctx, int32_t *rank, int32_t *nranks) {
  if (!ctx) return ESIKF_ERR_ARG;
  if (rank) *rank = ctx->rank;
  if (nranks) *nranks = ctx->nranks;
  return ESIKF_OK;
}

int esikf_set_phase_stamps(esikf_ctx *ctx, int32_t enable) {
  if (!ctx) return ESIKF_ERR_ARG;
  ctx->want_stamps = enable != 0;
  return ESIKF_OK;
}
int esikf_get_phase_stamps(esikf_ctx *ctx, uint64_t *out /* 800 */) {
  if (!ctx || !out) return ESIKF_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaMemcpyAsync(out, ctx->stamps.p, 800 * sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return ESIKF_OK;
}

int esikf_get_vio_chain_stamps(esikf_ctx *ctx, uint64_t *out) {
  if (!ctx || !out) return ESIKF_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaMemcpyAsync(out, ctx->stamps.p + 800, ESIKF_VIO_CHAIN_STAMP_WORDS * sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return ESIKF_OK;
}

int esikf_set_kernel_timing(esikf_ctx *ctx, int32_t enable) {
  if (!ctx) return ESIKF_ERR_ARG;
  ctx->timing = enable != 0;
  return ESIKF_OK;
}

int esikf_get_kernel_timing(esikf_ctx *ctx, float *lio_residual_ms, float *lio_solve_ms, float *vio_patch_ms, float *vio_solve_ms) {
  if (!ctx) return ESIKF_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int pass = 0; pass < 2; pass++) {
    const bool timed = pass == 0 ? ctx->lio_timed : ctx->vio_timed;
    const int slots = pass == 0 ? ctx->lio_slots : ctx->vio_slots, base = pass == 0 ? EV_LIO_BASE : EV_VIO_BASE, cap = pass == 0 ? 8 : 64;
    float *a = pass == 0 ? lio_residual_ms : vio_patch_ms, *b = pass == 0 ? lio_solve_ms : vio_solve_ms;
    for (int i = 0; i < cap; i++) {
      if (a) a[i] = 0.f;
      if (b) b[i] = 0.f;
    }
    if (!timed) continue;
    for (int i = 0; i < slots && i < cap; i++) {
      cudaEvent_t *e = &ctx->ev[(size_t)(base + i) * 3];
      float ms = 0.f;
      if (a && cudaEventElapsedTime(&ms, e[0], e[1]) == cudaSuccess) a[i] = ms;
      if (b && cudaEventElapsedTime(&ms, e[1], e[2]) == cudaSuccess) b[i] = ms;
    }
  }
  return ESIKF_OK;
}

}  // extern "C"
