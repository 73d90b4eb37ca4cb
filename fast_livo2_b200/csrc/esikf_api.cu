// Host side of the C ABI declared in include/esikf_b200.h: context, device mirror of the voxel map, staging of the
// per-tick inputs, and the launch sequences of the LIO / VIO update loops. No CPU fallback: every entry point fails
// with a status code when the device or an input is missing.
#include <cuda.h>
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <initializer_list>
#include <string>
#include <utility>
#include <vector>

#include "esikf_dev.cuh"
#include "scratch_layout.hpp"

// single translation unit: the kernels are included so the whole library builds with one nvcc invocation
#include "esikf_lio.cu"
#include "esikf_solve.cu"
#include "esikf_vio.cu"
#include "esikf_fused.cu"
#include "esikf_map.cu"
#include "esikf_color.cu"
#include "esikf_generate.cu"
#include "esikf_observe.cu"
#include "esikf_retrieve.cu"
#include "esikf_find.cu"
#include "esikf_refpatch.cu"
#include "esikf_vmap.cu"
#include "esikf_vretrieve.cu"

using namespace esikf;

// ---------------------------------------------------------------------------------------------------------------------
// NCCL through dlopen: the library has no link-time dependency on NCCL; when the process already holds a libnccl.so.2
// (e.g. torch's bundled one) that copy is reused.
typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
struct NcclApi {
  void *handle = nullptr;
  int (*GetUniqueId)(ncclUniqueId *) = nullptr;
  int (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  int (*AllReduce)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  const char *(*GetErrorString)(int) = nullptr;
  bool load() {
    if (handle) return true;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *n : names) {
      handle = dlopen(n, RTLD_NOW | RTLD_NOLOAD);
      if (handle) break;
    }
    if (!handle)
      for (const char *n : names) {
        handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (handle) break;
      }
    if (!handle) return false;
    GetUniqueId = (int (*)(ncclUniqueId *))dlsym(handle, "ncclGetUniqueId");
    CommInitRank = (int (*)(ncclComm_t *, int, ncclUniqueId, int))dlsym(handle, "ncclCommInitRank");
    AllReduce = (int (*)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t))dlsym(handle, "ncclAllReduce");
    CommDestroy = (int (*)(ncclComm_t))dlsym(handle, "ncclCommDestroy");
    GetErrorString = (const char *(*)(int))dlsym(handle, "ncclGetErrorString");
    return GetUniqueId && CommInitRank && AllReduce && CommDestroy;
  }
};
static NcclApi g_nccl;
enum { NCCL_FLOAT64 = 8, NCCL_SUM = 0 };

// ---------------------------------------------------------------------------------------------------------------------
// Device allocation owned by its holder: freed on destruction, moved but never copied.
template <typename T> struct DevBuf {
  T *p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr, o.cap = 0; }
  DevBuf &operator=(DevBuf &&o) noexcept {
    std::swap(p, o.p), std::swap(cap, o.cap);  // the old allocation leaves with `o`
    return *this;
  }
  ~DevBuf() {
    if (p) cudaFree(p);
  }
  // grow to at least n elements (with headroom); the old contents are discarded
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr, cap = 0;
    size_t want = n + n / 4 + 64;
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
};

// Pinned host bytes owned by their holder: freed on destruction, grown like DevBuf (n + n / 4); growing discards the contents.
struct PinnedBlock {
  uint8_t *p = nullptr;
  size_t cap = 0;
  PinnedBlock() = default;
  PinnedBlock(const PinnedBlock &) = delete;
  PinnedBlock &operator=(const PinnedBlock &) = delete;
  ~PinnedBlock() {
    if (p) cudaFreeHost(p);
  }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr, cap = 0;
    const cudaError_t e = cudaMallocHost((void **)&p, n + n / 4);
    if (e == cudaSuccess) cap = n + n / 4;
    return e;
  }
};

// The buffers of one device-map arena (MapArena, esikf_map.cuh) and the capacities they were reserved for. The slots,
// planes and recs buffers of the live arena also hold a host-uploaded map (esikf_map_upload).
struct MapArenaBufs {
  DevBuf<HashSlot> slots;
  DevBuf<int> slot_root, slot_cap;
  DevBuf<MapNode> nodes;
  DevBuf<double> pool;
  DevBuf<PlaneRec> recs;
  DevBuf<esikf_plane> planes;
  DevBuf<int> rec_node, counters;
  DevBuf<unsigned long long> counters64;
  uint32_t hash_cap = 0;
  int node_cap = 0, rec_cap = 0;
  long long pool_cap = 0;  // points
  cudaError_t reserve(uint32_t hash_cap_, int node_cap_, int rec_cap_, long long pool_cap_) {
    cudaError_t e;
    if ((e = slots.reserve(hash_cap_)) || (e = slot_root.reserve(hash_cap_)) || (e = slot_cap.reserve(hash_cap_)) || (e = nodes.reserve((size_t)node_cap_)) ||
        (e = pool.reserve((size_t)pool_cap_ * MAP_PT_D)) || (e = recs.reserve((size_t)rec_cap_)) || (e = planes.reserve((size_t)rec_cap_)) ||
        (e = rec_node.reserve((size_t)rec_cap_)) || (e = counters.reserve(8)) || (e = counters64.reserve(2)))
      return e;
    hash_cap = hash_cap_, node_cap = node_cap_, rec_cap = rec_cap_, pool_cap = pool_cap_;
    return cudaSuccess;
  }
  MapArena view(const MapCfg &cfg) const {
    MapArena A;
    A.slots = slots.p, A.hash_mask = hash_cap - 1, A.slot_root = slot_root.p, A.slot_cap = slot_cap.p;
    A.nodes = nodes.p, A.node_cap = node_cap, A.pool = pool.p, A.pool_cap = pool_cap;
    A.recs = recs.p, A.planes = planes.p, A.rec_node = rec_node.p, A.rec_cap = rec_cap;
    A.counters = counters.p, A.counters64 = counters64.p, A.cfg = cfg;
    return A;
  }
};

#define VIO_PERSIST_SMEM (sizeof(VioSmem) + sizeof(FusedSolveSmem))

struct esikf_ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  std::string err;
  int64_t launches = 0;
  int solve_mode = 0;
  int loop_mode = 2;      // >= 1: one persistent cooperative kernel per update (gain solve replicated in every CTA, one
                          //    grid exchange per iteration; carries the NVLink peer exchange when peers are attached),
                          // 0: one residual + one solve launch per iteration (NCCL communicator, kernel timing)
  int coop_ok = 0;
  int coop_lio = 0, coop_vio = 0;  // co-resident CTAs per SM of the persistent kernels
  uint32_t tuning = 0;             // ESIKF_TUNE_* flags (measurement variants)
  DevBuf<unsigned int> barrier;          // LIO kernel: two grid barriers {counter @ +0, release word @ +128 B}, 256 B apart; launches alternate
  DevBuf<unsigned long long> grid_mbox;  // VIO kernel: the grid mailbox (grid_mbox_words), then the exchange counter
  unsigned int *exchange_seq = nullptr;  // device word: exchanges executed so far (the tag of both mailboxes follows it)
  DevBuf<unsigned long long> stamps;  // 8 per slot: 8 LIO slots then 64 VIO slots; debug, LIO per-CTA; the VIO chain stamps
  bool want_stamps = false;
  // The inputs the entry points read, one group each with one validity marker: `need` checks them, `void_inputs` voids them.
  // Besides the input it sets, a call voids:
  //   esikf_vio_set_camera: the retrieval; the image when width or height changed; the sub-map and its inverse refs when
  //     patch_pyrimid_level changed (re-setting an identical camera voids neither)
  //   esikf_vio_set_ref_images: the inverse refs (their indices point into the images it releases); esikf_vmap_init: the placement
  //   esikf_lio_run, esikf_vio_run: the posterior until their launch has succeeded; esikf_lio_run also the normals
  //   esikf_map_upload: the normals; esikf_map_device_init: the normals and the export
  //   esikf_map_device_build / update: the export and the pv list until they succeed
  //   esikf_map_device_update_points: the export, the pv list and the normals; esikf_map_device_slide: the export and the normals
  //   a device map call that fails: the map, until esikf_map_device_init
  //   esikf_rgb_set_cloud, esikf_vio_retrieve_scan: the cloud, the retrieval, until they succeed
  // extrinsics: as set, and extR | extT on the device (what the LIO precompute reads)
  esikf_extrinsics ext{};
  double ext_host[12] = {};
  DevBuf<double> ext_dev;
  bool have_ext = false;

  // camera and VIO config: cam.width == 0 before the first esikf_vio_set_camera
  esikf_camera cam{};
  esikf_vio_cfg vio_cfg{};

  // current image: img_w == 0 when there is none of the camera's size
  DevBuf<uint8_t> img;
  int img_w = 0, img_h = 0;
  VioTma tma;                      // tensor maps of `img` (ESIKF_TUNE_VIO_TMA), encoded for tma_img / tma_w x tma_h
  const uint8_t *tma_img = nullptr;
  int tma_w = 0, tma_h = 0;

  // installed sub-map (set_patches, warp_patches(keep_on_device), select_patches), laid out for submap_levels levels (0: none
  // installed), and the inverse-compositional references of its first n_inv_refs patches
  DevBuf<double> vis_pos, inv_expo;
  DevBuf<float> warp_patch, errors;
  DevBuf<int32_t> search_levels;
  int n_patches = 0, submap_levels = 0;
  DevBuf<double> inv_ref_px, inv_ref_f, inv_ref_R, inv_ref_pos, H_sub_inv;
  DevBuf<int32_t> inv_ref_idx;
  int n_inv_refs = 0;

  // reference images of the warp producers: none while ref_imgs is empty
  std::vector<DevBuf<uint8_t>> ref_imgs;
  DevBuf<const uint8_t *> ref_img_ptrs;
  int ref_w = 0, ref_h = 0;

  // resident scan and its precompute: SCAN_SET until an esikf_lio_run ran it; a fresh context's empty one (SCAN_NONE) needs no run
  DevBuf<float> pts;
  DevBuf<double> pre;
  DevBuf<int32_t> match_plane, normal_plane;
  DevBuf<float> dis;
  int n_pts = 0;
  int pre_stride = 0;
  enum { SCAN_NONE, SCAN_SET, SCAN_RUN } scan = SCAN_NONE;
  double pre_ext[12] = {};   // the extR extT and dept_err / beam_err the precompute in `pre` was made with
  float pre_dept_err = 0.f, pre_beam_err = 0.f;
  esikf_lio_cfg lio_cfg{};
  DevBuf<double> lio_slot_block;  // lane slots of the LIO kernels' L2-slot warps: [partial_blocks][LIO_L2_WARPS * 32][SLOT_D]

  // voxel map: map.slots / planes (as uploaded, 256-byte records) / recs (what the residual kernel reads, 144 bytes) serve the
  // host-uploaded and the device-resident map; MAP_DEVICE_VOID: one a failed call voided (only map_device_* calls reach it)
  enum { MAP_NONE, MAP_HOST, MAP_DEVICE, MAP_DEVICE_VOID } map_kind = MAP_NONE;
  MapArenaBufs map;
  uint32_t hash_mask = 0;
  int n_planes = 0;  // of the host-uploaded map
  esikf_map_cfg map_cfg{};  // device-resident map (esikf_map_device_*): octree nodes, point lists and refits stay on the GPU
  MapCfg arena_cfg{};
  MapArenaBufs spare;  // esikf_map_device_slide copies the surviving roots into it, then it and `map` change roles
  DevBuf<int> map_work, map_survivors;
  DevBuf<unsigned long long> map_demand;  // map_demand_kernel's sums and defer word (capacity growth)
  DevBuf<unsigned int> map_key_in, map_key_out, map_idx_in, map_idx_out;
  DevBuf<MapTouched> map_touched;
  DevBuf<unsigned char> map_sort_tmp;
  int map_hash_bits = 0;
  esikf_map_stats map_last{};

  // the last map update's points, -1 for none: map_export_points of its tick (touched list map_touched) for map_device_export;
  // pv_n of its pv list (pv_list_, LIVMapper.cpp:413-424) in map_pt (point_w | var) and map_pt_normal (pv.normal) for
  // generate_points / retrieve_scan(point_w = NULL); normals_n whose pv.normal of the current LIO run map_pt_normal holds
  DevBuf<double> map_pt, map_pt_normal;
  int map_export_points = -1, pv_n = -1, normals_n = -1;

  // last posterior: which update's posterior `state` holds, what a call's state = NULL stands for (state_or_posterior)
  enum Resident { RESIDENT_NONE, RESIDENT_LIO, RESIDENT_VIO } resident = RESIDENT_NONE;
  DevBuf<double> state_prop;             // [state 386 | prop 386] contiguous: one H2D copy per update
  double *state = nullptr, *prop = nullptr;
  DevBuf<double> info, partials, old_state, G;
  // pinned staging ring for the two packed states of an update (slot reuse guarded by an event)
  enum { STAGE_SLOTS = 16 };
  double *stage = nullptr;
  unsigned char *stage_ctrl = nullptr;   // pinned copy of the loop-control block read by the fetch calls
  cudaEvent_t stage_ev[STAGE_SLOTS] = {};
  unsigned stage_idx = 0;
  unsigned launch_parity = 0;            // the persistent kernels alternate between two grid-barrier counters
  DevBuf<unsigned char> ctl_block;  // [esikf_lio_stats | Ctrl | 64 B pad | esikf_vio_stats]; initialised by CTA 0 of the persistent kernels,
                                    // by a memset on the per-iteration launch path
  esikf_lio_stats *lio_stats = nullptr;
  Ctrl *ctrl = nullptr;
  esikf_vio_stats *vio_stats = nullptr;
  int partial_blocks = 0;

  // coloured cloud (esikf_rgb_*): the world cloud of the last esikf_rgb_set_cloud, rgb_n == -1 when there is none
  DevBuf<float> rgb_cloud;
  int rgb_n = -1;

  // retrieval: the depth image of the last esikf_vio_retrieve_scan (ret_w == 0: none) and the frame pose it was made with
  DevBuf<double> ret_state;
  DevBuf<float> ret_depth;
  double ret_Rci[9] = {}, ret_Pci[3] = {};
  int ret_w = 0, ret_h = 0;

  // observation store (esikf_vmap_*, esikf_vmap.cu): vmap_cap point records (0: no store), the first vmap_points in use
  DevBuf<uint8_t> vmap;
  int64_t vmap_cap = 0, vmap_points = 0;
  std::vector<uint32_t> vmap_seen;  // per point, the last call (vmap_epoch) that named it: the repeated-id check in O(n)
  uint32_t vmap_epoch = 0;
  // placement: the device feat_map of the store's points (esikf_vmap_place_points, esikf_vretrieve.cu): vpl_cap point records,
  // ids below vpl_hi possibly placed, vpl_placed of them placed (the next sequence number); vpl_done mirrors which
  DevBuf<uint8_t> vpl;
  int64_t vpl_cap = 0, vpl_hi = 0, vpl_placed = 0;
  std::vector<uint8_t> vpl_done;

  // What the front-end entry points need for the length of one call only (lay_out_scratch). Every such call runs on `stream`
  // and synchronises it before it returns, so they can share it; nothing a later call reads may be kept here.
  DevBuf<uint8_t> scratch;
  PinnedBlock host;  // the same in pinned host memory: every such call stages its inputs and reads its answers back through it

  // multi-GPU
  int rank = 0, nranks = 1;
  ncclComm_t comm = nullptr;
  // NVLink peer-memory all-reduce inside the persistent kernels
  unsigned long long *mailbox = nullptr;             // own mailbox [2][PEER_MAX_RANKS][PEER_SLOT_WORDS]
  std::vector<unsigned long long *> peer_ptrs;       // mailbox of every rank as mapped into this process
  DevBuf<unsigned long long *> peer_ptrs_dev;
  bool p2p = false;

  // measurement
  bool timing = false;
  std::vector<cudaEvent_t> ev;      // 3 per slot: before residual, after residual, after solve
  int lio_slots = 0, vio_slots = 0;
  bool lio_timed = false, vio_timed = false;
  DevBuf<uint8_t> flush;
  DevBuf<double> scratch_state;

  MapArena arena() const { return map.view(arena_cfg); }  // the live device map as the kernels see it

  // Runs before the members are destroyed: the stream is drained first, then what is not a DevBuf is released here.
  ~esikf_ctx() {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    if (comm && g_nccl.CommDestroy) g_nccl.CommDestroy(comm);
    for (size_t r = 0; r < peer_ptrs.size(); r++)
      if ((int)r != rank && peer_ptrs[r]) cudaIpcCloseMemHandle(peer_ptrs[r]);
    if (mailbox) cudaFree(mailbox);
    if (stage) cudaFreeHost(stage);
    if (stage_ctrl) cudaFreeHost(stage_ctrl);
    for (cudaEvent_t e : stage_ev)
      if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }
};

static int fail(esikf_ctx *c, int code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (c) c->err = buf;
  return code;
}
#define CK(call)                                                                                                   \
  do {                                                                                                             \
    cudaError_t e__ = (call);                                                                                      \
    if (e__ != cudaSuccess) return fail(ctx, ESIKF_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

// The inputs of the context's groups (esikf_ctx), one bit each.
enum Input : unsigned {
  IN_EXT = 1u << 0, IN_CAMERA = 1u << 1, IN_IMAGE = 1u << 2, IN_SUBMAP = 1u << 3, IN_INV_REFS = 1u << 4, IN_REF_IMAGES = 1u << 5,
  IN_SCAN = 1u << 6, IN_RUN_SCAN = 1u << 7, IN_MAP = 1u << 8, IN_HOST_MAP = 1u << 9, IN_DEVICE_MAP = 1u << 10, IN_EXPORT = 1u << 11,
  IN_PV_LIST = 1u << 12, IN_NORMALS = 1u << 13, IN_CLOUD = 1u << 14, IN_RETRIEVAL = 1u << 15, IN_STORE = 1u << 16, IN_POSTERIOR = 1u << 17,
};

// The one check of each input: ESIKF_ERR_STATE naming `call` and the first of `inputs` missing (the posterior: state_or_posterior).
static int need(esikf_ctx *ctx, const char *call, unsigned inputs) {
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

// The one way to void an input; the table at esikf_ctx says when. A voided device map stays reachable to map_device_* calls.
static void void_inputs(esikf_ctx *ctx, unsigned inputs) {
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

// One call's layout of the scratch: its host inputs first, then its work arrays, then its answers as one span that ends the
// layout. `lay` marks where the inputs end and where the answers begin.
struct CallLayout : ScratchLayout {
  size_t in_bytes = 0, answers_at = SIZE_MAX;
  void end_inputs() { in_bytes = bytes; }
  void begin_answers() { answers_at = bytes; }
};

// The device scratch of ctx laid out by `lay`, and the pinned block reserved for the larger of the call's inputs and its
// answer span, so that neither staging nor read_back regrows the block while a copy from or to it may still be queued.
template <typename F> static cudaError_t lay_out_scratch(esikf_ctx *ctx, F &&lay) {
  CallLayout s;
  lay(s);
  const size_t answers = s.bytes - std::min(s.answers_at, s.bytes);
  if (const cudaError_t e = ctx->scratch.reserve(s.bytes)) return e;
  if (const cudaError_t e = ctx->host.reserve(std::max(s.in_bytes, answers))) return e;
  s = CallLayout{};
  s.base = (uintptr_t)ctx->scratch.p;
  lay(s);
  return cudaSuccess;
}

// One host input of a call and where it goes in scratch; a null src leaves zeros there.
struct HostIn {
  const void *dst, *src;
  size_t bytes;
};
// The call's inputs, staged in the pinned block at their scratch offsets, then uploaded with one copy of the scratch up to the
// end of the last one.
static cudaError_t upload(esikf_ctx *ctx, std::initializer_list<HostIn> in) {
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

// The one readback of answers that lie between the device addresses `first` and `end`: a copy into the pinned block and a
// synchronisation. copy_out then hands them to the caller, whose buffers a failed call thus leaves untouched.
static cudaError_t read_back(esikf_ctx *ctx, const void *first, const void *end) {
  const size_t bytes = (const uint8_t *)end - (const uint8_t *)first;
  if (bytes > ctx->host.cap) return cudaErrorInvalidValue;  // the layout did not mark these answers
  const cudaError_t e = cudaMemcpyAsync(ctx->host.p, first, bytes, cudaMemcpyDeviceToHost, ctx->stream);
  return e == cudaSuccess ? cudaStreamSynchronize(ctx->stream) : e;
}
static void copy_out(const esikf_ctx *ctx, void *dst, const void *first, const void *src, size_t bytes) {
  memcpy(dst, ctx->host.p + ((const uint8_t *)src - (const uint8_t *)first), bytes);
}
// The same for k answers of one array at p, or a count the rest of the call depends on, straight into out.
template <typename T> static cudaError_t read_back_to(esikf_ctx *ctx, const T *p, T *out, size_t k = 1) {
  const cudaError_t e = read_back(ctx, p, p + k);
  if (e == cudaSuccess) copy_out(ctx, out, p, p, k * sizeof(T));
  return e;
}

static cudaEvent_t *timing_events(esikf_ctx *ctx, int base, int slot) {
  size_t need = (size_t)(base + slot + 1) * 3;
  while (ctx->ev.size() < need) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return nullptr;
    ctx->ev.push_back(e);
  }
  return &ctx->ev[(size_t)(base + slot) * 3];
}
enum { EV_LIO_BASE = 0, EV_VIO_BASE = 8 };

static void shard_of(int n, int rank, int nranks, int &begin, int &count) {
  // contiguous blocks, remainder spread over the first ranks
  int base = n / nranks, rem = n % nranks;
  begin = rank * base + (rank < rem ? rank : rem);
  count = base + (rank < rem ? 1 : 0);
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
template <int L2W> static void launch_lio_residual(int grid, cudaStream_t st, const LioKernelArgs &ka) {
  lio_residual_kernel<L2W><<<grid, LioSmem<L2W>::THREADS, sizeof(LioSmem<L2W>), st>>>(ka);
}
static void launch_lio_residual(bool l2_slots, int grid, cudaStream_t st, const LioKernelArgs &ka) {
  if (l2_slots) launch_lio_residual<LIO_L2_WARPS>(grid, st, ka);
  else launch_lio_residual<0>(grid, st, ka);
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
       ctx->barrier.reserve(128) == cudaSuccess && ctx->grid_mbox.reserve(grid_mbox_words(ctx->partial_blocks) + 1) == cudaSuccess &&
       ctx->lio_slot_block.reserve((size_t)ctx->partial_blocks * LIO_L2_WARPS * 32 * SLOT_D) == cudaSuccess;
  if (ok) cudaMemsetAsync(ctx->barrier.p, 0, 128 * sizeof(unsigned int), ctx->stream);
  if (ok) {  // tag 0 is never sent
    cudaMemsetAsync(ctx->grid_mbox.p, 0, ctx->grid_mbox.cap * sizeof(unsigned long long), ctx->stream);
    ctx->exchange_seq = reinterpret_cast<unsigned int *>(ctx->grid_mbox.p + grid_mbox_words(ctx->partial_blocks));
  }
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
  if (!ok) {
    delete ctx;
    return ESIKF_ERR_CUDA;
  }
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

// ---------------------------------------------------------------------------------------------------------------- map
int esikf_map_upload(esikf_ctx *ctx, const int64_t *keys, const int32_t *first, const int32_t *count, int32_t n_roots,
                     const esikf_plane *planes, int32_t n_planes, double voxel_size) {
  if (!ctx || n_roots < 0 || n_planes < 0 || (n_roots > 0 && (!keys || !first || !count)) || (n_planes > 0 && !planes) || !(voxel_size > 0))
    return fail(ctx, ESIKF_ERR_ARG, "map_upload: bad argument");
  CK(cudaSetDevice(ctx->device));
  uint32_t cap = 1024;
  while (cap < (uint32_t)n_roots * 2u) cap <<= 1;
  std::vector<HashSlot> table(cap);
  for (auto &s : table) s.key = ESIKF_KEY_EMPTY, s.first = 0, s.count = 0;
  for (int r = 0; r < n_roots; r++) {
    long long x = keys[3 * r], y = keys[3 * r + 1], z = keys[3 * r + 2];
    if (!key_in_range(x, y, z)) return fail(ctx, ESIKF_ERR_ARG, "map_upload: voxel key (%lld,%lld,%lld) outside +-2^20", x, y, z);
    if (first[r] < 0 || count[r] < 0 || first[r] + count[r] > n_planes) return fail(ctx, ESIKF_ERR_ARG, "map_upload: root %d plane range", r);
    unsigned long long k = pack_key(x, y, z);
    uint32_t s = hash_key(k) & (cap - 1);
    while (table[s].key != ESIKF_KEY_EMPTY) {
      if (table[s].key == k) return fail(ctx, ESIKF_ERR_ARG, "map_upload: duplicate voxel key");
      s = (s + 1) & (cap - 1);
    }
    table[s].key = k, table[s].first = (uint32_t)first[r], table[s].count = (uint32_t)count[r];
  }
  CK(ctx->map.slots.reserve(cap));
  CK(ctx->map.planes.reserve((size_t)n_planes + 1));
  CK(ctx->map.recs.reserve((size_t)n_planes + 1));
  CK(cudaMemcpyAsync(ctx->map.slots.p, table.data(), cap * sizeof(HashSlot), cudaMemcpyHostToDevice, ctx->stream));
  if (n_planes) {
    CK(cudaMemcpyAsync(ctx->map.planes.p, planes, (size_t)n_planes * sizeof(esikf_plane), cudaMemcpyHostToDevice, ctx->stream));
    plane_compact_kernel<<<(n_planes + 127) / 128, 128, 0, ctx->stream>>>(ctx->map.planes.p, nullptr, n_planes, ctx->map.recs.p);
    ctx->launches++;
  }
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->hash_mask = cap - 1;
  ctx->n_planes = n_planes;
  ctx->map_kind = esikf_ctx::MAP_HOST;  // a host-flattened map replaces a device-resident one
  void_inputs(ctx, IN_NORMALS);
  return ESIKF_OK;
}

int esikf_map_patch(esikf_ctx *ctx, const int32_t *plane_ids, const esikf_plane *planes, int32_t n) {
  if (!ctx || n < 0 || (n > 0 && (!plane_ids || !planes))) return fail(ctx, ESIKF_ERR_ARG, "map_patch: bad argument");
  if (int rc = need(ctx, "map_patch", IN_HOST_MAP)) return rc;
  CK(cudaSetDevice(ctx->device));
  for (int i = 0; i < n; i++)
    if (plane_ids[i] < 0 || plane_ids[i] >= ctx->n_planes) return fail(ctx, ESIKF_ERR_ARG, "map_patch: plane id %d", plane_ids[i]);
  for (int i = 0; i < n;) {
    int j = i + 1;
    while (j < n && plane_ids[j] == plane_ids[j - 1] + 1) j++;  // a run of consecutive ids travels as one copy
    CK(cudaMemcpyAsync(ctx->map.planes.p + plane_ids[i], planes + i, (size_t)(j - i) * sizeof(esikf_plane), cudaMemcpyHostToDevice, ctx->stream));
    i = j;
  }
  if (n > 0) {
    int32_t *ids;
    auto lay = [&](CallLayout &s) { ids = s.take<int32_t>(n), s.end_inputs(); };
    CK(lay_out_scratch(ctx, lay));
    CK(upload(ctx, {{ids, plane_ids, (size_t)n * sizeof(int32_t)}}));
    plane_compact_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(ctx->map.planes.p, ids, n, ctx->map.recs.p);
    ctx->launches++;
  }
  CK(cudaStreamSynchronize(ctx->stream));
  return ESIKF_OK;
}

// ------------------------------------------------------------------------------------------------ device-resident map (f1)
__global__ void gather_normals_kernel(const int32_t *__restrict__ match_plane, const PlaneRec *__restrict__ recs, int n, double *__restrict__ out);

static int map_check_errors(esikf_ctx *ctx, const char *what) {
  int c[4];
  unsigned long long pool_used = 0;
  CK(cudaMemcpyAsync(c, ctx->map.counters.p, sizeof(c), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(&pool_used, ctx->map.counters64.p, sizeof(pool_used), cudaMemcpyDeviceToHost, ctx->stream));
  int work[2];
  CK(cudaMemcpyAsync(work, ctx->map_work.p, sizeof(work), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->map_last.nodes = c[0], ctx->map_last.records = c[1], ctx->map_last.errors = c[2], ctx->map_last.roots = c[3];
  ctx->map_last.pool_points = (int64_t)pool_used, ctx->map_last.touched_roots = work[0];
  if (c[2]) {
    void_inputs(ctx, IN_MAP);  // the map is not trustworthy any more: the next lio_run must not use it
    return fail(ctx, ESIKF_ERR_STATE, "%s: device map capacity exceeded (flags 0x%x:%s%s%s%s%s%s) — raise the esikf_map_cfg capacities and rebuild", what, c[2],
                (c[2] & MAP_ERR_NODES) ? " nodes" : "", (c[2] & MAP_ERR_POOL) ? " point-pool" : "", (c[2] & MAP_ERR_RECS) ? " records" : "",
                (c[2] & MAP_ERR_HASH) ? " hash" : "", (c[2] & MAP_ERR_KEY) ? " key-range" : "", (c[2] & MAP_ERR_STACK) ? " octree-depth" : "");
  }
  return ESIKF_OK;
}

int esikf_map_device_init(esikf_ctx *ctx, const esikf_map_cfg *cfg) {
  if (!ctx || !cfg || !(cfg->voxel_size > 0) || cfg->max_layer < 0 || cfg->max_layer >= MAP_MAX_LAYERS || cfg->max_points_num < 1 || (cfg->grow != 0 && cfg->grow != 1))
    return fail(ctx, ESIKF_ERR_ARG, "map_device_init: bad argument");
  for (int k = 0; k <= cfg->max_layer; k++)
    if (cfg->layer_init_num[k] < 1) return fail(ctx, ESIKF_ERR_ARG, "map_device_init: layer_init_num[%d] = %d", k, cfg->layer_init_num[k]);
  CK(cudaSetDevice(ctx->device));
  const int64_t roots = cfg->root_capacity > 0 ? cfg->root_capacity : (1 << 20);
  uint32_t cap = 1024;
  int bits = 10;
  while ((int64_t)cap < 2 * roots) cap <<= 1, bits++;
  const int64_t node_cap = cfg->node_capacity > 0 ? cfg->node_capacity : 4 * roots;
  const int64_t rec_cap = cfg->record_capacity > 0 ? cfg->record_capacity : 4 * roots;
  const int64_t pool_cap = cfg->point_capacity > 0 ? cfg->point_capacity : 64 * roots;
  if (node_cap > 0x7fffffff || rec_cap > 0x7fffffff || pool_cap > 0x7fffffff) return fail(ctx, ESIKF_ERR_ARG, "map_device_init: capacity above 2^31");
  CK(ctx->map.reserve(cap, (int)node_cap, (int)rec_cap, pool_cap));
  CK(ctx->map_work.reserve(4));
  if (cfg->grow) CK(ctx->map_demand.reserve(MAP_DEMAND_WORDS));
  MapCfg &mc = ctx->arena_cfg;
  mc.voxel_size = (float)cfg->voxel_size, mc.planer_threshold = (float)cfg->min_eigen_value;
  mc.max_layer = cfg->max_layer, mc.max_points_num = cfg->max_points_num;
  for (int k = 0; k < MAP_MAX_LAYERS; k++) mc.layer_init_num[k] = cfg->layer_init_num[k <= cfg->max_layer ? k : cfg->max_layer];
  map_reset_kernel<<<(cap + 255) / 256, 256, 0, ctx->stream>>>(ctx->arena());
  CK(cudaMemsetAsync(ctx->map_work.p, 0, 4 * sizeof(int), ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->launches++;
  ctx->map_cfg = *cfg;
  ctx->map_hash_bits = bits;
  ctx->hash_mask = cap - 1;
  ctx->map_kind = esikf_ctx::MAP_DEVICE;  // an empty map is a valid map (nothing matches)
  void_inputs(ctx, IN_NORMALS | IN_EXPORT);
  memset(&ctx->map_last, 0, sizeof(ctx->map_last));
  return ESIKF_OK;
}

// sort by slot, list the touched roots, (growth on) bound what they need, replay them unless that does not fit
static int map_replay_tick(esikf_ctx *ctx, int n, bool build) {
  cudaStream_t st = ctx->stream;
  const unsigned int invalid = ctx->map.hash_cap;
  size_t tmp_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, ctx->map_key_in.p, ctx->map_key_out.p, ctx->map_idx_in.p, ctx->map_idx_out.p, n, 0, ctx->map_hash_bits + 1, st);
  CK(ctx->map_sort_tmp.reserve(tmp_bytes + 16));
  CK(cub::DeviceRadixSort::SortPairs(ctx->map_sort_tmp.p, tmp_bytes, ctx->map_key_in.p, ctx->map_key_out.p, ctx->map_idx_in.p, ctx->map_idx_out.p, n, 0,
                                     ctx->map_hash_bits + 1, st));
  CK(cudaMemsetAsync(ctx->map_work.p, 0, 2 * sizeof(int), st));
  map_heads_kernel<<<(n + 255) / 256, 256, 0, st>>>(ctx->map_key_out.p, n, invalid, ctx->map_touched.p, ctx->map_work.p);
  const unsigned long long *defer = nullptr;
  if (ctx->map_cfg.grow) {
    CK(cudaMemsetAsync(ctx->map_demand.p, 0, MAP_DEMAND_WORDS * sizeof(unsigned long long), st));
    map_demand_kernel<<<ctx->sm_count * 4, 128, 0, st>>>(ctx->arena(), ctx->map_touched.p, ctx->map_work.p, ctx->map_demand.p, build ? 1 : 0);
    defer = ctx->map_demand.p + 5;
    ctx->launches++;
  }
  map_replay_kernel<<<ctx->sm_count * 4, 128, 0, st>>>(ctx->arena(), ctx->map_touched.p, ctx->map_work.p, ctx->map_idx_out.p, ctx->map_pt.p, build ? 1 : 0, defer);
  ctx->launches += 4;
  CK(cudaGetLastError());
  return ESIKF_OK;
}

static int map_capacity_error(esikf_ctx *ctx, const char *what, const char *resource, long long want) {
  void_inputs(ctx, IN_MAP);
  return fail(ctx, ESIKF_ERR_STATE, "%s: the device map cannot grow to %lld %s (the limit is 2^31)", what, want, resource);
}

// Capacity growth: copy the live arena into one of the given capacities with the slide's machinery and an unbounded box (the
// copy only compacts, so it fits any arena at least as large), make it the map and free the old one. Roots without a root
// node (keys inserted by a tick that was deferred) are not copied. When an allocation fails the map is invalidated: a
// deferred tick may have inserted keys already, and the LIO probe would treat them as present voxels.
static int map_grow(esikf_ctx *ctx, long long hash_cap, long long node_cap, long long rec_cap, long long pool_cap, const char *what) {
  if (hash_cap > (1ll << 31)) return map_capacity_error(ctx, what, "hash slots", hash_cap);
  if (node_cap > 0x7fffffff) return map_capacity_error(ctx, what, "nodes", node_cap);
  if (rec_cap > 0x7fffffff) return map_capacity_error(ctx, what, "records", rec_cap);
  if (pool_cap > 0x7fffffff) return map_capacity_error(ctx, what, "stored points", pool_cap);
  cudaStream_t st = ctx->stream;
  MapArenaBufs fresh;
  cudaError_t e = fresh.reserve((uint32_t)hash_cap, (int)node_cap, (int)rec_cap, pool_cap);
  if (e == cudaSuccess) e = ctx->map_survivors.reserve((size_t)(ctx->map_last.roots > 0 ? ctx->map_last.roots : 1) + 1);
  if (e != cudaSuccess) {
    cudaGetLastError();  // a failed allocation is not sticky: later calls must not report it again
    void_inputs(ctx, IN_MAP);
    return fail(ctx, ESIKF_ERR_CUDA, "%s: growing the device map to %lld hash slots / %lld nodes / %lld records / %lld points failed: %s", what, hash_cap, node_cap,
                rec_cap, pool_cap, cudaGetErrorString(e));
  }
  const MapArena S = ctx->arena(), D = fresh.view(ctx->arena_cfg);
  const long long big = 1ll << 40;
  map_reset_kernel<<<(unsigned)((hash_cap + 255) / 256), 256, 0, st>>>(D);
  CK(cudaMemsetAsync(ctx->map_work.p, 0, 2 * sizeof(int), st));
  map_survivors_kernel<<<(ctx->map.hash_cap + 255) / 256, 256, 0, st>>>(S, -big, -big, -big, big, big, big, ctx->map_survivors.p, ctx->map_work.p);
  map_copy_kernel<<<ctx->sm_count * 4, 128, 0, st>>>(S, D, ctx->map_survivors.p, ctx->map_work.p);
  ctx->launches += 3;
  CK(cudaGetLastError());
  std::swap(ctx->map, fresh);
  int bits = 0;
  while ((1ll << bits) < hash_cap) bits++;
  ctx->hash_mask = (uint32_t)(hash_cap - 1), ctx->map_hash_bits = bits;  // what the LIO probe and the key sort read
  return map_check_errors(ctx, what);  // synchronises: the old arena (now in `fresh`) is no longer read when it is freed
}

// growth on: room in the hash table for n new roots (at most one per point) before any key of the tick is inserted
static bool map_hash_short(const esikf_ctx *ctx, int n) { return ctx->map_cfg.grow && (long long)ctx->map_last.roots + n > (long long)ctx->map.hash_cap / 2; }
static int map_grow_hash(esikf_ctx *ctx, int n, const char *what) {
  const MapArenaBufs &m = ctx->map;
  return map_grow(ctx, map_grown_hash(m.hash_cap, ctx->map_last.roots, n), m.node_cap, m.rec_cap, m.pool_cap, what);
}

// Apply the keyed tick (map_key_in / map_idx_in, points in map_pt). With growth on, a tick the demand bound says might not
// fit is not replayed: each short resource grows to map_grown_capacity, the points are keyed again into the new arena and
// the tick is applied there (a tick that fits costs no extra round trip: the defer word rides on the error check's sync).
static int map_apply_points(esikf_ctx *ctx, int n, bool build) {
  const char *what = build ? "map_device_build" : "map_device_update";
  cudaStream_t st = ctx->stream;
  int rc = map_replay_tick(ctx, n, build);
  if (rc || !ctx->map_cfg.grow) return rc ? rc : map_check_errors(ctx, what);
  unsigned long long d[MAP_DEMAND_WORDS];
  CK(cudaMemcpyAsync(d, ctx->map_demand.p, sizeof(d), cudaMemcpyDeviceToHost, st));
  if ((rc = map_check_errors(ctx, what)) || !d[5]) return rc;
  const MapArenaBufs &m = ctx->map;
  const esikf_map_stats &u = ctx->map_last;  // the counters before the deferred tick
  const long long node_cap = (d[5] & MAP_ERR_NODES) ? map_grown_capacity(m.node_cap, u.nodes, (long long)d[0]) : m.node_cap;
  const long long pool_cap = (d[5] & MAP_ERR_POOL) ? map_grown_capacity(m.pool_cap, u.pool_points, (long long)d[1]) : m.pool_cap;
  const long long rec_cap = (d[5] & MAP_ERR_RECS) ? map_grown_capacity(m.rec_cap, u.records, (long long)d[2]) : m.rec_cap;
  if ((rc = map_grow(ctx, m.hash_cap, node_cap, rec_cap, pool_cap, what))) return rc;
  map_keys_kernel<<<(n + 255) / 256, 256, 0, st>>>(ctx->arena(), ctx->map_pt.p, n, ctx->map_key_in.p, ctx->map_idx_in.p, ctx->map.hash_cap);
  ctx->launches++;
  if ((rc = map_replay_tick(ctx, n, build))) return rc;
  CK(cudaMemcpyAsync(d, ctx->map_demand.p, sizeof(d), cudaMemcpyDeviceToHost, st));
  if ((rc = map_check_errors(ctx, what))) return rc;
  if (d[5]) {  // the grown arena holds used + demand of every short resource: the bound itself would be broken
    void_inputs(ctx, IN_MAP);
    return fail(ctx, ESIKF_ERR_STATE, "%s: the tick was deferred again after the map grew (flags 0x%x)", what, (unsigned)d[5]);
  }
  return ESIKF_OK;
}

static int map_reserve_tick(esikf_ctx *ctx, int n) {
  CK(ctx->map_pt.reserve((size_t)n * MAP_PT_D + 16));
  CK(ctx->map_pt_normal.reserve((size_t)n * 3 + 4));
  CK(ctx->map_key_in.reserve(n + 1));
  CK(ctx->map_key_out.reserve(n + 1));
  CK(ctx->map_idx_in.reserve(n + 1));
  CK(ctx->map_idx_out.reserve(n + 1));
  CK(ctx->map_touched.reserve(n + 1));
  return ESIKF_OK;
}

static int map_from_scan(esikf_ctx *ctx, const double *state, bool build) {
  if (!ctx) return ESIKF_ERR_ARG;
  const char *what = build ? "map_device_build" : "map_device_update";
  void_inputs(ctx, IN_EXPORT | IN_PV_LIST);  // map_pt is rewritten below
  if (int rc = need(ctx, what, IN_DEVICE_MAP | IN_EXT | (build ? 0 : IN_RUN_SCAN))) return rc;
  if (build && ctx->map_last.roots > 0) return fail(ctx, ESIKF_ERR_STATE, "map_device_build needs an empty map (esikf_map_device_init resets it)");
  CK(cudaSetDevice(ctx->device));
  const int n = ctx->n_pts;
  if (n == 0) return ctx->map_export_points = 0, ctx->pv_n = build ? -1 : 0, ESIKF_OK;
  int rc = map_reserve_tick(ctx, n);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  const double *dev_state = ctx->state;  // the posterior the last update left on the device
  if (state) {
    CK(ctx->scratch_state.reserve(S_N));
    CK(cudaMemcpyAsync(ctx->scratch_state.p, state, S_N * sizeof(double), cudaMemcpyHostToDevice, st));
    dev_state = ctx->scratch_state.p;
  }
  const int32_t *match_plane = build ? nullptr : ctx->normal_plane.p;
  if (map_hash_short(ctx, n)) {
    // pv.normal refers to the records of the last LIO run: snapshot it before the copy moves them
    if (match_plane) {
      gather_normals_kernel<<<(n + 255) / 256, 256, 0, st>>>(match_plane, ctx->map.recs.p, n, ctx->map_pt_normal.p);
      ctx->launches++;
      match_plane = nullptr;
    }
    if ((rc = map_grow_hash(ctx, n, what))) return rc;
  }
  MapPointArgs a;
  memset(&a, 0, sizeof(a));
  a.pts = ctx->pts.p, a.pre = ctx->pre.p, a.pre_stride = ctx->pre_stride, a.n = n, a.state = dev_state;
  memcpy(a.extR, ctx->ext.extR, 72), memcpy(a.extT, ctx->ext.extT, 24);
  a.build = build ? 1 : 0, a.dept_err = (float)ctx->map_cfg.dept_err, a.beam_err = (float)ctx->map_cfg.beam_err;
  a.match_plane = match_plane, a.recs = ctx->map.recs.p, a.pt_normal = ctx->map_pt_normal.p;
  a.pt = ctx->map_pt.p, a.pt_slot = ctx->map_key_in.p, a.pt_idx = ctx->map_idx_in.p, a.invalid_slot = ctx->map.hash_cap;
  map_points_kernel<<<(n + 255) / 256, 256, 0, st>>>(ctx->arena(), a);
  ctx->normals_n = build ? -1 : n;
  if ((rc = map_apply_points(ctx, n, build))) return rc;
  return ctx->map_export_points = n, ctx->pv_n = build ? -1 : n, ESIKF_OK;
}

int esikf_map_device_build(esikf_ctx *ctx, const double *state) {
  if (ctx && !state) return fail(ctx, ESIKF_ERR_ARG, "map_device_build: the pose the scan is mapped with is required");
  return map_from_scan(ctx, state, true);
}
int esikf_map_device_update(esikf_ctx *ctx, const double *state) { return map_from_scan(ctx, state, false); }

int esikf_map_device_update_points(esikf_ctx *ctx, const double *point_w, const double *var, int32_t n) {
  if (ctx) void_inputs(ctx, IN_EXPORT | IN_PV_LIST);
  if (!ctx || n < 0 || (n > 0 && (!point_w || !var))) return fail(ctx, ESIKF_ERR_ARG, "map_device_update_points: bad argument");
  if (int rc = need(ctx, "map_device_update_points", IN_DEVICE_MAP)) return rc;
  if (n == 0) return ctx->map_export_points = 0, ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  int rc = map_reserve_tick(ctx, n);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  // [n][12] = point_w | var: two strided copies
  CK(cudaMemcpy2DAsync(ctx->map_pt.p, MAP_PT_D * sizeof(double), point_w, 3 * sizeof(double), 3 * sizeof(double), n, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpy2DAsync(ctx->map_pt.p + 3, MAP_PT_D * sizeof(double), var, 9 * sizeof(double), 9 * sizeof(double), n, cudaMemcpyHostToDevice, st));
  if (map_hash_short(ctx, n) && (rc = map_grow_hash(ctx, n, "map_device_update"))) return rc;
  map_keys_kernel<<<(n + 255) / 256, 256, 0, st>>>(ctx->arena(), ctx->map_pt.p, n, ctx->map_key_in.p, ctx->map_idx_in.p, ctx->map.hash_cap);
  ctx->launches++;
  void_inputs(ctx, IN_NORMALS);
  if ((rc = map_apply_points(ctx, n, false))) return rc;
  return ctx->map_export_points = n, ESIKF_OK;
}

// mapSliding / clearMemOutOfMap (src/voxel_map.cpp:924-971)
int esikf_map_device_slide(esikf_ctx *ctx, const int64_t key_min[3], const int64_t key_max[3]) {
  if (!ctx) return ESIKF_ERR_ARG;
  void_inputs(ctx, IN_EXPORT);
  if (int rc = need(ctx, "map_device_slide", IN_DEVICE_MAP)) return rc;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const MapArenaBufs &live = ctx->map;
  const unsigned cap = live.hash_cap;
  CK(ctx->spare.reserve(cap, live.node_cap, live.rec_cap, live.pool_cap));
  CK(ctx->map_survivors.reserve((size_t)(ctx->map_last.roots > 0 ? ctx->map_last.roots : 1) + 1));
  const MapArena S = ctx->arena(), D = ctx->spare.view(ctx->arena_cfg);
  const long long big = 1ll << 40;
  const long long lo[3] = {key_min ? key_min[0] : -big, key_min ? key_min[1] : -big, key_min ? key_min[2] : -big};
  const long long hi[3] = {key_max ? key_max[0] : big, key_max ? key_max[1] : big, key_max ? key_max[2] : big};
  map_reset_kernel<<<(cap + 255) / 256, 256, 0, st>>>(D);
  CK(cudaMemsetAsync(ctx->map_work.p, 0, 2 * sizeof(int), st));
  map_survivors_kernel<<<(cap + 255) / 256, 256, 0, st>>>(S, lo[0], lo[1], lo[2], hi[0], hi[1], hi[2], ctx->map_survivors.p, ctx->map_work.p);
  map_copy_kernel<<<ctx->sm_count * 4, 128, 0, st>>>(S, D, ctx->map_survivors.p, ctx->map_work.p);
  ctx->launches += 3;
  CK(cudaGetLastError());
  // the fresh arena becomes the map (also when the copy reports an error: the status says so and the map is invalidated)
  std::swap(ctx->map, ctx->spare);
  void_inputs(ctx, IN_NORMALS);  // record positions of the last update are gone
  return map_check_errors(ctx, "map_device_slide");
}

int esikf_map_device_capacity(esikf_ctx *ctx, esikf_map_cfg *out) {
  if (!ctx || !out) return fail(ctx, ESIKF_ERR_ARG, "map_device_capacity: bad argument");
  if (int rc = need(ctx, "map_device_capacity", IN_DEVICE_MAP)) return rc;
  out->root_capacity = ctx->map.hash_cap / 2, out->node_capacity = ctx->map.node_cap;
  out->record_capacity = ctx->map.rec_cap, out->point_capacity = ctx->map.pool_cap;
  out->grow = ctx->map_cfg.grow;
  return ESIKF_OK;
}

int esikf_map_device_stats(esikf_ctx *ctx, esikf_map_stats *out) {
  if (!ctx || !out) return fail(ctx, ESIKF_ERR_ARG, "map_device_stats: bad argument");
  if (int rc = need(ctx, "map_device_stats", IN_DEVICE_MAP)) return rc;
  *out = ctx->map_last;
  return ESIKF_OK;
}

int esikf_map_device_download(esikf_ctx *ctx, int64_t *keys, int32_t *first, int32_t *count, int32_t roots_cap, esikf_plane *planes, int32_t planes_cap, int32_t *n_roots,
                              int32_t *n_planes) {
  if (!ctx || !n_roots || !n_planes) return fail(ctx, ESIKF_ERR_ARG, "map_device_download: bad argument");
  if (int rc = need(ctx, "map_device_download", IN_DEVICE_MAP)) return rc;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const bool fill = keys && first && count && planes && roots_cap > 0;
  const size_t R = fill ? (size_t)roots_cap : 0, P = fill && planes_cap > 0 ? (size_t)planes_cap : 0;
  int *d_out;
  long long *d_keys;
  int32_t *d_first, *d_count;
  esikf_plane *d_planes;
  auto lay = [&](CallLayout &s) {
    s.begin_answers();  // the counts, then the buffers' worth of roots and planes
    d_out = s.take<int>(2), d_keys = s.take<long long>(3 * R), d_first = s.take<int32_t>(R), d_count = s.take<int32_t>(R), d_planes = s.take<esikf_plane>(P);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(cudaMemsetAsync(d_out, 0, 2 * sizeof(int), st));
  const unsigned cap = ctx->map.hash_cap;
  map_download_kernel<<<(cap + 255) / 256, 256, 0, st>>>(ctx->arena(), fill ? d_keys : nullptr, d_first, d_count, d_planes, fill ? roots_cap : 0, fill ? planes_cap : 0, d_out);
  ctx->launches++;
  int out[2];
  CK(read_back_to(ctx, d_out, out, 2));
  *n_roots = out[0], *n_planes = out[1];
  if (!fill) return ESIKF_OK;
  if (out[0] > roots_cap || out[1] > planes_cap)
    return fail(ctx, ESIKF_ERR_ARG, "map_device_download: %d roots / %d planes do not fit the buffers (%d / %d)", out[0], out[1], roots_cap, planes_cap);
  const size_t nr = (size_t)out[0], np = (size_t)out[1];
  CK(read_back(ctx, d_keys, d_planes + np));
  copy_out(ctx, keys, d_keys, d_keys, nr * 3 * sizeof(int64_t)), copy_out(ctx, first, d_keys, d_first, nr * sizeof(int32_t));
  copy_out(ctx, count, d_keys, d_count, nr * sizeof(int32_t)), copy_out(ctx, planes, d_keys, d_planes, np * sizeof(esikf_plane));
  return ESIKF_OK;
}

int esikf_map_device_export(esikf_ctx *ctx, int64_t *keys, int32_t *first, int32_t *count, int32_t roots_cap, esikf_map_node *nodes, int32_t nodes_cap, int32_t *n_roots,
                            int32_t *n_nodes) {
  if (!ctx || !n_roots || !n_nodes) return fail(ctx, ESIKF_ERR_ARG, "map_device_export: bad argument");
  if (int rc = need(ctx, "map_device_export", IN_DEVICE_MAP | IN_EXPORT)) return rc;
  *n_roots = 0, *n_nodes = 0;
  const int n = ctx->map_export_points;
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const bool fill = keys && first && count && nodes && roots_cap > 0;
  // laid out for the buffers' worth of roots and nodes: the scan's offsets must stay in place for the write pass
  const size_t R = fill ? (size_t)roots_cap : 0, NN = fill && nodes_cap > 0 ? (size_t)nodes_cap : 0;
  unsigned long long *packed, *offs;
  long long *d_keys;
  int32_t *d_first, *d_count, *d_rows;
  esikf_map_node *d_nodes;
  auto lay = [&](CallLayout &s) {
    packed = s.take<unsigned long long>((size_t)n + 1), d_rows = s.take<int32_t>(NN);
    d_keys = s.take<long long>(3 * R), d_first = s.take<int32_t>(R), d_count = s.take<int32_t>(R), d_nodes = s.take<esikf_map_node>(NN);
    s.begin_answers(), offs = s.take<unsigned long long>((size_t)n + 1);  // the last offset holds the totals
  };
  CK(lay_out_scratch(ctx, lay));
  // position n stays 0: the exclusive scan leaves the totals there
  CK(cudaMemsetAsync(packed, 0, ((size_t)n + 1) * sizeof(unsigned long long), st));
  map_export_count_kernel<<<ctx->sm_count * 4, 128, 0, st>>>(ctx->arena(), ctx->map_touched.p, ctx->map_work.p, packed);
  size_t tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, packed, offs, n + 1, st);
  CK(ctx->map_sort_tmp.reserve(tmp_bytes + 16));
  CK(cub::DeviceScan::ExclusiveSum(ctx->map_sort_tmp.p, tmp_bytes, packed, offs, n + 1, st));
  ctx->launches += 2;
  unsigned long long total;
  CK(read_back_to(ctx, offs + n, &total));
  const int nr = (int)(total >> 32), nn = (int)(total & 0xffffffffull);
  *n_roots = nr, *n_nodes = nn;
  if (!fill) return ESIKF_OK;
  if (nr > roots_cap || nn > nodes_cap)
    return fail(ctx, ESIKF_ERR_ARG, "map_device_export: %d roots / %d nodes do not fit the buffers (%d / %d)", nr, nn, roots_cap, nodes_cap);
  map_export_kernel<<<ctx->sm_count * 4, 128, 0, st>>>(ctx->arena(), ctx->map_touched.p, ctx->map_work.p, offs, d_keys, d_first, d_count, d_nodes, d_rows);
  ctx->launches++;
  CK(cudaGetLastError());
  // direct copies: read back through the pinned block, config 2's export (6.5 MB) took 2.0-2.1 ms a call against 1.75 ms (H100, 700 W)
  CK(cudaMemcpyAsync(keys, d_keys, (size_t)nr * 3 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(first, d_first, (size_t)nr * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(count, d_count, (size_t)nr * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(nodes, d_nodes, (size_t)nn * sizeof(esikf_map_node), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ESIKF_OK;
}

int esikf_map_device_find(esikf_ctx *ctx, const double *points, int32_t n, int32_t rule, uint8_t *status, int64_t *keys, esikf_plane *rows) {
  if (!ctx || n < 0 || (rule != ESIKF_FIND_RULE_PATCH && rule != ESIKF_FIND_RULE_RAYCAST) || (n > 0 && (!points || !status || !keys || !rows)))
    return fail(ctx, ESIKF_ERR_ARG, "map_device_find: bad argument");
  if (int rc = need(ctx, "map_device_find", IN_DEVICE_MAP | IN_MAP)) return rc;
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)n;
  MapFindArgs a;
  a.n = n, a.rule = rule;
  auto lay = [&](CallLayout &s) {
    a.pts = s.take<double>(3 * N), s.end_inputs(), s.begin_answers();
    a.rows = s.take<esikf_plane>(N), a.keys = s.take<long long>(3 * N), a.status = s.take<uint8_t>(N);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{a.pts, points, 3 * N * sizeof(double)}}));
  map_find_kernel<<<(n + FIND_THREADS - 1) / FIND_THREADS, FIND_THREADS, 0, st>>>(ctx->arena(), a);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(read_back(ctx, a.rows, a.status + N));
  copy_out(ctx, rows, a.rows, a.rows, N * sizeof(esikf_plane));
  copy_out(ctx, keys, a.rows, a.keys, 3 * N * sizeof(int64_t));
  copy_out(ctx, status, a.rows, a.status, N);
  return ESIKF_OK;
}

// pv.normal of every point of the last update (voxel_map.cpp:744: the plane that last became the point's best candidate in any
// iteration — normal_plane, not the final match; zero when there never was one): snapshotted by esikf_map_device_update
// before the records may move, otherwise gathered from the records now
__global__ void gather_normals_kernel(const int32_t *__restrict__ match_plane, const PlaneRec *__restrict__ recs, int n, double *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int m = match_plane[i];
  for (int k = 0; k < 3; k++) out[3 * (size_t)i + k] = m >= 0 ? recs[m].n[k] : 0.0;
}
int esikf_lio_fetch_normals(esikf_ctx *ctx, double *normals) {
  if (!ctx || !normals) return fail(ctx, ESIKF_ERR_ARG, "lio_fetch_normals: bad argument");
  if (int rc = need(ctx, "lio_fetch_normals", IN_MAP | IN_RUN_SCAN)) return rc;
  CK(cudaSetDevice(ctx->device));
  const int n = ctx->n_pts;
  if (n == 0) return ESIKF_OK;
  double *normal;  // not map_pt_normal: it keeps the pv list's normals for a later generate_points
  auto lay = [&](CallLayout &s) { s.begin_answers(), normal = s.take<double>((size_t)n * 3 + 4); };
  CK(lay_out_scratch(ctx, lay));
  const double *src = ctx->map_pt_normal.p;
  if (ctx->normals_n != n) {
    gather_normals_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(ctx->normal_plane.p, ctx->map.recs.p, n, normal);
    ctx->launches++;
    src = normal;
  }
  CK(read_back_to(ctx, src, normals, (size_t)n * 3));
  return ESIKF_OK;
}

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
static void lio_precompute(esikf_ctx *ctx, float dept_err, float beam_err) {
  lio_precompute_kernel<<<(ctx->n_pts + 255) / 256, 256, 0, ctx->stream>>>(ctx->pts.p, ctx->n_pts, ctx->pre.p, ctx->pre_stride, ctx->ext_dev.p, dept_err, beam_err);
  memcpy(ctx->pre_ext, ctx->ext_host, sizeof(ctx->pre_ext));
  ctx->pre_dept_err = dept_err, ctx->pre_beam_err = beam_err;
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
    if (n > 0) {
      lio_precompute(ctx, dept_err, beam_err);
      ctx->launches++;
    }
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
    if (e) cudaEventRecord(e[0], st);
    ka.init_normal = (it == 0);
    launch_lio_residual(l2_slots, grid, st, ka);
    if (e) cudaEventRecord(e[1], st);
    int rc = allreduce_info(ctx);
    if (rc) return rc;
    lio_solve_kernel<<<1, SOLVE_THREADS, 0, st>>>(sa);
    if (e) cudaEventRecord(e[2], st);
    ctx->launches += 2;
  }
  CK(cudaGetLastError());
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
    cudaMemsetAsync(&ctx->ctrl->comm_error, 0, sizeof(int), ctx->stream);
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
  expand_point_cov_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(ctx->pre.p, ctx->pre_stride, n, body_cov9 ? body : nullptr, cross_mat9 ? cross : nullptr);
  ctx->launches++;
  const double *f0 = body_cov9 ? body : cross;
  CK(read_back(ctx, f0, cross_mat9 ? cross + N9 : body_cov9 ? body + N9 : f0));
  if (body_cov9) copy_out(ctx, body_cov9, f0, body, N9 * sizeof(double));
  if (cross_mat9) copy_out(ctx, cross_mat9, f0, cross, N9 * sizeof(double));
  return ESIKF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- VIO
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
  CK(ctx->vis_pos.reserve((size_t)n * 3 + 4));
  CK(ctx->warp_patch.reserve((size_t)n * 64 * L + 64));
  CK(ctx->search_levels.reserve(n + 1));
  CK(ctx->inv_expo.reserve(n + 1));
  CK(ctx->errors.reserve(n + 1));
  cudaStream_t st = ctx->stream;
  if (n) {
    CK(cudaMemcpyAsync(ctx->vis_pos.p, pos, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->warp_patch.p, warp_patch, (size_t)n * 64 * L * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->search_levels.p, search_levels, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->inv_expo.p, inv_expo_list, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  ctx->n_patches = n, ctx->submap_levels = L;
  return ESIKF_OK;
}

static void vio_consts(const esikf_ctx *ctx, double Rci[9], double Pci[3], double Jdp_dR[9]) {
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
static void cam_dev(const esikf_ctx *ctx, CamDev &c) {
  c.model = ctx->cam.model, c.width = ctx->cam.width, c.height = ctx->cam.height;
  c.fx = ctx->cam.fx, c.fy = ctx->cam.fy, c.cx = ctx->cam.cx, c.cy = ctx->cam.cy;
  for (int i = 0; i < 5; i++) c.d[i] = ctx->cam.d[i];
}
// The camera and the camera-from-IMU extrinsics the front-end kernels project with.
static void frame_consts(const esikf_ctx *ctx, CamDev &cam, double Rci[9], double Pci[3]) {
  cam_dev(ctx, cam);
  double Jdp_dR[9];
  vio_consts(ctx, Rci, Pci, Jdp_dR);
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
    if (inverse) {  // has_ref_patch_cache = false at every level (vio.cpp:794): H_sub_inv of this level's tap stride
      vio_inverse_precompute_kernel<<<(ka.count + 7) / 8, 256, 0, st>>>(ka, iv, level);
      ctx->launches++;
    }
    for (int it = 0; it < ctx->vio_cfg.max_iterations; it++, slot++) {
      ka.level = level, ka.slot_iter = it;
      cudaEvent_t *e = ctx->timing ? timing_events(ctx, EV_VIO_BASE, slot) : nullptr;
      if (e) cudaEventRecord(e[0], st);
      if (inverse)
        vio_inverse_patch_kernel<<<grid, VIO_THREADS, sizeof(VioSmem), st>>>(ka, iv);
      else
        vio_patch_kernel<<<grid, VIO_THREADS, sizeof(VioSmem), st>>>(ka);
      if (e) cudaEventRecord(e[1], st);
      int rc = allreduce_info(ctx);
      if (rc) return rc;
      sa.level = level, sa.slot_iter = it, sa.last_slot = (level == 0 && it == ctx->vio_cfg.max_iterations - 1);
      vio_solve_kernel<<<1, SOLVE_THREADS, 0, st>>>(sa);
      if (e) cudaEventRecord(e[2], st);
      ctx->launches += 2;
    }
  }
  CK(cudaGetLastError());
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
  image_patch_kernel<<<(n * 64 + 255) / 256, 256, 0, ctx->stream>>>(ctx->img.p, ctx->img_w, ctx->img_h, pc_d, n, level, patch);
  ctx->launches++;
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
    if (ref_img_index[i] < 0 || ref_img_index[i] >= (int)ctx->ref_imgs.size()) return fail(ctx, ESIKF_ERR_ARG, "warp_patches: ref image index %d", ref_img_index[i]);
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
  CK(ctx->search_levels.reserve(n + 1));
  CK(ctx->warp_patch.reserve(N * 64 * L + 64));
  const std::vector<double> one(keep_on_device ? N : 0, 1.0);
  CK(upload(ctx, {{ones, one.data(), one.size() * sizeof(double)}, {ref_idx, ref_img_index, N * sizeof(int32_t)}, {px, px_ref, N * 2 * sizeof(double)},
                  {pos, pos_w, N * 3 * sizeof(double)}, {normal, normal_w, N * 3 * sizeof(double)}, {T_ref, T_ref_w, N * 12 * sizeof(double)},
                  {T_cur, T_cur_w, 12 * sizeof(double)}}));
  CamDev cam;
  cam_dev(ctx, cam);
  warp_matrix_kernel<<<(n + 127) / 128, 128, 0, st>>>(cam, n, px, pos, normal, T_ref, T_cur, A, ctx->search_levels.p);
  CK(cudaMemsetAsync(ctx->warp_patch.p, 0, N * 64 * L * sizeof(float), st));
  warp_affine_kernel<<<(n * L * 64 + 255) / 256, 256, 0, st>>>(ctx->ref_img_ptrs.p, ref_idx, ctx->ref_w, ctx->ref_h, n, L, A, px, ctx->search_levels.p,
                                                              ctx->warp_patch.p);
  ctx->launches += 2;
  if (search_level_out) CK(cudaMemcpyAsync(levels, ctx->search_levels.p, N * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  if (warp_patch_out) CK(cudaMemcpyAsync(warp, ctx->warp_patch.p, N * 64 * L * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (keep_on_device) {
    // install as the visual sub-map of the coming update: pos = pos_w, inv_expo filled by the caller through set_patches otherwise
    CK(ctx->vis_pos.reserve((size_t)n * 3 + 4));
    CK(ctx->inv_expo.reserve(n + 1));
    CK(ctx->errors.reserve(n + 1));
    CK(cudaMemcpyAsync(ctx->vis_pos.p, pos, N * 3 * sizeof(double), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(ctx->inv_expo.p, ones, N * sizeof(double), cudaMemcpyDeviceToDevice, st));
  }
  CK(read_back(ctx, A, warp_patch_out ? (const void *)(warp + N * 64 * L) : search_level_out ? (const void *)(levels + N) : (const void *)(A + 4 * N)));
  if (keep_on_device) ctx->n_patches = n, ctx->submap_levels = L;
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
    if (ref_img_index[i] < 0 || ref_img_index[i] >= (int)ctx->ref_imgs.size()) return fail(ctx, ESIKF_ERR_ARG, "select_patches: ref image index %d", ref_img_index[i]);
    if (!homography && (ref_level[i] < 0 || ref_level[i] > 8)) return fail(ctx, ESIKF_ERR_ARG, "select_patches: ref level %d", ref_level[i]);
  }
  CK(cudaSetDevice(ctx->device));
  const int L = ctx->vio_cfg.patch_pyrimid_level;
  cudaStream_t st = ctx->stream;
  // every argument check is above: from here on the call replaces the installed sub-map
  CK(ctx->vis_pos.reserve((size_t)n * 3 + 4));
  CK(ctx->warp_patch.reserve((size_t)n * 64 * L + 64));
  CK(ctx->search_levels.reserve(n + 1));
  CK(ctx->inv_expo.reserve(n + 1));
  CK(ctx->errors.reserve(n + 1));
  *n_kept = 0;
  if (n == 0) return ctx->n_patches = 0, ctx->submap_levels = L, ESIKF_OK;
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
    warp_matrix_kernel<<<(n + 127) / 128, 128, 0, st>>>(cam, n, d_px, d_pos, d_nrm, d_T, d_Tc, d_A, d_sl);
  else
    warp_matrix_depth_kernel<<<(n + 127) / 128, 128, 0, st>>>(cam, n, d_px, d_f, d_rp, d_pos, d_T, d_Tc, d_lvl, d_key, d_A, d_sl);
  // patch_wrap is a fresh zero vector per candidate (:646): a NaN inverse leaves it zero (:297-301)
  CK(cudaMemsetAsync(d_warp, 0, N * 64 * L * sizeof(float), st));
  warp_affine_kernel<<<(n * L * 64 + 255) / 256, 256, 0, st>>>(ctx->ref_img_ptrs.p, d_idx, ctx->ref_w, ctx->ref_h, n, L, d_A, d_px, d_sl, d_warp);
  SelectGateArgs ga;
  ga.img = ctx->img.p, ga.width = ctx->img_w, ga.height = ctx->img_h, ga.n = n, ga.levels = L, ga.ncc_en = cfg->ncc_en != 0;
  ga.pc = d_pc, ga.warp = d_warp, ga.ref_inv_expo = d_ie;
  ga.cur_inv_expo = inv_expo_time, ga.ncc_thre = cfg->ncc_thre, ga.outlier_threshold = cfg->outlier_threshold;
  ga.error = d_err, ga.keep = d_keep;
  select_gate_kernel<<<(n + SELECT_GATE_WARPS - 1) / SELECT_GATE_WARPS, 32 * SELECT_GATE_WARPS, 0, st>>>(ga);
  select_scan_kernel<<<1, SELECT_SCAN_THREADS, 0, st>>>(d_keep, n, d_dst, d_nk);
  SelectScatterArgs sa;
  sa.n = n, sa.levels = L, sa.keep = d_keep, sa.dst = d_dst, sa.search_level = d_sl, sa.pos_w = d_pos, sa.ref_inv_expo = d_ie, sa.A = d_A;
  sa.warp = d_warp, sa.error = d_err;
  sa.vis_pos = ctx->vis_pos.p, sa.inv_expo = ctx->inv_expo.p, sa.A_kept = d_Akept, sa.warp_patch = ctx->warp_patch.p, sa.errors = ctx->errors.p;
  sa.search_levels = ctx->search_levels.p, sa.kept_index = d_kept;
  select_scatter_kernel<<<(n + 7) / 8, 256, 0, st>>>(sa);
  ctx->launches += 5;
  CK(cudaGetLastError());
  int32_t nk;
  CK(read_back_to(ctx, d_nk, &nk));
  ctx->n_patches = nk, ctx->submap_levels = L;
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
    if (ref_img_index[i] < 0 || ref_img_index[i] >= (int)ctx->ref_imgs.size()) return fail(ctx, ESIKF_ERR_ARG, "set_inverse_refs: ref image index %d", ref_img_index[i]);
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
    if (ref_img_index[i] < 0 || ref_img_index[i] >= (int)ctx->ref_imgs.size()) return fail(ctx, ESIKF_ERR_ARG, "warp_affine: ref image index %d", ref_img_index[i]);
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
  warp_affine_kernel<<<(n * L * 64 + 255) / 256, 256, 0, st>>>(ctx->ref_img_ptrs.p, ref_idx, ctx->ref_w, ctx->ref_h, n, L, A, px, levels, out);
  ctx->launches += 1;
  CK(cudaGetLastError());
  CK(read_back_to(ctx, out, warp_patch_out, N * 64 * L));
  return ESIKF_OK;
}

// ---------------------------------------------------------------------------------------------------------------- coloured scan
// The device copy of the state a call projects with: a packed host state staged into scratch_state, or (state == NULL) the
// posterior resident on the device, which must be the one an update of kind `want` left there.
static int state_or_posterior(esikf_ctx *ctx, const double *state, esikf_ctx::Resident want, const char *what, const double **out) {
  if (!state && ctx->resident != want)
    return fail(ctx, ESIKF_ERR_STATE, "%s(state = NULL): the device holds no %s posterior", what, want == esikf_ctx::RESIDENT_LIO ? "LIO" : "VIO");
  if (!state) return *out = ctx->state, ESIKF_OK;
  CK(ctx->scratch_state.reserve(S_N));
  CK(cudaMemcpyAsync(ctx->scratch_state.p, state, S_N * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  *out = ctx->scratch_state.p;
  return ESIKF_OK;
}

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
    rgb_world_kernel<<<(n + 255) / 256, 256, 0, st>>>(a);
    ctx->launches++;
    CK(cudaGetLastError());
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
  if (n > 0) cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, (int32_t *)nullptr, (int32_t *)nullptr, n + 1, st);
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
    rgb_color_kernel<<<(n + 1 + 255) / 256, 256, 0, st>>>(a);
    CK(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, keep, dst, n + 1, st));
    rgb_scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(keep, dst, n, ctx->rgb_cloud.p, color, xyz, bgr_kept, index);
    ctx->launches += 4;
    CK(cudaGetLastError());
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
  gen_score_kernel<<<(n + n_add + GEN_THREADS - 1) / GEN_THREADS, GEN_THREADS, 0, st>>>(a);
  gen_cells_kernel<<<(L + 255) / 256, 256, 0, st>>>(a.key, L, d_keep);
  select_scan_kernel<<<1, SELECT_SCAN_THREADS, 0, st>>>(d_keep, L, d_dst, d_nk);
  gen_scatter_kernel<<<(L + GEN_THREADS - 1) / GEN_THREADS, GEN_THREADS, 0, st>>>(a, d_keep, d_dst, o);
  ctx->launches += 4;
  CK(cudaGetLastError());
  int32_t nk = 0;
  CK(cudaMemcpyAsync(&nk, d_nk, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));  // also: the caller may reuse its buffers on return
  *n_out = nk;
  if (nk > cap) return fail(ctx, ESIKF_ERR_ARG, "vio_generate_points: %d new points, room for %d", nk, cap);
  if (nk == 0) return ESIKF_OK;
  if (patch_out) {
    image_patch_kernel<<<(nk * 64 + 255) / 256, 256, 0, st>>>(ctx->img.p, ctx->img_w, ctx->img_h, o.pc, nk, 0, d_patch);
    ctx->launches++;
    CK(cudaGetLastError());
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
  cudaStream_t st = ctx->stream;
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
  obs_flag_kernel<<<(n + OBS_THREADS - 1) / OBS_THREADS, OBS_THREADS, 0, st>>>(a);
  select_scan_kernel<<<1, SELECT_SCAN_THREADS, 0, st>>>(d_keep, n, d_dst, d_nk);
  obs_scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_keep, d_dst, a.pc, n, d_entry, out_pc);
  ctx->launches += 3;
  CK(cudaGetLastError());
  int32_t nk;
  CK(read_back_to(ctx, d_nk, &nk));
  *n_out = nk;
  if (nk > cap) return fail(ctx, ESIKF_ERR_ARG, "vio_update_points: %d new observations, room for %d", nk, cap);
  const size_t K = (size_t)nk;
  if (nk > 0 && patch_out) {
    image_patch_kernel<<<(nk * 64 + 255) / 256, 256, 0, st>>>(ctx->img.p, ctx->img_w, ctx->img_h, out_pc, nk, 0, patch);
    ctx->launches++;
    CK(cudaGetLastError());
  }
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
  cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, n, 0, 63, st);
  cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int32_t *)nullptr, (int32_t *)nullptr, n + 1, st);
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
  if (n > 0) ret_scan_kernel<<<(n + RET_THREADS - 1) / RET_THREADS, RET_THREADS, 0, st>>>(a);
  ret_depth_kernel<<<(int)((npix + 255) / 256), 256, 0, st>>>(a.win, a.depth_pt, (int)npix, ctx->ret_depth.p);
  ctx->launches += n > 0 ? 2 : 1;
  int32_t counts[2] = {0, 0};  // distinct keys, bad
  if (n > 0) {
    CK(cub::DeviceRadixSort::SortPairs(tmp, sort_bytes, a.key, k_out, a.idx, i_out, n, 0, 63, st));
    ret_head_kernel<<<(n + 1 + 255) / 256, 256, 0, st>>>(k_out, i_out, n, d_head);
    CK(cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, d_head, d_dst, n + 1, st));
    ret_keys_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_head, d_dst, a.key, n, d_keys);
    ctx->launches += 4;  // sort passes counted as one
  }
  CK(cudaGetLastError());
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
  cudaStream_t st = ctx->stream;
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
  ret_depth_check_kernel<<<(n + RET_THREADS - 1) / RET_THREADS, RET_THREADS, 0, st>>>(a);
  ctx->launches++;
  CK(cudaGetLastError());
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
  refpatch_score_kernel<<<(n + RP_WARPS - 1) / RP_WARPS, RP_WARPS * 32, 0, st>>>(a, RpPacked{d_first});
  ctx->launches++;
  CK(cudaGetLastError());
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
  vmap_pack_kernel<<<(n + VMAP_WARPS - 1) / VMAP_WARPS, VMAP_WARPS * 32, 0, st>>>(a);
  ctx->launches++;
  CK(cudaGetLastError());
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
  cudaStream_t st = ctx->stream;
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
  vmap_last_kernel<<<(n + 255) / 256, 256, 0, st>>>(e.s, d_pid, n, last_T, last_px);
  frame_consts(ctx, a.cam, a.Rci, a.Pci);
  a.state = dev_state, a.pos = ctx->vis_pos.p, a.converged = conv, a.last_T = last_T, a.last_px = last_px;
  a.n = n, a.cos_max = cos_max, a.keep = d_keep;
  obs_flag_kernel<<<(n + OBS_THREADS - 1) / OBS_THREADS, OBS_THREADS, 0, st>>>(a);
  select_scan_kernel<<<1, SELECT_SCAN_THREADS, 0, st>>>(d_keep, n, d_dst, d_nk);
  obs_scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_keep, d_dst, a.pc, n, d_entry, out_pc);
  ctx->launches += 4;
  CK(cudaGetLastError());
  int32_t nk;
  CK(read_back_to(ctx, d_nk, &nk));
  *n_out = nk;
  // the store is edited only once the answers fit: a call refused here can be repeated with a larger cap
  if (nk > cap) return fail(ctx, ESIKF_ERR_ARG, "vmap_update_points: %d new observations, room for %d", nk, cap);
  if (nk > 0) image_patch_kernel<<<(nk * 64 + 255) / 256, 256, 0, st>>>(ctx->img.p, ctx->img_w, ctx->img_h, out_pc, nk, 0, patch);
  e.pid = d_pid, e.dst = d_dst, e.new_pc = out_pc, e.new_patch = patch, e.T_f_w = T_f_w ? d_Tnew : nullptr, e.frame_id = frame_id;
  e.evicted = d_evicted, e.count = d_count;
  vmap_edit_kernel<<<(n + VMAP_WARPS - 1) / VMAP_WARPS, VMAP_WARPS * 32, 0, st>>>(e);
  ctx->launches += nk > 0 ? 2 : 1;
  CK(cudaGetLastError());
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
  cudaStream_t st = ctx->stream;
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
  refpatch_score_kernel<<<(n + RP_WARPS - 1) / RP_WARPS, RP_WARPS * 32, 0, st>>>(a, RpStore{d_pid, v.count, v.ref});
  ctx->launches++;
  if (score_out || mean_out) {
    vmap_rows_kernel<<<(n * VMAP_SLOTS + 255) / 256, 256, 0, st>>>(v, d_pid, n, nullptr, d_score, d_mean);
    ctx->launches++;
  }
  CK(cudaGetLastError());
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
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)n;
  VmapChooseArgs a;
  int32_t *d_pid;
  double *d_pos;
  auto lay = [&](CallLayout &s) { d_pid = s.take<int32_t>(N), d_pos = s.take<double>(3 * N), s.end_inputs(), s.begin_answers(), a.ref = s.take<int32_t>(N); };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{d_pid, point_id, N * sizeof(int32_t)}, {d_pos, pos, 3 * N * sizeof(double)}}));
  a.s = vmap_of(ctx), a.pid = d_pid, a.pos = d_pos, a.n = n, a.normal_en = normal_en != 0;
  for (int k = 0; k < 3; k++) a.frame_pos[k] = frame_pos ? frame_pos[k] : 0.0;
  vmap_choose_kernel<<<(n + VMAP_WARPS - 1) / VMAP_WARPS, VMAP_WARPS * 32, 0, st>>>(a);
  ctx->launches++;
  CK(cudaGetLastError());
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
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)n;
  int32_t *d_pid, *d_count;
  auto lay1 = [&](CallLayout &s) { d_pid = s.take<int32_t>(N), s.end_inputs(), s.begin_answers(), d_count = s.take<int32_t>(N); };
  CK(lay_out_scratch(ctx, lay1));
  CK(upload(ctx, {{d_pid, point_id, N * sizeof(int32_t)}}));
  const VmapView v = vmap_of(ctx);
  vmap_rows_kernel<<<(n * VMAP_SLOTS + 255) / 256, 256, 0, st>>>(v, d_pid, n, d_count, nullptr, nullptr);
  ctx->launches++;
  CK(cudaGetLastError());
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
  vmap_pack_kernel<<<(n + VMAP_WARPS - 1) / VMAP_WARPS, VMAP_WARPS * 32, 0, st>>>(a);
  ctx->launches++;
  CK(cudaGetLastError());
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
  vpl_key_kernel<<<(n + 255) / 256, 256, 0, st>>>(a);
  vpl_commit_kernel<<<(n + 255) / 256, 256, 0, st>>>(a);  // writes nothing when a key was out of range
  ctx->launches += 2;
  CK(cudaGetLastError());
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
  vrt_hash_kernel<<<(n_keys + 255) / 256, 256, 0, st>>>(d_keys, n_keys, table, (int32_t *)a.wrank, T - 1);
  CamDev cam;
  frame_consts(ctx, cam, a.Rci, a.Pci);
  memcpy(a.Rci, ctx->ret_Rci, sizeof(a.Rci)), memcpy(a.Pci, ctx->ret_Pci, sizeof(a.Pci));  // the scan call's
  a.cam = cam, a.state = ctx->ret_state.p, a.v = vpl_view(ctx->vpl.p, (size_t)ctx->vpl_cap), a.count = vmap_of(ctx).count, a.n_pts = (int)ctx->vpl_hi;
  a.wkey = table, a.wmask = T - 1, a.grid_size = grid_size, a.grid_n_width = grid_n_width, a.length = L, a.border = border, a.frame_pos = fpos;
  vrt_init_kernel<<<(L + 255) / 256, 256, 0, st>>>(a);
  const int pb = (a.n_pts + VRT_THREADS - 1) / VRT_THREADS;
  vrt_walk_kernel<0><<<pb, VRT_THREADS, 0, st>>>(a);
  vrt_walk_kernel<1><<<pb, VRT_THREADS, 0, st>>>(a);
  vrt_walk_kernel<2><<<pb, VRT_THREADS, 0, st>>>(a);
  DepthCheckArgs dc;  // K11's check on every cell's winner (a cell without one is not read)
  memcpy(dc.Rci, ctx->ret_Rci, sizeof(dc.Rci)), memcpy(dc.Pci, ctx->ret_Pci, sizeof(dc.Pci));
  dc.state = ctx->ret_state.p, dc.pos = a.wpos, dc.pc = a.pc, dc.n = L, dc.width = W, dc.height = H, dc.depth = ctx->ret_depth.p, dc.flag = disc;
  ret_depth_check_kernel<<<(L + RET_THREADS - 1) / RET_THREADS, RET_THREADS, 0, st>>>(dc);
  c.length = L, c.type = a.type, c.disc = disc, c.ninit = a.v.ninit, c.win = a.win, c.pc = a.pc, c.wpos = a.wpos;
  vrt_cells_kernel<true><<<(L + 255) / 256, 256, 0, st>>>(c);
  select_scan_kernel<<<1, SELECT_SCAN_THREADS, 0, st>>>(c.keep, L, c.dst, cnt);
  select_scan_kernel<<<1, SELECT_SCAN_THREADS, 0, st>>>(c.skeep, L, c.sdst, cnt + 1);
  vrt_cells_kernel<false><<<(L + 255) / 256, 256, 0, st>>>(c);
  ctx->launches += 10;
  CK(cudaGetLastError());
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
    vmap_choose_kernel<<<(ns + VMAP_WARPS - 1) / VMAP_WARPS, VMAP_WARPS * 32, 0, st>>>(ca);
    vrt_refs_kernel<<<(ns + 255) / 256, 256, 0, st>>>(ref_tmp, c.sat, ns, c.ref_out, c.status_out);
    ctx->launches += 2;
    CK(cudaGetLastError());
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
    if (which == 0) launch_lio_residual(lio_use_l2_slots(la.count, grid), grid, st, la);
    else if (which == 1) lio_solve_kernel<<<1, SOLVE_THREADS, 0, st>>>(sa);
    else if (which == 2) vio_patch_kernel<<<grid, VIO_THREADS, sizeof(VioSmem), st>>>(va);
    else lio_precompute(ctx, (float)ctx->lio_cfg.dept_err, (float)ctx->lio_cfg.beam_err);
    CK(cudaEventRecord(e1, st));
    CK(cudaEventSynchronize(e1));
    ctx->launches++;
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (r >= 3) total += ms;
  }
  CK(cudaGetLastError());
  *avg_ms = (float)(total / reps);
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
