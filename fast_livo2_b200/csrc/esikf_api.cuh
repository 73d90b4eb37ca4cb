// What the host files of the C ABI (include/esikf_b200.h) share: the context and the resources it owns, the status and
// precondition helpers, the staging of a call's inputs and answers, and the kernels launched from more than one of them.
//   esikf_api_ctx.cu    : context, setters, multi-GPU, phase stamps and kernel timing; the helpers declared here
//   esikf_api_update.cu : LIO / VIO set, run and fetch, the patch producers, esikf_profile_kernel
//   esikf_api_map.cu    : host-uploaded and device-resident voxel map, find_correspond, lio_fetch_normals
//   esikf_api_front.cu  : colouring, new points and observations, retrieval, reference patches, observation store
// No CPU fallback: every entry point fails with a status code when the device or an input is missing.
#pragma once
#include <dlfcn.h>
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <initializer_list>
#include <string>
#include <utility>
#include <vector>

#include "esikf_dev.cuh"
#include "esikf_map.cuh"
#include "esikf_vio.cuh"
#include "scratch_layout.hpp"

namespace esikf {
// Kernels launched from more than one host file, defined once in the kernel file named.
__global__ void plane_compact_kernel(const esikf_plane *__restrict__ planes, const int32_t *__restrict__ ids, int n, PlaneRec *__restrict__ recs);  // esikf_lio.cu
__global__ void image_patch_kernel(const uint8_t *__restrict__ img, int width, int height, const double *__restrict__ pc, int n, int level,
                                   float *__restrict__ out);  // esikf_vio.cu
__global__ void select_scan_kernel(const int32_t *__restrict__ keep, int n, int32_t *__restrict__ dst, int32_t *__restrict__ n_kept);  // esikf_vio.cu
}  // namespace esikf

using namespace esikf;

// The helpers below are shared by the host files only: kept out of the library's export table, as static functions were.
#define ESIKF_HIDDEN __attribute__((visibility("hidden")))

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
extern ESIKF_HIDDEN NcclApi g_nccl;  // esikf_api_ctx.cu
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
  // hidden: where the compiler does not inline it, the copy it emits stays out of the library's export table
  ESIKF_HIDDEN cudaError_t reserve(uint32_t hash_cap_, int node_cap_, int rec_cap_, long long pool_cap_) {
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

ESIKF_HIDDEN int fail(esikf_ctx *c, int code, const char *fmt, ...);
#define CK(call)                                                                                                   \
  do {                                                                                                             \
    cudaError_t e__ = (call);                                                                                      \
    if (e__ != cudaSuccess) return fail(ctx, ESIKF_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

// The one launch path of the entry points' kernels: `kernel` on the context's stream, its launch error returned, and one
// launch added to esikf_launch_count once it is enqueued. Only launch_persistent's cooperative launch goes another way.
// cudaGetLastError() also returns an error an earlier runtime call left, so every runtime call on an entry point's path is
// checked (CK) or has its error cleared where it is handled: the error returned here is this launch's.
template <typename... P, typename... A>
static cudaError_t launch(esikf_ctx *ctx, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A &&...args) {
  kernel<<<grid, block, smem, ctx->stream>>>(std::forward<A>(args)...);
  const cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) ctx->launches++;
  return e;
}
// A CUB device-wide call: whatever number of kernels it runs, it counts as one launch.
static inline cudaError_t counted(esikf_ctx *ctx, cudaError_t e) { return e == cudaSuccess ? (ctx->launches++, e) : e; }

// The inputs of the context's groups (esikf_ctx), one bit each.
enum Input : unsigned {
  IN_EXT = 1u << 0, IN_CAMERA = 1u << 1, IN_IMAGE = 1u << 2, IN_SUBMAP = 1u << 3, IN_INV_REFS = 1u << 4, IN_REF_IMAGES = 1u << 5,
  IN_SCAN = 1u << 6, IN_RUN_SCAN = 1u << 7, IN_MAP = 1u << 8, IN_HOST_MAP = 1u << 9, IN_DEVICE_MAP = 1u << 10, IN_EXPORT = 1u << 11,
  IN_PV_LIST = 1u << 12, IN_NORMALS = 1u << 13, IN_CLOUD = 1u << 14, IN_RETRIEVAL = 1u << 15, IN_STORE = 1u << 16, IN_POSTERIOR = 1u << 17,
};

// The one check of each input: ESIKF_ERR_STATE naming `call` and the first of `inputs` missing (the posterior: state_or_posterior).
ESIKF_HIDDEN int need(esikf_ctx *ctx, const char *call, unsigned inputs);

// The one way to void an input; the table at esikf_ctx says when. A voided device map stays reachable to map_device_* calls.
ESIKF_HIDDEN void void_inputs(esikf_ctx *ctx, unsigned inputs);

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
ESIKF_HIDDEN cudaError_t upload(esikf_ctx *ctx, std::initializer_list<HostIn> in);

// The one readback of answers that lie between the device addresses `first` and `end`: a copy into the pinned block and a
// synchronisation. copy_out then hands them to the caller, whose buffers a failed call thus leaves untouched.
ESIKF_HIDDEN cudaError_t read_back(esikf_ctx *ctx, const void *first, const void *end);
ESIKF_HIDDEN void copy_out(const esikf_ctx *ctx, void *dst, const void *first, const void *src, size_t bytes);
// The same for k answers of one array at p, or a count the rest of the call depends on, straight into out.
template <typename T> static cudaError_t read_back_to(esikf_ctx *ctx, const T *p, T *out, size_t k = 1) {
  const cudaError_t e = read_back(ctx, p, p + k);
  if (e == cudaSuccess) copy_out(ctx, out, p, p, k * sizeof(T));
  return e;
}

enum { EV_LIO_BASE = 0, EV_VIO_BASE = 8 };  // esikf_ctx::ev: the LIO update's timing slots, then the VIO update's
ESIKF_HIDDEN void shard_of(int n, int rank, int nranks, int &begin, int &count);

// The persistent update kernels' grid mailbox and LIO lane slots, their shared memory and how many CTAs of each an SM holds
// (esikf_api_update.cu, run by esikf_create).
ESIKF_HIDDEN cudaError_t update_kernels_setup(esikf_ctx *ctx);

// The device copy of the state a call projects with: a packed host state staged into scratch_state, or (state == NULL) the
// posterior resident on the device, which must be the one an update of kind `want` left there.
ESIKF_HIDDEN int state_or_posterior(esikf_ctx *ctx, const double *state, esikf_ctx::Resident want, const char *what, const double **out);

ESIKF_HIDDEN void vio_consts(const esikf_ctx *ctx, double Rci[9], double Pci[3], double Jdp_dR[9]);
ESIKF_HIDDEN void cam_dev(const esikf_ctx *ctx, CamDev &c);
// The camera and the camera-from-IMU extrinsics the front-end kernels project with.
ESIKF_HIDDEN void frame_consts(const esikf_ctx *ctx, CamDev &cam, double Rci[9], double Pci[3]);
