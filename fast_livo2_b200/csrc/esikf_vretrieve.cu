// The map side of the visual sub-map retrieval, K15 (H100, sm_90a): the visual points placed in their 0.5 m voxels as
// VIOManager::insertPointIntoVoxelMap places them (reference src/vio.cpp:227-250), and the walk of retrieveFromVisualSparseMap
// over them (:438-484): per grid cell the nearest point in view. The depth check (:614-640, ret_depth_check_kernel) and the
// reference-feature choice (:651-697, vmap_choose_kernel) run after it unchanged.
//
// The device feat_map is kept per point: its packed voxel key (patch_voxel_key, the insertion rule: the double quotient
// narrowed to float, one less when negative, truncated) and its placement sequence number. A voxel's voxel_points list is its
// points in placement order, because the reference only ever appends to it and never removes from it; so (key, sequence) is
// a point's voxel and its position in that voxel's list. The walk is then one pass over the placed points, each finding its
// voxel among the walk's keys (a hash of the keys built per call, key -> rank in the walk order).
//
//   vpl_key_kernel    : per new point, its packed voxel key; a flag when a key leaves [-2^20, 2^20)
//   vpl_commit_kernel : per new point, pos_, key, sequence and is_normal_initialized_ into the point arrays, unless flagged
//   vrt_hash_kernel   : the walk keys into an open-addressing table (linear probing) with their rank in the walk order
//   vrt_init_kernel   : per grid cell: not TYPE_MAP, map_dist 10000.0f, no winner
//   vrt_walk_kernel<P>: per placed point, three passes over the same candidates (obs_ count > 0, a walk voxel, dir[2] >= 0,
//                       isInFrame(pc.cast<int>(), border)): P0 marks the cell TYPE_MAP and takes the atomicMin of the float
//                       distance's bits (distances are >= 0, so the bits order as the floats; NaN and > 10000 never take part);
//                       P1, among the points at that minimum, the atomicMax of (walk rank, sequence): the point the serial
//                       `cur_dist <= map_dist` leaves last; P2 writes that point's id, pc and pos_ to its cell
//   vrt_cells_kernel  : per cell: TYPE_MAP flags for the compaction, then (after it) the answers in cell order, the status of
//                       the skips and the survivors for the choice
//   vrt_refs_kernel   : each survivor's chosen reference back to its cell
//
// Every double is single-rounded in the reference's operation order (Rn), as in K11: with a pinhole camera the answers are
// the host's bit for bit; the fisheye projection calls atan (DESIGN.md §4). No result depends on the launch geometry or the
// order in which threads run.

namespace esikf {

#define VRT_THREADS 256

enum { VRT_KEPT = 0, VRT_DEPTH = 1, VRT_NOT_INIT = 2, VRT_NO_REF = 3, VRT_NO_WINNER = 4 };

// the point arrays of the device feat_map, one allocation of `cap` points
struct VplView {
  double *pos;             // [cap][3] VisualPoint::pos_
  unsigned long long *key; // [cap] packed voxel key, ESIKF_KEY_EMPTY while the point is not placed
  int32_t *seq;            // [cap] placement order
  uint8_t *ninit;          // [cap] is_normal_initialized_
};
static inline size_t vpl_bytes(size_t cap) { return cap * (3 * 8 + 8 + 4 + 1); }
static inline VplView vpl_view(uint8_t *b, size_t cap) {
  VplView v;
  v.pos = (double *)b, v.key = (unsigned long long *)(v.pos + 3 * cap), v.seq = (int32_t *)(v.key + cap), v.ninit = (uint8_t *)(v.seq + cap);
  return v;
}

struct VplArgs {
  VplView v;
  const int32_t *pid;     // [n]
  const double *pos;      // [n][3]
  const uint8_t *ninit;   // [n] or NULL (all initialised)
  int n;
  int32_t seq0;           // the sequence number of the call's first point
  unsigned long long *key;
  int32_t *bad;
};

__global__ void vpl_key_kernel(const VplArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  long long k[3];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 3; j++) ok = patch_voxel_key(a.pos[3 * (size_t)i + j], k[j]) && ok;
  if (!ok) atomicOr(a.bad, 1);
  a.key[i] = ok ? pack_key(k[0], k[1], k[2]) : 0ull;
}

__global__ void vpl_commit_kernel(const VplArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n || *a.bad) return;
  const size_t p = (size_t)a.pid[i];
  for (int j = 0; j < 3; j++) a.v.pos[3 * p + j] = a.pos[3 * (size_t)i + j];
  a.v.key[p] = a.key[i], a.v.seq[p] = a.seq0 + i, a.v.ninit[p] = a.ninit ? (a.ninit[i] != 0) : 1;
}

__global__ void vrt_hash_kernel(const int32_t *__restrict__ keys, int n, unsigned long long *table, int32_t *rank, uint32_t mask) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = pack_key(keys[3 * i], keys[3 * i + 1], keys[3 * i + 2]);
  for (uint32_t h = hash_key(k) & mask;; h = (h + 1) & mask)
    if (atomicCAS(table + h, ESIKF_KEY_EMPTY, k) == ESIKF_KEY_EMPTY) {  // every key is different (checked by the caller)
      rank[h] = i;
      return;
    }
}

struct VrtArgs {
  CamDev cam;
  double Rci[9], Pci[3];
  const double *state;                 // the packed state of the scan call's frame pose
  VplView v;
  const int32_t *count;                // the observation store's obs_ counts
  int n_pts;                           // point ids below this may be placed
  const unsigned long long *wkey;      // the walk's hash table
  const int32_t *wrank;
  uint32_t wmask;
  int grid_size, grid_n_width, length, border;
  uint8_t *type;                       // [length] TYPE_MAP
  uint32_t *dist;                      // [length] bits of map_dist
  unsigned long long *tie;             // [length] (rank + 1) << 32 | sequence of the winner
  int32_t *win;                        // [length] the winner's point id, -1 none
  double *pc, *wpos;                   // [length][2], [length][3] its pc and pos_
  double *frame_pos;                   // [3] out: Frame::pos() of the pose
};

// The walk's test of point p (:446-472): its rank in the walk, cell, float distance and pc; false when it is no candidate.
__device__ __forceinline__ bool vrt_candidate(const VrtArgs &a, const double *Rcw, const double *Pcw, const double *fp, int p, int &rank, int &cell, float &d,
                                              Rn &u, Rn &v) {
  const unsigned long long k = a.v.key[p];
  if (k == ESIKF_KEY_EMPTY) return false;
  rank = -1;
  for (uint32_t h = hash_key(k) & a.wmask;; h = (h + 1) & a.wmask) {
    const unsigned long long w = a.wkey[h];
    if (w == ESIKF_KEY_EMPTY) break;
    if (w == k) {
      rank = a.wrank[h];
      break;
    }
  }
  if (rank < 0 || a.count[p] <= 0) return false;
  const double *q = a.v.pos + 3 * (size_t)p;
  Rn pf[3];
  frame_point(Rcw, Pcw, Rn(q[0]), Rn(q[1]), Rn(q[2]), pf);
  if (pf[2].v < 0) return false;  // dir[2] < 0
  world2cam(a.cam, pf[0], pf[1], pf[2], u, v);
  // pc.cast<int>(), as ret_scan_kernel: NaN fails the host's test (INT_MIN) and is rejected here
  if (u.v != u.v || v.v != v.v) return false;
  const int ui = (int)u.v, vi = (int)v.v;
  if (!(ui >= a.border && ui < a.cam.width - a.border && vi >= a.border && vi < a.cam.height - a.border)) return false;
  const Rn gs = (double)a.grid_size;
  cell = (int)(v / gs).v * a.grid_n_width + (int)(u / gs).v;
  if (cell < 0 || cell >= a.length) return false;  // not reached: the caller's grid covers every pixel isInFrame passes
  // (new_frame_->pos() - pos_).norm() narrowed to float
  const Rn o0 = Rn(fp[0]) - Rn(q[0]), o1 = Rn(fp[1]) - Rn(q[1]), o2 = Rn(fp[2]) - Rn(q[2]);
  d = __double2float_rn(sqrt((o0 * o0 + o1 * o1 + o2 * o2).v));
  return true;
}

template <int PASS> __global__ void __launch_bounds__(VRT_THREADS) vrt_walk_kernel(const VrtArgs a) {
  __shared__ double Rcw[9], Pcw[3], fp[3];
  ret_frame_pose(a.Rci, a.Pci, a.state, Rcw, Pcw);
  // Frame::pos() = T_f_w_.inverse().translation() = (R^T t) * -1.0, each row of R^T t summed left to right
  if (threadIdx.x < 3) {
    const int r = threadIdx.x;
    fp[r] = (-(Rn(Rcw[r]) * Rn(Pcw[0]) + Rn(Rcw[3 + r]) * Rn(Pcw[1]) + Rn(Rcw[6 + r]) * Rn(Pcw[2]))).v;
    if (PASS == 0 && blockIdx.x == 0) a.frame_pos[r] = fp[r];
  }
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n_pts) return;
  int rank, cell;
  float d;
  Rn u, v;
  if (!vrt_candidate(a, Rcw, Pcw, fp, p, rank, cell, d, u, v)) return;
  if (PASS == 0) a.type[cell] = 1;
  if (!(d <= 10000.0f)) return;  // map_dist starts at 10000.0f; NaN never passes `cur_dist <= map_dist`
  const uint32_t bits = __float_as_uint(d);
  if (PASS == 0) {
    atomicMin(a.dist + cell, bits);
    return;
  }
  if (bits != a.dist[cell]) return;
  const unsigned long long t = ((unsigned long long)(rank + 1) << 32) | (uint32_t)a.v.seq[p];
  if (PASS == 1) {
    atomicMax(a.tie + cell, t);
    return;
  }
  if (t != a.tie[cell]) return;
  a.win[cell] = p;
  a.pc[2 * cell] = u.v, a.pc[2 * cell + 1] = v.v;
  for (int j = 0; j < 3; j++) a.wpos[3 * cell + j] = a.v.pos[3 * (size_t)p + j];
}

__global__ void vrt_init_kernel(const VrtArgs a) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.length) return;
  a.type[c] = 0, a.dist[c] = 0x461c4000u /* 10000.0f */, a.tie[c] = 0ull, a.win[c] = -1;
  a.pc[2 * c] = a.pc[2 * c + 1] = 0.0;
  for (int j = 0; j < 3; j++) a.wpos[3 * c + j] = 0.0;
}

struct VrtCellArgs {
  int length;
  const uint8_t *type, *disc, *ninit;  // ninit: the point arrays' is_normal_initialized_
  const int32_t *win;
  const double *pc, *wpos;
  int32_t *keep, *dst;                 // [length] TYPE_MAP flags, their offsets
  int32_t *skeep, *sdst;               // [length] survivor flags, their offsets
  // answers in cell order
  int32_t *cell_out, *id_out, *status_out, *ref_out;
  double *pc_out;
  // survivors in cell order: point id, pos_, and the position of their cell among the answers
  int32_t *spid, *sat;
  double *spos;
};

// FLAGS: keep = TYPE_MAP; skeep = the cell's winner passes the depth check and is_normal_initialized_. Else the answers at dst.
template <bool FLAGS> __global__ void vrt_cells_kernel(const VrtCellArgs a) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.length) return;
  const int w = a.win[c];
  const bool marked = a.type[c] != 0;
  const int status = w < 0 ? VRT_NO_WINNER : a.disc[c] ? VRT_DEPTH : !a.ninit[w] ? VRT_NOT_INIT : VRT_KEPT;
  if (FLAGS) {
    a.keep[c] = marked;
    a.skeep[c] = marked && status == VRT_KEPT;
    return;
  }
  if (!marked) return;
  const int o = a.dst[c];
  a.cell_out[o] = c, a.id_out[o] = w, a.status_out[o] = status, a.ref_out[o] = -1;
  a.pc_out[2 * o] = a.pc[2 * c], a.pc_out[2 * o + 1] = a.pc[2 * c + 1];
  if (status != VRT_KEPT) return;
  const int s = a.sdst[c];
  a.spid[s] = w, a.sat[s] = o;
  for (int j = 0; j < 3; j++) a.spos[3 * s + j] = a.wpos[3 * c + j];
}

__global__ void vrt_refs_kernel(const int32_t *__restrict__ ref, const int32_t *__restrict__ sat, int n, int32_t *__restrict__ ref_out,
                                int32_t *__restrict__ status_out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  ref_out[sat[s]] = ref[s];
  if (ref[s] < 0) status_out[sat[s]] = VRT_NO_REF;
}

}  // namespace esikf
