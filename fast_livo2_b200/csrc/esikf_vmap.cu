// The visual map's observation store, K14 (H100, sm_90a): every visual point's obs_ list (VisualPoint::obs_, the Feature
// objects) kept on the device, fed by new points and new observations, edited by the bookkeeping of
// VIOManager::updateVisualMapPoints (reference src/vio.cpp:914-964), scored in place by K13 and read by the reference-feature
// choice of retrieveFromVisualSparseMap (:651-697).
//
// A point id is a slot of the store. Slot p holds count[p] (0 .. VMAP_SLOTS) observations in obs_ order, the newest first
// (addFrameRef pushes at the front), and ref[p], the position of ref_patch in that list or -1 (has_ref_patch_ false). Per
// observation the store keeps what device code reads: px_, T_f_w_ (R row-major, then t), patch_, id_, mean_ and score_.
// updateVisualMapPoints evicts one observation at 30 before it adds one, and a new point has one, so no list ever holds more
// than 30: a fixed record of 30 slots a point (11,408 bytes).
//
//   vmap_last_kernel  : per update entry, obs_.back()'s T_f_w_ and px_ into the arrays K10's obs_flag_kernel reads
//   vmap_edit_kernel  : one warp per update entry: deleteNonRefPatchFeatures of a converged point, the eviction of the first
//                       strict minimum of score_ at 30 observations, and addFrameRef of a flagged one
//   vmap_choose_kernel: one warp per retrieved point: the reference-feature choice (normal_en) or getCloseViewObs
//   vmap_pack_kernel  : observations of the given points into packed lists (download), or back (add)
//
// Every double is single-rounded in the reference's operation order (Rn), every float sum runs in the reference's order, and
// no result depends on the launch geometry. Every entry of one call names a different point, so the warps never share a slot.

namespace esikf {

#define VMAP_SLOTS 30
#define VMAP_WARPS 4

// the store's device arrays, laid out in one allocation of `cap` point records
struct VmapView {
  double *T;             // [cap][30][12] T_f_w_
  double *px;            // [cap][30][2]  px_
  float *patch;          // [cap][30][64] patch_
  float *mean, *score;   // [cap][30]     mean_, score_
  int32_t *id;           // [cap][30]     id_
  int32_t *count, *ref;  // [cap]
};
static inline size_t vmap_bytes(size_t cap) { return cap * (8 + VMAP_SLOTS * (12 * 8 + 2 * 8 + 64 * 4 + 3 * 4)); }
static inline VmapView vmap_view(uint8_t *b, size_t cap) {
  VmapView v;
  const size_t o = cap * VMAP_SLOTS;
  v.T = (double *)b, v.px = v.T + 12 * o, v.patch = (float *)(v.px + 2 * o), v.mean = v.patch + 64 * o, v.score = v.mean + o;
  v.id = (int32_t *)(v.score + o), v.count = v.id + o, v.ref = v.count + cap;
  return v;
}

// K13 on the store: entry i is point pid[i], whose list starts at its first slot; a ref is stored where one is chosen (the
// reference leaves ref_patch alone otherwise)
struct RpStore {
  const int32_t *pid, *counts;
  int32_t *ref;
  __device__ __forceinline__ int begin(int i) const { return pid[i] * VMAP_SLOTS; }
  __device__ __forceinline__ int count(int i) const { return counts[pid[i]]; }
  __device__ __forceinline__ void set_ref(int i, int r) const {
    if (r >= 0) ref[pid[i]] = r;
  }
};

// obs_.back() of entry i's point. A point without observations (a converged point whose deleteNonRefPatchFeatures kept none;
// the reference would read obs_.back() of an empty list) gets NaN, which adds no observation (DESIGN.md §4).
__global__ void vmap_last_kernel(const VmapView s, const int32_t *__restrict__ pid, int n, double *__restrict__ last_T, double *__restrict__ last_px) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = pid[i], c = s.count[p];
  const size_t o = (size_t)p * VMAP_SLOTS + (c - 1);
  for (int k = 0; k < 12; k++) last_T[12 * (size_t)i + k] = c > 0 ? s.T[12 * o + k] : __longlong_as_double(0x7ff8000000000000ll);
  for (int k = 0; k < 2; k++) last_px[2 * (size_t)i + k] = c > 0 ? s.px[2 * o + k] : __longlong_as_double(0x7ff8000000000000ll);
}

// One field of a point's list rearranged by the lanes: lane d (< 30) writes slot d from old slot src (-1: the new observation
// `fresh`) when d is live and src != d. Every lane reads before any lane writes.
template <class T> __device__ __forceinline__ void vmap_move(T *rows, int E, int lane, int src, bool live, const T *fresh) {
  const bool write = lane < VMAP_SLOTS && live && src != lane;
  for (int k = 0; k < E; k++) {
    T v = T();
    if (write) v = src >= 0 ? rows[src * E + k] : fresh[k];
    __syncwarp();
    if (write) rows[lane * E + k] = v;
    __syncwarp();
  }
}

struct VmapEditArgs {
  ObsArgs obs;               // K10's arguments: the frame pose, the entries' convergence and flags
  VmapView s;
  const int32_t *pid;        // [n]
  const int32_t *dst;        // [n] offset of a flagged entry among the new observations
  const double *new_pc;      // [k][2] their px_
  const float *new_patch;    // [k][64] their patch_
  const double *T_f_w;       // [12] T_f_w_ of the new observations; NULL: the frame pose of the flags
  int32_t frame_id;
  int32_t *evicted, *count;  // [n] outputs
};

__global__ void __launch_bounds__(VMAP_WARPS * 32) vmap_edit_kernel(const VmapEditArgs a) {
  __shared__ double Rcw[9], Pcw[3], Tinv[3], Tnew[12];
  obs_frame_pose(a.obs, Rcw, Pcw, Tinv);
  if (threadIdx.x < 12) Tnew[threadIdx.x] = a.T_f_w ? a.T_f_w[threadIdx.x] : threadIdx.x < 9 ? Rcw[threadIdx.x] : Pcw[threadIdx.x - 9];
  __syncthreads();
  const int lane = threadIdx.x & 31, i = blockIdx.x * VMAP_WARPS + (threadIdx.x >> 5);
  if (i >= a.obs.n) return;
  const int p = a.pid[i], c = a.s.count[p];
  int r = a.s.ref[p], e = -1, c2;
  const bool add = a.obs.flag[i];
  const size_t o = (size_t)p * VMAP_SLOTS;
  int src;  // the old slot lane d's new slot comes from (-1: the new observation)
  if (a.obs.converged[i]) {
    // deleteNonRefPatchFeatures: only ref_patch stays; with no ref_patch (nullptr, or never set) every observation goes
    c2 = r >= 0 ? 1 : 0;
    src = r;
    r = r >= 0 ? 0 : -1;
  } else {
    if (c >= VMAP_SLOTS) {
      // findMinScoreFeature: the first score_ below the running minimum, which starts at FLT_MAX; obs_.begin() when none is
      e = 0;
      float m = 3.402823466e+38f;
      for (int j = 0; j < c; j++) {
        const float v = a.s.score[o + j];
        if (v < m) m = v, e = j;
      }
      if (r == e) r = -1;  // deleteFeatureRef
      else if (r > e) r--;
    }
    const int kept = c - (e >= 0);
    c2 = kept + add;
    int j = add ? lane - 1 : lane;  // position among the kept observations
    src = j < 0 ? -1 : (e >= 0 && j >= e ? j + 1 : j);
    if (add && r >= 0) r++;
  }
  const bool live = lane < c2;
  const int q = add ? a.dst[i] : 0;
  vmap_move(a.s.T + 12 * o, 12, lane, src, live, Tnew);
  vmap_move(a.s.px + 2 * o, 2, lane, src, live, add ? a.new_pc + 2 * (size_t)q : nullptr);
  vmap_move(a.s.patch + 64 * o, 64, lane, src, live, add ? a.new_patch + 64 * (size_t)q : nullptr);
  const float zero = 0.0f;
  vmap_move(a.s.mean + o, 1, lane, src, live, &zero);
  vmap_move(a.s.score + o, 1, lane, src, live, &zero);
  vmap_move(a.s.id + o, 1, lane, src, live, &a.frame_id);
  if (lane == 0) {
    a.s.count[p] = c2, a.s.ref[p] = r;
    a.evicted[i] = e, a.count[i] = c2;
  }
}

struct VmapChooseArgs {
  VmapView s;
  const int32_t *pid;     // [n]
  const double *pos;      // [n][3] VisualPoint::pos_
  double frame_pos[3];    // new_frame_->pos()
  int n, normal_en;
  int32_t *ref;           // [n] output
};

// The reference feature of each retrieved point (:651-697). normal_en: one observation -> it; no ref_patch -> the first strict
// minimum, from FLT_MAX, of the float sum of squared patch differences against every observation of another id_, in list
// order, divided by their count; else the stored ref. The first two are stored as ref_patch. Without normal_en,
// getCloseViewObs: the first strict maximum, from 0, of the cosine between the frame's and the observation's viewing rays,
// -1 below 0.5. -1 also where the reference leaves ref_ftr unset: no error beats FLT_MAX (DESIGN.md §4).
__global__ void __launch_bounds__(VMAP_WARPS * 32) vmap_choose_kernel(const VmapChooseArgs a) {
  const int lane = threadIdx.x & 31, i = blockIdx.x * VMAP_WARPS + (threadIdx.x >> 5);
  if (i >= a.n) return;
  const int p = a.pid[i], c = a.s.count[p], r0 = a.s.ref[p];
  const size_t o = (size_t)p * VMAP_SLOTS;
  int best = -1;
  if (a.normal_en) {
    if (c == 1) {
      best = 0;
    } else if (r0 >= 0) {
      best = r0;
    } else {
      float err = 0.0f;
      if (lane < c) {
        const float *pa = a.s.patch + 64 * (o + lane);
        const int idr = a.s.id[o + lane];
        int count = 0;
        for (int j = 0; j < c; j++) {
          if (a.s.id[o + j] == idr) continue;
          const float *pb = a.s.patch + 64 * (o + j);
          for (int k = 0; k < 64; k++) {
            const float d = __fsub_rn(pa[k], pb[k]);
            err = __fadd_rn(err, __fmul_rn(d, d));
          }
          count++;
        }
        err = __fdiv_rn(err, (float)count);
      }
      float m = 3.402823466e+38f;
      for (int j = 0; j < c; j++) {
        const float v = __shfl_sync(0xffffffffu, err, j);
        if (v < m) m = v, best = j;
      }
    }
  } else {
    const Rn px = a.frame_pos[0], py = a.frame_pos[1], pz = a.frame_pos[2];
    const double *pw = a.pos + 3 * (size_t)i;
    Rn od[3] = {px - Rn(pw[0]), py - Rn(pw[1]), pz - Rn(pw[2])};
    const Rn on = sqrt(Rn(0.0) + od[0] * od[0] + od[1] * od[1] + od[2] * od[2]);
    for (int k = 0; k < 3; k++) od[k] = od[k] / on;
    double cs = 0.0;
    if (lane < c) {
      // T_f_w_.inverse().translation() = (R^T t) * -1.0, then minus pos_, normalised
      const double *T = a.s.T + 12 * (o + lane);
      Rn d[3];
      for (int k = 0; k < 3; k++) d[k] = -(Rn(0.0) + Rn(T[k]) * Rn(T[9]) + Rn(T[3 + k]) * Rn(T[10]) + Rn(T[6 + k]) * Rn(T[11])) - Rn(pw[k]);
      const Rn dn = sqrt(Rn(0.0) + d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
      for (int k = 0; k < 3; k++) d[k] = d[k] / dn;
      cs = (Rn(0.0) + od[0] * d[0] + od[1] * d[1] + od[2] * d[2]).v;
    }
    double m = 0.0;
    int at = 0;
    for (int j = 0; j < c; j++) {
      const double v = __shfl_sync(0xffffffffu, cs, j);
      if (v > m) m = v, at = j;
    }
    best = c > 0 && !(m < 0.5) ? at : -1;
  }
  if (lane == 0) {
    a.ref[i] = best;
    if (a.normal_en && best >= 0) a.s.ref[p] = best;
  }
}

// Packed lists <-> store slots, one warp per point: to_store copies point i's observations first[i] .. first[i + 1] - 1
// into slot pid[i] and sets its count and ref; else the other way.
template <class T> __device__ __forceinline__ void vmap_xfer(T *slot, T *packed, bool to_store) {
  if (to_store) *slot = *packed;
  else *packed = *slot;
}
struct VmapPackArgs {
  VmapView s;
  const int32_t *pid, *first;  // [n], [n + 1]
  int n, to_store;
  double *T, *px;
  float *patch, *mean, *score;
  int32_t *id, *ref;
};
__global__ void __launch_bounds__(VMAP_WARPS * 32) vmap_pack_kernel(const VmapPackArgs a) {
  const int lane = threadIdx.x & 31, i = blockIdx.x * VMAP_WARPS + (threadIdx.x >> 5);
  if (i >= a.n) return;
  const int b = a.first[i], c = a.first[i + 1] - b;
  const size_t o = (size_t)a.pid[i] * VMAP_SLOTS;
  const bool in = a.to_store;
  for (int e = lane; e < 64 * c; e += 32) vmap_xfer(a.s.patch + 64 * o + e, a.patch + 64 * (size_t)b + e, in);
  for (int e = lane; e < 12 * c; e += 32) vmap_xfer(a.s.T + 12 * o + e, a.T + 12 * (size_t)b + e, in);
  for (int e = lane; e < 2 * c; e += 32) vmap_xfer(a.s.px + 2 * o + e, a.px + 2 * (size_t)b + e, in);
  if (lane < c) {
    vmap_xfer(a.s.mean + o + lane, a.mean + b + lane, in);
    vmap_xfer(a.s.score + o + lane, a.score + b + lane, in);
    vmap_xfer(a.s.id + o + lane, a.id + b + lane, in);
  }
  if (lane == 0) {
    if (in) a.s.count[a.pid[i]] = c;
    vmap_xfer(a.s.ref + a.pid[i], a.ref + i, in);
  }
}

// count and ref of the given points (download's sizes), and the rows [n][30] of score_ and mean_ after esikf_vmap_score
// (0 past a point's count)
__global__ void vmap_rows_kernel(const VmapView s, const int32_t *__restrict__ pid, int n, int32_t *__restrict__ count, float *__restrict__ score,
                                 float *__restrict__ mean) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * VMAP_SLOTS) return;
  const int i = t / VMAP_SLOTS, j = t % VMAP_SLOTS, p = pid[i], c = s.count[p];
  if (count && j == 0) count[i] = c;
  const size_t o = (size_t)p * VMAP_SLOTS + j;
  if (score) score[t] = j < c ? s.score[o] : 0.0f;
  if (mean) mean[t] = j < c ? s.mean[o] : 0.0f;
}

}  // namespace esikf
