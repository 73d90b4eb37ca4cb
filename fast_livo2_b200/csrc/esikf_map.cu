// Device-side BuildVoxelMap / UpdateVoxelMap (SURVEY §8 f1; state machine in esikf_map.cuh):
//
//   map_points_kernel   : LIVMapper.cpp:413-424 (world point of every scan point with the posterior pose, float-rounded; its
//                         covariance R extR Sigma_b (R extR)^T + [c]x P_rot [c]x^T + P_pos) or voxel_map.cpp:541-556 (the
//                         BuildVoxelMap form), the voxel key (:620-625) and the hash slot of the root (inserted when new);
//                         also snapshots the normal of every point's matched plane (pv.normal) before records may move
//   cub radix sort      : (slot, scan index) pairs by slot — stable, so every root sees its points in scan order
//   map_heads_kernel    : one entry per touched root {slot, first sorted position, count}
//   map_demand_kernel   : (capacity growth on) one warp per touched root sums map_root_demand and raises the defer word when
//                         the tick might not fit the arena
//   map_replay_kernel   : one warp per touched root, work handed out through an atomic counter (roots differ a lot in work)
//   map_download_kernel : the map in esikf_map_upload's flat form (tests, visualisation, serialisation)
//   map_export_*_kernel : the subtrees of the roots the last replay touched, node by node (a host mirror of the map)
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "esikf_map.cuh"

namespace esikf {

struct MapPointArgs {
  const float *pts;        // [n][3] body-frame scan
  const double *pre;       // SoA [9][pre_stride] of lio_precompute_kernel (update form)
  int pre_stride, n;
  const double *state;     // packed state the points are transformed with
  double extR[9], extT[3];
  int build;               // 1: BuildVoxelMap's covariance (cross matrix of the raw body point, calcBodyCov's own z fix)
  float dept_err, beam_err;
  const int32_t *match_plane;  // normal_plane of the last update: the plane behind pv.normal (nullptr: no snapshot)
  const PlaneRec *recs;
  double *pt_normal;       // [n][3]
  double *pt;              // [n][12] out: point_w | var
  unsigned int *pt_slot, *pt_idx;
  unsigned int invalid_slot;  // sorts behind every real slot
};

// calcBodyCov (voxel_map.cpp:15-34) of a point whose z is already fixed; upper triangle xx xy xz yy yz zz
__device__ __forceinline__ void map_body_cov(double px, double py, double pz, float dept_err, float beam_err, double *c6) {
  const float range = (float)sqrt(px * px + py * py + pz * pz);
  const float range_var = dept_err * dept_err;
  const double sdv = sin((double)beam_err * 0.017453293);
  const double dv = sdv * sdv;
  const double nrm = sqrt(px * px + py * py + pz * pz);
  const double dx = px / nrm, dy = py / nrm, dz = pz / nrm;
  double b1x = 1.0, b1y = 1.0, b1z = -(dx + dy) / dz;
  const double n1 = sqrt(b1x * b1x + b1y * b1y + b1z * b1z);
  b1x /= n1, b1y /= n1, b1z /= n1;
  double b2x = b1y * dz - b1z * dy, b2y = b1z * dx - b1x * dz, b2z = b1x * dy - b1y * dx;
  const double n2 = sqrt(b2x * b2x + b2y * b2y + b2z * b2z);
  b2x /= n2, b2y /= n2, b2z /= n2;
  const double r = (double)range, rv = (double)range_var;
  const double a00 = r * (-dz * b1y + dy * b1z), a01 = r * (-dz * b2y + dy * b2z);
  const double a10 = r * (dz * b1x - dx * b1z), a11 = r * (dz * b2x - dx * b2z);
  const double a20 = r * (-dy * b1x + dx * b1y), a21 = r * (-dy * b2x + dx * b2y);
  c6[0] = dx * rv * dx + dv * (a00 * a00 + a01 * a01), c6[1] = dx * rv * dy + dv * (a00 * a10 + a01 * a11), c6[2] = dx * rv * dz + dv * (a00 * a20 + a01 * a21);
  c6[3] = dy * rv * dy + dv * (a10 * a10 + a11 * a11), c6[4] = dy * rv * dz + dv * (a10 * a20 + a11 * a21), c6[5] = dz * rv * dz + dv * (a20 * a20 + a21 * a21);
}

__global__ void __launch_bounds__(256) map_points_kernel(const MapArena A, const MapPointArgs a) {
  __shared__ double sR[9], st[3], sM[9], sPr[9], sPp[9];
  if (threadIdx.x < 9) {
    const int r = threadIdx.x / 3, c = threadIdx.x % 3;
    sR[threadIdx.x] = a.state[S_R + threadIdx.x];
    sPr[threadIdx.x] = a.state[S_COV + r * 19 + c];            // cov.block<3,3>(0,0)
    sPp[threadIdx.x] = a.state[S_COV + (3 + r) * 19 + 3 + c];  // cov.block<3,3>(3,3)
    // M = rot_end * extR
    sM[threadIdx.x] = m_dot3(a.state[S_R + 3 * r], a.extR[c], a.state[S_R + 3 * r + 1], a.extR[3 + c], a.state[S_R + 3 * r + 2], a.extR[6 + c]);
  }
  if (threadIdx.x < 3) st[threadIdx.x] = a.state[S_P + threadIdx.x];
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const float fx = a.pts[3 * (size_t)i], fy = a.pts[3 * (size_t)i + 1], fz = a.pts[3 * (size_t)i + 2];
  // world point: rot * (extR p + extT) + t, stored as float (LIVMapper.cpp:645-649)
  float wf[3];
  world_point_f(sR, st, a.extR, a.extT, fx, fy, fz, wf);
  const double pw[3] = {wf[0], wf[1], wf[2]};
  // covariance
  double b6[6], cv[3];
  if (a.build) {
    double px = fx, py = fy, pz = fz;
    if (pz == 0) pz = 0.0001;  // calcBodyCov's own fix (:17), which BuildVoxelMap's point_this keeps (:545-549)
    map_body_cov(px, py, pz, a.dept_err, a.beam_err, b6);
    cv[0] = px, cv[1] = py, cv[2] = pz;
  } else {
    const size_t ns = (size_t)a.pre_stride;
    for (int k = 0; k < 3; k++) cv[k] = a.pre[k * ns + i];
    for (int k = 0; k < 6; k++) b6[k] = a.pre[(3 + k) * ns + i];
  }
  const double B[9] = {b6[0], b6[1], b6[2], b6[1], b6[3], b6[4], b6[2], b6[4], b6[5]};
  // (M B) M^T
  double MB[9], var[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) MB[3 * r + c] = m_dot3(sM[3 * r], B[c], sM[3 * r + 1], B[3 + c], sM[3 * r + 2], B[6 + c]);
  // (-C) P_rot (-C)^T with C = [cv]x
  const double nC[9] = {-0.0, cv[2], -cv[1], -cv[2], -0.0, cv[0], cv[1], -cv[0], -0.0};
  double CP[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) CP[3 * r + c] = m_dot3(nC[3 * r], sPr[c], nC[3 * r + 1], sPr[3 + c], nC[3 * r + 2], sPr[6 + c]);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      // single-rounded, uncontracted, in the order of the reference's matrix expression (the fits amplify input rounding)
      const double t1 = m_dot3(MB[3 * r], sM[3 * c], MB[3 * r + 1], sM[3 * c + 1], MB[3 * r + 2], sM[3 * c + 2]);
      const double t2 = m_dot3(CP[3 * r], nC[3 * c], CP[3 * r + 1], nC[3 * c + 1], CP[3 * r + 2], nC[3 * c + 2]);
      var[3 * r + c] = m_add(m_add(t1, t2), sPp[3 * r + c]);
    }
  double *o = a.pt + (size_t)i * MAP_PT_D;
  for (int k = 0; k < 3; k++) o[k] = pw[k];
  for (int k = 0; k < 9; k++) o[3 + k] = var[k];
  // root voxel
  long long key[3];
  map_voxel_key(pw, A.cfg.voxel_size, key);
  unsigned int slot = a.invalid_slot;
  if (!key_in_range(key[0], key[1], key[2])) {
    map_raise(A, MAP_ERR_KEY);
  } else {
    const int s = map_slot_of(A, pack_key(key[0], key[1], key[2]));
    if (s < 0)
      map_raise(A, MAP_ERR_HASH);
    else
      slot = (unsigned int)s;
  }
  a.pt_slot[i] = slot, a.pt_idx[i] = (unsigned int)i;
  if (a.match_plane) {
    const int m = a.match_plane[i];
    for (int k = 0; k < 3; k++) a.pt_normal[3 * (size_t)i + k] = m >= 0 ? a.recs[m].n[k] : 0.0;
  }
}

// UpdateVoxelMap(input_points) with the caller's own lists: only key + slot
__global__ void __launch_bounds__(256) map_keys_kernel(const MapArena A, const double *__restrict__ pt, int n, unsigned int *pt_slot, unsigned int *pt_idx, unsigned int invalid_slot) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long key[3];
  map_voxel_key(pt + (size_t)i * MAP_PT_D, A.cfg.voxel_size, key);
  unsigned int slot = invalid_slot;
  if (!key_in_range(key[0], key[1], key[2])) {
    map_raise(A, MAP_ERR_KEY);
  } else {
    const int s = map_slot_of(A, pack_key(key[0], key[1], key[2]));
    if (s < 0)
      map_raise(A, MAP_ERR_HASH);
    else
      slot = (unsigned int)s;
  }
  pt_slot[i] = slot, pt_idx[i] = (unsigned int)i;
}

// work[0] = touched roots, work[1] = next root to hand out
__global__ void __launch_bounds__(256) map_heads_kernel(const unsigned int *__restrict__ sorted_slot, int n, unsigned int invalid_slot, MapTouched *touched, int *work) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const unsigned int s = sorted_slot[j];
  if (s == invalid_slot || (j > 0 && sorted_slot[j - 1] == s)) return;
  int lo = j + 1, hi = n;  // first position whose slot differs
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sorted_slot[mid] == s) lo = mid + 1; else hi = mid;
  }
  const int t = atomicAdd(&work[0], 1);
  touched[t].slot = s, touched[t].start = j, touched[t].count = lo - j;
}

// Capacity growth: demand[0..2] the summed map_root_demand (nodes, pool points, records), [3] next root to hand out, [4] warps
// done, [5] the defer word: the MAP_ERR_NODES / _POOL / _RECS bits of every resource whose free space is short of the sum.
// The last warp to finish compares, so the replay that follows only reads one word.
enum { MAP_DEMAND_WORDS = 8 };
__global__ void __launch_bounds__(128) map_demand_kernel(const MapArena A, const MapTouched *__restrict__ touched, const int *work, unsigned long long *demand, int build) {
  const WarpCoop co;
  const int n_touched = *reinterpret_cast<const volatile int *>(&work[0]);
  for (;;) {
    int t = 0;
    if (co.lane() == 0) t = (int)atomicAdd(&demand[3], 1ull);
    t = co.bcast(t);
    if (t >= n_touched) break;
    if (co.lane() == 0) {
      const MapTouched w = touched[t];
      const MapDemand d = map_root_demand(A, (int)w.slot, w.count, build != 0);
      atomicAdd(&demand[0], (unsigned long long)d.nodes), atomicAdd(&demand[1], (unsigned long long)d.pool), atomicAdd(&demand[2], (unsigned long long)d.recs);
    }
  }
  if (co.lane() != 0) return;
  __threadfence();
  const unsigned long long warps = (unsigned long long)gridDim.x * (blockDim.x / 32);
  if (atomicAdd(&demand[4], 1ull) != warps - 1) return;
  __threadfence();
  const volatile unsigned long long *v = demand;
  int defer = 0;
  if ((long long)A.counters[0] + (long long)v[0] > (long long)A.node_cap) defer |= MAP_ERR_NODES;
  if ((long long)A.counters64[0] + (long long)v[1] > A.pool_cap) defer |= MAP_ERR_POOL;
  if ((long long)A.counters[1] + (long long)v[2] > (long long)A.rec_cap) defer |= MAP_ERR_RECS;
  demand[5] = (unsigned long long)defer;
}

// defer (growth on): the word map_demand_kernel set; when it is non-zero the tick does not fit and nothing is touched
__global__ void __launch_bounds__(128) map_replay_kernel(const MapArena A, const MapTouched *__restrict__ touched, int *work, const unsigned int *__restrict__ order,
                                                         const double *__restrict__ pt, int build, const unsigned long long *defer) {
  const WarpCoop co;
  if (defer && *reinterpret_cast<const volatile unsigned long long *>(defer)) return;
  const int n_touched = *reinterpret_cast<volatile int *>(&work[0]);
  for (;;) {
    int t = 0;
    if (co.lane() == 0) t = atomicAdd(&work[1], 1);
    t = co.bcast(t);
    if (t >= n_touched) break;
    const MapTouched w = touched[t];
    map_replay_root(A, co, (int)w.slot, order, w.start, w.count, pt, build != 0);
  }
}

// out_counts[0] roots written, [1] candidate planes written
__global__ void __launch_bounds__(256) map_download_kernel(const MapArena A, long long *keys, int32_t *first, int32_t *count, esikf_plane *planes, int roots_cap, int planes_cap,
                                                           int *out_counts) {
  const unsigned int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > A.hash_mask) return;
  if (A.slots[s].key == ESIKF_KEY_EMPTY || A.slot_root[s] < 0) return;
  const int c = (int)A.slots[s].count;
  const int r = atomicAdd(&out_counts[0], 1);
  const int off = atomicAdd(&out_counts[1], c);
  if (!keys || r >= roots_cap || off + c > planes_cap) return;
  const unsigned long long k = A.slots[s].key;
  keys[3 * (size_t)r] = (long long)(k >> 42) - ESIKF_KEY_BIAS, keys[3 * (size_t)r + 1] = (long long)((k >> 21) & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS;
  keys[3 * (size_t)r + 2] = (long long)(k & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS;
  first[r] = off, count[r] = c;
  for (int j = 0; j < c; j++) planes[off + j] = A.planes[A.slots[s].first + j];
}

// Export of the touched roots (esikf_map_device_export), one warp per root, in two passes over the touched list of the last
// replay. The count pass writes (1 << 32 | subtree size) at the root's first position in the slot-sorted points (every other
// position holds 0); an exclusive scan over those positions turns it into (root index << 32 | first row), so the roots come
// out in slot order whatever order map_heads_kernel listed them in. The write pass lays out the rows.
__global__ void __launch_bounds__(128) map_export_count_kernel(const MapArena A, const MapTouched *__restrict__ touched, const int *work, unsigned long long *packed) {
  const WarpCoop co;
  const int n_touched = work[0], warps = gridDim.x * (blockDim.x / 32);
  for (int t = (blockIdx.x * blockDim.x + threadIdx.x) / 32; t < n_touched; t += warps) {
    const MapTouched w = touched[t];
    const int c = map_export_root(A, co, (int)w.slot, nullptr, nullptr);
    if (co.lane() == 0) packed[w.start] = (1ull << 32) | (unsigned)c;
  }
}
__global__ void __launch_bounds__(128) map_export_kernel(const MapArena A, const MapTouched *__restrict__ touched, const int *work, const unsigned long long *__restrict__ offs,
                                                         long long *keys, int32_t *first, int32_t *count, esikf_map_node *nodes, int *rows) {
  const WarpCoop co;
  const int n_touched = work[0], warps = gridDim.x * (blockDim.x / 32);
  for (int t = (blockIdx.x * blockDim.x + threadIdx.x) / 32; t < n_touched; t += warps) {
    const MapTouched w = touched[t];
    const unsigned long long o = offs[w.start];
    const int r = (int)(o >> 32), f = (int)(o & 0xffffffffull);
    const int c = map_export_root(A, co, (int)w.slot, nodes + f, rows + f);
    if (co.lane() == 0) {
      for (int q = 0; q < 3; q++) keys[3 * (size_t)r + q] = nodes[f].key[q];
      first[r] = f, count[r] = c;
    }
  }
}

// mapSliding: list the occupied slots inside the box, then one warp per surviving root copies it into the fresh arena
__global__ void __launch_bounds__(256) map_survivors_kernel(const MapArena S, long long lx, long long ly, long long lz, long long hx, long long hy, long long hz, int *survivors, int *work) {
  const unsigned int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > S.hash_mask) return;
  const unsigned long long k = S.slots[s].key;
  if (k == ESIKF_KEY_EMPTY || S.slot_root[s] < 0) return;
  const long long lo[3] = {lx, ly, lz}, hi[3] = {hx, hy, hz};
  if (!map_key_in_box(k, lo, hi)) return;
  survivors[atomicAdd(&work[0], 1)] = (int)s;
}
__global__ void __launch_bounds__(128) map_copy_kernel(const MapArena S, const MapArena D, const int *__restrict__ survivors, int *work) {
  const WarpCoop co;
  const int n = *reinterpret_cast<volatile int *>(&work[0]);
  for (;;) {
    int t = 0;
    if (co.lane() == 0) t = atomicAdd(&work[1], 1);
    t = co.bcast(t);
    if (t >= n) break;
    map_copy_root(S, D, co, survivors[t]);
  }
}

__global__ void map_reset_kernel(const MapArena A) {
  const unsigned int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s <= A.hash_mask) {
    A.slots[s].key = ESIKF_KEY_EMPTY, A.slots[s].first = 0, A.slots[s].count = 0;
    A.slot_root[s] = -1, A.slot_cap[s] = 0;
  }
  if (s < 4) A.counters[s] = 0;
  if (s == 0) A.counters64[0] = 0;
}

}  // namespace esikf
