// Device-side common definitions of the ESIKF update (H100, sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/esikf_b200.h"

namespace esikf {

// ---- packed state offsets (ESIKF_STATE_DOUBLES doubles, see include/esikf_b200.h)
enum { S_R = 0, S_P = 9, S_EXPO = 12, S_V = 13, S_BG = 16, S_BA = 19, S_G = 22, S_COV = 25, S_N = ESIKF_STATE_DOUBLES };

// ---- device hash of root voxels: open addressing, linear probing, 16-byte slots
struct HashSlot {
  unsigned long long key;  // packed VOXEL_LOCATION (21 bits / axis, biased), ~0 = empty
  uint32_t first;          // first candidate plane
  uint32_t count;          // number of candidate planes (DFS order)
};
#define ESIKF_KEY_EMPTY 0xFFFFFFFFFFFFFFFFull
#define ESIKF_KEY_BIAS (1 << 20)
#define ESIKF_KEY_RANGE (1 << 21)

__host__ __device__ inline bool key_in_range(long long x, long long y, long long z) {
  return x >= -ESIKF_KEY_BIAS && x < ESIKF_KEY_BIAS && y >= -ESIKF_KEY_BIAS && y < ESIKF_KEY_BIAS && z >= -ESIKF_KEY_BIAS &&
         z < ESIKF_KEY_BIAS;
}
__host__ __device__ inline unsigned long long pack_key(long long x, long long y, long long z) {
  return ((unsigned long long)(x + ESIKF_KEY_BIAS) << 42) | ((unsigned long long)(y + ESIKF_KEY_BIAS) << 21) |
         (unsigned long long)(z + ESIKF_KEY_BIAS);
}
__host__ __device__ inline uint32_t hash_key(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return (uint32_t)k;
}

// ---- plane record as the residual kernel consumes it (derived on the device from the 256-byte esikf_plane at map upload /
// patch time, plane_compact_kernel). sigma_l = J plane_var J^T with J = [p - c, -n] (src/voxel_map.cpp:733-735) expands to
//   e^T Paa e + 2 e^T (Pab n) + n^T Pbb n,   e = c - p,
// and only e depends on the point: b = Pab n and cnn = n^T Pbb n are properties of the plane. 18 doubles = 144 bytes
// (9 x 16 B: one cp.async.bulk per record, conflict-free lane stride in shared memory).
struct PlaneRec {
  double c[3];    // center_
  double n[3];    // normal_
  double paa[6];  // plane_var_[0:3,0:3], upper triangle xx xy xz yy yz zz
  double b[3];    // plane_var_[0:3,3:6] * normal_
  double cnn;     // normal_^T plane_var_[3:6,3:6] normal_
  float d;        // d_
  float radius;   // radius_
  double pad;
};
static_assert(sizeof(PlaneRec) == 144, "compact plane record is 9 x 16 bytes");

// ---- arithmetic of a plane fit: single-rounded products and sums in the written order, never contracted into FMAs, so that the
// device reproduces the host evaluation of the same expressions (and with it the oracle's) bit for bit
__host__ __device__ __forceinline__ double m_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double m_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ double m_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ double m_dot3(double a0, double b0, double a1, double b1, double a2, double b2) { return m_add(m_add(m_mul(a0, b0), m_mul(a1, b1)), m_mul(a2, b2)); }

// a00 a11 - a01 a10 with both products rounded, as the reference's 2 x 2 determinant (getBestSearchLevel, warpAffine's
// inverse). Contracted into an FMA it can land on the other side of getBestSearchLevel's thresholds 3 / 12 when it lies
// within an ulp of one, and it gives a different float inverse when the products cancel.
__device__ __forceinline__ double det2_rn(double a00, double a11, double a01, double a10) { return __dsub_rn(__dmul_rn(a00, a11), __dmul_rn(a01, a10)); }

// 256-byte map plane -> the 144-byte record (one definition for the upload / patch kernel and the device-resident map, evaluated
// without FMA contraction: both paths hand the residual kernel bit-identical records for the same plane)
__host__ __device__ constexpr int tri6u(int i, int j) { return i * 6 - (i * (i - 1)) / 2 + (j - i); }  // i <= j
__host__ __device__ __forceinline__ void compact_plane(const esikf_plane &p, PlaneRec &r) {
  const double n0 = p.normal[0], n1 = p.normal[1], n2 = p.normal[2];
  for (int j = 0; j < 3; j++) r.c[j] = p.center[j], r.n[j] = p.normal[j];
  r.paa[0] = p.plane_var[tri6u(0, 0)], r.paa[1] = p.plane_var[tri6u(0, 1)], r.paa[2] = p.plane_var[tri6u(0, 2)];
  r.paa[3] = p.plane_var[tri6u(1, 1)], r.paa[4] = p.plane_var[tri6u(1, 2)], r.paa[5] = p.plane_var[tri6u(2, 2)];
  for (int i = 0; i < 3; i++) r.b[i] = m_dot3(p.plane_var[tri6u(i, 3)], n0, p.plane_var[tri6u(i, 4)], n1, p.plane_var[tri6u(i, 5)], n2);
  const double *v = p.plane_var;
  // n^T Pbb n as (n^T Pbb) n
  const double t0 = m_dot3(n0, v[tri6u(3, 3)], n1, v[tri6u(3, 4)], n2, v[tri6u(3, 5)]);
  const double t1 = m_dot3(n0, v[tri6u(3, 4)], n1, v[tri6u(4, 4)], n2, v[tri6u(4, 5)]);
  const double t2 = m_dot3(n0, v[tri6u(3, 5)], n1, v[tri6u(4, 5)], n2, v[tri6u(5, 5)]);
  r.cnn = m_dot3(t0, n0, t1, n1, t2, n2);
  r.d = p.d, r.radius = p.radius, r.pad = 0.0;
}

// ---- reduced information of one iteration, compact: for an m-column measurement (m = 6 LIO, 7 VIO)
//   [0, T)          upper triangle of H^T R^-1 H, row-major (i <= j),  T = m (m + 1) / 2
//   [T, T + m)      H^T R^-1 z
//   [T + m]         sum |dis_to_plane| (LIO) / sum res^2 (VIO)
//   [T + m + 1]     matched points (LIO) / n_meas (VIO)
// 29 entries for LIO, 37 for VIO; buffers are sized NE_MAX.
#define NE_MAX 40
__host__ __device__ constexpr int ne_of(int m) { return m * (m + 1) / 2 + m + 2; }
__host__ __device__ constexpr int tri_of(int m, int i, int j) { return i * m - (i * (i - 1)) / 2 + (j - i); }  // i <= j

// ---- loop-control block shared by the kernels of one update (device memory)
struct Ctrl {
  int stop;         // LIO: EKF_stop_flg ; VIO: whole update finished
  int iter;         // LIO: iterations executed so far ; VIO: total iterations
  int rematch_num;  // LIO (voxel_map.cpp:365,482)
  int level_done;   // VIO: EKF_end of the current level
  int level;        // VIO: level being processed
  int level_iter;   // VIO: iteration counter inside the level
  float last_error; // VIO (vio.cpp:1528)
  int has_G;        // VIO: G valid (at least one accepted update)
  unsigned int block_counter;  // last-block-done counter of the per-iteration residual kernels
  int accepted_in_level;       // VIO: accepted updates of the current level (diagnostics)
  int comm_error;              // a bounded wait (grid barrier / peer mailbox) expired: results of this update are invalid
  int pad[5];
};

#ifdef __CUDACC__
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// fp64 tensor-core contraction step: D(8x8) += A(8x4) * B(4x8), mma.sync.m8n8k4.f64 (SASS DMMA).
// Lane l holds A[l/4][l%4], B[l%4][l/4] and D[l/4][2*(l%4) + {0,1}].
__device__ __forceinline__ void dmma_m8n8k4(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// Compact entry of element (g, h) of a warp's 8x8 block D = sum_i a_i b_i^T, or -1 when the element is not needed.
// LIO rows a = [A(3) n(3) z 1], b = [w a(0:7), |d|]: H^T R^-1 H = D[0:6,0:6], H^T R^-1 z = D[0:6,6], sum|d| = D[7][7].
// VIO rows a = b = [JdR(3) Jdt(3) cur res]:          H^T H = D[0:7,0:7],      H^T z = D[0:7,7],      sum res^2 = D[7][7].
template <int M> __device__ __forceinline__ int compact_entry(int g, int h) {
  constexpr int T = M * (M + 1) / 2;
  constexpr int ZC = (M == 6) ? 6 : 7;
  if (g < M && h < M) return (g <= h) ? tri_of(M, g, h) : -1;
  if (g < M && h == ZC) return T + g;
  if (g == 7 && h == 7) return T + M;
  return -1;
}

// Per-CTA scratch of the fixed-order reduction: one compact vector per warp.
template <int WARPS> struct ReduceSmem {
  double w[WARPS][NE_MAX];
  int is_last;
};

// warp fragments -> per-CTA compact vector -> global partial column `blockIdx.x` of the entry-major array
// partials[entry][partial_stride]. Fixed order (warp 0, 1, ...), so the result does not depend on timing.
template <int WARPS, int M>
__device__ __forceinline__ void store_partials(ReduceSmem<WARPS> &rs, double D0, double D1, double cnt, double *partials, int partial_stride) {
  constexpr int NE = ne_of(M);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  {
    const int g = lane >> 2, t = lane & 3;
    const int e0 = compact_entry<M>(g, 2 * t), e1 = compact_entry<M>(g, 2 * t + 1);
    if (e0 >= 0) rs.w[warp][e0] = D0;
    if (e1 >= 0) rs.w[warp][e1] = D1;
    if (lane == 0) rs.w[warp][NE - 1] = cnt;
  }
  __syncthreads();
  if (tid < NE) {
    double s = rs.w[0][tid];
#pragma unroll
    for (int w = 1; w < WARPS; w++) s += rs.w[w][tid];
    partials[(size_t)tid * partial_stride + blockIdx.x] = s;
  }
}

// Fixed-order sum over the per-CTA partial columns by the calling CTA (nb <= 160 columns): warp w owns entries w,
// w + nwarps, ...; lane l adds columns l, l + 32, ... in order, then a fixed xor-shuffle tree. Every load is issued before
// the first add, so the whole sum costs ONE L2 round trip. Bit-identical in every CTA that runs it.
#define SUM_MAXC 5
template <int M> __device__ __forceinline__ void sum_partials(const double *partials, int partial_stride, int nb, double *out, int nwarps) {
  constexpr int NE = ne_of(M);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int MAXE = 3;  // NE <= 3 * nwarps for nwarps >= 14
  double v[MAXE][SUM_MAXC];
#pragma unroll
  for (int k = 0; k < MAXE; k++) {
    const int e = warp + k * nwarps;
    const double *__restrict__ p = partials + (size_t)e * partial_stride;
#pragma unroll
    for (int c = 0; c < SUM_MAXC; c++) {
      const int b = lane + 32 * c;
      v[k][c] = (e < NE && b < nb) ? __ldcg(p + b) : 0.0;
    }
  }
#pragma unroll
  for (int k = 0; k < MAXE; k++) {
    const int e = warp + k * nwarps;
    double s = v[k][0];
#pragma unroll
    for (int c = 1; c < SUM_MAXC; c++) s += v[k][c];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0 && e < NE) out[e] = s;
  }
}

// Per-iteration kernels (loop_mode 0): the last CTA to finish sums the partial columns into info[] (global).
template <int WARPS, int M>
__device__ __forceinline__ void reduce_info(ReduceSmem<WARPS> &rs, double D0, double D1, double cnt, double *partials, int partial_stride, double *info, Ctrl *ctrl) {
  const int tid = threadIdx.x;
  store_partials<WARPS, M>(rs, D0, D1, cnt, partials, partial_stride);
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    unsigned int prev = atomicAdd(&ctrl->block_counter, 1u);
    rs.is_last = (prev == gridDim.x - 1);
  }
  __syncthreads();
  if (!rs.is_last) return;
  __threadfence();
  sum_partials<M>(partials, partial_stride, gridDim.x, info, WARPS);
  if (tid == 0) ctrl->block_counter = 0;
}

// ---- mbarrier / bulk-copy (TMA engine, 1-D) helpers: one plane record per instruction, completion counted in bytes.
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, unsigned bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes),
               "r"(smem_u32(bar))
               : "memory");
}
// 2-D tiled TMA load (cp.async.bulk.tensor, SASS UTMALDG): box of the tensor map at element coordinates (x, y) -> shared
// memory, completion on the mbarrier. Out-of-bounds elements arrive as zeros and still count towards the byte total.
__device__ __forceinline__ void tma_load_2d(void *dst_smem, const void *tmap, int x, int y, unsigned long long *bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst_smem)), "l"(tmap), "r"(x),
               "r"(y), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#endif

}  // namespace esikf
