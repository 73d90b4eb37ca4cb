// Reference-patch scoring of VIOManager::updateReferencePatch (reference src/vio.cpp:1036-1097), K13, on the device (H100,
// sm_90a): for every scored visual point, every observation's score_, mean_, and the observation that becomes ref_patch.
//
//   refpatch_score_kernel : one warp per point. Lane q scores the observations q, q + 32, ... of the point's list: the cosine
//                           between its viewing ray and the point's normal, and the NCC against every observation of another
//                           frame id; then lane 0 takes the first strict maximum above -1000 in list order. Templated on where a
//                           point's list lies: packed by first[] offsets (RpPacked, esikf_vio_score_ref_patches) or a slot of
//                           the visual map's observation store (RpStore in esikf_vmap.cu, esikf_vmap_score), whose mean_ and
//                           score_ it reads and writes in place.
//
// What is computed, per point with observations o_0 .. o_{n-1} in obs_ order (the newest first):
//   mean(o)   : o.mean_ when abs(mean_) >= 1e-6 (float abs, compared in double), else the double sum of the 64 taps in order,
//               narrowed to float, divided by 64 in float. The reference caches what it computes in mean_; a mean below 1e-6
//               is recomputed at every read, to the same value.
//   score(r)  : up = d1 = d2 = ncc = 0 (float); for each o_j in list order with id_ != o_r.id_, for k = 0..63:
//               up += (a_k - mean(o_r)) (b_k - mean(o_j)), d1 += (a_k - mean(o_r))^2, d2 += (b_k - mean(o_j))^2; then
//               ncc += fabs(up / sqrt(d1 * d2)) and count++. The three sums are declared per reference observation (:1039-1041)
//               and are not reset between the other observations: each term reads the running sums over every pair so far.
//               ncc / count is float by int (NaN when count is 0); score = ncc + cos_angle in double, narrowed to float.
//   ref       : the first r with score(r) > the running maximum, which starts at -1000 (strict >, so a tie keeps the earlier
//               observation and NaN never wins); -1 when no score beats -1000.
// The reference declares ref_mean / other_mean without a value and assigns them only when mean_ is below 1e-6, so from the
// second read of a cached mean on it reads an uninitialised float. Here both are the observation's mean as defined above: the
// cached value the code means to use (DESIGN.md §4).
//
// Every float operation is single-rounded (__fadd_rn / __fmul_rn / __fdiv_rn / __fsqrt_rn: no FMA contraction) and every sum
// runs in the reference's order, so the results are the host's bit for bit and do not depend on the launch geometry. A point
// with at most RP_CAP observations has its centred patches staged in shared memory (65 floats a row: the lanes' rows fall in
// different banks); a larger one reads them from global memory, with the same arithmetic.

namespace esikf {

#define RP_WARPS 4
#define RP_CAP 32
#define RP_STRIDE 65

struct RefPatchArgs {
  const double *pos, *normal;   // [n][3] VisualPoint::pos_, normal_
  const double *T;              // [m][12] Feature::T_f_w_: R row-major, then t
  const float *patch;           // [m][64] Feature::patch_
  const float *mean;            // [m] Feature::mean_ on entry
  const int32_t *id;            // [m] Feature::id_
  int n;
  float *score, *mean_out;      // [m]; mean_out is read back by the warp that wrote it (it may be `mean`: the lane that reads
                                // an observation's mean is the one that writes it, and a __syncwarp precedes every other read)
  int32_t *ref;                 // [n]
};

// point i owns the observations first[i] .. first[i + 1] - 1
struct RpPacked {
  const int32_t *first;
  __device__ __forceinline__ int begin(int i) const { return first[i]; }
  __device__ __forceinline__ int count(int i) const { return first[i + 1] - first[i]; }
  __device__ __forceinline__ void set_ref(int, int) const {}
};

// The mean the scoring uses for an observation whose cached mean_ is `cached` (std::accumulate from 0.0, then float / int)
__device__ __forceinline__ float rp_mean(const float *p, float cached) {
  if (!(fabsf(cached) < 1e-6)) return cached;
  double s = 0.0;
  for (int k = 0; k < 64; k++) s = __dadd_rn(s, (double)p[k]);
  return __fdiv_rn(__double2float_rn(s), 64.0f);
}

// the centred tap k of observation j: staged in shared memory, or the patch minus its mean from global memory
struct RpSmemTaps {
  const float *s;
  __device__ __forceinline__ float operator()(int j, int k) const { return s[j * RP_STRIDE + k]; }
};
struct RpGlobalTaps {
  const float *p, *mu;
  __device__ __forceinline__ float operator()(int j, int k) const { return __fsub_rn(p[64 * j + k], mu[j]); }
};

// NCC / count of observation r against the n observations of the point (:1038-1090)
template <class Taps> __device__ __forceinline__ float rp_ncc(const Taps &t, const int32_t *id, int n, int r) {
  float up = 0.0f, d1 = 0.0f, d2 = 0.0f, ncc = 0.0f;
  int count = 0;
  const int idr = id[r];
  for (int j = 0; j < n; j++) {
    if (id[j] == idr) continue;
#pragma unroll 8
    for (int k = 0; k < 64; k++) {
      const float a = t(r, k), b = t(j, k);
      up = __fadd_rn(up, __fmul_rn(a, b));
      d1 = __fadd_rn(d1, __fmul_rn(a, a));
      d2 = __fadd_rn(d2, __fmul_rn(b, b));
    }
    ncc = __fadd_rn(ncc, fabsf(__fdiv_rn(up, __fsqrt_rn(__fmul_rn(d1, d2)))));
    count++;
  }
  return __fdiv_rn(ncc, (float)count);
}

template <class Lists> __global__ void __launch_bounds__(RP_WARPS * 32) refpatch_score_kernel(const RefPatchArgs a, const Lists L) {
  __shared__ float taps[RP_WARPS][RP_CAP * RP_STRIDE];
  __shared__ int32_t ids[RP_WARPS][RP_CAP];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * RP_WARPS + w;
  if (i >= a.n) return;
  const int b = L.begin(i), n = L.count(i);
  const double *pos = a.pos + 3 * (size_t)i, *normal = a.normal + 3 * (size_t)i;
  float *score = a.score + b;
  if (n <= RP_CAP) {
    float *s = taps[w];
    const float *p = a.patch + 64 * (size_t)b;
    for (int e = lane; e < 64 * n; e += 32) s[(e >> 6) * RP_STRIDE + (e & 63)] = p[e];
    __syncwarp();
    if (lane < n) {
      float *row = s + lane * RP_STRIDE;
      const float mu = rp_mean(row, a.mean[b + lane]);
      a.mean_out[b + lane] = mu;
      for (int k = 0; k < 64; k++) row[k] = __fsub_rn(row[k], mu);
      ids[w][lane] = a.id[b + lane];
    }
    __syncwarp();
    if (lane < n) {
      Rn pf[3];
      const double *T = a.T + 12 * (size_t)(b + lane);
      frame_point(T, T + 9, Rn(pos[0]), Rn(pos[1]), Rn(pos[2]), pf);
      const Rn cos_angle = view_cos(T, pf, normal);
      score[lane] = __double2float_rn(__dadd_rn((double)rp_ncc(RpSmemTaps{s}, ids[w], n, lane), cos_angle.v));
    }
  } else {
    for (int j = lane; j < n; j += 32) a.mean_out[b + j] = rp_mean(a.patch + 64 * (size_t)(b + j), a.mean[b + j]);
    __syncwarp();
    const RpGlobalTaps t{a.patch + 64 * (size_t)b, a.mean_out + b};
    for (int r = lane; r < n; r += 32) {
      Rn pf[3];
      const double *T = a.T + 12 * (size_t)(b + r);
      frame_point(T, T + 9, Rn(pos[0]), Rn(pos[1]), Rn(pos[2]), pf);
      const Rn cos_angle = view_cos(T, pf, normal);
      score[r] = __double2float_rn(__dadd_rn((double)rp_ncc(t, a.id + b, n, r), cos_angle.v));
    }
  }
  __syncwarp();
  if (lane == 0) {
    float best = -1000.0f;
    int ref = -1;
    for (int r = 0; r < n; r++)
      if (score[r] > best) best = score[r], ref = r;
    a.ref[i] = ref;
    L.set_ref(i, ref);
  }
}

}  // namespace esikf
