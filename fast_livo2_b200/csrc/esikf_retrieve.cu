// Scan side of the visual sub-map retrieval, VIOManager::retrieveFromVisualSparseMap (reference src/vio.cpp:386-428 and
// 605-640), on the device (H100, sm_90a): the scan's voxel keys in first-occurrence order, its depth image, and the
// depth-continuity check of the retrieved points against that image.
//
//   ret_scan_kernel        : per scan point (:390-426), one thread: the 0.5 m voxel key as the retrieval spells it
//                            (floor(c / 0.5f) in double, then one less when negative), packed for the sort; the frame pose of
//                            updateFrameState, w2f / w2c, the pt_c[2] > 0 and isInFrame(px.cast<int>(), border) gates, and
//                            the pixel's last writer in scan order by atomicMax of the scan index
//   ret_depth_kernel       : per pixel, the depth float(pt_c[2]) of its last writer, 0 where nobody wrote (the serial loop's
//                            overwrite, whatever order the threads ran in)
//   cub DeviceRadixSort    : stable sort of (packed key, scan index): within a run of equal keys the scan indices ascend
//   ret_head_kernel        : per sorted position, 1 at the head of each run, stored at the head's scan index
//   cub DeviceScan         : exclusive sum of those flags in scan order (entry n: the number of distinct keys)
//   ret_keys_kernel        : each distinct key at its offset: the order of the scan index of the key's first point, which
//                            is the insertion order of sub_feat_map
//   ret_depth_check_kernel : per retrieved point (:614-640), one thread: pt_cam[2] = w2f(pos)[2] with the pose of the scan
//                            call, and the 8 x 8 + 1 taps around (int)pc (the centre skipped, empty taps skipped), discontinuous
//                            when any |pt_cam[2] - depth| > 0.5 in double
//
// Everything is evaluated without FMA contraction in the reference's operation order (Rn, frame_point, world2cam<Rn>): with a
// pinhole camera the depth image is the host's bit for bit. The fisheye projection calls atan, where CUDA's and the host's may
// differ in the last ulp (DESIGN.md §4).

namespace esikf {

#define RET_THREADS 256
#define RET_HALF 4  // patch_size_half of the 8 x 8 patches

struct RetArgs {
  CamDev cam;
  double Rci[9], Pci[3];
  const double *state;      // packed state (device) of the frame pose
  const double *pt;         // [n][pt_stride]: point_w first
  int pt_stride, n, border;
  unsigned long long *key;  // [n] out: packed voxel key
  uint32_t *idx;            // [n] out: the scan index (the sort's values)
  float *depth_pt;          // [n] out: float(pt_c[2]) of the points that write a pixel
  int32_t *win;             // [width * height] set to -1 before: the largest scan index writing the pixel
  int32_t *bad;             // set to 0 before: nonzero when a key leaves the map's key range
};

__device__ __forceinline__ void ret_frame_pose(const double *Rci, const double *Pci, const double *state, double *Rcw, double *Pcw) {
  if (threadIdx.x < 9) Rcw[threadIdx.x] = frame_rcw<Rn>(Rci, state, true, threadIdx.x);
  __syncthreads();
  if (threadIdx.x < 3) Pcw[threadIdx.x] = frame_pcw<Rn>(Rcw, Pci, state, true, threadIdx.x);
  __syncthreads();
}

__global__ void __launch_bounds__(RET_THREADS) ret_scan_kernel(const RetArgs a) {
  __shared__ double Rcw[9], Pcw[3];
  ret_frame_pose(a.Rci, a.Pci, a.state, Rcw, Pcw);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const double *p = a.pt + (size_t)i * a.pt_stride;
  long long k[3];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 3; j++) ok = ret_voxel_key(p[j], k[j]) && ok;
  if (!ok) atomicOr(a.bad, 1);
  a.key[i] = ok ? pack_key(k[0], k[1], k[2]) : 0ull;
  a.idx[i] = (uint32_t)i;
  Rn pf[3];
  frame_point(Rcw, Pcw, Rn(p[0]), Rn(p[1]), Rn(p[2]), pf);
  if (!(pf[2].v > 0.0)) return;
  Rn u, v;
  world2cam(a.cam, pf[0], pf[1], pf[2], u, v);
  // px.cast<int>(): truncation toward zero. Out of int range the host's conversion gives INT_MIN and the device's saturates:
  // both fail the test. NaN gives INT_MIN on the host, 0 on the device: rejected here, as the host's INT_MIN is.
  if (u.v != u.v || v.v != v.v) return;
  const int ui = (int)u.v, vi = (int)v.v;
  if (!(ui >= a.border && ui < a.cam.width - a.border && vi >= a.border && vi < a.cam.height - a.border)) return;
  a.depth_pt[i] = (float)pf[2].v;
  atomicMax(a.win + (long)a.cam.width * vi + ui, i);
}

__global__ void ret_depth_kernel(const int32_t *__restrict__ win, const float *__restrict__ depth_pt, int npix, float *__restrict__ depth) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= npix) return;
  const int w = win[q];
  depth[q] = w < 0 ? 0.0f : depth_pt[w];
}

// head[sidx[j]] = 1 when sorted position j starts a run of equal keys (its scan index is the run's smallest); head[n] = 0
__global__ void ret_head_kernel(const unsigned long long *__restrict__ skey, const uint32_t *__restrict__ sidx, int n, int32_t *__restrict__ head) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j > n) return;
  if (j == n) {
    head[n] = 0;
    return;
  }
  head[sidx[j]] = (j == 0 || skey[j] != skey[j - 1]) ? 1 : 0;
}

__global__ void ret_keys_kernel(const int32_t *__restrict__ head, const int32_t *__restrict__ dst, const unsigned long long *__restrict__ key, int n,
                                int32_t *__restrict__ keys_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !head[i]) return;
  const unsigned long long k = key[i];
  int32_t *o = keys_out + 3 * (size_t)dst[i];
  o[0] = (int32_t)((long long)(k >> 42) - ESIKF_KEY_BIAS);
  o[1] = (int32_t)((long long)((k >> 21) & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS);
  o[2] = (int32_t)((long long)(k & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS);
}

struct DepthCheckArgs {
  double Rci[9], Pci[3];
  const double *state;  // the packed state the depth image was made with
  const double *pos;    // [n][3] VisualPoint::pos_
  const double *pc;     // [n][2] the caller's w2c(pos_)
  int n, width, height;
  const float *depth;   // [height][width]
  uint8_t *flag;        // [n] out: depth_continous
};

__global__ void __launch_bounds__(RET_THREADS) ret_depth_check_kernel(const DepthCheckArgs a) {
  __shared__ double Rcw[9], Pcw[3];
  ret_frame_pose(a.Rci, a.Pci, a.state, Rcw, Pcw);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const double *p = a.pos + 3 * (size_t)i;
  Rn pf[3];
  frame_point(Rcw, Pcw, Rn(p[0]), Rn(p[1]), Rn(p[2]), pf);
  const double z = pf[2].v;
  // int(pc[0]), int(pc[1]); a tap outside the image is empty (the reference's linear index would leave the row or the buffer,
  // which a retrieved point, inside isInFrame(·, border >= 4), never makes it do)
  const long long u0 = (long long)(int)a.pc[2 * (size_t)i], v0 = (long long)(int)a.pc[2 * (size_t)i + 1];
  bool disc = false;
  for (int u = -RET_HALF; u <= RET_HALF && !disc; u++)
    for (int v = -RET_HALF; v <= RET_HALF; v++) {
      if (u == 0 && v == 0) continue;
      const long long x = u0 + u, y = v0 + v;
      if (x < 0 || x >= a.width || y < 0 || y >= a.height) continue;
      const float d = a.depth[a.width * y + x];
      if (d == 0.0f) continue;
      if (fabs(__dsub_rn(z, (double)d)) > 0.5) {  // std::abs(double) of pt_cam[2] - depth
        disc = true;
        break;
      }
    }
  a.flag[i] = disc ? 1 : 0;
}

}  // namespace esikf
