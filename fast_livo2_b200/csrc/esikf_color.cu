// Coloured scan of LIVMapper::publish_frame_world (reference src/LIVMapper.cpp:1140-1173) on the device (H100, sm_90a).
//
//   rgb_world_kernel   : the world cloud of a LIO tick, RGBpointBodyToWorld (:435-443, 682-690), one thread per point
//   rgb_color_kernel   : per point of that cloud: the frame pose of updateFrameState (vio.cpp:1690-1697), w2f / w2c, the pf[2]
//                        and isInFrame(pc.cast<int>(), 3) gates, getInterpolatedPixel (vio.cpp:1742-1760) on the BGR image and
//                        the strict pf.norm() > blind_rgb_points gate; one thread per point, a keep flag and B G R out
//   cub DeviceScan     : stable offsets of the kept points (exclusive sum of the keep flags; entry n is the number kept)
//   rgb_scatter_kernel : the survivors in cloud order: xyz, B G R, cloud index
//
// Everything is evaluated without FMA contraction (Rn, dot3_rn, explicit float rounding), in the reference's operation order:
// with a pinhole camera the kept set, xyz and colours are the host's bit for bit. The fisheye projection calls atan, where
// CUDA's and the host's may differ in the last ulp (DESIGN.md §4).

namespace esikf {

struct RgbWorldArgs {
  const float *body;    // [n][3] body-frame points (may alias `world`: each thread reads its point before writing it)
  float *world;         // [n][3] out
  int n;
  const double *state;  // packed state (device): rot_end, pos_end
  double extR[9], extT[3];
};
__global__ void __launch_bounds__(256) rgb_world_kernel(const RgbWorldArgs a) {
  __shared__ double sR[9], st[3];
  if (threadIdx.x < 9) sR[threadIdx.x] = a.state[S_R + threadIdx.x];
  if (threadIdx.x < 3) st[threadIdx.x] = a.state[S_P + threadIdx.x];
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  float w[3];
  world_point_f(sR, st, a.extR, a.extT, a.body[3 * (size_t)i], a.body[3 * (size_t)i + 1], a.body[3 * (size_t)i + 2], w);
  for (int k = 0; k < 3; k++) a.world[3 * (size_t)i + k] = w[k];
}

struct RgbColorArgs {
  const float *cloud;   // [n][3] world points
  int n;
  const uint8_t *bgr;   // [height][width][3], 8-bit B G R
  CamDev cam;
  double Rci[9], Pci[3];
  const double *state;  // packed state (device) of the frame pose
  double blind;         // publish/blind_rgb_points
  int32_t *keep;        // [n + 1] out: 1 = published; keep[n] = 0
  uint8_t *color;       // [n][3] out: B G R (written where keep)
};
__global__ void __launch_bounds__(256) rgb_color_kernel(const RgbColorArgs a) {
  __shared__ double Rcw[9], Pcw[3];
  if (threadIdx.x < 9) Rcw[threadIdx.x] = frame_rcw<Rn>(a.Rci, a.state, true, threadIdx.x);
  __syncthreads();
  if (threadIdx.x < 3) Pcw[threadIdx.x] = frame_pcw<Rn>(Rcw, a.Pci, a.state, true, threadIdx.x);
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) {
    if (i == a.n) a.keep[i] = 0;
    return;
  }
  // V3D p_w(float x, y, z); pf = new_frame_->w2f(p_w) = Rcw p_w + Pcw
  const Rn X = (double)a.cloud[3 * (size_t)i], Y = (double)a.cloud[3 * (size_t)i + 1], Z = (double)a.cloud[3 * (size_t)i + 2];
  Rn pf[3];
  frame_point(Rcw, Pcw, X, Y, Z, pf);
  const Rn pf0 = pf[0], pf1 = pf[1], pf2 = pf[2];
  int keep = 0;
  if (!(pf2 < 0.0)) {
    Rn u, v;
    world2cam(a.cam, pf0, pf1, pf2, u, v);
    // isInFrame(pc.cast<int>(), 3): truncation toward zero. Out of int range (pf2 near 0) the host's conversion gives INT_MIN
    // and the device's saturates: both fail the test, as does NaN (host INT_MIN, device 0).
    const int ui = (int)u.v, vi = (int)v.v;
    const int W = a.cam.width;
    if (ui >= 3 && ui < W - 3 && vi >= 3 && vi < a.cam.height - 3) {
      // getInterpolatedPixel: float pixel position, weights through double (1.0 - s), float sums left to right
      const float u_ref = (float)u.v, v_ref = (float)v.v;
      const int u_i = (int)floorf(u_ref), v_i = (int)floorf(v_ref);
      const float su = __fsub_rn(u_ref, (float)u_i), sv = __fsub_rn(v_ref, (float)v_i);
      const float w_tl = (float)__dmul_rn(__dsub_rn(1.0, (double)su), __dsub_rn(1.0, (double)sv));
      const float w_tr = (float)__dmul_rn((double)su, __dsub_rn(1.0, (double)sv));
      const float w_bl = (float)__dmul_rn(__dsub_rn(1.0, (double)su), (double)sv);
      const float w_br = __fmul_rn(su, sv);
      const long row = 3L * W;
      const uint8_t *p = a.bgr + ((long)v_i * W + u_i) * 3;
      uint8_t *c = a.color + 3 * (size_t)i;
#pragma unroll
      for (int ch = 0; ch < 3; ch++)  // B, G, R; PointXYZRGB's uint8 fields take the float by truncation
        c[ch] = (uint8_t)bil(w_tl, w_tr, w_bl, w_br, (float)p[ch], (float)p[ch + 3], (float)p[ch + row], (float)p[ch + row + 3]);
      keep = sqrt(pf0 * pf0 + pf1 * pf1 + pf2 * pf2) > a.blind;  // pf.norm() > blind_rgb_points
    }
  }
  a.keep[i] = keep;
}

// laserCloudWorldRGB->push_back of every kept point i at dst[i] (the exclusive sum of the keep flags).
__global__ void rgb_scatter_kernel(const int32_t *__restrict__ keep, const int32_t *__restrict__ dst, int n, const float *__restrict__ cloud,
                                   const uint8_t *__restrict__ color, float *__restrict__ xyz_out, uint8_t *__restrict__ bgr_out, int32_t *__restrict__ index_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !keep[i]) return;
  const size_t p = (size_t)dst[i];
  for (int k = 0; k < 3; k++) xyz_out[3 * p + k] = cloud[3 * (size_t)i + k], bgr_out[3 * p + k] = color[3 * (size_t)i + k];
  index_out[p] = i;
}

}  // namespace esikf
