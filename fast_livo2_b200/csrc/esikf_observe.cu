// New observations of the visual sub-map in a VIO tick, VIOManager::updateVisualMapPoints (reference src/vio.cpp:908-967), on
// the device (H100, sm_90a): which entries of the installed sub-map the current frame becomes a new Feature of, and that
// Feature's pixel and level-0 patch.
//
//   obs_flag_kernel    : per sub-map entry, one thread: the converged skip, pc = new_frame_->w2c(pos), delta_pose =
//                        pose_ref * pose_cur.inverse() of the entry's oldest observation, and the add rule
//                        delta_p > 0.5 || delta_theta > 0.3 || |pc - last_px| > 40 (:918-944)
//   select_scan_kernel : stable offsets in entry order (the sub-map selection's single-CTA scan: sub-map counts)
//   obs_scatter_kernel : entry index and pc of every added entry at its offset
//   image_patch_kernel : getImagePatch(img, pc, patch, 0) of the added entries (:928)
//
// Everything is evaluated without FMA contraction in the operation order of the reference's stand-in Eigen / SE3 (Rn): pc is
// the coloured scan's and generateVisualMapPoints' path, and the pose product, the trace and both norms are summed from 0 left
// to right as Matrix::operator*, trace() and squaredNorm() do. delta_theta > 0.3 is not evaluated with acos (CUDA's is not
// glibc's): acos is decreasing, so for x = 0.5 * (trace - 1) it holds exactly when -1 <= x <= cos_max, where cos_max, the
// largest double whose host acos exceeds 0.3, is found on the host (x < -1 makes acos NaN, which fails the test). With a pinhole
// camera every output is the host's bit for bit; the fisheye projection calls atan (DESIGN.md §4).

namespace esikf {

#define OBS_THREADS 256

struct ObsArgs {
  CamDev cam;
  double Rci[9], Pci[3];
  const double *state;        // packed state (device) of the frame pose
  const double *pos;          // [n][3] VisualPoint::pos_ of the installed sub-map
  const uint8_t *converged;   // [n] VisualPoint::is_converged_
  const double *last_T;       // [n][12] obs_.back()->T_f_w_: R row-major, then t
  const double *last_px;      // [n][2] obs_.back()->px_
  int n;
  double cos_max;             // largest x with acos(x) > 0.3 on the host
  uint8_t *flag;              // [n] update_flag
  int32_t *keep;              // [n] the same, for the scan
  double *pc;                 // [n][2] w2c(pos) of every entry that is not converged
};

// pose_cur = new_frame_->T_f_w_ = (Rcw, Pcw) as updateFrameState builds it, and the translation of pose_cur.inverse():
// (Rcw^T Pcw) * -1.0
__device__ __forceinline__ void obs_frame_pose(const ObsArgs &a, double *Rcw, double *Pcw, double *Tinv) {
  if (threadIdx.x < 9) Rcw[threadIdx.x] = frame_rcw<Rn>(a.Rci, a.state, true, threadIdx.x);
  __syncthreads();
  if (threadIdx.x < 3) Pcw[threadIdx.x] = frame_pcw<Rn>(Rcw, a.Pci, a.state, true, threadIdx.x);
  __syncthreads();
  if (threadIdx.x < 3) {
    const int r = threadIdx.x;
    Tinv[r] = -(Rn(0.0) + Rn(Rcw[r]) * Rn(Pcw[0]) + Rn(Rcw[3 + r]) * Rn(Pcw[1]) + Rn(Rcw[6 + r]) * Rn(Pcw[2])).v;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(OBS_THREADS) obs_flag_kernel(const ObsArgs a) {
  __shared__ double Rcw[9], Pcw[3], Tinv[3];
  obs_frame_pose(a, Rcw, Pcw, Tinv);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  bool add = false;
  if (!a.converged[i]) {
    const double *p = a.pos + 3 * (size_t)i;
    Rn pf[3], u, v;
    frame_point(Rcw, Pcw, Rn(p[0]), Rn(p[1]), Rn(p[2]), pf);
    world2cam(a.cam, pf[0], pf[1], pf[2], u, v);
    a.pc[2 * (size_t)i] = u.v, a.pc[2 * (size_t)i + 1] = v.v;
    const double *T = a.last_T + 12 * (size_t)i;
    // delta_pose = pose_ref * pose_cur.inverse(): rotation R_ref Rcw^T (only its diagonal is read), translation
    // t_ref + R_ref Tinv
    Rn trace = 0.0, dp2 = 0.0;
#pragma unroll
    for (int r = 0; r < 3; r++) {
      const Rn d = Rn(0.0) + Rn(T[3 * r]) * Rn(Rcw[3 * r]) + Rn(T[3 * r + 1]) * Rn(Rcw[3 * r + 1]) + Rn(T[3 * r + 2]) * Rn(Rcw[3 * r + 2]);
      const Rn t = Rn(T[9 + r]) + (Rn(0.0) + Rn(T[3 * r]) * Rn(Tinv[0]) + Rn(T[3 * r + 1]) * Rn(Tinv[1]) + Rn(T[3 * r + 2]) * Rn(Tinv[2]));
      trace += d;
      dp2 += t * t;
    }
    const double x = (Rn(0.5) * (trace - Rn(1.0))).v;
    const bool theta = !(trace.v > 3.0 - 1e-6) && x >= -1.0 && x <= a.cos_max;
    const Rn du = u - Rn(a.last_px[2 * (size_t)i]), dv = v - Rn(a.last_px[2 * (size_t)i + 1]);
    add = sqrt(dp2).v > 0.5 || theta || sqrt(Rn(0.0) + du * du + dv * dv).v > 40.0;
  }
  a.flag[i] = add;
  a.keep[i] = add;
}

// entry index and pc of every added entry at its stable offset
__global__ void obs_scatter_kernel(const int32_t *__restrict__ keep, const int32_t *__restrict__ dst, const double *__restrict__ pc, int n,
                                   int32_t *__restrict__ entry_out, double *__restrict__ pc_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !keep[i]) return;
  const int p = dst[i];
  entry_out[p] = i;
  pc_out[2 * (size_t)p] = pc[2 * (size_t)i], pc_out[2 * (size_t)p + 1] = pc[2 * (size_t)i + 1];
}

}  // namespace esikf
