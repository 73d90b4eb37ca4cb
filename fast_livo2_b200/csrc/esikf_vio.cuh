// VIO declarations shared by the update kernels (esikf_vio.cu, esikf_fused.cu), the front-end kernels and the host files:
// the camera model, the frame pose, the image taps and the tensor maps of the image.
#pragma once
#include "esikf_dev.cuh"

namespace esikf {

struct CamDev {
  int model, width, height;
  double fx, fy, cx, cy;
  double d[5];
};

// A double whose every operation is rounded on its own, never contracted into an FMA: what a host compiled without FMA
// contraction (the reference, the oracle) computes. The camera projection and the frame pose below are written once, over
// their number type: plain double in the VIO update kernels (which nvcc contracts), Rn where a result must equal the host's
// bit for bit (the coloured scan, esikf_color.cu).
struct Rn {
  double v;
  __device__ __forceinline__ Rn(double x = 0.0) : v(x) {}
  __device__ __forceinline__ explicit operator double() const { return v; }
  friend __device__ __forceinline__ Rn operator+(Rn a, Rn b) { return __dadd_rn(a.v, b.v); }
  friend __device__ __forceinline__ Rn operator-(Rn a, Rn b) { return __dsub_rn(a.v, b.v); }
  friend __device__ __forceinline__ Rn operator*(Rn a, Rn b) { return __dmul_rn(a.v, b.v); }
  friend __device__ __forceinline__ Rn operator/(Rn a, Rn b) { return __ddiv_rn(a.v, b.v); }
  friend __device__ __forceinline__ Rn operator-(Rn a) { return -a.v; }
  friend __device__ __forceinline__ Rn &operator+=(Rn &a, Rn b) { return a = a + b; }
  friend __device__ __forceinline__ bool operator<(Rn a, Rn b) { return a.v < b.v; }
  friend __device__ __forceinline__ bool operator>(Rn a, Rn b) { return a.v > b.v; }
  friend __device__ __forceinline__ Rn sqrt(Rn a) { return __dsqrt_rn(a.v); }
  friend __device__ __forceinline__ Rn atan(Rn a) { return ::atan(a.v); }  // CUDA's atan: within 2 ulp, not always glibc's
};

// vk::PinholeCamera::world2cam / vk::EquidistantCamera::world2cam (vikit, unpinned; restated from its published algorithm)
template <class T> __device__ __forceinline__ void world2cam(const CamDev &cam, T X, T Y, T Z, T &u, T &v) {
  T x = X / Z, y = Y / Z;
  if (cam.model == 0) {
    if (!(fabs(cam.d[0]) > 0.0000001)) {
      u = cam.fx * x + cam.cx;
      v = cam.fy * y + cam.cy;
    } else {
      T r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
      T a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
      T cdist = 1 + cam.d[0] * r2 + cam.d[1] * r4 + cam.d[4] * r6;
      T xd = x * cdist + cam.d[2] * a1 + cam.d[3] * a2;
      T yd = y * cdist + cam.d[2] * a3 + cam.d[3] * a1;
      u = xd * cam.fx + cam.cx;
      v = yd * cam.fy + cam.cy;
    }
  } else {
    T r = sqrt(x * x + y * y);
    T theta = atan(r);
    T t2 = theta * theta, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
    T theta_d = theta * (1 + cam.d[0] * t2 + cam.d[1] * t4 + cam.d[2] * t6 + cam.d[3] * t8);
    T scaling = (r > 1e-8) ? theta_d / r : 1.0;
    u = cam.fx * x * scaling + cam.cx;
    v = cam.fy * y * scaling + cam.cy;
  }
}
// cam2world -> unit bearing (distorted pinhole: 5 fixed-point iterations as cv::undistortPoints)
__device__ __forceinline__ void cam2world(const CamDev &cam, double u, double v, double f[3]) {
  double x0 = (u - cam.cx) / cam.fx, y0 = (v - cam.cy) / cam.fy;
  double x = x0, y = y0;
  if (cam.model == 0) {
    if (fabs(cam.d[0]) > 0.0000001) {
      for (int it = 0; it < 5; it++) {
        double r2 = x * x + y * y;
        double icdist = 1.0 / (1 + ((cam.d[4] * r2 + cam.d[1]) * r2 + cam.d[0]) * r2);
        double dx = 2 * cam.d[2] * x * y + cam.d[3] * (r2 + 2 * x * x);
        double dy = cam.d[2] * (r2 + 2 * y * y) + 2 * cam.d[3] * x * y;
        x = (x0 - dx) * icdist;
        y = (y0 - dy) * icdist;
      }
    }
  } else {
    double theta_d = sqrt(x0 * x0 + y0 * y0);
    if (theta_d > 1e-8) {
      double theta = theta_d;
      for (int it = 0; it < 10; it++) {
        double t2 = theta * theta, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
        theta = theta_d / (1 + cam.d[0] * t2 + cam.d[1] * t4 + cam.d[2] * t6 + cam.d[3] * t8);
      }
      double scaling = tan(theta) / theta_d;
      x = x0 * scaling;
      y = y0 * scaling;
    }
  }
  double n = sqrt(x * x + y * y + 1.0);
  f[0] = x / n, f[1] = y / n, f[2] = 1.0 / n;
}

// raw img.data + offset reads of the reference, with 0 outside the buffer (the reference would read out of bounds there)
__device__ __forceinline__ float tap(const uint8_t *__restrict__ img, long idx, long npix) {
  return (idx >= 0 && idx < npix) ? (float)__ldg(img + idx) : 0.0f;
}
// w_tl*a + w_tr*b + w_bl*c + w_br*d in float, left to right, no FMA contraction (vio.cpp:1600-1620)
__device__ __forceinline__ float bil(float wtl, float wtr, float wbl, float wbr, float a, float b, float c, float d) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(wtl, a), __fmul_rn(wtr, b)), __fmul_rn(wbl, c)), __fmul_rn(wbr, d));
}

// Tap footprints through the TMA unit (tuning flag ESIKF_TUNE_VIO_TMA): one tiled tensor map of the u8 image per tap
// stride s = 1, 2, 4, 8 — box {W_s bytes, 11 s rows} traversed with elementStrides {1, s} (TMA cannot stride the
// innermost dimension), i.e. 11 image rows of W_s contiguous bytes land in shared memory with ONE instruction issued by
// one lane; the 11 x 11 taps are then picked out at stride s. The box must START on a 16-byte boundary of the innermost
// dimension (an unaligned x coordinate is not a valid start for this descriptor form), so the start pixel is rounded down to a multiple of 16 and W_s = 16 ceil((16 + 10 s) / 16)
// covers the worst offset: 32, 48, 64, 96 bytes. Footprints that leave the image (the reference's raw linear-index reads
// wrap to the neighbouring row there, TMA would zero-fill) and strides 16 / 32 (elementStrides <= 8) keep the per-lane loads.
#define VIO_TMA_MAXLVL 3
#define VIO_TMA_INNER(l) (16u * ((16u + (10u << (l)) + 15u) / 16u))
#define VIO_TMA_TILE_BYTES (11 * 96 + 96)
struct VioTma {
  alignas(64) unsigned char map[VIO_TMA_MAXLVL + 1][128];  // CUtensorMap per level (opaque 128-byte descriptors)
  int enabled;
};

// The frame pose of the packed state `st`, one element per call: Rcw = Rci * Rwi^T (vio.cpp:1542) and, from it,
// Pcw = -Rci Rwi^T Pwi + Pci (:1543). updateFrameState (:1690-1697) is the same arithmetic. global: `st` lies in global memory,
// written by an earlier launch, else it is the CTA's resident copy.
template <class T> __device__ __forceinline__ double frame_rcw(const double *Rci, const double *st, bool global, int e) {
  const int r = e / 3, c = e % 3;
  T s = 0.0;
  for (int k = 0; k < 3; k++) s += T(Rci[r * 3 + k]) * T(ld_state(st + S_R + c * 3 + k, global));
  return (double)s;
}
template <class T> __device__ __forceinline__ double frame_pcw(const double *Rcw, const double *Pci, const double *st, bool global, int r) {
  T s = 0.0;
  for (int k = 0; k < 3; k++) s += T(Rcw[r * 3 + k]) * T(ld_state(st + S_P + k, global));
  return (double)(-s + T(Pci[r]));
}
// Frame::w2f of a world point with that pose: pf = Rcw p_w + Pcw, each row summed left to right
template <class T> __device__ __forceinline__ void frame_point(const double *Rcw, const double *Pcw, T X, T Y, T Z, T pf[3]) {
#pragma unroll
  for (int r = 0; r < 3; r++) pf[r] = T(Rcw[3 * r]) * X + T(Rcw[3 * r + 1]) * Y + T(Rcw[3 * r + 2]) * Z + T(Pcw[r]);
}

// the single-CTA scan of select_scan_kernel (esikf_vio.cu)
#define SELECT_SCAN_THREADS 1024

}  // namespace esikf
