// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header). PARITY UNPINNED.
// Restatement of src/vio.cpp (VIO ESIKF update, patch extraction, affine warp) and of the
// vikit camera arithmetic it calls.
#include "orc_vio.hpp"
#include <cfloat>
#include <limits>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace orc {

// vikit PinholeCamera::world2cam / EquidistantCamera::world2cam (restated, unpinned).
V2 Camera::world2cam(const V3 &xyz_c) const {
  double x = xyz_c[0] / xyz_c[2], y = xyz_c[1] / xyz_c[2];  // vk::project2d
  V2 px;
  if (model == 0) {
    bool distortion = std::fabs(d[0]) > 0.0000001;
    if (!distortion) {
      px[0] = fx * x + cx;
      px[1] = fy * y + cy;
    } else {
      double r2 = x * x + y * y;
      double r4 = r2 * r2;
      double r6 = r4 * r2;
      double a1 = 2 * x * y;
      double a2 = r2 + 2 * x * x;
      double a3 = r2 + 2 * y * y;
      double cdist = 1 + d[0] * r2 + d[1] * r4 + d[4] * r6;
      double xd = x * cdist + d[2] * a1 + d[3] * a2;
      double yd = y * cdist + d[2] * a3 + d[3] * a1;
      px[0] = xd * fx + cx;
      px[1] = yd * fy + cy;
    }
  } else {
    double r = std::sqrt(x * x + y * y);
    double theta = std::atan(r);
    double t2 = theta * theta, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
    double theta_d = theta * (1 + d[0] * t2 + d[1] * t4 + d[2] * t6 + d[3] * t8);
    double scaling = (r > 1e-8) ? theta_d / r : 1.0;
    px[0] = fx * x * scaling + cx;
    px[1] = fy * y * scaling + cy;
  }
  return px;
}

// vikit cam2world returns a unit bearing vector. The distorted pinhole path of vikit calls
// cv::undistortPoints (float, 5 fixed-point iterations); restated here in double.
V3 Camera::cam2world(const V2 &px) const {
  double x0 = (px[0] - cx) / fx, y0 = (px[1] - cy) / fy;
  double x = x0, y = y0;
  if (model == 0) {
    if (std::fabs(d[0]) > 0.0000001) {
      for (int it = 0; it < 5; it++) {
        double r2 = x * x + y * y;
        double icdist = 1.0 / (1 + ((d[4] * r2 + d[1]) * r2 + d[0]) * r2);
        double dx = 2 * d[2] * x * y + d[3] * (r2 + 2 * x * x);
        double dy = d[2] * (r2 + 2 * y * y) + 2 * d[3] * x * y;
        x = (x0 - dx) * icdist;
        y = (y0 - dy) * icdist;
      }
    }
  } else {
    double theta_d = std::sqrt(x0 * x0 + y0 * y0);
    if (theta_d > 1e-8) {
      double theta = theta_d;
      for (int it = 0; it < 10; it++) {
        double t2 = theta * theta, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
        theta = theta_d / (1 + d[0] * t2 + d[1] * t4 + d[2] * t6 + d[3] * t8);
      }
      double scaling = std::tan(theta) / theta_d;
      x = x0 * scaling;
      y = y0 * scaling;
    }
  }
  V3 f = v3(x, y, 1.0);
  return f / norm(f);
}

// vk::interpolateMat_8u (vikit/vision.h): floor + 4-tap bilinear on uint8, float weights.
float interpolateMat_8u(const Image &mat, float u, float v) {
  int x = (int)std::floor(u);
  int y = (int)std::floor(v);
  float subpix_x = u - x;
  float subpix_y = v - y;
  float w00 = (1.0f - subpix_x) * (1.0f - subpix_y);
  float w01 = (1.0f - subpix_x) * subpix_y;
  float w10 = subpix_x * (1.0f - subpix_y);
  float w11 = 1.0f - w00 - w01 - w10;  // vikit computes the last weight as the remainder, not as a product
  const int stride = mat.cols;
  const uint8_t *ptr = mat.data + y * stride + x;
  return w00 * ptr[0] + w01 * ptr[stride] + w10 * ptr[1] + w11 * ptr[stride + 1];
}

// src/vio.cpp:29-39
void VIOManager::setImuToLidarExtrinsic(const V3 &transl, const M3 &rot) {
  Pli = -(T(rot) * transl);
  Rli = T(rot);
}
void VIOManager::setLidarToCameraExtrinsic(const M3 &R, const V3 &P) {
  Rcl = R;
  Pcl = P;
}
// src/vio.cpp:41-65,150-154
void VIOManager::initializeVIO() {
  fx = cam.fx;
  fy = cam.fy;
  width = cam.width;
  height = cam.height;
  Rci = Rcl * Rli;
  Pci = Rcl * Pli + Pcl;
  Jdphi_dR = Rci;
  V3 Pic = -(T(Rci) * Pci);
  M3 tmp = skew(Pic);
  Jdp_dR = -(Rci * tmp);
  patch_size_total = patch_size * patch_size;
  patch_size_half = patch_size / 2;
  G = M19::Zero();
  H_T_H = M19::Zero();
}

// src/vio.cpp:189-201
void VIOManager::computeProjectionJacobian(const V3 &p, Mat<2, 3> &J) {
  const double x = p[0];
  const double y = p[1];
  const double z_inv = 1. / p[2];
  const double z_inv_2 = z_inv * z_inv;
  J(0, 0) = fx * z_inv;
  J(0, 1) = 0.0;
  J(0, 2) = -fx * x * z_inv_2;
  J(1, 0) = 0.0;
  J(1, 1) = fy * z_inv;
  J(1, 2) = -fy * y * z_inv_2;
}

// Raw pointer reads in the reference (img.data + linear offset). The oracle reproduces the
// linear addressing and returns 0 outside [0, rows*cols) where the reference would read
// out of the buffer (SURVEY §7 "out-of-bounds image reads").
static inline int pix(const Image &img, long idx) {
  if (idx < 0 || idx >= (long)img.rows * img.cols) return 0;
  return img.data[idx];
}

// src/vio.cpp:203-225
void VIOManager::getImagePatch(const Image &img, const V2 &pc, float *patch_tmp, int level) {
  const float u_ref = pc[0];
  const float v_ref = pc[1];
  const int scale = (1 << level);
  const int u_ref_i = floorf(pc[0] / scale) * scale;
  const int v_ref_i = floorf(pc[1] / scale) * scale;
  const float subpix_u_ref = (u_ref - u_ref_i) / scale;
  const float subpix_v_ref = (v_ref - v_ref_i) / scale;
  const float w_ref_tl = (1.0 - subpix_u_ref) * (1.0 - subpix_v_ref);
  const float w_ref_tr = subpix_u_ref * (1.0 - subpix_v_ref);
  const float w_ref_bl = (1.0 - subpix_u_ref) * subpix_v_ref;
  const float w_ref_br = subpix_u_ref * subpix_v_ref;
  for (int x = 0; x < patch_size; x++) {
    long base = (long)(v_ref_i - patch_size_half * scale + x * scale) * width + (u_ref_i - patch_size_half * scale);
    for (int y = 0; y < patch_size; y++, base += scale) {
      patch_tmp[patch_size_total * level + x * patch_size + y] = w_ref_tl * pix(img, base) + w_ref_tr * pix(img, base + scale) +
                                                                 w_ref_bl * pix(img, base + (long)scale * width) +
                                                                 w_ref_br * pix(img, base + (long)scale * width + scale);
    }
  }
}

// src/vio.cpp:252-273
void VIOManager::getWarpMatrixAffineHomography(const Camera &cam, const V2 &px_ref, const V3 &xyz_ref, const V3 &normal_ref,
                                               const SE3 &T_cur_ref, const int level_ref, M2 &A_cur_ref) {
  const V3 t = T_cur_ref.inverse().t;
  const M3 H_cur_ref = T_cur_ref.R * (dot(normal_ref, xyz_ref) * M3::Identity() - t * T(normal_ref));
  const int kHalfPatchSize = 4;
  V2 du, dv;
  du[0] = px_ref[0] + (double)(kHalfPatchSize * (1 << level_ref)), du[1] = px_ref[1];
  dv[0] = px_ref[0], dv[1] = px_ref[1] + (double)(kHalfPatchSize * (1 << level_ref));
  V3 f_du_ref = cam.cam2world(du);
  V3 f_dv_ref = cam.cam2world(dv);
  const V3 f_cur = H_cur_ref * xyz_ref;
  const V3 f_du_cur = H_cur_ref * f_du_ref;
  const V3 f_dv_cur = H_cur_ref * f_dv_ref;
  V2 px_cur = cam.world2cam(f_cur);
  V2 px_du_cur = cam.world2cam(f_du_cur);
  V2 px_dv_cur = cam.world2cam(f_dv_cur);
  A_cur_ref(0, 0) = (px_du_cur[0] - px_cur[0]) / kHalfPatchSize;
  A_cur_ref(1, 0) = (px_du_cur[1] - px_cur[1]) / kHalfPatchSize;
  A_cur_ref(0, 1) = (px_dv_cur[0] - px_cur[0]) / kHalfPatchSize;
  A_cur_ref(1, 1) = (px_dv_cur[1] - px_cur[1]) / kHalfPatchSize;
}

// src/vio.cpp:292-318
void VIOManager::warpAffine(const M2 &A_cur_ref, const Image &img_ref, const V2 &px_ref, const int level_ref, const int search_level,
                            const int pyramid_level, const int halfpatch_size, float *patch) {
  (void)level_ref;
  const int patch_size = halfpatch_size * 2;
  const M2 Ainv = inverse2(A_cur_ref);
  const float A00 = (float)Ainv(0, 0), A01 = (float)Ainv(0, 1), A10 = (float)Ainv(1, 0), A11 = (float)Ainv(1, 1);  // .cast<float>()
  if (std::isnan(A00)) return;  // :297-301
  const float pxr0 = (float)px_ref[0], pxr1 = (float)px_ref[1];
  float *patch_ptr = patch;
  for (int y = 0; y < patch_size; ++y) {
    for (int x = 0; x < patch_size; ++x) {
      float pp0 = (float)(x - halfpatch_size), pp1 = (float)(y - halfpatch_size);
      pp0 *= (1 << search_level), pp1 *= (1 << search_level);
      pp0 *= (1 << pyramid_level), pp1 *= (1 << pyramid_level);
      const float px0 = (A00 * pp0 + A01 * pp1) + pxr0;
      const float px1 = (A10 * pp0 + A11 * pp1) + pxr1;
      // the reference's in-frame test (:312) written so that a NaN position (singular A with non-zero entries: inf * 0 or
      // inf - inf) counts as outside; the reference would hand NaN to vk::interpolateMat_8u and read out of bounds
      if (!(px0 >= 0 && px1 >= 0 && px0 < img_ref.cols - 1 && px1 < img_ref.rows - 1))
        patch_ptr[patch_size_total * pyramid_level + y * patch_size + x] = 0;
      else
        patch_ptr[patch_size_total * pyramid_level + y * patch_size + x] = (float)interpolateMat_8u(img_ref, px0, px1);
    }
  }
}

// src/vio.cpp:320-331
int VIOManager::getBestSearchLevel(const M2 &A_cur_ref, const int max_level) {
  int search_level = 0;
  double D = A_cur_ref(0, 0) * A_cur_ref(1, 1) - A_cur_ref(0, 1) * A_cur_ref(1, 0);
  while (D > 3.0 && search_level < max_level) {
    search_level += 1;
    D *= 0.25;
  }
  return search_level;
}

// src/vio.cpp:784-802
void VIOManager::computeJacobianAndUpdateEKF(const Image &img) {
  memset(&stats_, 0, sizeof(stats_));
  if (total_points == 0) return;
  for (int level = patch_pyrimid_level - 1; level >= 0; level--) {  // :790-798
    if (inverse_composition_en) {
      has_ref_patch_cache = false;
      updateStateInverse(img, level);
    } else {
      updateState(img, level);
    }
  }
  state->cov = state->cov - G * state->cov;  // :800
  // updateFrameState(*state) :801 / :1690-1697
  M3 Rwi = state->rot_end;
  V3 Pwi = state->pos_end;
  Rcw = Rci * T(Rwi);
  Pcw = -((Rci * T(Rwi)) * Pwi) + Pci;
}

// src/vio.cpp:1520-1688
void VIOManager::updateState(const Image &img, int level) {
  if (total_points == 0) return;
  StatesGroup old_state = (*state);
  bool EKF_end = false;
  float last_error = std::numeric_limits<float>::max();
  const int H_DIM = total_points * patch_size_total;
  std::vector<double> z(H_DIM, 0.0);               // VectorXd z      :1531-1532
  std::vector<double> H_sub((size_t)H_DIM * 7, 0.0);  // MatrixXd H_sub  :1533-1534
  errors.resize(total_points);

  for (int iteration = 0; iteration < max_iterations; iteration++) {
    M3 Rwi = state->rot_end;
    V3 Pwi = state->pos_end;
    Rcw = Rci * T(Rwi);
    Pcw = -((Rci * T(Rwi)) * Pwi) + Pci;
    Jdp_dt = Rci * T(Rwi);

    float error = 0.0;
    int n_meas = 0;
    // #pragma omp parallel for reduction(+:error, n_meas)  (:1552-1555). The reduction
    // order is unspecified in the reference; here each thread owns a contiguous static
    // chunk and the partial sums are combined in thread order, so results are reproducible.
    int nthreads = omp_threads_ < 1 ? 1 : omp_threads_;
    std::vector<float> error_part(nthreads, 0.0f);
    std::vector<int> n_part(nthreads, 0);
#ifdef _OPENMP
#pragma omp parallel for num_threads(nthreads) schedule(static, 1)
#endif
    for (int th = 0; th < nthreads; th++) {
      int chunk = (total_points + nthreads - 1) / nthreads;
      int i0 = th * chunk, i1 = (i0 + chunk < total_points) ? i0 + chunk : total_points;
      float error_t = 0.0f;
      int n_t = 0;
      for (int i = i0; i < i1; i++) {
        Mat<1, 2> Jimg;
        Mat<2, 3> Jdpi;
        Mat<1, 3> Jdphi, Jdp, JdR, Jdt;
        float patch_error = 0.0;
        int search_level = search_levels[i];
        int pyramid_level = level + search_level;
        int scale = (1 << pyramid_level);
        float inv_scale = 1.0f / scale;

        V3 pt_pos = v3(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]);
        V3 pf = Rcw * pt_pos + Pcw;
        V2 pc = cam.world2cam(pf);
        computeProjectionJacobian(pf, Jdpi);
        M3 p_hat = skew(pf);

        float u_ref = pc[0];
        float v_ref = pc[1];
        int u_ref_i = floorf(pc[0] / scale) * scale;
        int v_ref_i = floorf(pc[1] / scale) * scale;
        float subpix_u_ref = (u_ref - u_ref_i) / scale;
        float subpix_v_ref = (v_ref - v_ref_i) / scale;
        float w_ref_tl = (1.0 - subpix_u_ref) * (1.0 - subpix_v_ref);
        float w_ref_tr = subpix_u_ref * (1.0 - subpix_v_ref);
        float w_ref_bl = (1.0 - subpix_u_ref) * subpix_v_ref;
        float w_ref_br = subpix_u_ref * subpix_v_ref;

        std::vector<float> P(warp_patch.begin() + (size_t)i * patch_size_total * patch_pyrimid_level,
                             warp_patch.begin() + (size_t)(i + 1) * patch_size_total * patch_pyrimid_level);  // copy at :1591
        double inv_ref_expo = inv_expo_list[i];

        for (int x = 0; x < patch_size; x++) {
          long b = (long)(v_ref_i + x * scale - patch_size_half * scale) * width + u_ref_i - patch_size_half * scale;
          const long sw = (long)scale * width;
          for (int y = 0; y < patch_size; ++y, b += scale) {
            float du = 0.5f * ((w_ref_tl * pix(img, b + scale) + w_ref_tr * pix(img, b + scale * 2) + w_ref_bl * pix(img, b + sw + scale) +
                                w_ref_br * pix(img, b + sw + scale * 2)) -
                               (w_ref_tl * pix(img, b - scale) + w_ref_tr * pix(img, b) + w_ref_bl * pix(img, b + sw - scale) +
                                w_ref_br * pix(img, b + sw)));
            float dv = 0.5f * ((w_ref_tl * pix(img, b + sw) + w_ref_tr * pix(img, b + scale + sw) + w_ref_bl * pix(img, b + 2 * sw) +
                                w_ref_br * pix(img, b + 2 * sw + scale)) -
                               (w_ref_tl * pix(img, b - sw) + w_ref_tr * pix(img, b - sw + scale) + w_ref_bl * pix(img, b) +
                                w_ref_br * pix(img, b + scale)));
            Jimg(0, 0) = du, Jimg(0, 1) = dv;
            Jimg = Jimg * state->inv_expo_time;
            Jimg = Jimg * (double)inv_scale;
            Jdphi = (Jimg * Jdpi) * p_hat;
            Jdp = (-Jimg) * Jdpi;
            JdR = Jdphi * Jdphi_dR + Jdp * Jdp_dR;
            Jdt = Jdp * Jdp_dt;

            double cur_value = w_ref_tl * pix(img, b) + w_ref_tr * pix(img, b + scale) + w_ref_bl * pix(img, b + sw) + w_ref_br * pix(img, b + sw + scale);
            double res = state->inv_expo_time * cur_value - inv_ref_expo * P[patch_size_total * level + x * patch_size + y];

            size_t row = (size_t)i * patch_size_total + x * patch_size + y;
            z[row] = res;
            patch_error += res * res;
            n_t += 1;
            double *h = &H_sub[row * 7];
            h[0] = JdR(0, 0), h[1] = JdR(0, 1), h[2] = JdR(0, 2), h[3] = Jdt(0, 0), h[4] = Jdt(0, 1), h[5] = Jdt(0, 2);
            if (exposure_estimate_en) h[6] = cur_value;
          }
        }
        errors[i] = patch_error;
        error_t += patch_error;
      }
      error_part[th] = error_t;
      n_part[th] = n_t;
    }
    for (int th = 0; th < nthreads; th++) error += error_part[th], n_meas += n_part[th];

    error = error / n_meas;
    if (level < 8 && iteration < 8) stats_.error_trace[level][iteration] = error;
    if (level < 8) stats_.iters_per_level[level] = iteration + 1;
    stats_.total_iters++;

    if (error <= last_error) {
      old_state = (*state);
      last_error = error;
      H_T_H = M19::Zero();
      G = M19::Zero();
      // H_T_H.block<7,7>(0,0) = H_sub_T * H_sub  (:1660) ; HTz = H_sub_T * z  (:1662)
      Mat<7, 7> HTH7 = Mat<7, 7>::Zero();
      Mat<7, 1> HTz = Mat<7, 1>::Zero();
      for (int r = 0; r < H_DIM; r++) {
        const double *h = &H_sub[(size_t)r * 7];
        for (int a = 0; a < 7; a++) {
          HTz[a] += h[a] * z[r];
          for (int b = 0; b < 7; b++) HTH7(a, b) += h[a] * h[b];
        }
      }
      set_block(H_T_H, 0, 0, HTH7);
      M19 K_1 = inverse_pplu(H_T_H + inverse_pplu(state->cov / img_point_cov));  // :1661
      V19 vec = state_propagat->boxminus(*state);                                 // :1664
      Mat<19, 7> K17 = block<19, 7>(K_1, 0, 0);
      Mat<19, 7> G7 = K17 * HTH7;  // :1665
      set_block(G, 0, 0, G7);
      V19 solution = (-K17) * HTz + vec - G7 * block<7, 1>(vec, 0, 0);  // :1667
      if (level < 8 && iteration < 8) {
        memcpy(stats_.HTH[level][iteration], HTH7.a, sizeof(double) * 49);
        memcpy(stats_.HTz[level][iteration], HTz.a, sizeof(double) * 7);
        memcpy(stats_.solution[level][iteration], solution.a, sizeof(double) * 19);
      }
      state->boxplus(solution);
      V3 rot_add = block<3, 1>(solution, 0, 0);
      V3 t_add = block<3, 1>(solution, 3, 0);
      if (level < 8) stats_.accepted_per_level[level]++;
      if ((norm(rot_add) * 57.3f < 0.001f) && (norm(t_add) * 100.0f < 0.001f)) EKF_end = true;  // :1675
    } else {
      (*state) = old_state;
      EKF_end = true;
    }
    if (iteration == max_iterations || EKF_end) break;
  }
}

// src/vio.cpp:1327-1396 — Jacobian rows of every reference patch pixel w.r.t. the WORLD-frame pose perturbation, from the
// gradients of the reference image (the pyramid level only sets the tap stride; search levels are not used here).
void VIOManager::precomputeReferencePatches(int level) {
  if (total_points == 0) return;
  const int H_DIM = total_points * patch_size_total;
  H_sub_inv.assign((size_t)H_DIM * 6, 0.0);
  for (int i = 0; i < total_points; i++) {
    const int scale = (1 << level);
    const Image &img = ref_imgs[ref_img_index[i]];
    V3 pt_pos = v3(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]);
    V3 rp = v3(ref_pos[3 * i], ref_pos[3 * i + 1], ref_pos[3 * i + 2]);
    double depth = norm(pt_pos - rp);
    V3 pf = v3(ref_f[3 * i], ref_f[3 * i + 1], ref_f[3 * i + 2]) * depth;
    V2 pc;
    pc[0] = ref_px[2 * i], pc[1] = ref_px[2 * i + 1];
    M3 R_ref_w;
    for (int k = 0; k < 9; k++) R_ref_w.a[k] = ref_R[9 * (size_t)i + k];
    Mat<2, 3> Jdpi;
    computeProjectionJacobian(pf, Jdpi);
    M3 p_w_hat = skew(pt_pos);

    const float u_ref = pc[0];
    const float v_ref = pc[1];
    const int u_ref_i = floorf(pc[0] / scale) * scale;
    const int v_ref_i = floorf(pc[1] / scale) * scale;
    const float subpix_u_ref = (u_ref - u_ref_i) / scale;
    const float subpix_v_ref = (v_ref - v_ref_i) / scale;
    const float w_ref_tl = (1.0 - subpix_u_ref) * (1.0 - subpix_v_ref);
    const float w_ref_tr = subpix_u_ref * (1.0 - subpix_v_ref);
    const float w_ref_bl = (1.0 - subpix_u_ref) * subpix_v_ref;
    const float w_ref_br = subpix_u_ref * subpix_v_ref;
    const int w = img.cols;  // the reference indexes the reference image with the manager's `width`; same size here
    for (int x = 0; x < patch_size; x++) {
      long b = (long)(v_ref_i + x * scale - patch_size_half * scale) * w + u_ref_i - patch_size_half * scale;
      const long sw = (long)scale * w;
      for (int y = 0; y < patch_size; ++y, b += scale) {
        float du = 0.5f * ((w_ref_tl * pix(img, b + scale) + w_ref_tr * pix(img, b + scale * 2) + w_ref_bl * pix(img, b + sw + scale) +
                            w_ref_br * pix(img, b + sw + scale * 2)) -
                           (w_ref_tl * pix(img, b - scale) + w_ref_tr * pix(img, b) + w_ref_bl * pix(img, b + sw - scale) + w_ref_br * pix(img, b + sw)));
        float dv = 0.5f * ((w_ref_tl * pix(img, b + sw) + w_ref_tr * pix(img, b + scale + sw) + w_ref_bl * pix(img, b + 2 * sw) +
                            w_ref_br * pix(img, b + 2 * sw + scale)) -
                           (w_ref_tl * pix(img, b - sw) + w_ref_tr * pix(img, b - sw + scale) + w_ref_bl * pix(img, b) + w_ref_br * pix(img, b + scale)));
        Mat<1, 2> Jimg;
        Jimg(0, 0) = du, Jimg(0, 1) = dv;
        Jimg = Jimg * (1.0 / scale);
        Mat<1, 3> JdR = ((Jimg * Jdpi) * R_ref_w) * p_w_hat;  // :1387
        Mat<1, 3> Jdt = ((-Jimg) * Jdpi) * R_ref_w;           // :1388
        double *h = &H_sub_inv[((size_t)i * patch_size_total + x * patch_size + y) * 6];
        h[0] = JdR(0, 0), h[1] = JdR(0, 1), h[2] = JdR(0, 2), h[3] = Jdt(0, 0), h[4] = Jdt(0, 1), h[5] = Jdt(0, 2);
      }
    }
  }
  has_ref_patch_cache = true;
}

// src/vio.cpp:1398-1518 — serial in the reference (no OpenMP); 6-column H (no exposure column, no exposure factors in the
// residual); the residual is formed in FLOAT (bilinear sum minus the float reference value) and then widened (:1466-1468).
void VIOManager::updateStateInverse(const Image &img, int level) {
  if (total_points == 0) return;
  StatesGroup old_state = (*state);
  bool EKF_end = false;
  float last_error = std::numeric_limits<float>::max();
  const int H_DIM = total_points * patch_size_total;
  std::vector<double> z(H_DIM, 0.0);
  std::vector<double> H_sub((size_t)H_DIM * 6, 0.0);
  errors.resize(total_points);

  for (int iteration = 0; iteration < max_iterations; iteration++) {
    if (has_ref_patch_cache == false) precomputeReferencePatches(level);
    int n_meas = 0;
    float error = 0.0;
    M3 Rwi = state->rot_end;
    V3 Pwi = state->pos_end;
    M3 P_wi_hat = skew(Pwi);
    Rcw = Rci * T(Rwi);
    Pcw = -((Rci * T(Rwi)) * Pwi) + Pci;

    for (int i = 0; i < total_points; i++) {
      float patch_error = 0.0;
      const int scale = (1 << level);
      V3 pt_pos = v3(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]);
      V3 pf = Rcw * pt_pos + Pcw;
      V2 pc = cam.world2cam(pf);

      const float u_ref = pc[0];
      const float v_ref = pc[1];
      const int u_ref_i = floorf(pc[0] / scale) * scale;
      const int v_ref_i = floorf(pc[1] / scale) * scale;
      const float subpix_u_ref = (u_ref - u_ref_i) / scale;
      const float subpix_v_ref = (v_ref - v_ref_i) / scale;
      const float w_ref_tl = (1.0 - subpix_u_ref) * (1.0 - subpix_v_ref);
      const float w_ref_tr = subpix_u_ref * (1.0 - subpix_v_ref);
      const float w_ref_bl = (1.0 - subpix_u_ref) * subpix_v_ref;
      const float w_ref_br = subpix_u_ref * subpix_v_ref;

      const float *P = &warp_patch[(size_t)i * patch_size_total * patch_pyrimid_level];
      for (int x = 0; x < patch_size; x++) {
        long b = (long)(v_ref_i + x * scale - patch_size_half * scale) * width + u_ref_i - patch_size_half * scale;
        const long sw = (long)scale * width;
        for (int y = 0; y < patch_size; ++y, b += scale) {
          double res = w_ref_tl * pix(img, b) + w_ref_tr * pix(img, b + scale) + w_ref_bl * pix(img, b + sw) + w_ref_br * pix(img, b + sw + scale) -
                       P[patch_size_total * level + x * patch_size + y];
          const size_t row = (size_t)i * patch_size_total + x * patch_size + y;
          z[row] = res;
          patch_error += res * res;
          Mat<1, 3> J_dR, J_dt;
          const double *hi = &H_sub_inv[row * 6];
          J_dR(0, 0) = hi[0], J_dR(0, 1) = hi[1], J_dR(0, 2) = hi[2];
          J_dt(0, 0) = hi[3], J_dt(0, 1) = hi[4], J_dt(0, 2) = hi[5];
          Mat<1, 3> JdR = J_dR * Rwi + (J_dt * P_wi_hat) * Rwi;  // :1471
          Mat<1, 3> Jdt = J_dt * Rwi;                            // :1472
          double *h = &H_sub[row * 6];
          h[0] = JdR(0, 0), h[1] = JdR(0, 1), h[2] = JdR(0, 2), h[3] = Jdt(0, 0), h[4] = Jdt(0, 1), h[5] = Jdt(0, 2);
          n_meas++;
        }
      }
      errors[i] = patch_error;
      error += patch_error;
    }
    error = error / n_meas;
    if (level < 8 && iteration < 8) stats_.error_trace[level][iteration] = error;
    if (level < 8) stats_.iters_per_level[level] = iteration + 1;
    stats_.total_iters++;

    if (error <= last_error) {
      old_state = (*state);
      last_error = error;
      H_T_H = M19::Zero();
      G = M19::Zero();
      Mat<6, 6> HTH6 = Mat<6, 6>::Zero();
      Mat<6, 1> HTz = Mat<6, 1>::Zero();
      for (int r = 0; r < H_DIM; r++) {
        const double *h = &H_sub[(size_t)r * 6];
        for (int a = 0; a < 6; a++) {
          HTz[a] += h[a] * z[r];
          for (int b = 0; b < 6; b++) HTH6(a, b) += h[a] * h[b];
        }
      }
      set_block(H_T_H, 0, 0, HTH6);
      M19 K_1 = inverse_pplu(H_T_H + inverse_pplu(state->cov / img_point_cov));  // :1492
      V19 vec = state_propagat->boxminus(*state);
      Mat<19, 6> K16 = block<19, 6>(K_1, 0, 0);
      Mat<19, 6> G6 = K16 * HTH6;  // :1495
      set_block(G, 0, 0, G6);
      V19 solution = (-K16) * HTz + vec - G6 * block<6, 1>(vec, 0, 0);  // :1496
      if (level < 8 && iteration < 8) {
        // diagnostics share the 7 x 7 / 7-vector slots of the forward variant (last row / column zero)
        for (int a = 0; a < 6; a++) {
          stats_.HTz[level][iteration][a] = HTz[a];
          for (int b = 0; b < 6; b++) stats_.HTH[level][iteration][a * 7 + b] = HTH6(a, b);
        }
        memcpy(stats_.solution[level][iteration], solution.a, sizeof(double) * 19);
      }
      state->boxplus(solution);
      V3 rot_add = block<3, 1>(solution, 0, 0);
      V3 t_add = block<3, 1>(solution, 3, 0);
      if (level < 8) stats_.accepted_per_level[level]++;
      if ((norm(rot_add) * 57.3f < 0.001f) && (norm(t_add) * 100.0f < 0.001f)) EKF_end = true;  // :1501
    } else {
      (*state) = old_state;
      EKF_end = true;
    }
    if (iteration == max_iterations || EKF_end) break;
  }
}

}  // namespace orc
