// TEST INFRASTRUCTURE — pins the oracle's VIO half to the reference SOURCE: the reference's own src/vio.cpp, src/frame.cpp and
// src/visual_point.cpp are compiled from where they lie under /root/reference (nothing copied) against the stand-in headers of
// ref_shim/ (a small matrix library answering the Eigen calls, an owning 8-bit cv::Mat with no-op drawing, a matrix-backed
// Sophus::SE3, boost::noncopyable, empty PCL / ROS shells) and driven through C entry points shaped like oracle/orc_capi.cpp's.
// What is NOT the reference's code on this path: vikit (un-vendored, no version pin — README.md:80-84): the pinhole camera model
// and vk::interpolateMat_8u in ref_shim/vikit/ are restatements of the published algorithm. Everything else that
// VIOManager::computeJacobianAndUpdateEKF / updateState / updateStateInverse / precomputeReferencePatches / getImagePatch /
// warpAffine / getWarpMatrixAffineHomography / getBestSearchLevel compute is the reference's own arithmetic.
// Built by oracle/Makefile into oracle/_ref/libfl2_ref_vio.so only where /root/reference exists.
#include <iomanip>
#include <list>
#include <set>
#include <deque>
#include <vector>
#include <numeric>
#include <chrono>
#include <unordered_map>
using namespace std;
typedef unsigned char uchar;
#include <vikit/equidistant_camera.h>
#include "/root/reference/src/voxel_map.cpp"  // VoxelOctoTree::find_correspond etc., referenced by the retrieval code of vio.cpp
#include "/root/reference/src/frame.cpp"
#include "/root/reference/src/visual_point.cpp"
#include "/root/reference/src/vio.cpp"

static void unpack_state(const double *s, StatesGroup &x) {  // packed layout of include/esikf_b200.h
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) x.rot_end(r, c) = s[3 * r + c];
  for (int i = 0; i < 3; i++) x.pos_end[i] = s[9 + i], x.vel_end[i] = s[13 + i], x.bias_g[i] = s[16 + i], x.bias_a[i] = s[19 + i], x.gravity[i] = s[22 + i];
  x.inv_expo_time = s[12];
  for (int r = 0; r < 19; r++)
    for (int c = 0; c < 19; c++) x.cov(r, c) = s[25 + 19 * r + c];
}
static void pack_state(const StatesGroup &x, double *s) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) s[3 * r + c] = x.rot_end(r, c);
  for (int i = 0; i < 3; i++) s[9 + i] = x.pos_end[i], s[13 + i] = x.vel_end[i], s[16 + i] = x.bias_g[i], s[19 + i] = x.bias_a[i], s[22 + i] = x.gravity[i];
  s[12] = x.inv_expo_time;
  for (int r = 0; r < 19; r++)
    for (int c = 0; c < 19; c++) s[25 + 19 * r + c] = x.cov(r, c);
}

struct RefVio {
  VIOManager v;
  StatesGroup st, prop;
  std::vector<VisualPoint *> owned;
  std::vector<cv::Mat> ref_imgs;
  ~RefVio() {
    for (auto *p : owned) delete p;  // ~VisualPoint deletes its observations (and their patches)
    delete v.cam;
  }
};

extern "C" {

// Version of this library: 2 = the stand-in matrix library inverts a fixed 2 x 2 by Eigen's closed form (warpAffine's
// A_cur_ref.inverse()); an older build inverted it by LU, which differs in the last bits when the determinant cancels.
// tests/oracle_bind.py uses the library live only at this version; the Makefile rebuilds a library that does not export it.
int ref_vio_driver_version_2(void) { return 2; }

// cam = [model (0 pinhole / radtan, 1 equidistant), width, height, fx, fy, cx, cy, d0..d4]; cfg = [patch_pyrimid_level, max_iterations, img_point_cov, exposure_estimate_en]
void *ref_vio_create(const double *cam, const double *extR, const double *extT, const double *Rcl, const double *Pcl, const double *cfg) {
  if ((int)cam[0] != 0 && (int)cam[0] != 1) return nullptr;
  RefVio *r = new RefVio;
  VIOManager &v = r->v;
  if ((int)cam[0] == 0)
    v.cam = new vk::PinholeCamera(cam[1], cam[2], 1.0, cam[3], cam[4], cam[5], cam[6], cam[7], cam[8], cam[9], cam[10], cam[11]);
  else
    v.cam = new vk::EquidistantCamera(cam[1], cam[2], 1.0, cam[3], cam[4], cam[5], cam[6], cam[7], cam[8], cam[9], cam[10]);
  M3D R;
  V3D t;
  for (int i = 0; i < 3; i++) {
    t[i] = extT[i];
    for (int j = 0; j < 3; j++) R(i, j) = extR[3 * i + j];
  }
  v.setImuToLidarExtrinsic(t, R);  // LIVMapper.cpp:125-126 -> vio.cpp:29-33
  std::vector<double> Rv(Rcl, Rcl + 9), Pv(Pcl, Pcl + 3);
  v.setLidarToCameraExtrinsic(Rv, Pv);  // vio.cpp:35-39
  v.grid_size = 40, v.grid_n_width = 0, v.grid_n_height = 0;
  v.patch_size = 8, v.patch_pyrimid_level = (int)cfg[0], v.max_iterations = (int)cfg[1], v.img_point_cov = cfg[2];
  v.exposure_estimate_en = cfg[3] != 0, v.normal_en = true, v.inverse_composition_en = false, v.raycast_en = false, v.colmap_output_en = false, v.ncc_en = false;
  v.outlier_threshold = 1000, v.ncc_thre = 0, v.plot_flag = false, v.has_ref_patch_cache = false;
  v.state = &r->st, v.state_propagat = &r->prop;
  v.initializeVIO();
  return r;
}
void ref_vio_destroy(void *h) { delete (RefVio *)h; }

static void fill_submap(RefVio *r, int n_pts, const double *pos, const float *warp_patch, const int32_t *search_levels, const double *inv_expo_list) {
  VIOManager &v = r->v;
  SubSparseMap &sub = *v.visual_submap;
  sub.reset();
  for (auto *p : r->owned) delete p;
  r->owned.clear();
  const int wl = v.warp_len;
  for (int i = 0; i < n_pts; i++) {
    VisualPoint *pt = new VisualPoint(V3D(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]));
    r->owned.push_back(pt);
    sub.voxel_points.push_back(pt);
    sub.warp_patch.emplace_back(warp_patch + (size_t)i * wl, warp_patch + (size_t)(i + 1) * wl);
    sub.search_levels.push_back(search_levels[i]);
    sub.inv_expo_list.push_back(inv_expo_list[i]);
    sub.errors.push_back(0.f);
  }
  v.total_points = n_pts;
}

// VIOManager::computeJacobianAndUpdateEKF (src/vio.cpp:784-802) on a caller-provided visual sub-map (what retrieveFromVisualSparseMap
// would have produced). diag: [0..3] iterations are not exposed by the reference; G and H_T_H are returned (19 x 19 each, row-major).
double ref_vio_update(void *h, const uint8_t *img, int n_pts, const double *pos, const float *warp_patch, const int32_t *search_levels, const double *inv_expo_list,
                      const double *state_in, const double *state_prop, double *state_out, float *errors_out, double *G_out, double *HTH_out) {
  RefVio *r = (RefVio *)h;
  VIOManager &v = r->v;
  unpack_state(state_in, r->st);
  unpack_state(state_prop, r->prop);
  cv::Mat im(v.height, v.width, CV_8UC1, (void *)img);
  cv::Mat own = im.clone();
  v.new_frame_.reset(new Frame(v.cam, own));
  fill_submap(r, n_pts, pos, warp_patch, search_levels, inv_expo_list);
  auto t0 = std::chrono::steady_clock::now();
  v.computeJacobianAndUpdateEKF(own);
  auto t1 = std::chrono::steady_clock::now();
  pack_state(r->st, state_out);
  if (errors_out)
    for (int i = 0; i < n_pts; i++) errors_out[i] = v.visual_submap->errors[i];
  for (int a = 0; a < 19; a++)
    for (int b = 0; b < 19; b++) {
      if (G_out) G_out[19 * a + b] = v.G(a, b);
      if (HTH_out) HTH_out[19 * a + b] = v.H_T_H(a, b);
    }
  return std::chrono::duration<double>(t1 - t0).count();
}

// inverse-compositional variant: the reference features the points were first seen in (Feature::img_, px_, f_, T_f_w_)
void ref_vio_set_inverse(void *h, int enable) { ((RefVio *)h)->v.inverse_composition_en = enable != 0; }
double ref_vio_update_inverse(void *h, const uint8_t *img, int n_pts, const double *pos, const float *warp_patch, const int32_t *search_levels, const double *inv_expo_list,
                              const uint8_t *const *ref_imgs, int n_imgs, const int32_t *ref_img_index, const double *ref_px, const double *ref_f, const double *ref_R,
                              const double *ref_pos /* translation t of T_f_w_ = (R, t) */, const double *state_in, const double *state_prop, double *state_out, float *errors_out) {
  RefVio *r = (RefVio *)h;
  VIOManager &v = r->v;
  unpack_state(state_in, r->st);
  unpack_state(state_prop, r->prop);
  cv::Mat im(v.height, v.width, CV_8UC1, (void *)img);
  cv::Mat own = im.clone();
  v.new_frame_.reset(new Frame(v.cam, own));
  fill_submap(r, n_pts, pos, warp_patch, search_levels, inv_expo_list);
  r->ref_imgs.clear();
  for (int k = 0; k < n_imgs; k++) r->ref_imgs.push_back(cv::Mat(v.height, v.width, CV_8UC1, (void *)ref_imgs[k]).clone());
  for (int i = 0; i < n_pts; i++) {
    M3D R;
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) R(a, b) = ref_R[9 * i + 3 * a + b];
    const V3D t(ref_pos[3 * i], ref_pos[3 * i + 1], ref_pos[3 * i + 2]);  // translation of T_f_w_ (Feature::pos() is then -R^T t)
    Feature *f = new Feature(r->owned[i], new float[64], V2D(ref_px[2 * i], ref_px[2 * i + 1]), V3D(ref_f[3 * i], ref_f[3 * i + 1], ref_f[3 * i + 2]), SE3(R, t), 0);
    f->img_ = r->ref_imgs[ref_img_index[i]];
    r->owned[i]->ref_patch = f;
    r->owned[i]->has_ref_patch_ = true;
    r->owned[i]->obs_.push_back(f);
  }
  v.inverse_composition_en = true;
  auto t0 = std::chrono::steady_clock::now();
  v.computeJacobianAndUpdateEKF(own);
  auto t1 = std::chrono::steady_clock::now();
  v.inverse_composition_en = false;
  pack_state(r->st, state_out);
  if (errors_out)
    for (int i = 0; i < n_pts; i++) errors_out[i] = v.visual_submap->errors[i];
  return std::chrono::duration<double>(t1 - t0).count();
}

// H_sub_inv of the last precomputeReferencePatches (the last level processed: level 0), row-major [n * 64][6]
int ref_vio_get_h_sub_inv(void *h, double *out, int max_doubles) {
  VIOManager &v = ((RefVio *)h)->v;
  const int rows = (int)v.H_sub_inv.rows();
  if (rows * 6 > max_doubles) return -1;
  for (int r = 0; r < rows; r++)
    for (int c = 0; c < 6; c++) out[6 * r + c] = v.H_sub_inv(r, c);
  return rows * 6;
}

// getImagePatch (vio.cpp:203-225): patch_out must hold levels * 64 floats; only [level * 64, level * 64 + 64) is written
void ref_vio_get_image_patch(void *h, const uint8_t *img, const double *pc, int level, float *patch_out) {
  VIOManager &v = ((RefVio *)h)->v;
  cv::Mat im(v.height, v.width, CV_8UC1, (void *)img);
  v.getImagePatch(im, V2D(pc[0], pc[1]), patch_out, level);
}
// warpAffine (vio.cpp:292-318) for one pyramid level into patch_out[pyramid_level * 64 ...]
void ref_vio_warp_affine(void *h, const uint8_t *img_ref, int cols, int rows, const double *A_cur_ref /* row-major 2x2 */, const double *px_ref, int search_level,
                         int pyramid_level, float *patch_out) {
  VIOManager &v = ((RefVio *)h)->v;
  cv::Mat im(rows, cols, CV_8UC1, (void *)img_ref);
  Matrix2d A;
  A(0, 0) = A_cur_ref[0], A(0, 1) = A_cur_ref[1], A(1, 0) = A_cur_ref[2], A(1, 1) = A_cur_ref[3];
  v.warpAffine(A, im, V2D(px_ref[0], px_ref[1]), 0, search_level, pyramid_level, v.patch_size_half, patch_out);
}
// getWarpMatrixAffineHomography + getBestSearchLevel as retrieveFromVisualSparseMap chains them (vio.cpp:699-715)
int ref_vio_warp_matrix(void *h, const double *px_ref, const double *pos_w, const double *normal_w, const double *R_ref_w, const double *t_ref_w, const double *R_cur_w,
                        const double *t_cur_w, double *A_out /* row-major 2x2 */) {
  VIOManager &v = ((RefVio *)h)->v;
  M3D Rr, Rc;
  V3D tr, tc;
  for (int a = 0; a < 3; a++) {
    tr[a] = t_ref_w[a], tc[a] = t_cur_w[a];
    for (int b = 0; b < 3; b++) Rr(a, b) = R_ref_w[3 * a + b], Rc(a, b) = R_cur_w[3 * a + b];
  }
  const SE3 T_ref(Rr, tr), T_cur(Rc, tc);
  const V3D pos(pos_w[0], pos_w[1], pos_w[2]), normal(normal_w[0], normal_w[1], normal_w[2]);
  V3D norm_vec = (T_ref.rotation_matrix() * normal).normalized();  // :701
  V3D pf(T_ref * pos);                                             // :703
  SE3 T_cur_ref = T_cur * T_ref.inverse();                         // :710
  Matrix2d A_cur_ref;
  v.getWarpMatrixAffineHomography(*v.cam, V2D(px_ref[0], px_ref[1]), pf, norm_vec, T_cur_ref, 0, A_cur_ref);  // :712
  A_out[0] = A_cur_ref(0, 0), A_out[1] = A_cur_ref(0, 1), A_out[2] = A_cur_ref(1, 0), A_out[3] = A_cur_ref(1, 1);
  return v.getBestSearchLevel(A_cur_ref, 2);  // :714
}
}
