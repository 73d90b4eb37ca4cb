// oracle/_ref — the reference's OWN VIOManager::getWarpMatrixAffine + getBestSearchLevel (src/vio.cpp:275-290, 320-331, chained
// as retrieveFromVisualSparseMap does at :726-729) and VIOManager::calculateNCC (:333-350), on the VIOManager the driver
// ref_vio.cpp (included as it is) creates. TEST INFRASTRUCTURE ONLY: pins the oracle's restatement (oracle/orc_select.cpp) in
// tests/test_oracle_select.py. Built by oracle/select.mk where the reference source exists.
#include "ref_vio.cpp"

extern "C" {

// depth = (ref_ftr->pos() - pt->pos_).norm(), T_cur_ref = new_frame_->T_f_w_ * ref_ftr->T_f_w_.inverse(), pyramid level 0,
// halfpatch patch_size_half; T_* as R(9) t(3); A_out row-major 2 x 2. Returns getBestSearchLevel(A, 2).
int ref_vio_warp_matrix_affine(void *h, const double *px_ref, const double *f_ref, const double *ref_pos, const double *pos_w, const double *T_ref,
                               const double *T_cur, int level_ref, double *A_out) {
  VIOManager &v = ((RefVio *)h)->v;
  M3D Rr, Rc;
  V3D tr, tc;
  for (int a = 0; a < 3; a++) {
    tr[a] = T_ref[9 + a], tc[a] = T_cur[9 + a];
    for (int b = 0; b < 3; b++) Rr(a, b) = T_ref[3 * a + b], Rc(a, b) = T_cur[3 * a + b];
  }
  const SE3 Tref(Rr, tr), Tcur(Rc, tc);
  const V3D rp(ref_pos[0], ref_pos[1], ref_pos[2]), pw(pos_w[0], pos_w[1], pos_w[2]);
  Matrix2d A;
  v.getWarpMatrixAffine(*v.cam, V2D(px_ref[0], px_ref[1]), V3D(f_ref[0], f_ref[1], f_ref[2]), (rp - pw).norm(), Tcur * Tref.inverse(), level_ref, 0,
                        v.patch_size_half, A);
  A_out[0] = A(0, 0), A_out[1] = A(0, 1), A_out[2] = A(1, 0), A_out[3] = A(1, 1);
  return v.getBestSearchLevel(A, 2);
}

double ref_vio_calculate_ncc(void *h, const float *ref_patch, const float *cur_patch) {
  VIOManager &v = ((RefVio *)h)->v;
  float r[64], c[64];
  for (int i = 0; i < 64; i++) r[i] = ref_patch[i], c[i] = cur_patch[i];
  return v.calculateNCC(r, c, 64);
}
}
