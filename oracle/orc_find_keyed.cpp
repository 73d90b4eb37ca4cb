// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header). The lookups of the VIO front end as the reference keys them:
// VIOManager::updateReferencePatch (src/vio.cpp:983-993) and the ray-casting branch of the retrieval (:508-514, :572-575), each
// with its own key rule over the literal 0.5, then find_correspond (orc_find.cpp's restatement of src/voxel_map.cpp:292-305) on
// the oracle's map. orc_lio_find_correspond (orc_find.cpp, included here) keys with the map's voxel size instead; both are in
// this library. Built by oracle/find_keyed.mk with -ffp-contract=off, handed OracleLIO handles of liborc_parity.so.
#include <cmath>
#include <cstdint>

#include "orc_find.cpp"

namespace {
const int64_t KEY_RANGE = 1 << 20;  // the device map's keys lie in [-2^20, 2^20)

// rule 0, updateReferencePatch (:983-989): float loc_xyz[j] = p_w[j] / 0.5; if (loc_xyz[j] < 0) loc_xyz[j] -= 1.0; (int64_t)loc
bool key_patch(double c, int64_t *k) {
  float loc = c / 0.5;
  if (loc < 0) loc -= 1.0;
  if (!(loc > -(float)(KEY_RANGE + 1) && loc < (float)KEY_RANGE)) return false;  // trunc(loc) inside the range (NaN, inf fail)
  *k = (int64_t)loc;
  return true;
}
// rule 1, ray casting (:508-514) with an int loc_xyz: loc = floor(p / 0.5); if (loc < 0) loc -= 1.0
bool key_raycast(double c, int64_t *k) {
  const double f = floor(c / 0.5);
  if (!(f >= -(double)KEY_RANGE && f < (double)KEY_RANGE)) return false;
  int loc = (int)f;
  if (loc < 0) loc -= 1.0;
  *k = loc;
  return loc >= -KEY_RANGE;
}
}  // namespace

extern "C" {

// For every point (n x 3) and the key rule (0: updateReferencePatch, 1: ray casting): out n x 6 int64 = status (0 no root,
// 1 a node that is not a plane, 2 a plane), key x y z (INT64_MIN on every axis when it leaves [-2^20, 2^20)), layer, path of the
// node find_correspond returns; f n x 29 doubles = that node's plane_ptr_ center_, normal_, the upper triangle of plane_var_, d_,
// radius_ (zeros where there is no root).
void orc_lio_find_correspond_keyed(void *h, const double *pts, int n, int rule, int64_t *out, double *f) {
  const VoxelMapManager *m = (const VoxelMapManager *)h;
  for (int i = 0; i < n; i++) {
    const double *p = pts + 3 * (size_t)i;
    int64_t *o = out + 6 * (size_t)i;
    double *g = f + 29 * (size_t)i;
    for (int j = 0; j < 6; j++) o[j] = 0;
    for (int j = 0; j < 29; j++) g[j] = 0;
    int64_t k[3];
    bool ok = true;
    for (int j = 0; j < 3; j++) ok = (rule == 1 ? key_raycast(p[j], &k[j]) : key_patch(p[j], &k[j])) && ok;
    for (int j = 0; j < 3; j++) o[1 + j] = ok ? k[j] : INT64_MIN;
    if (!ok) continue;
    auto it = m->voxel_map_.find(VOXEL_LOCATION(k[0], k[1], k[2]));
    if (it == m->voxel_map_.end()) continue;
    int64_t path = 0;
    const VoxelOctoTree *t = find_correspond(it->second, p, &path);
    const VoxelPlane &pl = *t->plane_ptr_;
    o[0] = pl.is_plane_ ? 2 : 1, o[4] = t->layer_, o[5] = path;
    for (int j = 0; j < 3; j++) g[j] = pl.center_.a[j], g[3 + j] = pl.normal_.a[j];
    for (int a = 0, q = 6; a < 6; a++)
      for (int b = a; b < 6; b++) g[q++] = pl.plane_var_(a, b);
    g[27] = pl.d_, g[28] = pl.radius_;
  }
}
}
