// ORACLE — TEST INFRASTRUCTURE ONLY. Restates the parts of VIOManager::retrieveFromVisualSparseMap (src/vio.cpp:352-484 and
// 593-640, raycast_en off) that esikf_vio_retrieve_scan / esikf_vio_depth_check run on the device, and the map-side walk the
// caller keeps between them:
//   orc_retrieve_scan : the scan's voxel keys (floor(c / 0.5f) in double, one less when negative) inserted into a
//                       std::unordered_map<VOXEL_LOCATION, int> with the reference's hash, returned in first-occurrence order,
//                       and the depth image (pt_c[2] > 0, isInFrame(px.cast<int>(), border), the last writer wins)
//   orc_submap_*      : a persistent sub_feat_map (the same container, hash and operation sequence as the reference's member)
//   orc_retrieve_walk : clear, insert the keys in the given order, walk the map in its iteration order over a flat visual map
//                       (voxel key -> points with position and obs_ count), the grid argmin (cur_dist <= map_dist) and the
//                       erase of DeleteKeyList
//   orc_depth_check   : the 8-neighbourhood test of :614-640 (a tap outside the image is empty)
// Checks tests/test_gpu_retrieve_scan.py; pinned to the reference source's own retrieveFromVisualSparseMap
// (oracle/ref_retrieve.cpp, tests/test_oracle_retrieve.py). Built by oracle/retrieve.mk with the parity oracle's translation
// units (handles of orc_vio_create: the camera and Rci / Pci).
#include <cmath>
#include <cstdint>
#include <unordered_map>
#include <vector>

#include "orc_vio.hpp"

using namespace orc;

namespace {

struct VoxelLoc {  // VOXEL_LOCATION (include/voxel_map.h:96-104)
  int64_t x, y, z;
  bool operator==(const VoxelLoc &o) const { return x == o.x && y == o.y && z == o.z; }
};
struct VoxelHash {  // std::hash<VOXEL_LOCATION> (include/voxel_map.h:109-117): VOXELMAP_HASH_P 116101, VOXELMAP_MAX_N 1e10
  int64_t operator()(const VoxelLoc &s) const {
    return ((((s.z) * 116101LL) % 10000000000LL + (s.y)) * 116101LL) % 10000000000LL + (s.x);
  }
};
typedef std::unordered_map<VoxelLoc, int, VoxelHash> SubFeatMap;

SE3 frame_pose(const VIOManager &v, const double *state) {  // updateFrameState (:1690-1697)
  M3 Rwi;
  for (int k = 0; k < 9; k++) Rwi.a[k] = state[k];
  const M3 Rcw = v.Rci * T(Rwi);
  const V3 Pcw = -((v.Rci * T(Rwi)) * v3(state[9], state[10], state[11])) + v.Pci;
  return SE3(Rcw, Pcw);
}

bool in_frame(const Camera &cam, const V2 &px, int border) {  // isInFrame(px.cast<int>(), border)
  const int u = (int)px[0], v = (int)px[1];
  return u >= border && u < cam.width - border && v >= border && v < cam.height - border;
}

}  // namespace

extern "C" {

void *orc_submap_create() { return new SubFeatMap(); }
void orc_submap_destroy(void *s) { delete (SubFeatMap *)s; }
// the keys of the map in its iteration order (room for its size); returns the size
int orc_submap_keys(void *s, int64_t *keys) {
  int k = 0;
  for (auto &kv : *(SubFeatMap *)s) keys[3 * k] = kv.first.x, keys[3 * k + 1] = kv.first.y, keys[3 * k + 2] = kv.first.z, k++;
  return k;
}
// clear(), then insert keys (n x 3) in the given order, as :365 and :402-404 do
void orc_submap_fill(void *s, const int64_t *keys, int n) {
  SubFeatMap &m = *(SubFeatMap *)s;
  m.clear();
  for (int i = 0; i < n; i++) {
    const VoxelLoc p{keys[3 * i], keys[3 * i + 1], keys[3 * i + 2]};
    auto it = m.find(p);
    if (it == m.end()) m[p] = 0;
    else it->second = 0;
  }
}

// :386-428 on n scan points (point_w: n x 3) with the frame pose of `state`: keys (room for n x 3) in first-occurrence order,
// depth (width x height floats). Returns the number of keys, or -1 when a key leaves [-2^20, 2^20).
int orc_retrieve_scan(void *h, const double *state, const double *point_w, int n, int border, int64_t *keys, float *depth) {
  const VIOManager &v = *(VIOManager *)h;
  const SE3 T_f_w = frame_pose(v, state);
  const float voxel_size = 0.5;
  const int width = v.width;
  for (int q = 0; q < v.width * v.height; q++) depth[q] = 0.0f;
  SubFeatMap seen;
  int k = 0;
  for (int i = 0; i < n; i++) {
    const V3 pt_w = v3(point_w[3 * i], point_w[3 * i + 1], point_w[3 * i + 2]);
    int loc_xyz[3];
    for (int j = 0; j < 3; j++) {
      const double f = std::floor(pt_w[j] / voxel_size);
      if (!(f >= -1048576.0 && f < 1048576.0)) return -1;
      loc_xyz[j] = (int)f;
      if (loc_xyz[j] < 0) loc_xyz[j] -= 1.0;
      if (loc_xyz[j] < -1048576) return -1;
    }
    const VoxelLoc position{loc_xyz[0], loc_xyz[1], loc_xyz[2]};
    if (seen.find(position) == seen.end()) {
      seen[position] = 0;
      keys[3 * k] = position.x, keys[3 * k + 1] = position.y, keys[3 * k + 2] = position.z, k++;
    }
    const V3 pt_c = T_f_w * pt_w;
    if (pt_c[2] > 0) {
      const V2 px = v.cam.world2cam(pt_c);
      if (in_frame(v.cam, px, border)) {
        const float d = pt_c[2];
        depth[width * (int)px[1] + (int)px[0]] = d;
      }
    }
  }
  return k;
}

// :438-484 and :593-596 on the persistent sub_feat_map `s`: clear, insert keys (n_keys x 3) in order, then walk it in its
// iteration order over the flat visual map (n_vox voxels: vkeys n_vox x 3, vfirst / vcount into the points; points: pos P x 3,
// n_obs P) and erase the keys whose voxel holds no point in view. Grid as initializeVIO leaves it. Outputs per cell (length =
// grid_n_width * grid_n_height): grid_type (1 = TYPE_MAP), cell_pt (the retrieved point's index, -1 none), cell_pc (its w2c,
// 2 each). Returns the map's size after the erase (its keys: orc_submap_keys).
int orc_retrieve_walk(void *h, void *s, const double *state, const int64_t *keys, int n_keys, const int64_t *vkeys, const int32_t *vfirst, const int32_t *vcount,
                      int n_vox, const double *pos, const int32_t *n_obs, int grid_size, int grid_n_width, int grid_n_height, int border,
                      uint8_t *grid_type, int32_t *cell_pt, double *cell_pc) {
  const VIOManager &v = *(VIOManager *)h;
  SubFeatMap &sub = *(SubFeatMap *)s;
  const SE3 T_f_w = frame_pose(v, state);
  const V3 frame_pos = T_f_w.inverse().t;  // Frame::pos()
  const int length = grid_n_width * grid_n_height;
  std::vector<float> map_dist(length, 10000.0f);
  for (int c = 0; c < length; c++) grid_type[c] = 0, cell_pt[c] = -1, cell_pc[2 * c] = cell_pc[2 * c + 1] = 0.0;
  SubFeatMap feat_map;
  for (int j = 0; j < n_vox; j++) feat_map[VoxelLoc{vkeys[3 * j], vkeys[3 * j + 1], vkeys[3 * j + 2]}] = j;
  orc_submap_fill(s, keys, n_keys);
  std::vector<VoxelLoc> DeleteKeyList;
  for (auto &iter : sub) {
    const VoxelLoc position = iter.first;
    auto corre_voxel = feat_map.find(position);
    if (corre_voxel == feat_map.end()) continue;
    bool voxel_in_fov = false;
    const int j = corre_voxel->second;
    for (int q = vfirst[j]; q < vfirst[j] + vcount[j]; q++) {
      if (n_obs[q] == 0) continue;
      const V3 p = v3(pos[3 * q], pos[3 * q + 1], pos[3 * q + 2]);
      const V3 dir = T_f_w * p;
      if (dir[2] < 0) continue;
      const V2 pc = v.cam.world2cam(T_f_w * p);
      if (!in_frame(v.cam, pc, border)) continue;
      voxel_in_fov = true;
      const int index = static_cast<int>(pc[1] / grid_size) * grid_n_width + static_cast<int>(pc[0] / grid_size);
      grid_type[index] = 1;
      const float cur_dist = norm(V3(frame_pos - p));
      if (cur_dist <= map_dist[index]) {
        map_dist[index] = cur_dist;
        cell_pt[index] = q;
        cell_pc[2 * index] = pc[0], cell_pc[2 * index + 1] = pc[1];
      }
    }
    if (!voxel_in_fov) DeleteKeyList.push_back(position);
  }
  for (auto &key : DeleteKeyList) sub.erase(key);
  return (int)sub.size();
}

// :614-640 for n points (pos n x 3, pc n x 2) against the depth image (the camera's size) with the frame pose of `state`:
// flag = depth_continous
void orc_depth_check(void *h, const double *state, const float *depth, int n, const double *pos, const double *pc, uint8_t *flag) {
  const VIOManager &v = *(VIOManager *)h;
  const SE3 T_f_w = frame_pose(v, state);
  const int width = v.width, half = v.patch_size_half;
  for (int i = 0; i < n; i++) {
    const V3 pt_cam = T_f_w * v3(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]);
    const int u0 = (int)pc[2 * i], v0 = (int)pc[2 * i + 1];
    bool depth_continous = false;
    for (int u = -half; u <= half && !depth_continous; u++)
      for (int w = -half; w <= half; w++) {
        if (u == 0 && w == 0) continue;
        const long x = (long)u0 + u, y = (long)v0 + w;
        if (x < 0 || x >= width || y < 0 || y >= v.height) continue;  // outside the image: empty
        const float d = depth[width * y + x];
        if (d == 0.) continue;
        const double delta_dist = std::abs(pt_cam[2] - d);
        if (delta_dist > 0.5) {
          depth_continous = true;
          break;
        }
      }
    flag[i] = depth_continous;
  }
}

}  // extern "C"
