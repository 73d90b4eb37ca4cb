// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header). VoxelOctoTree::find_correspond (src/voxel_map.cpp:292-305)
// restated on the oracle's map, the lookup VIOManager::updateReferencePatch (src/vio.cpp:969-1034) and the ray-casting branch
// of the retrieval (:572-583) make per visual point. Built on its own (oracle/find.mk) and handed the handle of an OracleLIO
// of liborc_parity.so: it only reads the map (orc_lio.hpp's types, same compiler and flags).
#include "orc_lio.hpp"

using namespace orc;

namespace {
// :292-305: descend while the node is a cut, non-plane node above the last layer and the point's leaf exists; the leaf is
// picked by a strict comparison with the node's centre per axis (x: 4, y: 2, z: 1). path collects the leaves taken (3 bits
// per layer, as the flat plane records).
const VoxelOctoTree *find_correspond(const VoxelOctoTree *t, const double *pw, int64_t *path) {
  while (t->init_octo_ && !t->plane_ptr_->is_plane_ && t->layer_ < t->max_layer_) {
    const int leaf = (pw[0] > t->voxel_center_[0]) * 4 + (pw[1] > t->voxel_center_[1]) * 2 + (pw[2] > t->voxel_center_[2]);
    if (!t->leaves_[leaf]) break;
    *path |= (int64_t)leaf << (3 * t->layer_);
    t = t->leaves_[leaf];
  }
  return t;
}
}  // namespace

extern "C" {

// For every point (n x 3): the root voxel by the float quotient of updateReferencePatch (vio.cpp:983-989, with the map's voxel
// size), then find_correspond from that root. out: n x 4 int64 = found (0: no such root), layer, path, is_plane of the node.
void orc_lio_find_correspond(void *h, const double *pts, int n, int64_t *out) {
  const VoxelMapManager *m = (const VoxelMapManager *)h;
  for (int i = 0; i < n; i++) {
    const double *p = pts + 3 * (size_t)i;
    float loc[3];
    for (int j = 0; j < 3; j++) {
      loc[j] = p[j] / m->config_setting_.max_voxel_size_;
      if (loc[j] < 0) loc[j] -= 1.0;
    }
    int64_t *o = out + 4 * (size_t)i;
    o[0] = o[1] = o[2] = o[3] = 0;
    auto it = m->voxel_map_.find(VOXEL_LOCATION((int64_t)loc[0], (int64_t)loc[1], (int64_t)loc[2]));
    if (it == m->voxel_map_.end()) continue;
    int64_t path = 0;
    const VoxelOctoTree *t = find_correspond(it->second, p, &path);
    o[0] = 1, o[1] = t->layer_, o[2] = path, o[3] = t->plane_ptr_->is_plane_;
  }
}
}
