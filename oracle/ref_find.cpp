// oracle/_ref — the reference's OWN VoxelOctoTree::find_correspond (src/voxel_map.cpp:292-305) on the reference source's map
// (the driver ref_voxel_map.cpp, included as it is, builds and updates it). TEST INFRASTRUCTURE ONLY: pins the oracle's
// restatement (oracle/orc_find.cpp) in tests/test_map_mirror_host.py. Built by oracle/find.mk where the reference source exists.
#include "ref_voxel_map.cpp"

namespace {
// the path (3 bits per layer) of `target` below `node`, -1 when it is not in that subtree
int64_t ref_path_of(const VoxelOctoTree *node, const VoxelOctoTree *target, int64_t path) {
  if (node == target) return path;
  for (int l = 0; l < 8; l++)
    if (node->leaves_[l]) {
      const int64_t p = ref_path_of(node->leaves_[l], target, path | ((int64_t)l << (3 * node->layer_)));
      if (p >= 0) return p;
    }
  return -1;
}
}  // namespace

extern "C" {

// As orc_lio_find_correspond: out n x 4 int64 = found, layer, path, is_plane of the node find_correspond returns.
void ref_map_find_correspond(void *h, const double *pts, int n, int64_t *out) {
  RefMap *r = static_cast<RefMap *>(h);
  const auto &vm = r->mgr->voxel_map_;
  for (int i = 0; i < n; i++) {
    const double *p = pts + 3 * (size_t)i;
    float loc_xyz[3];
    for (int j = 0; j < 3; j++) {
      loc_xyz[j] = p[j] / r->config.max_voxel_size_;
      if (loc_xyz[j] < 0) loc_xyz[j] -= 1.0;
    }
    int64_t *o = out + 4 * (size_t)i;
    o[0] = o[1] = o[2] = o[3] = 0;
    auto it = vm.find(VOXEL_LOCATION((int64_t)loc_xyz[0], (int64_t)loc_xyz[1], (int64_t)loc_xyz[2]));
    if (it == vm.end()) continue;
    Eigen::Vector3d pw;
    pw << p[0], p[1], p[2];
    const VoxelOctoTree *t = it->second->find_correspond(pw);
    o[0] = 1, o[1] = t->layer_, o[2] = ref_path_of(it->second, t, 0), o[3] = t->plane_ptr_->is_plane_;
  }
}
}
