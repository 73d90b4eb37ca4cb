// The VIO front end's find_correspond lookups on the device-resident voxel map (K12), without a host mirror: the root voxel
// updateReferencePatch (reference src/vio.cpp:983-993) or the retrieval's ray casting (:508-514, :572-575) looks up, then
// VoxelOctoTree::find_correspond (src/voxel_map.cpp:292-305) from it.
//
//   map_find_kernel : one thread per point. The key by the call site's rule (patch_voxel_key / ret_voxel_key, esikf_dev.cuh),
//                     range-checked before it is packed; the slot by a find-only probe (map_find_slot: no key is inserted);
//                     then the descent while the node is a cut, non-plane node above max_layer, the leaf picked by a strict
//                     `>` against the node's centre per axis (x: 4, y: 2, z: 1), stopping where that leaf is absent.
//
// A pure read of the arena: no atomics, no write into the map, and each point's answer depends on that point alone.

namespace esikf {

#define FIND_THREADS 256

struct MapFindArgs {
  const double *pts;     // [n][3]
  int n, rule;           // ESIKF_FIND_RULE_*
  uint8_t *status;       // [n] ESIKF_FIND_*
  long long *keys;       // [n][3]
  esikf_plane *rows;     // [n]
};

__global__ void __launch_bounds__(FIND_THREADS) map_find_kernel(const MapArena A, const MapFindArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const double p[3] = {a.pts[3 * (size_t)i], a.pts[3 * (size_t)i + 1], a.pts[3 * (size_t)i + 2]};
  long long k[3];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 3; j++) ok = (a.rule == ESIKF_FIND_RULE_RAYCAST ? ret_voxel_key(p[j], k[j]) : patch_voxel_key(p[j], k[j])) && ok;
  const int slot = ok ? map_find_slot(A, pack_key(k[0], k[1], k[2])) : -1;
  int id = slot < 0 ? -1 : A.slot_root[slot];  // a slot can hold a key without a root (a deferred tick inserted it)
  int path = 0;
  while (id >= 0) {
    const MapNode &n = A.nodes[id];
    if (!(n.init_octo && !n.is_plane && n.layer < A.cfg.max_layer)) break;
    const int leaf = (p[0] > n.center[0]) * 4 + (p[1] > n.center[1]) * 2 + (p[2] > n.center[2]);
    const int c = n.children[leaf];
    if (c < 0) break;
    path |= leaf << (3 * n.layer);
    id = c;
  }
  long long *ko = a.keys + 3 * (size_t)i;
  for (int j = 0; j < 3; j++) ko[j] = ok ? k[j] : (long long)INT64_MIN;
  esikf_plane &o = a.rows[i];
  for (int q = 0; q < 6; q++) o.pad[q] = 0;
  if (id < 0) {
    a.status[i] = ESIKF_FIND_NO_ROOT;
    for (int q = 0; q < 3; q++) o.center[q] = 0.0, o.normal[q] = 0.0;
    for (int q = 0; q < 21; q++) o.plane_var[q] = 0.0;
    o.d = 0.f, o.radius = 0.f, o.layer = 0, o.path = 0;
    return;
  }
  const MapNode &n = A.nodes[id];
  a.status[i] = n.is_plane ? ESIKF_FIND_PLANE : ESIKF_FIND_NODE;
  for (int q = 0; q < 3; q++) o.center[q] = n.pc[q], o.normal[q] = n.pn[q];
  for (int q = 0; q < 21; q++) o.plane_var[q] = n.plane_var[q];
  o.d = n.d, o.radius = n.radius, o.layer = n.layer, o.path = path;
}

}  // namespace esikf
