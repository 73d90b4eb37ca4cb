// Test infrastructure, not product code: the device voxel-map state machine (fast_livo2_b200/csrc/esikf_map.cuh) compiled
// for the HOST with the serial cooperation policy, so that tests/test_map_host.py can replay BuildVoxelMap / UpdateVoxelMap
// tick by tick against the oracle without a GPU. The product runs the same functions under WarpCoop inside map_replay_kernel.
//   nvcc -std=c++17 -O2 -shared -Xcompiler -fPIC -o tests/_build/libmap_host.so tests/map_host_harness.cu
#include <algorithm>
#include <cstring>
#include <vector>

#include "../fast_livo2_b200/csrc/esikf_map.cuh"

using namespace esikf;

struct HostMap {
  MapArena A;
  std::vector<HashSlot> slots;
  std::vector<int> slot_root, slot_cap, rec_node;
  std::vector<MapNode> nodes;
  std::vector<double> pool;
  std::vector<PlaneRec> recs;
  std::vector<esikf_plane> planes;
  int counters[4];
  unsigned long long counters64[1];
};

extern "C" {

void *maph_create(float voxel_size, float planer_threshold, int max_layer, int max_points_num, const int *layer_init_num, int hash_cap, int node_cap, long long pool_cap,
                  int rec_cap) {
  HostMap *m = new HostMap;
  m->slots.resize(hash_cap);
  for (auto &s : m->slots) s.key = ESIKF_KEY_EMPTY, s.first = 0, s.count = 0;
  m->slot_root.assign(hash_cap, -1), m->slot_cap.assign(hash_cap, 0), m->rec_node.assign(rec_cap, -1);
  m->nodes.resize(node_cap), m->pool.resize((size_t)pool_cap * MAP_PT_D), m->recs.resize(rec_cap), m->planes.resize(rec_cap);
  memset(m->counters, 0, sizeof(m->counters)), m->counters64[0] = 0;
  MapArena &A = m->A;
  A.slots = m->slots.data(), A.hash_mask = (uint32_t)hash_cap - 1, A.slot_root = m->slot_root.data(), A.slot_cap = m->slot_cap.data();
  A.nodes = m->nodes.data(), A.node_cap = node_cap, A.pool = m->pool.data(), A.pool_cap = pool_cap;
  A.recs = m->recs.data(), A.planes = m->planes.data(), A.rec_node = m->rec_node.data(), A.rec_cap = rec_cap;
  A.counters = m->counters, A.counters64 = m->counters64;
  A.cfg.voxel_size = voxel_size, A.cfg.planer_threshold = planer_threshold, A.cfg.max_layer = max_layer, A.cfg.max_points_num = max_points_num;
  for (int k = 0; k < MAP_MAX_LAYERS; k++) A.cfg.layer_init_num[k] = layer_init_num[k];
  return m;
}
void maph_destroy(void *h) { delete (HostMap *)h; }

// pt12: [n][12] = point_w | var (row-major). build != 0: BuildVoxelMap form, else UpdateVoxelMap.
int maph_apply(void *h, const double *pt12, int n, int build) {
  HostMap *m = (HostMap *)h;
  MapArena &A = m->A;
  std::vector<unsigned> slot(n), order(n);
  for (int i = 0; i < n; i++) {
    long long k[3];
    map_voxel_key(pt12 + (size_t)i * MAP_PT_D, A.cfg.voxel_size, k);
    if (!key_in_range(k[0], k[1], k[2])) {
      A.counters[2] |= MAP_ERR_KEY;
      return A.counters[2];
    }
    const int s = map_slot_of(A, pack_key(k[0], k[1], k[2]));
    if (s < 0) {
      A.counters[2] |= MAP_ERR_HASH;
      return A.counters[2];
    }
    slot[i] = (unsigned)s, order[i] = (unsigned)i;
  }
  std::stable_sort(order.begin(), order.end(), [&](unsigned a, unsigned b) { return slot[a] < slot[b]; });
  SerialCoop co;
  for (int a = 0; a < n;) {
    int b = a + 1;
    while (b < n && slot[order[b]] == slot[order[a]]) b++;
    map_replay_root(A, co, (int)slot[order[a]], order.data(), a, b - a, pt12, build != 0);
    a = b;
  }
  return A.counters[2];
}

// sizes first (planes == NULL), then fill; roots in slot order
void maph_flatten(void *h, int *n_roots, int *n_planes, long long *keys, int *first, int *count, esikf_plane *planes) {
  HostMap *m = (HostMap *)h;
  int nr = 0, np = 0;
  for (size_t s = 0; s < m->slots.size(); s++) {
    if (m->slots[s].key == ESIKF_KEY_EMPTY || m->slot_root[s] < 0) continue;
    const unsigned long long k = m->slots[s].key;
    if (planes) {
      keys[3 * nr] = (long long)(k >> 42) - ESIKF_KEY_BIAS, keys[3 * nr + 1] = (long long)((k >> 21) & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS;
      keys[3 * nr + 2] = (long long)(k & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS;
      first[nr] = np, count[nr] = (int)m->slots[s].count;
      for (unsigned j = 0; j < m->slots[s].count; j++) planes[np + j] = m->planes[m->slots[s].first + j];
    }
    nr++, np += (int)m->slots[s].count;
  }
  *n_roots = nr, *n_planes = np;
}
// mapSliding: keep the roots with lo <= key <= hi (component-wise), rebuilt into a fresh arena of the same capacities
int maph_slide(void *h, const long long *lo, const long long *hi) {
  HostMap *m = (HostMap *)h;
  const MapArena &S = m->A;
  HostMap *d = (HostMap *)maph_create(S.cfg.voxel_size, S.cfg.planer_threshold, S.cfg.max_layer, S.cfg.max_points_num, S.cfg.layer_init_num, (int)S.hash_mask + 1, S.node_cap,
                                     S.pool_cap, S.rec_cap);
  SerialCoop co;
  for (size_t s = 0; s < m->slots.size(); s++)
    if (m->slots[s].key != ESIKF_KEY_EMPTY && m->slot_root[s] >= 0 && map_key_in_box(m->slots[s].key, lo, hi)) map_copy_root(S, d->A, co, (int)s);
  const int err = d->counters[2];
  // the handle keeps its identity: move the new storage in
  m->slots.swap(d->slots), m->slot_root.swap(d->slot_root), m->slot_cap.swap(d->slot_cap), m->rec_node.swap(d->rec_node), m->nodes.swap(d->nodes);
  m->pool.swap(d->pool), m->recs.swap(d->recs), m->planes.swap(d->planes);
  memcpy(m->counters, d->counters, sizeof(m->counters)), m->counters64[0] = d->counters64[0];
  MapArena &A = m->A;
  A.slots = m->slots.data(), A.slot_root = m->slot_root.data(), A.slot_cap = m->slot_cap.data(), A.nodes = m->nodes.data(), A.pool = m->pool.data();
  A.recs = m->recs.data(), A.planes = m->planes.data(), A.rec_node = m->rec_node.data();
  delete d;
  return err;
}
void maph_usage(void *h, long long *out4) {
  HostMap *m = (HostMap *)h;
  out4[0] = m->counters[0], out4[1] = m->counters[1], out4[2] = (long long)m->counters64[0], out4[3] = m->counters[3];
}
// Every node of every root (roots in slot order, nodes in DFS pre-order, leaves 0..7), MAP_DUMP_COLS int64 a row:
// key x y z | layer path | init_octo octo_state update_enable is_plane | new_points temp_points_.size() points_size.
// Returns the number of nodes; rows beyond cap are counted, not written.
#define MAP_DUMP_COLS 12
static void dump_node(const MapArena &A, int id, long long path, const long long *key, long long *out, int cap, int *n) {
  const MapNode &nd = A.nodes[id];
  if (*n < cap) {
    long long *r = out + (size_t)(*n) * MAP_DUMP_COLS;
    r[0] = key[0], r[1] = key[1], r[2] = key[2], r[3] = nd.layer, r[4] = path;
    r[5] = nd.init_octo, r[6] = nd.octo_state, r[7] = nd.update_enable, r[8] = nd.is_plane;
    r[9] = nd.new_points, r[10] = nd.list_size, r[11] = nd.points_size;
  }
  (*n)++;
  for (int l = 0; l < 8; l++)
    if (nd.children[l] >= 0) dump_node(A, nd.children[l], path | ((long long)l << (3 * nd.layer)), key, out, cap, n);
}
int maph_dump_nodes(void *h, long long *out, int cap) {
  HostMap *m = (HostMap *)h;
  int n = 0;
  for (size_t s = 0; s < m->slots.size(); s++) {
    if (m->slots[s].key == ESIKF_KEY_EMPTY || m->slot_root[s] < 0) continue;
    const unsigned long long k = m->slots[s].key;
    const long long key[3] = {(long long)(k >> 42) - ESIKF_KEY_BIAS, (long long)((k >> 21) & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS,
                              (long long)(k & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS};
    dump_node(m->A, m->slot_root[s], 0, key, out, cap, &n);
  }
  return n;
}
// slots in use (occupied keys, whether or not their root was created)
int maph_slots_used(void *h) {
  HostMap *m = (HostMap *)h;
  int n = 0;
  for (auto &s : m->slots) n += s.key != ESIKF_KEY_EMPTY;
  return n;
}
}
