// Test infrastructure, not product code: the host build of the device voxel-map state machine (tests/map_host_harness.cu,
// included as it is) plus what tests/test_map_growth_host.py needs to check capacity growth (esikf_map_cfg.grow) without a
// GPU: the demand bound of a tick (map_root_demand), a root-by-root apply that reports every root's bound next to what its
// replay took, a copy into larger capacities, and a tick under the demand -> grow -> apply policy of esikf_map_device_*.
//   nvcc -std=c++17 -O2 -shared -Xcompiler -fPIC -o tests/_build/libmap_growth.so tests/map_growth_harness.cu
#include "map_host_harness.cu"

// The keying of a tick (map_points_kernel / map_keys_kernel + the stable sort): the slot of every point (inserted when new)
// and the scan indices ordered by slot. Returns the error flags.
static int key_tick(MapArena &A, const double *pt12, int n, std::vector<unsigned> &slot, std::vector<unsigned> &order) {
  slot.resize(n), order.resize(n);
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
  return 0;
}
// calls f(slot, first sorted position, count) for every touched root (map_heads_kernel)
template <class F>
static void for_each_root(int n, const std::vector<unsigned> &slot, const std::vector<unsigned> &order, F f) {
  for (int a = 0; a < n;) {
    int b = a + 1;
    while (b < n && slot[order[b]] == slot[order[a]]) b++;
    f((int)slot[order[a]], a, b - a);
    a = b;
  }
}

// Every root copied into a fresh arena of the given capacities (map_copy_root, as maph_slide does with the same capacities
// and a box), whose storage then moves into the handle.
static int copy_into(HostMap *m, int hash_cap, int node_cap, long long pool_cap, int rec_cap) {
  const MapArena &S = m->A;
  HostMap *d = (HostMap *)maph_create(S.cfg.voxel_size, S.cfg.planer_threshold, S.cfg.max_layer, S.cfg.max_points_num, S.cfg.layer_init_num, hash_cap, node_cap, pool_cap,
                                     rec_cap);
  SerialCoop co;
  for (size_t s = 0; s < m->slots.size(); s++)
    if (m->slots[s].key != ESIKF_KEY_EMPTY && m->slot_root[s] >= 0) map_copy_root(S, d->A, co, (int)s);
  const int err = d->counters[2];
  m->slots.swap(d->slots), m->slot_root.swap(d->slot_root), m->slot_cap.swap(d->slot_cap), m->rec_node.swap(d->rec_node), m->nodes.swap(d->nodes);
  m->pool.swap(d->pool), m->recs.swap(d->recs), m->planes.swap(d->planes);
  memcpy(m->counters, d->counters, sizeof(m->counters)), m->counters64[0] = d->counters64[0];
  MapArena &A = m->A;
  A.slots = m->slots.data(), A.slot_root = m->slot_root.data(), A.slot_cap = m->slot_cap.data(), A.nodes = m->nodes.data(), A.pool = m->pool.data();
  A.recs = m->recs.data(), A.planes = m->planes.data(), A.rec_node = m->rec_node.data();
  A.hash_mask = (uint32_t)hash_cap - 1, A.node_cap = node_cap, A.pool_cap = pool_cap, A.rec_cap = rec_cap;
  delete d;
  return err;
}

extern "C" {

// The tick root by root: row r of out ([roots][6]) is map_root_demand of the r-th touched root (nodes, pool points, records)
// and what its replay then took from the three counters. Returns the number of touched roots; *err the error flags.
int maph_apply_roots(void *h, const double *pt12, int n, int build, long long *out, int cap, int *err) {
  HostMap *m = (HostMap *)h;
  MapArena &A = m->A;
  std::vector<unsigned> slot, order;
  int r = 0;
  if (!(*err = key_tick(A, pt12, n, slot, order))) {
    SerialCoop co;
    for_each_root(n, slot, order, [&](int s, int a, int c) {
      const MapDemand d = map_root_demand(A, s, c, build != 0);
      const long long before[3] = {A.counters[0], (long long)A.counters64[0], A.counters[1]};
      map_replay_root(A, co, s, order.data(), a, c, pt12, build != 0);
      if (r < cap) {
        long long *o = out + 6 * (size_t)r;
        o[0] = d.nodes, o[1] = d.pool, o[2] = d.recs;
        o[3] = A.counters[0] - before[0], o[4] = (long long)A.counters64[0] - before[1], o[5] = A.counters[1] - before[2];
      }
      r++;
    });
    *err = A.counters[2];
  }
  return r;
}

// The summed demand bound of a tick (map_demand_kernel's sums), after keying it (which inserts its new keys, as the device's
// keying does). out3: nodes, pool points, records. Returns the error flags.
int maph_demand(void *h, const double *pt12, int n, int build, long long *out3) {
  HostMap *m = (HostMap *)h;
  std::vector<unsigned> slot, order;
  out3[0] = out3[1] = out3[2] = 0;
  if (key_tick(m->A, pt12, n, slot, order)) return m->A.counters[2];
  for_each_root(n, slot, order, [&](int s, int, int c) {
    const MapDemand d = map_root_demand(m->A, s, c, build != 0);
    out3[0] += d.nodes, out3[1] += d.pool, out3[2] += d.recs;
  });
  return 0;
}

// Capacity growth: every root copied into an arena of the given (larger) capacities, as esikf_map_device_* grows the map
int maph_grow(void *h, int hash_cap, int node_cap, long long pool_cap, int rec_cap) { return copy_into((HostMap *)h, hash_cap, node_cap, pool_cap, rec_cap); }

// hash slots, nodes, pool points, records
void maph_capacity(void *h, long long *out4) {
  const MapArena &A = ((HostMap *)h)->A;
  out4[0] = (long long)A.hash_mask + 1, out4[1] = A.node_cap, out4[2] = A.pool_cap, out4[3] = A.rec_cap;
}

// A tick with capacity growth, in the order esikf_map_device_update_points takes: the hash table grows first when the tick
// could overfill it; after keying, the summed demand bound is checked against the free space; a short resource grows to
// map_grown_capacity, the tick is keyed again into the grown arena and applied. *grew: the MAP_ERR_* bits of the resources
// that grew. Returns the error flags (-1: deferred again after growing, which would mean the bound is broken).
int maph_apply_grow(void *h, const double *pt12, int n, int build, int *grew) {
  HostMap *m = (HostMap *)h;
  *grew = 0;
  {
    const MapArena &A = m->A;
    const long long hash_cap = (long long)A.hash_mask + 1;
    if ((long long)A.counters[3] + n > hash_cap / 2) {
      if (int e = maph_grow(h, (int)map_grown_hash(hash_cap, A.counters[3], n), A.node_cap, A.pool_cap, A.rec_cap)) return e;
      *grew |= MAP_ERR_HASH;
    }
  }
  for (int pass = 0; pass < 2; pass++) {
    const MapArena &A = m->A;
    long long d[3];
    if (int e = maph_demand(h, pt12, n, build, d)) return e;
    const long long used[3] = {A.counters[0], (long long)A.counters64[0], A.counters[1]}, cap[3] = {A.node_cap, A.pool_cap, A.rec_cap};
    const int flag[3] = {MAP_ERR_NODES, MAP_ERR_POOL, MAP_ERR_RECS};
    long long want[3];
    int short_ = 0;
    for (int r = 0; r < 3; r++) {
      want[r] = cap[r];
      if (used[r] + d[r] > cap[r]) short_ |= flag[r], want[r] = map_grown_capacity(cap[r], used[r], d[r]);
    }
    if (!short_) return maph_apply(h, pt12, n, build);  // keys are found again: the same slots
    if (pass == 1) return -1;
    if (int e = maph_grow(h, (int)A.hash_mask + 1, (int)want[0], want[1], (int)want[2])) return e;
    *grew |= short_;
  }
  return -1;
}
}
