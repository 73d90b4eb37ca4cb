// Test infrastructure, not product code: the host build of the device voxel-map state machine (tests/map_host_harness.cu,
// included as it is) plus the export of a tick's touched roots (map_export_root, what map_export_kernel runs per warp), so
// that tests/test_map_mirror_host.py can check the export and the host mirror built from it without a GPU.
//   nvcc -std=c++17 -O2 -shared -Xcompiler -fPIC -o tests/_build/libmap_mirror.so tests/map_mirror_harness.cu
#include "map_host_harness.cu"

extern "C" {

// maph_apply, also listing the roots the tick touched in slot order (the order esikf_map_device_export writes them in):
// slots_out has room for n. Returns the number of touched roots; *err the error flags.
int maph_apply_touched(void *h, const double *pt12, int n, int build, int *slots_out, int *err) {
  HostMap *m = (HostMap *)h;
  MapArena &A = m->A;
  std::vector<unsigned> slot(n), order(n);
  *err = 0;
  for (int i = 0; i < n; i++) {
    long long k[3];
    map_voxel_key(pt12 + (size_t)i * MAP_PT_D, A.cfg.voxel_size, k);
    if (!key_in_range(k[0], k[1], k[2])) return *err = (A.counters[2] |= MAP_ERR_KEY), 0;
    const int s = map_slot_of(A, pack_key(k[0], k[1], k[2]));
    if (s < 0) return *err = (A.counters[2] |= MAP_ERR_HASH), 0;
    slot[i] = (unsigned)s, order[i] = (unsigned)i;
  }
  std::stable_sort(order.begin(), order.end(), [&](unsigned a, unsigned b) { return slot[a] < slot[b]; });
  SerialCoop co;
  int r = 0;
  for (int a = 0; a < n;) {
    int b = a + 1;
    while (b < n && slot[order[b]] == slot[order[a]]) b++;
    map_replay_root(A, co, (int)slot[order[a]], order.data(), a, b - a, pt12, build != 0);
    slots_out[r++] = (int)slot[order[a]];
    a = b;
  }
  *err = A.counters[2];
  return r;
}

// The export of the given roots (esikf_map_device_export's layout): root r owns nodes [first[r], first[r] + count[r]).
// nodes == NULL: sizes only. Returns the number of nodes; rows beyond cap are counted, not written.
int maph_export(void *h, const int *slots, int n_slots, long long *keys, int *first, int *count, esikf_map_node *nodes, int cap) {
  HostMap *m = (HostMap *)h;
  SerialCoop co;
  int total = 0;
  std::vector<int> rows;
  std::vector<esikf_map_node> buf;
  for (int r = 0; r < n_slots; r++) {
    const int c = map_export_root(m->A, co, slots[r], nullptr, nullptr);
    if (nodes && total + c <= cap) {
      rows.resize(c), buf.resize(c);
      map_export_root(m->A, co, slots[r], buf.data(), rows.data());
      memcpy(nodes + total, buf.data(), (size_t)c * sizeof(esikf_map_node));
      for (int q = 0; q < 3; q++) keys[3 * r + q] = buf[0].key[q];
      first[r] = total, count[r] = c;
    }
    total += c;
  }
  return total;
}
}

extern "C" {
// the slot of a root key, -1 when the key is not in the table (nothing is inserted)
int maph_slot_of_key(void *h, long long x, long long y, long long z) {
  const MapArena &A = ((HostMap *)h)->A;
  const unsigned long long k = pack_key(x, y, z);
  uint32_t s = hash_key(k) & A.hash_mask;
  for (uint32_t probes = 0; probes <= A.hash_mask; probes++, s = (s + 1) & A.hash_mask) {
    if (A.slots[s].key == k) return (int)s;
    if (A.slots[s].key == ESIKF_KEY_EMPTY) return -1;
  }
  return -1;
}
}
