// esikf_map.cuh — the adaptive voxel map kept and refitted on the device (SURVEY §8 f1):
//
//   VoxelMapManager::BuildVoxelMap / UpdateVoxelMap      src/voxel_map.cpp:532-591, 609-641
//   VoxelOctoTree::init_octo_tree / cut_octo_tree / UpdateOctoTree   :137-161, 163-217, 219-290
//   VoxelOctoTree::init_plane                            :55-135
//
// The reference walks the scan serially: every point is pushed into the octree of its root voxel, and a node refits its
// plane whenever enough new points arrived. Root voxels never interact, and inside one root only the ORDER of its points
// matters. The device form therefore is: key every point -> stable sort by root -> ONE WARP PER TOUCHED ROOT replays that
// root's points in scan order through the same state machine (the lanes share the control flow; the per-point sums of a
// refit — second moments, J var J^T — are spread over the lanes) -> the root's candidate planes are re-emitted in DFS order
// into the record block the residual kernel reads (relocated to a larger block when the list outgrows it). No plane, point
// list or key crosses PCIe: the map patch of round 1 (host refit + host flatten + diff + esikf_map_patch) is gone.
//
// Storage (all in HBM, sized once at esikf_map_device_init, nothing allocated per tick):
//   slots[]      open-addressing hash of root keys  {key, first, count}   — what lio_update_kernel probes
//   slot_root[]  root node of a slot / slot_cap[] capacity of its record block
//   nodes[]      octree nodes: geometry, flags, counters, the node's plane fit, its temp_points_ list (offset, size, capacity)
//   pool[]       point storage, 12 doubles a point (point_w | var row-major): pointWithVar reduced to what init_plane reads
//   recs[] / planes[] / rec_node[]   144-byte records for the residual kernel, the 256-byte form for download, owner node
//
// Everything that decides something is written MAP_HD (host + device) on top of a cooperation policy: `WarpCoop` on the GPU,
// `SerialCoop` when the same code is compiled for the host by the test harness (tests/map_host_harness.cu), which replays it
// against the oracle's UpdateVoxelMap without a GPU. The product never runs the host form.
#pragma once
#include "esikf_dev.cuh"

namespace esikf {

#define MAP_HD __host__ __device__ __forceinline__
#define MAP_PT_D 12                // doubles per stored point
#define MAP_UPDATE_THRESHOLD 5     // VoxelOctoTree::update_size_threshold_ (include/voxel_map.h:157)
#define MAP_MAX_LAYERS 8           // layer_init_num entries kept
#define MAP_STACK 64               // explicit DFS / cut stack (8 children x max_layer, max_layer <= 7)

enum { MAP_ERR_NODES = 1, MAP_ERR_POOL = 2, MAP_ERR_RECS = 4, MAP_ERR_HASH = 8, MAP_ERR_KEY = 16, MAP_ERR_STACK = 32 };

struct MapCfg {
  float voxel_size;        // float voxel_size = config_setting_.max_voxel_size_  (:534, :611)
  float planer_threshold;  // float planer_threshold_                            (:535; compared as evalsReal(evalsMin) < planer_threshold_)
  int max_layer, max_points_num;
  int layer_init_num[MAP_MAX_LAYERS];
};

struct MapNode {
  double center[3];  // voxel_center_
  float quarter;     // quater_length_
  int layer;
  int children[8];   // leaves_, -1 = nullptr
  int list_off, list_size, list_cap;  // temp_points_ in pool[] (units: points)
  int new_points;
  unsigned char init_octo, update_enable, octo_state, is_plane;
  int points_size;   // plane_ptr_->points_size_
  // the node's VoxelPlane, what the residual build and the flat download read
  double pc[3], pn[3];
  double plane_var[21];  // upper triangle of plane_var_, row-major i <= j
  float d, radius;
};

struct MapArena {
  HashSlot *slots;
  uint32_t hash_mask;
  int *slot_root;
  int *slot_cap;
  MapNode *nodes;
  int node_cap;
  double *pool;
  long long pool_cap;  // points
  PlaneRec *recs;
  esikf_plane *planes;
  int *rec_node;
  int rec_cap;
  // counters[0] nodes used, [1] records used, [2] error flags, [3] roots; counters64[0] pool points used
  int *counters;
  unsigned long long *counters64;
  MapCfg cfg;
};

struct MapTouched {
  unsigned int slot;
  int start, count;
};

// ---- atomics that degrade to plain operations on the host (single thread there)
MAP_HD int map_atomic_add(int *p, int v) {
#ifdef __CUDA_ARCH__
  return atomicAdd(p, v);
#else
  int o = *p;
  *p = o + v;
  return o;
#endif
}
MAP_HD unsigned long long map_atomic_add64(unsigned long long *p, unsigned long long v) {
#ifdef __CUDA_ARCH__
  return atomicAdd(p, v);
#else
  unsigned long long o = *p;
  *p = o + v;
  return o;
#endif
}
MAP_HD void map_raise(const MapArena &A, int flag) {
#ifdef __CUDA_ARCH__
  atomicOr(&A.counters[2], flag);
#else
  A.counters[2] |= flag;
#endif
}

// ---- cooperation policies. ordered_add<K>: acc[k] += term[k] of lane 0, then of lane 1, ... — the lanes hold consecutive
// points, so the sum runs in the serial order of the reference's loop and every lane ends with the bit-identical total.
struct SerialCoop {
  static constexpr int N = 1;
  MAP_HD int lane() const { return 0; }
  MAP_HD int bcast(int v) const { return v; }
  MAP_HD void sync() const {}
  template <int K>
  MAP_HD void ordered_add(double *acc, const double *term, int valid_lanes) const {
    if (valid_lanes > 0)
      for (int k = 0; k < K; k++) acc[k] = m_add(acc[k], term[k]);
  }
};
#ifdef __CUDACC__
struct WarpCoop {
  static constexpr int N = 32;
  __device__ __forceinline__ int lane() const { return threadIdx.x & 31; }
  __device__ __forceinline__ int bcast(int v) const { return __shfl_sync(0xffffffffu, v, 0); }
  __device__ __forceinline__ void sync() const { __syncwarp(); }
  template <int K>
  __device__ __forceinline__ void ordered_add(double *acc, const double *term, int valid_lanes) const {
    for (int j = 0; j < valid_lanes; j++) {  // valid_lanes is warp-uniform
#pragma unroll
      for (int k = 0; k < K; k++) acc[k] = __dadd_rn(acc[k], __shfl_sync(0xffffffffu, term[k], j));
    }
  }
};
#endif

// ---- voxel key of a world point, float quotient semantics of BuildVoxelMap / UpdateVoxelMap (:566-571, :620-625)
MAP_HD void map_voxel_key(const double *pw, float voxel_size, long long key[3]) {
  for (int j = 0; j < 3; j++) {
    float loc = (float)(pw[j] / (double)voxel_size);
    if (loc < 0) loc = (float)((double)loc - 1.0);
    key[j] = (long long)loc;
  }
}

// find the slot of a key, inserting it when absent (concurrent inserts of the same key agree on one slot). -1: table full.
MAP_HD int map_slot_of(const MapArena &A, unsigned long long k) {
  uint32_t s = hash_key(k) & A.hash_mask;
  for (uint32_t probes = 0; probes <= A.hash_mask; probes++, s = (s + 1) & A.hash_mask) {
#ifdef __CUDA_ARCH__
    unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(&A.slots[s].key);
    if (cur == ESIKF_KEY_EMPTY) cur = atomicCAS(&A.slots[s].key, ESIKF_KEY_EMPTY, k), cur = (cur == ESIKF_KEY_EMPTY) ? k : cur;
#else
    unsigned long long cur = A.slots[s].key;
    if (cur == ESIKF_KEY_EMPTY) A.slots[s].key = cur = k;
#endif
    if (cur == k) return (int)s;
  }
  return -1;
}

// find the slot of a key without inserting it: a pure read of the table. -1: absent. Keys are never removed from a live
// table (a slide or a growth copies the survivors into a fresh one), so the first empty slot ends the probe. lio_update_kernel's
// `probe` (esikf_lio.cu) walks the same table the same way with 16-byte slot loads and no probe bound; keep the two in step.
MAP_HD int map_find_slot(const MapArena &A, unsigned long long k) {
  uint32_t s = hash_key(k) & A.hash_mask;
  for (uint32_t probes = 0; probes <= A.hash_mask; probes++, s = (s + 1) & A.hash_mask) {
    const unsigned long long cur = A.slots[s].key;
    if (cur == k) return (int)s;
    if (cur == ESIKF_KEY_EMPTY) return -1;
  }
  return -1;
}

// ---- nodes
template <class C>
MAP_HD int map_new_node(const MapArena &A, const C &co, int layer, const double *center, float quarter) {
  int id = 0;
  if (co.lane() == 0) id = map_atomic_add(&A.counters[0], 1);
  id = co.bcast(id);
  if (id >= A.node_cap) {
    map_raise(A, MAP_ERR_NODES);
    return -1;
  }
  if (co.lane() == 0) {
    MapNode &n = A.nodes[id];
    for (int k = 0; k < 3; k++) n.center[k] = center[k], n.pc[k] = 0.0, n.pn[k] = 0.0;
    n.quarter = quarter, n.layer = layer;
    for (int k = 0; k < 8; k++) n.children[k] = -1;
    n.list_off = -1, n.list_size = 0, n.list_cap = 0, n.new_points = 0;
    n.init_octo = 0, n.update_enable = 1, n.octo_state = 0, n.is_plane = 0, n.points_size = 0;
    for (int k = 0; k < 21; k++) n.plane_var[k] = 0.0;
    n.d = 0.f, n.radius = 0.f;
  }
  co.sync();
  return id;
}

// leaves_[leafnum] of a node for a point, created on demand (:171-187, :258-273)
template <class C>
MAP_HD int map_child_for(const MapArena &A, const C &co, int node, const double *pw) {
  MapNode &n = A.nodes[node];
  int xyz[3];
  for (int k = 0; k < 3; k++) xyz[k] = pw[k] > n.center[k] ? 1 : 0;
  const int leaf = 4 * xyz[0] + 2 * xyz[1] + xyz[2];
  int c = n.children[leaf];
  if (c >= 0) return c;
  double cc[3];
  for (int k = 0; k < 3; k++) cc[k] = n.center[k] + (double)((float)(2 * xyz[k] - 1) * n.quarter);  // int * float -> float, then double + float
  c = map_new_node(A, co, n.layer + 1, cc, n.quarter / 2);
  if (c < 0) return -1;
  if (co.lane() == 0) n.children[leaf] = c;
  co.sync();
  return c;
}

// temp_points_.push_back(pv)
template <class C>
MAP_HD bool map_list_push(const MapArena &A, const C &co, int node, const double *pt, int reserve = 0) {
  MapNode &n = A.nodes[node];
  if (n.list_size >= n.list_cap) {
    int want = n.list_cap < 8 ? 8 : 2 * n.list_cap;
    if (want < reserve) want = reserve;
    unsigned long long off = 0;
    if (co.lane() == 0) off = map_atomic_add64(&A.counters64[0], (unsigned long long)want);
    const int lo = co.bcast((int)(off & 0xffffffffull)), hi = co.bcast((int)(off >> 32));
    off = ((unsigned long long)(unsigned)hi << 32) | (unsigned)lo;
    if ((long long)(off + want) > A.pool_cap) {
      map_raise(A, MAP_ERR_POOL);
      return false;
    }
    const double *src = A.pool + (size_t)(n.list_off < 0 ? 0 : n.list_off) * MAP_PT_D;
    double *dst = A.pool + off * MAP_PT_D;
    const int words = n.list_size * MAP_PT_D;
    for (int w = co.lane(); w < words; w += C::N) dst[w] = src[w];
    co.sync();
    if (co.lane() == 0) n.list_off = (int)off, n.list_cap = want;
    co.sync();
  }
  double *dst = A.pool + ((size_t)n.list_off + n.list_size) * MAP_PT_D;
  for (int w = co.lane(); w < MAP_PT_D; w += C::N) dst[w] = pt[w];
  co.sync();
  if (co.lane() == 0) n.list_size = n.list_size + 1;
  co.sync();
  return true;
}
// std::vector<pointWithVar>().swap(temp_points_)
template <class C>
MAP_HD void map_list_free(const MapArena &A, const C &co, int node) {
  if (co.lane() == 0) {
    MapNode &n = A.nodes[node];
    n.list_off = -1, n.list_size = 0, n.list_cap = 0;
  }
  co.sync();
}

// Symmetric 3 x 3 eigen-decomposition, cyclic Jacobi (the reference calls Eigen::EigenSolver, :70; eigenvector sign / order
// freedom cancels in everything downstream: the F rows pair each eigenvector with itself, the normal's sign cancels in the
// residual and its Jacobian).
MAP_HD void map_eig_sym3(const double *A9, double evals[3], double V[9]) {
  double a[9];
  for (int k = 0; k < 9; k++) a[k] = A9[k], V[k] = (k % 4 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; sweep++) {
    const double off = m_add(m_add(fabs(a[1]), fabs(a[2])), fabs(a[5]));
    const double diag = m_add(m_add(fabs(a[0]), fabs(a[4])), fabs(a[8]));
    if (off <= m_mul(1e-18, diag) || off == 0.0) break;
    for (int p = 0; p < 2; p++)
      for (int q = p + 1; q < 3; q++) {
        if (a[p * 3 + q] == 0.0) continue;
        const double theta = m_sub(a[q * 3 + q], a[p * 3 + p]) / m_mul(2.0, a[p * 3 + q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / m_add(fabs(theta), sqrt(m_add(m_mul(theta, theta), 1.0)));
        const double c = 1.0 / sqrt(m_add(m_mul(t, t), 1.0)), s = m_mul(t, c);
        for (int k = 0; k < 3; k++) {
          const double akp = a[k * 3 + p], akq = a[k * 3 + q];
          a[k * 3 + p] = m_sub(m_mul(c, akp), m_mul(s, akq));
          a[k * 3 + q] = m_add(m_mul(s, akp), m_mul(c, akq));
        }
        for (int k = 0; k < 3; k++) {
          const double apk = a[p * 3 + k], aqk = a[q * 3 + k];
          a[p * 3 + k] = m_sub(m_mul(c, apk), m_mul(s, aqk));
          a[q * 3 + k] = m_add(m_mul(s, apk), m_mul(c, aqk));
        }
        for (int k = 0; k < 3; k++) {
          const double vkp = V[k * 3 + p], vkq = V[k * 3 + q];
          V[k * 3 + p] = m_sub(m_mul(c, vkp), m_mul(s, vkq));
          V[k * 3 + q] = m_add(m_mul(s, vkp), m_mul(c, vkq));
        }
      }
  }
  for (int i = 0; i < 3; i++) evals[i] = a[i * 3 + i];
}

MAP_HD constexpr int map_tri6(int i, int j) { return i * 6 - (i * (i - 1)) / 2 + (j - i); }  // i <= j

// init_plane(temp_points_, plane_ptr_)   (:55-135). Lane l of a round holds point base + l; the per-point terms are added in
// point order (ordered_add), every lane ends with the same fit, and it is the fit the serial host evaluation produces.
template <class C>
MAP_HD void map_init_plane(const MapArena &A, const C &co, int node) {
  MapNode &n = A.nodes[node];
  const int np = n.list_size;
  const double *pts = A.pool + (size_t)(n.list_off < 0 ? 0 : n.list_off) * MAP_PT_D;
  // covariance_ += p p^T ; center_ += p   (:64-68)
  double s[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};  // xx xy xz yy yz zz | x y z
  for (int base = 0; base < np; base += C::N) {
    const int i = base + co.lane();
    double t[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (i < np) {
      const double *p = pts + (size_t)i * MAP_PT_D;
      t[0] = m_mul(p[0], p[0]), t[1] = m_mul(p[0], p[1]), t[2] = m_mul(p[0], p[2]), t[3] = m_mul(p[1], p[1]), t[4] = m_mul(p[1], p[2]), t[5] = m_mul(p[2], p[2]);
      t[6] = p[0], t[7] = p[1], t[8] = p[2];
    }
    co.template ordered_add<9>(s, t, np - base < C::N ? np - base : C::N);
  }
  const double dn = (double)np;
  const double c[3] = {s[6] / dn, s[7] / dn, s[8] / dn};
  double cov[9];
  cov[0] = m_sub(s[0] / dn, m_mul(c[0], c[0])), cov[1] = m_sub(s[1] / dn, m_mul(c[0], c[1])), cov[2] = m_sub(s[2] / dn, m_mul(c[0], c[2]));
  cov[4] = m_sub(s[3] / dn, m_mul(c[1], c[1])), cov[5] = m_sub(s[4] / dn, m_mul(c[1], c[2])), cov[8] = m_sub(s[5] / dn, m_mul(c[2], c[2]));
  cov[3] = cov[1], cov[6] = cov[2], cov[7] = cov[5];
  double ev[3], V[9];
  map_eig_sym3(cov, ev, V);
  int imin = 0, imax = 0;  // minCoeff / maxCoeff: first index on ties (:76-77)
  for (int i = 1; i < 3; i++) {
    if (ev[i] < ev[imin]) imin = i;
    if (ev[i] > ev[imax]) imax = i;
  }
  const bool is_plane = ev[imin] < (double)A.cfg.planer_threshold;
  double P[21];
  for (int k = 0; k < 21; k++) P[k] = 0.0;
  if (is_plane) {
    const double vmin[3] = {V[imin], V[3 + imin], V[6 + imin]};
    const double jq = 1.0 / np;  // J_Q = I / points_size_ (:83-84)
    for (int base = 0; base < np; base += C::N) {
      const int i = base + co.lane();
      double T[21];
      for (int k = 0; k < 21; k++) T[k] = 0.0;
      if (i < np) {
        const double *p = pts + (size_t)i * MAP_PT_D, *var = p + 3;
        // F rows (:95-108): F_m = (p - c)^T / (n (l_min - l_m)) * (v_m v_min^T + v_min v_m^T), zero for m = min
        double F[9];
        for (int m = 0; m < 3; m++) {
          if (m == imin) {
            F[3 * m] = F[3 * m + 1] = F[3 * m + 2] = 0.0;
            continue;
          }
          const double den = m_mul((double)np, m_sub(ev[imin], ev[m]));
          const double r[3] = {m_sub(p[0], c[0]) / den, m_sub(p[1], c[1]) / den, m_sub(p[2], c[2]) / den};
          const double vm[3] = {V[m], V[3 + m], V[6 + m]};
          for (int cc = 0; cc < 3; cc++) {
            double acc = 0.0;
            for (int k = 0; k < 3; k++) acc = m_add(acc, m_mul(r[k], m_add(m_mul(vm[k], vmin[cc]), m_mul(vmin[k], vm[cc]))));
            F[3 * m + cc] = acc;
          }
        }
        // J = [evecs F ; J_Q]  (6 x 3), plane_var_ += J var J^T  (:110-112)
        double J[18];
        for (int a = 0; a < 3; a++)
          for (int cc = 0; cc < 3; cc++) {
            double acc = 0.0;
            for (int m = 0; m < 3; m++) acc = m_add(acc, m_mul(V[a * 3 + m], F[3 * m + cc]));
            J[a * 3 + cc] = acc;
            J[(3 + a) * 3 + cc] = (a == cc) ? jq : 0.0;
          }
        double JV[18];
        for (int a = 0; a < 6; a++)
          for (int l = 0; l < 3; l++) JV[a * 3 + l] = m_dot3(J[a * 3], var[l], J[a * 3 + 1], var[3 + l], J[a * 3 + 2], var[6 + l]);
        for (int a = 0; a < 6; a++)
          for (int b = a; b < 6; b++) T[map_tri6(a, b)] = m_dot3(JV[a * 3], J[b * 3], JV[a * 3 + 1], J[b * 3 + 1], JV[a * 3 + 2], J[b * 3 + 2]);
      }
      co.template ordered_add<21>(P, T, np - base < C::N ? np - base : C::N);
    }
  }
  if (co.lane() == 0) {
    n.points_size = np;
    for (int k = 0; k < 3; k++) n.pc[k] = c[k];
    for (int k = 0; k < 21; k++) n.plane_var[k] = P[k];
    if (is_plane) {
      for (int k = 0; k < 3; k++) n.pn[k] = V[k * 3 + imin];
      n.radius = (float)sqrt(ev[imax]);
      n.d = (float)(-m_dot3(n.pn[0], c[0], n.pn[1], c[1], n.pn[2], c[2]));
      n.is_plane = 1;
    } else {
      for (int k = 0; k < 3; k++) n.pn[k] = 0.0;
      n.radius = 0.f;
      n.is_plane = 0;
    }
  }
  co.sync();
}

// cut_octo_tree (:163-217), the recursion unrolled onto an explicit stack (sub-trees are independent: the visiting order of the
// leaves changes nothing that is kept)
template <class C>
MAP_HD void map_cut(const MapArena &A, const C &co, int start) {
  int stack[MAP_STACK];
  int sp = 0;
  stack[sp++] = start;
  while (sp > 0) {
    const int id = stack[--sp];
    MapNode &n = A.nodes[id];
    if (n.layer >= A.cfg.max_layer) {
      if (co.lane() == 0) n.octo_state = 0;
      co.sync();
      continue;
    }
    const int np = n.list_size;
    // how many points every leaf receives: its list is reserved once
    int cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const double *pts = A.pool + (size_t)(n.list_off < 0 ? 0 : n.list_off) * MAP_PT_D;
    for (int i = 0; i < np; i++) {
      const double *p = pts + (size_t)i * MAP_PT_D;
      cnt[4 * (p[0] > n.center[0] ? 1 : 0) + 2 * (p[1] > n.center[1] ? 1 : 0) + (p[2] > n.center[2] ? 1 : 0)]++;
    }
    for (int i = 0; i < np; i++) {
      const double *p = A.pool + ((size_t)n.list_off + i) * MAP_PT_D;  // re-derived: a child's push may not move this list, but stay explicit
      const int leaf = 4 * (p[0] > n.center[0] ? 1 : 0) + 2 * (p[1] > n.center[1] ? 1 : 0) + (p[2] > n.center[2] ? 1 : 0);
      const int c = map_child_for(A, co, id, p);
      if (c < 0) return;
      if (!map_list_push(A, co, c, p, cnt[leaf] + 1)) return;
      if (co.lane() == 0) A.nodes[c].new_points++;
      co.sync();
    }
    // the reference keeps the distributed temp_points_ of this node, but never reads them again (a non-plane node above the
    // last layer only forwards points): the storage is released here
    map_list_free(A, co, id);
    for (int l = 0; l < 8; l++) {
      const int c = n.children[l];
      if (c < 0) continue;
      MapNode &ch = A.nodes[c];
      if (ch.list_size > A.cfg.layer_init_num[ch.layer]) {
        map_init_plane(A, co, c);
        if (ch.is_plane) {
          if (co.lane() == 0) ch.octo_state = 0;
          co.sync();
          if (ch.list_size > A.cfg.max_points_num) {
            if (co.lane() == 0) ch.update_enable = 0, n.new_points = 0;  // "new_points_ = 0" is the PARENT's counter there (:203)
            map_list_free(A, co, c);
          }
        } else {
          if (co.lane() == 0) ch.octo_state = 1;
          co.sync();
          if (sp >= MAP_STACK) {
            map_raise(A, MAP_ERR_STACK);
            return;
          }
          stack[sp++] = c;
        }
        if (co.lane() == 0) ch.init_octo = 1, ch.new_points = 0;
        co.sync();
      }
    }
  }
}

// init_octo_tree (:137-161)
template <class C>
MAP_HD void map_init_octo_tree(const MapArena &A, const C &co, int id) {
  MapNode &n = A.nodes[id];
  if (n.list_size > A.cfg.layer_init_num[n.layer]) {
    map_init_plane(A, co, id);
    if (n.is_plane) {
      if (co.lane() == 0) n.octo_state = 0;
      co.sync();
      if (n.list_size > A.cfg.max_points_num) {
        if (co.lane() == 0) n.update_enable = 0, n.new_points = 0;
        map_list_free(A, co, id);
      }
    } else {
      if (co.lane() == 0) n.octo_state = 1;
      co.sync();
      map_cut(A, co, id);
    }
    if (co.lane() == 0) n.init_octo = 1, n.new_points = 0;
    co.sync();
  }
}

// UpdateOctoTree(pv) (:219-290), the tail recursion into the leaf as a loop
template <class C>
MAP_HD void map_update_octo_tree(const MapArena &A, const C &co, int root, const double *pt) {
  int id = root;
  for (int depth = 0; depth <= MAP_MAX_LAYERS; depth++) {
    MapNode &n = A.nodes[id];
    if (!n.init_octo) {
      if (co.lane() == 0) n.new_points++;
      if (!map_list_push(A, co, id, pt)) return;
      if (n.list_size > A.cfg.layer_init_num[n.layer]) map_init_octo_tree(A, co, id);
      return;
    }
    const bool leaf_level = !(n.layer < A.cfg.max_layer);
    const bool was_plane = n.is_plane != 0;  // the branch is chosen before the refit below may change it
    if (was_plane || leaf_level) {
      if (n.update_enable) {
        if (co.lane() == 0) n.new_points++;
        if (!map_list_push(A, co, id, pt)) return;
        if (n.new_points > MAP_UPDATE_THRESHOLD) {
          map_init_plane(A, co, id);
          if (co.lane() == 0) n.new_points = 0;
          co.sync();
        }
        // a plane node stops at size >= max_points_num_ (:237), a non-plane node of the last layer at size > max_points_num_ (:276)
        const bool full = was_plane ? (n.list_size >= A.cfg.max_points_num) : (n.list_size > A.cfg.max_points_num);
        if (full) {
          if (co.lane() == 0) n.update_enable = 0, n.new_points = 0;
          map_list_free(A, co, id);
        }
      }
      return;
    }
    const int c = map_child_for(A, co, id, pt);
    if (c < 0) return;
    id = c;
  }
}

// ---- what the residual kernel reads: the 144-byte record of a fitted plane (same expressions as plane_compact_kernel)
MAP_HD void map_full_record(const MapNode &n, int path, esikf_plane &f) {
  for (int k = 0; k < 3; k++) f.center[k] = n.pc[k], f.normal[k] = n.pn[k];
  for (int k = 0; k < 21; k++) f.plane_var[k] = n.plane_var[k];
  f.d = n.d, f.radius = n.radius, f.layer = n.layer, f.path = path;
  for (int k = 0; k < 6; k++) f.pad[k] = 0;
}
MAP_HD void map_compact_record(const esikf_plane &p, PlaneRec &r) { compact_plane(p, r); }

// Candidate planes of a root in the order build_single_residual visits them (:721, :771-784): a node that is a plane is a
// candidate, otherwise its existing leaves are searched while layer < max_layer. emit == false only counts.
template <class C>
MAP_HD int map_walk_candidates(const MapArena &A, const C &co, int root, bool emit, int first) {
  int node_stack[MAP_STACK], path_stack[MAP_STACK];
  int sp = 0, count = 0;
  node_stack[sp] = root, path_stack[sp] = 0, sp++;
  while (sp > 0) {
    --sp;
    const int id = node_stack[sp], path = path_stack[sp];
    const MapNode &n = A.nodes[id];
    if (n.is_plane) {
      if (emit && co.lane() == 0) {
        esikf_plane f;
        map_full_record(n, path, f);
        A.planes[first + count] = f;
        map_compact_record(f, A.recs[first + count]);
        A.rec_node[first + count] = id;
      }
      count++;
      continue;
    }
    if (n.layer < A.cfg.max_layer) {
      if (sp + 8 > MAP_STACK) {
        map_raise(A, MAP_ERR_STACK);
        return count;
      }
      for (int l = 7; l >= 0; l--)  // pushed in reverse: leaf 0 is popped (visited) first
        if (n.children[l] >= 0) node_stack[sp] = n.children[l], path_stack[sp] = path | (l << (3 * n.layer)), sp++;
    }
  }
  return count;
}

// Re-emit the candidate block of a slot; a list that outgrew its block moves to a fresh, larger one (the old block is dead
// space until the next full rebuild — a root grows at most from 1 to 8^max_layer candidates over its life).
template <class C>
MAP_HD void map_emit_root(const MapArena &A, const C &co, int slot) {
  const int root = A.slot_root[slot];
  const int count = map_walk_candidates(A, co, root, false, 0);
  int first = (int)A.slots[slot].first;
  if (count > A.slot_cap[slot]) {
    int cap = count <= 1 ? 1 : 8;
    while (cap < count) cap *= 2;
    int f = 0;
    if (co.lane() == 0) f = map_atomic_add(&A.counters[1], cap);
    f = co.bcast(f);
    if (f + cap > A.rec_cap) {
      map_raise(A, MAP_ERR_RECS);
      return;
    }
    first = f;
    if (co.lane() == 0) A.slot_cap[slot] = cap;
  }
  map_walk_candidates(A, co, root, true, first);
  co.sync();
  if (co.lane() == 0) {
    // count first drops to 0 so that no reader of a half-written slot exists even in principle (readers are stream-ordered anyway)
    A.slots[slot].first = (uint32_t)first;
    A.slots[slot].count = (uint32_t)count;
  }
  co.sync();
}

// One touched root: its points (indices order[start .. start + count) into pt, ascending scan order) through UpdateOctoTree
// (build == false) or the BuildVoxelMap form: all pushed first, then init_octo_tree (:572-590).
template <class C>
MAP_HD void map_replay_root(const MapArena &A, const C &co, int slot, const unsigned int *order, int start, int count, const double *pt, bool build) {
  int root = A.slot_root[slot];
  if (root < 0) {
    const unsigned long long k = A.slots[slot].key;
    const long long kx = (long long)(k >> 42) - ESIKF_KEY_BIAS, ky = (long long)((k >> 21) & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS,
                    kz = (long long)(k & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS;
    const double vs = (double)A.cfg.voxel_size;
    const double c[3] = {(0.5 + (double)kx) * vs, (0.5 + (double)ky) * vs, (0.5 + (double)kz) * vs};  // (:578-581, :634-636)
    root = map_new_node(A, co, 0, c, A.cfg.voxel_size / 4);
    if (root < 0) return;
    if (co.lane() == 0) {
      A.slot_root[slot] = root, A.slot_cap[slot] = 0;
      A.slots[slot].first = 0, A.slots[slot].count = 0;
      map_atomic_add(&A.counters[3], 1);
    }
    co.sync();
  }
  if (build) {
    for (int j = 0; j < count; j++) {
      if (!map_list_push(A, co, root, pt + (size_t)order[start + j] * MAP_PT_D, count + 1)) return;
      if (co.lane() == 0) A.nodes[root].new_points++;
      co.sync();
    }
    map_init_octo_tree(A, co, root);
  } else {
    for (int j = 0; j < count; j++) map_update_octo_tree(A, co, root, pt + (size_t)order[start + j] * MAP_PT_D);
  }
  map_emit_root(A, co, slot);
}

// ---- Export of one root's subtree for a host mirror (esikf_map_device_export): one esikf_map_node a node, in DFS pre-order
// with leaves 0..7 (the order of the node dumps). Lane 0 walks the tree and lays out the rows (rows[r] = node of row r), then
// the lanes fill the records. out == nullptr: the subtree size only. A pure read of the arena.
MAP_HD void map_export_fields(const MapNode &n, esikf_map_node &o) {
  for (int k = 0; k < 3; k++) o.voxel_center[k] = n.center[k], o.center[k] = n.pc[k], o.normal[k] = n.pn[k];
  o.quater_length = n.quarter;
  o.init_octo = n.init_octo, o.octo_state = n.octo_state, o.update_enable = n.update_enable, o.is_plane = n.is_plane;
  o.new_points = n.new_points, o.points_size = n.points_size, o.temp_points = n.list_size, o.pad_ = 0;
  for (int k = 0; k < 21; k++) o.plane_var[k] = n.plane_var[k];
  o.d = n.d, o.radius = n.radius;
}
template <class C>
MAP_HD int map_export_root(const MapArena &A, const C &co, int slot, esikf_map_node *out, int *rows) {
  int count = 0;
  if (co.lane() == 0) {
    const unsigned long long k = A.slots[slot].key;
    const long long key[3] = {(long long)(k >> 42) - ESIKF_KEY_BIAS, (long long)((k >> 21) & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS,
                              (long long)(k & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS};
    // (node, path, parent row, leaf) entries; a pre-order walk holds at most 7 siblings a layer plus one: < MAP_STACK for ML <= 7
    int st_node[MAP_STACK], st_path[MAP_STACK], st_parent[MAP_STACK], st_leaf[MAP_STACK];
    int sp = 0;
    st_node[sp] = A.slot_root[slot], st_path[sp] = 0, st_parent[sp] = -1, st_leaf[sp] = -1, sp++;
    while (sp > 0) {
      --sp;
      const int id = st_node[sp];
      const MapNode &n = A.nodes[id];
      if (out) {
        esikf_map_node &o = out[count];
        for (int q = 0; q < 3; q++) o.key[q] = key[q];
        o.layer = n.layer, o.path = st_path[sp], o.parent = st_parent[sp], o.leaf = st_leaf[sp];
        rows[count] = id;
      }
      const int row = count++, path = st_path[sp];
      for (int l = 7; l >= 0; l--)  // pushed in reverse: leaf 0 is visited first
        if (n.children[l] >= 0) st_node[sp] = n.children[l], st_path[sp] = path | (l << (3 * n.layer)), st_parent[sp] = row, st_leaf[sp] = l, sp++;
    }
  }
  count = co.bcast(count);
  if (out) {
    co.sync();
    for (int r = co.lane(); r < count; r += C::N) map_export_fields(A.nodes[rows[r]], out[r]);
  }
  return count;
}

// ---- Capacity growth (esikf_map_cfg.grow): what map_replay_root can consume, known before any root is touched.
//
// Upper bounds on the nodes, pool points and record slots one map_replay_root(slot, k points, build) can hand out, from the
// root's subtree at tick start. The derivation, with ML = cfg.max_layer:
//  * Point copies. Only map_cut moves stored points, and it runs only on a node with init_octo == 0 (map_init_octo_tree) or
//    on a child it just filled. An init_octo == 0 node has no children (children are made by a cut, which sets init_octo,
//    or by a descent, which needs init_octo). So every copy moves a point one layer down into a fresh child, and the list it
//    left is freed: a point lives in one list at a time and enters each layer at most once. The points that can move are
//    the k new ones and S, those stored in init_octo == 0 lists at tick start. The build form pushes into the root whatever
//    its state and may cut every list of the subtree: there S counts every stored point.
//  * Nodes. A node is made only when a point enters a layer below 0 (map_child_for, by a descent or a copy), plus the root
//    when it is new: nodes <= [new root] + ML (k + S).
//  * Pushes. A new point is pushed once at the node it stops at, then copied at most ML times; a stored point only copied:
//    pushes <= k (ML + 1) + S ML.
//  * Pool. map_list_push grows a list from capacity c to max(8 or 2c, reserve), only when it is full, and the reserve (a
//    cut's count for one fresh child + 1, or the build's k + 1) never exceeds the list's peak size P + 1. The capacities a
//    list takes in one tick double at least, and all but the last equal its size at a later growth (<= P): they sum to
//    <= 2P, the last is <= max(8, 2P, P + 1). So one list takes <= 4P + 8 points, P <= its size at tick start + its pushes.
//    Lists that can take a push: the init_octo == 0 nodes, the plane / last-layer nodes still updating (every node in the
//    build form), and the new ones. Summed: pool <= 4 (U + pushes) + 8 min(pushes, L + new nodes), U / L the stored points
//    / the number of those pushable lists at tick start.
//  * Records. Candidates are nodes, so a root ends the tick with at most T = (nodes now) + (new nodes) of them.
//    map_emit_root relocates at most once per replay, only when the count exceeds the block it has, into the power-of-two
//    block of the count (1 for one candidate, else 8 or more): records <= 0 if T fits the block, else that block of T.
// The bound only sizes headroom; it may be loose but is never exceeded (tests/test_map_growth_host.py checks it root by root).
struct MapDemand {
  long long nodes, pool, recs;
};
MAP_HD MapDemand map_root_demand(const MapArena &A, int slot, int k, bool build) {
  const long long ML = A.cfg.max_layer;
  const int root = A.slot_root[slot];
  long long S = 0, U = 0, L = 0, have = 0;
  if (root >= 0) {
    int stack[MAP_STACK];  // every node, 8 children a layer, ML <= 7: at most 8 ML + 1 entries
    int sp = 0;
    stack[sp++] = root;
    while (sp > 0) {
      const MapNode &n = A.nodes[stack[--sp]];
      have++;
      const bool init0 = build || !n.init_octo;
      const bool pushable = init0 || (n.update_enable && (n.is_plane || n.layer >= A.cfg.max_layer));
      if (init0) S += n.list_size;
      if (pushable) U += n.list_size, L++;
      for (int l = 0; l < 8; l++)
        if (n.children[l] >= 0 && sp < MAP_STACK) stack[sp++] = n.children[l];
    }
  }
  MapDemand d;
  d.nodes = (root < 0 ? 1 : 0) + ML * (k + S);
  const long long pushes = (long long)k * (ML + 1) + S * ML;
  const long long lists = L + d.nodes;
  d.pool = 4 * (U + pushes) + 8 * (pushes < lists ? pushes : lists);
  const long long T = have + d.nodes;
  long long blk = T <= 1 ? 1 : 8;
  while (blk < T) blk *= 2;
  d.recs = (root >= 0 && T <= A.slot_cap[slot]) ? 0 : blk;
  return d;
}

// The capacity a short resource grows to: twice the old one, or what the tick needs if that is more. The host API and the
// test harness both size their arenas with it.
MAP_HD long long map_grown_capacity(long long cap, long long used, long long demand) { return 2 * cap > used + demand ? 2 * cap : used + demand; }
// Hash slots for `roots` roots plus up to n new ones at a load of at most 1/2 (esikf_map_device_init's sizing): a power of two.
MAP_HD long long map_grown_hash(long long cap, long long roots, long long n) {
  const long long want = map_grown_capacity(cap, 2 * roots, 2 * n);
  long long c = cap;
  while (c < want) c *= 2;
  return c;
}

// ---- mapSliding / clearMemOutOfMap (:924-971) as a copy into a fresh arena: the roots inside the box are re-inserted with their
// whole sub-trees, point lists sized to their content and a tight record block — which also reclaims the dead record
// blocks and the list space earlier growth left behind. S is read-only.
template <class C>
MAP_HD bool map_copy_root(const MapArena &S, const MapArena &D, const C &co, int src_slot) {
  const unsigned long long k = S.slots[src_slot].key;
  const int dslot = map_slot_of(D, k);
  if (dslot < 0) {
    map_raise(D, MAP_ERR_HASH);
    return false;
  }
  int src_stack[MAP_STACK], dst_stack[MAP_STACK];
  int sp = 0;
  const MapNode &sr = S.nodes[S.slot_root[src_slot]];
  const int droot = map_new_node(D, co, 0, sr.center, sr.quarter);
  if (droot < 0) return false;
  src_stack[sp] = S.slot_root[src_slot], dst_stack[sp] = droot, sp++;
  while (sp > 0) {
    --sp;
    const int si = src_stack[sp], di = dst_stack[sp];
    const MapNode &sn = S.nodes[si];
    MapNode &dn = D.nodes[di];
    if (co.lane() == 0) {
      dn.new_points = sn.new_points, dn.init_octo = sn.init_octo, dn.update_enable = sn.update_enable, dn.octo_state = sn.octo_state;
      dn.is_plane = sn.is_plane, dn.points_size = sn.points_size, dn.d = sn.d, dn.radius = sn.radius;
      for (int q = 0; q < 3; q++) dn.pc[q] = sn.pc[q], dn.pn[q] = sn.pn[q];
      for (int q = 0; q < 21; q++) dn.plane_var[q] = sn.plane_var[q];
    }
    co.sync();
    if (sn.list_size > 0) {
      const int want = sn.list_size < 8 ? 8 : sn.list_size;
      unsigned long long off = 0;
      if (co.lane() == 0) off = map_atomic_add64(&D.counters64[0], (unsigned long long)want);
      const int lo = co.bcast((int)(off & 0xffffffffull)), hi = co.bcast((int)(off >> 32));
      off = ((unsigned long long)(unsigned)hi << 32) | (unsigned)lo;
      if ((long long)(off + want) > D.pool_cap) {
        map_raise(D, MAP_ERR_POOL);
        return false;
      }
      const double *src = S.pool + (size_t)sn.list_off * MAP_PT_D;
      double *dst = D.pool + off * MAP_PT_D;
      for (int w = co.lane(); w < sn.list_size * MAP_PT_D; w += C::N) dst[w] = src[w];
      if (co.lane() == 0) dn.list_off = (int)off, dn.list_size = sn.list_size, dn.list_cap = want;
      co.sync();
    }
    for (int l = 0; l < 8; l++) {
      const int sc = sn.children[l];
      if (sc < 0) continue;
      const int dc = map_new_node(D, co, S.nodes[sc].layer, S.nodes[sc].center, S.nodes[sc].quarter);
      if (dc < 0) return false;
      if (co.lane() == 0) dn.children[l] = dc;
      co.sync();
      if (sp >= MAP_STACK) {
        map_raise(D, MAP_ERR_STACK);
        return false;
      }
      src_stack[sp] = sc, dst_stack[sp] = dc, sp++;
    }
  }
  if (co.lane() == 0) {
    D.slot_root[dslot] = droot, D.slot_cap[dslot] = 0;
    D.slots[dslot].first = 0, D.slots[dslot].count = 0;
    map_atomic_add(&D.counters[3], 1);
  }
  co.sync();
  map_emit_root(D, co, dslot);
  return true;
}
// should_remove of clearMemOutOfMap (:958) negated
MAP_HD bool map_key_in_box(unsigned long long k, const long long *lo, const long long *hi) {
  const long long x = (long long)(k >> 42) - ESIKF_KEY_BIAS, y = (long long)((k >> 21) & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS, z = (long long)(k & (ESIKF_KEY_RANGE - 1)) - ESIKF_KEY_BIAS;
  return !(x > hi[0] || x < lo[0] || y > hi[1] || y < lo[1] || z > hi[2] || z < lo[2]);
}

}  // namespace esikf
