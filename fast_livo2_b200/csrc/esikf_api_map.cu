// The voxel map: a host-uploaded map and its patches, the device-resident map (build, update, slide, growth, download and
// export), find_correspond on it, and the pv.normal of the last LIO run.
#include "esikf_api.cuh"

#include "esikf_map.cu"
#include "esikf_find.cu"

extern "C" {

// ---------------------------------------------------------------------------------------------------------------- map
int esikf_map_upload(esikf_ctx *ctx, const int64_t *keys, const int32_t *first, const int32_t *count, int32_t n_roots,
                     const esikf_plane *planes, int32_t n_planes, double voxel_size) {
  if (!ctx || n_roots < 0 || n_planes < 0 || (n_roots > 0 && (!keys || !first || !count)) || (n_planes > 0 && !planes) || !(voxel_size > 0))
    return fail(ctx, ESIKF_ERR_ARG, "map_upload: bad argument");
  CK(cudaSetDevice(ctx->device));
  uint32_t cap = 1024;
  while (cap < (uint32_t)n_roots * 2u) cap <<= 1;
  std::vector<HashSlot> table(cap);
  for (auto &s : table) s.key = ESIKF_KEY_EMPTY, s.first = 0, s.count = 0;
  for (int r = 0; r < n_roots; r++) {
    long long x = keys[3 * r], y = keys[3 * r + 1], z = keys[3 * r + 2];
    if (!key_in_range(x, y, z)) return fail(ctx, ESIKF_ERR_ARG, "map_upload: voxel key (%lld,%lld,%lld) outside +-2^20", x, y, z);
    if (first[r] < 0 || count[r] < 0 || first[r] + count[r] > n_planes) return fail(ctx, ESIKF_ERR_ARG, "map_upload: root %d plane range", r);
    unsigned long long k = pack_key(x, y, z);
    uint32_t s = hash_key(k) & (cap - 1);
    while (table[s].key != ESIKF_KEY_EMPTY) {
      if (table[s].key == k) return fail(ctx, ESIKF_ERR_ARG, "map_upload: duplicate voxel key");
      s = (s + 1) & (cap - 1);
    }
    table[s].key = k, table[s].first = (uint32_t)first[r], table[s].count = (uint32_t)count[r];
  }
  CK(ctx->map.slots.reserve(cap));
  CK(ctx->map.planes.reserve((size_t)n_planes + 1));
  CK(ctx->map.recs.reserve((size_t)n_planes + 1));
  CK(cudaMemcpyAsync(ctx->map.slots.p, table.data(), cap * sizeof(HashSlot), cudaMemcpyHostToDevice, ctx->stream));
  if (n_planes) {
    CK(cudaMemcpyAsync(ctx->map.planes.p, planes, (size_t)n_planes * sizeof(esikf_plane), cudaMemcpyHostToDevice, ctx->stream));
    CK(launch(ctx, plane_compact_kernel, (n_planes + 127) / 128, 128, 0, ctx->map.planes.p, nullptr, n_planes, ctx->map.recs.p));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->hash_mask = cap - 1;
  ctx->n_planes = n_planes;
  ctx->map_kind = esikf_ctx::MAP_HOST;  // a host-flattened map replaces a device-resident one
  void_inputs(ctx, IN_NORMALS);
  return ESIKF_OK;
}

int esikf_map_patch(esikf_ctx *ctx, const int32_t *plane_ids, const esikf_plane *planes, int32_t n) {
  if (!ctx || n < 0 || (n > 0 && (!plane_ids || !planes))) return fail(ctx, ESIKF_ERR_ARG, "map_patch: bad argument");
  if (int rc = need(ctx, "map_patch", IN_HOST_MAP)) return rc;
  CK(cudaSetDevice(ctx->device));
  for (int i = 0; i < n; i++)
    if (plane_ids[i] < 0 || plane_ids[i] >= ctx->n_planes) return fail(ctx, ESIKF_ERR_ARG, "map_patch: plane id %d", plane_ids[i]);
  for (int i = 0; i < n;) {
    int j = i + 1;
    while (j < n && plane_ids[j] == plane_ids[j - 1] + 1) j++;  // a run of consecutive ids travels as one copy
    CK(cudaMemcpyAsync(ctx->map.planes.p + plane_ids[i], planes + i, (size_t)(j - i) * sizeof(esikf_plane), cudaMemcpyHostToDevice, ctx->stream));
    i = j;
  }
  if (n > 0) {
    int32_t *ids;
    auto lay = [&](CallLayout &s) { ids = s.take<int32_t>(n), s.end_inputs(); };
    CK(lay_out_scratch(ctx, lay));
    CK(upload(ctx, {{ids, plane_ids, (size_t)n * sizeof(int32_t)}}));
    CK(launch(ctx, plane_compact_kernel, (n + 127) / 128, 128, 0, ctx->map.planes.p, ids, n, ctx->map.recs.p));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  return ESIKF_OK;
}

// ------------------------------------------------------------------------------------------------ device-resident map (f1)
// pv.normal of every point of the last update (voxel_map.cpp:744: the plane that last became the point's best candidate in any
// iteration — normal_plane, not the final match; zero when there never was one): snapshotted by esikf_map_device_update
// before the records may move, otherwise gathered from the records now
__global__ void gather_normals_kernel(const int32_t *__restrict__ match_plane, const PlaneRec *__restrict__ recs, int n, double *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int m = match_plane[i];
  for (int k = 0; k < 3; k++) out[3 * (size_t)i + k] = m >= 0 ? recs[m].n[k] : 0.0;
}

static int map_check_errors(esikf_ctx *ctx, const char *what) {
  int c[4];
  unsigned long long pool_used = 0;
  CK(cudaMemcpyAsync(c, ctx->map.counters.p, sizeof(c), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(&pool_used, ctx->map.counters64.p, sizeof(pool_used), cudaMemcpyDeviceToHost, ctx->stream));
  int work[2];
  CK(cudaMemcpyAsync(work, ctx->map_work.p, sizeof(work), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->map_last.nodes = c[0], ctx->map_last.records = c[1], ctx->map_last.errors = c[2], ctx->map_last.roots = c[3];
  ctx->map_last.pool_points = (int64_t)pool_used, ctx->map_last.touched_roots = work[0];
  if (c[2]) {
    void_inputs(ctx, IN_MAP);  // the map is not trustworthy any more: the next lio_run must not use it
    return fail(ctx, ESIKF_ERR_STATE, "%s: device map capacity exceeded (flags 0x%x:%s%s%s%s%s%s) — raise the esikf_map_cfg capacities and rebuild", what, c[2],
                (c[2] & MAP_ERR_NODES) ? " nodes" : "", (c[2] & MAP_ERR_POOL) ? " point-pool" : "", (c[2] & MAP_ERR_RECS) ? " records" : "",
                (c[2] & MAP_ERR_HASH) ? " hash" : "", (c[2] & MAP_ERR_KEY) ? " key-range" : "", (c[2] & MAP_ERR_STACK) ? " octree-depth" : "");
  }
  return ESIKF_OK;
}

int esikf_map_device_init(esikf_ctx *ctx, const esikf_map_cfg *cfg) {
  if (!ctx || !cfg || !(cfg->voxel_size > 0) || cfg->max_layer < 0 || cfg->max_layer >= MAP_MAX_LAYERS || cfg->max_points_num < 1 || (cfg->grow != 0 && cfg->grow != 1))
    return fail(ctx, ESIKF_ERR_ARG, "map_device_init: bad argument");
  for (int k = 0; k <= cfg->max_layer; k++)
    if (cfg->layer_init_num[k] < 1) return fail(ctx, ESIKF_ERR_ARG, "map_device_init: layer_init_num[%d] = %d", k, cfg->layer_init_num[k]);
  CK(cudaSetDevice(ctx->device));
  const int64_t roots = cfg->root_capacity > 0 ? cfg->root_capacity : (1 << 20);
  uint32_t cap = 1024;
  int bits = 10;
  while ((int64_t)cap < 2 * roots) cap <<= 1, bits++;
  const int64_t node_cap = cfg->node_capacity > 0 ? cfg->node_capacity : 4 * roots;
  const int64_t rec_cap = cfg->record_capacity > 0 ? cfg->record_capacity : 4 * roots;
  const int64_t pool_cap = cfg->point_capacity > 0 ? cfg->point_capacity : 64 * roots;
  if (node_cap > 0x7fffffff || rec_cap > 0x7fffffff || pool_cap > 0x7fffffff) return fail(ctx, ESIKF_ERR_ARG, "map_device_init: capacity above 2^31");
  CK(ctx->map.reserve(cap, (int)node_cap, (int)rec_cap, pool_cap));
  CK(ctx->map_work.reserve(4));
  if (cfg->grow) CK(ctx->map_demand.reserve(MAP_DEMAND_WORDS));
  MapCfg &mc = ctx->arena_cfg;
  mc.voxel_size = (float)cfg->voxel_size, mc.planer_threshold = (float)cfg->min_eigen_value;
  mc.max_layer = cfg->max_layer, mc.max_points_num = cfg->max_points_num;
  for (int k = 0; k < MAP_MAX_LAYERS; k++) mc.layer_init_num[k] = cfg->layer_init_num[k <= cfg->max_layer ? k : cfg->max_layer];
  CK(launch(ctx, map_reset_kernel, (cap + 255) / 256, 256, 0, ctx->arena()));
  CK(cudaMemsetAsync(ctx->map_work.p, 0, 4 * sizeof(int), ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->map_cfg = *cfg;
  ctx->map_hash_bits = bits;
  ctx->hash_mask = cap - 1;
  ctx->map_kind = esikf_ctx::MAP_DEVICE;  // an empty map is a valid map (nothing matches)
  void_inputs(ctx, IN_NORMALS | IN_EXPORT);
  memset(&ctx->map_last, 0, sizeof(ctx->map_last));
  return ESIKF_OK;
}

// sort by slot, list the touched roots, (growth on) bound what they need, replay them unless that does not fit
static int map_replay_tick(esikf_ctx *ctx, int n, bool build) {
  cudaStream_t st = ctx->stream;
  const unsigned int invalid = ctx->map.hash_cap;
  size_t tmp_bytes = 0;
  CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, ctx->map_key_in.p, ctx->map_key_out.p, ctx->map_idx_in.p, ctx->map_idx_out.p, n, 0, ctx->map_hash_bits + 1,
                                     st));
  CK(ctx->map_sort_tmp.reserve(tmp_bytes + 16));
  CK(counted(ctx, cub::DeviceRadixSort::SortPairs(ctx->map_sort_tmp.p, tmp_bytes, ctx->map_key_in.p, ctx->map_key_out.p, ctx->map_idx_in.p, ctx->map_idx_out.p, n,
                                                  0, ctx->map_hash_bits + 1, st)));
  CK(cudaMemsetAsync(ctx->map_work.p, 0, 2 * sizeof(int), st));
  CK(launch(ctx, map_heads_kernel, (n + 255) / 256, 256, 0, ctx->map_key_out.p, n, invalid, ctx->map_touched.p, ctx->map_work.p));
  const unsigned long long *defer = nullptr;
  if (ctx->map_cfg.grow) {
    CK(cudaMemsetAsync(ctx->map_demand.p, 0, MAP_DEMAND_WORDS * sizeof(unsigned long long), st));
    CK(launch(ctx, map_demand_kernel, ctx->sm_count * 4, 128, 0, ctx->arena(), ctx->map_touched.p, ctx->map_work.p, ctx->map_demand.p, build ? 1 : 0));
    defer = ctx->map_demand.p + 5;
  }
  CK(launch(ctx, map_replay_kernel, ctx->sm_count * 4, 128, 0, ctx->arena(), ctx->map_touched.p, ctx->map_work.p, ctx->map_idx_out.p, ctx->map_pt.p, build ? 1 : 0, defer));
  return ESIKF_OK;
}

static int map_capacity_error(esikf_ctx *ctx, const char *what, const char *resource, long long want) {
  void_inputs(ctx, IN_MAP);
  return fail(ctx, ESIKF_ERR_STATE, "%s: the device map cannot grow to %lld %s (the limit is 2^31)", what, want, resource);
}

// Capacity growth: copy the live arena into one of the given capacities with the slide's machinery and an unbounded box (the
// copy only compacts, so it fits any arena at least as large), make it the map and free the old one. Roots without a root
// node (keys inserted by a tick that was deferred) are not copied. When an allocation fails the map is invalidated: a
// deferred tick may have inserted keys already, and the LIO probe would treat them as present voxels.
static int map_grow(esikf_ctx *ctx, long long hash_cap, long long node_cap, long long rec_cap, long long pool_cap, const char *what) {
  if (hash_cap > (1ll << 31)) return map_capacity_error(ctx, what, "hash slots", hash_cap);
  if (node_cap > 0x7fffffff) return map_capacity_error(ctx, what, "nodes", node_cap);
  if (rec_cap > 0x7fffffff) return map_capacity_error(ctx, what, "records", rec_cap);
  if (pool_cap > 0x7fffffff) return map_capacity_error(ctx, what, "stored points", pool_cap);
  cudaStream_t st = ctx->stream;
  MapArenaBufs fresh;
  cudaError_t e = fresh.reserve((uint32_t)hash_cap, (int)node_cap, (int)rec_cap, pool_cap);
  if (e == cudaSuccess) e = ctx->map_survivors.reserve((size_t)(ctx->map_last.roots > 0 ? ctx->map_last.roots : 1) + 1);
  if (e != cudaSuccess) {
    cudaGetLastError();  // a failed allocation is not sticky: later calls must not report it again
    void_inputs(ctx, IN_MAP);
    return fail(ctx, ESIKF_ERR_CUDA, "%s: growing the device map to %lld hash slots / %lld nodes / %lld records / %lld points failed: %s", what, hash_cap, node_cap,
                rec_cap, pool_cap, cudaGetErrorString(e));
  }
  const MapArena S = ctx->arena(), D = fresh.view(ctx->arena_cfg);
  const long long big = 1ll << 40;
  CK(launch(ctx, map_reset_kernel, (unsigned)((hash_cap + 255) / 256), 256, 0, D));
  CK(cudaMemsetAsync(ctx->map_work.p, 0, 2 * sizeof(int), st));
  CK(launch(ctx, map_survivors_kernel, (ctx->map.hash_cap + 255) / 256, 256, 0, S, -big, -big, -big, big, big, big, ctx->map_survivors.p, ctx->map_work.p));
  CK(launch(ctx, map_copy_kernel, ctx->sm_count * 4, 128, 0, S, D, ctx->map_survivors.p, ctx->map_work.p));
  std::swap(ctx->map, fresh);
  int bits = 0;
  while ((1ll << bits) < hash_cap) bits++;
  ctx->hash_mask = (uint32_t)(hash_cap - 1), ctx->map_hash_bits = bits;  // what the LIO probe and the key sort read
  return map_check_errors(ctx, what);  // synchronises: the old arena (now in `fresh`) is no longer read when it is freed
}

// growth on: room in the hash table for n new roots (at most one per point) before any key of the tick is inserted
static bool map_hash_short(const esikf_ctx *ctx, int n) { return ctx->map_cfg.grow && (long long)ctx->map_last.roots + n > (long long)ctx->map.hash_cap / 2; }
static int map_grow_hash(esikf_ctx *ctx, int n, const char *what) {
  const MapArenaBufs &m = ctx->map;
  return map_grow(ctx, map_grown_hash(m.hash_cap, ctx->map_last.roots, n), m.node_cap, m.rec_cap, m.pool_cap, what);
}

// Apply the keyed tick (map_key_in / map_idx_in, points in map_pt). With growth on, a tick the demand bound says might not
// fit is not replayed: each short resource grows to map_grown_capacity, the points are keyed again into the new arena and
// the tick is applied there (a tick that fits costs no extra round trip: the defer word rides on the error check's sync).
static int map_apply_points(esikf_ctx *ctx, int n, bool build) {
  const char *what = build ? "map_device_build" : "map_device_update";
  cudaStream_t st = ctx->stream;
  int rc = map_replay_tick(ctx, n, build);
  if (rc || !ctx->map_cfg.grow) return rc ? rc : map_check_errors(ctx, what);
  unsigned long long d[MAP_DEMAND_WORDS];
  CK(cudaMemcpyAsync(d, ctx->map_demand.p, sizeof(d), cudaMemcpyDeviceToHost, st));
  if ((rc = map_check_errors(ctx, what)) || !d[5]) return rc;
  const MapArenaBufs &m = ctx->map;
  const esikf_map_stats &u = ctx->map_last;  // the counters before the deferred tick
  const long long node_cap = (d[5] & MAP_ERR_NODES) ? map_grown_capacity(m.node_cap, u.nodes, (long long)d[0]) : m.node_cap;
  const long long pool_cap = (d[5] & MAP_ERR_POOL) ? map_grown_capacity(m.pool_cap, u.pool_points, (long long)d[1]) : m.pool_cap;
  const long long rec_cap = (d[5] & MAP_ERR_RECS) ? map_grown_capacity(m.rec_cap, u.records, (long long)d[2]) : m.rec_cap;
  if ((rc = map_grow(ctx, m.hash_cap, node_cap, rec_cap, pool_cap, what))) return rc;
  CK(launch(ctx, map_keys_kernel, (n + 255) / 256, 256, 0, ctx->arena(), ctx->map_pt.p, n, ctx->map_key_in.p, ctx->map_idx_in.p, ctx->map.hash_cap));
  if ((rc = map_replay_tick(ctx, n, build))) return rc;
  CK(cudaMemcpyAsync(d, ctx->map_demand.p, sizeof(d), cudaMemcpyDeviceToHost, st));
  if ((rc = map_check_errors(ctx, what))) return rc;
  if (d[5]) {  // the grown arena holds used + demand of every short resource: the bound itself would be broken
    void_inputs(ctx, IN_MAP);
    return fail(ctx, ESIKF_ERR_STATE, "%s: the tick was deferred again after the map grew (flags 0x%x)", what, (unsigned)d[5]);
  }
  return ESIKF_OK;
}

static int map_reserve_tick(esikf_ctx *ctx, int n) {
  CK(ctx->map_pt.reserve((size_t)n * MAP_PT_D + 16));
  CK(ctx->map_pt_normal.reserve((size_t)n * 3 + 4));
  CK(ctx->map_key_in.reserve(n + 1));
  CK(ctx->map_key_out.reserve(n + 1));
  CK(ctx->map_idx_in.reserve(n + 1));
  CK(ctx->map_idx_out.reserve(n + 1));
  CK(ctx->map_touched.reserve(n + 1));
  return ESIKF_OK;
}

static int map_from_scan(esikf_ctx *ctx, const double *state, bool build) {
  if (!ctx) return ESIKF_ERR_ARG;
  const char *what = build ? "map_device_build" : "map_device_update";
  void_inputs(ctx, IN_EXPORT | IN_PV_LIST);  // map_pt is rewritten below
  if (int rc = need(ctx, what, IN_DEVICE_MAP | IN_EXT | (build ? 0 : IN_RUN_SCAN))) return rc;
  if (build && ctx->map_last.roots > 0) return fail(ctx, ESIKF_ERR_STATE, "map_device_build needs an empty map (esikf_map_device_init resets it)");
  CK(cudaSetDevice(ctx->device));
  const int n = ctx->n_pts;
  if (n == 0) return ctx->map_export_points = 0, ctx->pv_n = build ? -1 : 0, ESIKF_OK;
  int rc = map_reserve_tick(ctx, n);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  const double *dev_state = ctx->state;  // the posterior the last update left on the device
  if (state) {
    CK(ctx->scratch_state.reserve(S_N));
    CK(cudaMemcpyAsync(ctx->scratch_state.p, state, S_N * sizeof(double), cudaMemcpyHostToDevice, st));
    dev_state = ctx->scratch_state.p;
  }
  const int32_t *match_plane = build ? nullptr : ctx->normal_plane.p;
  if (map_hash_short(ctx, n)) {
    // pv.normal refers to the records of the last LIO run: snapshot it before the copy moves them
    if (match_plane) {
      CK(launch(ctx, gather_normals_kernel, (n + 255) / 256, 256, 0, match_plane, ctx->map.recs.p, n, ctx->map_pt_normal.p));
      match_plane = nullptr;
    }
    if ((rc = map_grow_hash(ctx, n, what))) return rc;
  }
  MapPointArgs a;
  memset(&a, 0, sizeof(a));
  a.pts = ctx->pts.p, a.pre = ctx->pre.p, a.pre_stride = ctx->pre_stride, a.n = n, a.state = dev_state;
  memcpy(a.extR, ctx->ext.extR, 72), memcpy(a.extT, ctx->ext.extT, 24);
  a.build = build ? 1 : 0, a.dept_err = (float)ctx->map_cfg.dept_err, a.beam_err = (float)ctx->map_cfg.beam_err;
  a.match_plane = match_plane, a.recs = ctx->map.recs.p, a.pt_normal = ctx->map_pt_normal.p;
  a.pt = ctx->map_pt.p, a.pt_slot = ctx->map_key_in.p, a.pt_idx = ctx->map_idx_in.p, a.invalid_slot = ctx->map.hash_cap;
  CK(launch(ctx, map_points_kernel, (n + 255) / 256, 256, 0, ctx->arena(), a));
  ctx->normals_n = build ? -1 : n;
  if ((rc = map_apply_points(ctx, n, build))) return rc;
  return ctx->map_export_points = n, ctx->pv_n = build ? -1 : n, ESIKF_OK;
}

int esikf_map_device_build(esikf_ctx *ctx, const double *state) {
  if (ctx && !state) return fail(ctx, ESIKF_ERR_ARG, "map_device_build: the pose the scan is mapped with is required");
  return map_from_scan(ctx, state, true);
}
int esikf_map_device_update(esikf_ctx *ctx, const double *state) { return map_from_scan(ctx, state, false); }

int esikf_map_device_update_points(esikf_ctx *ctx, const double *point_w, const double *var, int32_t n) {
  if (ctx) void_inputs(ctx, IN_EXPORT | IN_PV_LIST);
  if (!ctx || n < 0 || (n > 0 && (!point_w || !var))) return fail(ctx, ESIKF_ERR_ARG, "map_device_update_points: bad argument");
  if (int rc = need(ctx, "map_device_update_points", IN_DEVICE_MAP)) return rc;
  if (n == 0) return ctx->map_export_points = 0, ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  int rc = map_reserve_tick(ctx, n);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  // [n][12] = point_w | var: two strided copies
  CK(cudaMemcpy2DAsync(ctx->map_pt.p, MAP_PT_D * sizeof(double), point_w, 3 * sizeof(double), 3 * sizeof(double), n, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpy2DAsync(ctx->map_pt.p + 3, MAP_PT_D * sizeof(double), var, 9 * sizeof(double), 9 * sizeof(double), n, cudaMemcpyHostToDevice, st));
  if (map_hash_short(ctx, n) && (rc = map_grow_hash(ctx, n, "map_device_update"))) return rc;
  CK(launch(ctx, map_keys_kernel, (n + 255) / 256, 256, 0, ctx->arena(), ctx->map_pt.p, n, ctx->map_key_in.p, ctx->map_idx_in.p, ctx->map.hash_cap));
  void_inputs(ctx, IN_NORMALS);
  if ((rc = map_apply_points(ctx, n, false))) return rc;
  return ctx->map_export_points = n, ESIKF_OK;
}

// mapSliding / clearMemOutOfMap (src/voxel_map.cpp:924-971)
int esikf_map_device_slide(esikf_ctx *ctx, const int64_t key_min[3], const int64_t key_max[3]) {
  if (!ctx) return ESIKF_ERR_ARG;
  void_inputs(ctx, IN_EXPORT);
  if (int rc = need(ctx, "map_device_slide", IN_DEVICE_MAP)) return rc;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const MapArenaBufs &live = ctx->map;
  const unsigned cap = live.hash_cap;
  CK(ctx->spare.reserve(cap, live.node_cap, live.rec_cap, live.pool_cap));
  CK(ctx->map_survivors.reserve((size_t)(ctx->map_last.roots > 0 ? ctx->map_last.roots : 1) + 1));
  const MapArena S = ctx->arena(), D = ctx->spare.view(ctx->arena_cfg);
  const long long big = 1ll << 40;
  const long long lo[3] = {key_min ? key_min[0] : -big, key_min ? key_min[1] : -big, key_min ? key_min[2] : -big};
  const long long hi[3] = {key_max ? key_max[0] : big, key_max ? key_max[1] : big, key_max ? key_max[2] : big};
  CK(launch(ctx, map_reset_kernel, (cap + 255) / 256, 256, 0, D));
  CK(cudaMemsetAsync(ctx->map_work.p, 0, 2 * sizeof(int), st));
  CK(launch(ctx, map_survivors_kernel, (cap + 255) / 256, 256, 0, S, lo[0], lo[1], lo[2], hi[0], hi[1], hi[2], ctx->map_survivors.p, ctx->map_work.p));
  CK(launch(ctx, map_copy_kernel, ctx->sm_count * 4, 128, 0, S, D, ctx->map_survivors.p, ctx->map_work.p));
  // the fresh arena becomes the map (also when the copy reports an error: the status says so and the map is invalidated)
  std::swap(ctx->map, ctx->spare);
  void_inputs(ctx, IN_NORMALS);  // record positions of the last update are gone
  return map_check_errors(ctx, "map_device_slide");
}

int esikf_map_device_capacity(esikf_ctx *ctx, esikf_map_cfg *out) {
  if (!ctx || !out) return fail(ctx, ESIKF_ERR_ARG, "map_device_capacity: bad argument");
  if (int rc = need(ctx, "map_device_capacity", IN_DEVICE_MAP)) return rc;
  out->root_capacity = ctx->map.hash_cap / 2, out->node_capacity = ctx->map.node_cap;
  out->record_capacity = ctx->map.rec_cap, out->point_capacity = ctx->map.pool_cap;
  out->grow = ctx->map_cfg.grow;
  return ESIKF_OK;
}

int esikf_map_device_stats(esikf_ctx *ctx, esikf_map_stats *out) {
  if (!ctx || !out) return fail(ctx, ESIKF_ERR_ARG, "map_device_stats: bad argument");
  if (int rc = need(ctx, "map_device_stats", IN_DEVICE_MAP)) return rc;
  *out = ctx->map_last;
  return ESIKF_OK;
}

int esikf_map_device_download(esikf_ctx *ctx, int64_t *keys, int32_t *first, int32_t *count, int32_t roots_cap, esikf_plane *planes, int32_t planes_cap, int32_t *n_roots,
                              int32_t *n_planes) {
  if (!ctx || !n_roots || !n_planes) return fail(ctx, ESIKF_ERR_ARG, "map_device_download: bad argument");
  if (int rc = need(ctx, "map_device_download", IN_DEVICE_MAP)) return rc;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const bool fill = keys && first && count && planes && roots_cap > 0;
  const size_t R = fill ? (size_t)roots_cap : 0, P = fill && planes_cap > 0 ? (size_t)planes_cap : 0;
  int *d_out;
  long long *d_keys;
  int32_t *d_first, *d_count;
  esikf_plane *d_planes;
  auto lay = [&](CallLayout &s) {
    s.begin_answers();  // the counts, then the buffers' worth of roots and planes
    d_out = s.take<int>(2), d_keys = s.take<long long>(3 * R), d_first = s.take<int32_t>(R), d_count = s.take<int32_t>(R), d_planes = s.take<esikf_plane>(P);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(cudaMemsetAsync(d_out, 0, 2 * sizeof(int), st));
  const unsigned cap = ctx->map.hash_cap;
  CK(launch(ctx, map_download_kernel, (cap + 255) / 256, 256, 0, ctx->arena(), fill ? d_keys : nullptr, d_first, d_count, d_planes, fill ? roots_cap : 0,
            fill ? planes_cap : 0, d_out));
  int out[2];
  CK(read_back_to(ctx, d_out, out, 2));
  *n_roots = out[0], *n_planes = out[1];
  if (!fill) return ESIKF_OK;
  if (out[0] > roots_cap || out[1] > planes_cap)
    return fail(ctx, ESIKF_ERR_ARG, "map_device_download: %d roots / %d planes do not fit the buffers (%d / %d)", out[0], out[1], roots_cap, planes_cap);
  const size_t nr = (size_t)out[0], np = (size_t)out[1];
  CK(read_back(ctx, d_keys, d_planes + np));
  copy_out(ctx, keys, d_keys, d_keys, nr * 3 * sizeof(int64_t)), copy_out(ctx, first, d_keys, d_first, nr * sizeof(int32_t));
  copy_out(ctx, count, d_keys, d_count, nr * sizeof(int32_t)), copy_out(ctx, planes, d_keys, d_planes, np * sizeof(esikf_plane));
  return ESIKF_OK;
}

int esikf_map_device_export(esikf_ctx *ctx, int64_t *keys, int32_t *first, int32_t *count, int32_t roots_cap, esikf_map_node *nodes, int32_t nodes_cap, int32_t *n_roots,
                            int32_t *n_nodes) {
  if (!ctx || !n_roots || !n_nodes) return fail(ctx, ESIKF_ERR_ARG, "map_device_export: bad argument");
  if (int rc = need(ctx, "map_device_export", IN_DEVICE_MAP | IN_EXPORT)) return rc;
  *n_roots = 0, *n_nodes = 0;
  const int n = ctx->map_export_points;
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const bool fill = keys && first && count && nodes && roots_cap > 0;
  // laid out for the buffers' worth of roots and nodes: the scan's offsets must stay in place for the write pass
  const size_t R = fill ? (size_t)roots_cap : 0, NN = fill && nodes_cap > 0 ? (size_t)nodes_cap : 0;
  unsigned long long *packed, *offs;
  long long *d_keys;
  int32_t *d_first, *d_count, *d_rows;
  esikf_map_node *d_nodes;
  auto lay = [&](CallLayout &s) {
    packed = s.take<unsigned long long>((size_t)n + 1), d_rows = s.take<int32_t>(NN);
    d_keys = s.take<long long>(3 * R), d_first = s.take<int32_t>(R), d_count = s.take<int32_t>(R), d_nodes = s.take<esikf_map_node>(NN);
    s.begin_answers(), offs = s.take<unsigned long long>((size_t)n + 1);  // the last offset holds the totals
  };
  CK(lay_out_scratch(ctx, lay));
  // position n stays 0: the exclusive scan leaves the totals there
  CK(cudaMemsetAsync(packed, 0, ((size_t)n + 1) * sizeof(unsigned long long), st));
  CK(launch(ctx, map_export_count_kernel, ctx->sm_count * 4, 128, 0, ctx->arena(), ctx->map_touched.p, ctx->map_work.p, packed));
  size_t tmp_bytes = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, packed, offs, n + 1, st));
  CK(ctx->map_sort_tmp.reserve(tmp_bytes + 16));
  CK(counted(ctx, cub::DeviceScan::ExclusiveSum(ctx->map_sort_tmp.p, tmp_bytes, packed, offs, n + 1, st)));
  unsigned long long total;
  CK(read_back_to(ctx, offs + n, &total));
  const int nr = (int)(total >> 32), nn = (int)(total & 0xffffffffull);
  *n_roots = nr, *n_nodes = nn;
  if (!fill) return ESIKF_OK;
  if (nr > roots_cap || nn > nodes_cap)
    return fail(ctx, ESIKF_ERR_ARG, "map_device_export: %d roots / %d nodes do not fit the buffers (%d / %d)", nr, nn, roots_cap, nodes_cap);
  CK(launch(ctx, map_export_kernel, ctx->sm_count * 4, 128, 0, ctx->arena(), ctx->map_touched.p, ctx->map_work.p, offs, d_keys, d_first, d_count, d_nodes, d_rows));
  // direct copies: read back through the pinned block, config 2's export (6.5 MB) took 2.0-2.1 ms a call against 1.75 ms (H100, 700 W)
  CK(cudaMemcpyAsync(keys, d_keys, (size_t)nr * 3 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(first, d_first, (size_t)nr * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(count, d_count, (size_t)nr * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(nodes, d_nodes, (size_t)nn * sizeof(esikf_map_node), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return ESIKF_OK;
}

int esikf_map_device_find(esikf_ctx *ctx, const double *points, int32_t n, int32_t rule, uint8_t *status, int64_t *keys, esikf_plane *rows) {
  if (!ctx || n < 0 || (rule != ESIKF_FIND_RULE_PATCH && rule != ESIKF_FIND_RULE_RAYCAST) || (n > 0 && (!points || !status || !keys || !rows)))
    return fail(ctx, ESIKF_ERR_ARG, "map_device_find: bad argument");
  if (int rc = need(ctx, "map_device_find", IN_DEVICE_MAP | IN_MAP)) return rc;
  if (n == 0) return ESIKF_OK;
  CK(cudaSetDevice(ctx->device));
  const size_t N = (size_t)n;
  MapFindArgs a;
  a.n = n, a.rule = rule;
  auto lay = [&](CallLayout &s) {
    a.pts = s.take<double>(3 * N), s.end_inputs(), s.begin_answers();
    a.rows = s.take<esikf_plane>(N), a.keys = s.take<long long>(3 * N), a.status = s.take<uint8_t>(N);
  };
  CK(lay_out_scratch(ctx, lay));
  CK(upload(ctx, {{a.pts, points, 3 * N * sizeof(double)}}));
  CK(launch(ctx, map_find_kernel, (n + FIND_THREADS - 1) / FIND_THREADS, FIND_THREADS, 0, ctx->arena(), a));
  CK(read_back(ctx, a.rows, a.status + N));
  copy_out(ctx, rows, a.rows, a.rows, N * sizeof(esikf_plane));
  copy_out(ctx, keys, a.rows, a.keys, 3 * N * sizeof(int64_t));
  copy_out(ctx, status, a.rows, a.status, N);
  return ESIKF_OK;
}

int esikf_lio_fetch_normals(esikf_ctx *ctx, double *normals) {
  if (!ctx || !normals) return fail(ctx, ESIKF_ERR_ARG, "lio_fetch_normals: bad argument");
  if (int rc = need(ctx, "lio_fetch_normals", IN_MAP | IN_RUN_SCAN)) return rc;
  CK(cudaSetDevice(ctx->device));
  const int n = ctx->n_pts;
  if (n == 0) return ESIKF_OK;
  double *normal;  // not map_pt_normal: it keeps the pv list's normals for a later generate_points
  auto lay = [&](CallLayout &s) { s.begin_answers(), normal = s.take<double>((size_t)n * 3 + 4); };
  CK(lay_out_scratch(ctx, lay));
  const double *src = ctx->map_pt_normal.p;
  if (ctx->normals_n != n) {
    CK(launch(ctx, gather_normals_kernel, (n + 255) / 256, 256, 0, ctx->normal_plane.p, ctx->map.recs.p, n, normal));
    src = normal;
  }
  CK(read_back_to(ctx, src, normals, (size_t)n * 3));
  return ESIKF_OK;
}
}  // extern "C"
