// Drives the shim managers of fast_livo2_b200/csrc/fl2_shim.hpp through the calls of a LIVMapper tick on inputs written by
// tests/test_gpu_shim_staging.py, and writes every answer to <out>/<tag>.<name>.bin for the test to compare bit for bit.
//   shim_staging_driver <in> <out> <command>...
// Commands run in order on one manager pair ("new" replaces it with a fresh one):
//   tick:<size>:<tag>    StateEstimation .. warpAffine on the inputs of <size> (L or S); none of them changes the map
//   lazy:<size>:<tag>    StateEstimation with lazy point lists; UpdateVoxelMap(), FindCorrespond and SetWorldCloud of the
//                        other size; then the lists
//   select:<size>:<tag>  SelectSubSparseMap; the other size's LIO and front-end calls but the selection and the update; then
//                        MaterializeWarpPatches and computeJacobianAndUpdateEKF on the sub-map the selection left
//   select_now:<size>:<tag>  the same without the calls in between
//   failbuild:<tag>      BuildVoxelMap of the large scan on the non-empty map (fails after uploading the scan)
//   resident:<tag>       UpdateVoxelMap() of the wide scan (more voxel keys than RetrieveScanVoxels' first room), then
//                        RetrieveScanVoxels of the resident scan
//   score:<case>:<tag>   ScoreReferencePatches on the arrays <case>_first, <case>_pts and <case>_obs
//   generate:<tag>       GenerateVisualMapPoints on its own context, camera and image (the gen_* arrays)
//   time:<size>:<reps>   milliseconds per call of the four methods that moved to pinned memory and of a LIO + VIO tick pair
// Where a method is compared with the plain C-ABI call, the call runs on the managers' context right after the method, with
// the same inputs in ordinary host arrays, and its answer is written as <name>_abi in the method's format.
#include <chrono>
#include <cstdio>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "../fast_livo2_b200/csrc/fl2_shim.hpp"

using namespace fl2b200;

static std::string in_dir, out_dir;

template <typename T> static std::vector<T> load(const std::string &name) {
  std::vector<T> v;
  FILE *f = std::fopen((in_dir + "/" + name + ".bin").c_str(), "rb");
  if (!f) return v;
  std::fseek(f, 0, SEEK_END);
  v.resize(std::ftell(f) / sizeof(T));
  std::fseek(f, 0, SEEK_SET);
  if (std::fread(v.data(), sizeof(T), v.size(), f) != v.size()) v.clear();
  std::fclose(f);
  return v;
}
static void dump(const std::string &tag, const std::string &name, const void *p, size_t bytes) {
  FILE *f = std::fopen((out_dir + "/" + tag + "." + name + ".bin").c_str(), "wb");
  if (bytes) std::fwrite(p, 1, bytes, f);
  std::fclose(f);
}
template <typename T> static void dumpv(const std::string &tag, const std::string &name, const std::vector<T> &v) { dump(tag, name, v.data(), v.size() * sizeof(T)); }
// the fields of records whose padding is not part of the answer, as doubles
template <typename T, typename F> static void dumpf(const std::string &tag, const std::string &name, const std::vector<T> &v, F &&fields) {
  std::vector<double> o;
  for (const T &e : v) fields(e, o);
  dumpv(tag, name, o);
}
static void put(std::vector<double> &o, const double *p, int n) { o.insert(o.end(), p, p + n); }
static void putf(std::vector<double> &o, const float *p, int n) { o.insert(o.end(), p, p + n); }

struct Inputs {
  std::vector<PointXYZ> pts, dense;
  std::vector<double> state, query;
  std::vector<SubMapCandidate> cands;
};

struct Pair {
  VoxelMapConfig cfg;
  VoxelMap map;
  VoxelMapManager *mgr = nullptr;
  VIOManager *vio = nullptr;
  StatesGroup st, stp;
  SubSparseMap sub;
  std::vector<uint8_t> img, ref, bgr;
  GrayImage gimg, gref;
  int W = 0, H = 0;
  std::vector<SubMapCandidate> cands_of_selection;
  ~Pair() { delete vio, delete mgr, ClearVoxelMap(map); }
};

static Inputs inputs[3];  // L, S and the wide scan W (L's state)
static std::vector<double> meta;  // cam fx fy cx cy w h | extR 9 extT 3 Rcl 9 Pcl 3 | T_cur_w 12 (the camera pose of the frame)

static Pair *make_pair() {
  Pair *p = new Pair;
  p->cfg.device_root_capacity_ = 1 << 16, p->cfg.device_map_grow_ = true;
  p->mgr = new VoxelMapManager(p->cfg, p->map, 0);
  VoxelMapManager &m = *p->mgr;
  const double *e = meta.data() + 6;
  memcpy(m.extR_.m, e, 72), memcpy(m.extT_.v, e + 9, 24);
  m.EnableDeviceMap();
  p->vio = new VIOManager(m.context());
  VIOManager &v = *p->vio;
  p->W = (int)meta[4], p->H = (int)meta[5];
  v.cam.model = 0, v.cam.width = p->W, v.cam.height = p->H, v.cam.fx = meta[0], v.cam.fy = meta[1], v.cam.cx = meta[2], v.cam.cy = meta[3];
  memcpy(v.extR.m, e, 72), memcpy(v.extT.v, e + 9, 24), memcpy(v.Rcl.m, e + 12, 72), memcpy(v.Pcl.v, e + 21, 24);
  v.state = &p->st, v.state_propagat = &p->stp, v.visual_submap = &p->sub;
  v.initializeVIO();
  p->img = load<uint8_t>("img"), p->ref = load<uint8_t>("ref"), p->bgr = load<uint8_t>("bgr");
  p->gimg = GrayImage{p->img.data(), p->W, p->H}, p->gref = GrayImage{p->ref.data(), p->W, p->H};
  // the map: the small scan at its state, so that both sizes find planes
  m.feats_down_body_ = inputs[1].pts, m.feats_down_size_ = (int)inputs[1].pts.size();
  m.state_.unpack(inputs[1].state.data());
  m.BuildVoxelMap();
  return p;
}

static void status(const std::string &tag, const std::string &name, int s) { dump(tag, name + ".status", &s, sizeof(s)); }
static std::vector<double> packed(const StatesGroup &st) {
  std::vector<double> s(ESIKF_STATE_DOUBLES);
  st.pack(s.data());
  return s;
}
static void put_keys(std::vector<double> &o, const int32_t *kb, int k) { o.insert(o.end(), kb, kb + 3 * k); }
static void put_plane(std::vector<double> &o, const double *c, const double *nrm, const double *var36, double d, double radius, bool is_plane) {
  put(o, c, 3), put(o, nrm, 3), put(o, var36, 36), o.push_back(d), o.push_back(radius), o.push_back(is_plane);
}

static void lio(Pair &p, const Inputs &in, const std::string &tag) {
  VoxelMapManager &m = *p.mgr;
  m.feats_down_body_ = in.pts, m.feats_down_size_ = (int)in.pts.size();
  m.state_.unpack(in.state.data());
  StatesGroup prop = m.state_;
  m.StateEstimation(prop);
  status(tag, "lio", m.last_status_);
  std::vector<double> s(ESIKF_STATE_DOUBLES);
  m.state_.pack(s.data());
  dumpv(tag, "lio.state", s);
}

static void lists(Pair &p, const std::string &tag) {
  VoxelMapManager &m = *p.mgr;
  m.MaterializePointLists();
  status(tag, "lists", m.last_status_);
  dumpv(tag, "lists.pv", m.pv_list_), dumpv(tag, "lists.body_cov", m.body_cov_list_), dumpv(tag, "lists.cross", m.cross_mat_list_);
  dumpf(tag, "lists.ptpl", m.ptpl_list_, [](const PointToPlane &q, std::vector<double> &o) {
    put(o, q.point_w_.v, 3), put(o, q.normal_.v, 3), put(o, q.center_.v, 3), put(o, q.plane_var_, 36), o.push_back(q.d_), o.push_back(q.dis_to_plane_), o.push_back(q.layer_);
  });
}

// the plain C-ABI form of the candidates
struct CandArrays {
  std::vector<int32_t> idx, lvl, key;
  std::vector<double> px, f, rp, pw, nw, T, ie, pc;
  explicit CandArrays(const std::vector<SubMapCandidate> &c) {
    for (const SubMapCandidate &k : c) {
      idx.push_back(k.ref_img_index), lvl.push_back(k.ref_level), key.push_back(k.ref_key), ie.push_back(k.ref_inv_expo);
      px.insert(px.end(), k.px_ref, k.px_ref + 2), f.insert(f.end(), k.ref_f, k.ref_f + 3), rp.insert(rp.end(), k.ref_pos, k.ref_pos + 3);
      pw.insert(pw.end(), k.pos_w, k.pos_w + 3), nw.insert(nw.end(), k.normal_w, k.normal_w + 3), T.insert(T.end(), k.T_ref_w, k.T_ref_w + 12);
      pc.insert(pc.end(), k.pc, k.pc + 2);
    }
  }
};
static std::vector<double> sel_A;  // the matrices of the last C-ABI selection, for the C-ABI form of MaterializeWarpPatches
static std::vector<int32_t> sel_kept, sel_sl;

static void select(Pair &p, const Inputs &in, const std::string &tag) {
  VIOManager &v = *p.vio;
  const double *T_cur_w = meta.data() + 30;
  v.SetReferenceImages(&p.gref, 1);
  v.SelectSubSparseMap(in.cands.data(), (int)in.cands.size(), p.gimg, T_cur_w);
  p.cands_of_selection = in.cands;
  status(tag, "select", v.last_status_);
  dumpv(tag, "select.errors", p.sub.errors), dumpv(tag, "select.levels", p.sub.search_levels), dumpv(tag, "select.index", p.sub.candidate_index);
  const int n = (int)in.cands.size();
  CandArrays c(in.cands);
  esikf_vio_select_cfg cfg;
  cfg.normal_en = v.normal_en, cfg.ncc_en = v.ncc_en, cfg.ncc_thre = v.ncc_thre, cfg.outlier_threshold = v.outlier_threshold;
  std::vector<float> err(n);
  sel_kept.assign(n, 0), sel_sl.assign(n, 0), sel_A.assign(4 * n, 0.0);
  int32_t nk = 0;
  status(tag, "select_abi", esikf_vio_select_patches(p.mgr->context(), n, c.idx.data(), c.px.data(), c.lvl.data(), c.f.data(), c.rp.data(), c.pw.data(), c.nw.data(), c.T.data(),
                                                     c.ie.data(), c.key.data(), c.pc.data(), T_cur_w, p.st.inv_expo_time, &cfg, &nk, sel_kept.data(), err.data(),
                                                     sel_sl.data(), sel_A.data(), nullptr));
  err.resize(nk), sel_kept.resize(nk), sel_sl.resize(nk), sel_A.resize(4 * nk);
  dumpv(tag, "select.errors_abi", err), dumpv(tag, "select.levels_abi", sel_sl), dumpv(tag, "select.index_abi", sel_kept);
}

static void materialize_and_update(Pair &p, const std::string &tag) {
  VIOManager &v = *p.vio;
  v.MaterializeWarpPatches();
  status(tag, "warp", v.last_status_);
  std::vector<float> wp;
  for (const std::vector<float> &w : p.sub.warp_patch) wp.insert(wp.end(), w.begin(), w.end());
  dumpv(tag, "warp.patches", wp);
  std::vector<int32_t> idx;
  std::vector<double> px;
  for (int32_t j : sel_kept) idx.push_back(p.cands_of_selection[j].ref_img_index), px.insert(px.end(), p.cands_of_selection[j].px_ref, p.cands_of_selection[j].px_ref + 2);
  std::vector<float> wa(wp.size());
  status(tag, "warp_abi", esikf_vio_warp_affine(p.mgr->context(), (int)idx.size(), idx.data(), px.data(), sel_A.data(), sel_sl.data(), wa.data()));
  dumpv(tag, "warp.patches_abi", wa);
  p.stp = p.st;
  v.computeJacobianAndUpdateEKF(p.gimg);
  status(tag, "vio", v.last_status_);
  std::vector<double> s(ESIKF_STATE_DOUBLES);
  p.st.pack(s.data());
  dumpv(tag, "vio.state", s), dumpv(tag, "vio.errors", p.sub.errors);
}

static void dump_points_abi(const std::string &tag, const std::string &name, int k, const int32_t *src, const int32_t *cell, const double *pos, const double *pc,
                            const double *nrm, const double *var, const float *score, const float *patch) {
  std::vector<double> o;
  for (int i = 0; i < k; i++)
    o.push_back(src[i]), o.push_back(cell[i]), put(o, pos + 3 * i, 3), put(o, pc + 2 * i, 2), put(o, nrm + 3 * i, 3), put(o, var + 9 * i, 9), putf(o, score + i, 1),
        putf(o, patch + 64 * i, 64);
  dumpv(tag, name, o);
}
static void dump_points(const std::string &tag, const std::string &name, const std::vector<NewVisualPoint> &np) {
  dumpf(tag, name, np, [](const NewVisualPoint &q, std::vector<double> &o) {
    o.push_back(q.source), o.push_back(q.cell), put(o, q.pos, 3), put(o, q.pc, 2), put(o, q.normal, 3), put(o, q.var, 9), putf(o, &q.score, 1), putf(o, q.patch, 64);
  });
}
// esikf_vio_score_ref_patches on the records of ScoreReferencePatches, unpacked into plain arrays
static void score_abi(esikf_ctx *ctx, const std::string &tag, const std::vector<int32_t> &first, const std::vector<ScoredPoint> &sp, const std::vector<PatchObservation> &po) {
  const size_t n = sp.size(), m = po.size();
  std::vector<double> pos, nrm, T;
  std::vector<float> patch, mean, sc(m + 1), mu(m + 1);
  std::vector<int32_t> id, ref(n + 1);
  for (const ScoredPoint &s : sp) pos.insert(pos.end(), s.pos, s.pos + 3), nrm.insert(nrm.end(), s.normal, s.normal + 3);
  for (const PatchObservation &o : po) T.insert(T.end(), o.T_f_w, o.T_f_w + 12), patch.insert(patch.end(), o.patch, o.patch + 64), mean.push_back(o.mean), id.push_back(o.id);
  status(tag, "score_abi", esikf_vio_score_ref_patches(ctx, (int)n, first.data(), (int)m, pos.data(), nrm.data(), patch.data(), mean.data(), id.data(), T.data(), sc.data(),
                                                       mu.data(), ref.data()));
  sc.resize(m), mu.resize(m), ref.resize(n);
  dumpv(tag, "score.score_abi", sc), dumpv(tag, "score.mean_abi", mu), dumpv(tag, "score.ref_abi", ref);
}

// the front-end calls after the LIO half, in the order of a tick, on the point lists of the last StateEstimation
static void front_end(Pair &p, const Inputs &in, const std::string &tag, bool select_and_update) {
  VoxelMapManager &m = *p.mgr;
  VIOManager &v = *p.vio;
  m.SetWorldCloud(&in.dense);
  status(tag, "world_cloud", m.last_status_);
  p.st = m.state_;
  std::vector<VOXEL_LOCATION> keys;
  v.RetrieveScanVoxels(5 << 2, &m.pv_list_, keys);
  status(tag, "retrieve", v.last_status_), dumpf(tag, "retrieve.keys", keys, [](const VOXEL_LOCATION &q, std::vector<double> &o) { o.push_back(q.x), o.push_back(q.y), o.push_back(q.z); });
  esikf_ctx *ctx = m.context();
  const int npv = (int)m.pv_list_.size();
  std::vector<double> pvw(3 * npv + 3), pvn(3 * npv + 3), pvv(9 * npv + 9);
  for (int i = 0; i < npv; i++) {
    memcpy(&pvw[3 * i], m.pv_list_[i].point_w.v, 24), memcpy(&pvn[3 * i], m.pv_list_[i].normal.v, 24), memcpy(&pvv[9 * i], m.pv_list_[i].var.m, 72);
  }
  {
    std::vector<int32_t> kb(3 * npv + 3);
    int32_t k = 0;
    status(tag, "retrieve_abi", esikf_vio_retrieve_scan(ctx, pvw.data(), npv, 5 << 2, packed(p.st).data(), npv, &k, kb.data(), nullptr));
    std::vector<double> o;
    put_keys(o, kb.data(), k);
    dumpv(tag, "retrieve.keys_abi", o);
  }
  const size_t n = in.cands.size();
  std::vector<double> pos(3 * n), pc(2 * n);
  for (size_t i = 0; i < n; i++) memcpy(&pos[3 * i], in.cands[i].pos_w, 24), memcpy(&pc[2 * i], in.cands[i].pc, 16);
  std::vector<uint8_t> disc;
  v.CheckDepthContinuity((int)n, pos.data(), pc.data(), disc);
  status(tag, "depth", v.last_status_), dumpv(tag, "depth.flags", disc);
  std::vector<uint8_t> disc_abi(n);
  status(tag, "depth_abi", esikf_vio_depth_check(ctx, (int)n, pos.data(), pc.data(), disc_abi.data()));
  dumpv(tag, "depth.flags_abi", disc_abi);
  const size_t q = in.query.size() / 3;
  std::vector<uint8_t> fs(q);
  std::vector<VoxelPlane> planes(q);
  m.FindCorrespond((int)q, reinterpret_cast<const V3D *>(in.query.data()), ESIKF_FIND_RULE_PATCH, fs.data(), planes.data());
  status(tag, "find", m.last_status_), dumpv(tag, "find.found", fs), dumpf(tag, "find.planes", planes, [](const VoxelPlane &q, std::vector<double> &o) {
    put_plane(o, q.center_.v, q.normal_.v, q.plane_var_, q.d_, q.radius_, q.is_plane_);
  });
  {
    std::vector<uint8_t> fa(q);
    std::vector<int64_t> fk(3 * q);
    std::vector<esikf_plane> rows(q);
    status(tag, "find_abi", esikf_map_device_find(ctx, in.query.data(), (int)q, ESIKF_FIND_RULE_PATCH, fa.data(), fk.data(), rows.data()));
    std::vector<double> o;
    for (size_t i = 0; i < q; i++) {
      double var[36] = {0}, zero[3] = {0, 0, 0};
      const esikf_plane &r = rows[i];
      if (fa[i] == ESIKF_FIND_NO_ROOT) {
        put_plane(o, zero, zero, var, 0, 0, false);
        continue;
      }
      for (int a = 0, t = 0; a < 6; a++)
        for (int b = a; b < 6; b++, t++) var[6 * a + b] = var[6 * b + a] = r.plane_var[t];
      put_plane(o, r.center, r.normal, var, r.d, r.radius, fa[i] == ESIKF_FIND_PLANE);
    }
    dumpv(tag, "find.found_abi", fa), dumpv(tag, "find.planes_abi", o);
  }
  if (select_and_update) select(p, in, tag), materialize_and_update(p, tag);
  std::vector<PointXYZRGB> rgb;
  v.ColorizeFrameWorld(BgrImage{p.bgr.data(), p.W, p.H}, 0.01, rgb);
  status(tag, "colorize", v.last_status_), dumpf(tag, "colorize.cloud", rgb, [](const PointXYZRGB &q, std::vector<double> &o) {
    putf(o, &q.x, 1), putf(o, &q.y, 1), putf(o, &q.z, 1), o.push_back(q.r), o.push_back(q.g), o.push_back(q.b);
  });
  {  // SetWorldCloud and ColorizeFrameWorld together
    const int nd = (int)in.dense.size();
    std::vector<float> xyz_in(3 * nd), xyz(3 * nd + 3);
    std::vector<uint8_t> bgr(3 * nd + 3);
    for (int i = 0; i < nd; i++) xyz_in[3 * i] = in.dense[i].x, xyz_in[3 * i + 1] = in.dense[i].y, xyz_in[3 * i + 2] = in.dense[i].z;
    int32_t kept = 0;
    int rc = esikf_rgb_set_cloud(ctx, xyz_in.data(), nd, packed(m.state_).data());
    if (!rc) rc = esikf_rgb_colorize(ctx, p.bgr.data(), p.W, p.H, packed(p.st).data(), 0.01, nd, &kept, xyz.data(), bgr.data(), nullptr);
    status(tag, "colorize_abi", rc);
    std::vector<double> o;
    for (int i = 0; i < kept; i++) putf(o, &xyz[3 * i], 3), o.push_back(bgr[3 * i + 2]), o.push_back(bgr[3 * i + 1]), o.push_back(bgr[3 * i]);
    dumpv(tag, "colorize.cloud_abi", o);
  }
  const int gw = p.W / 10, gh = p.H / 10;
  std::vector<uint8_t> type_map(gw * gh, 0);
  for (size_t i = 0; i < type_map.size(); i += 7) type_map[i] = 1;
  std::vector<NewVisualPoint> np;
  v.GenerateVisualMapPoints(type_map, 10, gw, gh, 5 << 2, &m.pv_list_, nullptr, np);
  status(tag, "generate", v.last_status_), dump_points(tag, "generate.points", np);
  {
    const int cap = gw * gh;
    std::vector<int32_t> src(cap + 1), cell(cap + 1);
    std::vector<double> gpos(3 * cap + 3), gpc(2 * cap + 2), gn(3 * cap + 3), gv(9 * cap + 9);
    std::vector<float> gs(cap + 1), gp(64 * cap + 64);
    int32_t k = 0;
    status(tag, "generate_abi", esikf_vio_generate_points(ctx, pvw.data(), pvn.data(), pvv.data(), npv, nullptr, nullptr, 0, type_map.data(), cap, 10, gw, gh, 5 << 2,
                                                          packed(p.st).data(), cap, &k, src.data(), cell.data(), gpos.data(), gpc.data(), gs.data(), gn.data(),
                                                          gv.data(), gp.data()));
    dump_points_abi(tag, "generate.points_abi", k, src.data(), cell.data(), gpos.data(), gpc.data(), gn.data(), gv.data(), gs.data(), gp.data());
  }
  std::vector<uint8_t> conv(v.total_points, 0), flags;
  std::vector<LastObservation> last(v.total_points);
  for (int i = 0; i < v.total_points; i++) {
    const SubMapCandidate &c = in.cands[v.visual_submap->candidate_index[i]];
    memcpy(last[i].T_f_w, c.T_ref_w, 96), memcpy(last[i].px, c.px_ref, 16);
  }
  std::vector<NewObservation> obs;
  v.UpdateVisualMapPoints(conv, last, flags, obs);
  status(tag, "observe", v.last_status_), dumpv(tag, "observe.flags", flags), dumpf(tag, "observe.new", obs, [](const NewObservation &q, std::vector<double> &o) { o.push_back(q.entry), put(o, q.pc, 2), putf(o, q.patch, 64); });
  {
    const int t = v.total_points;
    std::vector<double> T(12 * t + 12), px(2 * t + 2), opc(2 * t + 2);
    std::vector<uint8_t> fl(t + 1);
    std::vector<int32_t> entry(t + 1);
    std::vector<float> patch(64 * t + 64);
    for (int i = 0; i < t; i++) memcpy(&T[12 * i], last[i].T_f_w, 96), memcpy(&px[2 * i], last[i].px, 16);
    int32_t k = 0;
    status(tag, "observe_abi", esikf_vio_update_points(ctx, t, conv.data(), T.data(), px.data(), packed(p.st).data(), t, &k, fl.data(), entry.data(), opc.data(), patch.data()));
    fl.resize(t);
    std::vector<double> o;
    for (int i = 0; i < k; i++) o.push_back(entry[i]), put(o, &opc[2 * i], 2), putf(o, &patch[64 * i], 64);
    dumpv(tag, "observe.flags_abi", fl), dumpv(tag, "observe.new_abi", o);
  }
  // every candidate scored against its reference patch and its current one, seen from both poses
  std::vector<int32_t> first(1, 0);
  std::vector<ScoredPoint> sp;
  std::vector<PatchObservation> po;
  for (size_t i = 0; i < n; i++) {
    const SubMapCandidate &c = in.cands[i];
    ScoredPoint s;
    memcpy(s.pos, c.pos_w, 24), memcpy(s.normal, c.normal_w, 24);
    sp.push_back(s);
    for (int k = 0; k < 2; k++) {
      PatchObservation o;
      memcpy(o.T_f_w, c.T_ref_w, 96);
      v.getImagePatch(k ? p.gimg : p.gref, k ? c.pc : c.px_ref, o.patch, 0);
      o.mean = 0.0f, o.id = (int32_t)(2 * i + k);
      po.push_back(o);
    }
    first.push_back((int32_t)po.size());
  }
  status(tag, "patches", v.last_status_);
  {  // getImagePatch of the current image against one batched call
    std::vector<float> cur, cur_abi(64 * n);
    for (size_t i = 0; i < n; i++) cur.insert(cur.end(), po[2 * i + 1].patch, po[2 * i + 1].patch + 64);
    int rc = esikf_vio_set_image(ctx, p.gimg.data, p.W, p.H);
    if (!rc) rc = esikf_vio_get_image_patch(ctx, pc.data(), (int)n, 0, cur_abi.data());
    v.InvalidatePatchImages();
    status(tag, "patches_abi", rc), dumpv(tag, "patches.cur", cur), dumpv(tag, "patches.cur_abi", cur_abi);
  }
  std::vector<float> score, mean;
  std::vector<int32_t> ref;
  v.ScoreReferencePatches(first, sp, po, score, mean, ref);
  status(tag, "score", v.last_status_), dumpv(tag, "score.score", score), dumpv(tag, "score.mean", mean), dumpv(tag, "score.ref", ref);
  score_abi(ctx, tag, first, sp, po);
  std::vector<float> wp(64 * v.patch_pyrimid_level, 0.0f);
  const double A[4] = {1.02, 0.01, -0.02, 0.98};
  v.warpAffine(A, p.gref, in.cands[0].px_ref, 0, 1, 1, 4, wp.data());
  status(tag, "affine", v.last_status_), dumpv(tag, "affine.patch", wp);
  std::vector<float> wa(64 * v.patch_pyrimid_level);
  const int32_t idx0 = 0, sl1 = 1;
  status(tag, "affine_abi", esikf_vio_warp_affine(ctx, 1, &idx0, in.cands[0].px_ref, A, &sl1, wa.data()));
  dump(tag, "affine.level", wp.data() + 64, 64 * sizeof(float)), dump(tag, "affine.level_abi", wa.data() + 64, 64 * sizeof(float));
}

static double ms_per_call(int reps, const std::function<void()> &f) {
  f();
  const auto t0 = std::chrono::steady_clock::now();
  for (int r = 0; r < reps; r++) f();
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() / reps;
}

int main(int argc, char **argv) {
  if (argc < 4) return 2;
  in_dir = argv[1], out_dir = argv[2];
  meta = load<double>("meta");
  for (int s = 0; s < 2; s++) {
    const std::string k = s ? "S" : "L";
    inputs[s].pts = load<PointXYZ>(k + "_pts"), inputs[s].dense = load<PointXYZ>(k + "_dense");
    inputs[s].state = load<double>(k + "_state"), inputs[s].query = load<double>(k + "_query"), inputs[s].cands = load<SubMapCandidate>(k + "_cands");
  }
  inputs[2].pts = load<PointXYZ>("W_pts"), inputs[2].state = inputs[0].state;
  Pair *p = make_pair();
  if (p->mgr->last_status_) {
    std::printf("set-up failed: %s\n", p->mgr->last_error_.c_str());
    return 1;
  }
  for (int a = 3; a < argc; a++) {
    std::string cmd = argv[a], tag;
    const size_t c1 = cmd.find(':'), c2 = cmd.find(':', c1 + 1);
    const std::string verb = cmd.substr(0, c1), arg = c1 == std::string::npos ? "" : cmd.substr(c1 + 1, c2 - c1 - 1);
    tag = c2 == std::string::npos ? arg : cmd.substr(c2 + 1);
    const int s = arg == "S" ? 1 : 0;
    if (verb == "new") {
      delete p;
      p = make_pair();
    } else if (verb == "tick") {
      lio(*p, inputs[s], tag);
      lists(*p, tag);
      front_end(*p, inputs[s], tag, true);
    } else if (verb == "lazy") {
      p->mgr->lazy_point_lists_ = true;
      lio(*p, inputs[s], tag);
      const Inputs &o = inputs[1 - s];
      const size_t q = o.query.size() / 3;
      std::vector<uint8_t> fs(q);
      std::vector<VoxelPlane> planes(q);
      p->mgr->UpdateVoxelMap();
      p->mgr->FindCorrespond((int)q, reinterpret_cast<const V3D *>(o.query.data()), ESIKF_FIND_RULE_PATCH, fs.data(), planes.data());
      p->mgr->SetWorldCloud(&o.dense);
      lists(*p, tag);
      p->mgr->lazy_point_lists_ = false;
    } else if (verb == "select" || verb == "select_now") {
      p->st = p->mgr->state_;
      select(*p, inputs[s], tag);
      const StatesGroup st = p->st;
      if (verb == "select") {
        lio(*p, inputs[1 - s], tag + "_between"), lists(*p, tag + "_between");
        front_end(*p, inputs[1 - s], tag + "_between", false);
      }
      p->st = st;
      materialize_and_update(*p, tag);
    } else if (verb == "failbuild") {
      VoxelMapManager &m = *p->mgr;
      m.feats_down_body_ = inputs[0].pts, m.feats_down_size_ = (int)inputs[0].pts.size();
      m.BuildVoxelMap();
      status(tag, "build", m.last_status_);
    } else if (verb == "resident") {
      VoxelMapManager &m = *p->mgr;
      lio(*p, inputs[2], tag);
      m.UpdateVoxelMap();
      status(tag, "update_map", m.last_status_);
      p->st = m.state_;
      std::vector<VOXEL_LOCATION> keys;
      p->vio->RetrieveScanVoxels(5 << 2, nullptr, keys);
      status(tag, "resident", p->vio->last_status_);
      dumpf(tag, "resident.keys", keys, [](const VOXEL_LOCATION &q, std::vector<double> &o) { o.push_back(q.x), o.push_back(q.y), o.push_back(q.z); });
      std::vector<int32_t> kb(3 * inputs[2].pts.size() + 3);
      int32_t k = 0;
      status(tag, "resident_abi", esikf_vio_retrieve_scan(m.context(), nullptr, 0, 5 << 2, packed(p->st).data(), (int32_t)inputs[2].pts.size(), &k, kb.data(), nullptr));
      std::vector<double> o;
      put_keys(o, kb.data(), k);
      dumpv(tag, "resident.keys_abi", o);
    } else if (verb == "score") {
      const std::vector<int32_t> first = load<int32_t>(arg + "_first");
      const std::vector<ScoredPoint> sp = load<ScoredPoint>(arg + "_pts");
      const std::vector<PatchObservation> po = load<PatchObservation>(arg + "_obs");
      std::vector<float> score, mean;
      std::vector<int32_t> ref;
      p->vio->ScoreReferencePatches(first, sp, po, score, mean, ref);
      status(tag, "score", p->vio->last_status_), dumpv(tag, "score.score", score), dumpv(tag, "score.mean", mean), dumpv(tag, "score.ref", ref);
    } else if (verb == "generate") {
      // gen_meta: fx fy cx cy w h d0..d4 | extR 9 extT 3 Rcl 9 Pcl 3 | grid_size grid_n_width grid_n_height border
      const std::vector<double> gm = load<double>("gen_meta"), pw = load<double>("gen_pw"), nrm = load<double>("gen_normal"), var = load<double>("gen_var");
      const std::vector<double> ap = load<double>("gen_add_pos"), an = load<double>("gen_add_normal"), gs = load<double>("gen_state");
      std::vector<uint8_t> img = load<uint8_t>("gen_img"), mask = load<uint8_t>("gen_mask");
      esikf_ctx *ctx = nullptr;
      if (esikf_create(&ctx, 0)) return 1;
      {
        VIOManager v(ctx);
        v.cam.model = 0, v.cam.width = (int)gm[4], v.cam.height = (int)gm[5], v.cam.fx = gm[0], v.cam.fy = gm[1], v.cam.cx = gm[2], v.cam.cy = gm[3];
        for (int k = 0; k < 5; k++) v.cam.d[k] = gm[6 + k];
        memcpy(v.extR.m, &gm[11], 72), memcpy(v.extT.v, &gm[20], 24), memcpy(v.Rcl.m, &gm[23], 72), memcpy(v.Pcl.v, &gm[32], 24);
        StatesGroup st;
        st.unpack(gs.data());
        v.state = &st;
        v.initializeVIO();
        float tmp[64];
        const double centre[2] = {gm[4] / 2, gm[5] / 2};
        v.getImagePatch(GrayImage{img.data(), v.cam.width, v.cam.height}, centre, tmp, 0);  // uploads the frame's image
        std::vector<pointWithVar> pg(pw.size() / 3), add(ap.size() / 3);
        for (size_t i = 0; i < pg.size(); i++) memcpy(pg[i].point_w.v, &pw[3 * i], 24), memcpy(pg[i].normal.v, &nrm[3 * i], 24), memcpy(pg[i].var.m, &var[9 * i], 72);
        for (size_t i = 0; i < add.size(); i++) memcpy(add[i].point_w.v, &ap[3 * i], 24), memcpy(add[i].normal.v, &an[3 * i], 24);
        std::vector<NewVisualPoint> np;
        v.GenerateVisualMapPoints(mask, (int)gm[35], (int)gm[36], (int)gm[37], (int)gm[38], &pg, &add, np);
        status(tag, "generate", v.last_status_), dump_points(tag, "generate.points", np);
      }
      esikf_destroy(ctx);
    } else if (verb == "time") {
      const int reps = std::stoi(tag);
      const Inputs &in = inputs[s];
      VIOManager &v = *p->vio;
      lio(*p, in, "time"), lists(*p, "time"), front_end(*p, in, "time", true);
      const int gw = p->W / 10, gh = p->H / 10;
      std::vector<uint8_t> type_map(gw * gh, 0), conv(v.total_points, 0), flags;
      for (size_t i = 0; i < type_map.size(); i += 7) type_map[i] = 1;
      std::vector<LastObservation> last(v.total_points);
      std::vector<NewVisualPoint> np;
      std::vector<NewObservation> obs;
      std::vector<PointXYZRGB> rgb;
      const double *T_cur_w = meta.data() + 30;
      v.SetReferenceImages(&p->gref, 1);  // the tick's warpAffine replaced them
      const double g = ms_per_call(reps, [&] { v.GenerateVisualMapPoints(type_map, 10, gw, gh, 5 << 2, &p->mgr->pv_list_, nullptr, np); });
      const double u = ms_per_call(reps, [&] { v.UpdateVisualMapPoints(conv, last, flags, obs); });
      const double c = ms_per_call(reps, [&] { v.ColorizeFrameWorld(BgrImage{p->bgr.data(), p->W, p->H}, 0.01, rgb); });
      const double sel = ms_per_call(reps, [&] { v.SelectSubSparseMap(in.cands.data(), (int)in.cands.size(), p->gimg, T_cur_w); });
      // the tick pair of LIVMapper: StateEstimation (lazy point lists) and the update on a host-assembled sub-map
      v.MaterializeWarpPatches();  // the last selection's patches, which the host-assembled sub-map carries
      SubSparseMap host = p->sub;
      v.visual_submap = &host;
      p->mgr->lazy_point_lists_ = true;
      StatesGroup prop;
      prop.unpack(in.state.data());
      const double e = ms_per_call(reps, [&] {
        p->mgr->state_ = prop, p->mgr->StateEstimation(prop);
        p->st = p->stp = p->mgr->state_, v.computeJacobianAndUpdateEKF(p->gimg);
      });
      v.visual_submap = &p->sub, p->mgr->lazy_point_lists_ = false;
      std::printf("time generate %.4f update_points %.4f colorize %.4f select %.4f tick_pair %.4f ms (status %d, %zu points, %zu observations, %zu coloured, %d kept)\n",
                  g, u, c, sel, e, v.last_status_, np.size(), obs.size(), rgb.size(), v.total_points);
    } else {
      std::printf("unknown command %s\n", cmd.c_str());
      return 2;
    }
  }
  delete p;
  return 0;
}
