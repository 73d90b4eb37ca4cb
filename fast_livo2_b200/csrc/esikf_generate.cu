// New visual map points of a VIO tick, VIOManager::generateVisualMapPoints (reference src/vio.cpp:804-906), on the device
// (H100, sm_90a): at most one winner per grid cell of the current frame, in cell order.
//
//   gen_score_kernel   : per point of the scan pg, then of add_from_voxel_map (:809-854), one thread each: the frame pose of
//                        updateFrameState, w2c, the isInFrame(pc.cast<int>(), border) gate, the grid cell, the TYPE_MAP mask
//                        and vk::shiTomasiScore; the cell's winner by atomicMax on a 64-bit key {score bits | ~source}
//   gen_cells_kernel   : keep flag of every cell that has a winner
//   select_scan_kernel : stable offsets in cell order (the sub-map selection's single-CTA scan: a few hundred cells)
//   gen_scatter_kernel : per winning cell (:860-890): source, pos, pc, score, var and the normal with the cos_theta sign flip
//   image_patch_kernel : getImagePatch(img, pc, patch, 0) of the winners (:875)
//
// The reference keeps a cell's point when cur_value > scan_value[index] with scan_value reset to 0: the winner is the first
// point, in the order scan then add_from, with the cell's largest positive score. A positive float orders as its bit pattern,
// so max {score bits << 32 | (2^32 - 1 - source)} over the cell is that point whatever order the threads run in; a score
// <= 0 or NaN is never entered. Everything is evaluated without FMA contraction in the reference's operation order (Rn,
// explicit float rounding): with a pinhole camera the winners and every output are the host's bit for bit. The fisheye
// projection calls atan, where CUDA's and the host's may differ in the last ulp (DESIGN.md §4).

namespace esikf {

#define GEN_THREADS 256

struct GenArgs {
  const uint8_t *img;      // current grey image (esikf_vio_set_image)
  CamDev cam;
  double Rci[9], Pci[3];
  const double *state;     // packed state (device) of the frame pose
  const double *pt;        // [n][pt_stride]: point_w (3) then var (9) of every scan point
  int pt_stride;
  const double *normal;    // [n][3] pv.normal of every scan point
  int n;
  const double *add_pos;   // [n_add][3] add_from_voxel_map[j].point_w
  const double *add_normal;
  int n_add;
  const uint8_t *type_map; // [length] nonzero: grid_num[cell] == TYPE_MAP
  int grid_size, grid_n_width, length, border;
  unsigned long long *key; // [length] zeroed before gen_score_kernel: the cell's winner key, 0 = none
};

__device__ __forceinline__ void gen_frame_pose(const GenArgs &a, double *Rcw, double *Pcw) {
  if (threadIdx.x < 9) Rcw[threadIdx.x] = frame_rcw<Rn>(a.Rci, a.state, true, threadIdx.x);
  __syncthreads();
  if (threadIdx.x < 3) Pcw[threadIdx.x] = frame_pcw<Rn>(Rcw, a.Pci, a.state, true, threadIdx.x);
  __syncthreads();
}

// point_w of source s: scan point s < n, else add_from point s - n
__device__ __forceinline__ const double *gen_pos(const GenArgs &a, int s) {
  return s < a.n ? a.pt + (size_t)s * a.pt_stride : a.add_pos + 3 * (size_t)(s - a.n);
}

// vk::shiTomasiScore(img, u, v) (vikit, unpinned; the restatement of oracle/ref_shim/vikit/vision.h): the 8 x 8 box of central
// differences around (u, v), float sums in y-then-x order, each sum divided in double by 2 * box_area, the smaller eigenvalue
// of the structure tensor in float; 0 when the box and its one-pixel ring leave the image.
__device__ __forceinline__ float shi_tomasi_score(const uint8_t *__restrict__ img, int W, int H, int u, int v) {
  const int x_min = u - 4, x_max = u + 4, y_min = v - 4, y_max = v + 4;
  if (x_min < 1 || x_max >= W - 1 || y_min < 1 || y_max >= H - 1) return 0.0f;
  float dXX = 0.0f, dYY = 0.0f, dXY = 0.0f;
  for (int y = y_min; y < y_max; ++y) {
    const uint8_t *row = img + (long)W * y + x_min, *up = row - W, *down = row + W;
#pragma unroll
    for (int x = 0; x < 8; ++x) {
      const float dx = (float)((int)__ldg(row + x + 1) - (int)__ldg(row + x - 1)), dy = (float)((int)__ldg(down + x) - (int)__ldg(up + x));
      dXX = __fadd_rn(dXX, __fmul_rn(dx, dx)), dYY = __fadd_rn(dYY, __fmul_rn(dy, dy)), dXY = __fadd_rn(dXY, __fmul_rn(dx, dy));
    }
  }
  dXX = (float)__ddiv_rn((double)dXX, 128.0), dYY = (float)__ddiv_rn((double)dYY, 128.0), dXY = (float)__ddiv_rn((double)dXY, 128.0);
  const float s = __fadd_rn(dXX, dYY);
  const float disc = __fsub_rn(__fmul_rn(s, s), __fmul_rn(4.0f, __fsub_rn(__fmul_rn(dXX, dYY), __fmul_rn(dXY, dXY))));
  return (float)__dmul_rn(0.5, (double)__fsub_rn(s, __fsqrt_rn(disc)));
}

// w2c of a world point (pc in double) and its grid cell; false when isInFrame(pc.cast<int>(), border) fails or (where the
// reference would index past grid_num) the cell lies outside the grid
__device__ __forceinline__ bool gen_cell(const GenArgs &a, const double *Rcw, const double *Pcw, const double *p, Rn pf[3], Rn &u, Rn &v, int &cell) {
  frame_point(Rcw, Pcw, Rn(p[0]), Rn(p[1]), Rn(p[2]), pf);
  world2cam(a.cam, pf[0], pf[1], pf[2], u, v);
  // truncation toward zero; out of int range the host's conversion gives INT_MIN and the device's saturates: both fail the
  // test. NaN gives INT_MIN on the host and 0 on the device, which passes with border 0, where the score box (u - 4 < 1) is 0.
  const int ui = (int)u.v, vi = (int)v.v;
  if (!(ui >= a.border && ui < a.cam.width - a.border && vi >= a.border && vi < a.cam.height - a.border)) return false;
  const double g = (double)a.grid_size;
  cell = (int)__ddiv_rn(v.v, g) * a.grid_n_width + (int)__ddiv_rn(u.v, g);
  return cell >= 0 && cell < a.length;
}

__global__ void __launch_bounds__(GEN_THREADS) gen_score_kernel(const GenArgs a) {
  __shared__ double Rcw[9], Pcw[3];
  gen_frame_pose(a, Rcw, Pcw);
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= a.n + a.n_add) return;
  if (s < a.n) {  // pg[i].normal == V3D(0, 0, 0): skipped (add_from points are not tested)
    const double *nv = a.normal + 3 * (size_t)s;
    if (nv[0] == 0.0 && nv[1] == 0.0 && nv[2] == 0.0) return;
  }
  Rn pf[3], u, v;
  int cell;
  if (!gen_cell(a, Rcw, Pcw, gen_pos(a, s), pf, u, v, cell) || a.type_map[cell]) return;
  const float score = shi_tomasi_score(a.img, a.cam.width, a.cam.height, (int)u.v, (int)v.v);
  if (!(score > 0.0f)) return;
  atomicMax(a.key + cell, ((unsigned long long)__float_as_uint(score) << 32) | (0xffffffffu - (unsigned)s));
}

__global__ void gen_cells_kernel(const unsigned long long *__restrict__ key, int length, int32_t *__restrict__ keep) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < length) keep[c] = key[c] != 0ull;
}

struct GenOut {
  int32_t *source, *cell;  // [length] source (scan index, or ESIKF_GEN_ADD_FROM | add_from index), grid cell
  double *pos, *pc, *normal, *var;  // [length][3], [2], [3], [9]
  float *score;            // [length]
};

// append_voxel_points[cell] of every TYPE_POINTCLOUD cell at dst[cell]: the record :864-890 builds its VisualPoint from
__global__ void __launch_bounds__(GEN_THREADS) gen_scatter_kernel(const GenArgs a, const int32_t *__restrict__ keep, const int32_t *__restrict__ dst,
                                                                   const GenOut o) {
  __shared__ double Rcw[9], Pcw[3];
  gen_frame_pose(a, Rcw, Pcw);
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.length || !keep[c]) return;
  const unsigned long long k = a.key[c];
  const int s = (int)(0xffffffffu - (unsigned)k), p = dst[c];
  const double *pw = gen_pos(a, s);
  const double *nw = s < a.n ? a.normal + 3 * (size_t)s : a.add_normal + 3 * (size_t)(s - a.n);
  Rn pf[3], u, v;
  int cell;
  gen_cell(a, Rcw, Pcw, pw, pf, u, v, cell);  // the winner passed it: pf, pc as when it was scored
  const Rn cos_theta = view_cos(Rcw, pf, nw);
  const bool flip = cos_theta.v < 0.0;
  o.source[p] = s < a.n ? s : (ESIKF_GEN_ADD_FROM | (s - a.n));
  o.cell[p] = c;
  o.score[p] = __uint_as_float((unsigned)(k >> 32));
  for (int r = 0; r < 3; r++) o.pos[3 * (size_t)p + r] = pw[r], o.normal[3 * (size_t)p + r] = flip ? -nw[r] : nw[r];
  o.pc[2 * (size_t)p] = u.v, o.pc[2 * (size_t)p + 1] = v.v;
  for (int r = 0; r < 9; r++) o.var[9 * (size_t)p + r] = s < a.n ? pw[3 + r] : 0.0;  // add_from: a default pointWithVar's zero var
}

}  // namespace esikf
