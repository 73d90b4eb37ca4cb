// Persistent update kernels of the ESIKF update (H100, sm_90a): the WHOLE iteration loop of one LIO / VIO update in a
// single cooperative launch, so a tick costs one launch instead of 2 x iterations, the state never leaves the chip between
// iterations and no kernel boundary separates the residual build from the gain solve.
//
//   lio_update_kernel : VoxelMapManager::StateEstimation's loop          (reference src/voxel_map.cpp:372-500)
//   vio_update_kernel : VIOManager::computeJacobianAndUpdateEKF's loops   (src/vio.cpp:784-802, 1520-1688)
//
// Every CTA (one per SM, co-resident) keeps its own copy of P, the current / prior pose and the loop control in shared
// memory for the whole update. Per iteration: build the residual / Jacobian rows of the CTA's slice and contract them on
// the fp64 tensor-core path -> combine the CTAs' compact partial vectors in a fixed order (VIO: tagged-word reduce-scatter /
// all-gather through the grid mailbox; LIO: one grid barrier, then every CTA sums every column; state_propagat (-) state is
// evaluated inside the wait) -> every CTA runs the same m x m gain solve and boxplus — same instructions on the same
// inputs, so all copies stay bit-identical. Only the LAST CTA writes results and diagnostics (its
// slice is never the largest, so the stores stay off the critical path of the grid). With peer GPUs attached (PEER) CTA 0
// additionally pushes the rank's vector into every rank's NVLink mailbox and every CTA adds the rank-ordered sum pulled
// from the local one.
#include "esikf_dev.cuh"

namespace esikf {

// Optional phase timestamps (ns, %globaltimer) written by CTA 0 / thread 0 — measurement only.
// The VIO kernel's finer stamps (builds with ESIKF_VIO_CHAIN_STAMPS; VioKernelArgs::chain, 8 per (level, iteration) slot,
// 64 slots; tools/ab_timing.py): warp 0's first patch
// (vio_process_range) at 8 slot + 0..3, every CTA's slice end (its partial summed) at VIO_CHAIN_CTA + VIO_CHAIN_MAX_CTAS slot
// + blockIdx.x.
#define VIO_CHAIN_CTA (8 * 64)
#define VIO_CHAIN_MAX_CTAS 160
__device__ __forceinline__ void stamp(unsigned long long *stamps, int &k) {
  if (stamps && blockIdx.x == 0 && threadIdx.x == 0) stamps[k] = globaltimer_ns();
  k++;
}

// Every wait inside the persistent kernels (grid barrier, grid mailbox, peer mailbox) is bounded: a rank that never arrives must not
// hang the other seven. On expiry the waiter raises Ctrl::comm_error (host: ESIKF_ERR_COMM at fetch) and stops waiting for
// the rest of the launch; the numbers of that update are invalid but the kernel terminates.
#define ESIKF_WAIT_NS 2000000000ull
struct WaitGuard {
  int *error_flag;  // Ctrl::comm_error in global memory
  bool dead;
};
__device__ __forceinline__ bool wait_expired(WaitGuard &w, unsigned long long t0, unsigned &spins) {
  if ((++spins & 1023u) != 0) return false;
  if (globaltimer_ns() - t0 < ESIKF_WAIT_NS) return false;
  w.dead = true;
  *reinterpret_cast<volatile int *>(w.error_flag) = 1;
  return true;
}

// ---------------------------------------------------------------------------------------------------------------------
// In-kernel all-reduce of the compact information vector over NVLink peer memory (one process per GPU, mailboxes
// exchanged with CUDA IPC), low-latency flavour: no fence, no separate flag. Every rank owns a mailbox
// [2 parities][nranks][NE_MAX entries][2 words] in its own HBM. A double travels as two 64-bit words {payload half |
// 32-bit sequence tag}; aligned 64-bit stores are single-copy atomic, so a reader that sees the expected tag in both words
// has the whole value — one NVLink one-way trip instead of store + system fence + flag. CTA 0 of rank r stores its entries
// into slot (parity, r) of EVERY rank's mailbox (its own included); every CTA of every rank then spins on the nranks slots
// of the LOCAL mailbox and adds them in rank order, so every CTA of every rank forms the bit-identical sum with no
// broadcast, no NCCL call and no kernel boundary.
// Tag and parity follow `seq`, the number of exchanges executed since peer_attach — the context's device-resident exchange
// counter, which also tags the grid mailbox below and persists across launches (levels may end early, updates may stop
// early: a per-launch formula would reuse a parity). Two parities suffice because exchanges strictly alternate: a rank's
// CTA 0 writes exchange k + 2 only after it received every peer's k + 1, which a peer's CTA 0 sends after its own grid
// exchange k + 1 — and every CTA of that peer completes that grid exchange only after it finished pulling exchange k.
struct PeerArgs {
  unsigned long long *const *mbox;  // device array: mailbox base of every rank (own entry = local memory)
  unsigned int *seq;                // device word: exchanges executed so far (same on every rank); set without peers too
  int rank, nranks;
};

// A double as two 64-bit words {payload half | 32-bit tag}: {low half | tag}, {high half | tag}.
__device__ __forceinline__ unsigned long long tagged_lo(double v, unsigned int tag) { return ((unsigned long long)__double_as_longlong(v) << 32) | tag; }
__device__ __forceinline__ unsigned long long tagged_hi(double v, unsigned int tag) {
  return ((unsigned long long)__double_as_longlong(v) & 0xffffffff00000000ull) | tag;
}
__device__ __forceinline__ bool tags_match(unsigned long long a, unsigned long long b, unsigned int tag) { return (unsigned int)a == tag && (unsigned int)b == tag; }
__device__ __forceinline__ double untagged(unsigned long long a, unsigned long long b) { return __longlong_as_double((long long)((b & 0xffffffff00000000ull) | (a >> 32))); }

__device__ __forceinline__ void peer_push(const double *info, const PeerArgs &p, unsigned int seq) {
  const int tid = threadIdx.x;
  const unsigned int tag = seq + 1u;  // never 0 (the mailbox starts zeroed)
  const int par = seq & 1;
  if (tid < NE_MAX) {
    const unsigned long long w0 = tagged_lo(info[tid], tag), w1 = tagged_hi(info[tid], tag);
    const size_t off = (size_t)(par * p.nranks + p.rank) * PEER_SLOT_WORDS + 2 * tid;
    for (int r = 0; r < p.nranks; r++) {
      unsigned long long *dst = p.mbox[r] + off;
      asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(dst), "l"(w0) : "memory");
      asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(dst + 1), "l"(w1) : "memory");
    }
  }
}
__device__ __forceinline__ void peer_pull(double *info, const PeerArgs &p, unsigned int seq, WaitGuard &wg) {
  const int tid = threadIdx.x;
  const unsigned int tag = seq + 1u;
  const int par = seq & 1;
  if (tid < NE_MAX) {
    const unsigned long long *own = p.mbox[p.rank] + (size_t)par * p.nranks * PEER_SLOT_WORDS + 2 * tid;
    double s = 0.0;
    const unsigned long long t0 = globaltimer_ns();
    unsigned spins = 0;
    for (int r = 0; r < p.nranks; r++) {
      const unsigned long long *src = own + (size_t)r * PEER_SLOT_WORDS;
      unsigned long long a, b;
      for (;;) {
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(a) : "l"(src) : "memory");
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(b) : "l"(src + 1) : "memory");
        if (tags_match(a, b, tag) || wg.dead || wait_expired(wg, t0, spins)) break;
      }
      s += untagged(a, b);
    }
    info[tid] = s;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// How the CTAs of a persistent launch combine their partial vectors. Both forms give the same sums, bit for bit; which one a
// kernel uses was measured on H100 (DESIGN §8): the grid mailbox cuts the VIO iteration (short slices, 125 CTAs) from
// 11.0 to 10.1 us on config 2, while the LIO update is 1-6 % slower with it than with the grid barrier on configs 2-5.
template <int M> __host__ __device__ constexpr bool uses_grid_mailbox() { return M == 7; }  // VIO

// Counting grid barrier over all CTAs of a cooperative launch: arrivals are release-increments, thread 0 of every CTA polls
// the same counter with acquire loads; the k-th barrier (k = 0, 1, ...) completes when it reaches (k + 1) * gridDim.x. The
// counter is zeroed for this launch by the previous launch (launches alternate between two counters). The waiting time does
// useful work: every thread but thread 0 runs `work` meanwhile. A variant with a separate release word written by the last
// arriver costs an extra L2 hop per barrier.
template <class F> __device__ __forceinline__ void grid_barrier_overlap(unsigned int *counter, unsigned int &epoch, WaitGuard &wg, F work) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int target = (epoch + 1) * gridDim.x;
    // release-increment: orders this CTA's earlier writes (made visible to thread 0 by the CTA barrier above) before the
    // arrival, without a separate membar; the acquire poll orders the other CTAs' writes before everything after it.
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
    unsigned int v;
    const unsigned long long t0 = globaltimer_ns();
    unsigned spins = 0;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
    } while (v < target && !wg.dead && !wait_expired(wg, t0, spins));
  } else {
    work();
  }
  epoch++;
  __syncthreads();
}

// Grid mailbox: the peer mailbox's tagged words (above) inside one GPU, so no fence, no counter and no grid barrier. The
// context owns one zero-initialised grid mailbox of tagged u64 words:
//   partial columns [2 parities][NE_MAX][partial_stride][2 words]   entry-major like `partials`: a warp's loads coalesce
//   entry totals    [2 parities][NE_MAX][2 words]
// Exchange k (tag k + 1, parity k & 1, k = the context's exchange counter `seq`) runs in two hops:
//   reduce-scatter: every CTA stores its column; entry e is summed by one warp of CTA e mod gridDim.x, which polls the
//                   entry's gridDim.x columns and stores the tagged total;
//   all-gather:     every CTA polls the NE totals.
// Parity reuse: CTA c stores its column of exchange k + 2 only after its all-gather k + 1 saw every total of k + 1; the
// warp that stored a total of k + 1 had read its columns of k + 1, which it polled after it had read (and summed into the
// stored total) those of k. The same chain covers the totals: a total of k + 2 needs every CTA's column of k + 2, stored
// after that CTA's all-gather k + 1, which it ran after its all-gather k. The stores that close each chain carry the values
// those reads returned, so no read is left outstanding behind them.
// Tags across launches: the per-iteration launches (loop_mode 0) use `partials`, never this buffer (the low word of a plain
// double could equal a tag). A launch reads only columns below its own grid size, and every exchange writes all of those
// with its own tag, so a column left behind by a wider launch is never read. The counter only grows (the LIO kernel leaves
// it alone without peers), so a stale word never carries a current tag until it wraps after 2^32 exchanges.
__host__ __device__ constexpr size_t grid_mbox_cols_words(int partial_stride) { return (size_t)NE_MAX * partial_stride * 2; }  // per parity
__host__ __device__ constexpr size_t grid_mbox_words(int partial_stride) { return 2 * grid_mbox_cols_words(partial_stride) + 2 * NE_MAX * 2; }

__device__ __forceinline__ void st_tagged(unsigned long long *dst, double v, unsigned int tag) {
  asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(tagged_lo(v, tag)), "l"(tagged_hi(v, tag)) : "memory");
}
__device__ __forceinline__ void ld_tagged(const unsigned long long *src, unsigned long long &a, unsigned long long &b) {
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(src) : "memory");
}

// Entry e of exchange `tag` by one warp: the nb tagged columns of `col` (entry e's row), summed in sum_partials' order; lane 0
// stores the tagged total. Every pass issues all the still-missing loads before it checks any of them.
__device__ __forceinline__ void reduce_entry(const unsigned long long *col, int nb, unsigned int tag, unsigned long long *total, WaitGuard &wg) {
  const int lane = threadIdx.x & 31;
  unsigned long long w[SUM_MAXC][2];
  unsigned pending = 0;
#pragma unroll
  for (int c = 0; c < SUM_MAXC; c++) {
    w[c][0] = w[c][1] = 0ull;
    if (lane + 32 * c < nb) pending |= 1u << c;
  }
  const unsigned long long t0 = globaltimer_ns();
  unsigned spins = 0;
  while (pending) {
    const unsigned want = pending;
#pragma unroll
    for (int c = 0; c < SUM_MAXC; c++)
      if ((want >> c) & 1u) ld_tagged(col + 2 * (lane + 32 * c), w[c][0], w[c][1]);
#pragma unroll
    for (int c = 0; c < SUM_MAXC; c++)
      if (((want >> c) & 1u) && tags_match(w[c][0], w[c][1], tag)) pending &= ~(1u << c);
    if (pending && (wg.dead || wait_expired(wg, t0, spins))) break;
  }
  double v[SUM_MAXC];
#pragma unroll
  for (int c = 0; c < SUM_MAXC; c++) v[c] = (lane + 32 * c < nb) ? untagged(w[c][0], w[c][1]) : 0.0;
  const double s = column_sum(v);
  if (lane == 0) st_tagged(total, s, tag);
}

// The grid-sync arguments of both persistent kernels: the LIO kernel's grid barrier (this launch's counter, and the next
// launch's, which CTA 0 zeroes: no host memset per update) and the VIO kernel's grid mailbox.
struct GridSync {
  unsigned int *barrier, *barrier_next;
  unsigned long long *mbox;
};

struct FusedSolveSmem {
  SolveSmem sm;
  SolveIO io;
  Ctrl ctrl;  // the CTA's working copy of the loop-control block
  WaitGuard wg;
};
static_assert(sizeof(FusedSolveSmem) % 8 == 0, "what follows it in shared memory holds doubles");

// Prologue of both persistent kernels: the CTA's loop control, wait guard and literal-mode workspace (solve_mode 1 borrows
// `lit`), the next launch's barrier counter, zeroed stats, P and the poses staged once for the whole update, and the gain's
// loop invariants on the last warp. `setup` is the kernel's own set-up and ends with a CTA barrier (fs.sm.P is in place
// after it). Returns the exchange counter where the kernel uses it (grid mailbox or peers), else 0.
template <int M, int WARPS, bool PEER, class F>
__device__ __forceinline__ unsigned int persist_prologue(FusedSolveSmem &fs, SolveLiteralScratch &lit, SolveArgs &sa, const GridSync &gs, const PeerArgs &peer,
                                                         double pscale, F setup) {
  const bool publisher = (blockIdx.x == gridDim.x - 1);
  sa.no_publish = !publisher;
  if (threadIdx.x == 0) {
    Ctrl z;
    memset(&z, 0, sizeof(z));
    fs.ctrl = z;
    fs.wg.error_flag = &sa.ctrl->comm_error, fs.wg.dead = false;
    fs.sm.W = lit.W, fs.sm.K = lit.K;
    if (blockIdx.x == 0) gs.barrier_next[0] = 0u, gs.barrier_next[32] = 0u;
  }
  int *const stats = (M == 6) ? reinterpret_cast<int *>(sa.lio_stats) : reinterpret_cast<int *>(sa.vio_stats);
  const int stats_words = (int)((M == 6) ? sizeof(esikf_lio_stats) : sizeof(esikf_vio_stats)) / 4;
  if (publisher && stats)
    for (int t = threadIdx.x; t < stats_words; t += blockDim.x) stats[t] = 0;
  solve_load(fs.sm, fs.io, sa, false);
  const unsigned int seq = (PEER || uses_grid_mailbox<M>()) ? __ldcg(peer.seq) : 0u;
  setup();
  if ((threadIdx.x >> 5) == WARPS - 1 && sa.solve_mode == 0) gain_setup<M>(fs.sm, pscale, threadIdx.x & 31);  // first used after two CTA barriers
  return seq;
}

// Exchange step of one iteration: warp 1 evaluates vec = state_propagat (-) state (voxel_map.cpp:470 / vio.cpp:1664) while
// the CTA waits for the other CTAs; the fixed-order sum lands in fs.io.info and, with peers, is replaced by the rank-ordered
// sum over the peer mailboxes. Ends with a CTA barrier. Phase stamp: this CTA sees every CTA's contribution. cta_done
// (grid mailbox, measurement only): when this CTA's partial was summed, at cta_done[blockIdx.x].
//   grid mailbox (VIO): the CTA's tagged column, the reduce-scatter of the entries this CTA owns, the all-gather of the
//                       totals;
//   grid barrier (LIO): the CTA's column of `partials` (double-buffered by the launch's exchange count `epoch`), the
//                       barrier, every CTA sums every column.
template <int WARPS, int M, bool PEER>
__device__ __forceinline__ void persist_exchange(FusedSolveSmem &fs, ReduceSmem<WARPS> &red, double D0, double D1, double cnt, const GridSync &gs, double *partials,
                                                 int partial_stride, unsigned int &epoch, const PeerArgs &peer, unsigned int &seq, unsigned long long *stamps, int &sk,
                                                 unsigned long long *cta_done = nullptr) {
  constexpr int NE = ne_of(M);
  const int tid = threadIdx.x, warp = tid >> 5, nb = gridDim.x;
  if constexpr (uses_grid_mailbox<M>()) {
    const unsigned int tag = seq + 1u;  // never 0 (the mailbox starts zeroed)
    unsigned long long *cols = gs.mbox + (seq & 1) * grid_mbox_cols_words(partial_stride);
    unsigned long long *totals = gs.mbox + 2 * grid_mbox_cols_words(partial_stride) + (seq & 1) * NE_MAX * 2;
    const double s = cta_partial<WARPS, M>(red, D0, D1, cnt);
    if (cta_done && tid == 0) stamp_after(cta_done + blockIdx.x, s);
    if (tid < NE) st_tagged(cols + 2 * ((size_t)tid * partial_stride + blockIdx.x), s, tag);
    if (warp == 1) boxminus_warp(fs.io.pr, fs.io.st, fs.sm.vec, tid & 31);
    for (int e = blockIdx.x + warp * nb; e < NE; e += WARPS * nb) reduce_entry(cols + 2 * (size_t)e * partial_stride, nb, tag, totals + 2 * e, fs.wg);
    if (tid < NE) {
      unsigned long long a, b;
      const unsigned long long t0 = globaltimer_ns();
      unsigned spins = 0;
      for (;;) {
        ld_tagged(totals + 2 * tid, a, b);
        if (tags_match(a, b, tag) || fs.wg.dead || wait_expired(fs.wg, t0, spins)) break;
      }
      fs.io.info[tid] = untagged(a, b);
    }
    __syncthreads();
    stamp(stamps, sk);
  } else {
    double *part = partials + (size_t)(epoch & 1) * partial_stride * NE_MAX;
    store_partials<WARPS, M>(red, D0, D1, cnt, part, partial_stride);
    grid_barrier_overlap(gs.barrier, epoch, fs.wg, [&]() {
      if (warp == 1) boxminus_warp(fs.io.pr, fs.io.st, fs.sm.vec, tid & 31);
    });
    stamp(stamps, sk);
    sum_partials<M>(part, partial_stride, nb, fs.io.info, WARPS);
    __syncthreads();
  }
  if (PEER) {
    if (blockIdx.x == 0) peer_push(fs.io.info, peer, seq);
    peer_pull(fs.io.info, peer, seq, fs.wg);
    __syncthreads();
  }
  if (PEER || uses_grid_mailbox<M>()) seq++;
}

// Epilogue, publisher only: the loop-control block and, where the kernel uses it, the exchange counter back to global
// memory. An expired wait stays raised, whether this CTA or another one saw it.
template <int M, bool PEER> __device__ __forceinline__ void persist_epilogue(FusedSolveSmem &fs, Ctrl *ctrl, const PeerArgs &peer, unsigned int seq) {
  if (threadIdx.x == 0) {
    fs.ctrl.comm_error = fs.wg.dead ? 1 : 0;
    const int err = *reinterpret_cast<volatile int *>(&ctrl->comm_error);
    *ctrl = fs.ctrl;
    if (err) ctrl->comm_error = 1;
    if (PEER || uses_grid_mailbox<M>()) *peer.seq = seq;
  }
}

template <bool PEER, int L2W>
__global__ void __launch_bounds__(LioSmem<L2W>::THREADS, 1) lio_update_kernel(const LioKernelArgs a, const SolveArgs sa_in, const GridSync gs, unsigned long long *stamps,
                                                                              const PeerArgs peer) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  LioSmem<L2W> &sm = *reinterpret_cast<LioSmem<L2W> *>(smem_raw);
  static_assert(sizeof(FusedSolveSmem) <= sizeof(sm.fs_raw), "solve state must fit");
  static_assert(sizeof(SolveLiteralScratch) <= sizeof(sm.rec), "literal scratch must fit in the record slots");
  FusedSolveSmem &fs = *reinterpret_cast<FusedSolveSmem *>(sm.fs_raw);
  SolveLiteralScratch &lit = *reinterpret_cast<SolveLiteralScratch *>(&sm.rec[0][0][0]);
  SolveArgs sa = sa_in;
  unsigned int epoch = 0;
  int lo, hi;
  lio_block_range(a.count, lo, hi);
  unsigned int seq = persist_prologue<6, LioSmem<L2W>::WARPS, PEER>(fs, lit, sa, gs, peer, 1.0, [&]() {
    lio_prior_consts(sm, a);  // never change inside the loop
    lio_init_cold(sm, a);
    lio_init_barriers(sm);    // fs.sm.P is in place
    lio_pose_consts(sm, fs.io.st, fs.sm.P, false);  // Ptt / Ppp for the whole update
  });
  int sk = 0;
  LaneCache lc;
  lane_cache_init(lc);
  for (int it = 0; it < sa.max_iterations; it++) {
    stamp(stamps, sk);  // 0: iteration start
    lio_pose_consts(sm, fs.io.st, nullptr, false);
    stamp(stamps, sk);  // 1: constants in place
    double D0 = 0.0, D1 = 0.0;
    int cnt = 0;
    // literal solve mode borrows the record slots as workspace: the per-point outputs cannot wait there for the last iteration
    lio_process_range(a, sm, lo, hi, D0, D1, cnt, lc, it == 0, sa.solve_mode == 1);
    if (stamps && it == 3) {  // measurement only: when did every CTA finish its slice of iteration 3?
      __syncthreads();
      if (threadIdx.x == 0) stamps[640 + blockIdx.x] = globaltimer_ns();
    }
    stamp(stamps, sk);  // 2: this CTA's warps issued their slice (CTA 0 / thread 0)
    persist_exchange<LioSmem<L2W>::WARPS, 6, PEER>(fs, sm.red, D0, D1, (double)cnt, gs, a.partials, a.partial_stride, epoch, peer, seq, stamps,
                                                   sk);  // 3: all CTAs arrived
    stamp(stamps, sk);  // 4: information vector complete
    sa.dbg = (stamps && blockIdx.x == 0) ? stamps + sk + 1 : nullptr;  // 6: gain rows done, 7: boxplus done
    lio_solve_block(sa, fs.sm, fs.io, fs.ctrl);
    if (sa.solve_mode == 1) lane_cache_reset(lc);  // the literal workspace borrowed the record slots
    stamp(stamps, sk);  // 5: solved (state, loop control current in every CTA)
    sk += 2;            // 6, 7: spare
    if (fs.ctrl.stop) break;  // EKF_stop_flg (voxel_map.cpp:499)
  }
  if (sa.solve_mode != 1) lio_write_outputs(a, sm, lo, hi, lc);
  if (!sa.no_publish) persist_epilogue<6, PEER>(fs, a.ctrl, peer, seq);
}

// INVERSE: the inverse-compositional variant (vio/inverse_composition_en, src/vio.cpp:792-795, 1327-1518) in the same loop:
// every warp precomputes H_sub_inv of ITS patches when a level starts (precomputeReferencePatches; written and later read by
// the same lanes, so no barrier is involved) and the per-iteration build is vio_inverse_process_range.
template <bool PEER, bool INVERSE>
__global__ void __launch_bounds__(VIO_THREADS, 1) vio_update_kernel(const VioKernelArgs a, SolveArgs sa, const GridSync gs, unsigned long long *stamps, const PeerArgs peer, const VioInvArgs inv,
                                                                     const __grid_constant__ VioTma tma) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  VioSmem &sm = *reinterpret_cast<VioSmem *>(smem_raw);
  FusedSolveSmem &fs = *reinterpret_cast<FusedSolveSmem *>(smem_raw + sizeof(VioSmem));
  SolveLiteralScratch &lit = *reinterpret_cast<SolveLiteralScratch *>(&sm.rows[0][0][0]);
  static_assert(sizeof(SolveLiteralScratch) <= sizeof(sm.rows), "literal scratch must fit in the row staging area");
  unsigned int epoch = 0;
  int lo, hi;
  vio_block_range(a.count, lo, hi);
  const bool cached = (hi - lo) <= VIO_WARPS * VIO_KMAX;
  unsigned tma_phase = 0;  // parity of this warp's TMA barrier
  unsigned int seq = persist_prologue<7, VIO_WARPS, PEER>(fs, lit, sa, gs, peer, 1.0 / sa.img_point_cov, [&]() {
    vio_cache_reset(sm);
    if (threadIdx.x < VIO_WARPS) mbar_init(&sm.tma_bar[threadIdx.x], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
  });
  for (int level = a.levels - 1; level >= 0; level--) {      // vio.cpp:790
    for (int it = 0; it < sa.max_iterations; it++) {          // :1536
      int sk = 8 * ((a.levels - 1 - level) * sa.max_iterations + it);
      if (a.chain && threadIdx.x == 0) sm.stamp_slot = sk >> 3;
      stamp(stamps, sk);
      vio_load_consts(sm, a, fs.io.st, false);
      stamp(stamps, sk);
      double D0 = 0.0, D1 = 0.0, n_meas = 0.0;
      if (INVERSE) {
        if (it == 0)
          for (int lp = lo + (int)(threadIdx.x >> 5); lp < hi; lp += VIO_WARPS) vio_inverse_precompute_patch(a, inv, level, lp, threadIdx.x & 31);
        vio_inverse_process_range(a, inv, sm, level, lo, hi, fs.io.st + S_R, fs.io.st + S_P, D0, D1, n_meas);
      } else {
        vio_process_range(a, sm, level, lo, hi, D0, D1, n_meas, cached, tma.enabled ? &tma : nullptr, &tma_phase);
      }
      stamp(stamps, sk);
#ifdef ESIKF_VIO_CHAIN_STAMPS
      unsigned long long *const cta_done = a.chain ? a.chain + VIO_CHAIN_CTA + VIO_CHAIN_MAX_CTAS * (sk >> 3) : nullptr;
#else
      unsigned long long *const cta_done = nullptr;
#endif
      persist_exchange<VIO_WARPS, 7, PEER>(fs, sm.red, D0, D1, n_meas, gs, a.partials, a.partial_stride, epoch, peer, seq, stamps, sk, cta_done);
      stamp(stamps, sk);
      sa.level = level, sa.slot_iter = it;
      sa.dbg = (stamps && blockIdx.x == 0) ? stamps + sk + 1 : nullptr;  // 6: gain rows done, 7: boxplus done
      vio_solve_block(sa, fs.sm, fs.io, fs.ctrl);
      if (sa.solve_mode == 1) {  // the literal workspace borrowed the row area; nothing cached lives there
        __syncthreads();
      }
      stamp(stamps, sk);
      if (fs.ctrl.level_done) break;  // EKF_end (:1685)
    }
  }
  if (!sa.no_publish) {
    __syncthreads();  // this CTA's threads stored every accepted G
    if (fs.ctrl.has_G) vio_final_cov(sa, fs.sm, fs.io, false);
    persist_epilogue<7, PEER>(fs, a.ctrl, peer, seq);
  }
}

}  // namespace esikf
