// fit_tc.cu -- the sm_90a fast path: TMA-staged series tiles, wgmma moment GEMM with the
// centred series as the register A operand, per-row epilogue.
//
// What it computes (reference 02_Fine_Grained_Demand_Forecasting.py:435-494 for every group of the
// applyInPandas fan-out 02:523-528, in the whitened calendar basis of DESIGN.md section 2):
//     b_i  = A_fit^T (y_i - c_i)          [128 series x T] x [T x 16]  -> wgmma tf32
//     yhat = c_i + A_pred b_i             (fully observed series: G_i = I, gamma_i = b_i)
// fp32-grade accuracy on the tf32 tensor path comes from an exact 2-term split of both operands
//     y - c = hi + lo,  A = A_hi + A_lo  ->  D = hi*[A_hi | A_lo] + lo*[A_hi | A_lo]   (N = 32 each, b = D[:, p] + D[:, P + p])
// (lo*A_lo is below fp32 rounding; it is computed only so that both MMAs have the same shape and may chain on one
// accumulator -- wgmma orders accumulator accesses only between MMAs of the same shape)
// Rows that contain a non-finite value poison only their own accumulator row (NaN/Inf); the epilogue
// detects that, marks the row MMF_STATUS_PENDING and the masked warp kernel finishes them.
//
// CTA = 13 warps, 1 CTA per SM, persistent over 128-series tiles, every stage decoupled by mbarriers:
//   warp 12    TMA producer: y box {32 t x 128 series} + design box {32 t x 32 (hi|lo columns)} per stage.
//   warps 0-3 / 4-7   two consumer warpgroups taking alternate 32-step chunks.  Per chunk each thread first scans
//              series row r of the tile (r = its index in the warpgroup) for gaps, then loads its m16n8k8 fragments
//              of both 64-row halves from the TMA-swizzled stage, centres and splits them hi/lo and issues the
//              wgmma.mma_async chain into register accumulators.  At the end of a tile both warpgroups hand their
//              partial moments (and gap counts) to the epilogue through a double-buffered shared-memory slot.
//   warps 8-11 epilogue: sum the two partials of a finished tile, release the slot at once, then forecast + store
//              while the next tile is already streaming.
// Algorithmic HBM bytes per series: 4*t_fit read + 4*n_pred written (DESIGN.md section 4).
#include "mmf_internal.cuh"
#include "sm90_ptx.cuh"

namespace mmf {
namespace {

using namespace sm90;

constexpr int TILE_M = 128;            // series per tile
constexpr int KC = 32;                 // time steps per stage == one 128-B swizzle row
// The shared-memory ring (20 KB per stage) and the number of forecast staging tiles are template parameters of the
// kernel: <8 stages, 1 staging tile> is the product configuration, <6, 2> (a second staging tile lets tile k+1 be
// assembled while the NVLink stores of tile k are still reading tile k's) an experiment.
constexpr int NGROUPS = 2;             // consumer warpgroups (alternate chunks)
// A wgmma accumulator rounds every addition relative to the running partial sum, which grows with the fit window, so
// summing a long window in one accumulator has an error that grows linearly with t_fit (36x the parity tolerance at
// 70,001 rows).  Each consumer group therefore adds its accumulator into a running fp32 sum (kept in the tile's slot
// of partial moments in shared memory) and restarts it after every FOLD_CHUNKS of its chunks.  Tiles of up to 2 * 18 chunks (t_fit <= 1,152) never fold and are summed exactly as
// without folding.
constexpr int FOLD_CHUNKS = 18;
constexpr int MAX_PRED = 64;           // forecast rows the epilogue supports
constexpr int BULK_MAX_PRED = 28;      // forecast rows the staged bulk-store epilogue supports (14 KB of smem)
constexpr int Y_STAGE_BYTES = TILE_M * KC * 4;      // 16384
constexpr int AT_STAGE_BYTES = 2 * P * KC * 4;      // 4096
constexpr int THREADS = 416;
constexpr int TILE_RING = 4;           // tiles the producer has claimed and published, not yet taken by every warp
constexpr int WARP_EPI0 = 8, WARP_PROD = 12;
// named barriers: 1-3 epilogue, 4 + g consumer warpgroup g

template <int STAGES, int OBUF, bool SE = false>
struct SmemLayoutT {
  // offsets from the 1024-aligned base
  static constexpr int y = 0;
  static constexpr int at = y + STAGES * Y_STAGE_BYTES;
  static constexpr int apred = at + STAGES * AT_STAGE_BYTES;
  static constexpr int ostage = apred + MAX_PRED * P * 4;            // forecast tile staged for the bulk stores
  static constexpr int acc = ostage + OBUF * TILE_M * BULK_MAX_PRED * 4;   // partial moments: [2 slots][2 groups][128][P] f32
  static constexpr int nm = acc + 2 * NGROUPS * TILE_M * P * 4;      // gap counts: [2 slots][2 chunk parities][128] u16
  static constexpr int cc = nm + 2 * NGROUPS * TILE_M * 2;           // centring constants: [2 slots][128] f32
  static constexpr int tiles = cc + 2 * TILE_M * 4;                // claimed tiles in flight: [TILE_RING] int
  static constexpr int bars = tiles + TILE_RING * 4;
  static constexpr int n_bars = 2 * STAGES + 6 + 2 * TILE_RING;
  // SE only: S per row, [2 slots][2 groups][128] f64, and sqrt(1 + h_t) of the prediction rows
  static constexpr int ss = bars + n_bars * 8;
  static constexpr int sfac = ss + (SE ? 2 * NGROUPS * TILE_M * 8 : 0);
  static constexpr int total = sfac + (SE ? MAX_PRED * 4 : 0);
  static_assert(total + 1024 <= 232448, "exceeds the 227 KB of shared memory a CTA can opt into");
};

__device__ __forceinline__ float dot16(const float* __restrict__ arow, const float (&g)[P], float s) {
  const float4* ap = reinterpret_cast<const float4*>(arow);
  const float4 a0 = ap[0], a1 = ap[1], a2 = ap[2], a3 = ap[3];
  s = fmaf(a0.x, g[0], s);  s = fmaf(a0.y, g[1], s);  s = fmaf(a0.z, g[2], s);  s = fmaf(a0.w, g[3], s);
  s = fmaf(a1.x, g[4], s);  s = fmaf(a1.y, g[5], s);  s = fmaf(a1.z, g[6], s);  s = fmaf(a1.w, g[7], s);
  s = fmaf(a2.x, g[8], s);  s = fmaf(a2.y, g[9], s);  s = fmaf(a2.z, g[10], s); s = fmaf(a2.w, g[11], s);
  s = fmaf(a3.x, g[12], s); s = fmaf(a3.y, g[13], s); s = fmaf(a3.z, g[14], s); s = fmaf(a3.w, g[15], s);
  return s;
}

__device__ __forceinline__ bool is_finite_bits(float x) { return (__float_as_uint(x) & 0x7f800000u) != 0x7f800000u; }

// Centring constant of a series: its first finite value among the first 8 (any constant works -- the intercept
// absorbs it exactly -- it only has to be near the series' level and identical in every warp role that uses it).
// NaN when all 8 are missing: the row then takes the general pass.  Taken from the row's first 8 values as staged in
// chunk 0 (a, b), so the row head is not read from global memory again; positions from t_fit on count as missing --
// the TMA clip stages them as 0, not NaN.
__device__ __forceinline__ float centring_constant(const float4& a, const float4& b, int t_fit) {
  const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  float c = t_fit > 7 ? v[7] : __int_as_float(0x7fc00000);
#pragma unroll
  for (int i = 6; i >= 0; --i) c = (i < t_fit && is_finite_bits(v[i])) ? v[i] : c;
  return c;
}

// Backtest: a consumer group's running moments of its four fragment rows at origin k -> bt.mom, folded (hi + lo
// columns, plus the restarted accumulators' sum in the tile's slot) exactly like the tile's hand-off to the epilogue.
__device__ __forceinline__ void bt_write_moments(const BtArgs& bt, int k, int grp, int64_t n, const TileRec& tr, int frow0,
                                                 int t4, const float (&acc)[2][P], bool folded, const float* sacc) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int rt = 64 * h + frow0 + 8 * j;
      if (rt >= tr.nrows) continue;
      float* __restrict__ dst = bt.mom + (((int64_t)k * 2 + grp) * n + tr.row0 + rt) * P + 2 * t4;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int q = 4 * i + 2 * j;                    // acc[h][q + 8] is the lo column of acc[h][q]
        float2 v = make_float2(acc[h][q] + acc[h][q + P / 2], acc[h][q + 1] + acc[h][q + 1 + P / 2]);
        if (folded) {
          const float2 o = *reinterpret_cast<const float2*>(sacc + rt * P + 8 * i + 2 * t4);
          v.x = o.x + v.x; v.y = o.y + v.y;
        }
        *reinterpret_cast<float2*>(dst + 8 * i) = v;
      }
    }
}

__device__ __forceinline__ float lds32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}

// MULTI: a ragged launch -- every 128-row tile names its calendar (mv.tiles / mv.cals); `n_chunks` is then only the
// minimum over the calendars (>= 2).  MULTI == false compiles to the single-calendar kernel.
// SE (standard-error calls, single calendar): the consumers also sum S = sum (y - c)^2 of their fragment rows and the
// epilogue writes sigma / dof (and the se row in future mode) of the gap-free rows; the MMA inputs are unchanged.
// BT (backtest calls, single calendar, d = the longest window t_K): a consumer group writes its running moments to
// bt.mom at every earlier origin t_k -- a chunk that contains t_k is issued twice, first with its values at t >= t_k
// zeroed, then with the complementary ones -- and the epilogue finishes every origin of a row (DESIGN.md section 4.12).
template <int STAGES, int OBUF, bool MULTI, bool SE = false, bool BT = false>
__global__ void __launch_bounds__(THREADS, 1)
fit_tc_kernel(const __grid_constant__ TcLaunch tl, const DesignView d, const FitArgs a,
              uint32_t* __restrict__ pending_count, const int n_tiles, const int n_chunks, const MultiView mv,
              const SeArgs se, const BtArgs bt) {
  static_assert(!SE || !MULTI, "standard errors are built for the single-calendar launch");
  static_assert(!BT || !(MULTI || SE), "backtests are built for the single-calendar launch");
  using SmemLayout = SmemLayoutT<STAGES, OBUF, SE>;
  auto tile_rec = [&](int ti) -> TileRec {
    if (MULTI) {
      if (ti >= n_tiles) return TileRec{0, 0, 0, 1};
      const int4 v = __ldg(reinterpret_cast<const int4*>(mv.tiles) + ti);
      return TileRec{v.x, v.y, v.z, v.w};
    }
    const int64_t left = a.n - (int64_t)ti * TILE_M;
    return TileRec{ti * TILE_M, (int)(left >= TILE_M ? TILE_M : (left > 0 ? left : 0)), 0, n_chunks};
  };
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  const uint32_t sbase = smem_u32(smem);
  const uint32_t s_y = sbase + SmemLayout::y;
  const uint32_t s_at = sbase + SmemLayout::at;
  float* s_apred = reinterpret_cast<float*>(smem + SmemLayout::apred);
  float* s_ostage = reinterpret_cast<float*>(smem + SmemLayout::ostage);
  float* s_acc = reinterpret_cast<float*>(smem + SmemLayout::acc);
  uint16_t* s_nm = reinterpret_cast<uint16_t*>(smem + SmemLayout::nm);
  float* s_cc = reinterpret_cast<float*>(smem + SmemLayout::cc);
  double* s_ss = reinterpret_cast<double*>(smem + SmemLayout::ss);
  float* s_sfac = reinterpret_cast<float*>(smem + SmemLayout::sfac);
  // series with gaps: substitute the centring constant for missing values (so the moments stay exact), record
  // where they were, and let the epilogue queue a SolveRec for solve_rows_kernel instead of a second pass
#ifdef MMF_TC_NO_COLLECT
  const bool collect = false;
#else
  const bool collect = a.recs != nullptr && d.t_fit <= 65535;      // ragged: d.t_fit is the longest calendar's
#endif
  const uint32_t s_bars = sbase + SmemLayout::bars;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  auto bar_full = [&](int s) { return s_bars + 8u * s; };
  auto bar_empty = [&](int s) { return s_bars + 8u * (STAGES + s); };
  auto bar_accfull = [&](int b) { return s_bars + 8u * (2 * STAGES + b); };
  auto bar_accempty = [&](int b) { return s_bars + 8u * (2 * STAGES + 2 + b); };
  auto bar_cc = [&](int b) { return s_bars + 8u * (2 * STAGES + 4 + b); };
  auto bar_tfull = [&](int s) { return s_bars + 8u * (2 * STAGES + 6 + s); };
  auto bar_tempty = [&](int s) { return s_bars + 8u * (2 * STAGES + 6 + TILE_RING + s); };
  int* s_tiles = reinterpret_cast<int*>(smem + SmemLayout::tiles);
  // the tile of the CTA's lt-th turn, as the producer claimed it (-1: no more); every consumer and epilogue warp
  // takes every entry once
  auto take_tile = [&](int lt) -> int {
    const int sl = lt % TILE_RING;
    mbar_wait(bar_tfull(sl), (lt / TILE_RING) & 1);
    const int t = *reinterpret_cast<volatile int*>(s_tiles + sl);
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_tempty(sl));
    return t;
  };

  // ---- one-time setup
  if (blockIdx.x == 0 && threadIdx.x == 0 && a.zero_next != nullptr) {
#pragma unroll
    for (int i = 0; i < CTR_WORDS; ++i) a.zero_next[i] = 0u;
  }
  if (warp == WARP_PROD) {
    if (lane == 0) {
      for (int s = 0; s < STAGES; ++s) {
        mbar_init(bar_full(s), 1);        // producer's expect_tx arrive (+ TMA bytes)
        mbar_init(bar_empty(s), 4);       // 4 warps of the consuming warpgroup, after their MMAs have retired
      }
      for (int b = 0; b < 2; ++b) {
        // partial moments + gap counts of a tile: every consumer THREAD arrives after writing its entries (release),
        // the epilogue's wait acquires them (the writer of each entry synchronises with its reader directly)
        mbar_init(bar_accfull(b), NGROUPS * 128);
        mbar_init(bar_accempty(b), 4);    // 4 epilogue warps have read the slot
        // centring constants of the tile in slot b: every thread of the group that consumes the tile's chunk 0 arrives
        // after writing its row's constant
        mbar_init(bar_cc(b), 128);
      }
      for (int sl = 0; sl < TILE_RING; ++sl) {
        mbar_init(bar_tfull(sl), 1);                       // the producer published the entry
        mbar_init(bar_tempty(sl), NGROUPS * 4 + 4);        // every consumer and epilogue warp has taken it
      }
      fence_mbar_init();
      prefetch_tensormap(tl.tmap_y);
      prefetch_tensormap(tl.tmap_at);
    }
  } else if (warp >= WARP_EPI0) {
    // prediction rows of the whitened design -> shared (broadcast-read in the epilogue); ragged launches reload
    // them whenever the epilogue reaches a tile of another calendar
    if (!a.skip_pred && !MULTI)
      for (int i = threadIdx.x - WARP_EPI0 * 32; i < a.n_pred * P; i += 128)
        s_apred[i] = __ldg(d.apred + (size_t)a.pred_start * P + i);
    if (SE && !a.skip_pred)
      for (int i = threadIdx.x - WARP_EPI0 * 32; i < a.n_pred; i += 128) s_sfac[i] = __ldg(se.sfac + a.pred_start + i);
  }
  __syncthreads();
  // This CTA is resident: a dependent kernel launched behind this one with programmatic stream serialisation may start
  // once EVERY CTA has said so -- the early-exit fix-up kernels hide their launch latency under this kernel's tail.
  if (threadIdx.x == 0) pdl_launch_dependents();

  if (warp == WARP_PROD) {
    // =========================== TMA producer ===========================
    // whole warp converged, one elected lane issues (keeps the tensor-map / barrier operands uniform)
    int stage = 0;
    uint32_t phase = 0;
    int last_cal = -1;
    // Tiles are claimed, not assigned by a stride: the first is blockIdx.x, every later one the next value of the call's
    // claim counter (counted from gridDim.x), so an SM that streams faster takes more tiles and the launch does not wait
    // for the slowest one.  The claim for the next tile is issued before this one streams, so its latency hides.
    uint32_t* claim_ctr = pending_count + CTR_TILE_CLAIM;
    int tile = blockIdx.x;
    for (int lt = 0;; ++lt) {
      const int sl = lt % TILE_RING;
      mbar_wait(bar_tempty(sl), ((lt / TILE_RING) & 1) ^ 1u);
      const bool more = tile < n_tiles;
      uint32_t claim = 0;
      if (lane == 0) {
        if (more) claim = atomicAdd(claim_ctr, 1u);
        s_tiles[sl] = more ? tile : -1;
        mbar_arrive(bar_tfull(sl));
      }
      __syncwarp();
      if (!more) break;
      const TileRec tr = tile_rec(tile);
      // ragged: the y buffer seen through the calendar's own tensor map (clipped at ITS t_fit: later columns, which
      // hold the held-out values or another calendar's padding, arrive as zeros) and the calendar's block of the
      // stacked design
      const void* tmy = MULTI ? static_cast<const void*>(mv.tmaps_y + (size_t)tr.cal * 128) : static_cast<const void*>(tl.tmap_y);
      if (MULTI && tr.cal != last_cal) { fence_tensormap_acquire(tmy); last_cal = tr.cal; }
      const int at_row = MULTI ? tr.cal * 2 * P : 0;
      for (int ch = 0; ch < tr.n_chunks; ++ch) {
        mbar_wait(bar_empty(stage), phase ^ 1u);
        tma_load_2d_x2_elect(bar_full(stage), Y_STAGE_BYTES + AT_STAGE_BYTES,
                             // series: evict-normal, not evict-first.  A row's 128 B of one chunk straddle two L2
                             // lines unless the pitch is 128-B aligned, and the next chunk's box reads the second one
                             // again: under evict-first it is often gone by then (H100 SXM, 700 W: the step is 1.2 %
                             // faster with evict-normal)
                             s_y + stage * Y_STAGE_BYTES, tmy, ch * KC, tr.row0, L2_EVICT_NORMAL,
                             s_at + stage * AT_STAGE_BYTES, tl.tmap_at, ch * KC, at_row,
                             MULTI ? L2_EVICT_NORMAL : L2_EVICT_LAST);   // one design stays in L2; a thousand do not
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      tile = static_cast<int>(gridDim.x + __shfl_sync(0xffffffffu, claim, 0));
    }
  } else if (warp < NGROUPS * 4) {
    // =========================== consumer warpgroups (warps 0-3, 4-7) ===========================
    // Chunk k of the CTA's stream (counted over all its tiles) sits in stage k % STAGES and belongs to group k & 1.
    const int grp = warp >> 2;
    const int r = threadIdx.x & 127;                    // gap scan: row r of the tile
    const uint32_t row_off = static_cast<uint32_t>(r) * 128u;
    const uint32_t sw = static_cast<uint32_t>(r & 7);
    const int g8 = lane >> 2, t4 = lane & 3;            // MMA fragments: rows 64h + 16*(warp & 3) + g8 (+8), cols t4 (+4)
    const int frow0 = 16 * (warp & 3) + g8;
    uint32_t gc = 0;                                    // first chunk of the current tile in the CTA's stream
    for (int lt = 0;; ++lt) {
      const int tile = take_tile(lt);
      if (tile < 0) break;
      const TileRec tr = tile_rec(tile);
      // cannot centre on a missing first value: general path (flagged by the group that forms the constants; the
      // epilogue ORs both groups' flags)
      bool bad = false;
      float cf[2][2];                                   // centring constants of this thread's four fragment rows
      float acc[2][P];                                  // m64n32 accumulators of the two 64-row halves
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < P; ++i) acc[h][i] = 0.f;
      const bool scan = collect && (!MULTI || r < tr.nrows);   // short tiles: rows beyond belong to ANOTHER tile
      // segment = parity of the chunk inside the TILE (all of a group's chunks of one tile share it), not the group:
      // with an odd chunk count the groups swap roles from tile to tile, and the order in which the solve applies
      // the gaps -- hence the forecast's last bits -- must not depend on where in a launch the series sits
      const int seg = (grp ^ (int)gc) & 1;
      int nm = 0;                                       // missing values this thread saw in the tile
      unsigned long long packq = 0ull;                  // the last (nm & 3) gap positions, newest in the top lanes
      // the tile's slot of partial moments for the epilogue; a long tile keeps the folded sums of its restarted
      // accumulators there (each thread its own entries), which costs no registers
      const int ab = lt & 1;
      float* __restrict__ sacc = s_acc + (ab * NGROUPS + grp) * TILE_M * P;
      auto sacc_at = [&](int h, int j, int i) {
        return reinterpret_cast<float2*>(sacc + (64 * h + frow0 + 8 * j) * P + 8 * i + 2 * t4);
      };
      bool folded = false;
      int since_fold = 0;
      // SE: S of the four fragment rows over this thread's columns.  A chunk's 8 squares are summed in fp32 and the
      // chunk sums in f64, so the rounding does not grow with the fit window (the moments restart for the same reason)
      double ssq[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
      for (int ch = seg; ch < tr.n_chunks; ch += NGROUPS) {
        const uint32_t k = gc + static_cast<uint32_t>(ch);
        const int stage = static_cast<int>(k % STAGES);
        mbar_wait(bar_full(stage), (k / STAGES) & 1u);
        const uint32_t sy = s_y + stage * Y_STAGE_BYTES;
        if (ch == seg) {                                // this group's first chunk of the tile
          if (seg == 0) {
            // chunk 0: row r's centring constant from its staged head, into the tile's slot of constants.  The slot's
            // previous tile (lt - 2) must be done with it: its epilogue has read it once it released the partials slot
            mbar_wait(bar_accempty(ab), ((lt >> 1) & 1) ^ 1u);
            float c = 0.f;
            if (d.has_constant && r < tr.nrows) {
              const uint32_t rowp = sy + row_off;
              // (a ragged calendar's t_fit is at least 33, so none of its first 8 positions is clipped)
              c = centring_constant(lds128(rowp + (sw << 4)), lds128(rowp + ((1u ^ sw) << 4)), MULTI ? KC : d.t_fit);
            }
            bad = collect && !is_finite_bits(c);
            s_cc[ab * TILE_M + r] = bad ? 0.f : c;
            mbar_arrive(bar_cc(ab));
          }
          mbar_wait(bar_cc(ab), (lt >> 1) & 1);
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 2; ++j) cf[h][j] = s_cc[ab * TILE_M + 64 * h + frow0 + 8 * j];
        }
        if (scan) {
          const uint32_t rowp = sy + row_off;
          float4 v[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) v[q] = lds128(rowp + ((static_cast<uint32_t>(q) ^ sw) << 4));
          float chk = 0.f;                              // 0 * x is NaN exactly when x is NaN or Inf
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            chk = fmaf(v[q].x, 0.f, chk); chk = fmaf(v[q].y, 0.f, chk);
            chk = fmaf(v[q].z, 0.f, chk); chk = fmaf(v[q].w, 0.f, chk);
          }
          if (!(chk == 0.f)) {                          // rare: this row has a gap inside this chunk
            // a bit mask of the gap positions, then a short loop over the set bits; positions are shifted into a
            // 64-bit register and leave four at a time (one 8-B store, the unit the solve kernel reads)
            unsigned gaps = 0u;
#pragma unroll
            for (int q = 0; q < 8; ++q)
              gaps |= (is_finite_bits(v[q].x) ? 0u : 1u << (4 * q)) | (is_finite_bits(v[q].y) ? 0u : 2u << (4 * q)) |
                      (is_finite_bits(v[q].z) ? 0u : 4u << (4 * q)) | (is_finite_bits(v[q].w) ? 0u : 8u << (4 * q));
            uint16_t* __restrict__ mt = a.recs[(int64_t)tr.row0 + r].miss_t + seg * SOLVE_SEG;
            const int tbase = ch * KC;
            while (gaps) {
              const int pos = __ffs(gaps) - 1;
              gaps &= gaps - 1u;
              packq = (packq >> 16) | (static_cast<unsigned long long>(tbase + pos) << 48);
              ++nm;
              if ((nm & 3) == 0 && nm <= SOLVE_SEG) *reinterpret_cast<unsigned long long*>(mt + nm - 4) = packq;
              // BT: the first position the segment cannot hold, so that the epilogue can tell for every origin whether
              // more than SOLVE_SEG of its gaps fall into the segment (kept in the record's `ss` word, unused here)
              if constexpr (BT) if (nm == SOLVE_SEG + 1)
                reinterpret_cast<uint16_t*>(&a.recs[(int64_t)tr.row0 + r].ss)[seg] = static_cast<uint16_t>(tbase + pos);
            }
          }
        }
        // A fragments of both 64-row halves: centre (missing values take the centring constant, so they add
        // (c - c) = 0 to every moment), split into tf32 hi + fp32 residual lo
        uint32_t ahi[2][KC / 8][4], alo[2][KC / 8][4];
        const int lim = d.t_fit - ch * KC;              // SE: columns from t_fit on arrive as zeros (TMA clip), not c
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const uint32_t rowp = sy + static_cast<uint32_t>(64 * h + frow0 + 8 * j) * 128u + t4 * 4;   // row & 7 == g8
            float part = 0.f;
#pragma unroll
            for (int kk = 0; kk < KC / 8; ++kk)
#pragma unroll
              for (int hf = 0; hf < 2; ++hf) {
                float x = lds32(rowp + ((static_cast<uint32_t>(2 * kk + hf) ^ static_cast<uint32_t>(g8)) << 4));
                if (collect) x = is_finite_bits(x) ? x : cf[h][j];
                const float rr = x - cf[h][j];
                const uint32_t hb = __float_as_uint(rr) & 0xFFFFE000u;
                ahi[h][kk][j + 2 * hf] = hb;
                alo[h][kk][j + 2 * hf] = __float_as_uint(rr - __uint_as_float(hb));
                if (SE) {
                  const float rs = 4 * (2 * kk + hf) + t4 < lim ? rr : 0.f;
                  part = fmaf(rs, rs, part);
                }
              }
            if (SE) ssq[h][j] += static_cast<double>(part);
          }
        const uint64_t bdesc0 = gmma_desc_k_sw128(s_at + stage * AT_STAGE_BYTES);
        uint32_t bt_in = 0;                             // BT: earlier origins strictly inside this chunk
        if constexpr (BT) {
          // origins in [start - 32, start]: this group's previous chunk ended at or below them and the other group's
          // chunk lies in between, so the accumulator holds exactly this group's share of their moments (origins
          // inside a chunk of this group are split below, origins beyond its last chunk written at the tile's end)
          const int s0 = ch * KC;
          uint32_t pre = 0;
#pragma unroll
          for (int k = 0; k < MMF_BT_MAX_ORIGINS - 1; ++k) {
            pre |= (bt.t_orig[k] >= s0 - KC && bt.t_orig[k] <= s0 ? 1u : 0u) << k;
            bt_in |= (bt.t_orig[k] > s0 && bt.t_orig[k] < s0 + KC ? 1u : 0u) << k;
          }
          while (pre) {
            const int k = __ffs(pre) - 1;
            pre &= pre - 1u;
            bt_write_moments(bt, k, grp, a.n, tr, frow0, t4, acc, folded, sacc);
          }
        }
        // (if constexpr, and the plain chunk below written out twice: the other instantiations must compile to exactly
        // the code they had before the backtest existed)
        if constexpr (BT) {
        if (bt_in != 0u) {
          // the chunk in column ranges [lo, hi) split at its origins: the A fragments of the other columns are zero,
          // the B tiles are the stage's as always; after each range that ends at an origin the moments are written
          int lo = 0;
          uint32_t m = bt_in;
          for (;;) {
            const int k = m ? __ffs(m) - 1 : -1;
            const int hi = k >= 0 ? __ldg(&bt.cals[k].t_fit) - ch * KC : KC;
            wgmma_fence();
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int kk = 0; kk < KC / 8; ++kk) {
                const uint64_t bdesc = bdesc0 + static_cast<uint64_t>(kk * 2);
                uint32_t fh[4], fl[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {                 // element e: column 8 kk + 4 (e >> 1) + t4
                  const int col = 8 * kk + 4 * (e >> 1) + t4;
                  const bool in = col >= lo && col < hi;
                  fh[e] = in ? ahi[h][kk][e] : 0u;
                  fl[e] = in ? alo[h][kk][e] : 0u;
                }
                wgmma_m64n32k8_tf32_rs(acc[h], fh, bdesc);
#ifndef MMF_TC_NO_LO_TERM
                wgmma_m64n32k8_tf32_rs(acc[h], fl, bdesc);
#endif
              }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(acc[0]);
            wgmma_fence_regs(acc[1]);
            if (k < 0) break;
            bt_write_moments(bt, k, grp, a.n, tr, frow0, t4, acc, folded, sacc);
            m &= m - 1u;
            lo = hi;
          }
        } else {
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int kk = 0; kk < KC / 8; ++kk) {
            const uint64_t bdesc = bdesc0 + static_cast<uint64_t>(kk * 2);       // +32 B (16-B units)
            wgmma_m64n32k8_tf32_rs(acc[h], ahi[h][kk], bdesc);
#ifndef MMF_TC_NO_LO_TERM      // negative-control build (tests): without the lo term the path is tf32-grade and must FAIL parity
            wgmma_m64n32k8_tf32_rs(acc[h], alo[h][kk], bdesc);
#endif
          }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc[0]);
        wgmma_fence_regs(acc[1]);
        }
        } else {
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int kk = 0; kk < KC / 8; ++kk) {
            const uint64_t bdesc = bdesc0 + static_cast<uint64_t>(kk * 2);       // +32 B (16-B units)
            wgmma_m64n32k8_tf32_rs(acc[h], ahi[h][kk], bdesc);
#ifndef MMF_TC_NO_LO_TERM      // negative-control build (tests): without the lo term the path is tf32-grade and must FAIL parity
            wgmma_m64n32k8_tf32_rs(acc[h], alo[h][kk], bdesc);
#endif
          }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc[0]);
        wgmma_fence_regs(acc[1]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty(stage));   // this warp's MMAs and smem reads of the stage are done
        if (++since_fold == FOLD_CHUNKS && ch + NGROUPS < tr.n_chunks) {   // more chunks follow: fold and restart
          if (!folded) mbar_wait(bar_accempty(ab), ((lt >> 1) & 1) ^ 1u);  // epilogue of tile lt-2 has drained the slot
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const int q = 4 * i + 2 * j;            // acc[h][q + 8] is the lo column of acc[h][q]
                float2 f = make_float2(acc[h][q] + acc[h][q + P / 2], acc[h][q + 1] + acc[h][q + 1 + P / 2]);
                if (folded) { const float2 o = *sacc_at(h, j, i); f.x = o.x + f.x; f.y = o.y + f.y; }
                *sacc_at(h, j, i) = f;
              }
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < P; ++i) acc[h][i] = 0.f;
          folded = true;
          since_fold = 0;
        }
      }
      if (scan && (nm & 3) != 0 && nm < SOLVE_SEG) {    // flush the partial group (right-aligned: oldest first)
        uint16_t* __restrict__ mt = a.recs[(int64_t)tr.row0 + r].miss_t + seg * SOLVE_SEG;
        *reinterpret_cast<unsigned long long*>(mt + (nm & ~3)) = packq >> (16 * (4 - (nm & 3)));
      }
      if constexpr (BT) {                                         // earlier origins at or beyond the end of this group's last chunk
        const int s_end = ((tr.n_chunks - 1 - seg) / NGROUPS * NGROUPS + seg + 1) * KC;
        uint32_t rest = 0;
#pragma unroll
        for (int k = 0; k < MMF_BT_MAX_ORIGINS - 1; ++k) rest |= (bt.t_orig[k] != INT32_MAX && bt.t_orig[k] >= s_end ? 1u : 0u) << k;
        while (rest) {
          const int k = __ffs(rest) - 1;
          rest &= rest - 1u;
          bt_write_moments(bt, k, grp, a.n, tr, frow0, t4, acc, folded, sacc);
        }
      }
      // hand the tile's partial moments (hi and lo columns folded: b = D[:, p] + D[:, P + p]) to the epilogue
      if (!folded) mbar_wait(bar_accempty(ab), ((lt >> 1) & 1) ^ 1u);  // epilogue of tile lt-2 has drained this slot
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int q = 4 * i + 2 * j;                // acc[h][q + 8] is the lo column of acc[h][q]
            float2 v = make_float2(acc[h][q] + acc[h][q + P / 2], acc[h][q + 1] + acc[h][q + 1 + P / 2]);
            if (folded) { const float2 o = *sacc_at(h, j, i); v.x = o.x + v.x; v.y = o.y + v.y; }
            *sacc_at(h, j, i) = v;
          }
      if (SE) {                                         // the quad's four column sets -> one S per fragment row
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            double v = ssq[h][j];
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            if (t4 == 0) s_ss[(ab * NGROUPS + grp) * TILE_M + 64 * h + frow0 + 8 * j] = v;
          }
      }
      const int cnt = nm > 0x7ffe ? 0x7ffe : nm;
      s_nm[(ab * NGROUPS + seg) * TILE_M + r] = static_cast<uint16_t>(cnt | (bad ? 0x8000 : 0));
      mbar_arrive(bar_accfull(ab));
      gc += static_cast<uint32_t>(tr.n_chunks);
    }
  } else {
    // =========================== epilogue (warps 8-11) ===========================
    const int r = threadIdx.x & 127;
    bool vec_out = (a.n_pred % 4 == 0) && (a.ld_out % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.out) & 15u) == 0);
    for (int i = 0; i + 1 < a.n_out; ++i) vec_out = vec_out && ((reinterpret_cast<uintptr_t>(a.out_more[i]) & 15u) == 0);
    // Staged epilogue: the tile's forecasts are one contiguous block of the table (rows are dense), so they are
    // assembled in shared memory: the local table leaves as coalesced warp stores, each peer's copy as ONE bulk (TMA)
    // store -- full-size NVLink packets instead of 16-B stores scattered at a 112-B stride.
#ifdef MMF_TC_NO_BULK
    const bool bulk = false;
#else
    const bool bulk = !a.skip_pred && vec_out && a.out_multimem != 1 && a.ld_out == a.n_pred && a.n_pred <= BULK_MAX_PRED;
#endif
    const uint32_t s_ostage_u32 = smem_u32(s_ostage);
    const uint64_t l2_policy = l2_evict_first_policy();
    // SE: 16-B stores of the se rows when the table allows them (the same test as vec_out)
    const bool se_vec = SE && (a.n_pred % 4 == 0) && (se.ld_se % 4 == 0) &&
                        ((reinterpret_cast<uintptr_t>(se.out_se) & 15u) == 0);
    int lt = 0;
    int cur_cal = MULTI ? -1 : 0;
    uint32_t kept_mask = d.kept_mask;
    int t_fit_c = d.t_fit;
    for (;; ++lt) {
      const int tile = take_tile(lt);
      if (tile < 0) break;
      const int ab = lt & 1;
      const TileRec tr = tile_rec(tile);
      const int64_t row = (int64_t)tr.row0 + r;
      const bool live = r < tr.nrows;
      if (MULTI && tr.cal != cur_cal) {                 // uniform over the four epilogue warps: they walk the same tiles
        const int4* cp = reinterpret_cast<const int4*>(mv.cals + tr.cal);
        const int4 m0 = __ldg(cp), m1 = __ldg(cp + 1);  // {t_fit, n_chunks, n_rows, kept_mask}, {row_off, pred_start, ..}
        t_fit_c = m0.x;
        kept_mask = static_cast<uint32_t>(m0.w);
        if (!a.skip_pred) {
          named_bar_sync(2, 128);                       // the previous tile's forecasts no longer read s_apred
          const float* __restrict__ src = d.apred + (size_t)(m1.x + m1.y) * P;
          for (int i = threadIdx.x - WARP_EPI0 * 32; i < a.n_pred * P; i += 128) s_apred[i] = __ldg(src + i);
          named_bar_sync(2, 128);
        }
        cur_cal = tr.cal;
      }
      mbar_wait(bar_accfull(ab), (lt >> 1) & 1);
      float c = s_cc[ab * TILE_M + r];                  // the constant the consumers centred row r on
      float g[P];
      {
        const float4* p0 = reinterpret_cast<const float4*>(s_acc + (ab * NGROUPS + 0) * TILE_M * P + r * P);
        const float4* p1 = reinterpret_cast<const float4*>(s_acc + (ab * NGROUPS + 1) * TILE_M * P + r * P);
#pragma unroll
        for (int q = 0; q < P / 4; ++q) {
          const float4 u = p0[q], w = p1[q];
          g[4 * q] = u.x + w.x; g[4 * q + 1] = u.y + w.y; g[4 * q + 2] = u.z + w.z; g[4 * q + 3] = u.w + w.w;
        }
      }
      // gaps the consumer warpgroups saw in this tile, by chunk parity
      const unsigned f0 = s_nm[(ab * NGROUPS + 0) * TILE_M + r], f1 = s_nm[(ab * NGROUPS + 1) * TILE_M + r];
      const double ss = SE ? s_ss[(ab * NGROUPS + 0) * TILE_M + r] + s_ss[(ab * NGROUPS + 1) * TILE_M + r] : 0.0;
      if constexpr (BT) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_accempty(ab));   // g, f0 and f1 are in registers
        // every origin of the row by the plain epilogue's rules, with origin k's own gap counts and t_k; the last
        // origin (t_K) is the tile's hand-off itself, the earlier ones the two groups' moments in bt.mom
        for (int k = 0; k < bt.n_origin; ++k) {
          const bool last = k == bt.n_origin - 1;
          const int4 m0 = __ldg(reinterpret_cast<const int4*>(bt.cals + k));   // {t_k, n_chunks, n_rows, kept_mask}
          const int tk = m0.x;
          float gk[P];
          if (last || !live) {
#pragma unroll
            for (int p = 0; p < P; ++p) gk[p] = g[p];
          } else {
            const float4* p0 = reinterpret_cast<const float4*>(bt.mom + (((int64_t)k * NGROUPS + 0) * a.n + row) * P);
            const float4* p1 = reinterpret_cast<const float4*>(bt.mom + (((int64_t)k * NGROUPS + 1) * a.n + row) * P);
#pragma unroll
            for (int q = 0; q < P / 4; ++q) {
              const float4 u = p0[q], w = p1[q];
              gk[4 * q] = u.x + w.x; gk[4 * q + 1] = u.y + w.y; gk[4 * q + 2] = u.z + w.z; gk[4 * q + 3] = u.w + w.w;
            }
          }
          // gaps below t_k per segment: a prefix of the positions recorded in the last origin's record (ascending per
          // segment); a segment that overflowed holds its first SOLVE_SEG positions and, in `ss`, the next one
          const SolveRec* __restrict__ src = collect ? a.recs + row : nullptr;
          int n0 = f0 & 0x7fff, n1 = f1 & 0x7fff;
          bool over = false;
          if (collect && !last && live && (n0 | n1) != 0) {
#pragma unroll
            for (int sg = 0; sg < 2; ++sg) {
              const int tot = sg ? n1 : n0;
              const uint16_t* mt = src->miss_t + sg * SOLVE_SEG;
              const int have = tot < SOLVE_SEG ? tot : SOLVE_SEG;
              int cnt = 0;
              while (cnt < have && mt[cnt] < tk) ++cnt;
              if (cnt == SOLVE_SEG && tot > SOLVE_SEG && reinterpret_cast<const uint16_t*>(&src->ss)[sg] < tk) over = true;
              if (sg) n1 = cnt; else n0 = cnt;
            }
          }
          bool general = false;
          if (collect)
            general = ((f0 | f1) & 0x8000u) != 0u || over || n0 > SOLVE_SEG || n1 > SOLVE_SEG || 2 * (n0 + n1) > tk;
          bool finite = true;
#pragma unroll
          for (int p = 0; p < P; ++p) {
            finite = finite && is_finite_bits(gk[p]);
            if (!((kept_mask >> p) & 1u)) gk[p] = 0.f;
          }
          const bool pend = live && (!finite || general);
          const bool defer = live && !pend && (n0 + n1) > 0;
          const unsigned pm = __ballot_sync(0xffffffffu, pend);
          if (lane == 0 && pm != 0u) {
            atomicAdd(pending_count, __popc(pm));
            atomicAdd(bt.pending + k, __popc(pm));
          }
          const unsigned dm = __ballot_sync(0xffffffffu, defer);
          if (dm != 0u) {
            unsigned base = 0;
            if (lane == 0) base = atomicAdd(bt.rec_count + k, __popc(dm));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (defer) {
              SolveRec& rec = bt.recs[(int64_t)k * a.n + row];
              float bk[P];
              if (last) {
#pragma unroll
                for (int p = 0; p < P; ++p) bk[p] = gk[p];
              } else {                                  // into origin k's own basis: b^(k) = T_k^T b_k
                const float* __restrict__ tm = bt.tmat + (size_t)k * P * P;
#pragma unroll
                for (int p = 0; p < P; ++p) {
                  float s = 0.f;
#pragma unroll
                  for (int q = 0; q < P; ++q) s = fmaf(__ldg(tm + q * P + p), gk[q], s);
                  bk[p] = s;
                }
                for (int sg = 0; sg < 2; ++sg) {
                  const int cnt = sg ? n1 : n0;
                  for (int e = 0; e < cnt; ++e) rec.miss_t[sg * SOLVE_SEG + e] = src->miss_t[sg * SOLVE_SEG + e];
                }
              }
              float4* bp = reinterpret_cast<float4*>(rec.b);
              bp[0] = make_float4(bk[0], bk[1], bk[2], bk[3]);    bp[1] = make_float4(bk[4], bk[5], bk[6], bk[7]);
              bp[2] = make_float4(bk[8], bk[9], bk[10], bk[11]);  bp[3] = make_float4(bk[12], bk[13], bk[14], bk[15]);
              rec.c = c;
              rec.nm[0] = static_cast<uint16_t>(n0);
              rec.nm[1] = static_cast<uint16_t>(n1);
              rec.cal = k;
              const unsigned slot = base + __popc(dm & ((1u << lane) - 1u));
              if (slot < a.rec_cap) bt.rec_rows[(int64_t)k * a.n + slot] = row;
            }
          }
          if (live && !pend && !defer) {
            const float* __restrict__ pk = bt.pred + (size_t)k * a.n_pred * P;
            const int64_t off = ((int64_t)k * bt.out_kstride + row) * a.ld_out;
            if (vec_out) {
              for (int j = 0; j < a.n_pred; j += 4) {
                float o[4];
#pragma unroll
                for (int w = 0; w < 4; ++w) o[w] = dot16(pk + (j + w) * P, gk, c);
                store_out4(a, off + j, make_float4(o[0], o[1], o[2], o[3]));
              }
            } else {
              for (int j = 0; j < a.n_pred; ++j) store_out1(a, off + j, dot16(pk + j * P, gk, c));
            }
          }
          if (live) a.status[(int64_t)k * bt.st_kstride + row] = pend ? MMF_STATUS_PENDING : (defer ? MMF_STATUS_DEFERRED : MMF_STATUS_OK);
        }
        continue;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_accempty(ab));     // the consumers may overwrite this slot now
      int nm0 = 0, nm1 = 0;
      bool general = false;
      if (collect) {
        nm0 = f0 & 0x7fff; nm1 = f1 & 0x7fff;
        // mostly-missing rows: the downdate I - sum a a^T cancels catastrophically; fit_warp builds their Gram
        // directly over the observed rows (same rule as fit_warp.cu)
        general = ((f0 | f1) & 0x8000u) != 0u || nm0 > SOLVE_SEG || nm1 > SOLVE_SEG || 2 * (nm0 + nm1) > t_fit_c;
        if (general) c = 0.f;
      }
      bool finite = true;
#pragma unroll
      for (int p = 0; p < P; ++p) {
        finite = finite && is_finite_bits(g[p]);
        if (!((kept_mask >> p) & 1u)) g[p] = 0.f;
      }
      const bool pend = live && (!finite || general);            // -> general warp pass
      const bool defer = live && !pend && (nm0 + nm1) > 0;       // -> thread-per-series solve of the queued record
      const unsigned pm = __ballot_sync(0xffffffffu, pend);
      if (lane == 0 && pm != 0u) {
        atomicAdd(pending_count, __popc(pm));
        if (MULTI) atomicAdd(mv.pending_by_cal + tr.cal, __popc(pm));      // the general pass runs per calendar
      }
      const unsigned dm = __ballot_sync(0xffffffffu, defer);
      if (dm != 0u) {
        unsigned base = 0;
        if (lane == 0) base = atomicAdd(a.rec_count, __popc(dm));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (defer) {
          SolveRec& rec = a.recs[row];
          float4* bp = reinterpret_cast<float4*>(rec.b);
          bp[0] = make_float4(g[0], g[1], g[2], g[3]);    bp[1] = make_float4(g[4], g[5], g[6], g[7]);
          bp[2] = make_float4(g[8], g[9], g[10], g[11]);  bp[3] = make_float4(g[12], g[13], g[14], g[15]);
          rec.c = c;
          if (SE) rec.ss = static_cast<float>(ss);
          rec.nm[0] = static_cast<uint16_t>(nm0);
          rec.nm[1] = static_cast<uint16_t>(nm1);
          rec.cal = tr.cal;
          const unsigned slot = base + __popc(dm & ((1u << lane) - 1u));
          if (slot < a.rec_cap) a.rec_rows[slot] = row;
        }
      }
      if (bulk) {
        // staging tile lt % OBUF: the bulk stores that read it last (tile lt - OBUF) must have drained it
        const int ob = OBUF > 1 ? (lt % OBUF) : 0;
        if (warp == WARP_EPI0) { if (OBUF > 1) bulk_wait_read1_elect(); else bulk_wait_read_elect(); }
        named_bar_sync(1, 128);
        float* __restrict__ srow = s_ostage + ob * (TILE_M * BULK_MAX_PRED) + r * a.n_pred;
        for (int k = 0; k < a.n_pred; k += 4) {          // PENDING rows stage garbage; the fix-up pass rewrites them
          float o[4];
#pragma unroll
          for (int w = 0; w < 4; ++w) o[w] = dot16(s_apred + (k + w) * P, g, c);
          *reinterpret_cast<float4*>(srow + k) = make_float4(o[0], o[1], o[2], o[3]);
        }
        fence_proxy_async_smem();
        named_bar_sync(1, 128);
        const uint32_t bytes = static_cast<uint32_t>(tr.nrows) * a.n_pred * 4u;
        const int64_t off = (int64_t)tr.row0 * a.n_pred;
        const uint32_t src = s_ostage_u32 + static_cast<uint32_t>(ob) * (TILE_M * BULK_MAX_PRED * 4);
        // the local table: coalesced 16-B stores of the staged tile by all four warps (512 contiguous bytes per warp
        // instruction), evict-first -- the table is not read again by this kernel, and its dirty lines leave L2 early
        // instead of piling up amid the series stream.  On an H100 SXM at 700 W this is 0.6 % faster than one
        // evict-first bulk store per tile, which queues on the TMA unit that also feeds the load ring
        for (uint32_t i = r; i < bytes / 16u; i += 128u)
          stg128_hint(reinterpret_cast<float4*>(a.out + off) + i, lds128(src + 16u * i), l2_policy);
        if (warp == WARP_EPI0) {
          // peers: every tile starts at another peer, so at any moment this GPU's store queues target all
          // peers evenly instead of all hammering the first one in the list (NVLink ingress hot spot)
          const int n_peer = a.n_out - 1;
          int j = n_peer > 1 ? tile % n_peer : 0;
          for (int i = 0; i < n_peer; ++i) {
            bulk_store_elect(reinterpret_cast<uint64_t>(a.out_more[j] + off), src, bytes);
            if (++j == n_peer) j = 0;
          }
          bulk_commit_elect();
        }
      } else if (live && !pend && !defer && !a.skip_pred) {
        const int64_t off = row * a.ld_out;
        if (vec_out) {
          for (int k = 0; k < a.n_pred; k += 4) {
            float o[4];
#pragma unroll
            for (int w = 0; w < 4; ++w) o[w] = dot16(s_apred + (k + w) * P, g, c);
            store_out4(a, off + k, make_float4(o[0], o[1], o[2], o[3]));
          }
        } else {
          for (int k = 0; k < a.n_pred; ++k) store_out1(a, off + k, dot16(s_apred + k * P, g, c));
        }
      }
      if (live) {
        if (!pend && !defer) {
          if (a.out_gamma != nullptr) {
            float4* gp = reinterpret_cast<float4*>(a.out_gamma + row * P);
            gp[0] = make_float4(g[0], g[1], g[2], g[3]);    gp[1] = make_float4(g[4], g[5], g[6], g[7]);
            gp[2] = make_float4(g[8], g[9], g[10], g[11]);  gp[3] = make_float4(g[12], g[13], g[14], g[15]);
            a.out_c[row] = c;
          }
          if (a.out_beta != nullptr) {
            float* __restrict__ br = a.out_beta + row * P;
            for (int p = 0; p < P; ++p) {
              float s = (p == 0 && d.has_constant) ? c : 0.f;
#pragma unroll
              for (int q = 0; q < P; ++q) s = fmaf(__ldg(d.w + p * P + q), g[q], s);
              br[p] = s;
            }
          }
          if (SE) {
            // gap-free: G_i = I, so b'gamma = |gamma|^2, every kept column is used and h_t = |a_t|^2
            double bg = 0.0;
#pragma unroll
            for (int p = 0; p < P; ++p) bg = fma(static_cast<double>(g[p]), static_cast<double>(g[p]), bg);
            const int dof = t_fit_c - __popc(kept_mask);
            const double rss = fmax(ss - bg, 0.0);
            const float sig = dof > 0 ? static_cast<float>(sqrt(rss / dof)) : __int_as_float(0x7fc00000);
            se.sigma[row] = sig;
            if (se.dof != nullptr) se.dof[row] = dof;
            if (se.out_se != nullptr && !a.skip_pred) {
              float* __restrict__ srow = se.out_se + row * se.ld_se;
              int k = 0;
              if (se_vec)
                for (; k < a.n_pred; k += 4)
                  __stcs(reinterpret_cast<float4*>(srow + k),
                         make_float4(sig * s_sfac[k], sig * s_sfac[k + 1], sig * s_sfac[k + 2], sig * s_sfac[k + 3]));
              for (; k < a.n_pred; ++k) __stcs(srow + k, sig * s_sfac[k]);
            }
          }
        }
        stg32_hint(a.status + row, pend ? MMF_STATUS_PENDING : (defer ? MMF_STATUS_DEFERRED : MMF_STATUS_OK), l2_policy);
      }
    }
    if (bulk && warp == WARP_EPI0) bulk_wait_all_elect();   // global writes complete before the kernel retires
  }
}

}  // namespace

bool fit_tc_supported(const DesignView& d, const FitArgs& a, const char** why) {
  const char* w = nullptr;
  if (!a.skip_pred && a.n_pred > MAX_PRED) w = "n_pred > 64 needs the fit + predict_tc_kernel pair";
  else if (a.n_pred < 1) w = "n_pred < 1";
  else if (a.ld_y % 4 != 0) w = "ld_y not a multiple of 4 floats (TMA needs 16-B row pitch)";
  else if ((reinterpret_cast<uintptr_t>(a.y) & 15u) != 0) w = "y not 16-B aligned";
  else if (d.t_fit < 1) w = "t_fit < 1";
  else if (a.n > (int64_t)0x7fffffff - TILE_M) w = "n too large for 32-bit TMA coordinates";
  if (why) *why = w;
  return w == nullptr;
}

template <int STAGES, int OBUF, bool MULTI, bool SE = false, bool BT = false>
static cudaError_t launch_variant(const DesignView& d, const FitArgs& a, const TcLaunch& tl, uint32_t* pending_count,
                                  int sm_count, cudaStream_t s, int n_tiles, int n_chunks, const MultiView& mv,
                                  const SeArgs& se = SeArgs{}, const BtArgs& bt = BtArgs{}) {
  const size_t smem = SmemLayoutT<STAGES, OBUF, SE>::total + 1024;
  cudaError_t e = cudaFuncSetAttribute(fit_tc_kernel<STAGES, OBUF, MULTI, SE, BT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const int grid = n_tiles < sm_count ? n_tiles : sm_count;
  fit_tc_kernel<STAGES, OBUF, MULTI, SE, BT><<<grid, THREADS, smem, s>>>(tl, d, a, pending_count, n_tiles, n_chunks, mv, se, bt);
  return cudaGetLastError();
}

cudaError_t launch_fit_tc(const DesignView& d, const FitArgs& a, const TcLaunch& tl, uint32_t* pending_count,
                          int sm_count, cudaStream_t s, int variant, const MultiView* multi) {
  if (a.n <= 0) return cudaSuccess;
  if (multi != nullptr)      // ragged: the tile table names rows and calendars; d.t_pad / KC is the LONGEST calendar's count
    return launch_variant<8, 1, true>(d, a, tl, pending_count, sm_count, s, multi->n_tiles, 2, *multi);
  const int n_tiles = (int)((a.n + TILE_M - 1) / TILE_M);
  const int n_chunks = d.t_pad / KC;
  const MultiView none{};
  // variant 2: <6 stages, 2 staging tiles> (tile k+1 staged while the peer stores of tile k still read theirs; the
  // second tile costs two stages of the 227 KB); any other value: eight stages, one staging tile
  return variant == 2 ? launch_variant<6, 2, false>(d, a, tl, pending_count, sm_count, s, n_tiles, n_chunks, none)
                      : launch_variant<8, 1, false>(d, a, tl, pending_count, sm_count, s, n_tiles, n_chunks, none);
}

cudaError_t launch_fit_tc_se(const DesignView& d, const FitArgs& a, const TcLaunch& tl, uint32_t* pending_count,
                             int sm_count, cudaStream_t s, const SeArgs& se) {
  if (a.n <= 0) return cudaSuccess;
  const int n_tiles = (int)((a.n + TILE_M - 1) / TILE_M);
  return launch_variant<8, 1, false, true>(d, a, tl, pending_count, sm_count, s, n_tiles, d.t_pad / KC, MultiView{}, se);
}

cudaError_t launch_fit_tc_bt(const DesignView& d, const FitArgs& a, const TcLaunch& tl, uint32_t* pending_count,
                             int sm_count, cudaStream_t s, const BtArgs& bt) {
  if (a.n <= 0) return cudaSuccess;
  const int n_tiles = (int)((a.n + TILE_M - 1) / TILE_M);
  return launch_variant<8, 1, false, false, true>(d, a, tl, pending_count, sm_count, s, n_tiles, d.t_pad / KC,
                                                  MultiView{}, SeArgs{}, bt);
}

}  // namespace mmf
