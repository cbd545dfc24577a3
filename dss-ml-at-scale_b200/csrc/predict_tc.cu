// predict_tc.cu -- fitted values + forecasts for every requested date: out[n, n_pred] = c + gamma A_pred^T.
//
// The reference's per-group UDF returns Demand_Fitted for EVERY date of the group (in-sample fits for the train
// dates + the forecast for the held-out dates, group_apply/02_Fine_Grained_Demand_Forecasting.py:484-494).  With
// T dates per series that is as many bytes out as the fit read in, and 16 FMAs per output element -- too much for
// the CUDA cores at HBM speed, so it is a second tensor-core GEMM, the mirror image of fit_tc.cu:
//   A operand  gamma tile [128 series x 16] (fp32 split hi/lo, m16n8k8 register fragments)
//   B operand  prediction rows of the whitened design, [128 t x 16] K-major tiles (hi and lo), TMA, 64-B swizzle
//   D          [64 series x 128 t] fp32 per warpgroup (registers):  hi*Bhi + hi*Blo + lo*Bhi  (fp32-grade)
//   epilogue   each warpgroup owns one 64-row half of every tile: D + c -> 128-B-swizzled shared tiles (double
//              buffered) -> TMA 2-D stores (clipped at n / n_pred)
// Bound: HBM writes, 4*n_pred bytes per series (DESIGN.md section 4).
#include "mmf_internal.cuh"
#include "sm90_ptx.cuh"

namespace mmf {
namespace {

using namespace sm90;

constexpr int TILE_M = 128;                   // series per tile
constexpr int WG_M = 64;                      // series per warpgroup (one wgmma M)
constexpr int TN = 128;                       // prediction rows per chunk == D columns
constexpr int SB = 3;                         // B-operand stages
constexpr int B_TILE_BYTES = TN * P * 4;      // 8192 (hi) ; same for lo
constexpr int B_STAGE_BYTES = 2 * B_TILE_BYTES;
constexpr int OUT_SUB_BYTES = WG_M * 32 * 4;            // one {32 t x 64 series} store box: 8192
constexpr int OUT_BUF_BYTES = (TN / 32) * OUT_SUB_BYTES;     // 32768
constexpr int THREADS = 288;
constexpr int WARP_PROD = 8;                  // warps 0-3 / 4-7: the two warpgroups

struct Smem {
  static constexpr int b = 0;
  static constexpr int out = b + SB * B_STAGE_BYTES;                // 49152
  static constexpr int bars = out + 2 * 2 * OUT_BUF_BYTES;          // + 2 warpgroups x 2 buffers
  static constexpr int n_bars = 2 * SB;
  static constexpr int total = bars + n_bars * 8;
  static_assert(total + 1024 <= 232448, "exceeds the 227 KB of shared memory a CTA can opt into");
};

__device__ __forceinline__ void sts64(uint32_t addr, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x), "f"(y) : "memory");
}

// MULTI: a ragged batch (mmf_fit_forecast_ragged_f32, holdout-style requests): the work units come from a table
// (rows, calendar, chunk of THAT calendar's prediction rows, first row of the chunk in the stacked design table) and the
// output goes through the calendar's own tensor map -- the table clipped to that calendar's rows and columns, so a tile
// that straddles two calendars or a chunk that runs past the calendar's last date never writes outside its own block.
template <bool MULTI>
__global__ void __launch_bounds__(THREADS, 1)
predict_tc_kernel(const __grid_constant__ PredictLaunch pl, const DesignView d, const FitArgs a, const int n_tiles,
                  const int n_chunks, const PredUnit* __restrict__ units, const unsigned char* __restrict__ tmaps_out,
                  const int64_t n_units_multi) {
  const int64_t n_units = MULTI ? n_units_multi : (int64_t)n_tiles * n_chunks;
  auto unit_at = [&](int64_t u) -> PredUnit {
    if (MULTI) {
      const int4* p = reinterpret_cast<const int4*>(units + u);
      const int4 v0 = __ldg(p), v1 = __ldg(p + 1);
      return PredUnit{v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
    }
    const int tile = (int)(u / n_chunks), ch = (int)(u % n_chunks);
    const int64_t left = a.n - (int64_t)tile * TILE_M;
    return PredUnit{tile * TILE_M, (int)(left >= TILE_M ? TILE_M : left), 0, ch, a.pred_start + ch * TN, tile * TILE_M, 0, 0};
  };
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  const uint32_t sbase = smem_u32(smem);
  const uint32_t s_b = sbase + Smem::b;
  const uint32_t s_out = sbase + Smem::out;
  const uint32_t s_bars = sbase + Smem::bars;
  auto bar_bfull = [&](int s) { return s_bars + 8u * s; };
  auto bar_bempty = [&](int s) { return s_bars + 8u * (SB + s); };
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == WARP_PROD && lane == 0) {
    for (int s = 0; s < SB; ++s) {
      mbar_init(bar_bfull(s), 1);
      mbar_init(bar_bempty(s), 8);     // the 8 MMA warps, after their MMAs have retired
    }
    fence_mbar_init();
    prefetch_tensormap(pl.tmap_bhi);
    prefetch_tensormap(pl.tmap_blo);
    prefetch_tensormap(pl.tmap_out);
  }
  __syncthreads();

  if (warp == WARP_PROD) {
    // =========================== TMA producer: design rows of the prediction window ===========================
    // Work units are (tile, chunk) pairs in chunk-major order, dealt round-robin to the CTAs: at any moment the
    // CTAs with neighbouring ids write neighbouring 512-B pieces of the SAME 128 rows, i.e. one contiguous region
    // of the table, instead of unrelated row sets (DRAM write locality).
    int stage = 0;
    uint32_t phase = 0;
    for (int64_t u = blockIdx.x; u < n_units; u += gridDim.x) {
      const int t0 = unit_at(u).b_row;
      mbar_wait(bar_bempty(stage), phase ^ 1u);
      tma_load_2d_x2_elect(bar_bfull(stage), B_STAGE_BYTES,
                           s_b + stage * B_STAGE_BYTES, pl.tmap_bhi, 0, t0, L2_EVICT_LAST,
                           s_b + stage * B_STAGE_BYTES + B_TILE_BYTES, pl.tmap_blo, 0, t0, L2_EVICT_LAST);
      if (++stage == SB) { stage = 0; phase ^= 1u; }
    }
  } else {
    // =========================== warpgroups: gamma fragments -> wgmma -> + c -> swizzled tiles -> TMA store ===========
    const int wg = warp >> 2;                              // rows 64*wg .. 64*wg + 63 of every tile
    const int g8 = lane >> 2, t4 = lane & 3;
    const int frow = 16 * (warp & 3) + g8;                 // fragment rows frow, frow + 8 of the warpgroup's 64
    const bool leader = (warp & 3) == 0;
    int stage = 0;
    uint32_t phase = 0;
    int64_t k = 0;                                         // this CTA's unit counter: staging buffer k & 1
    for (int64_t u = blockIdx.x; u < n_units; u += gridDim.x, ++k) {
      const PredUnit pu = unit_at(u);
      uint32_t ahi[2][4], alo[2][4];                       // [k-step][fragment register]
      float c[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int rl = WG_M * wg + frow + 8 * j;
        const bool live = rl < pu.nrows;
        const float* __restrict__ gp = a.out_gamma + ((int64_t)pu.row0 + rl) * P;
        c[j] = live ? __ldg(a.out_c + pu.row0 + rl) : 0.f;
#pragma unroll
        for (int kk = 0; kk < 2; ++kk)
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            const float gv = live ? __ldg(gp + 8 * kk + 4 * hf + t4) : 0.f;
            const uint32_t h = __float_as_uint(gv) & 0xFFFFE000u;
            ahi[kk][j + 2 * hf] = h;
            alo[kk][j + 2 * hf] = __float_as_uint(gv - __uint_as_float(h));
          }
      }
      float acc[TN / 2];
#pragma unroll
      for (int i = 0; i < TN / 2; ++i) acc[i] = 0.f;
      mbar_wait(bar_bfull(stage), phase);
      const uint64_t bhi = gmma_desc_k_sw64(s_b + stage * B_STAGE_BYTES);
      const uint64_t blo = gmma_desc_k_sw64(s_b + stage * B_STAGE_BYTES + B_TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        wgmma_m64n128k8_tf32_rs(acc, ahi[kk], bhi + static_cast<uint64_t>(kk * 2));
        wgmma_m64n128k8_tf32_rs(acc, ahi[kk], blo + static_cast<uint64_t>(kk * 2));
        wgmma_m64n128k8_tf32_rs(acc, alo[kk], bhi + static_cast<uint64_t>(kk * 2));
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_bempty(stage));      // design tile free for the producer
      if (++stage == SB) { stage = 0; phase ^= 1u; }

      const uint32_t obase = s_out + static_cast<uint32_t>(wg * 2 + (int)(k & 1)) * OUT_BUF_BYTES;
      if (leader) bulk_wait_read1_elect();                 // the stores of unit k - 2 have read this buffer
      named_bar_sync(1 + wg, 128);
#pragma unroll
      for (int i = 0; i < TN / 8; ++i) {                   // n8 block i: columns 8i + 2t4, +1 of rows frow, frow + 8
        const uint32_t q = static_cast<uint32_t>(2 * (i & 3) + (t4 >> 1));
        const uint32_t col = obase + (i >> 2) * OUT_SUB_BYTES + ((q ^ static_cast<uint32_t>(g8)) << 4) + (t4 & 1) * 8;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float v0 = acc[4 * i + 2 * j] + c[j], v1 = acc[4 * i + 2 * j + 1] + c[j];
          sts64(col + static_cast<uint32_t>(frow + 8 * j) * 128u, v0, v1);
          if (!MULTI) {
            // the table's last n_pred % 4 columns: a TMA store would also write the caller's columns up to the next
            // multiple of 4, so these few go out as plain stores
            const int tcol = pu.ch * TN + 8 * i + 2 * t4;
            const int rl = WG_M * wg + frow + 8 * j;
            if (tcol + 1 >= pl.n_tma && tcol < a.n_pred && rl < pu.nrows) {
              float* __restrict__ orow = a.out + ((int64_t)pu.row0 + rl) * a.ld_out;
              if (tcol >= pl.n_tma) orow[tcol] = v0;
              if (tcol + 1 < a.n_pred) orow[tcol + 1] = v1;
            }
          }
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + wg, 128);
      if (leader) {
        if (WG_M * wg < pu.nrows) {
          const void* tmo = MULTI ? static_cast<const void*>(tmaps_out + (size_t)pu.cal * 128) : static_cast<const void*>(pl.tmap_out);
          if (MULTI) fence_tensormap_acquire(tmo);
#pragma unroll
          for (int j = 0; j < TN / 32; ++j)
            if (MULTI || pu.ch * TN + j * 32 < pl.n_tma)
              tma_store_2d_elect(tmo, obase + j * OUT_SUB_BYTES, pu.ch * TN + j * 32, pu.row_in_map + WG_M * wg);
        }
        bulk_commit_elect();
      }
    }
    if (leader) bulk_wait_all_elect();
  }
}

// Standard errors of the gap-free rows of a fit + predict_tc call: se[i, k] = sigma_i * sqrt(1 + h_{pred_start+k}), an
// outer product and a pure HBM write (one warp per row, coalesced).  It runs right after fit_tc_kernel: MMF_STATUS_OK
// then marks exactly the rows that kernel finished; the passes behind it write the se rows of all the others.
__global__ void __launch_bounds__(256)
se_outer_kernel(const int32_t* __restrict__ status, const float* __restrict__ sigma, const float* __restrict__ sfac,
                int32_t pred_start, int32_t n_pred, int64_t n, float* __restrict__ out_se, int64_t ld_se) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * 8;
  for (int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); row < n; row += warps) {
    if (status[row] != MMF_STATUS_OK) continue;
    const float sg = sigma[row];
    float* __restrict__ o = out_se + row * ld_se;
    for (int k = lane; k < n_pred; k += 32) __stcs(o + k, sg * __ldg(sfac + pred_start + k));
  }
}

}  // namespace

cudaError_t launch_se_outer(const FitArgs& a, const SeArgs& se, int sm_count, cudaStream_t s) {
  if (a.n <= 0 || se.out_se == nullptr) return cudaSuccess;
  const int64_t want = (a.n + 7) / 8, cap = (int64_t)sm_count * 8;
  se_outer_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, s>>>(a.status, se.sigma, se.sfac, a.pred_start, a.n_pred,
                                                                     a.n, se.out_se, se.ld_se);
  return cudaGetLastError();
}

cudaError_t launch_predict_tc(const DesignView& d, const FitArgs& a, const PredictLaunch& pl, int sm_count,
                              cudaStream_t s, const PredUnit* units, int64_t n_units_multi, const unsigned char* tmaps_out) {
  if (a.n <= 0) return cudaSuccess;
  const size_t smem = Smem::total + 1024;
  if (units != nullptr) {
    if (n_units_multi <= 0) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(predict_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = n_units_multi < sm_count ? (int)n_units_multi : sm_count;
    predict_tc_kernel<true><<<grid, THREADS, smem, s>>>(pl, d, a, 0, 1, units, tmaps_out, n_units_multi);
    return cudaGetLastError();
  }
  const int n_tiles = (int)((a.n + TILE_M - 1) / TILE_M);
  const int n_chunks = (a.n_pred + TN - 1) / TN;
  cudaError_t e = cudaFuncSetAttribute(predict_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const int64_t n_units = (int64_t)n_tiles * n_chunks;
  const int grid = n_units < sm_count ? (int)n_units : sm_count;
  predict_tc_kernel<false><<<grid, THREADS, smem, s>>>(pl, d, a, n_tiles, n_chunks, nullptr, nullptr, 0);
  return cudaGetLastError();
}

}  // namespace mmf
