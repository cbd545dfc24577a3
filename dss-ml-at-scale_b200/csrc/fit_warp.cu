// fit_warp.cu -- warp-per-series-group fit + forecast on CUDA cores (general path).
//
// One warp owns S = MMF_WARP_S (2) consecutive series ((Product,SKU) groups of the reference fan-out,
// group_apply/02_Fine_Grained_Demand_Forecasting.py:523-528) and does what the reference UDF does
// for each (02:435-494) in the whitened calendar basis:
//   b   = sum_{t observed} a_t (y_t - c)     lanes stride over t (coalesced 128-B row segments); one
//                                            LDS.128 x4 design-row fetch feeds S series = 16*S FMAs
//   fully observed series : G_i = I, gamma = b
//   series with gaps      : second pass over the (L2-hot) row builds D = sum_{missing} a_t a_t^T
//                           warp-cooperatively (or the Gram over the observed rows when most are
//                           missing), then an in-order Cholesky of G_i in shared memory with pivot
//                           dropping and two triangular solves -- one warp per series
//   yhat_t = c + a_t . gamma                  for the requested rows, again S series per design row
// It handles everything (NaN masks, any leading dimension, any number of prediction rows: the
// reference's "Demand_Fitted for every date" contract, 02:484-494) and is also the masked fix-up
// pass behind the tensor-core kernel.  Bound: HBM; see DESIGN.md section 4.
#include "mmf_internal.cuh"

namespace mmf {
namespace {

#ifndef MMF_WARP_S
#define MMF_WARP_S 2
#endif
#ifndef MMF_WARP_U
#define MMF_WARP_U 8
#endif
#ifndef MMF_WARP_WARPS
#define MMF_WARP_WARPS 16
#endif
constexpr int S = MMF_WARP_S;               // series per warp pass (share each design-row fetch)
constexpr int WARPS = MMF_WARP_WARPS;       // one CTA per SM: the design table is staged once per SM
constexpr int THREADS = WARPS * 32;
constexpr int U = MMF_WARP_U;               // time blocks (32 t) per pass: U*S independent 128-B loads per warp
constexpr int MISS_CAP = 96;                // missing positions remembered per series (else: second pass)
constexpr int DPL = (NPAIR + 31) / 32;      // packed Gram entries per lane (5)

struct WarpScratch {
  float G[P][P + 1];
  float diag0[P];
  float b[P];
  int miss_n[S];                       // missing positions seen in the streaming pass
  unsigned short miss_t[S][MISS_CAP];
};

__device__ __forceinline__ bool is_finite_bits(float v) {
  return (__float_as_uint(v) & 0x7f800000u) != 0x7f800000u;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct ARows {
  const float4* s;    // shared copy [4][srows]
  const float4* g;    // global      [4][n_rows_pad]
  int srows;
  int grows;
  __device__ __forceinline__ float4 vec(int j, int t) const {
    return (t < srows) ? s[j * srows + t] : __ldg(&g[(size_t)j * grows + t]);
  }
  __device__ __forceinline__ float elem(int t, int i) const {
    const float* base = (t < srows) ? reinterpret_cast<const float*>(s + (i >> 2) * srows + t)
                                    : reinterpret_cast<const float*>(g + (size_t)(i >> 2) * grows + t);
    return base[i & 3];
  }
};

#define MMF_DOT16(acc_, a0, a1, a2, a3, val_)                                                   \
  acc_[0] = fmaf(a0.x, val_, acc_[0]);   acc_[1] = fmaf(a0.y, val_, acc_[1]);                   \
  acc_[2] = fmaf(a0.z, val_, acc_[2]);   acc_[3] = fmaf(a0.w, val_, acc_[3]);                   \
  acc_[4] = fmaf(a1.x, val_, acc_[4]);   acc_[5] = fmaf(a1.y, val_, acc_[5]);                   \
  acc_[6] = fmaf(a1.z, val_, acc_[6]);   acc_[7] = fmaf(a1.w, val_, acc_[7]);                   \
  acc_[8] = fmaf(a2.x, val_, acc_[8]);   acc_[9] = fmaf(a2.y, val_, acc_[9]);                   \
  acc_[10] = fmaf(a2.z, val_, acc_[10]); acc_[11] = fmaf(a2.w, val_, acc_[11]);                 \
  acc_[12] = fmaf(a3.x, val_, acc_[12]); acc_[13] = fmaf(a3.y, val_, acc_[13]);                 \
  acc_[14] = fmaf(a3.z, val_, acc_[14]); acc_[15] = fmaf(a3.w, val_, acc_[15]);

__device__ __forceinline__ float dot16(const float4& a0, const float4& a1, const float4& a2, const float4& a3,
                                       const float (&g)[P], float s) {
  s = fmaf(a0.x, g[0], s);  s = fmaf(a0.y, g[1], s);  s = fmaf(a0.z, g[2], s);  s = fmaf(a0.w, g[3], s);
  s = fmaf(a1.x, g[4], s);  s = fmaf(a1.y, g[5], s);  s = fmaf(a1.z, g[6], s);  s = fmaf(a1.w, g[7], s);
  s = fmaf(a2.x, g[8], s);  s = fmaf(a2.y, g[9], s);  s = fmaf(a2.z, g[10], s); s = fmaf(a2.w, g[11], s);
  s = fmaf(a3.x, g[12], s); s = fmaf(a3.y, g[13], s); s = fmaf(a3.z, g[14], s); s = fmaf(a3.w, g[15], s);
  return s;
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One masked series: Gram (down)date over the row, in-order Cholesky with pivot dropping, two solves.
// `b` (moments, identical in every lane) in, gamma out; returns the status.  Deliberately not inlined
// into the S-unrolled paths: it is the rare path and would quadruple the hot loop's I-cache footprint.
// SE: zz = |z|^2 of the forward solve (= b'gamma); the factor stays in scr.G for the se rows.
template <bool SE>
__device__ __noinline__ int solve_masked(const DesignView& d, const ARows& A, const float* __restrict__ yr,
                                         int nmiss, const unsigned short* __restrict__ miss_list,
                                         WarpScratch& scr, float (&g)[P], int lane, float& zz, unsigned& omask,
                                         bool gram_direct) {
  const int t_fit = d.t_fit;
  int pi[DPL], pj[DPL];
#pragma unroll
  for (int k = 0; k < DPL; ++k) {           // packed lower-triangular entries owned by this lane
    const int e = lane + 32 * k;
    int i = 0;
    while ((i + 1) * (i + 2) / 2 <= e) ++i;
    pi[k] = (e < NPAIR) ? i : 0;
    pj[k] = (e < NPAIR) ? e - i * (i + 1) / 2 : 0;
  }
  // Mostly-missing rows: G_i = I - D would cancel catastrophically in fp32, so accumulate the Gram
  // directly over the (few) observed rows instead of downdating over the (many) missing ones.
  bool direct = 2 * nmiss > t_fit;
  float dacc[DPL];
#pragma unroll 1
  for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
  for (int k = 0; k < DPL; ++k) dacc[k] = 0.f;
  if (!direct && nmiss <= MISS_CAP && t_fit <= 65535) {
    // positions were recorded while streaming: no second trip to memory
#pragma unroll 1
    for (int m = 0; m < nmiss; ++m) {
      const int tt = miss_list[m];
#pragma unroll
      for (int k = 0; k < DPL; ++k) dacc[k] = fmaf(A.elem(tt, pi[k]), A.elem(tt, pj[k]), dacc[k]);
    }
  } else {
    // second pass over the row (L2-hot), 8 independent 128-B loads in flight per trip.  Every lane sums its entries
    // over the whole row; for a long row (a mostly-missing one sums every observed position) the partial sums grow and
    // so does the rounding of each addition, so the sums restart every FOLD_T positions and are added up in dsum.  Rows
    // of up to FOLD_T fit values are summed exactly as without folding.
    constexpr int FOLD_T = 2048;
    float dsum[DPL];
    bool folded = false;
#pragma unroll 1
    for (int t0 = 0; t0 < t_fit; t0 += 256) {
      if (t0 > 0 && t0 % FOLD_T == 0) {
#pragma unroll
        for (int k = 0; k < DPL; ++k) { dsum[k] = folded ? dsum[k] + dacc[k] : dacc[k]; dacc[k] = 0.f; }
        folded = true;
      }
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int t = t0 + u * 32 + lane;
        v[u] = (t < t_fit) ? __ldg(yr + t) : (direct ? __int_as_float(0x7fc00000) : 0.f);
      }
#pragma unroll 1
      for (int u = 0; u < 8; ++u) {
        float vu = v[0];
#pragma unroll
        for (int q = 1; q < 8; ++q) vu = (q == u) ? v[q] : vu;
        unsigned mm = __ballot_sync(0xffffffffu, is_finite_bits(vu) == direct);
#pragma unroll 1
        while (mm) {
          const int tt = t0 + u * 32 + __ffs(mm) - 1;
          mm &= mm - 1;
#pragma unroll
          for (int k = 0; k < DPL; ++k) dacc[k] = fmaf(A.elem(tt, pi[k]), A.elem(tt, pj[k]), dacc[k]);
        }
      }
    }
    if (folded) {
#pragma unroll
      for (int k = 0; k < DPL; ++k) dacc[k] = dsum[k] + dacc[k];
    }
  }
  if (!gram_direct || direct) break;
  // the general pass after the tensor-core kernel (gram_direct): its rows start with a gap, and when the missing rows
  // carry more than 40 % of the design's leverage (trace D > 0.4 x kept columns) I - D cancels to pivots near
  // MMF_PIVOT_TOL even with fewer than half of the values missing -- sum the Gram over the observed rows instead
  float tr = 0.f;
#pragma unroll
  for (int k = 0; k < DPL; ++k)
    if (lane + 32 * k < NPAIR && pi[k] == pj[k] && ((d.kept_mask >> pi[k]) & 1u)) tr += dacc[k];
  if (warp_sum(tr) <= 0.4f * static_cast<float>(__popc(d.kept_mask & 0xFFFFu))) break;
  direct = true;
  }
  __syncwarp();
#pragma unroll
  for (int k = 0; k < DPL; ++k) {
    const int e = lane + 32 * k;
    if (e < NPAIR) {
      const int i = pi[k], j = pj[k];
      const float full = (i == j && ((d.kept_mask >> i) & 1u)) ? 1.f : 0.f;
      const float gij = direct ? dacc[k] : full - dacc[k];
      scr.G[i][j] = gij;
      scr.G[j][i] = gij;
      if (i == j) scr.diag0[i] = gij;
    }
  }
  if (lane < P) {
    float bl = 0.f;
#pragma unroll
    for (int p = 0; p < P; ++p) bl = (lane == p) ? g[p] : bl;
    scr.b[lane] = bl;
  }
  __syncwarp();
  // right-looking Cholesky, lane -> (row i = lane&15, column half h = lane>>4)
  const int ri = lane & 15, ch = lane >> 4;
  unsigned dropped = 0u, kept_cols = 0u;
#pragma unroll 1
  for (int j = 0; j < P; ++j) {
    const float dj = scr.G[j][j];
    const float d0 = scr.diag0[j];
    const bool globally_out = !((d.kept_mask >> j) & 1u);
    const bool keep = !globally_out && d0 > 0.f && dj > MMF_PIVOT_TOL * d0;
    if (SE && keep) kept_cols |= 1u << j;
    __syncwarp();
    if (keep) {
      const float inv = rsqrtf(dj);
      const float lij = (ri > j) ? scr.G[ri][j] * inv : 0.f;     // column j of L, row ri
      __syncwarp();
      if (ch == 0) {
        if (ri > j) scr.G[ri][j] = lij;
        if (ri == j) scr.G[j][j] = dj * inv;                      // sqrt(dj)
      }
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {                            // trailing update of this lane's column half
        const int k = ch * 8 + kk;
        const float lkj = __shfl_sync(0xffffffffu, lij, k);       // lane k (half 0) holds L[k][j]
        if (ri > j && k > j) scr.G[ri][k] = fmaf(-lij, lkj, scr.G[ri][k]);
      }
    } else {
      if (!globally_out && d0 > 0.f) dropped |= 1u << j;
      if (ch == 0) {
        if (ri > j) scr.G[ri][j] = 0.f;
        if (ri == j) scr.G[j][j] = 1.f;
      }
      if (lane == 0) scr.b[j] = 0.f;                              // gamma_j = 0
    }
    __syncwarp();
  }
  const unsigned outmask = dropped | ~d.kept_mask;
  if (SE) omask = ~kept_cols & 0xFFFFu;              // also the columns no observed row touches (pivot 0)
#pragma unroll 1
  for (int j = 0; j < P; ++j) {                                   // forward solve L z = b
    float zj = 0.f;
    if (!((outmask >> j) & 1u)) zj = scr.b[j] / scr.G[j][j];
    __syncwarp();
    if (lane == j) scr.b[j] = zj;
    if (lane > j && lane < P) scr.b[lane] = fmaf(-scr.G[lane][j], zj, scr.b[lane]);
    __syncwarp();
  }
  if (SE) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < P; ++j) s = fmaf(scr.b[j], scr.b[j], s);
    zz = s;
    __syncwarp();
  }
#pragma unroll 1
  for (int j = P - 1; j >= 0; --j) {                              // backward solve L^T gamma = z
    float gj = 0.f;
    if (!((outmask >> j) & 1u)) gj = scr.b[j] / scr.G[j][j];
    __syncwarp();
    if (lane == j) scr.b[j] = gj;
    if (lane < j) scr.b[lane] = fmaf(-scr.G[j][lane], gj, scr.b[lane]);
    __syncwarp();
  }
#pragma unroll
  for (int p = 0; p < P; ++p) g[p] = ((outmask >> p) & 1u) ? 0.f : scr.b[p];
  __syncwarp();
  return dropped ? MMF_STATUS_RANKDEF : MMF_STATUS_OK;
}

// se row of one series after solve_masked: h_t = |L^-1 a_t|^2 with the factor in scr.G, lanes over the rows
__device__ __forceinline__ void se_row_masked(const DesignView& d, const FitArgs& a, const SeArgs& se, const ARows& A,
                                              const WarpScratch& scr, unsigned outmask, float sig, int64_t row,
                                              int lane) {
  float rinv[P];                                  // 1 / L_jj once per series: no division per prediction row
#pragma unroll
  for (int j = 0; j < P; ++j) rinv[j] = ((outmask >> j) & 1u) ? 0.f : 1.f / scr.G[j][j];
#pragma unroll 1
  for (int k = lane; k < a.n_pred; k += 32) {
    const int t = a.pred_start + k;
    const float4 a0 = A.vec(0, t), a1 = A.vec(1, t), a2 = A.vec(2, t), a3 = A.vec(3, t);
    const float av[P] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w, a3.x, a3.y, a3.z, a3.w};
    float w[P];
    float h = 0.f;
#pragma unroll
    for (int j = 0; j < P; ++j) {
      float s = av[j];
#pragma unroll
      for (int q = 0; q < j; ++q) s = fmaf(-scr.G[j][q], w[q], s);
      w[j] = s * rinv[j];
      h = fmaf(w[j], w[j], h);
    }
    se.out_se[row * se.ld_se + k] = sig * sqrtf(1.f + h);
  }
}

__device__ __forceinline__ float sigma_of(double ss, double bg, int dof) {
  return dof > 0 ? static_cast<float>(sqrt(fmax(ss - bg, 0.0) / dof)) : __int_as_float(0x7fc00000);
}

template <bool SE>
__global__ void __launch_bounds__(THREADS, 1)
fit_warp_kernel(const DesignView d, const FitArgs a, const int smem_rows, const SeArgs se) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  // programmatic dependent launch: this kernel may have been scheduled before its producer finished; its work starts
  // once the producer has completed.  (Releasing ITS dependent -- solve_rows_kernel -- early as well was measured: the
  // pre-launched solve blocks cost the 2 %-missing workload 6 % and small batches more; not done.)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (a.pending_count != nullptr && *a.pending_count == 0u) return;   // grid-uniform early exit

  float4* s_a4 = reinterpret_cast<float4*>(smem_raw);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  WarpScratch& scr = reinterpret_cast<WarpScratch*>(smem_raw + (size_t)4 * smem_rows * sizeof(float4))[warp];

  for (int i = threadIdx.x; i < 4 * smem_rows; i += THREADS) {
    const int j = i / smem_rows, t = i - j * smem_rows;
    s_a4[i] = d.a4[(size_t)j * d.n_rows_pad + t];
  }
  __syncthreads();

  const ARows A{s_a4, d.a4, smem_rows, d.n_rows_pad};
  const int t_fit = d.t_fit;
  const float qnan = __int_as_float(0x7fc00000);
  const int64_t n_groups = (a.n + S - 1) / S;
  const int64_t warps_total = (int64_t)gridDim.x * WARPS;

  for (int64_t grp = (int64_t)blockIdx.x * WARPS + warp; grp < n_groups; grp += warps_total) {
    const int64_t row0 = grp * S;
    bool act[S];
    bool any_act = false;
#pragma unroll
    for (int s = 0; s < S; ++s) {
      act[s] = row0 + s < a.n;
      if (act[s] && a.only_pending) act[s] = a.status[row0 + s] == MMF_STATUS_PENDING;
      any_act = any_act || act[s];
    }
    if (!any_act) continue;
    const float* __restrict__ yr0 = a.y + row0 * a.ld_y;

    // ---- centring constant per series: its first observed value (needs X[:,0] == 1); empty detection
    float c[S];
    bool any[S];
#pragma unroll
    for (int s = 0; s < S; ++s) {
      c[s] = 0.f;
      any[s] = false;
      if (act[s]) {
#pragma unroll 1
        for (int t0 = 0; t0 < t_fit; t0 += 32) {
          const int t = t0 + lane;
          const float v = (t < t_fit) ? __ldg(yr0 + s * a.ld_y + t) : qnan;
          const unsigned m = __ballot_sync(0xffffffffu, is_finite_bits(v));
          if (m) {
            c[s] = __shfl_sync(0xffffffffu, v, __ffs(m) - 1);
            any[s] = true;
            break;
          }
        }
        if (!d.has_constant) c[s] = 0.f;
      }
    }

    // ---- moments of the S series
    float acc[S][P];
    int miss[S];
    double ssq[S];                                   // SE: S = sum (y - c)^2 over the observed rows (f64: no restarts)
    if (lane < S) scr.miss_n[lane] = 0;
    __syncwarp();
#pragma unroll
    for (int s = 0; s < S; ++s) {
      miss[s] = 0;
      ssq[s] = 0.0;
#pragma unroll
      for (int p = 0; p < P; ++p) acc[s][p] = 0.f;
    }
#pragma unroll 1
    for (int t0 = 0; t0 < t_fit; t0 += 32 * U) {
      float v[U][S];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int t = t0 + u * 32 + lane;
#pragma unroll
        for (int s = 0; s < S; ++s) v[u][s] = (act[s] && t < t_fit) ? __ldcs(yr0 + s * a.ld_y + t) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int tb = t0 + u * 32;
        if (tb < t_fit) {                          // warp-uniform
          const int t = tb + lane;
          const bool inr = t < t_fit;
          const float4 a0 = A.vec(0, t), a1 = A.vec(1, t), a2 = A.vec(2, t), a3 = A.vec(3, t);
#pragma unroll
          for (int s = 0; s < S; ++s) {
            const bool fin = is_finite_bits(v[u][s]);
            const float r = (inr && fin) ? v[u][s] - c[s] : 0.f;
            if (inr && !fin) {                     // rare: remember where, for the Gram downdate
              ++miss[s];
              const int pos = atomicAdd(&scr.miss_n[s], 1);
              if (pos < MISS_CAP) scr.miss_t[s][pos] = (unsigned short)t;
            }
            MMF_DOT16(acc[s], a0, a1, a2, a3, r)
            if (SE) ssq[s] = fma(static_cast<double>(r), static_cast<double>(r), ssq[s]);
          }
        }
      }
    }
#pragma unroll
    for (int s = 0; s < S; ++s) {
#pragma unroll
      for (int p = 0; p < P; ++p) {
        acc[s][p] = warp_sum(acc[s][p]);
        if (!((d.kept_mask >> p) & 1u)) acc[s][p] = 0.f;         // fully observed: G_i = I, gamma = b
      }
      miss[s] = __reduce_add_sync(0xffffffffu, miss[s]);
      if (SE) ssq[s] = warp_sum_d(ssq[s]);
    }

    __syncwarp();                                    // missing positions recorded by other lanes are visible now
    // ---- series with gaps: per-series normal equations (rare path, one copy of the code)
    int st[S];
    bool deferred[S];
    bool se_done[S];                                 // SE: sigma / dof / se row already written by the masked solve
#pragma unroll
    for (int s = 0; s < S; ++s) { st[s] = any[s] ? MMF_STATUS_OK : MMF_STATUS_EMPTY; deferred[s] = false; se_done[s] = false; }
#pragma unroll 1
    for (int s = 0; s < S; ++s) {
      bool need = false;
      int nm = 0;
#pragma unroll
      for (int q = 0; q < S; ++q)
        if (q == s) { need = act[q] && any[q] && miss[q] > 0; nm = miss[q]; }
      if (!need) continue;                          // warp-uniform
      // (not in the general pass after the tensor-core kernel: its rows are solved here, on a Gram over the observed rows)
      if (a.recs != nullptr && !a.only_pending && nm <= SOLVE_MISS_CAP && nm <= MISS_CAP && 2 * nm <= t_fit && t_fit <= 65535) {
        // common case: hand the series to the thread-per-series solve kernel (moments + missing positions)
        SolveRec& rec = a.recs[row0 + s];
        float bl = 0.f, cs = 0.f;
#pragma unroll
        for (int q = 0; q < S; ++q) {
          if (q == s) {
            cs = c[q];
#pragma unroll
            for (int p = 0; p < P; ++p) bl = (lane == p) ? acc[q][p] : bl;
          }
        }
        if (lane < P) rec.b[lane] = bl;
        if (lane == P) {
          rec.c = cs;
          if (SE) {
            double sq = ssq[0];
#pragma unroll
            for (int q = 1; q < S; ++q) sq = (q == s) ? ssq[q] : sq;
            rec.ss = static_cast<float>(sq);
          }
          rec.nm[0] = (uint16_t)(nm < SOLVE_SEG ? nm : SOLVE_SEG);
          rec.nm[1] = (uint16_t)(nm < SOLVE_SEG ? 0 : nm - SOLVE_SEG);
          rec.cal = a.cal_id;
          const unsigned slot = atomicAdd(a.rec_count, 1u);
          if (slot < a.rec_cap) a.rec_rows[slot] = a.row_base + row0 + s;
        }
        for (int m = lane; m < nm; m += 32) rec.miss_t[m] = scr.miss_t[s][m];   // segment 1 starts at SOLVE_SEG
        if (lane < ((nm + 3) & ~3) - nm) rec.miss_t[nm + lane] = 0;             // the solve kernel reads whole 8-B groups
#pragma unroll
        for (int q = 0; q < S; ++q) if (q == s) deferred[q] = true;
        continue;
      }
      float g[P];
#pragma unroll
      for (int p = 0; p < P; ++p) {
        float x = acc[0][p];
#pragma unroll
        for (int q = 1; q < S; ++q) x = (q == s) ? acc[q][p] : x;
        g[p] = x;
      }
      float zz = 0.f;
      unsigned outmask = 0u;
      const int rs = solve_masked<SE>(d, A, yr0 + s * a.ld_y, nm, scr.miss_t[s], scr, g, lane, zz, outmask,
                                      a.only_pending != 0);
#pragma unroll
      for (int q = 0; q < S; ++q) {
        if (q == s) {
          st[q] = rs;
#pragma unroll
          for (int p = 0; p < P; ++p) acc[q][p] = g[p];
        }
      }
      if (SE) {                                      // the factor is still in scr.G: this series' se row now
        double sq = ssq[0];
#pragma unroll
        for (int q = 1; q < S; ++q) sq = (q == s) ? ssq[q] : sq;
        const int dof = t_fit - nm - __popc(~outmask & 0xFFFFu);
        const float sg = sigma_of(sq, static_cast<double>(zz), dof);
        if (se.out_se != nullptr) se_row_masked(d, a, se, A, scr, outmask, sg, row0 + s, lane);
        if (lane == 0) {
          se.sigma[row0 + s] = sg;
          if (se.dof != nullptr) se.dof[row0 + s] = dof;
        }
#pragma unroll
        for (int q = 0; q < S; ++q) if (q == s) se_done[q] = true;
        __syncwarp();                                // scr.G is read until here; the next series overwrites it
      }
    }

    // ---- predictions for rows [pred_start, pred_start + n_pred): 4 series per design-row fetch
    const int64_t off0 = row0 * a.ld_out;
    if (a.out_gamma != nullptr) {
#pragma unroll
      for (int s = 0; s < S; ++s) {
        if (act[s] && !deferred[s]) {
          float gl = 0.f;
#pragma unroll
          for (int p = 0; p < P; ++p) gl = (lane == p) ? acc[s][p] : gl;
          if (lane < P) a.out_gamma[(row0 + s) * P + lane] = any[s] ? gl : qnan;
          if (lane == P) a.out_c[row0 + s] = any[s] ? c[s] : qnan;
        }
      }
    }
#pragma unroll 1
    for (int k = lane; k < (a.skip_pred ? 0 : a.n_pred); k += 32) {
      const int t = a.pred_start + k;
      const float4 a0 = A.vec(0, t), a1 = A.vec(1, t), a2 = A.vec(2, t), a3 = A.vec(3, t);
#pragma unroll
      for (int s = 0; s < S; ++s) {
        if (act[s] && !deferred[s]) {
          const float yhat = any[s] ? dot16(a0, a1, a2, a3, acc[s], c[s]) : qnan;
          store_out1(a, off0 + s * a.ld_out + k, yhat);
        }
      }
    }
    if (SE) {                                      // fully observed (G_i = I, b'gamma = |gamma|^2) and empty rows
#pragma unroll
      for (int s = 0; s < S; ++s) {
        if (!act[s] || deferred[s] || se_done[s]) continue;
        double bg = 0.0;
#pragma unroll
        for (int p = 0; p < P; ++p) bg = fma(static_cast<double>(acc[s][p]), static_cast<double>(acc[s][p]), bg);
        const int dof = any[s] ? t_fit - __popc(d.kept_mask) : 0;
        const float sg = sigma_of(ssq[s], bg, dof);
        if (se.out_se != nullptr)
          for (int k = lane; k < a.n_pred; k += 32)
            se.out_se[(row0 + s) * se.ld_se + k] = sg * __ldg(se.sfac + a.pred_start + k);
        if (lane == 0) {
          se.sigma[row0 + s] = sg;
          if (se.dof != nullptr) se.dof[row0 + s] = dof;
        }
      }
    }
    if (a.out_beta != nullptr && lane < P) {       // beta = W gamma (+ c on the intercept)
#pragma unroll
      for (int s = 0; s < S; ++s) {
        if (act[s] && !deferred[s]) {
          float b = (lane == 0 && d.has_constant) ? c[s] : 0.f;
#pragma unroll
          for (int q = 0; q < P; ++q) b = fmaf(__ldg(d.w + lane * P + q), acc[s][q], b);
          a.out_beta[(row0 + s) * P + lane] = any[s] ? b : qnan;
        }
      }
    }
    if (lane == 0) {
#pragma unroll
      for (int s = 0; s < S; ++s)
        if (act[s]) a.status[row0 + s] = deferred[s] ? MMF_STATUS_DEFERRED : st[s];
    }
  }
}

}  // namespace

constexpr size_t FIT_WARP_SMEM_MAX = 200 * 1024;

size_t fit_warp_smem_bytes(const DesignView& d, int* smem_rows) {
  // one CTA per SM: keep as many design rows resident as fit beside the per-warp scratch
  const size_t scratch = sizeof(WarpScratch) * WARPS;
  const size_t budget = FIT_WARP_SMEM_MAX - scratch;
  int rows = d.n_rows_pad;
  const int max_rows = (int)(budget / (4 * sizeof(float4))) & ~31;
  if (rows > max_rows) rows = max_rows;
  *smem_rows = rows;
  return (size_t)rows * 4 * sizeof(float4) + scratch;
}

cudaError_t launch_fit_warp(const DesignView& d, const FitArgs& a, int sm_count, cudaStream_t s, const SeArgs* se) {
  if (a.n <= 0) return cudaSuccess;
  int smem_rows = 0;
  const size_t smem = fit_warp_smem_bytes(d, &smem_rows);
  auto kern = se != nullptr ? fit_warp_kernel<true> : fit_warp_kernel<false>;
  // the attribute is per function and process-wide: always the same value, the most any design needs, so that a
  // context on another host thread cannot lower it between this launch's set and the launch
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FIT_WARP_SMEM_MAX);
  if (e != cudaSuccess) return e;
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, THREADS, smem);
  if (e != cudaSuccess) return e;
  if (per_sm < 1) per_sm = 1;
  const int64_t groups = (a.n + S - 1) / S;
  int64_t blocks = (groups + WARPS - 1) / WARPS;
  const int64_t cap = (int64_t)sm_count * per_sm;
  if (blocks > cap) blocks = cap;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)blocks);
  cfg.blockDim = dim3(THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;      // launch latency hides under the producer
  attr[0].val.programmaticStreamSerializationAllowed = a.only_pending ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, d, a, smem_rows, se != nullptr ? *se : SeArgs{});
}

}  // namespace mmf
