// solve_rows.cu -- thread-per-series normal equations for series with gaps.
//
// The streaming kernel (fit_warp.cu) leaves, for every masked series, a 256-B record: the moments
// b = A_fit^T (y - c) over its observed rows, the centring constant and the grid positions of its missing
// rows.  Here ONE THREAD owns one series and does the rest of build_tune_and_score_model's fit/predict
// (reference 02:435-494) for it without touching shared memory or a barrier:
//   G_i = diag(kept) - sum_{t missing} a_t a_t^T        136 packed entries, in registers
//   in-order Cholesky of G_i with relative pivot dropping (MMF_PIVOT_TOL), fully unrolled
//   L z = b, L^T gamma = z ; yhat_t = c + a_t . gamma ; beta = W gamma on request
// A warp therefore factors 32 different 16x16 systems at once at full lane utilisation -- two orders of
// magnitude fewer issue slots per series than a warp-cooperative Cholesky with a barrier per column.
#include "mmf_internal.cuh"
#include "solve_math.cuh"

namespace mmf {
namespace {

constexpr int THREADS = 128;

// both 128-B lines of a record into L1: the record is read piecemeal (moments, then one gap position at a time),
// and every new 32-B sector would otherwise be its own trip to DRAM in the middle of the dependent chain
__device__ __forceinline__ void prefetch_rec(const SolveRec* r) {
  asm volatile("prefetch.global.L1 [%0];" ::"l"(r));
  asm volatile("prefetch.global.L1 [%0];" ::"l"(reinterpret_cast<const char*>(r) + 128));
}

// One queued series: Gram downdate, Cholesky with pivot dropping, both solves, forecasts, status.
// SE: also sigma / dof from S (rec.ss) and |z|^2, and the se row with h_t = |L^-1 a_t|^2 from the row's own factor.
template <bool MULTI, bool SE = false>
__device__ __forceinline__ void solve_one(const DesignView& d0, const FitArgs& a, const CalMeta* __restrict__ cals,
                                          const int64_t row, const bool vec_out, const SeArgs& se = SeArgs{}) {
  const SolveRec& rec = a.recs[row];
  float b[P];
  {
    const float4* bp = reinterpret_cast<const float4*>(rec.b);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = bp[q];
      b[4 * q] = v.x; b[4 * q + 1] = v.y; b[4 * q + 2] = v.z; b[4 * q + 3] = v.w;
    }
  }
  const float c = rec.c;
  const int nm0 = rec.nm[0], nm1 = rec.nm[1];
  // ragged launches: the record names its calendar; the stacked design tables are indexed from that calendar's row 0
  DesignView d = d0;
  int pred_start = a.pred_start;
  if (MULTI) {
    const int4* cp = reinterpret_cast<const int4*>(cals + rec.cal);
    const int4 m0 = __ldg(cp), m1 = __ldg(cp + 1);
    d.t_fit = m0.x;
    d.kept_mask = static_cast<uint32_t>(m0.w);
    d.apred = d0.apred + (size_t)m1.x * P;
    pred_start = m1.y;
  }

  // ---- G_i = I - sum over the missing rows of a_t a_t^T, Cholesky with pivot dropping, both solves (solve_math.cuh)
  auto load_group = [&](int seg, int gi) {
    return reinterpret_cast<const unsigned long long*>(rec.miss_t + seg * SOLVE_SEG)[gi];
  };
  auto se_tail = [&](const float (&G)[NPAIR], unsigned outmask, float zz) {
    if (!SE) return;
    const int dof = d.t_fit - nm0 - nm1 - __popc(~outmask & 0xFFFFu);
    const double rss = fmax(static_cast<double>(rec.ss) - static_cast<double>(zz), 0.0);
    const float sig = dof > 0 ? static_cast<float>(sqrt(rss / dof)) : __int_as_float(0x7fc00000);
    se.sigma[row] = sig;
    if (se.dof != nullptr) se.dof[row] = dof;
    if (se.out_se == nullptr) return;
    float rinv[P];
#pragma unroll
    for (int j = 0; j < P; ++j) rinv[j] = ((outmask >> j) & 1u) ? 0.f : 1.f / G[tri(j, j)];
#pragma unroll 1
    for (int k = 0; k < a.n_pred; ++k) {
      const float4* ap = reinterpret_cast<const float4*>(d.apred + (size_t)(pred_start + k) * P);
      const float4 a0 = __ldg(ap), a1 = __ldg(ap + 1), a2 = __ldg(ap + 2), a3 = __ldg(ap + 3);
      const float av[P] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w, a3.x, a3.y, a3.z, a3.w};
      se.out_se[row * se.ld_se + k] = sig * sqrtf(1.f + leverage_packed(G, rinv, av));
    }
  };
  const unsigned dropped = masked_solve(d, b, nm0, nm1, load_group, se_tail);

  if (a.out_gamma != nullptr) {
    float4* gp = reinterpret_cast<float4*>(a.out_gamma + row * P);
    gp[0] = make_float4(b[0], b[1], b[2], b[3]);    gp[1] = make_float4(b[4], b[5], b[6], b[7]);
    gp[2] = make_float4(b[8], b[9], b[10], b[11]);  gp[3] = make_float4(b[12], b[13], b[14], b[15]);
    a.out_c[row] = c;
  }
  // ---- forecasts (16-B stores when the table allows it: a thread owns a whole row of it)
  const int64_t off = row * a.ld_out;
  auto predict = [&](int k) -> float {
    const float4* ap = reinterpret_cast<const float4*>(d.apred + (size_t)(pred_start + k) * P);
    const float4 a0 = __ldg(ap), a1 = __ldg(ap + 1), a2 = __ldg(ap + 2), a3 = __ldg(ap + 3);
    float s = c;
    s = fmaf(a0.x, b[0], s);  s = fmaf(a0.y, b[1], s);  s = fmaf(a0.z, b[2], s);  s = fmaf(a0.w, b[3], s);
    s = fmaf(a1.x, b[4], s);  s = fmaf(a1.y, b[5], s);  s = fmaf(a1.z, b[6], s);  s = fmaf(a1.w, b[7], s);
    s = fmaf(a2.x, b[8], s);  s = fmaf(a2.y, b[9], s);  s = fmaf(a2.z, b[10], s); s = fmaf(a2.w, b[11], s);
    s = fmaf(a3.x, b[12], s); s = fmaf(a3.y, b[13], s); s = fmaf(a3.z, b[14], s); s = fmaf(a3.w, b[15], s);
    return s;
  };
  const int n_pred = a.skip_pred ? 0 : a.n_pred;
  int k = 0;
  if (vec_out) {
#pragma unroll 1
    for (; k + 4 <= n_pred; k += 4)
      store_out4(a, off + k, make_float4(predict(k), predict(k + 1), predict(k + 2), predict(k + 3)));
  }
#pragma unroll 1
  for (; k < n_pred; ++k) store_out1(a, off + k, predict(k));
  if (a.out_beta != nullptr) {
#pragma unroll 1
    for (int p = 0; p < P; ++p) {
      float s = (p == 0 && d.has_constant) ? c : 0.f;
#pragma unroll
      for (int q = 0; q < P; ++q) s = fmaf(__ldg(d.w + p * P + q), b[q], s);
      a.out_beta[row * P + p] = s;
    }
  }
  a.status[row] = dropped ? MMF_STATUS_RANKDEF : MMF_STATUS_OK;
}

__device__ __forceinline__ bool vec_out_ok(const FitArgs& a) {
  bool v = (a.ld_out % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.out) & 15u) == 0);
  for (int q = 0; q + 1 < a.n_out; ++q) v = v && ((reinterpret_cast<uintptr_t>(a.out_more[q]) & 15u) == 0);
  return v;
}

// The pass over the whole work list, after the producers have finished.
template <bool MULTI, bool SE = false>
__global__ void __launch_bounds__(THREADS, 2)
solve_rows_kernel(const DesignView d0, const FitArgs a, const CalMeta* __restrict__ cals, const SeArgs se) {
  asm volatile("griddepcontrol.wait;" ::: "memory");    // programmatic dependent launch: the producer kernels are done
  const uint32_t count = min(*a.rec_count, a.rec_cap);
  const uint32_t stride = gridDim.x * THREADS;
  const bool vec_out = vec_out_ok(a);
  uint32_t i = blockIdx.x * THREADS + threadIdx.x;
  int64_t row_next = i < count ? a.rec_rows[i] : 0;
  if (i < count) prefetch_rec(a.recs + row_next);
  for (; i < count; i += stride) {
    const int64_t row = row_next;
    if (i + stride < count) {                           // the next series' record arrives while this one is solved
      row_next = a.rec_rows[i + stride];
      prefetch_rec(a.recs + row_next);
    }
    solve_one<MULTI, SE>(d0, a, cals, row, vec_out, se);
  }
}

}  // namespace

cudaError_t launch_solve_rows(const DesignView& d, const FitArgs& a, int sm_count, cudaStream_t s, const CalMeta* cals,
                              const SeArgs* se) {
  if (a.recs == nullptr || a.rec_cap == 0) return cudaSuccess;
  const int64_t want = ((int64_t)a.rec_cap + THREADS - 1) / THREADS;
  const int64_t cap = (int64_t)sm_count * 8;
  const unsigned grid = (unsigned)(want < cap ? want : cap);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(THREADS);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;      // launch latency hides under the producer
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const SeArgs none{};
  if (se != nullptr) return cudaLaunchKernelEx(&cfg, solve_rows_kernel<false, true>, d, a, cals, *se);
  return cals != nullptr ? cudaLaunchKernelEx(&cfg, solve_rows_kernel<true>, d, a, cals, none)
                         : cudaLaunchKernelEx(&cfg, solve_rows_kernel<false>, d, a, cals, none);
}

}  // namespace mmf
