// select.cu -- per-series model selection on the device: the GPU analogue of the reference's per-group
// hyperopt loop (group_apply/02_Fine_Grained_Demand_Forecasting.py:435-469: fit candidate models on the train
// rows, score each by the MSE of its forecast over the held-out rows, keep the best, 02:472-488 refit + predict).
//
// Candidates are the nested models spanned by the first m whitened design columns (m in a small list, e.g.
// mean / +trend / +day-of-week / +yearly Fourier / +calendar dummies).  The whitened basis is orthonormal on
// the calendar, so for a gap-free series the least-squares fit of candidate m is simply the first m entries of
// the full coefficient vector gamma -- all candidates come from the ONE streaming pass that produced gamma.
// For a series with gaps the same truncation rule is used (a deterministic approximation of refitting).
// One thread per series: held-out rows are scored with running prefix sums, the winner's tail is zeroed in
// place, and predict_tc_kernel then writes fitted values + forecast for every date from the chosen model.
#include "mmf_internal.cuh"

namespace mmf {
namespace {

constexpr int THREADS = 128;

__global__ void __launch_bounds__(THREADS)
select_kernel(const DesignView d, const FitArgs a, const SelectArgs sel) {
  extern __shared__ float s_hold[];                 // [n_hold][P] whitened design rows of the held-out dates
  asm volatile("griddepcontrol.wait;" ::: "memory");
  for (int i = threadIdx.x; i < sel.n_hold * P; i += THREADS) s_hold[i] = __ldg(d.apred + (size_t)d.t_fit * P + i);
  __syncthreads();
  for (int64_t row = (int64_t)blockIdx.x * THREADS + threadIdx.x; row < a.n; row += (int64_t)gridDim.x * THREADS) {
    const int st = a.status[row];
    if (st != MMF_STATUS_OK && st != MMF_STATUS_RANKDEF) {      // empty series: nothing to choose
      if (sel.out_choice) sel.out_choice[row] = 0;
      if (sel.out_mse) sel.out_mse[row] = __int_as_float(0x7fc00000);
      continue;
    }
    float g[P];
    const float4* gp = reinterpret_cast<const float4*>(a.out_gamma + row * P);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = gp[q];
      g[4 * q] = v.x; g[4 * q + 1] = v.y; g[4 * q + 2] = v.z; g[4 * q + 3] = v.w;
    }
    const float c = a.out_c[row];
    // Running prefix sums over the whitened columns give every nested model's residual at once: after column p the
    // partial sum IS the prediction of the model made of columns 0..p, so each held-out row costs 16 FMAs for the
    // predictions and 16 for the squared errors of all 16 prefix lengths (statically indexed registers); the
    // candidates' scores are picked out of those 16 at the end.  (Testing every column against every candidate
    // inside the loop made this kernel issue-bound at ~4x the instructions.)
    float sse[P];
#pragma unroll
    for (int p = 0; p < P; ++p) sse[p] = 0.f;
    int n_obs = 0;
    const float* __restrict__ yh = a.y + row * a.ld_y + d.t_fit;
    for (int t = 0; t < sel.n_hold; ++t) {
      const float y = __ldg(yh + t);
      if ((__float_as_uint(y) & 0x7f800000u) == 0x7f800000u) continue;      // missing held-out value
      ++n_obs;
      const float4* arow = reinterpret_cast<const float4*>(s_hold + t * P);
      const float4 a0 = arow[0], a1 = arow[1], a2 = arow[2], a3 = arow[3];
      const float av[P] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w, a3.x, a3.y, a3.z, a3.w};
      float e = y - c;
#pragma unroll
      for (int p = 0; p < P; ++p) {
        e = fmaf(-av[p], g[p], e);                             // residual of the model on columns 0..p
        sse[p] = fmaf(e, e, sse[p]);
      }
    }
    auto sse_of = [&](int m) -> float {                        // m = number of leading columns, 1..16
      float v = sse[0];
#pragma unroll
      for (int p = 1; p < P; ++p) v = (m == p + 1) ? sse[p] : v;
      return v;
    };
    int best = sel.n_cand - 1;                                   // no observed held-out row: keep the full model
    float best_sse = sse_of(sel.cand[best]);
    if (n_obs > 0) {
      best = 0;
      best_sse = sse_of(sel.cand[0]);
#pragma unroll
      for (int kk = 1; kk < MMF_MAX_CAND; ++kk)
        if (kk < sel.n_cand) {
          const float v = sse_of(sel.cand[kk]);
          if (v < best_sse) { best = kk; best_sse = v; }
        }
    }
    const int m = sel.cand[best];
    float4* gw = reinterpret_cast<float4*>(a.out_gamma + row * P);
#pragma unroll
    for (int q = 0; q < 4; ++q)
      gw[q] = make_float4(4 * q < m ? g[4 * q] : 0.f, 4 * q + 1 < m ? g[4 * q + 1] : 0.f,
                          4 * q + 2 < m ? g[4 * q + 2] : 0.f, 4 * q + 3 < m ? g[4 * q + 3] : 0.f);
    if (sel.out_choice) sel.out_choice[row] = m;
    if (sel.out_mse) sel.out_mse[row] = n_obs > 0 ? best_sse / (float)n_obs : __int_as_float(0x7fc00000);
  }
}

}  // namespace

cudaError_t launch_select(const DesignView& d, const FitArgs& a, const SelectArgs& sel, int sm_count, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  const int64_t want = (a.n + THREADS - 1) / THREADS;
  const int64_t cap = (int64_t)sm_count * 16;
  const unsigned grid = (unsigned)(want < cap ? want : cap);
  const size_t smem = (size_t)sel.n_hold * P * sizeof(float);       // <= MMF_SELECT_MAX_HOLD * 64 B (validated at the ABI)
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  select_kernel<<<grid, THREADS, smem, s>>>(d, a, sel);
  return cudaGetLastError();
}

}  // namespace mmf
