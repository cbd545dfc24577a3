// ar.cu -- regression with AR(p) errors (DESIGN.md section 2 item 9, section 4.13): the two-step estimator behind
// mmf_fit_forecast_ar_f32.  The plain fit has already run and left gamma / c in the hand-off buffers (FitArgs::out_gamma,
// out_c) and the final status; this kernel
//   pass A  reads y over [0, t_fit) once: residuals e_t = y_t - c - a_t.gamma, lag products sum e_t e_{t-k} (k <= p) in
//           float64, n_obs; Levinson-Durbin in float64 gives the series' order, phi and the innovation variance;
//   pass B  re-reads y from s0 (the latest position <= min(pred_start, t_fit) whose p predecessors are all observed) and
//           writes c + a_t.gamma + sum_j phi_j u_{t-j} for the requested rows, filling missing residuals with their AR
//           prediction from the past (item 5).
// ar_select_kernel (section 2 item 10, section 4.14) adds per-series order selection by hold-out MSE.
// One warp per series, lanes over t, so y loads are coalesced 128-B segments (ar_common.cuh: staging and helpers).
#include "ar_common.cuh"

namespace mmf {
namespace {

__global__ void __launch_bounds__(THREADS, 3)
ar_kernel(const DesignView d, const FitArgs a, const ArArgs ar) {
  __shared__ float4 s_a[4][TC];
  __shared__ uint32_t s_nz[TC];
  __shared__ int s_lo;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * WARPS + warp;
  const bool live = row < a.n;
  const int p = ar.p;
  const int t_fit = d.t_fit;
  const int end = a.pred_start + a.n_pred;
  const int S = min(a.pred_start, t_fit);
  if (threadIdx.x == 0) s_lo = INT32_MAX;

  float g[P], c;
  const int st = load_fit(a, row, live, g, c);
  const bool work = live && st != MMF_STATUS_EMPTY;
  const float* __restrict__ yr = a.y + (live ? row : 0) * a.ld_y;

  // ---- pass A: residuals over the fit rows, lag products, and the restart position s0 of pass B
  double acc[AR_MAX + 1];
#pragma unroll
  for (int k = 0; k <= AR_MAX; ++k) acc[k] = 0.0;
  float eprev = 0.f;                       // residuals of the previous 32 rows (positions < 0: 0)
  uint32_t bprev = 0xffffffffu;            // their observed bits (positions < 0 count as observed: u = 0 there)
  int s0 = 0, n_obs = 0;
  uint32_t colmask = 0u;                   // whitened columns with a non-zero entry on an observed fit row
  // the chunk's y values are loaded one chunk ahead, so the loads of chunk c0 + TC are in flight while chunk c0 is
  // staged and processed
  float ys[NSUB];
#pragma unroll
  for (int q = 0; q < NSUB; ++q) ys[q] = work && 32 * q + lane < t_fit ? __ldg(yr + 32 * q + lane) : 0.f;
  for (int c0 = 0; c0 < t_fit; c0 += TC) {
    float yn[NSUB];
#pragma unroll
    for (int q = 0; q < NSUB; ++q) {
      const int t = c0 + TC + 32 * q + lane;
      yn[q] = work && t < t_fit ? __ldg(yr + t) : 0.f;
    }
    stage(s_a, s_nz, d, ar, c0);
    __syncthreads();
    if (work) {
#pragma unroll
      for (int q = 0; q < NSUB; ++q) {
        const int t0 = c0 + 32 * q;
        if (t0 >= t_fit) break;
        const int t = t0 + lane;
        const float yv = ys[q];
        const bool obs = t < t_fit && finite_f(yv);
        const float e = obs ? yv - fitted(s_a, t - c0, g, c) : 0.f;
        const uint32_t bal = __ballot_sync(0xffffffffu, obs);
        n_obs += __popc(bal);
        colmask |= obs ? s_nz[t - c0] : 0u;
        acc[0] = fma((double)e, (double)e, acc[0]);
#pragma unroll
        for (int k = 1; k <= AR_MAX; ++k)
          if (k <= p) acc[k] = fma((double)e, (double)lagged(e, eprev, k, lane), acc[k]);
        eprev = e;
        if (t0 < S) {
          // bit 32 + j of M: positions t0 + j - p + 1 .. t0 + j all observed, i.e. position t0 + 1 + j may start pass B
          const uint64_t comb = ((uint64_t)bal << 32) | bprev;
          uint64_t M = comb;
#pragma unroll
          for (int k = 2; k <= AR_MAX; ++k)
            if (k <= p) M &= comb << (k - 1);
          uint32_t ok = (uint32_t)(M >> 32);
          const int jmax = S - t0 - 1 + LATE_RESTART;            // t0 + 1 + j <= S
          if (jmax < 31) ok &= (2u << jmax) - 1u;
          if (ok) s0 = t0 + 1 + (31 - __clz(ok));
        }
        bprev = bal;
      }
    }
#pragma unroll
    for (int q = 0; q < NSUB; ++q) ys[q] = yn[q];
    __syncthreads();
  }

  // ---- order, Yule-Walker coefficients and innovation variance (float64 Levinson-Durbin, identical on every lane)
#pragma unroll
  for (int k = 0; k <= AR_MAX; ++k)
    if (k <= p)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  // used columns k of the dof rule (section 2 item 7): the calendar's kept columns that are non-zero on an observed fit
  // row (a column that is zero there has a zero pivot and is skipped, as in the fit kernels), less those the pivoted
  // solve dropped for the series' mask (status 2 only; a dropped column's gamma is pinned to exactly 0)
  const int k_used = used_columns(d, colmask, st, g);
  double phi[AR_MAX];
#pragma unroll
  for (int j = 0; j < AR_MAX; ++j) phi[j] = 0.0;
  int order = 0;
  double var = dnan();
  if (work) {
    const double inv = 1.0 / (double)max(n_obs, 1);
    double r[AR_MAX + 1];
#pragma unroll
    for (int k = 0; k <= AR_MAX; ++k) r[k] = acc[k] * inv;
    var = r[0];
    bool go = n_obs - k_used > p && r[0] > 0.0;
#pragma unroll
    for (int j = 1; j <= AR_MAX; ++j) {
      if (go && j <= p) {
        double num = r[j];
#pragma unroll
        for (int i = 1; i < j; ++i) num -= phi[i - 1] * r[j - i];
        const double kap = num / var;
        if (fabs(kap) >= (double)MMF_AR_KAPPA_MAX) {
          go = false;
        } else {
          double nxt[AR_MAX];
#pragma unroll
          for (int i = 1; i < j; ++i) nxt[i - 1] = phi[i - 1] - kap * phi[j - i - 1];
#pragma unroll
          for (int i = 1; i < j; ++i) phi[i - 1] = nxt[i - 1];
          phi[j - 1] = kap;
          var *= 1.0 - kap * kap;
          order = j;
        }
      }
    }
  }
  float f[AR_MAX];
#pragma unroll
  for (int j = 0; j < AR_MAX; ++j) f[j] = (float)phi[j];
  if (live) {
    store_row(ar.phi, row, lane, f);
    if (lane == 0) {
      if (ar.order != nullptr) ar.order[row] = order;
      if (ar.sigma != nullptr) ar.sigma[row] = (float)sqrt(var);
    }
    if (!work)                                                   // empty series: NaN predictions, as the plain call
      for (int k = lane; k < a.n_pred; k += 32) a.out[row * a.ld_out + k] = __int_as_float(0x7fc00000);
  }

  // ---- pass B from the aligned chunk that holds s0 - p: every state pass B needs is a plain residual
  const int b0 = max(s0 - p, 0) & ~31;
  if (work && lane == 0) atomicMin(&s_lo, b0);
  __syncthreads();
  const int lo = s_lo;
  float uprev = 0.f;                       // filled residuals u of the previous 32 rows
  for (int c0 = lo & ~(TC - 1); c0 < end; c0 += TC) {
    stage(s_a, s_nz, d, ar, c0);
    __syncthreads();
    if (work) {
#pragma unroll 1
      for (int t0 = max(c0, b0); t0 < min(c0 + TC, end); t0 += 32) {
        const int s = t0 + lane;
        const float fit = fitted(s_a, s - c0, g, c);
        const float yv = s < t_fit ? __ldg(yr + s) : 0.f;        // y is never read at or beyond t_fit
        const bool obs = s < t_fit && finite_f(yv);
        const float e = obs ? yv - fit : 0.f;
        const uint32_t bal = __ballot_sync(0xffffffffu, obs);
        const int nb = s0 - t0;                                  // lanes below nb lie before s0
        const uint32_t before = nb >= 32 ? 0xffffffffu : (nb <= 0 ? 0u : (1u << nb) - 1u);
        float u, arv = 0.f;
        if ((bal | before) == 0xffffffffu) {                     // no missing value at or after s0: all parallel
          u = e;
#pragma unroll
          for (int k = 1; k <= AR_MAX; ++k)
            if (k <= p) arv = fmaf(f[k - 1], lagged(u, uprev, k, lane), arv);
        } else {                                                 // fill (item 5) runs serially over the chunk
          float h[AR_MAX];
#pragma unroll
          for (int k = 0; k < AR_MAX; ++k) h[k] = __shfl_sync(0xffffffffu, uprev, 31 - k);   // h[k] = u_{t0-1-k}
          u = 0.f;
          // only the positions up to the last requested row are needed; the chain is p long (phi_k = 0 beyond p)
          const int jn = min(32, end - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            float pr = 0.f;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < p) pr = fmaf(f[k], h[k], pr);
            const float ej = __shfl_sync(0xffffffffu, e, j);
            const bool oj = (bal >> j) & 1u;
#ifdef MMF_AR_NO_FILL
            // negative control: a missing fit-window residual counts as 0 instead of its AR prediction
            const float v = (oj || t0 + j < s0 || t0 + j < t_fit) ? (oj ? ej : 0.f) : pr;
#else
            const float v = (oj || t0 + j < s0) ? (oj ? ej : 0.f) : pr;
#endif
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) h[k] = h[k - 1];
            h[0] = v;
            if (lane == j) { u = v; arv = pr; }
          }
        }
        uprev = u;
        if (s >= a.pred_start && s < end) a.out[row * a.ld_out + (s - a.pred_start)] = fit + arv;
      }
    }
    __syncthreads();
  }
}

// The selecting variant behind mmf_fit_select_ar_f32 (section 2 item 10, section 4.14): ar_kernel's pass A with p = ar.p,
// the largest candidate; Levinson-Durbin on lane j with its own bound sel.cand[j]; a scoring walk that forecasts the
// held-out rows with every candidate; the choice; and ar_kernel's pass B with the winner's order and coefficients.  It is
// a kernel of its own, not a template instantiation of ar_kernel, so that ar_kernel's code stays exactly as it was.
__global__ void __launch_bounds__(THREADS, 3)
ar_select_kernel(const DesignView d, const FitArgs a, const ArArgs ar, const ArSelArgs sel) {
  __shared__ float4 s_a[4][TC];
  __shared__ uint32_t s_nz[TC];
  __shared__ int s_lo;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * WARPS + warp;
  const bool live = row < a.n;
  const int p = ar.p;
  const int t_fit = d.t_fit;
  const int end = a.pred_start + a.n_pred;
  const int S = min(a.pred_start, t_fit);
  if (threadIdx.x == 0) s_lo = INT32_MAX;

  float g[P], c;
  const int st = load_fit(a, row, live, g, c);
  const bool work = live && st != MMF_STATUS_EMPTY;
  const float* __restrict__ yr = a.y + (live ? row : 0) * a.ld_y;

  // ---- pass A: residuals over the fit rows, lag products, and the restart position s0 of pass B
  double acc[AR_MAX + 1];
#pragma unroll
  for (int k = 0; k <= AR_MAX; ++k) acc[k] = 0.0;
  float eprev = 0.f;                       // residuals of the previous 32 rows (positions < 0: 0)
  uint32_t bprev = 0xffffffffu;            // their observed bits (positions < 0 count as observed: u = 0 there)
  int s0 = 0, n_obs = 0;
  int s0h = 0;                             // the latest position <= t_fit whose p predecessors are all observed
  uint32_t colmask = 0u;                   // whitened columns with a non-zero entry on an observed fit row
  // the chunk's y values are loaded one chunk ahead, so the loads of chunk c0 + TC are in flight while chunk c0 is
  // staged and processed
  float ys[NSUB];
#pragma unroll
  for (int q = 0; q < NSUB; ++q) ys[q] = work && 32 * q + lane < t_fit ? __ldg(yr + 32 * q + lane) : 0.f;
  for (int c0 = 0; c0 < t_fit; c0 += TC) {
    float yn[NSUB];
#pragma unroll
    for (int q = 0; q < NSUB; ++q) {
      const int t = c0 + TC + 32 * q + lane;
      yn[q] = work && t < t_fit ? __ldg(yr + t) : 0.f;
    }
    stage(s_a, s_nz, d, ar, c0);
    __syncthreads();
    if (work) {
#pragma unroll
      for (int q = 0; q < NSUB; ++q) {
        const int t0 = c0 + 32 * q;
        if (t0 >= t_fit) break;
        const int t = t0 + lane;
        const float yv = ys[q];
        const bool obs = t < t_fit && finite_f(yv);
        const float e = obs ? yv - fitted(s_a, t - c0, g, c) : 0.f;
        const uint32_t bal = __ballot_sync(0xffffffffu, obs);
        n_obs += __popc(bal);
        colmask |= obs ? s_nz[t - c0] : 0u;
        acc[0] = fma((double)e, (double)e, acc[0]);
#pragma unroll
        for (int k = 1; k <= AR_MAX; ++k)
          if (k <= p) acc[k] = fma((double)e, (double)lagged(e, eprev, k, lane), acc[k]);
        eprev = e;
        if (t0 < S) {
          // bit 32 + j of M: positions t0 + j - p + 1 .. t0 + j all observed, i.e. position t0 + 1 + j may start pass B
          const uint64_t comb = ((uint64_t)bal << 32) | bprev;
          uint64_t M = comb;
#pragma unroll
          for (int k = 2; k <= AR_MAX; ++k)
            if (k <= p) M &= comb << (k - 1);
          uint32_t ok = (uint32_t)(M >> 32);
          const int jmax = S - t0 - 1 + LATE_RESTART;            // t0 + 1 + j <= S
          if (jmax < 31) ok &= (2u << jmax) - 1u;
          if (ok) s0 = t0 + 1 + (31 - __clz(ok));
        }
        {                                                        // the same with the bound t_fit: the scoring walk's start
          const uint64_t comb = ((uint64_t)bal << 32) | bprev;
          uint64_t M = comb;
#pragma unroll
          for (int k = 2; k <= AR_MAX; ++k)
            if (k <= p) M &= comb << (k - 1);
          uint32_t ok = (uint32_t)(M >> 32);
          const int jmax = t_fit - t0 - 1;
          if (jmax < 31) ok &= (2u << jmax) - 1u;
          if (ok) s0h = t0 + 1 + (31 - __clz(ok));
        }
        bprev = bal;
      }
    }
#pragma unroll
    for (int q = 0; q < NSUB; ++q) ys[q] = yn[q];
    __syncthreads();
  }

  // ---- order, Yule-Walker coefficients and innovation variance (float64 Levinson-Durbin, bound pl on each lane)
#pragma unroll
  for (int k = 0; k <= AR_MAX; ++k)
    if (k <= p)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  // used columns k of the dof rule (section 2 item 7): the calendar's kept columns that are non-zero on an observed fit
  // row (a column that is zero there has a zero pivot and is skipped, as in the fit kernels), less those the pivoted
  // solve dropped for the series' mask (status 2 only; a dropped column's gamma is pinned to exactly 0)
  const int k_used = used_columns(d, colmask, st, g);
  // Levinson-Durbin bound of lane j: candidate j; lanes >= n_cand repeat the last candidate
  int pl = sel.cand[0];
#pragma unroll
  for (int j = 1; j < MMF_ARSEL_MAX_CAND; ++j)
    if (j < sel.n_cand && lane >= j) pl = sel.cand[j];
  double phi[AR_MAX];
#pragma unroll
  for (int j = 0; j < AR_MAX; ++j) phi[j] = 0.0;
  int order = 0;
  double var = dnan();
  if (work) {
    const double inv = 1.0 / (double)max(n_obs, 1);
    double r[AR_MAX + 1];
#pragma unroll
    for (int k = 0; k <= AR_MAX; ++k) r[k] = acc[k] * inv;
    var = r[0];
    bool go = n_obs - k_used > pl && r[0] > 0.0;
#pragma unroll
    for (int j = 1; j <= AR_MAX; ++j) {
      if (go && j <= pl) {
        double num = r[j];
#pragma unroll
        for (int i = 1; i < j; ++i) num -= phi[i - 1] * r[j - i];
        const double kap = num / var;
        if (fabs(kap) >= (double)MMF_AR_KAPPA_MAX) {
          go = false;
        } else {
          double nxt[AR_MAX];
#pragma unroll
          for (int i = 1; i < j; ++i) nxt[i - 1] = phi[i - 1] - kap * phi[j - i - 1];
#pragma unroll
          for (int i = 1; i < j; ++i) phi[i - 1] = nxt[i - 1];
          phi[j - 1] = kap;
          var *= 1.0 - kap * kap;
          order = j;
        }
      }
    }
  }
  float f[AR_MAX];
#pragma unroll
  for (int j = 0; j < AR_MAX; ++j) f[j] = (float)phi[j];
  int pb;                                  // order of pass B: the chosen candidate's
  {
    // ---- scoring walk: candidate lane j forecasts the held-out rows dynamically from origin t_fit with its own
    // coefficients and history u (e on observed fit rows, its own AR prediction elsewhere; held-out y never enters),
    // from the aligned chunk that holds s0h - p, with pass B's fmaf order
    __shared__ int s_wlo;
    if (threadIdx.x == 0) s_wlo = INT32_MAX;
    __syncthreads();
    const int hend = t_fit + sel.n_hold;
    const int w0 = max(s0h - p, 0) & ~31;
    if (work && lane == 0) atomicMin(&s_wlo, w0);
    __syncthreads();
    const int wlo = s_wlo;
    float h[AR_MAX];                       // h[k] = u_{s-1-k} of this lane's candidate
#pragma unroll
    for (int k = 0; k < AR_MAX; ++k) h[k] = 0.f;
    double sse = 0.0;
    int cnt = 0;
    for (int c0 = wlo & ~(TC - 1); c0 < hend; c0 += TC) {
      stage(s_a, s_nz, d, ar, c0);
      __syncthreads();
      if (work) {
#pragma unroll 1
        for (int t0 = max(c0, w0); t0 < min(c0 + TC, hend); t0 += 32) {
          const int s = t0 + lane;
          const float fit = fitted(s_a, s - c0, g, c);
          const float yv = s < hend ? __ldg(yr + s) : 0.f;     // y is never read at or beyond t_fit + n_hold
          const bool obs = s < t_fit && finite_f(yv);
          const float e = obs ? yv - fit : 0.f;
          const uint32_t bal = __ballot_sync(0xffffffffu, obs);
          const int jn = min(32, hend - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            float pr = 0.f;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < pl) pr = fmaf(f[k], h[k], pr);
            const float ej = __shfl_sync(0xffffffffu, e, j);
            const float fj = __shfl_sync(0xffffffffu, fit, j);
            const float yj = __shfl_sync(0xffffffffu, yv, j);
            const bool oj = (bal >> j) & 1u;
            float v = (oj || t0 + j < s0h) ? (oj ? ej : 0.f) : pr;
            if (t0 + j >= t_fit) {                               // held-out row: score the dynamic forecast
              const float fc = fj + pr;
              if (finite_f(yj) && finite_f(fc)) {
                const double dd = (double)yj - (double)fc;
                sse = fma(dd, dd, sse);
                ++cnt;
              }
#ifdef MMF_ARSEL_ONE_STEP
              // negative control: the observed held-out residual enters the history, a leaky one-step-ahead score
              if (finite_f(yj)) v = yj - fj;
#endif
            }
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) h[k] = h[k - 1];
            h[0] = v;
          }
        }
      }
      __syncthreads();
    }
    const double mse = cnt > 0 ? sse / (double)cnt : dnan();
    // ---- choice: the first minimum in list order; no scored point: the last candidate
    int win = -1;
    double best = 0.0;
    for (int j = 0; j < sel.n_cand; ++j) {
      const double v = __shfl_sync(0xffffffffu, mse, j);
      if (!isnan(v) && (win < 0 || v < best)) { best = v; win = j; }
    }
    if (win < 0) win = sel.n_cand - 1;
#pragma unroll
    for (int k = 0; k < AR_MAX; ++k) f[k] = __shfl_sync(0xffffffffu, f[k], win);
    order = __shfl_sync(0xffffffffu, order, win);
    var = __shfl_sync(0xffffffffu, var, win);
    pb = __shfl_sync(0xffffffffu, pl, win);
    const double mse_win = __shfl_sync(0xffffffffu, mse, win);
    if (live) {
      if (sel.cand_mse != nullptr && lane < sel.n_cand) sel.cand_mse[row * sel.n_cand + lane] = (float)mse;
      if (lane == 0) {
        if (sel.choice != nullptr) sel.choice[row] = work ? pb : -1;
        if (sel.mse != nullptr) sel.mse[row] = (float)mse_win;
      }
    }
  }
  if (live) {
    store_row(ar.phi, row, lane, f);
    if (lane == 0) {
      if (ar.order != nullptr) ar.order[row] = order;
      if (ar.sigma != nullptr) ar.sigma[row] = (float)sqrt(var);
    }
    if (!work)                                                   // empty series: NaN predictions, as the plain call
      for (int k = lane; k < a.n_pred; k += 32) a.out[row * a.ld_out + k] = __int_as_float(0x7fc00000);
  }

  // ---- pass B from the aligned chunk that holds s0 - p: every state pass B needs is a plain residual
  const int b0 = max(s0 - pb, 0) & ~31;
  if (work && lane == 0) atomicMin(&s_lo, b0);
  __syncthreads();
  const int lo = s_lo;
  float uprev = 0.f;                       // filled residuals u of the previous 32 rows
  for (int c0 = lo & ~(TC - 1); c0 < end; c0 += TC) {
    stage(s_a, s_nz, d, ar, c0);
    __syncthreads();
    if (work) {
#pragma unroll 1
      for (int t0 = max(c0, b0); t0 < min(c0 + TC, end); t0 += 32) {
        const int s = t0 + lane;
        const float fit = fitted(s_a, s - c0, g, c);
        const float yv = s < t_fit ? __ldg(yr + s) : 0.f;        // y is never read at or beyond t_fit
        const bool obs = s < t_fit && finite_f(yv);
        const float e = obs ? yv - fit : 0.f;
        const uint32_t bal = __ballot_sync(0xffffffffu, obs);
        const int nb = s0 - t0;                                  // lanes below nb lie before s0
        const uint32_t before = nb >= 32 ? 0xffffffffu : (nb <= 0 ? 0u : (1u << nb) - 1u);
        float u, arv = 0.f;
        if ((bal | before) == 0xffffffffu) {                     // no missing value at or after s0: all parallel
          u = e;
#pragma unroll
          for (int k = 1; k <= AR_MAX; ++k)
            if (k <= pb) arv = fmaf(f[k - 1], lagged(u, uprev, k, lane), arv);
        } else {                                                 // fill (item 5) runs serially over the chunk
          float h[AR_MAX];
#pragma unroll
          for (int k = 0; k < AR_MAX; ++k) h[k] = __shfl_sync(0xffffffffu, uprev, 31 - k);   // h[k] = u_{t0-1-k}
          u = 0.f;
          // only the positions up to the last requested row are needed; the chain is p long (phi_k = 0 beyond p)
          const int jn = min(32, end - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            float pr = 0.f;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < pb) pr = fmaf(f[k], h[k], pr);
            const float ej = __shfl_sync(0xffffffffu, e, j);
            const bool oj = (bal >> j) & 1u;
#ifdef MMF_AR_NO_FILL
            // negative control: a missing fit-window residual counts as 0 instead of its AR prediction
            const float v = (oj || t0 + j < s0 || t0 + j < t_fit) ? (oj ? ej : 0.f) : pr;
#else
            const float v = (oj || t0 + j < s0) ? (oj ? ej : 0.f) : pr;
#endif
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) h[k] = h[k - 1];
            h[0] = v;
            if (lane == j) { u = v; arv = pr; }
          }
        }
        uprev = u;
        if (s >= a.pred_start && s < end) a.out[row * a.ld_out + (s - a.pred_start)] = fit + arv;
      }
    }
    __syncthreads();
  }
}

}  // namespace

cudaError_t launch_ar(const DesignView& d, const FitArgs& a, const ArArgs& ar, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;
  ar_kernel<<<(unsigned)grid, THREADS, 0, s>>>(d, a, ar);
  return cudaGetLastError();
}

cudaError_t launch_ar_select(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArSelArgs& sel,
                             cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;
  ar_select_kernel<<<(unsigned)grid, THREADS, 0, s>>>(d, a, ar, sel);
  return cudaGetLastError();
}

}  // namespace mmf
