// arima.cu -- regression with ARIMA(p, d, 0) errors (DESIGN.md section 2 item 11, section 4.15), behind
// mmf_fit_forecast_arima_f32.  Per slab:
//   diff_kernel   writes the differenced series z'_s = Delta^d y_{s+d}, s in [0, t_fit - d), into a pitched scratch
//                 buffer (round4(t_fit - d) floats per row, so fit_tc's TMA path applies);
//   the fit passes run on z' with the plan of the differenced design D_d and hand gamma / c over (FitArgs::out_gamma);
//   arima_kernel  ar_kernel's pass A and Levinson-Durbin on z', and its pass B extended by the level state: the AR part
//                 gives zhat (the prediction of z'), which is integrated to the level prediction yhat with the filled
//                 levels ytilde (observed y on the fit rows, yhat elsewhere).
// arima_kernel is a kernel of its own, not a template of ar_kernel: wrapping ar_kernel moved its register allocation
// (section 4.14).  The z-space AR part and the level integration are separate steps of pass B, so a selecting variant can
// score every (p, d) candidate on levels: arima_select_kernel (section 2 item 12, section 4.16), behind
// mmf_fit_select_arima_f32.
#include "ar_common.cuh"

namespace mmf {
namespace {

// one warp per row, lanes over s: z' in the stated fp32 order; any non-finite level gives a non-finite z
__global__ void __launch_bounds__(THREADS)
diff_kernel(const ArimaArgs ma, float* __restrict__ z, int64_t ld_z, int64_t n) {
  const int64_t row = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (row >= n) return;
  const int lane = threadIdx.x & 31;
  const float* __restrict__ yr = ma.y + row * ma.ld_y;
  float* __restrict__ zr = z + row * ld_z;
  const int tz = ma.t_fit - ma.d;
  if (ma.d == 1) {
    for (int s = lane; s < tz; s += 32) zr[s] = __fsub_rn(__ldg(yr + s + 1), __ldg(yr + s));
  } else {
    for (int s = lane; s < tz; s += 32) {
      const float y0 = __ldg(yr + s), y1 = __ldg(yr + s + 1), y2 = __ldg(yr + s + 2);
      zr[s] = __fsub_rn(__fsub_rn(y2, y1), __fsub_rn(y1, y0));
    }
  }
}

// d.t_fit, d.n_rows: the differenced plan (t_fit - dd, n_rows - dd); a.y / a.ld_y: z'; a.pred_start / n_pred / out /
// ld_out: the caller's level rows
__global__ void __launch_bounds__(THREADS, 3)
arima_kernel(const DesignView d, const FitArgs a, const ArArgs ar, const ArimaArgs ma) {
  __shared__ float4 s_a[4][TC];
  __shared__ uint32_t s_nz[TC];
  __shared__ int s_lo;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * WARPS + warp;
  const bool live = row < a.n;
  const int p = ar.p;
  const int pm = max(p, 1);                // restart rule: max(p, 1) observed predecessors in z' (p = 0: the levels')
  const int dd = ma.d;
  const int t_fit = d.t_fit;               // z' fit rows
  const int T = ma.t_fit;                  // level fit rows
  const int end = a.pred_start + a.n_pred; // level rows [pred_start, end)
  const int endz = end - dd;               // z' rows whose prediction is a requested level
  const int S = min(a.pred_start, T) - dd; // the latest restart: no later than the first requested level's z' row
  if (threadIdx.x == 0) s_lo = INT32_MAX;

  float g[P], c;
  const int st = load_fit(a, row, live, g, c);
  const bool work = live && st != MMF_STATUS_EMPTY;
  const float* __restrict__ zr = a.y + (live ? row : 0) * a.ld_y;
  const float* __restrict__ yr = ma.y + (live ? row : 0) * ma.ld_y;

  // ---- pass A: residuals of z' over its fit rows, lag products, and the restart position s0 of pass B
  double acc[AR_MAX + 1];
#pragma unroll
  for (int k = 0; k <= AR_MAX; ++k) acc[k] = 0.0;
  float eprev = 0.f;                       // residuals of the previous 32 rows (positions < 0: 0)
  uint32_t bprev = 0xffffffffu;            // their observed bits (positions < 0 count as observed: u = 0 there)
  int s0 = 0, n_obs = 0;
  uint32_t colmask = 0u;                   // whitened columns with a non-zero entry on an observed fit row
  float ys[NSUB];
#pragma unroll
  for (int q = 0; q < NSUB; ++q) ys[q] = work && 32 * q + lane < t_fit ? __ldg(zr + 32 * q + lane) : 0.f;
  for (int c0 = 0; c0 < t_fit; c0 += TC) {
    float yn[NSUB];
#pragma unroll
    for (int q = 0; q < NSUB; ++q) {
      const int t = c0 + TC + 32 * q + lane;
      yn[q] = work && t < t_fit ? __ldg(zr + t) : 0.f;
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
          // bit 32 + j of M: z' positions t0 + j - pm + 1 .. t0 + j all observed, i.e. z' row t0 + 1 + j may start pass
          // B.  z'_{s-1} observed means levels y_{s-1} .. y_{s+d-1} are, so the d levels the integration of row s needs
          // are plain observations (for p = 0 this is the extra condition on the levels)
          const uint64_t comb = ((uint64_t)bal << 32) | bprev;
          uint64_t M = comb;
#pragma unroll
          for (int k = 2; k <= AR_MAX; ++k)
            if (k <= pm) M &= comb << (k - 1);
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
    // empty series: every requested level; otherwise the requested levels t < d, which have no prediction
    const int n_nan = work ? min(a.n_pred, dd - a.pred_start) : a.n_pred;
    for (int k = lane; k < n_nan; k += 32) a.out[row * a.ld_out + k] = qnan();
  }

  // ---- pass B from the aligned chunk that holds s0 - p: every state pass B needs is a plain residual, and the level
  // state at s0 is made of observed levels
  const int b0 = max(s0 - p, 0) & ~31;
  if (work && lane == 0) atomicMin(&s_lo, b0);
  __syncthreads();
  const int lo = s_lo;
  float uprev = 0.f;                       // filled residuals u of the previous 32 rows
  // filled levels ytilde_{t-1}, ytilde_{t-2} before the warp's first level row t = b0 + dd (read as they are: their
  // chain restarts at s0 at the latest)
  float l1 = qnan(), l2 = qnan();
  if (work) {
    const int i1 = b0 + dd - 1, i2 = b0 + dd - 2;
    const float v1 = i1 >= 0 && i1 < T ? __ldg(yr + i1) : qnan();
    const float v2 = i2 >= 0 && i2 < T ? __ldg(yr + i2) : qnan();
    l1 = finite_f(v1) ? v1 : qnan();
    l2 = finite_f(v2) ? v2 : qnan();
  }
  for (int c0 = lo & ~(TC - 1); c0 < endz; c0 += TC) {
    stage(s_a, s_nz, d, ar, c0);
    __syncthreads();
    if (work) {
#pragma unroll 1
      for (int t0 = max(c0, b0); t0 < min(c0 + TC, endz); t0 += 32) {
        // -- z-space: ar_kernel's pass B on z'
        const int s = t0 + lane;
        const float fit = fitted(s_a, s - c0, g, c);
        const float yv = s < t_fit ? __ldg(zr + s) : 0.f;        // z' is never read at or beyond its t_fit
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
          const int jn = min(32, endz - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            float pr = 0.f;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < p) pr = fmaf(f[k], h[k], pr);
            const float ej = __shfl_sync(0xffffffffu, e, j);
            const bool oj = (bal >> j) & 1u;
            const float v = (oj || t0 + j < s0) ? (oj ? ej : 0.f) : pr;
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) h[k] = h[k - 1];
            h[0] = v;
            if (lane == j) { u = v; arv = pr; }
          }
        }
        uprev = u;
        const float zh = fit + arv;                              // zhat of level row t = s + dd

        // -- levels: yhat_t from zhat_t and the filled levels before t (y is never read at or beyond t_fit)
        const int t = s + dd;
        const float lv = t < T ? __ldg(yr + t) : 0.f;
        const bool lobs = t < T && finite_f(lv);
        const uint32_t lbal = __ballot_sync(0xffffffffu, lobs);
        float yh;
        if (lbal == 0xffffffffu) {                               // every level of the chunk observed: ytilde = y
          const float p1 = __shfl_up_sync(0xffffffffu, lv, 1), p2 = __shfl_up_sync(0xffffffffu, lv, 2);
          yh = integrate(zh, lane >= 1 ? p1 : l1, lane >= 2 ? p2 : (lane == 1 ? l1 : l2), dd);
          l1 = __shfl_sync(0xffffffffu, lv, 31);
          l2 = __shfl_sync(0xffffffffu, lv, 30);
        } else {                                                 // a filled level: the chain runs serially
          yh = 0.f;
          const int jn = min(32, endz - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            const float hj = integrate(__shfl_sync(0xffffffffu, zh, j), l1, l2, dd);
            const float yj = __shfl_sync(0xffffffffu, lv, j);
#ifdef MMF_ARIMA_NO_LEVEL_FILL
            // negative control: a missing fit value's level is the last level instead of its prediction
            const float nl = (lbal >> j) & 1u ? yj : (t0 + j + dd < T ? l1 : hj);
#else
            const float nl = (lbal >> j) & 1u ? yj : hj;
#endif
            if (lane == j) yh = hj;
            l2 = l1;
            l1 = nl;
          }
        }
        if (t >= a.pred_start && t < end) a.out[row * a.ld_out + (t - a.pred_start)] = yh;
      }
    }
    __syncthreads();
  }
}

// The (p, d) selecting variant behind mmf_fit_select_arima_f32 (section 2 item 12, section 4.16), launched once per listed
// d behind that d's fit.  ma.d = 0: a.y is y and the level step is the identity (ar_select_kernel's candidates); ma.d >= 1:
// a.y is z' (arima_kernel's).  arima_kernel's pass A with ar.p = the largest order; Levinson-Durbin on lane j with bound
// sel.cand[j]; a scoring walk in which every candidate lane carries its own z-space history and its own filled levels
// ytilde_{t-1}, ytilde_{t-2} and forecasts the held-out levels from origin T; the first minimum of this d, compared with
// the running best of the earlier d's; and, only when this d takes the lead, pass B with the winner (arima_kernel's, or
// ar_kernel's for d = 0, in the same fp32 order), which writes the predictions and phi / order / sigma / status.
__global__ void __launch_bounds__(THREADS, 3)
arima_select_kernel(const DesignView d, const FitArgs a, const ArArgs ar, const ArimaArgs ma, const ArimaSelArgs sel) {
  __shared__ float4 s_a[4][TC];
  __shared__ uint32_t s_nz[TC];
  __shared__ int s_lo;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * WARPS + warp;
  const bool live = row < a.n;
  const int p = ar.p;                      // the largest candidate order
  const int pm = max(p, 1);                // restart rule: max(p, 1) observed predecessors
  const int dd = ma.d;
  const int t_fit = d.t_fit;               // fit rows of a.y (z': T - dd)
  const int T = ma.t_fit;                  // level fit rows
  const int end = a.pred_start + a.n_pred;
  const int endz = end - dd;
  const int S = min(a.pred_start, T) - dd;
  const bool first = sel.d_index == 0;
  if (threadIdx.x == 0) s_lo = INT32_MAX;

  float g[P], c;
  const int st = load_fit(a, row, live, g, c);
  const bool work = live && st != MMF_STATUS_EMPTY;     // eligible: the fit this d builds on is not empty
  const float* __restrict__ zr = a.y + (live ? row : 0) * a.ld_y;
  const float* __restrict__ yr = ma.y + (live ? row : 0) * ma.ld_y;

  // ---- pass A: residuals of a.y over its fit rows, lag products, the restart position s0 of pass B and s0h of the
  // scoring walk (the same rule with the bound t_fit)
  double acc[AR_MAX + 1];
#pragma unroll
  for (int k = 0; k <= AR_MAX; ++k) acc[k] = 0.0;
  float eprev = 0.f;
  uint32_t bprev = 0xffffffffu;
  int s0 = 0, s0h = 0, n_obs = 0;
  uint32_t colmask = 0u;
  float ys[NSUB];
#pragma unroll
  for (int q = 0; q < NSUB; ++q) ys[q] = work && 32 * q + lane < t_fit ? __ldg(zr + 32 * q + lane) : 0.f;
  for (int c0 = 0; c0 < t_fit; c0 += TC) {
    float yn[NSUB];
#pragma unroll
    for (int q = 0; q < NSUB; ++q) {
      const int t = c0 + TC + 32 * q + lane;
      yn[q] = work && t < t_fit ? __ldg(zr + t) : 0.f;
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
        // bit 32 + j of M: positions t0 + j - pm + 1 .. t0 + j all observed, i.e. position t0 + 1 + j may start a walk
        const uint64_t comb = ((uint64_t)bal << 32) | bprev;
        uint64_t M = comb;
#pragma unroll
        for (int k = 2; k <= AR_MAX; ++k)
          if (k <= pm) M &= comb << (k - 1);
        const uint32_t ok = (uint32_t)(M >> 32);
        if (t0 < S) {
          uint32_t okb = ok;
          const int jmax = S - t0 - 1 + LATE_RESTART;            // t0 + 1 + j <= S
          if (jmax < 31) okb &= (2u << jmax) - 1u;
          if (okb) s0 = t0 + 1 + (31 - __clz(okb));
        }
        {
          uint32_t okh = ok;
          const int jmax = t_fit - t0 - 1;                       // t0 + 1 + j <= t_fit
          if (jmax < 31) okh &= (2u << jmax) - 1u;
          if (okh) s0h = t0 + 1 + (31 - __clz(okh));
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
  const int k_used = used_columns(d, colmask, st, g);
  int pl = sel.cand[0];                    // lanes >= n_cand repeat the last candidate
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

  int pb;                                  // order of pass B: the winner's
  bool lead;                               // this d takes the lead (warp-uniform)
  {
    // ---- scoring walk: candidate lane j forecasts the held-out levels [T, T + n_hold) dynamically from origin T with
    // its own coefficients, z-space history u and filled levels (held-out y enters neither), from the aligned chunk
    // that holds s0h - p, with pass B's fp32 order
    __shared__ int s_wlo;
    if (threadIdx.x == 0) s_wlo = INT32_MAX;
    __syncthreads();
    const int hend = T + sel.n_hold;       // level rows read: [0, hend)
    const int hendz = hend - dd;
    const int w0 = max(s0h - p, 0) & ~31;
    if (work && lane == 0) atomicMin(&s_wlo, w0);
    __syncthreads();
    const int wlo = s_wlo;
    float h[AR_MAX];                       // h[k] = u_{s-1-k} of this lane's candidate
#pragma unroll
    for (int k = 0; k < AR_MAX; ++k) h[k] = 0.f;
    float l1 = qnan(), l2 = qnan();        // this lane's filled levels ytilde_{t-1}, ytilde_{t-2}
    if (work && dd > 0) {
      const int i1 = w0 + dd - 1, i2 = w0 + dd - 2;
      const float v1 = i1 >= 0 && i1 < T ? __ldg(yr + i1) : qnan();
      const float v2 = i2 >= 0 && i2 < T ? __ldg(yr + i2) : qnan();
      l1 = finite_f(v1) ? v1 : qnan();
      l2 = finite_f(v2) ? v2 : qnan();
    }
    double sse = 0.0;
    int cnt = 0;
    for (int c0 = wlo & ~(TC - 1); c0 < hendz; c0 += TC) {
      stage(s_a, s_nz, d, ar, c0);
      __syncthreads();
      if (work) {
#pragma unroll 1
        for (int t0 = max(c0, w0); t0 < min(c0 + TC, hendz); t0 += 32) {
          const int s = t0 + lane;
          const float fit = fitted(s_a, s - c0, g, c);
          const float zv = s < t_fit ? __ldg(zr + s) : 0.f;      // a.y is never read at or beyond its t_fit
          const bool obs = s < t_fit && finite_f(zv);
          const float e = obs ? zv - fit : 0.f;
          const uint32_t bal = __ballot_sync(0xffffffffu, obs);
          const float lv = s + dd < hend ? __ldg(yr + s + dd) : 0.f;   // y is never read at or beyond T + n_hold
          const int jn = min(32, hendz - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            float pr = 0.f;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < pl) pr = fmaf(f[k], h[k], pr);
            const float ej = __shfl_sync(0xffffffffu, e, j);
            const float fj = __shfl_sync(0xffffffffu, fit, j);
            const float yj = __shfl_sync(0xffffffffu, lv, j);
            const bool oj = (bal >> j) & 1u;
            const float v = (oj || t0 + j < s0h) ? (oj ? ej : 0.f) : pr;
            const float zh = fj + pr;
            const float hj = dd == 0 ? zh : integrate(zh, l1, l2, dd);
            const int tj = t0 + j + dd;                          // level row
            if (tj >= T) {                                       // held-out row: score the dynamic forecast
              if (finite_f(yj) && finite_f(hj)) {
                const double df = (double)yj - (double)hj;
                sse = fma(df, df, sse);
                ++cnt;
              }
            }
#ifdef MMF_ARIMASEL_ONE_STEP
            // negative control: an observed held-out level enters the level chain, a leaky one-step-ahead score
            const float nl = finite_f(yj) ? yj : hj;
#else
            const float nl = tj < T && finite_f(yj) ? yj : hj;
#endif
            l2 = l1;
            l1 = nl;
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) h[k] = h[k - 1];
            h[0] = v;
          }
        }
      }
      __syncthreads();
    }
    const double mse = cnt > 0 ? sse / (double)cnt : dnan();
    // ---- this d's first minimum in list order (no scored point: its last candidate), then the running best
    int win = -1;
    double best = 0.0;
    for (int j = 0; j < sel.n_cand; ++j) {
      const double v = __shfl_sync(0xffffffffu, mse, j);
      if (!isnan(v) && (win < 0 || v < best)) { best = v; win = j; }
    }
    const bool scored = win >= 0;
    if (win < 0) win = sel.n_cand - 1;
    ArimaSelBest rb{0.0, -1, -1, 0};       // the running best of the earlier d's
    if (live && !first) rb = sel.best[row];
    // the first minimum over the list (d ascending, then p): a later d leads only with a strictly smaller MSE; with no
    // scored point anywhere so far, the last eligible candidate leads
    const bool had = (rb.flags & ARIMASEL_SCORED) != 0;
    lead = work && (scored ? (!had || best < rb.mse) : !had);
#pragma unroll
    for (int k = 0; k < AR_MAX; ++k) f[k] = __shfl_sync(0xffffffffu, f[k], win);
    order = __shfl_sync(0xffffffffu, order, win);
    var = __shfl_sync(0xffffffffu, var, win);
    pb = __shfl_sync(0xffffffffu, pl, win);
    const double mse_win = __shfl_sync(0xffffffffu, mse, win);
    if (live) {
      if (sel.cand_mse != nullptr && lane < sel.n_cand)
        sel.cand_mse[(row * sel.n_diffs + sel.d_index) * sel.n_cand + lane] = (float)mse;
      if (lane == 0 && (first || work)) {
        if (lead) { rb.mse = best; rb.p = (int16_t)pb; rb.d = (int16_t)dd; }
        if (work) rb.flags |= ARIMASEL_ELIGIBLE | (scored ? ARIMASEL_SCORED : 0);
        sel.best[row] = rb;
      }
      // the first d writes every output of every row (NaN, -1, order 0, phi 0 where it is not eligible); a later d
      // only the rows it leads
      if (lane == 0 && (first || lead)) {
        if (sel.choice_p != nullptr) sel.choice_p[row] = lead ? pb : -1;
        if (sel.choice_d != nullptr) sel.choice_d[row] = lead ? dd : -1;
        if (sel.mse != nullptr) sel.mse[row] = lead ? (float)mse_win : qnan();
      }
    }
  }
  if (live && (first || lead)) {
    store_row(ar.phi, row, lane, f);
    if (lane == 0) {
      if (ar.order != nullptr) ar.order[row] = order;
      if (ar.sigma != nullptr) ar.sigma[row] = (float)sqrt(var);
      if (sel.status != nullptr) sel.status[row] = st;
    }
    // not eligible: every requested level; otherwise the requested levels t < d, which have no prediction
    const int n_nan = lead ? min(a.n_pred, dd - a.pred_start) : a.n_pred;
    for (int k = lane; k < n_nan; k += 32) a.out[row * a.ld_out + k] = qnan();
  }

  // ---- pass B with the winner, for the rows this d leads: arima_kernel's (ar_kernel's for d = 0) from the aligned chunk
  // that holds s0 - pb
  const bool wb = lead;
  const int b0 = max(s0 - pb, 0) & ~31;
  if (wb && lane == 0) atomicMin(&s_lo, b0);
  __syncthreads();
  const int lo = s_lo;
  float uprev = 0.f;
  float l1 = qnan(), l2 = qnan();
  if (wb && dd > 0) {
    const int i1 = b0 + dd - 1, i2 = b0 + dd - 2;
    const float v1 = i1 >= 0 && i1 < T ? __ldg(yr + i1) : qnan();
    const float v2 = i2 >= 0 && i2 < T ? __ldg(yr + i2) : qnan();
    l1 = finite_f(v1) ? v1 : qnan();
    l2 = finite_f(v2) ? v2 : qnan();
  }
  for (int c0 = lo & ~(TC - 1); c0 < endz; c0 += TC) {
    stage(s_a, s_nz, d, ar, c0);
    __syncthreads();
    if (wb) {
#pragma unroll 1
      for (int t0 = max(c0, b0); t0 < min(c0 + TC, endz); t0 += 32) {
        const int s = t0 + lane;
        const float fit = fitted(s_a, s - c0, g, c);
        const float yv = s < t_fit ? __ldg(zr + s) : 0.f;
        const bool obs = s < t_fit && finite_f(yv);
        const float e = obs ? yv - fit : 0.f;
        const uint32_t bal = __ballot_sync(0xffffffffu, obs);
        const int nb = s0 - t0;
        const uint32_t before = nb >= 32 ? 0xffffffffu : (nb <= 0 ? 0u : (1u << nb) - 1u);
        float u, arv = 0.f;
        if ((bal | before) == 0xffffffffu) {
          u = e;
#pragma unroll
          for (int k = 1; k <= AR_MAX; ++k)
            if (k <= pb) arv = fmaf(f[k - 1], lagged(u, uprev, k, lane), arv);
        } else {
          float h[AR_MAX];
#pragma unroll
          for (int k = 0; k < AR_MAX; ++k) h[k] = __shfl_sync(0xffffffffu, uprev, 31 - k);
          u = 0.f;
          const int jn = min(32, endz - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            float pr = 0.f;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < pb) pr = fmaf(f[k], h[k], pr);
            const float ej = __shfl_sync(0xffffffffu, e, j);
            const bool oj = (bal >> j) & 1u;
            const float v = (oj || t0 + j < s0) ? (oj ? ej : 0.f) : pr;
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) h[k] = h[k - 1];
            h[0] = v;
            if (lane == j) { u = v; arv = pr; }
          }
        }
        uprev = u;
        const float zh = fit + arv;
        const int t = s + dd;
        float yh = zh;                                           // d = 0: the level step is the identity
        if (dd > 0) {
          const float lv = t < T ? __ldg(yr + t) : 0.f;
          const bool lobs = t < T && finite_f(lv);
          const uint32_t lbal = __ballot_sync(0xffffffffu, lobs);
          if (lbal == 0xffffffffu) {
            const float p1 = __shfl_up_sync(0xffffffffu, lv, 1), p2 = __shfl_up_sync(0xffffffffu, lv, 2);
            yh = integrate(zh, lane >= 1 ? p1 : l1, lane >= 2 ? p2 : (lane == 1 ? l1 : l2), dd);
            l1 = __shfl_sync(0xffffffffu, lv, 31);
            l2 = __shfl_sync(0xffffffffu, lv, 30);
          } else {
            yh = 0.f;
            const int jn = min(32, endz - t0);
#pragma unroll 1
            for (int j = 0; j < jn; ++j) {
              const float hj = integrate(__shfl_sync(0xffffffffu, zh, j), l1, l2, dd);
              const float yj = __shfl_sync(0xffffffffu, lv, j);
              const float nl = (lbal >> j) & 1u ? yj : hj;
              if (lane == j) yh = hj;
              l2 = l1;
              l1 = nl;
            }
          }
        }
        if (t >= a.pred_start && t < end) a.out[row * a.ld_out + (t - a.pred_start)] = yh;
      }
    }
    __syncthreads();
  }
}

}  // namespace

cudaError_t launch_diff(const ArimaArgs& ma, float* z, int64_t ld_z, int64_t n, int sm_count, cudaStream_t s) {
  (void)sm_count;
  if (n <= 0) return cudaSuccess;
  const int64_t grid = (n + WARPS - 1) / WARPS;
  diff_kernel<<<(unsigned)grid, THREADS, 0, s>>>(ma, z, ld_z, n);
  return cudaGetLastError();
}

cudaError_t launch_arima(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;
  arima_kernel<<<(unsigned)grid, THREADS, 0, s>>>(d, a, ar, ma);
  return cudaGetLastError();
}

cudaError_t launch_arima_select(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                                const ArimaSelArgs& sel, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;
  arima_select_kernel<<<(unsigned)grid, THREADS, 0, s>>>(d, a, ar, ma, sel);
  return cudaGetLastError();
}

}  // namespace mmf
