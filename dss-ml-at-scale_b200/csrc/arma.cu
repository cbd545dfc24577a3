// arma.cu -- regression with ARIMA(p, d, q) errors (DESIGN.md section 2 item 13, section 4.17), behind
// mmf_fit_forecast_arma_f32.  Per slab, after the fit passes (on y for d = 0, on z' for d >= 1, gamma / c hand-off) and
// after ar_kernel / arima_kernel with order p, which write every row's fallback outputs:
//   arma_kernel  Hannan-Rissanen on the residuals e of the fit, one warp per series:
//     pass A   residuals and r_0..r_m (lane k sums lag k + 1 in float64 from the staged residuals of this and the previous
//              32 rows), then Levinson-Durbin to order m with psi spread over the lanes;
//     pass A2  the filled long-AR residuals u^L, the innovation estimates eps^ and the float64 normal equations of the
//              regression of e_t on (e_{t-1..t-p}, eps^_{t-1..t-q}) over the rows R, about three entries per lane;
//     solve    in-order float64 Cholesky and the step-down tests on lane 0; a series that fails the gate keeps the
//              fallback outputs;
//     pass B   the ARMA recursion from s = 0 (never restarted: MA terms have infinite memory), integrated to levels as
//              arima_kernel does for d >= 1, for the gated series only.
// The fit hand-off load, the ring shift, the theta store and the small helpers come from ar_common.cuh.  The other blocks
// it shares with arma_select_kernel (pass A, step 1, the pass-A2 rings, the solve, pass B) stay written out here: as
// shared functions they changed this kernel's code, and the ARMA calls were measured about 1 % slower (DESIGN.md 4.17).
#include "ar_common.cuh"

// timing builds only (scripts/bench_arma.py --split): 1 ends the kernel after pass A and step 1, 2 after the solve
#ifndef MMF_ARMA_STOP_AFTER
#define MMF_ARMA_STOP_AFTER 0
#endif

namespace mmf {
namespace {

constexpr int NC = AR_MAX + MA_MAX + 1;    // regressors + target: columns of the staged normal equations

// d.t_fit: fit rows of a.y (z' for d >= 1); ma: the levels (ma.d = 0: ma.y is a.y); ar.p / hr.q / hr.m: the orders
__global__ void __launch_bounds__(THREADS, 3)
arma_kernel(const DesignView d, const FitArgs a, const ArArgs ar, const ArimaArgs ma, const ArmaArgs hr) {
  __shared__ float4 s_a[4][TC];
  __shared__ uint32_t s_nz[TC];
  // float64 rings: every product of passes A and A2 reads them as float64, so each value is converted once, on store
  __shared__ double s_e[WARPS][64];        // residuals e of the previous and the current 32 rows (0 where missing)
  __shared__ double s_u[WARPS][64];        // filled long-AR residuals u^L, same rows
  __shared__ double s_v[WARPS][64];        // innovation estimates eps^, same rows (0 where missing)
  __shared__ double s_psi[WARPS][32];      // psi_1..psi_32
  __shared__ double s_g[WARPS][NC * NC];   // normal equations [G b; b' .], regressor-major
  __shared__ float s_beta[WARPS][AR_MAX + MA_MAX];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * WARPS + warp;
  const bool live = row < a.n;
  const int p = ar.p, q = hr.q, m = hr.m;
  const int nreg = p + q;
  const int L = max(p, q);                 // lags a row of R needs observed
  const int dd = ma.d;
  const int T = d.t_fit;                   // fit rows of a.y
  const int TL = ma.t_fit;                 // level fit rows
  const int end = a.pred_start + a.n_pred; // level rows [pred_start, end)
  const int endz = end - dd;
  double* __restrict__ sE = s_e[warp];
  double* __restrict__ sU = s_u[warp];
  double* __restrict__ sV = s_v[warp];

  float g[P], c;
  const int st = load_fit(a, row, live, g, c);
  const bool work = live && st != MMF_STATUS_EMPTY;
  const float* __restrict__ zr = a.y + (live ? row : 0) * a.ld_y;
  const float* __restrict__ yr = ma.y + (live ? row : 0) * ma.ld_y;

  // ---- pass A: residuals, n_obs, used columns and r_0 (own lane), r_{lane+1} (lane k sums lag k + 1)
  sE[lane] = 0.0;
  double acc0 = 0.0, accl = 0.0;
  int n_obs = 0;
  uint32_t colmask = 0u;
  for (int c0 = 0; c0 < T; c0 += TC) {
    stage(s_a, s_nz, d, ar, c0);
    __syncthreads();
    if (work) {
#pragma unroll 1
      for (int t0 = c0; t0 < min(c0 + TC, T); t0 += 32) {
        const int t = t0 + lane;
        const float yv = t < T ? __ldg(zr + t) : 0.f;
        const bool obs = t < T && finite_f(yv);
        const float e = obs ? yv - fitted(s_a, t - c0, g, c) : 0.f;
        n_obs += __popc(__ballot_sync(0xffffffffu, obs));
        colmask |= obs ? s_nz[t - c0] : 0u;
        acc0 = fma((double)e, (double)e, acc0);
        const double ed = (double)e;
        sE[32 + lane] = ed;
        __syncwarp();
        if (lane < m) {
#pragma unroll 8
          for (int j = 0; j < 32; ++j) accl = fma(sE[32 + j], sE[31 + j - lane], accl);
        }
        __syncwarp();
        sE[lane] = ed;
        __syncwarp();
      }
    }
    __syncthreads();
  }

  // ---- step 1: Levinson-Durbin to order m with the kappa stop; lane i holds psi_{i+1} and r_{i+1}
  acc0 = warp_sum(acc0);
  colmask = __reduce_or_sync(0xffffffffu, colmask);
  uint32_t used = d.kept_mask & colmask;
  if (st == MMF_STATUS_RANKDEF) {
#pragma unroll
    for (int k = 0; k < P; ++k) used &= g[k] != 0.f ? ~0u : ~(1u << k);
  }
  const int k_used = __popc(used);
  double psi = 0.0;
  int m_i = 0;
  if (work) {
    const double inv = 1.0 / (double)max(n_obs, 1);
    const double r0 = acc0 * inv, rl = accl * inv;
    double var = r0;
    bool go = n_obs - k_used > m && r0 > 0.0;
    for (int j = 1; j <= m && go; ++j) {
      const double rr = __shfl_sync(0xffffffffu, rl, (j - lane - 2) & 31);     // r_{j - (lane + 1)}
      const double num = __shfl_sync(0xffffffffu, rl, j - 1) - warp_sum(lane + 1 < j ? psi * rr : 0.0);
      const double kap = num / var;
      if (fabs(kap) >= (double)MMF_AR_KAPPA_MAX) {
        go = false;
      } else {
        const double mirror = __shfl_sync(0xffffffffu, psi, (j - lane - 2) & 31);  // psi_{j - (lane + 1)}
        psi = lane + 1 < j ? psi - kap * mirror : (lane + 1 == j ? kap : psi);
        var *= 1.0 - kap * kap;
        m_i = j;
      }
    }
  }
  s_psi[warp][lane] = psi;

#if MMF_ARMA_STOP_AFTER == 1
  return;                                  // timing build: pass A and step 1 only
#endif
  // ---- pass A2: u^L, eps^, and the normal equations over R (lane owns entries lane, lane + 32, lane + 64 of the upper
  // triangle of the (nreg + 1)-square system, the target's own square excluded)
  bool hr_ok = work && m_i >= 1;
  int ei[3], ej[3];
  double gacc[3] = {0.0, 0.0, 0.0};
  {
    int idx = 0;
#pragma unroll
    for (int s = 0; s < 3; ++s) { ei[s] = -1; ej[s] = -1; }
    for (int j = 0; j <= nreg; ++j)
      for (int i = 0; i <= j; ++i) {
        if (i == nreg) continue;
        const int s = (idx - lane) >> 5;
        if (idx >= lane && ((idx - lane) & 31) == 0 && s < 3) { ei[s] = i; ej[s] = j; }
        ++idx;
      }
  }
  int n_R = 0;
  sE[lane] = 0.0; sU[lane] = 0.0; sV[lane] = 0.0;
  __syncwarp();
  const int r_lo = m + q;                  // first row of R
  uint32_t bprev = 0u;
  if (__syncthreads_or(hr_ok)) {
    for (int c0 = 0; c0 < T; c0 += TC) {
      stage(s_a, s_nz, d, ar, c0);
      __syncthreads();
      if (hr_ok) {
#pragma unroll 1
        for (int t0 = c0; t0 < min(c0 + TC, T); t0 += 32) {
          const int t = t0 + lane;
          const float yv = t < T ? __ldg(zr + t) : 0.f;
          const bool obs = t < T && finite_f(yv);
          const float e = obs ? yv - fitted(s_a, t - c0, g, c) : 0.f;
          const uint32_t bal = __ballot_sync(0xffffffffu, obs);
          const double ed = (double)e;
          sE[32 + lane] = ed;
          sU[32 + lane] = ed;
          __syncwarp();
          // missing fit rows of the chunk, in order: u^L_s = sum_k psi_k u^L_{s-k}
          uint32_t miss = ~bal;
          if (T - t0 < 32) miss &= (1u << (T - t0)) - 1u;
          while (miss) {
            const int j = __ffs(miss) - 1;
            miss &= miss - 1u;
            const double v = warp_sum(lane < m_i ? psi * sU[31 + j - lane] : 0.0);
            if (lane == 0) sU[32 + j] = v;
            __syncwarp();
          }
          double ve = 0.0;
          if (obs) {
            ve = ed;
            for (int k = 1; k <= m_i; ++k) ve = fma(-s_psi[warp][k - 1], sU[32 + lane - k], ve);
          }
          sV[32 + lane] = ve;
          // R: t >= m + q and t, t-1, .., t-L observed (the control build: t observed, missing lags enter as 0)
          const uint64_t comb = ((uint64_t)bal << 32) | bprev;
          uint64_t M = comb;
#ifndef MMF_ARMA_GAPPY_REGRESSION
          for (int k = 1; k <= L; ++k) M &= comb << k;
#endif
          uint32_t rmask = (uint32_t)(M >> 32);
          if (r_lo > t0) rmask &= r_lo - t0 >= 32 ? 0u : ~((1u << (r_lo - t0)) - 1u);
          n_R += __popc(rmask);
          __syncwarp();
#pragma unroll
          for (int s = 0; s < 3; ++s) {
            if (ei[s] < 0) continue;
            const int ci = ei[s], cj = ej[s];
            const double* bi = ci < p ? sE + 31 - ci : sV + 31 - (ci - p);
            const double* bj = cj == nreg ? sE + 32 : (cj < p ? sE + 31 - cj : sV + 31 - (cj - p));
            uint32_t rm = rmask;
            double acc = gacc[s];
            while (rm) {
              const int j = __ffs(rm) - 1;
              rm &= rm - 1u;
              acc = fma(bi[j], bj[j], acc);
            }
            gacc[s] = acc;
          }
          __syncwarp();
          hr_rings_shift(sE, sU, sV, ed);
          bprev = bal;
          __syncwarp();
        }
      }
      __syncthreads();
    }
  }

  // ---- step 2: in-order float64 Cholesky of G, beta = G^-1 b, and the gate (lane 0)
  double* G = s_g[warp];
#pragma unroll
  for (int s = 0; s < 3; ++s)
    if (ei[s] >= 0) { G[ei[s] * NC + ej[s]] = gacc[s]; G[ej[s] * NC + ei[s]] = gacc[s]; }
  __syncwarp();
  if (hr_ok && lane == 0) {
    bool ok = n_R > nreg;
    // L in the strict lower triangle and diag[] (G's upper triangle and last column stay as they are)
    double diag[AR_MAX + MA_MAX], w[AR_MAX + MA_MAX];
    for (int j = 0; j < nreg && ok; ++j) {
      double dj = G[j * NC + j];
      for (int k = 0; k < j; ++k) dj -= G[j * NC + k] * G[j * NC + k];
      if (!(dj > (double)MMF_HR_PIVOT_TOL * G[j * NC + j])) { ok = false; break; }
      diag[j] = sqrt(dj);
      for (int i = j + 1; i < nreg; ++i) {
        double v = G[j * NC + i];
        for (int k = 0; k < j; ++k) v -= G[i * NC + k] * G[j * NC + k];
        G[i * NC + j] = v / diag[j];
      }
    }
    if (ok) {
      for (int i = 0; i < nreg; ++i) {
        double v = G[i * NC + nreg];
        for (int k = 0; k < i; ++k) v -= G[i * NC + k] * w[k];
        w[i] = v / diag[i];
      }
      for (int i = nreg - 1; i >= 0; --i) {
        double v = w[i];
        for (int k = i + 1; k < nreg; ++k) v -= G[k * NC + i] * w[k];
        w[i] = v / diag[i];
      }
      double fa[AR_MAX], fm[MA_MAX];
      for (int i = 0; i < p; ++i) fa[i] = w[i];
      for (int i = 0; i < q; ++i) fm[i] = -w[p + i];
      ok = step_down_ok(fa, p) && step_down_ok(fm, q);
      for (int i = 0; i < nreg; ++i) s_beta[warp][i] = (float)w[i];
    }
    G[0] = ok ? 1.0 : 0.0;
  }
  __syncwarp();
  hr_ok = hr_ok && __shfl_sync(0xffffffffu, G[0], 0) != 0.0;

  float f[AR_MAX], th[MA_MAX];
#pragma unroll
  for (int k = 0; k < AR_MAX; ++k) f[k] = hr_ok && k < p ? s_beta[warp][k] : 0.f;
#pragma unroll
  for (int k = 0; k < MA_MAX; ++k) th[k] = hr_ok && k < q ? s_beta[warp][p + k] : 0.f;
  if (live) {
    store_row(hr.theta, row, lane, th);
    if (lane == 0 && hr.ma_order != nullptr) hr.ma_order[row] = hr_ok ? q : 0;
    if (hr_ok) {
      if (ar.phi != nullptr && lane < AR_MAX) {
        float v = 0.f;
#pragma unroll
        for (int k = 0; k < AR_MAX; ++k) v = lane == k ? f[k] : v;
        ar.phi[row * AR_MAX + lane] = v;
      }
      if (lane == 0 && ar.order != nullptr) ar.order[row] = p;
    }
  }

#if MMF_ARMA_STOP_AFTER == 2
  return;                                  // timing build: passes A, A2 and the solve only
#endif
  // ---- pass B (gated series): the recursion from s = 0 over the z-space rows [0, max(endz, T)) -- sigma needs every
  // fit row whatever the window -- integrated to levels
  if (!__syncthreads_or(hr_ok)) return;
  const int endB = max(endz, T);
  float uprev = 0.f;                       // u of the previous 32 rows
  float he[MA_MAX];                        // he[k] = eps~_{s-1-k}, the same on every lane
#pragma unroll
  for (int k = 0; k < MA_MAX; ++k) he[k] = 0.f;
  double sse = 0.0;
  bprev = 0u;
  float l1 = qnan(), l2 = qnan();
  if (hr_ok && dd > 0) {
    const int i1 = dd - 1, i2 = dd - 2;
    const float v1 = __ldg(yr + i1);
    const float v2 = i2 >= 0 ? __ldg(yr + i2) : qnan();
    l1 = finite_f(v1) ? v1 : qnan();
    l2 = finite_f(v2) ? v2 : qnan();
  }
  for (int c0 = 0; c0 < endB; c0 += TC) {
    stage(s_a, s_nz, d, ar, c0);
    __syncthreads();
    if (hr_ok) {
#pragma unroll 1
      for (int t0 = c0; t0 < min(c0 + TC, endB); t0 += 32) {
        const int s = t0 + lane;
        const float fit = fitted(s_a, s - c0, g, c);
        const float yv = s < T ? __ldg(zr + s) : 0.f;            // never read at or beyond the fit rows
        const bool obs = s < T && finite_f(yv);
        const float e = obs ? yv - fit : 0.f;
        const uint32_t bal = __ballot_sync(0xffffffffu, obs);
        float u, pr, eps = 0.f;
        if (bal == 0xffffffffu) {                                // every row a fit row: AR part lane-parallel
          u = e;
          float arv = 0.f;
#pragma unroll
          for (int k = 1; k <= AR_MAX; ++k)
            if (k <= p) arv = fmaf(f[k - 1], lagged(u, uprev, k, lane), arv);
          const float w = e - arv;                               // eps~_s = w_s - sum theta_k eps~_{s-k}
          float mav = 0.f;
#pragma unroll 1
          for (int j = 0; j < 32; ++j) {
            float mj = 0.f;
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k)
              if (k < q) mj = fmaf(th[k], he[k], mj);
            const float ej = __shfl_sync(0xffffffffu, w, j) - mj;
#pragma unroll
            for (int k = MA_MAX - 1; k > 0; --k) he[k] = he[k - 1];
            he[0] = ej;
            if (lane == j) { eps = ej; mav = mj; }
          }
          pr = arv + mav;
        } else {                                                 // a missing or forecast row: all serial
          float hu[AR_MAX];
#pragma unroll
          for (int k = 0; k < AR_MAX; ++k) hu[k] = __shfl_sync(0xffffffffu, uprev, 31 - k);
          u = 0.f; pr = 0.f;
          const int jn = min(32, endB - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            float pj = 0.f;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < p) pj = fmaf(f[k], hu[k], pj);
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k)
              if (k < q) pj = fmaf(th[k], he[k], pj);
            const float ej = __shfl_sync(0xffffffffu, e, j);
            const bool oj = (bal >> j) & 1u;
            const float uj = oj ? ej : pj;
            const float xj = oj ? ej - pj : 0.f;
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) hu[k] = hu[k - 1];
            hu[0] = uj;
#pragma unroll
            for (int k = MA_MAX - 1; k > 0; --k) he[k] = he[k - 1];
            he[0] = xj;
            if (lane == j) { u = uj; pr = pj; eps = xj; }
          }
        }
        uprev = u;
        if (t0 < T) {                                            // sigma: eps~ over R
          const uint64_t comb = ((uint64_t)bal << 32) | bprev;
          uint64_t M = comb;
#ifndef MMF_ARMA_GAPPY_REGRESSION
          for (int k = 1; k <= L; ++k) M &= comb << k;
#endif
          const bool inR = ((M >> (32 + lane)) & 1u) && s >= r_lo;
          if (inR) sse = fma((double)eps, (double)eps, sse);
          bprev = bal;
        }
        const float zh = fit + pr;
        const int t = s + dd;
        float yh = zh;                                           // d = 0: the level step is the identity
        if (dd > 0) {
          const float lv = t < TL ? __ldg(yr + t) : 0.f;         // y is never read at or beyond t_fit
          const bool lobs = t < TL && finite_f(lv);
          const uint32_t lbal = __ballot_sync(0xffffffffu, lobs);
          if (lbal == 0xffffffffu) {
            const float p1 = __shfl_up_sync(0xffffffffu, lv, 1), p2 = __shfl_up_sync(0xffffffffu, lv, 2);
            yh = integrate(zh, lane >= 1 ? p1 : l1, lane >= 2 ? p2 : (lane == 1 ? l1 : l2), dd);
            l1 = __shfl_sync(0xffffffffu, lv, 31);
            l2 = __shfl_sync(0xffffffffu, lv, 30);
          } else {
            yh = 0.f;
            const int jn = min(32, endB - t0);
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
  sse = warp_sum(sse);
  if (hr_ok && lane == 0 && ar.sigma != nullptr) ar.sigma[row] = (float)sqrt(sse / (double)n_R);
}

}  // namespace

cudaError_t launch_arma(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                        const ArmaArgs& hr, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;
  arma_kernel<<<(unsigned)grid, THREADS, 0, s>>>(d, a, ar, ma, hr);
  return cudaGetLastError();
}

}  // namespace mmf
