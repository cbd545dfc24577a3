// arma_css.cu -- conditional least squares for regression with ARIMA(p, d, q) errors (DESIGN.md section 2 item 16,
// section 4.20), behind mmf_fit_forecast_arma_css_f32.  Per slab, after the whole HR call (fit passes, ar_kernel /
// arima_kernel, arma_kernel), which leaves every row's outputs and the Hannan-Rissanen (phi, theta) of the gated rows:
//   arma_css_kernel  Levenberg-Marquardt on S(x) = sum over C of eps~_s(x)^2, one warp per gated series, from x0 = the
//     HR estimate.  One pass reads the fit window once and evaluates S, g = J' eps~ and H = J'J at an fp32 point:
//       the recursion runs serially over the rows in float64 on every lane (u~, eps~ histories); lane i < p + q carries
//       the derivatives of u~ and eps~ by parameter i, so row s's Jacobian row J_s is spread over the lanes and goes
//       to shared memory with eps~_s; after each 32 rows the lanes accumulate the (p + q + 1)-square system [H g; g' S]
//       over the rows of C, about three entries per lane, each one sequential float64 FMA in row order;
//     the step: on lane 0, the in-order float64 Cholesky of H + lambda diag H, a trial point x' = fp32(x + delta) that
//       must pass the step-down tests, lambda x 10 until one does;
//     pass B: the rows that accepted a step run arma_kernel's pass B with the new (phi, theta); the others keep the HR
//       call's outputs bit for bit (their sigma excepted).
// The staging, fitted, load_fit, step_down_ok, integrate and the helpers come from ar_common.cuh; pass B is arma_kernel's,
// written out again (as a shared function it changed arma_kernel's code, DESIGN.md 4.17).
// arma_css_kernel is arma_css_kernel_t<false>.  The refit of a (p, d, q) selection's winners (section 4.22) runs
// refit_list_kernel, then arma_css_list_kernel, which is arma_css_kernel_t<true>: the same kernel over that list, with
// each row's own (p, q).
#include "ar_common.cuh"

namespace mmf {
namespace {

constexpr int NPAR = AR_MAX + MA_MAX;      // parameters (phi, theta)
constexpr int NENT = 96;                   // [H g; g' S] upper triangle, (p + q + 1)(p + q + 2) / 2 <= 91: 3 per lane
static_assert((NPAR + 1) * (NPAR + 2) / 2 <= NENT, "three Gram entries per lane");

// STOP codes of out_css_stop
constexpr int CSS_CONVERGED = 1, CSS_STALLED = 2, CSS_BUDGET = 3;

// packed index of entry (i, j), i <= j, of the (p + q + 1)-square system, column-major upper triangle
__device__ __forceinline__ int ent(int i, int j) { return j * (j + 1) / 2 + i; }

// lane 0: a trial point for (H + lam diag H) delta = -g, lam x 10 until the Cholesky pivots and the step-down tests
// pass; false when lam passes MMF_CSS_LAMBDA_MAX first.  H / g packed in hg, x the accepted point, xt the trial point,
// W an nreg x nreg work space (lower triangle of the factor).
__device__ bool css_step(const double* __restrict__ hg, const float* __restrict__ x, float* __restrict__ xt,
                         double* __restrict__ W, int p, int q, double& lam) {
  const int nreg = p + q;
  for (; lam <= (double)MMF_CSS_LAMBDA_MAX; lam *= 10.0) {
    bool ok = true;
    double diag[NPAR], w[NPAR];
    for (int j = 0; j < nreg && ok; ++j) {
      const double ajj = fma(lam, hg[ent(j, j)], hg[ent(j, j)]);
      double dj = ajj;
      for (int k = 0; k < j; ++k) dj -= W[j * NPAR + k] * W[j * NPAR + k];
      if (!(dj > (double)MMF_HR_PIVOT_TOL * ajj)) { ok = false; break; }
      diag[j] = sqrt(dj);
      for (int i = j + 1; i < nreg; ++i) {
#ifdef MMF_ARMACSS_DIAG_STEP
        double v = 0.0;                    // control build: diag(H) only, the off-diagonal entries ignored
#else
        double v = hg[ent(j, i)];
#endif
        for (int k = 0; k < j; ++k) v -= W[i * NPAR + k] * W[j * NPAR + k];
        W[i * NPAR + j] = v / diag[j];
      }
    }
    if (!ok) continue;
    for (int i = 0; i < nreg; ++i) {
      double v = -hg[ent(i, nreg)];
      for (int k = 0; k < i; ++k) v -= W[i * NPAR + k] * w[k];
      w[i] = v / diag[i];
    }
    for (int i = nreg - 1; i >= 0; --i) {
      double v = w[i];
      for (int k = i + 1; k < nreg; ++k) v -= W[k * NPAR + i] * w[k];
      w[i] = v / diag[i];
    }
    double fa[AR_MAX], fm[MA_MAX];
    for (int i = 0; i < nreg; ++i) xt[i] = (float)((double)x[i] + w[i]);
    for (int i = 0; i < p; ++i) fa[i] = (double)xt[i];
    for (int i = 0; i < q; ++i) fm[i] = -(double)xt[p + i];
    if (step_down_ok(fa, p) && step_down_ok(fm, q)) return true;
  }
  return false;
}

// d.t_fit: fit rows of a.y (z' for d >= 1); ma: the levels (ma.d = 0: ma.y is a.y); ar.p / hr.q: the orders; ar.phi,
// hr.theta, hr.ma_order: the HR call's outputs (caller buffers or scratch, never null here).  LIST: the rows of a
// (p, d, q) selection whose winner has q >= 1 and this d (the refit of DESIGN.md section 4.22).  Warp li takes row
// rf.rows[li] while li < *rf.count, at the orders that row's winner ships (ar.order, hr.ma_order; ar.p / hr.q are the
// call's largest listed orders); every other operation is the fixed-order kernel's, so that each row's outputs are the
// fixed-order CSS call's at its (p, d, q) bit for bit.  Warps past the count join the CTA's staging and __syncthreads_or
// as dead rows.  rf comes last and the fixed-order kernel never reads it, so that its parameter offsets and code stay
// those of a kernel without rf (scripts/compare_sass.py checks the code).
template <bool LIST>
__global__ void __launch_bounds__(THREADS, 1)
arma_css_kernel_t(const DesignView d, const FitArgs a, const ArArgs ar, const ArimaArgs ma, const ArmaArgs hr,
                  const CssArgs cs, const RefitArgs rf) {
  if constexpr (LIST) {
    if ((int64_t)blockIdx.x * WARPS >= (int64_t)*rf.count) return;   // a CTA past the list: uniform exit
  }
  __shared__ float4 s_a[4][TC];
  __shared__ uint32_t s_nz[TC];
  __shared__ double s_j[WARPS][32 * NPAR]; // J rows of the current 32 rows (row-major); the step's work space after a pass
  __shared__ double s_eps[WARPS][32];      // eps~ of the current 32 rows
  __shared__ double s_hg[WARPS][NENT];     // [H g; g' S] of the accepted point
  __shared__ float s_x[WARPS][2][NPAR];    // the accepted point and the trial point
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t li = (int64_t)blockIdx.x * WARPS + warp;
  const bool live = LIST ? li < (int64_t)*rf.count : li < a.n;
  const int64_t row = LIST ? (live ? (int64_t)rf.rows[li] : 0) : li;
#ifdef MMF_ARMASELCSS_CALL_ORDERS
  const int p = ar.p, q = hr.q;            // control build: every listed row at the call's largest listed (p, q)
#else
  const int p = LIST ? (live ? ar.order[row] : 0) : ar.p, q = LIST ? (live ? hr.ma_order[row] : 0) : hr.q;
#endif
  const int nreg = p + q;
  const int dd = ma.d;
  const int T = d.t_fit;                   // fit rows of a.y
  const int TL = ma.t_fit;                 // level fit rows
  const int end = a.pred_start + a.n_pred; // level rows [pred_start, end)
  const int endz = end - dd;
  double* __restrict__ sJ = s_j[warp];
  double* __restrict__ sX = s_eps[warp];
  float* __restrict__ xa = s_x[warp][0];
  float* __restrict__ xt = s_x[warp][1];

  float g[P], c;
  const int st = load_fit(a, row, live, g, c);
  const bool gated = live && st != MMF_STATUS_EMPTY && hr.ma_order[row] == q;
  const float* __restrict__ zr = a.y + (live ? row : 0) * a.ld_y;
  const float* __restrict__ yr = ma.y + (live ? row : 0) * ma.ld_y;
  if (gated && lane < nreg) xa[lane] = lane < p ? ar.phi[row * AR_MAX + lane] : hr.theta[row * MA_MAX + lane - p];
  if (lane < NPAR) xt[lane] = 0.f;
  __syncwarp();

  // this lane's entries of [H g; g' S]: index lane + 32 s, s < 3 (column-major upper triangle, S last)
  int ei[3], ej[3];
  {
    int idx = 0;
#pragma unroll
    for (int s = 0; s < 3; ++s) { ei[s] = -1; ej[s] = -1; }
    for (int j = 0; j <= nreg; ++j)
      for (int i = 0; i <= j; ++i) {
        const int s = (idx - lane) >> 5;
        if (idx >= lane && ((idx - lane) & 31) == 0 && s < 3) { ei[s] = i; ej[s] = j; }
        ++idx;
      }
  }
  const int idx_S = ent(nreg, nreg);

  // the LM state, the same on every lane
  bool active = gated;
  int passes = 0, n_acc = 0, stop = 0, n_C = 0;
  double S = 0.0, S0 = dnan(), lam = (double)MMF_CSS_LAMBDA0;
  double f[AR_MAX], th[MA_MAX];            // the point this pass evaluates
#pragma unroll
  for (int k = 0; k < AR_MAX; ++k) f[k] = gated && k < p ? (double)xa[k] : 0.0;
#pragma unroll
  for (int k = 0; k < MA_MAX; ++k) th[k] = gated && k < q ? (double)xa[p + k] : 0.0;

  while (__syncthreads_or(active)) {
    // ---- one pass: S, g and H at (f, th)
    double hu[AR_MAX], he[MA_MAX];         // u~_{s-1-k}, eps~_{s-1-k}
    double du[AR_MAX], de[MA_MAX];         // their derivatives by this lane's parameter (lane < nreg)
#pragma unroll
    for (int k = 0; k < AR_MAX; ++k) { hu[k] = 0.0; du[k] = 0.0; }
#pragma unroll
    for (int k = 0; k < MA_MAX; ++k) { he[k] = 0.0; de[k] = 0.0; }
    double gacc[3] = {0.0, 0.0, 0.0};
    bool gap_seen = false;                 // before the first missing row du = 0: the two-filter form
    int nc = 0;
    for (int c0 = 0; c0 < T; c0 += TC) {
      stage(s_a, s_nz, d, ar, c0);
      __syncthreads();
      if (active) {
#pragma unroll 1
        for (int t0 = c0; t0 < min(c0 + TC, T); t0 += 32) {
          const int s = t0 + lane;
          const float yv = s < T ? __ldg(zr + s) : 0.f;
          const bool obs = s < T && finite_f(yv);
          const float e = obs ? yv - fitted(s_a, s - c0, g, c) : 0.f;
          const uint32_t bal = __ballot_sync(0xffffffffu, obs);
          const double ed = (double)e;
          const int jn = min(32, T - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            double pr = 0.0;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < p) pr = fma(f[k], hu[k], pr);
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k)
              if (k < q) pr = fma(th[k], he[k], pr);
            // d pr / d x_lane: its own lag, then the lags of the derivatives
            double dpr = 0.0;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k) dpr = lane == k && k < p ? hu[k] : dpr;
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k) dpr = lane == p + k && k < q ? he[k] : dpr;
            if (gap_seen) {
#pragma unroll
              for (int k = 0; k < AR_MAX; ++k)
                if (k < p) dpr = fma(f[k], du[k], dpr);
            }
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k)
              if (k < q) dpr = fma(th[k], de[k], dpr);
            const double ej = __shfl_sync(0xffffffffu, ed, j);
            const bool oj = (bal >> j) & 1u;
            double uj, xj, duj, dej;
            if (oj) {                      // observed: u~ = e, eps~ = e - pr, d u~ = 0, d eps~ = -d pr
              uj = ej; xj = ej - pr; duj = 0.0; dej = -dpr;
            } else {                       // missing: u~ = pr, eps~ = 0, d u~ = d pr, d eps~ = 0
              uj = pr; xj = 0.0;
#ifdef MMF_ARMACSS_NO_GAP_JACOBIAN
              duj = 0.0; dej = -dpr;       // control build: the filled value taken as data (the two-filter form)
#else
              duj = dpr; dej = 0.0;
#endif
              gap_seen = true;
            }
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) { hu[k] = hu[k - 1]; du[k] = du[k - 1]; }
            hu[0] = uj; du[0] = duj;
#pragma unroll
            for (int k = MA_MAX - 1; k > 0; --k) { he[k] = he[k - 1]; de[k] = de[k - 1]; }
            he[0] = xj; de[0] = dej;
            if (lane < nreg) sJ[j * NPAR + lane] = dej;
            if (lane == 0) sX[j] = xj;
          }
          __syncwarp();
          // C: observed rows s >= p (bal is 0 at and beyond T)
          uint32_t cm = bal;
          if (p > t0) cm &= p - t0 >= 32 ? 0u : ~((1u << (p - t0)) - 1u);
          nc += __popc(cm);
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            if (ei[k] < 0) continue;
            const int ci = ei[k], cj = ej[k];
            const double* bi = ci == nreg ? sX : sJ + ci;
            const double* bj = cj == nreg ? sX : sJ + cj;
            const int si = ci == nreg ? 1 : NPAR, sj = cj == nreg ? 1 : NPAR;
            uint32_t rm = cm;
            double acc = gacc[k];
            while (rm) {
              const int j = __ffs(rm) - 1;
              rm &= rm - 1u;
              acc = fma(bi[j * si], bj[j * sj], acc);
            }
            gacc[k] = acc;
          }
          __syncwarp();
        }
      }
      __syncthreads();
    }
    if (!active) continue;                 // a warp that has stopped keeps its state while the others run on
    n_C = nc;

    // ---- accept or reject the point just evaluated, then the next trial point
    double mine = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) mine = k == (idx_S >> 5) ? gacc[k] : mine;
    const double Sn = __shfl_sync(0xffffffffu, mine, idx_S & 31);
    ++passes;
    bool take, conv = false;
    if (passes == 1) {
      take = true;
      S0 = Sn;
    } else {
      take = Sn < S;
      if (take) conv = S - Sn <= (double)MMF_CSS_RTOL * S;
    }
    if (take) {
      if (passes > 1) {
        ++n_acc;
        lam /= 10.0;
        if (lane < nreg) xa[lane] = xt[lane];
      }
      S = Sn;
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (ei[k] >= 0) s_hg[warp][ent(ei[k], ej[k])] = gacc[k];
    } else {
      lam *= 10.0;
    }
    __syncwarp();
    if (conv) stop = CSS_CONVERGED;
    else if (lam > (double)MMF_CSS_LAMBDA_MAX) stop = CSS_STALLED;
    else if (passes >= cs.max_iter) stop = CSS_BUDGET;
    if (stop == 0) {
      int ok = 0;
      if (lane == 0) ok = css_step(s_hg[warp], xa, xt, sJ, p, q, lam) ? 1 : 0;
      __syncwarp();
      ok = __shfl_sync(0xffffffffu, ok, 0);
      lam = __shfl_sync(0xffffffffu, lam, 0);
      if (!ok) stop = CSS_STALLED;
    }
    if (stop != 0) {
      active = false;
    } else {
#pragma unroll
      for (int k = 0; k < AR_MAX; ++k) f[k] = k < p ? (double)xt[k] : 0.0;
#pragma unroll
      for (int k = 0; k < MA_MAX; ++k) th[k] = k < q ? (double)xt[p + k] : 0.0;
    }
  }

  // ---- outputs: the objective columns of every live row, sigma of the gated rows, phi / theta of the refined rows
  if (live && lane == 0) {
    if (cs.css_start != nullptr) cs.css_start[row] = gated ? (float)S0 : qnan();
    if (cs.css != nullptr) cs.css[row] = gated ? (float)S : qnan();
    if (cs.css_stop != nullptr) cs.css_stop[row] = gated ? stop : 0;
    if (cs.iters != nullptr) cs.iters[row] = gated ? passes : 0;
    if (gated && ar.sigma != nullptr) ar.sigma[row] = (float)sqrt(S / (double)n_C);
  }
  const bool refined = gated && n_acc > 0;
  float fb[AR_MAX], tb[MA_MAX];
#pragma unroll
  for (int k = 0; k < AR_MAX; ++k) fb[k] = refined && k < p ? xa[k] : 0.f;
#pragma unroll
  for (int k = 0; k < MA_MAX; ++k) tb[k] = refined && k < q ? xa[p + k] : 0.f;
  if (refined) {
    store_row(ar.phi, row, lane, fb);
    store_row(hr.theta, row, lane, tb);
  }

  // ---- pass B (refined series): arma_kernel's, the recursion from s = 0 over the z-space rows [0, max(endz, T)),
  // integrated to levels; predictions only (sigma is the CSS one)
  if (!__syncthreads_or(refined)) return;
  const int endB = max(endz, T);
  float uprev = 0.f;                       // u of the previous 32 rows
  float hb[MA_MAX];                        // hb[k] = eps~_{s-1-k}, the same on every lane
#pragma unroll
  for (int k = 0; k < MA_MAX; ++k) hb[k] = 0.f;
  float l1 = qnan(), l2 = qnan();
  if (refined && dd > 0) {
    const int i1 = dd - 1, i2 = dd - 2;
    const float v1 = __ldg(yr + i1);
    const float v2 = i2 >= 0 ? __ldg(yr + i2) : qnan();
    l1 = finite_f(v1) ? v1 : qnan();
    l2 = finite_f(v2) ? v2 : qnan();
  }
  for (int c0 = 0; c0 < endB; c0 += TC) {
    stage(s_a, s_nz, d, ar, c0);
    __syncthreads();
    if (refined) {
#pragma unroll 1
      for (int t0 = c0; t0 < min(c0 + TC, endB); t0 += 32) {
        const int s = t0 + lane;
        const float fit = fitted(s_a, s - c0, g, c);
        const float yv = s < T ? __ldg(zr + s) : 0.f;            // never read at or beyond the fit rows
        const bool obs = s < T && finite_f(yv);
        const float e = obs ? yv - fit : 0.f;
        const uint32_t bal = __ballot_sync(0xffffffffu, obs);
        float u, pr;
        if (bal == 0xffffffffu) {                                // every row a fit row: AR part lane-parallel
          u = e;
          float arv = 0.f;
#pragma unroll
          for (int k = 1; k <= AR_MAX; ++k)
            if (k <= p) arv = fmaf(fb[k - 1], lagged(u, uprev, k, lane), arv);
          const float w = e - arv;                               // eps~_s = w_s - sum theta_k eps~_{s-k}
          float mav = 0.f;
#pragma unroll 1
          for (int j = 0; j < 32; ++j) {
            float mj = 0.f;
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k)
              if (k < q) mj = fmaf(tb[k], hb[k], mj);
            const float ej = __shfl_sync(0xffffffffu, w, j) - mj;
#pragma unroll
            for (int k = MA_MAX - 1; k > 0; --k) hb[k] = hb[k - 1];
            hb[0] = ej;
            if (lane == j) mav = mj;
          }
          pr = arv + mav;
        } else {                                                 // a missing or forecast row: all serial
          float hv[AR_MAX];
#pragma unroll
          for (int k = 0; k < AR_MAX; ++k) hv[k] = __shfl_sync(0xffffffffu, uprev, 31 - k);
          u = 0.f; pr = 0.f;
          const int jn = min(32, endB - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            float pj = 0.f;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < p) pj = fmaf(fb[k], hv[k], pj);
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k)
              if (k < q) pj = fmaf(tb[k], hb[k], pj);
            const float ej = __shfl_sync(0xffffffffu, e, j);
            const bool oj = (bal >> j) & 1u;
            const float uj = oj ? ej : pj;
            const float xj = oj ? ej - pj : 0.f;
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) hv[k] = hv[k - 1];
            hv[0] = uj;
#pragma unroll
            for (int k = MA_MAX - 1; k > 0; --k) hb[k] = hb[k - 1];
            hb[0] = xj;
            if (lane == j) { u = uj; pr = pj; }
          }
        }
        uprev = u;
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
}

// one thread per row of the slab, behind this d's fit (DESIGN.md section 4.22).  A row whose winner is (p, d, q >= 1), d
// this stage's, joins the list (warp-aggregated atomics: the list's order is arbitrary, and no output depends on it).  A
// row whose winner is (p, d, 0), and on the first stage a row with no eligible candidate, gets the refit outputs of a row
// no refit kernel touches: css_start, css NaN, css_stop, iters 0, and beta = W gamma (+ c on the intercept) of this d's
// fit in arma_joint_kernel's fp32 order (NaN for an empty fit and for a row with no winner).
__global__ void __launch_bounds__(256)
refit_list_kernel(const DesignView d, const FitArgs a, const ArimaArgs ma, const CssArgs cs, const JointArgs jt,
                  const RefitArgs rf) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool live = row < a.n;
  const int cd = live ? rf.choice_d[row] : -1, cq = live ? rf.choice_q[row] : -1;
  const bool listed = live && cd == ma.d && cq >= 1;
  const uint32_t bal = __ballot_sync(0xffffffffu, listed);
  uint32_t base = 0;
  if (lane == 0 && bal != 0u) base = atomicAdd(rf.count, (uint32_t)__popc(bal));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (listed) rf.rows[base + __popc(bal & ((1u << lane) - 1u))] = (int32_t)row;
  if (!live || listed || !(cd == ma.d || (rf.first && cd < 0))) return;
  if (cs.css_start != nullptr) cs.css_start[row] = qnan();
  if (cs.css != nullptr) cs.css[row] = qnan();
  if (cs.css_stop != nullptr) cs.css_stop[row] = 0;
  if (cs.iters != nullptr) cs.iters[row] = 0;
  if (jt.beta != nullptr) {
    float g[P], c;
    const int st = load_fit(a, row, cd == ma.d, g, c);
    for (int k = 0; k < P; ++k) {
      float b = (k == 0 && d.has_constant) ? c : 0.f;
#pragma unroll
      for (int j = 0; j < P; ++j) b = fmaf(__ldg(d.w + k * P + j), g[j], b);
      jt.beta[row * P + k] = st != MMF_STATUS_EMPTY ? b : qnan();
    }
  }
}

}  // namespace

cudaError_t launch_arma_css(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                            const ArmaArgs& hr, const CssArgs& cs, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;
  arma_css_kernel_t<false><<<(unsigned)grid, THREADS, 0, s>>>(d, a, ar, ma, hr, cs, RefitArgs{});
  return cudaGetLastError();
}

cudaError_t launch_arma_css_list(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                                 const ArmaArgs& hr, const CssArgs& cs, const RefitArgs& rf, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;          // the list's length is on the device: the slab's rows
  arma_css_kernel_t<true><<<(unsigned)grid, THREADS, 0, s>>>(d, a, ar, ma, hr, cs, rf);
  return cudaGetLastError();
}

cudaError_t launch_refit_list(const DesignView& d, const FitArgs& a, const ArimaArgs& ma, const CssArgs& cs,
                              const JointArgs& jt, const RefitArgs& rf, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  refit_list_kernel<<<(unsigned)((a.n + 255) / 256), 256, 0, s>>>(d, a, ma, cs, jt, rf);
  return cudaGetLastError();
}

}  // namespace mmf
