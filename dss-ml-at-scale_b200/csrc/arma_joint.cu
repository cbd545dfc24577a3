// arma_joint.cu -- regression with ARIMA(p, d, q) errors, beta estimated jointly with (phi, theta) by conditional least
// squares (DESIGN.md section 2 item 17, section 4.21), behind mmf_fit_forecast_arma_joint_f32.  Per slab, after the whole
// HR call (fit passes, ar_kernel / arima_kernel, arma_kernel), which leaves every row's outputs, the fit's gamma / c and
// the Hannan-Rissanen (phi, theta) of the gated rows:
//   arma_joint_kernel  arma_css_kernel's Levenberg-Marquardt with the whitened coefficients gamma_j of the series' used
//     columns J added to the parameter vector, x = (phi, theta, gamma_J), from x0 = (HR, the fit's gamma).  The residual
//     e_s = z'_s - fitted(a_s, gamma, c) is recomputed in fp32 at every pass's gamma (c held fixed); lane i < n_x carries
//     parameter i's derivative histories, a gamma lane reading a_{s,j} from the staged chunk.  The (n_x + 1)-square
//     system [H g; g' S] (at most 435 entries, 14 per lane) accumulates in shared memory after every 32 rows, each
//     entry one sequential float64 FMA chain in row order; the step's Cholesky is spread over the lanes (lane i owns
//     row i of the factor) with every entry computed by arma_css.cu's css_step operations in its order, so that with J
//     empty every output is the CSS call's bit for bit;
//   pass B: the rows that accepted a step run arma_kernel's pass B at the shipped (gamma, phi, theta); the others keep
//     the HR call's outputs bit for bit (their sigma excepted).  out_beta = W gamma (+ c on the intercept) for every
//     non-empty row, in the fit kernels' fmaf order.
// The negative-control build (-DMMF_ARMAJOINT_WHITE_BETA) drops the recursion from the gamma columns of the Jacobian,
// d eps~_s = -a_{s,j} on observed rows and 0 elsewhere (the regression derivative as if the errors were white).
// arma_joint_kernel is arma_joint_kernel_t<false>.  The joint refit of a (p, d, q) selection's winners (section 4.22) runs
// arma_joint_list_kernel, which is arma_joint_kernel_t<true>: the same kernel over arma_css.cu's refit list, with each
// row's own (p, q).
#include "ar_common.cuh"

namespace mmf {
namespace {

constexpr int NPAR = AR_MAX + MA_MAX;      // parameters (phi, theta)
constexpr int NX = NPAR + P;               // ... and gamma on at most P used columns
static_assert(NX <= 28, "one lane per parameter, (p + q <= 12) + (16 columns) <= 28");
constexpr int NENT = (NX + 1) * (NX + 2) / 2;   // [H g; g' S] upper triangle: 435 entries
constexpr int EPL = (NENT + 31) / 32;           // entries per lane: 14
static_assert(EPL == 14, "fourteen Gram entries per lane");

// CSS stop codes of out_css_stop (arma_css.cu's)
constexpr int CSS_CONVERGED = 1, CSS_STALLED = 2, CSS_BUDGET = 3;

// one warp's shared memory
struct JointWarp {
  double j[32 * NX];                       // J rows of the current 32 rows (row stride NX); the factor during a step
  double eps[32];                          // eps~ of the current 32 rows
  double acc[NENT];                        // [H g; g' S] of the point being evaluated
  double hg[NENT];                         // ... of the accepted point
  double w[NX];                            // the solves' vector
  double diag[NX];                         // the factor's diagonal
  float x[2][NX];                          // the accepted point and the trial point
};
struct JointSmem {
  float4 a[4][TC];                         // the staged chunk (ar_common's stage)
  uint32_t nz[TC];
  JointWarp w[WARPS];
};
static_assert(NX * NX <= 32 * NX, "the factor fits in the J rows");
static_assert(offsetof(JointSmem, w) % 16 == 0 && sizeof(JointWarp) % 8 == 0, "aligned per-warp blocks");
constexpr size_t JOINT_SMEM = sizeof(JointSmem);   // the kernel's fixed dynamic shared memory, every launch
static_assert(JOINT_SMEM <= 227 * 1024, "one CTA per SM");

// packed index of entry (i, j), i <= j, of the (n_x + 1)-square system, column-major upper triangle (arma_css.cu's)
__device__ __forceinline__ int ent(int i, int j) { return j * (j + 1) / 2 + i; }

// a trial point for (H + lam diag H) delta = -g, lam x 10 until the Cholesky pivots and the step-down tests on the
// (phi, theta) part pass; false when lam passes MMF_CSS_LAMBDA_MAX first.  Every lane runs the loop; lane i builds row i
// of the factor (ws.j, row stride NX), every lane forms the pivots (the same value on every lane), lane 0 solves.  Each
// entry is css_step's expression in css_step's order.
__device__ bool joint_step(JointWarp& ws, int p, int q, int nx, double& lam, int lane) {
  double* __restrict__ W = ws.j;
  const double* __restrict__ hg = ws.hg;
  for (; lam <= (double)MMF_CSS_LAMBDA_MAX; lam *= 10.0) {
    bool ok = true;
    for (int j = 0; j < nx; ++j) {
      const double ajj = fma(lam, hg[ent(j, j)], hg[ent(j, j)]);
      double dj = ajj;
      for (int k = 0; k < j; ++k) dj -= W[j * NX + k] * W[j * NX + k];
      if (!(dj > (double)MMF_HR_PIVOT_TOL * ajj)) { ok = false; break; }
      const double dg = sqrt(dj);
      const int i = lane;
      if (i > j && i < nx) {
        double v = hg[ent(j, i)];
        for (int k = 0; k < j; ++k) v -= W[i * NX + k] * W[j * NX + k];
        W[i * NX + j] = v / dg;
      }
      if (lane == 0) ws.diag[j] = dg;
      __syncwarp();
    }
    if (!ok) { __syncwarp(); continue; }
    int good = 0;
    if (lane == 0) {
      double* __restrict__ w = ws.w;
      const double* __restrict__ diag = ws.diag;
      for (int i = 0; i < nx; ++i) {
        double v = -hg[ent(i, nx)];
        for (int k = 0; k < i; ++k) v -= W[i * NX + k] * w[k];
        w[i] = v / diag[i];
      }
      for (int i = nx - 1; i >= 0; --i) {
        double v = w[i];
        for (int k = i + 1; k < nx; ++k) v -= W[k * NX + i] * w[k];
        w[i] = v / diag[i];
      }
      const float* __restrict__ x = ws.x[0];
      float* __restrict__ xt = ws.x[1];
      double fa[AR_MAX], fm[MA_MAX];
      for (int i = 0; i < nx; ++i) xt[i] = (float)((double)x[i] + w[i]);
      for (int i = 0; i < p; ++i) fa[i] = (double)xt[i];
      for (int i = 0; i < q; ++i) fm[i] = -(double)xt[p + i];
      good = step_down_ok(fa, p) && step_down_ok(fm, q) ? 1 : 0;
    }
    good = __shfl_sync(0xffffffffu, good, 0);
    __syncwarp();
    if (good) return true;
  }
  return false;
}

// gamma with the gamma lanes of point xp placed on the used columns (jmask ascending)
__device__ __forceinline__ void place_gamma(float (&g)[P], const float* __restrict__ xp, int nreg, uint32_t jmask) {
#pragma unroll
  for (int k = 0; k < P; ++k)
    if ((jmask >> k) & 1u) g[k] = xp[nreg + __popc(jmask & ((1u << k) - 1u))];
}

// d.t_fit: fit rows of a.y (z' for d >= 1); ma: the levels (ma.d = 0: ma.y is a.y); ar.p / hr.q: the orders; ar.phi,
// hr.theta, hr.ma_order: the HR call's outputs (caller buffers or scratch, never null here).  LIST: the rows of a
// (p, d, q) selection whose winner has q >= 1 and this d (DESIGN.md section 4.22), each at its winner's orders, by
// arma_css_kernel_t's rules for LIST and rf.
template <bool LIST>
__global__ void __launch_bounds__(THREADS, 1)
arma_joint_kernel_t(const DesignView d, const FitArgs a, const ArArgs ar, const ArimaArgs ma, const ArmaArgs hr,
                    const CssArgs cs, const JointArgs jt, const RefitArgs rf) {
  if constexpr (LIST) {
    if ((int64_t)blockIdx.x * WARPS >= (int64_t)*rf.count) return;   // a CTA past the list: uniform exit
  }
  extern __shared__ __align__(16) unsigned char smem_raw[];
  JointSmem& sm = *reinterpret_cast<JointSmem*>(smem_raw);
  float4 (*s_a)[TC] = sm.a;
  uint32_t* s_nz = sm.nz;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  JointWarp& ws = sm.w[warp];
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
  double* __restrict__ sJ = ws.j;
  double* __restrict__ sX = ws.eps;
  float* __restrict__ xa = ws.x[0];
  float* __restrict__ xt = ws.x[1];

  float g[P], c;
  const int st = load_fit(a, row, live, g, c);
  const bool gated = live && st != MMF_STATUS_EMPTY && hr.ma_order[row] == q;
  const float* __restrict__ zr = a.y + (live ? row : 0) * a.ld_y;
  const float* __restrict__ yr = ma.y + (live ? row : 0) * ma.ld_y;

  // J: the used columns of the dof rule, from one scan of the observed fit rows
  uint32_t colmask = 0u;
  for (int c0 = 0; c0 < T; c0 += TC) {
    if (threadIdx.x < TC) s_nz[threadIdx.x] = c0 + (int)threadIdx.x < d.n_rows ? __ldg(ar.nz + c0 + threadIdx.x) : 0u;
    __syncthreads();
    if (gated) {
#pragma unroll 1
      for (int s = c0 + lane; s < min(c0 + TC, T); s += 32)
        if (finite_f(__ldg(zr + s))) colmask |= s_nz[s - c0];
    }
    __syncthreads();
  }
  const uint32_t jmask = gated ? used_mask(d, colmask, st, g) : 0u;
  const int nx = nreg + __popc(jmask);
  int gcol = -1;                           // this lane's design column (gamma lanes nreg <= lane < nx)
  {
    int k = lane - nreg;
#pragma unroll
    for (int j = 0; j < P; ++j)
      if ((jmask >> j) & 1u) { if (k == 0) gcol = j; --k; }
  }
  if (gated && lane < nreg) xa[lane] = lane < p ? ar.phi[row * AR_MAX + lane] : hr.theta[row * MA_MAX + lane - p];
  if (gated && gcol >= 0) {
    float v = 0.f;
#pragma unroll
    for (int j = 0; j < P; ++j) v = gcol == j ? g[j] : v;
    xa[lane] = v;
  }
  if (lane < NX) xt[lane] = 0.f;
  __syncwarp();
  const int nent = (nx + 1) * (nx + 2) / 2;
  const int idx_S = ent(nx, nx);

  // the LM state, the same on every lane
  bool active = gated;
  int passes = 0, n_acc = 0, stop = 0, n_C = 0;
  double S = 0.0, S0 = dnan(), lam = (double)MMF_CSS_LAMBDA0;
  double f[AR_MAX], th[MA_MAX];            // the point this pass evaluates (and g: its gamma)
#pragma unroll
  for (int k = 0; k < AR_MAX; ++k) f[k] = gated && k < p ? (double)xa[k] : 0.0;
#pragma unroll
  for (int k = 0; k < MA_MAX; ++k) th[k] = gated && k < q ? (double)xa[p + k] : 0.0;

  while (__syncthreads_or(active)) {
    // ---- one pass: S, g and H at (f, th, g)
    double hu[AR_MAX], he[MA_MAX];         // u~_{s-1-k}, eps~_{s-1-k}
    double du[AR_MAX], de[MA_MAX];         // their derivatives by this lane's parameter (lane < nx)
#pragma unroll
    for (int k = 0; k < AR_MAX; ++k) { hu[k] = 0.0; du[k] = 0.0; }
#pragma unroll
    for (int k = 0; k < MA_MAX; ++k) { he[k] = 0.0; de[k] = 0.0; }
    if (active)
      for (int e = lane; e < nent; e += 32) ws.acc[e] = 0.0;
    bool gap_seen = false;                 // before the first missing row du = 0 on the (phi, theta) lanes
    const bool glane = gcol >= 0;          // gamma lanes: du is never 0 on them
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
          const float* arow = reinterpret_cast<const float*>(&s_a[glane ? gcol >> 2 : 0][t0 - c0]) + (gcol & 3);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            double pr = 0.0;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < p) pr = fma(f[k], hu[k], pr);
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k)
              if (k < q) pr = fma(th[k], he[k], pr);
            // d pr / d x_lane: its own lag ((phi, theta) lanes), then the lags of the derivatives
            double dpr = 0.0;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k) dpr = lane == k && k < p ? hu[k] : dpr;
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k) dpr = lane == p + k && k < q ? he[k] : dpr;
            if (gap_seen || glane) {
#pragma unroll
              for (int k = 0; k < AR_MAX; ++k)
                if (k < p) dpr = fma(f[k], du[k], dpr);
            }
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k)
              if (k < q) dpr = fma(th[k], de[k], dpr);
            const double ej = __shfl_sync(0xffffffffu, ed, j);
            const bool oj = (bal >> j) & 1u;
            const double av = glane ? (double)arow[4 * j] : 0.0;   // a_{s,j} of this lane's column (float4 rows)
            double uj, xj, duj, dej;
            if (oj) {                      // observed: u~ = e, eps~ = e - pr, d u~ = -a (gamma) or 0, d eps~ = d u~ - d pr
              uj = ej; xj = ej - pr;
#ifdef MMF_ARMAJOINT_WHITE_BETA
              duj = 0.0; dej = glane ? -av : -dpr;   // control build: the gamma columns as if the errors were white
#else
              duj = glane ? -av : 0.0; dej = glane ? -av - dpr : -dpr;
#endif
            } else {                       // missing: u~ = pr, eps~ = 0, d u~ = d pr, d eps~ = 0
              uj = pr; xj = 0.0;
#ifdef MMF_ARMAJOINT_WHITE_BETA
              duj = glane ? 0.0 : dpr; dej = 0.0;
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
            if (lane < nx) sJ[j * NX + lane] = dej;
            if (lane == 0) sX[j] = xj;
          }
          __syncwarp();
          // C: observed rows s >= p (bal is 0 at and beyond T)
          uint32_t cm = bal;
          if (p > t0) cm &= p - t0 >= 32 ? 0u : ~((1u << (p - t0)) - 1u);
          nc += __popc(cm);
          // this lane's entries lane + 32 k of [H g; g' S], (ci, cj) walked along the packed order
          int ci = lane, cj = 0;
          while (ci > cj) { ci -= cj + 1; ++cj; }
#pragma unroll 1
          for (int k = 0; k < EPL; ++k) {
            const int e = lane + 32 * k;
            if (e >= nent) break;
            const double* bi = ci == nx ? sX : sJ + ci;
            const double* bj = cj == nx ? sX : sJ + cj;
            const int si = ci == nx ? 1 : NX, sj = cj == nx ? 1 : NX;
            uint32_t rm = cm;
            double acc = ws.acc[e];
            while (rm) {
              const int jr = __ffs(rm) - 1;
              rm &= rm - 1u;
              acc = fma(bi[jr * si], bj[jr * sj], acc);
            }
            ws.acc[e] = acc;
            ci += 32;
            while (ci > cj) { ci -= cj + 1; ++cj; }
          }
          __syncwarp();
        }
      }
      __syncthreads();
    }
    if (!active) continue;                 // a warp that has stopped keeps its state while the others run on
    n_C = nc;

    // ---- accept or reject the point just evaluated, then the next trial point
    const double Sn = ws.acc[idx_S];
    ++passes;
    bool take, conv = false;
    if (passes == 1) {
      take = true;
      S0 = Sn;
    } else {
      take = Sn < S;
      if (take) conv = S - Sn <= (double)MMF_CSS_RTOL * S;
    }
    __syncwarp();
    if (take) {
      if (passes > 1) {
        ++n_acc;
        lam /= 10.0;
        if (lane < nx) xa[lane] = xt[lane];
      }
      S = Sn;
      for (int e = lane; e < nent; e += 32) ws.hg[e] = ws.acc[e];
    } else {
      lam *= 10.0;
    }
    __syncwarp();
    if (conv) stop = CSS_CONVERGED;
    else if (lam > (double)MMF_CSS_LAMBDA_MAX) stop = CSS_STALLED;
    else if (passes >= cs.max_iter) stop = CSS_BUDGET;
    if (stop == 0 && !joint_step(ws, p, q, nx, lam, lane)) stop = CSS_STALLED;
    if (stop != 0) {
      active = false;
    } else {
#pragma unroll
      for (int k = 0; k < AR_MAX; ++k) f[k] = k < p ? (double)xt[k] : 0.0;
#pragma unroll
      for (int k = 0; k < MA_MAX; ++k) th[k] = k < q ? (double)xt[p + k] : 0.0;
      place_gamma(g, xt, nreg, jmask);
    }
  }

  // ---- outputs: the objective columns of every live row, sigma of the gated rows, phi / theta / gamma of the refined
  // rows, beta of every live row
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
  if (gated) load_fit(a, row, live, g, c);                        // the fit's gamma where no step was accepted
  if (refined) {
    store_row(ar.phi, row, lane, fb);
    store_row(hr.theta, row, lane, tb);
    place_gamma(g, xa, nreg, jmask);
  }
  if (live && jt.beta != nullptr && lane < P) {                     // beta = W gamma (+ c on the intercept)
    float b = (lane == 0 && d.has_constant) ? c : 0.f;
#pragma unroll
    for (int k = 0; k < P; ++k) b = fmaf(__ldg(d.w + lane * P + k), g[k], b);
    jt.beta[row * P + lane] = st != MMF_STATUS_EMPTY ? b : qnan();
  }

  // ---- pass B (refined series): arma_kernel's, the recursion from s = 0 over the z-space rows [0, max(endz, T)),
  // integrated to levels, at the shipped gamma; predictions only (sigma is the CSS one)
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

}  // namespace

cudaError_t launch_arma_joint(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                              const ArmaArgs& hr, const CssArgs& cs, const JointArgs& jt, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  // the attribute is per function and process-wide: always the kernel's fixed bound, so that a context on another host
  // thread cannot lower it between this call's set and its launch
  cudaError_t e =
      cudaFuncSetAttribute(arma_joint_kernel_t<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)JOINT_SMEM);
  if (e != cudaSuccess) return e;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;
  arma_joint_kernel_t<false><<<(unsigned)grid, THREADS, JOINT_SMEM, s>>>(d, a, ar, ma, hr, cs, jt, RefitArgs{});
  return cudaGetLastError();
}

cudaError_t launch_arma_joint_list(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                                   const ArmaArgs& hr, const CssArgs& cs, const JointArgs& jt, const RefitArgs& rf,
                                   cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  // always the kernel's fixed bound, never this call's own need (launch_arma_joint's reason)
  cudaError_t e =
      cudaFuncSetAttribute(arma_joint_kernel_t<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)JOINT_SMEM);
  if (e != cudaSuccess) return e;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;          // the list's length is on the device: the slab's rows
  arma_joint_kernel_t<true><<<(unsigned)grid, THREADS, JOINT_SMEM, s>>>(d, a, ar, ma, hr, cs, jt, rf);
  return cudaGetLastError();
}

}  // namespace mmf
