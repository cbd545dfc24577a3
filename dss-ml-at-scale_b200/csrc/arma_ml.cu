// arma_ml.cu -- ARIMA(p, d, q) errors by exact Gaussian likelihood (DESIGN.md section 2 item 19, section 4.23), behind
// mmf_fit_forecast_arma_ml_f32.  Per slab, after the whole CSS call (fit passes, ar_kernel / arima_kernel, arma_kernel,
// arma_css_kernel), which leaves every row's outputs and the CSS (phi, theta) of the gated rows:
//   arma_ml_kernel  Levenberg-Marquardt on the scaled innovations r_s = G v_s / sqrt(F_s) of a Kalman filter in Harvey's
//     state-space form, one warp per gated series, from x0 = the CSS estimate.  One pass:
//       P_0: the stationary state covariance and its derivatives, (I - T (x) T) vec P = vec(R R') on the r (r + 1) / 2
//         symmetric unknowns by Gaussian elimination with partial pivoting in shared memory, the lanes over columns;
//         the derivatives solve the same factorisation with the right-hand sides d(R R') + dT P T' + T P dT';
//       the filter: serial over the rows in float64.  Lane l < p + q carries d a / d x_l (registers) and d P / d x_l
//         (shared memory, its own slot of ws.X), lane p + q carries a and P: every carried pair moves by the same
//         expression X' = T X T' + W K' + K W' + Q R' + R Q' + c K K', each lane with its own (W, Q, c).  Row s's
//         Jacobian row D~_s = d(v_s / sqrt F_s) is spread over the lanes and goes to shared memory with v_s / sqrt F_s;
//         after each 32 rows the lanes accumulate the (p + q + 1)-square system [sum D~'D~, sum D~'v~; ., S_w] over the
//         observed rows, in row order, as arma_css_kernel does;
//       after the pass the factor G enters H and g as a rank-2 correction from sum dF / F (the common G^2 cancels in
//         the step).  The objective is G^2 S_w = n exp(L / n).
//     the step: arma_css_kernel's, and a trial point whose P_0 solve fails counts as a failed step-down (lam x 10).
//     pass B: the rows that accepted a step run arma_kernel's pass B with the new (phi, theta); the others keep the CSS
//       call's outputs bit for bit (their sigma excepted).
// ml_step and pass B are arma_css_kernel's, written out again (as shared functions they changed that kernel's code).
// arma_ml_kernel is arma_ml_kernel_t<false>.  The ML refit of a (p, d, q) selection's winners (mmf_fit_select_arma_ml_f32,
// section 4.25) runs arma_ml_list_kernel, which is arma_ml_kernel_t<true>: the same kernel over a list of rows with each
// row's own (p, q); refit_ml_cols_kernel writes the rows outside the list.
#include "ar_common.cuh"
#ifdef MMF_REFIT_ASSERT
#include <assert.h>
#endif

namespace mmf {
namespace {

constexpr int NPAR = AR_MAX + MA_MAX;      // parameters (phi, theta)
constexpr int NENT = 96;                   // [H g; g' S] upper triangle, (p + q + 1)(p + q + 2) / 2 <= 91: 3 per lane
static_assert((NPAR + 1) * (NPAR + 2) / 2 <= NENT, "three Gram entries per lane");
constexpr int RMAX = AR_MAX > MA_MAX + 1 ? AR_MAX : MA_MAX + 1;   // state dimension r = max(p, q + 1)
constexpr int NSYM = RMAX * (RMAX + 1) / 2;                        // symmetric unknowns of P
constexpr int NSLOT = 16;                  // carried covariances per warp: d P by parameter l < p + q, then P
static_assert(NPAR + 1 <= NSLOT, "one slot per carrying lane");
constexpr int AUGW = NSYM + 1 + NPAR;      // [A | P's right-hand side | the derivatives' right-hand sides]

// STOP codes of out_ml_stop (the CSS call's)
constexpr int ML_CONVERGED = 1, ML_STALLED = 2, ML_BUDGET = 3;

// one warp's shared memory
struct MlWarp {
  double j[32 * NPAR];                     // D~ rows of the current 32 rows (row-major); the step's work space
  double vt[32];                           // v / sqrt F of the current 32 rows
  double hg[NENT];                         // [H g; g' S] of the accepted point, G's correction applied
  double raw[NENT];                        // ... of the point just evaluated, before it
  double gam[NPAR];                        // sum dF / F / (2 n) of the point just evaluated
  double ph[RMAX], rv[RMAX];               // phi and R of the point being evaluated, padded to RMAX
  double X[NSYM * NSLOT];                  // carried covariances, packed entry e of slot l at e * NSLOT + l
  double aug[NSYM * AUGW];                 // the P_0 system, row-major
  int perm[NSYM];                          // its row exchanges
  float x[2][NPAR];                        // the accepted point and the trial point
};
struct MlSmem {
  float4 a[4][TC];                         // the staged chunk (ar_common's stage)
  uint32_t nz[TC];
  MlWarp w[WARPS];
};
static_assert(offsetof(MlSmem, w) % 16 == 0 && sizeof(MlWarp) % 8 == 0, "aligned per-warp blocks");
static_assert(NPAR * NPAR <= 32 * NPAR, "the factor fits in the D~ rows");
constexpr size_t ML_SMEM = sizeof(MlSmem);  // the kernel's fixed dynamic shared memory, every launch
static_assert(ML_SMEM <= 227 * 1024, "one CTA per SM");

// packed index of entry (i, j), i <= j, column-major upper triangle (arma_css.cu's)
__device__ __forceinline__ int ent(int i, int j) { return j * (j + 1) / 2 + i; }

// lane 0: arma_css.cu's css_step
__device__ bool ml_step(const double* __restrict__ hg, const float* __restrict__ x, float* __restrict__ xt,
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
        double v = hg[ent(j, i)];
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

// (i, j) of packed entry k
__device__ __forceinline__ void unpack(int k, int& i, int& j) {
  j = 0;
  while ((j + 1) * (j + 2) / 2 <= k) ++j;
  i = k - j * (j + 1) / 2;
}

// back substitution of column col of the eliminated system (one lane)
__device__ void back_sub(double* __restrict__ A, int N, int col) {
  for (int i = N - 1; i >= 0; --i) {
    double v = A[i * AUGW + col];
    for (int c = i + 1; c < N; ++c) v = fma(-A[i * AUGW + c], A[c * AUGW + col], v);
    A[i * AUGW + col] = v / A[i * AUGW + i];
  }
}

// the whole warp: P_0 into slot np of ws.X and d P_0 / d x_l into slot l < np, from ws.ph / ws.rv.  False (on every
// lane) when a pivot |u_kk| <= MMF_HR_PIVOT_TOL x max |A|.
__device__ bool p0_solve(MlWarp& ws, int r, int p, int np, int lane) {
  const int N = r * (r + 1) / 2;
  double* __restrict__ A = ws.aug;
  double amax = 0.0;
  for (int k = lane; k < N; k += 32) {     // row k: P_ij - (T P T')_ij = R_i R_j
    double* row = A + k * AUGW;
    for (int c = 0; c <= N; ++c) row[c] = 0.0;
    int i, j;
    unpack(k, i, j);
    const double pi = ws.ph[i], pj = ws.ph[j];
    row[k] += 1.0;
    row[0] -= pi * pj;
    if (j + 1 < r) {
      row[ent(0, j + 1)] -= pi;
      row[ent(i + 1, j + 1)] -= 1.0;
    }
    if (i + 1 < r) row[ent(0, i + 1)] -= pj;
    row[N] = ws.rv[i] * ws.rv[j];
    for (int c = 0; c < N; ++c) amax = fmax(amax, fabs(row[c]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  __syncwarp();
  for (int k = 0; k < N; ++k) {
    double best = -1.0;
    int bi = k;
    for (int i = k + lane; i < N; i += 32) {
      const double v = fabs(A[i * AUGW + k]);
      if (v > best) { best = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (!(best > (double)MMF_HR_PIVOT_TOL * amax)) return false;
    if (lane == 0) ws.perm[k] = bi;
    if (bi != k)
      for (int c = lane; c <= N; c += 32) {
        const double t = A[k * AUGW + c];
        A[k * AUGW + c] = A[bi * AUGW + c];
        A[bi * AUGW + c] = t;
      }
    __syncwarp();
    const double inv = 1.0 / A[k * AUGW + k];
    __syncwarp();
    for (int i = k + 1 + lane; i < N; i += 32) A[i * AUGW + k] *= inv;   // the multipliers
    __syncwarp();
    for (int c = k + 1 + lane; c <= N; c += 32) {
      const double akc = A[k * AUGW + c];
      for (int i = k + 1; i < N; ++i) A[i * AUGW + c] = fma(-A[i * AUGW + k], akc, A[i * AUGW + c]);
    }
    __syncwarp();
  }
  if (lane == np) {
    back_sub(A, N, N);
    for (int k = 0; k < N; ++k) ws.X[k * NSLOT + np] = A[k * AUGW + N];
  }
  __syncwarp();
  if (lane < np) {                         // right-hand side of parameter `lane`, then the same factorisation
    const int col = N + 1 + lane;
    const int ip = lane < p ? lane : -1, iq = lane < p ? -1 : lane - p + 1;
    const double P00 = A[N];
    for (int k = 0; k < N; ++k) {
      int i, j;
      unpack(k, i, j);
      const double mi = ws.ph[i] * P00 + (i + 1 < r ? A[ent(0, i + 1) * AUGW + N] : 0.0);   // (T P_0 Z')_i
      const double mj = ws.ph[j] * P00 + (j + 1 < r ? A[ent(0, j + 1) * AUGW + N] : 0.0);
      double v = 0.0;
      if (i == iq) v += ws.rv[j];
      if (j == iq) v += ws.rv[i];
      if (i == ip) v += mj;
      if (j == ip) v += mi;
      A[k * AUGW + col] = v;
    }
    for (int k = 0; k < N; ++k) {
      const int b = ws.perm[k];
      if (b != k) {
        const double t = A[k * AUGW + col];
        A[k * AUGW + col] = A[b * AUGW + col];
        A[b * AUGW + col] = t;
      }
    }
    for (int k = 0; k < N; ++k) {
      const double bk = A[k * AUGW + col];
      for (int i = k + 1; i < N; ++i) A[i * AUGW + col] = fma(-A[i * AUGW + k], bk, A[i * AUGW + col]);
    }
    back_sub(A, N, col);
    for (int k = 0; k < N; ++k) ws.X[k * NSLOT + lane] = A[k * AUGW + col];
  }
  __syncwarp();
  return true;
}

// d.t_fit: fit rows of a.y (z' for d >= 1); ma: the levels (ma.d = 0: ma.y is a.y); ar.p / hr.q: the orders; ar.phi,
// hr.theta, hr.ma_order: the CSS call's outputs (caller buffers or scratch, never null here).  LIST: the rows of a
// (p, d, q) selection whose winner has q >= 1 and this d (the ML refit of DESIGN.md section 4.25), behind the CSS list
// kernel on the same list, each at its winner's orders, by arma_css_kernel_t's rules for LIST and rf.  Warps past the
// count index nothing by p or q.
template <bool LIST>
__global__ void __launch_bounds__(THREADS, 1)
arma_ml_kernel_t(const DesignView d, const FitArgs a, const ArArgs ar, const ArimaArgs ma, const ArmaArgs hr,
                 const MlArgs ml, const RefitArgs rf) {
  if constexpr (LIST) {
    if ((int64_t)blockIdx.x * WARPS >= (int64_t)*rf.count) return;   // a CTA past the list: uniform exit
  }
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MlSmem& sm = *reinterpret_cast<MlSmem*>(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  MlWarp& ws = sm.w[warp];
  const int64_t li = (int64_t)blockIdx.x * WARPS + warp;
  const bool live = LIST ? li < (int64_t)*rf.count : li < a.n;
  const int64_t row = LIST ? (live ? (int64_t)rf.rows[li] : 0) : li;
#ifdef MMF_ARMASELML_CALL_ORDERS
  const int p = ar.p, q = hr.q;            // control build: every listed row at the call's largest listed (p, q)
#else
  const int p = LIST ? (live ? ar.order[row] : 0) : ar.p, q = LIST ? (live ? hr.ma_order[row] : 0) : hr.q;
#endif
#ifdef MMF_REFIT_ASSERT
  if constexpr (LIST) assert(!live || (row < a.n && p >= 0 && p <= AR_MAX && q >= 1 && q <= MA_MAX));
#endif
  const int nreg = p + q;
  const int r = max(p, q + 1);
  const int dd = ma.d;
  const int T = d.t_fit;                   // fit rows of a.y
  const int TL = ma.t_fit;                 // level fit rows
  const int end = a.pred_start + a.n_pred; // level rows [pred_start, end)
  const int endz = end - dd;
  float* __restrict__ xa = ws.x[0];
  float* __restrict__ xt = ws.x[1];
  const bool carry = lane <= nreg;         // lanes with a slot of ws.X
  const bool isP = lane == nreg;           // ... the one that carries (a, P)
  const int ip = lane < p ? lane : -1;     // d phi_i = [i == ip]
  const int iq = lane >= p && lane < nreg ? lane - p + 1 : -1;   // d R_i = [i == iq]

  float g[P], c;
  const int st = load_fit(a, row, live, g, c);
  const bool gated = live && st != MMF_STATUS_EMPTY && hr.ma_order[row] == q;
  const float* __restrict__ zr = a.y + (live ? row : 0) * a.ld_y;
  const float* __restrict__ yr = ma.y + (live ? row : 0) * ma.ld_y;
  if (gated && lane < nreg) xa[lane] = lane < p ? ar.phi[row * AR_MAX + lane] : hr.theta[row * MA_MAX + lane - p];
  if (lane < NPAR) xt[lane] = gated && lane < nreg ? xa[lane] : 0.f;
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
  int passes = 0, n_acc = 0, stop = 0;
  double obj = 0.0, L0 = dnan(), L = dnan(), sig = dnan(), n_obs0 = 0.0, n_obs = 0.0;
  double lam = (double)MMF_CSS_LAMBDA0;

  while (__syncthreads_or(active)) {
    // ---- P_0 at the trial point xt; a failed solve is a failed step-down (no pass)
    while (active) {
      if (lane < RMAX) {
        ws.ph[lane] = lane < p ? (double)xt[lane] : 0.0;
        ws.rv[lane] = lane == 0 ? 1.0 : lane <= q ? (double)xt[p + lane - 1] : 0.0;
      }
      __syncwarp();
      if (p0_solve(ws, r, p, nreg, lane)) break;
      if (passes == 0) { active = false; break; }          // the CSS point's own solve: the row keeps its outputs
      lam *= 10.0;
      int ok = 0;
      if (lane == 0) ok = ml_step(ws.hg, xa, xt, ws.j, p, q, lam) ? 1 : 0;
      __syncwarp();
      ok = __shfl_sync(0xffffffffu, ok, 0);
      lam = __shfl_sync(0xffffffffu, lam, 0);
      if (!ok) { stop = ML_STALLED; active = false; }
    }
    // ---- one pass: the filter, S_w, sum log F and the system at the point
    double yv_[RMAX];                      // lane < np: d a / d x_lane; lane np: a
#pragma unroll
    for (int k = 0; k < RMAX; ++k) yv_[k] = 0.0;
    double gacc[3] = {0.0, 0.0, 0.0};
    double slf = 0.0, dlf = 0.0;           // sum log F (every lane), sum dF / F (this lane's parameter)
    int nc = 0;
    for (int c0 = 0; c0 < T; c0 += TC) {
      stage(sm.a, sm.nz, d, ar, c0);
      __syncthreads();
      if (active) {
#pragma unroll 1
        for (int t0 = c0; t0 < min(c0 + TC, T); t0 += 32) {
          const int s = t0 + lane;
          const float yv = s < T ? __ldg(zr + s) : 0.f;
          const bool obs = s < T && finite_f(yv);
          const float e = obs ? yv - fitted(sm.a, s - c0, g, c) : 0.f;
          const int jn = min(32, T - t0);
#ifdef MMF_ARMAML_GAP_AS_ZERO
          // control build: a missing row updates the filter with e = 0
          const uint32_t bal = jn == 32 ? 0xffffffffu : (1u << jn) - 1u;
#else
          const uint32_t bal = __ballot_sync(0xffffffffu, obs);
#endif
          const double ed = (double)e;
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            const double ej = __shfl_sync(0xffffffffu, ed, j);
            const bool oj = (bal >> j) & 1u;
            const double a0 = __shfl_sync(0xffffffffu, yv_[0], nreg);
            const double F = ws.X[nreg];                        // P_11
            double dc[RMAX + 1];                                // this lane's X e_1
#pragma unroll
            for (int i = 0; i < RMAX; ++i) dc[i] = carry && i < r ? ws.X[ent(0, i) * NSLOT + lane] : 0.0;
            dc[RMAX] = 0.0;
            const double dF = dc[0];
            const double invF = 1.0 / F;
            const double v = ej - a0;
            const double y0 = yv_[0];
            if (oj) {
              const double sF = sqrt(F);
              const double vt = v / sF;
              const double Dt = -y0 / sF - 0.5 * vt * dF * invF;
              slf += log(F);
              dlf += dF * invF;
              if (lane < nreg) ws.j[j * NPAR + lane] = Dt;
              if (lane == 0) ws.vt[j] = vt;
            }
            // Gv: K (observed) or T P Z' (missing); W this lane's; yv_ moves in ascending order
            double Gv[RMAX], W[RMAX];
#pragma unroll
            for (int i = 0; i < RMAX; ++i) {
              const double phi_i = ws.ph[i];
              const double M = i < r ? fma(phi_i, F, i + 1 < r ? ws.X[ent(0, i + 1) * NSLOT + nreg] : 0.0) : 0.0;
              const double dphi = i == ip ? 1.0 : 0.0;
              const double dM = dphi * F + phi_i * dF + dc[i + 1];
              double yK, B;
              if (oj) {                    // observed: K = M / F and its derivative
                const double K = M * invF;
                const double dK = (dM - K * dF) * invF;
                Gv[i] = K; yK = K;
                W[i] = isP ? 0.0 : dphi * F - dM;
                B = isP ? K * ej : dphi * a0 + dK * v;
              } else {                     // missing: predict only
                Gv[i] = M; yK = 0.0;
                W[i] = isP ? 0.0 : dphi;
                B = isP ? 0.0 : dphi * a0;
              }
              yv_[i] = phi_i * y0 + (i + 1 < RMAX ? yv_[i + 1] : 0.0) - yK * y0 + B;
            }
            const double cc = oj ? (isP ? -F : dF) : 0.0;
            __syncwarp();
            if (carry) {
#pragma unroll
              for (int i = 0; i < RMAX; ++i)
#pragma unroll
                for (int jj = i; jj < RMAX; ++jj) {
                  if (jj >= r) continue;
                  const double pi = ws.ph[i], pj = ws.ph[jj], ri = ws.rv[i], rj = ws.rv[jj];
                  const double qi = isP ? 0.5 * ri : i == iq ? 1.0 : 0.0, qj = isP ? 0.5 * rj : jj == iq ? 1.0 : 0.0;
                  double x = jj + 1 < r ? ws.X[ent(i + 1, jj + 1) * NSLOT + lane] : 0.0;
                  x = fma(pi * pj, dc[0], x);
                  x = fma(pi, dc[jj + 1], x);
                  x = fma(pj, dc[i + 1], x);
                  x = fma(W[i], Gv[jj], x);
                  x = fma(Gv[i], W[jj], x);
                  x = fma(qi, rj, x);
                  x = fma(ri, qj, x);
                  x = fma(cc * Gv[i], Gv[jj], x);
                  ws.X[ent(i, jj) * NSLOT + lane] = x;
                }
            }
            __syncwarp();
          }
          // the observed rows of the block
          const uint32_t cm = bal;
          nc += __popc(cm);
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            if (ei[k] < 0) continue;
            const int ci = ei[k], cj = ej[k];
            const double* bi = ci == nreg ? ws.vt : ws.j + ci;
            const double* bj = cj == nreg ? ws.vt : ws.j + cj;
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

    // ---- the objective, G's rank-2 correction, accept or reject, then the next trial point
    const double n = (double)nc;
    double mine = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) mine = k == (idx_S >> 5) ? gacc[k] : mine;
    const double Sw = __shfl_sync(0xffffffffu, mine, idx_S & 31);
#ifdef MMF_ARMAML_NO_LOGDET
    slf = 0.0;                             // control build: sum log F dropped (the objective is S_w)
    dlf = 0.0;
#endif
    const double Ln = n * log(Sw / n) + slf;
    const double on = exp(slf / n) * Sw;
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (ei[k] >= 0) ws.raw[ent(ei[k], ej[k])] = gacc[k];
    if (lane < nreg) ws.gam[lane] = dlf / (2.0 * n);
    __syncwarp();
    double cor[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      cor[k] = gacc[k];
      const int ci = ei[k], cj = ej[k];
      if (ci < 0 || ci == nreg) continue;
      if (cj == nreg) {
        cor[k] = fma(Sw, ws.gam[ci], gacc[k]);
      } else {
        const double gi = ws.gam[ci], gj = ws.gam[cj];
        double h = fma(gi, ws.raw[ent(cj, nreg)], gacc[k]);
        h = fma(ws.raw[ent(ci, nreg)], gj, h);
        cor[k] = fma(Sw * gi, gj, h);
      }
    }
    ++passes;
    bool take, conv = false;
    if (passes == 1) {
      take = true;
      L0 = Ln;
      n_obs0 = n;
    } else {
      take = on < obj;
      if (take) conv = obj - on <= (double)MMF_CSS_RTOL * obj;
    }
    if (take) {
      if (passes > 1) {
        ++n_acc;
        lam /= 10.0;
        if (lane < nreg) xa[lane] = xt[lane];
      }
      obj = on;
      L = Ln;
      n_obs = n;
      sig = sqrt(Sw / n);
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (ei[k] >= 0) ws.hg[ent(ei[k], ej[k])] = cor[k];
    } else {
      lam *= 10.0;
    }
    __syncwarp();
    if (conv) stop = ML_CONVERGED;
    else if (lam > (double)MMF_CSS_LAMBDA_MAX) stop = ML_STALLED;
    else if (passes >= ml.max_iter) stop = ML_BUDGET;
    if (stop == 0) {
      int ok = 0;
      if (lane == 0) ok = ml_step(ws.hg, xa, xt, ws.j, p, q, lam) ? 1 : 0;
      __syncwarp();
      ok = __shfl_sync(0xffffffffu, ok, 0);
      lam = __shfl_sync(0xffffffffu, lam, 0);
      if (!ok) stop = ML_STALLED;
    }
    if (stop != 0) active = false;
  }

  // ---- outputs: the likelihood columns of every live row, sigma of the solved rows, phi / theta of the refined rows
  const bool done = gated && passes > 0;          // false: no pass, the CSS point's P_0 solve failed
  if (live && lane == 0) {
    const double c1 = 1.0 + log(2.0 * 3.14159265358979323846);
    if (ml.loglik_start != nullptr) ml.loglik_start[row] = done ? (float)(-0.5 * (L0 + n_obs0 * c1)) : qnan();
    if (ml.loglik != nullptr) ml.loglik[row] = done ? (float)(-0.5 * (L + n_obs * c1)) : qnan();
    if (ml.stop != nullptr) ml.stop[row] = done ? stop : 0;
    if (ml.iters != nullptr) ml.iters[row] = done ? passes : 0;
    if (done && ar.sigma != nullptr) ar.sigma[row] = (float)sig;
  }
  const bool refined = done && n_acc > 0;
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
  // integrated to levels; predictions only (sigma is the ML one)
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
    stage(sm.a, sm.nz, d, ar, c0);
    __syncthreads();
    if (refined) {
#pragma unroll 1
      for (int t0 = c0; t0 < min(c0 + TC, endB); t0 += 32) {
        const int s = t0 + lane;
        const float fit = fitted(sm.a, s - c0, g, c);
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

// one thread per row of the slab, behind refit_list_kernel (DESIGN.md section 4.25): a row whose winner is (p, d, 0), d
// this stage's, and on the first stage a row with no eligible candidate, gets the ML columns of a row no refit kernel
// touches (loglik_start, loglik NaN, ml_stop, iters 0): refit_list_kernel's rule for the CSS columns
__global__ void __launch_bounds__(256)
refit_ml_cols_kernel(const FitArgs a, const ArimaArgs ma, const MlArgs ml, const RefitArgs rf) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= a.n) return;
  const int cd = rf.choice_d[row], cq = rf.choice_q[row];
  if (!(cd == ma.d ? cq < 1 : rf.first && cd < 0)) return;
  if (ml.loglik_start != nullptr) ml.loglik_start[row] = qnan();
  if (ml.loglik != nullptr) ml.loglik[row] = qnan();
  if (ml.stop != nullptr) ml.stop[row] = 0;
  if (ml.iters != nullptr) ml.iters[row] = 0;
}

}  // namespace

cudaError_t launch_arma_ml(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                           const ArmaArgs& hr, const MlArgs& ml, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  // the attribute is per function and process-wide: always the kernel's fixed bound (arma_joint.cu's rule)
  cudaError_t e =
      cudaFuncSetAttribute(arma_ml_kernel_t<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ML_SMEM);
  if (e != cudaSuccess) return e;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;
  arma_ml_kernel_t<false><<<(unsigned)grid, THREADS, ML_SMEM, s>>>(d, a, ar, ma, hr, ml, RefitArgs{});
  return cudaGetLastError();
}


cudaError_t launch_arma_ml_list(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                                const ArmaArgs& hr, const MlArgs& ml, const RefitArgs& rf, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  cudaError_t e =
      cudaFuncSetAttribute(arma_ml_kernel_t<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ML_SMEM);
  if (e != cudaSuccess) return e;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;          // the list's length is on the device: the slab's rows
  arma_ml_kernel_t<true><<<(unsigned)grid, THREADS, ML_SMEM, s>>>(d, a, ar, ma, hr, ml, rf);
  return cudaGetLastError();
}

cudaError_t launch_refit_ml_cols(const FitArgs& a, const ArimaArgs& ma, const MlArgs& ml, const RefitArgs& rf,
                                 cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  refit_ml_cols_kernel<<<(unsigned)((a.n + 255) / 256), 256, 0, s>>>(a, ma, ml, rf);
  return cudaGetLastError();
}

}  // namespace mmf
