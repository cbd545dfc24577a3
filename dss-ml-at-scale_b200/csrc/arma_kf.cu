// arma_kf.cu -- the Kalman predictor of the exact-likelihood ARIMA(p, d, q) fit (DESIGN.md section 2 item 20, section
// 4.24), behind mmf_fit_forecast_arma_ml_kf_f32.  Per slab, after the whole ML call (fit passes, ar_kernel /
// arima_kernel, arma_kernel, arma_css_kernel, arma_ml_kernel) and, when out_se is given, arima_se_kernel over every row:
//   arma_kf_kernel  one warp per gated series whose stationary P_0 solves at the shipped (phi, theta): the filter of
//     arma_ml_kernel's model, run once in float64 over the z-space rows [0, max(endz, T)), predicts e_s by a_{s,1} (a
//     missing row predicted, not updated; beyond T the dynamic forecast a <- T a).  The level prediction is fitted_s +
//     a_{s,1}, integrated to levels as pass B of arma_kernel integrates it.  Its error state is xi = (alpha - a, the level
//     errors of the d previous filled levels), k = r + d <= 10 components; their covariance C (units of sigma^2) moves
//     row by row as C' = U C U' + b b', every new component a sparse row of U:
//       alpha_i - a_i  <-  (phi_i - kappa_i) (alpha_1 - a_1) + (alpha_{i+1} - a_{i+1}) + R_i eps,  kappa = K observed, 0
//                           missing (K = T P Z' / F, P = C's alpha block: the filter's covariance);
//       newest level error  <-  lambda = (alpha_1 - a_1) + L . (level errors), L = (1) or (2, -1); 0 where y_t is observed;
//       the level error before it  <-  the newest one (d = 2).
//     se_t = sigma sqrt(Var lambda) before the row's update (sqrt(F) on an observed row for d = 0), NaN where
//     arima_se_kernel's level-chain flags give NaN, +Inf where the float64 variance overflowed.  The lanes own the packed
//     entries of C' (<= 55, two per lane); everything else is the same on every lane.
// P_0 is arma_ml.cu's elimination on the P column alone (no derivatives), written out again: the same operations in the
// same order, so that it fails exactly where arma_ml_kernel's fails at the same point.
// arma_kf_kernel is arma_kf_kernel_t<false>.  The ML + Kalman refit of a (p, d, q) selection's winners
// (mmf_fit_select_arma_ml_kf_f32, section 4.25) runs arma_kf_list_kernel, which is arma_kf_kernel_t<true>: the same
// kernel over a list of rows with each row's own (p, q).
#include "ar_common.cuh"
#ifdef MMF_REFIT_ASSERT
#include <assert.h>
#endif

namespace mmf {
namespace {

constexpr int RMAX = AR_MAX > MA_MAX + 1 ? AR_MAX : MA_MAX + 1;   // state dimension r = max(p, q + 1)
constexpr int NSYM = RMAX * (RMAX + 1) / 2;                        // symmetric unknowns of P_0
constexpr int AUGW = NSYM + 1;                                     // [A | vec(R R')]
constexpr int KM = RMAX + MMF_DIFF_MAX;                            // error state: alpha - a, then the level errors
constexpr int NSLOT = 2;                                           // packed entries of C per lane
static_assert(KM * (KM + 1) / 2 <= 32 * NSLOT, "two covariance entries per lane");

struct KfWarp {
  double C[2][KM * KM];                    // ping-pong covariance of the error state, dense, row-major
  double aug[NSYM * AUGW];                 // the P_0 system, row-major
  double ph[RMAX], rv[RMAX];               // phi and R, padded to RMAX
};
struct KfSmem {
  float4 a[4][TC];                         // the staged chunk (ar_common's stage)
  uint32_t nz[TC];
  KfWarp w[WARPS];
};
static_assert(offsetof(KfSmem, w) % 16 == 0 && sizeof(KfWarp) % 8 == 0, "aligned per-warp blocks");
constexpr size_t KF_SMEM = sizeof(KfSmem);
static_assert(2 * KF_SMEM <= 227 * 1024, "two CTAs per SM");

// packed index of entry (i, j), i <= j, column-major upper triangle (arma_ml.cu's)
__device__ __forceinline__ int ent(int i, int j) { return j * (j + 1) / 2 + i; }

// (i, j) of packed entry k
__device__ __forceinline__ void unpack(int k, int& i, int& j) {
  j = 0;
  while ((j + 1) * (j + 2) / 2 <= k) ++j;
  i = k - j * (j + 1) / 2;
}

// the whole warp: P_0 from ws.ph / ws.rv into the alpha block of ws.C[0] (the rest of it zero).  False (on every lane)
// when a pivot |u_kk| <= MMF_HR_PIVOT_TOL x max |A| (arma_ml.cu's p0_solve on its P column)
__device__ bool p0_solve(KfWarp& ws, int r, int k, int lane) {
  const int N = r * (r + 1) / 2;
  double* __restrict__ A = ws.aug;
  double amax = 0.0;
  for (int e = lane; e < N; e += 32) {     // row e: P_ij - (T P T')_ij = R_i R_j
    double* row = A + e * AUGW;
    for (int c = 0; c <= N; ++c) row[c] = 0.0;
    int i, j;
    unpack(e, i, j);
    const double pi = ws.ph[i], pj = ws.ph[j];
    row[e] += 1.0;
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
  for (int kk = 0; kk < N; ++kk) {
    double best = -1.0;
    int bi = kk;
    for (int i = kk + lane; i < N; i += 32) {
      const double v = fabs(A[i * AUGW + kk]);
      if (v > best) { best = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (!(best > (double)MMF_HR_PIVOT_TOL * amax)) return false;
    if (bi != kk)
      for (int c = lane; c <= N; c += 32) {
        const double t = A[kk * AUGW + c];
        A[kk * AUGW + c] = A[bi * AUGW + c];
        A[bi * AUGW + c] = t;
      }
    __syncwarp();
    const double inv = 1.0 / A[kk * AUGW + kk];
    __syncwarp();
    for (int i = kk + 1 + lane; i < N; i += 32) A[i * AUGW + kk] *= inv;   // the multipliers
    __syncwarp();
    for (int c = kk + 1 + lane; c <= N; c += 32) {
      const double akc = A[kk * AUGW + c];
      for (int i = kk + 1; i < N; ++i) A[i * AUGW + c] = fma(-A[i * AUGW + kk], akc, A[i * AUGW + c]);
    }
    __syncwarp();
  }
  if (lane == 0)                           // back substitution of the P column (arma_ml.cu's back_sub)
    for (int i = N - 1; i >= 0; --i) {
      double v = A[i * AUGW + N];
      for (int c = i + 1; c < N; ++c) v = fma(-A[i * AUGW + c], A[c * AUGW + N], v);
      A[i * AUGW + N] = v / A[i * AUGW + i];
    }
  __syncwarp();
  for (int e = lane; e < k * k; e += 32) {
    const int i = e / k, j = e - i * k;
    ws.C[0][i * KM + j] = i < r && j < r ? A[ent(min(i, j), max(i, j)) * AUGW + N] : 0.0;
  }
  __syncwarp();
  return true;
}

// the row of U of error component i: up to three (index, coefficient) terms; fi = phi_i - kappa_i for i < r
struct Row { int ix[3]; double cf[3]; };
__device__ __forceinline__ Row urow(int i, int r, int dd, double fi, double mu) {
  Row u{{0, 0, 0}, {0.0, 0.0, 0.0}};
  if (i < r) {
    u.ix[0] = 0; u.cf[0] = fi;
    if (i + 1 < r) { u.ix[1] = i + 1; u.cf[1] = 1.0; }
  } else if (i == r) {                     // the newest level error: mu lambda
    u.ix[0] = 0; u.cf[0] = mu;
    u.ix[1] = r; u.cf[1] = dd == 1 ? mu : 2.0 * mu;
    if (dd == 2) { u.ix[2] = r + 1; u.cf[2] = -mu; }
  } else {                                 // the level error before it
    u.ix[0] = r; u.cf[0] = 1.0;
  }
  return u;
}

// d.t_fit: fit rows of a.y (z' for d >= 1); ma: the levels (ma.d = 0: ma.y is a.y); ar.p / hr.q: the orders; ar.phi,
// hr.theta, hr.ma_order: the ML call's outputs (caller buffers or scratch, never null here); ar.sigma: never null when
// kf.se is given.  LIST: the rows of a (p, d, q) selection whose winner has q >= 1 and this d (the ML + Kalman refit of
// DESIGN.md section 4.25), behind the ML list kernel's outputs for the same list, each at its winner's orders, by
// arma_css_kernel_t's rules for LIST and rf.  Warps past the count index nothing by p or q.
template <bool LIST>
__global__ void __launch_bounds__(THREADS, 2)
arma_kf_kernel_t(const DesignView d, const FitArgs a, const ArArgs ar, const ArimaArgs ma, const ArmaArgs hr,
                 const KfArgs kf, const RefitArgs rf) {
  if constexpr (LIST) {
    if ((int64_t)blockIdx.x * WARPS >= (int64_t)*rf.count) return;   // a CTA past the list: uniform exit
  }
  extern __shared__ __align__(16) unsigned char smem_raw[];
  KfSmem& sm = *reinterpret_cast<KfSmem*>(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  KfWarp& ws = sm.w[warp];
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
  const int r = max(p, q + 1);
  const int dd = ma.d;
  const int k = r + dd;
  const int T = d.t_fit;                   // fit rows of a.y
  const int TL = ma.t_fit;                 // level fit rows
  const int end = a.pred_start + a.n_pred; // level rows [pred_start, end)
  const int endB = max(end - dd, T);

  float g[P], c;
  const int st = load_fit(a, row, live, g, c);
  const bool gated = live && st != MMF_STATUS_EMPTY && hr.ma_order[row] == q;
  const float* __restrict__ zr = a.y + (live ? row : 0) * a.ld_y;
  const float* __restrict__ yr = ma.y + (live ? row : 0) * ma.ld_y;
  if (lane < RMAX) {
    ws.ph[lane] = gated && lane < p ? (double)ar.phi[row * AR_MAX + lane] : 0.0;
    ws.rv[lane] = lane == 0 ? 1.0 : gated && lane <= q ? (double)hr.theta[row * MA_MAX + lane - 1] : 0.0;
  }
  __syncwarp();
  const bool covered = gated && p0_solve(ws, r, k, lane);
  if (!__syncthreads_or(covered)) return;

  const double* __restrict__ ph = ws.ph;
  const double* __restrict__ rv = ws.rv;
#ifdef MMF_ARMAKF_GAIN_P0
  // control build: the gain from P_0 on every row
  double k0[RMAX];
#pragma unroll
  for (int i = 0; i < RMAX; ++i)
    k0[i] = i < r ? fma(ph[i], ws.C[0][0], i + 1 < r ? ws.C[0][(i + 1) * KM] : 0.0) / ws.C[0][0] : 0.0;
#endif
  // this lane's packed entries of C
  int ei[NSLOT], ej[NSLOT];
#pragma unroll
  for (int m = 0; m < NSLOT; ++m) {
    const int e = lane + 32 * m;
    ei[m] = -1; ej[m] = -1;
    if (e < k * (k + 1) / 2) unpack(e, ei[m], ej[m]);
  }
  const bool want_se = covered && kf.se != nullptr;
  const double sig = want_se ? (double)ar.sigma[row] : 0.0;
  double av[RMAX];                         // a, the same on every lane
#pragma unroll
  for (int i = 0; i < RMAX; ++i) av[i] = 0.0;
  int cur = 0;
  // the level chain: l1, l2 the filled levels t - 1, t - 2 (pass B's); f0, f1 arima_se_kernel's NaN flags of level lags
  float l1 = qnan(), l2 = qnan();
  bool f0 = false, f1 = false;
  if (covered && dd > 0) {
    const int i1 = dd - 1, i2 = dd - 2;
    const float v1 = __ldg(yr + i1);
    const float v2 = i2 >= 0 ? __ldg(yr + i2) : qnan();
    l1 = finite_f(v1) ? v1 : qnan();
    l2 = finite_f(v2) ? v2 : qnan();
    f0 = !finite_f(v1);
    f1 = i2 >= 0 && !finite_f(v2);
  }
  for (int c0 = 0; c0 < endB; c0 += TC) {
    stage(sm.a, sm.nz, d, ar, c0);
    __syncthreads();
    if (covered) {
#pragma unroll 1
      for (int t0 = c0; t0 < min(c0 + TC, endB); t0 += 32) {
        const int s = t0 + lane;
        const float fit = fitted(sm.a, s - c0, g, c);
        const float yv = s < T ? __ldg(zr + s) : 0.f;            // never read at or beyond the fit rows
        const bool obs = s < T && finite_f(yv);
        const float e = obs ? yv - fit : 0.f;
        const uint32_t bal = __ballot_sync(0xffffffffu, obs);
        const int t = s + dd;
        const float lv = t < TL ? __ldg(yr + t) : 0.f;           // y is never read at or beyond t_fit
        const bool lobs = t < TL && finite_f(lv);
        const uint32_t lbal = __ballot_sync(0xffffffffu, lobs);
        const double ed = (double)e;
        const int jn = min(32, endB - t0);
        double eh = 0.0, vl = 0.0;                               // lane j: a_{s,1} and Var lambda of row t0 + j
        bool fl = false;                                         // ... and its NaN flag
#pragma unroll 1
        for (int j = 0; j < jn; ++j) {
          const double es = __shfl_sync(0xffffffffu, ed, j);
          const bool oj = (bal >> j) & 1u;
          const bool lj = (lbal >> j) & 1u;
          const double* __restrict__ Cc = ws.C[cur];
          const double F = Cc[0];
          // Var lambda = c' C c, c = e_1 (+ L on the level errors)
          double var = F;
          if (dd == 1) var = Cc[0] + 2.0 * Cc[r] + Cc[r * KM + r];
          if (dd == 2) {
            const double c0r = Cc[r], c0s = Cc[r + 1], crr = Cc[r * KM + r], crs = Cc[r * KM + r + 1];
            const double css = Cc[(r + 1) * KM + r + 1];
            var = Cc[0] + 4.0 * c0r - 2.0 * c0s + 4.0 * crr - 4.0 * crs + css;
          }
          const bool flagged = (dd >= 1 && f0) || (dd == 2 && f1);
          if (lane == j) { eh = av[0]; vl = var; fl = flagged; }
          const bool nf = !lj && flagged;
          f1 = f0; f0 = nf;
          // the gain (0 on a missing or forecast row) and phi - kappa
          double fk[RMAX];
          const double invF = 1.0 / F;
#pragma unroll
          for (int i = 0; i < RMAX; ++i) {
#ifdef MMF_ARMAKF_GAIN_P0
            const double K = k0[i];
#else
            const double K = i < r ? fma(ph[i], F, i + 1 < r ? Cc[(i + 1) * KM] : 0.0) * invF : 0.0;
#endif
            fk[i] = oj ? ph[i] - K : ph[i];
          }
          const double a0 = av[0];
#pragma unroll
          for (int i = 0; i < RMAX; ++i) {
            const double kap = ph[i] - fk[i];
            av[i] = fma(fk[i], a0, i + 1 < RMAX ? av[i + 1] : 0.0);
            if (oj) av[i] = fma(kap, es, av[i]);
          }
          const double mu = lj ? 0.0 : 1.0;
          double* __restrict__ Cn = ws.C[cur ^ 1];
#pragma unroll
          for (int m = 0; m < NSLOT; ++m) {
            if (ei[m] < 0) continue;
            const int i = ei[m], jj = ej[m];
            double fi = 0.0, fj = 0.0;
#pragma unroll
            for (int u = 0; u < RMAX; ++u) {
              fi = u == i ? fk[u] : fi;
              fj = u == jj ? fk[u] : fj;
            }
            const Row ui = urow(i, r, dd, fi, mu), uj = urow(jj, r, dd, fj, mu);
            double x = i < r && jj < r ? rv[i] * rv[jj] : 0.0;
#pragma unroll
            for (int u = 0; u < 3; ++u) {
              double h = 0.0;
#pragma unroll
              for (int w = 0; w < 3; ++w) h = fma(uj.cf[w], Cc[ui.ix[u] * KM + uj.ix[w]], h);
              x = fma(ui.cf[u], h, x);
            }
#ifdef MMF_ARMAKF_NO_CROSS
            if (i < r && jj >= r) x = 0.0;       // control build: no covariance between alpha - a and the level errors
#endif
            Cn[i * KM + jj] = x;
            Cn[jj * KM + i] = x;
          }
          __syncwarp();
          cur ^= 1;
        }
        // the level predictions of the block (pass B's integration) and their standard errors
        const float zh = fit + (float)eh;
        float yh = zh;                                           // d = 0: the level step is the identity
        if (dd > 0) {
          if (lbal == 0xffffffffu) {
            const float p1 = __shfl_up_sync(0xffffffffu, lv, 1), p2 = __shfl_up_sync(0xffffffffu, lv, 2);
            yh = integrate(zh, lane >= 1 ? p1 : l1, lane >= 2 ? p2 : (lane == 1 ? l1 : l2), dd);
            l1 = __shfl_sync(0xffffffffu, lv, 31);
            l2 = __shfl_sync(0xffffffffu, lv, 30);
          } else {
            yh = 0.f;
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
        if (t >= a.pred_start && t < end && lane < jn) {
          a.out[row * a.ld_out + (t - a.pred_start)] = yh;
          if (want_se) {
            const double sv = sig * sqrt(vl);
            kf.se[row * kf.ld_se + (t - a.pred_start)] = fl ? qnan() : (sv != sv ? __int_as_float(0x7f800000) : (float)sv);
          }
        }
      }
    }
    __syncthreads();
  }
}

}  // namespace

cudaError_t launch_arma_kf(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                           const ArmaArgs& hr, const KfArgs& kf, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  // the attribute is per function and process-wide: always the kernel's fixed bound (arma_joint.cu's rule)
  cudaError_t e =
      cudaFuncSetAttribute(arma_kf_kernel_t<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)KF_SMEM);
  if (e != cudaSuccess) return e;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;
  arma_kf_kernel_t<false><<<(unsigned)grid, THREADS, KF_SMEM, s>>>(d, a, ar, ma, hr, kf, RefitArgs{});
  return cudaGetLastError();
}


cudaError_t launch_arma_kf_list(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                                const ArmaArgs& hr, const KfArgs& kf, const RefitArgs& rf, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  cudaError_t e =
      cudaFuncSetAttribute(arma_kf_kernel_t<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)KF_SMEM);
  if (e != cudaSuccess) return e;
  const int64_t grid = (a.n + WARPS - 1) / WARPS;          // the list's length is on the device: the slab's rows
  arma_kf_kernel_t<true><<<(unsigned)grid, THREADS, KF_SMEM, s>>>(d, a, ar, ma, hr, kf, rf);
  return cudaGetLastError();
}

}  // namespace mmf
