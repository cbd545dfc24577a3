// arima_se.cu -- standard errors of the ARIMA-family forecasts (mmf_arima_se_f32, DESIGN.md section 2 item 15).
//
// One warp per series.  The forecast error of the predictor the ARIMA-family calls ship (one step ahead in sample, the
// dynamic forecast beyond t_fit, missing values filled with predictions) is a linear function of the innovations, with
// the fitted (phi, theta, sigma) taken as true and u_s = eps_s = 0 for s < 0.  Its variance comes from the covariance P
// (units of sigma^2, float64) of the predictor's error state
//   x = (du_{s-1..s-p}, deps_{s-1..s-q}, dy_{t-1..t-d}),   level row t, z-row s = t - d,
// propagated row by row as P' = A P A' + b b'.  Three rows of A are dense (the new du, deps and dy), every other row is a
// shift, so a row costs O(k^2) with k = p + q + d <= 14:
//   g_s = a.x (a = (phi, theta, 0)), the level error minus eps_s is c.x (c = (phi, theta, L)), L = (1) or (2, -1);
//   z'_s observed (t < t_fit, levels t-d..t finite): du_s = 0, deps_s = -g_s;  otherwise du_s = g_s + eps_s, deps_s = eps_s;
//   level t observed (t < t_fit, y_t finite): dy_t = 0;  otherwise dy_t = c.x + eps_s;
//   se_t = sigma sqrt(1 + c'Pc) (before the row's update), NaN for t < d and where a used level lag is NaN in the
//   predictor's level chain (a flag per lag: set by a missing level at t < d, carried by a missing level whose lags are
//   flagged), +Inf where the float64 variance overflowed.
// P is exactly 0 while every row is observed, so those rows cost no arithmetic: a warp in the zero state reads y 256
// rows at a time and writes sigma (NaN for t < d) for the observed run.  With q = 0 the state is zero again once the
// last p + d levels are observed: the walk re-enters the zero state there, and starts at min(pred_start, t_fit) when
// the p + d levels before it are observed.  With q >= 1 it never returns to zero after a missing row.
// Built with -DMMF_ARIMASE_NO_GAPS (tests/_build/libmmf_arimase_nogaps.so, negative control only), every fit row counts
// as observed: sigma in sample and the textbook psi-weight formula beyond, whatever the gaps.
#include "mmf_internal.cuh"

namespace mmf {
namespace {

constexpr int THREADS = 128;
constexpr int WARPS = THREADS / 32;
constexpr int KM = MMF_AR_MAX + MMF_MA_MAX + MMF_DIFF_MAX;    // largest state (14)
constexpr int FAST_CHUNKS = 8;                                // 32-row ballots of one zero-state read (256 rows in flight)

struct WarpSmem {
  double P[2][KM * KM];     // ping-pong covariance
  double a[KM], c[KM];      // g = a.x, level error - eps = c.x
  double pa[KM], pc[KM];    // P a, P c of the current row
};

__device__ __forceinline__ bool finite_bits(float x) { return (__float_as_uint(x) & 0x7f800000u) != 0x7f800000u; }

// level t counts as observed (t < t_fit is the caller's condition)
__device__ __forceinline__ bool level_obs(float v) {
#ifdef MMF_ARIMASE_NO_GAPS
  (void)v;
  return true;
#else
  return finite_bits(v);
#endif
}

struct Head { double sa, sc, b; };   // new head component = sa (a.x) + sc (c.x) + b eps

__global__ void __launch_bounds__(THREADS)
arima_se_kernel(const ArimaSeArgs g) {
  __shared__ WarpSmem smem[WARPS];
  const int lane = threadIdx.x & 31;
  WarpSmem& sm = smem[threadIdx.x >> 5];
  const float qnan = __int_as_float(0x7fc00000);
  const int64_t n_warps = (int64_t)gridDim.x * WARPS;
  const int32_t end = g.pred_start + g.n_pred;
  for (int64_t i = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5); i < g.n; i += n_warps) {
    const int p = __ldg(g.order + i);
    const int q = g.ma_order ? __ldg(g.ma_order + i) : 0;
    const int d = g.diffs ? __ldg(g.diffs + i) : g.diff_order;
    const float sigf = __ldg(g.sigma + i);
    float* __restrict__ out = g.out + i * g.ld_se - g.pred_start;       // out[t] for t in [pred_start, end)
    if (p < 0 || p > MMF_AR_MAX || q < 0 || q > MMF_MA_MAX || d < 0 || d > MMF_DIFF_MAX || !finite_bits(sigf)) {
      for (int t = g.pred_start + lane; t < end; t += 32) out[t] = qnan;
      continue;
    }
    const int pq = p + q, k = pq + d;
    const float* __restrict__ yr = g.y + i * g.ld_y;
    if (lane < k) {
      const double v = lane < p ? (double)__ldg(g.phi + i * MMF_AR_MAX + lane)
                     : lane < pq ? (double)__ldg(g.theta + i * MMF_MA_MAX + (lane - p)) : 0.0;
      sm.a[lane] = v;
      sm.c[lane] = lane < pq ? v : (lane == pq ? (d == 1 ? 1.0 : 2.0) : -1.0);
    }
    const double sig = (double)sigf;
    // start of the walk, in the zero state: row 0, or for q = 0 min(pred_start, t_fit) when its p + d levels before it
    // are observed
    int t = 0, run = 0;                  // run: consecutive observed levels ending at t - 1
    if (q == 0) {
      const int r = min(g.pred_start, g.t_fit), pd = p + d;
      if (r >= pd) {
        const bool ok = lane >= pd || level_obs(__ldg(yr + r - pd + lane));
        if (__all_sync(0xffffffffu, ok)) { t = r; run = pd; }
      }
    }
    __syncwarp();
    bool zero = true;
    int cur = 0;
    bool f0 = false, f1 = false;         // NaN flags of level lags 1 and 2
    int mbase = -32;                     // observed-level mask of rows [mbase, mbase + 32) for the general path
    uint32_t mask = 0u;
    while (t < end) {
      if (zero) {
        const int lim = min(end, g.t_fit);
        if (t < lim) {
          float v[FAST_CHUNKS];
#pragma unroll
          for (int j = 0; j < FAST_CHUNKS; ++j) {
            const int r = t + j * 32 + lane;
            v[j] = r < lim ? __ldg(yr + r) : qnan;
          }
          const int t0 = t;
          bool stop = false;
#pragma unroll
          for (int j = 0; j < FAST_CHUNKS; ++j) {
            if (!stop) {
              const int r = t0 + j * 32 + lane;
              const uint32_t m = __ballot_sync(0xffffffffu, r < lim && level_obs(v[j]));
              const int nrun = m == 0xffffffffu ? 32 : __ffs(~m) - 1;
              if (lane < nrun && r >= g.pred_start) out[r] = r < d ? qnan : sigf;
              run += nrun;
              if (nrun < 32) { t = t0 + j * 32 + nrun; stop = true; }
            }
          }
          if (!stop) { t = t0 + FAST_CHUNKS * 32; continue; }
          if (t >= end) break;
        }
        // row t is not observed: leave the zero state with P = 0 (flags are clear there)
        for (int e = lane; e < k * k; e += 32) sm.P[cur][(e / k) * KM + e % k] = 0.0;
        zero = false;
        __syncwarp();
      }
      // ---- general row t ----
      if (t - mbase >= 32) {
        mbase = t;
        const int r = t + lane;
        mask = __ballot_sync(0xffffffffu, r < g.t_fit && level_obs(__ldg(yr + min(r, g.t_fit - 1))));
      }
      const bool lobs = (mask >> (t - mbase)) & 1u;
      run = lobs ? run + 1 : 0;
      if (t < d) {
        if (lane == 0 && t >= g.pred_start) out[t] = qnan;
        f1 = f0; f0 = !lobs;
      } else {
        const bool zobs = run >= d + 1;
        const double* P = sm.P[cur];
        double pa = 0.0, pc = 0.0;
        if (lane < k) {
          for (int j = 0; j < k; ++j) {
            const double x = P[lane * KM + j];
            pa = fma(x, sm.a[j], pa);
            pc = fma(x, sm.c[j], pc);
          }
          sm.pa[lane] = pa;
          sm.pc[lane] = pc;
        }
        double apa = lane < k ? sm.a[lane] * pa : 0.0;
        double apc = lane < k ? sm.a[lane] * pc : 0.0;
        double cpc = lane < k ? sm.c[lane] * pc : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          apa += __shfl_xor_sync(0xffffffffu, apa, o);
          apc += __shfl_xor_sync(0xffffffffu, apc, o);
          cpc += __shfl_xor_sync(0xffffffffu, cpc, o);
        }
        const bool flagged = (d >= 1 && f0) || (d == 2 && f1);
        if (lane == 0 && t >= g.pred_start) {
          const double s = sig * sqrt(1.0 + cpc);
          out[t] = flagged ? qnan : (s != s ? __int_as_float(0x7f800000) : (float)s);
        }
        __syncwarp();
        const Head hu = zobs ? Head{0.0, 0.0, 0.0} : Head{1.0, 0.0, 1.0};
        const Head he = zobs ? Head{-1.0, 0.0, 0.0} : Head{0.0, 0.0, 1.0};
        const Head hy = lobs ? Head{0.0, 0.0, 0.0} : Head{0.0, 1.0, 1.0};
        double* Pn = sm.P[cur ^ 1];
        for (int e = lane; e < k * k; e += 32) {
          const int r = e / k, s = e - r * k;
          // a component is a block's head (its new value) or the shift of the component before it
          const bool hr = r == 0 || r == p || r == pq, hs = s == 0 || s == p || s == pq;
          const Head h1 = r < p ? hu : (r < pq ? he : hy);
          const Head h2 = s < p ? hu : (s < pq ? he : hy);
          double v;
          if (!hr && !hs) v = P[(r - 1) * KM + (s - 1)];
          else if (hr && !hs) v = h1.sa * sm.pa[s - 1] + h1.sc * sm.pc[s - 1];
          else if (!hr && hs) v = h2.sa * sm.pa[r - 1] + h2.sc * sm.pc[r - 1];
          else v = h1.sa * h2.sa * apa + (h1.sa * h2.sc + h1.sc * h2.sa) * apc + h1.sc * h2.sc * cpc + h1.b * h2.b;
          Pn[r * KM + s] = v;
        }
        cur ^= 1;
        const bool nf = !lobs && flagged;
        f1 = f0; f0 = nf;
        __syncwarp();
      }
      ++t;
      if (q == 0 && run >= p + d) zero = true;     // the last p + d levels observed: P = 0, flags clear
    }
    __syncwarp();
  }
}

}  // namespace

cudaError_t launch_arima_se(const ArimaSeArgs& a, int sm_count, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  const int64_t want = (a.n + WARPS - 1) / WARPS;
  const int64_t cap = (int64_t)sm_count * 16;
  arima_se_kernel<<<(unsigned)(want < cap ? want : cap), THREADS, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace mmf
