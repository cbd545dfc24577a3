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
// score every (p, d) candidate on levels.
#include "ar_common.cuh"

namespace mmf {
namespace {

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fc00000); }

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

// yhat_t from zhat_t and the filled levels ytilde_{t-1} (l1), ytilde_{t-2} (l2), in the order include/mmf.h states
__device__ __forceinline__ float integrate(float zh, float l1, float l2, int d) {
  return d == 1 ? __fadd_rn(zh, l1) : __fsub_rn(__fadd_rn(zh, __fmul_rn(2.f, l1)), l2);
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

  int st = MMF_STATUS_EMPTY;
  float g[P], c = 0.f;
#pragma unroll
  for (int q = 0; q < P; ++q) g[q] = 0.f;
  if (live) {
    st = a.status[row];
    const float4* gp = reinterpret_cast<const float4*>(a.out_gamma + row * P);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = gp[q];
      g[4 * q] = v.x; g[4 * q + 1] = v.y; g[4 * q + 2] = v.z; g[4 * q + 3] = v.w;
    }
    c = a.out_c[row];
  }
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
          const int jmax = S - t0 - 1;                           // t0 + 1 + j <= S
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
  colmask = __reduce_or_sync(0xffffffffu, colmask);
  uint32_t used = d.kept_mask & colmask;
  if (st == MMF_STATUS_RANKDEF) {
#pragma unroll
    for (int q = 0; q < P; ++q) used &= g[q] != 0.f ? ~0u : ~(1u << q);
  }
  const int k_used = __popc(used);
  double phi[AR_MAX];
#pragma unroll
  for (int j = 0; j < AR_MAX; ++j) phi[j] = 0.0;
  int order = 0;
  double var = __longlong_as_double(0x7ff8000000000000ll);
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
    if (ar.phi != nullptr && lane < AR_MAX) {
      float v = 0.f;
#pragma unroll
      for (int j = 0; j < AR_MAX; ++j) v = lane == j ? f[j] : v;
      ar.phi[row * AR_MAX + lane] = v;
    }
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

}  // namespace mmf
