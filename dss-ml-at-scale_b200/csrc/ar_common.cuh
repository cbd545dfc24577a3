// ar_common.cuh -- the building blocks of the ARIMA-family warp kernels (ar.cu: ar_kernel, ar_select_kernel; arima.cu:
// arima_kernel, arima_select_kernel; arma.cu: arma_kernel; arma_select.cu: arma_select_kernel): one warp per series,
// lanes over t, the whitened design rows staged in shared memory one TC-row chunk at a time and shared by the WARPS
// series of a CTA (all series share the calendar).  Each helper here exists once; a kernel uses one only where that
// leaves its SASS as it was (DESIGN.md 4.17), and keeps its other blocks written out.
#pragma once
#include "mmf_internal.cuh"

namespace mmf {
namespace {

constexpr int WARPS = 8;                   // series per CTA (80 registers: 3 CTAs per SM)
constexpr int THREADS = WARPS * 32;
constexpr int TC = 128;                    // design rows per staged chunk: 4 x 128 float4 = 8 KB
constexpr int NSUB = TC / 32;              // 32-row steps of a warp per staged chunk
static_assert((4 * TC) % THREADS == 0, "whole float4s of the staged chunk per thread");
constexpr int AR_MAX = MMF_AR_MAX;
constexpr int MA_MAX = MMF_MA_MAX;
// Rows past the latest restart of pass B that ar.cu and arima.cu allow: 0.  The negative-control build
// (-DMMF_AR_LATE_RESTART, tests/test_gpu_arima_contract.py) allows one row past S, where the state need not be made of
// observations, so that a prediction depends on the requested window.  Never loaded by the product.
#ifdef MMF_AR_LATE_RESTART
constexpr int LATE_RESTART = 1;
#else
constexpr int LATE_RESTART = 0;
#endif

__device__ __forceinline__ bool finite_f(float v) { return (__float_as_uint(v) & 0x7f800000u) != 0x7f800000u; }
__device__ __forceinline__ float qnan() { return __int_as_float(0x7fc00000); }
__device__ __forceinline__ double dnan() { return __longlong_as_double(0x7ff8000000000000ll); }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// value of lane (lane - k) of the sequence "previous chunk, this chunk": lanes below k read the previous chunk's tail
__device__ __forceinline__ float lagged(float cur, float prev, int k, int lane) {
  const float src = lane < 32 - k ? cur : prev;
  return __shfl_sync(0xffffffffu, src, (lane - k) & 31);
}

// stage design rows [c0, c0 + TC) of the column-blocked a4 table and their non-zero column masks (zero beyond the table)
__device__ __forceinline__ void stage(float4 (*s_a)[TC], uint32_t* s_nz, const DesignView& d, const ArArgs& ar, int c0) {
#pragma unroll
  for (int i = threadIdx.x; i < 4 * TC; i += THREADS) {
    const int j = i / TC, r = i % TC, t = c0 + r;
    s_a[j][r] = t < d.n_rows_pad ? __ldg(d.a4 + (size_t)j * d.n_rows_pad + t) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (threadIdx.x < TC) s_nz[threadIdx.x] = c0 + (int)threadIdx.x < d.n_rows ? __ldg(ar.nz + c0 + threadIdx.x) : 0u;
}

__device__ __forceinline__ float fitted(float4 (*s_a)[TC], int r, const float (&g)[P], float c) {
  float v = c;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 a4 = s_a[j][r];
    v = fmaf(a4.x, g[4 * j], v); v = fmaf(a4.y, g[4 * j + 1], v);
    v = fmaf(a4.z, g[4 * j + 2], v); v = fmaf(a4.w, g[4 * j + 3], v);
  }
  return v;
}

// the fit's hand-off of `row` (FitArgs::status, out_gamma, out_c): its status, gamma and c; EMPTY and zeros past the batch
__device__ __forceinline__ int load_fit(const FitArgs& a, int64_t row, bool live, float (&g)[P], float& c) {
  int st = MMF_STATUS_EMPTY;
  c = 0.f;
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
  return st;
}

// used columns k of the dof rule (section 2 item 7) and their mask (arma_joint.cu's J): the calendar's kept columns that are non-zero on an observed fit row
// (colmask, per lane; a column that is zero there has a zero pivot and is skipped, as in the fit kernels), less those the
// pivoted solve dropped for the series' mask (status 2 only; a dropped column's gamma is pinned to exactly 0)
__device__ __forceinline__ uint32_t used_mask(const DesignView& d, uint32_t colmask, int st, const float (&g)[P]) {
  uint32_t used = d.kept_mask & __reduce_or_sync(0xffffffffu, colmask);
  if (st == MMF_STATUS_RANKDEF) {
#pragma unroll
    for (int q = 0; q < P; ++q) used &= g[q] != 0.f ? ~0u : ~(1u << q);
  }
  return used;
}
__device__ __forceinline__ int used_columns(const DesignView& d, uint32_t colmask, int st, const float (&g)[P]) {
  return __popc(used_mask(d, colmask, st, g));
}

// out[row][0 .. N) = v, lane k writing v[k] (nothing when out is null)
template <int N>
__device__ __forceinline__ void store_row(float* out, int64_t row, int lane, const float (&v)[N]) {
  if (out != nullptr && lane < N) {
    float x = 0.f;
#pragma unroll
    for (int k = 0; k < N; ++k) x = lane == k ? v[k] : x;
    out[row * N + lane] = x;
  }
}

// yhat_t from zhat_t and the filled levels ytilde_{t-1} (l1), ytilde_{t-2} (l2), in the order include/mmf.h states
__device__ __forceinline__ float integrate(float zh, float l1, float l2, int d) {
  return d == 1 ? __fadd_rn(zh, l1) : __fsub_rn(__fadd_rn(zh, __fmul_rn(2.f, l1)), l2);
}

// ---- ARIMA(p, d, q): Hannan-Rissanen (arma.cu, arma_select.cu) ------------------------------------------------------

// step-down (reverse Levinson) of 1 - sum_j a_j z^j, a[0 .. k): true when every |kappa| < MMF_AR_KAPPA_MAX
template <int N>
__device__ bool step_down_ok(double (&a)[N], int k) {
  for (int j = k; j >= 1; --j) {
    const double kap = a[j - 1];
    if (!(fabs(kap) < (double)MMF_AR_KAPPA_MAX)) return false;
    const double den = 1.0 - kap * kap;
    double nxt[N];
    for (int i = 1; i < j; ++i) nxt[i - 1] = (a[i - 1] + kap * a[j - i - 1]) / den;
    for (int i = 1; i < j; ++i) a[i - 1] = nxt[i - 1];
  }
  return true;
}

// the rings move on by 32 rows: the current rows become the previous ones
__device__ __forceinline__ void hr_rings_shift(double* __restrict__ sE, double* __restrict__ sU, double* __restrict__ sV,
                                               double ed) {
  const int lane = threadIdx.x & 31;
  sE[lane] = ed;
  sU[lane] = sU[32 + lane];
  sV[lane] = sV[32 + lane];
}

}  // namespace
}  // namespace mmf
