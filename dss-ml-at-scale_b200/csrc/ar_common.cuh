// ar_common.cuh -- the warp-per-series building blocks of the AR-error kernels (ar.cu: ar_kernel, ar_select_kernel;
// arima.cu: arima_kernel): one warp per series, lanes over t, the whitened design rows staged in shared memory one
// TC-row chunk at a time and shared by the WARPS series of a CTA (all series share the calendar).
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

__device__ __forceinline__ bool finite_f(float v) { return (__float_as_uint(v) & 0x7f800000u) != 0x7f800000u; }

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

}  // namespace
}  // namespace mmf
