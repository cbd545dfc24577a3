// backtest.cu -- forecast errors of a rolling-origin backtest (mmf_backtest_f32, DESIGN.md section 2 item 8).
//
// One warp per (series, origin), lanes over the horizon: the warp reads origin k's forecast row of series i and the
// actual values y[i, t_k .. t_k + H) (both contiguous), scores the points where both are finite in float64 and
// reduces with shuffles.  Every row is scored here, whichever kernel finished its fit, so there is one definition of
// the metrics:
//   MSE = mean e^2, MAE = mean |e|, bias = mean e (e = forecast - actual), MAPE = mean |e| / |y| over the scored points
//   with y != 0; NaN where nothing is averaged.
// Reference: the hold-out MSE of build_tune_and_score_model (02:453-459) and the MAPE it imports (02:51).
#include "mmf_internal.cuh"

namespace mmf {
namespace {

constexpr int THREADS = 256;

__device__ __forceinline__ bool finite_bits(float x) { return (__float_as_uint(x) & 0x7f800000u) != 0x7f800000u; }

__global__ void __launch_bounds__(THREADS)
backtest_score_kernel(const ScoreArgs sa) {
  const int lane = threadIdx.x & 31;
  const int64_t n_warps = (int64_t)gridDim.x * (THREADS / 32);
  const int64_t total = sa.n * sa.n_origin;
  const bool vec = (reinterpret_cast<uintptr_t>(sa.metrics) & 15u) == 0;
  // origin-major: neighbouring warps read neighbouring rows of one origin block
  for (int64_t w = (int64_t)blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5); w < total; w += n_warps) {
    const int k = (int)(w / sa.n);
    const int64_t i = w - (int64_t)k * sa.n;
    const int tk = __ldg(&sa.cals[k].t_fit);
    const float* __restrict__ pr = sa.pred + ((int64_t)k * sa.pred_kstride + i) * sa.ld_pred;
    const float* __restrict__ yr = sa.y + i * sa.ld_y + tk;
    double se = 0.0, ae = 0.0, bias = 0.0, ape = 0.0;
    int cnt = 0, cnt_ape = 0;
    for (int h = lane; h < sa.horizon; h += 32) {
      const float f = __ldcs(pr + h), v = __ldcs(yr + h);
      if (finite_bits(f) && finite_bits(v)) {
        const double e = static_cast<double>(f) - static_cast<double>(v);
        se = fma(e, e, se);
        ae += fabs(e);
        bias += e;
        ++cnt;
        if (v != 0.f) { ape += fabs(e) / fabs(static_cast<double>(v)); ++cnt_ape; }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      se += __shfl_xor_sync(0xffffffffu, se, o);
      ae += __shfl_xor_sync(0xffffffffu, ae, o);
      bias += __shfl_xor_sync(0xffffffffu, bias, o);
      ape += __shfl_xor_sync(0xffffffffu, ape, o);
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      cnt_ape += __shfl_xor_sync(0xffffffffu, cnt_ape, o);
    }
    if (lane == 0) {
      const int64_t o = (int64_t)k * sa.out_kstride + i;
      if (sa.metrics != nullptr) {
        const float qnan = __int_as_float(0x7fc00000);
        const float4 m = cnt > 0 ? make_float4(static_cast<float>(se / cnt), static_cast<float>(ae / cnt),
                                               static_cast<float>(bias / cnt),
                                               cnt_ape > 0 ? static_cast<float>(ape / cnt_ape) : qnan)
                                 : make_float4(qnan, qnan, qnan, qnan);
        float* dst = sa.metrics + o * MMF_BT_NMETRIC;
        if (vec) {
          __stcs(reinterpret_cast<float4*>(dst), m);
        } else {
          dst[0] = m.x; dst[1] = m.y; dst[2] = m.z; dst[3] = m.w;
        }
      }
      if (sa.count != nullptr) sa.count[o] = cnt;
    }
  }
}

}  // namespace

cudaError_t launch_bt_score(const ScoreArgs& sa, int sm_count, cudaStream_t s) {
  const int64_t total = sa.n * sa.n_origin;
  if (total <= 0 || (sa.metrics == nullptr && sa.count == nullptr)) return cudaSuccess;
  const int64_t want = (total + THREADS / 32 - 1) / (THREADS / 32);
  const int64_t cap = (int64_t)sm_count * 16;
  backtest_score_kernel<<<(unsigned)(want < cap ? want : cap), THREADS, 0, s>>>(sa);
  return cudaGetLastError();
}

}  // namespace mmf
