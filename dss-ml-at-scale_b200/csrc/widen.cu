// widen.cu -- integer demand columns -> the float32 series rows the fit kernels read.
//
// The reference's demand is integer valued (01-data-generator.py:304 `round`) but travels as float32
// (enriched_schema, 02:360-370).  With host-resident input the whole path is PCIe-bound, so an int16 / uint16
// (or int32) value column halves (keeps) the bytes that cross the link; this kernel widens a staged chunk on the
// device: y32[i, t] = (float) y_int[i, t], the type's sentinel -> NaN (= missing, like a float NaN).
// Exact for every representable value (|v| < 2^24 for int32), so the forecasts are bit-equal to a float32 ingest.
// Bound: HBM, 2 (4) B read + 4 B written per value -- noise next to the PCIe copy that feeds it.
#include "mmf_internal.cuh"

namespace mmf {
namespace {

constexpr int TPB = 256;

template <typename T> struct Sentinel;
template <> struct Sentinel<int16_t>  { static constexpr int32_t v = -32768; };
template <> struct Sentinel<uint16_t> { static constexpr int32_t v = 65535; };
template <> struct Sentinel<int32_t>  { static constexpr int32_t v = INT32_MIN; };

template <typename T>
__device__ __forceinline__ float widen_one(T x) {
  return static_cast<int32_t>(x) == Sentinel<T>::v ? __int_as_float(0x7fc00000) : static_cast<float>(x);
}

// 8 values per 16-B (int16) / 32-B (int32) load, two 16-B stores.  A 64-thread quarter of the block owns a row at a time
// and strides over its groups of 8 (no integer division per element: the first version computed row = i / groups in 64
// bits for every group and ran at 1.3 TB/s whatever the unrolling); the loads of a row are
// issued before its stores.  Rows are walked with a pitch, so a group never straddles a row; the tail of a row (t % 8)
// takes the scalar path.
constexpr int QUART = 64;                      // threads per row
constexpr int ROWS_PER_BLOCK = TPB / QUART;    // 4 rows in flight per block
constexpr int MAXG = 4;                        // groups of 8 per thread and row handled in registers (t <= 2,048), else looped

template <typename T>
__global__ void __launch_bounds__(TPB)
widen_kernel(const T* __restrict__ src, int64_t ld_src, float* __restrict__ dst, int64_t ld_dst, int64_t n, int32_t t,
             int vec_ok) {
  const int sub = threadIdx.x / QUART, lane = threadIdx.x % QUART;
  const int groups = (t + 7) >> 3;
  for (int64_t row = (int64_t)blockIdx.x * ROWS_PER_BLOCK + sub; row < n; row += (int64_t)gridDim.x * ROWS_PER_BLOCK) {
    const T* __restrict__ s = src + row * ld_src;
    float* __restrict__ d = dst + row * ld_dst;
    for (int g0 = 0; g0 < groups; g0 += QUART * MAXG) {
      T v[MAXG][8];
#pragma unroll
      for (int u = 0; u < MAXG; ++u) {
        const int g = g0 + u * QUART + lane;
        if (g < groups && vec_ok && (g << 3) + 8 <= t) {
          if (sizeof(T) == 2) {
            *reinterpret_cast<uint4*>(v[u]) = __ldcs(reinterpret_cast<const uint4*>(s + (g << 3)));
          } else {
            reinterpret_cast<uint4*>(v[u])[0] = __ldcs(reinterpret_cast<const uint4*>(s + (g << 3)));
            reinterpret_cast<uint4*>(v[u])[1] = __ldcs(reinterpret_cast<const uint4*>(s + (g << 3)) + 1);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < MAXG; ++u) {
        const int g = g0 + u * QUART + lane;
        if (g >= groups) continue;
        const int c0 = g << 3;
        if (vec_ok && c0 + 8 <= t) {
          __stcs(reinterpret_cast<float4*>(d + c0), make_float4(widen_one(v[u][0]), widen_one(v[u][1]), widen_one(v[u][2]), widen_one(v[u][3])));
          __stcs(reinterpret_cast<float4*>(d + c0 + 4), make_float4(widen_one(v[u][4]), widen_one(v[u][5]), widen_one(v[u][6]), widen_one(v[u][7])));
        } else {
          for (int k = 0; k < 8 && c0 + k < t; ++k) d[c0 + k] = widen_one(s[c0 + k]);
        }
      }
    }
  }
}

template <typename T>
cudaError_t launch(const void* src, int64_t ld_src, float* dst, int64_t ld_dst, int64_t n, int32_t t, int sm, cudaStream_t s) {
  if (n <= 0 || t <= 0) return cudaSuccess;
  const int vec_ok = ((reinterpret_cast<uintptr_t>(src) & 15u) == 0 && (ld_src * sizeof(T)) % 16 == 0 &&
                      (reinterpret_cast<uintptr_t>(dst) & 15u) == 0 && ld_dst % 4 == 0) ? 1 : 0;
  const int64_t want = (n + ROWS_PER_BLOCK - 1) / ROWS_PER_BLOCK, cap = (int64_t)sm * 16;
  widen_kernel<T><<<(unsigned)(want < cap ? want : cap), TPB, 0, s>>>(static_cast<const T*>(src), ld_src, dst, ld_dst, n, t, vec_ok);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_widen(int dtype, const void* src, int64_t ld_src, float* dst, int64_t ld_dst, int64_t n, int32_t t,
                         int sm_count, cudaStream_t s) {
  switch (dtype) {
    case MMF_DT_I16: return launch<int16_t>(src, ld_src, dst, ld_dst, n, t, sm_count, s);
    case MMF_DT_U16: return launch<uint16_t>(src, ld_src, dst, ld_dst, n, t, sm_count, s);
    case MMF_DT_I32: return launch<int32_t>(src, ld_src, dst, ld_dst, n, t, sm_count, s);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace mmf
