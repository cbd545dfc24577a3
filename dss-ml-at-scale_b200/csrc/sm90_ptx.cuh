// sm90_ptx.cuh -- thin inline-PTX wrappers for the Hopper (sm_90a) features the tensor-core
// kernels use: mbarrier, TMA (cp.async.bulk.tensor / bulk stores) and wgmma.mma_async (tf32, A from
// registers, B from a swizzled shared-memory tile).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sm90 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier -------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a protocol bug traps after ~2 s (-> a CUDA error through the C ABI) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = global_timer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 1023u) == 0u && global_timer_ns() - t0 > 2000000000ull) __trap();
  }
}

// ---- programmatic dependent launch ----------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- TMA -------------------------------------------------------------------
constexpr uint64_t L2_EVICT_NORMAL = 0x1000000000000000ull;
constexpr uint64_t L2_EVICT_FIRST = 0x12F0000000000000ull;
constexpr uint64_t L2_EVICT_LAST = 0x14F0000000000000ull;

__device__ __forceinline__ void prefetch_tensormap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// A tensor map that lives in GLOBAL memory (written by the host before the launch, e.g. one map per calendar of a
// ragged batch) must be acquired by the tensormap proxy before its first use in a TMA instruction.
__device__ __forceinline__ void fence_tensormap_acquire(const void* tmap) {
  asm volatile("fence.proxy.tensormap::generic.acquire.sys [%0], 128;" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2-D tiled load global -> shared, completion on an mbarrier (complete_tx::bytes)
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const void* tmap, uint32_t bar,
                                            int32_t c0, int32_t c1, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}

// warp-converged: all lanes call with warp-uniform operands, one elected lane arms the barrier and issues
__device__ __forceinline__ void tma_load_2d_x2_elect(uint32_t bar, uint32_t tx_bytes,
                                                     uint32_t dst0, const void* tmap0, int32_t c00, int32_t c01, uint64_t hint0,
                                                     uint32_t dst1, const void* tmap1, int32_t c10, int32_t c11, uint64_t hint1) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t"
      "@pe cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%2], [%3, {%4, %5}], [%0], %6;\n\t"
      "@pe cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%7], [%8, {%9, %10}], [%0], %11;\n\t}"
      ::"r"(bar), "r"(tx_bytes),
        "r"(dst0), "l"(reinterpret_cast<uint64_t>(tmap0)), "r"(c00), "r"(c01), "l"(hint0),
        "r"(dst1), "l"(reinterpret_cast<uint64_t>(tmap1)), "r"(c10), "r"(c11), "l"(hint1)
      : "memory");
}

// split form: arm the barrier, then issue loads separately (lets the producer order its loads freely)
__device__ __forceinline__ void mbar_expect_tx_elect(uint32_t bar, uint32_t bytes) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}"
      ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_issue_2d_elect(uint32_t bar, uint32_t dst, const void* tmap, int32_t c0, int32_t c1,
                                                   uint64_t hint) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%1], [%2, {%3, %4}], [%0], %5;\n\t}"
      ::"r"(bar), "r"(dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_elect(uint32_t bar, uint32_t tx_bytes, uint32_t dst, const void* tmap,
                                                  int32_t c0, int32_t c1, uint64_t hint) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t"
      "@pe cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%2], [%3, {%4, %5}], [%0], %6;\n\t}"
      ::"r"(bar), "r"(tx_bytes), "r"(dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "l"(hint)
      : "memory");
}

// bulk (TMA, non-tensor) store shared -> global of a contiguous block; warp-converged, one elected lane issues.
// The destination may be local or a peer-mapped (NVLink) address.
__device__ __forceinline__ void bulk_store_elect(uint64_t dst_global, uint32_t src_smem, uint32_t bytes) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n\t}"
      ::"l"(dst_global), "r"(src_smem), "r"(bytes)
      : "memory");
}
// the same with an L2 cache-eviction policy for the written lines (L2_EVICT_*)
__device__ __forceinline__ void bulk_store_hint_elect(uint64_t dst_global, uint32_t src_smem, uint32_t bytes, uint64_t hint) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;\n\t}"
      ::"l"(dst_global), "r"(src_smem), "r"(bytes), "l"(hint)
      : "memory");
}
__device__ __forceinline__ void bulk_commit_elect() {
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe cp.async.bulk.commit_group;\n\t}" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_read_elect() {       // the elected lane's pending bulk stores have read smem
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe cp.async.bulk.wait_group.read 0;\n\t}" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_read1_elect() {      // all but the most recent bulk group have read smem
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe cp.async.bulk.wait_group.read 1;\n\t}" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_all_elect() {        // ... and have been written to global
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe cp.async.bulk.wait_group 0;\n\t}" ::: "memory");
}
// plain stores with an L2 eviction policy (a policy register made by createpolicy, not the TMA hint constants above)
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void stg128_hint(void* dst, float4 v, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
               ::"l"(dst), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(policy) : "memory");
}
__device__ __forceinline__ void stg32_hint(void* dst, uint32_t v, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.b32 [%0], %1, %2;" ::"l"(dst), "r"(v), "l"(policy) : "memory");
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// 2-D tiled store shared -> global through a tensor map (clips at the tensor bounds); warp-converged, elected lane
__device__ __forceinline__ void tma_store_2d_elect(const void* tmap, uint32_t src_smem, int32_t c0, int32_t c1) {
  asm volatile(
      "{\n\t.reg .pred pe;\n\t"
      "elect.sync _|pe, 0xffffffff;\n\t"
      "@pe cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];\n\t}"
      ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(src_smem), "r"(c0), "r"(c1)
      : "memory");
}

// ---- wgmma ---------------------------------------------------------------------
// Shared-memory matrix descriptor (sm_90 GMMA), K-major, 32-bit elements, tile base aligned to the swizzle atom:
//   SW128: rows are 128 B (32 elements), 8-row groups 1024 B apart;  SW64: rows are 64 B, 8-row groups 512 B apart.
// A k-step of 8 tf32 inside a row advances the start address by 32 B (+2 in 16-B units).
__device__ __forceinline__ uint64_t gmma_desc_k(uint32_t smem_addr, uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);        // start address  [0,14)
  d |= static_cast<uint64_t>(1) << 16;                            // LBO (unused for swizzled K-major) [16,30)
  d |= static_cast<uint64_t>(sbo_bytes >> 4) << 32;               // SBO            [32,46)
  d |= static_cast<uint64_t>(layout) << 62;                       // 1 = SWIZZLE_128B, 2 = SWIZZLE_64B
  return d;
}
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(uint32_t smem_addr) { return gmma_desc_k(smem_addr, 1024, 1); }
__device__ __forceinline__ uint64_t gmma_desc_k_sw64(uint32_t smem_addr) { return gmma_desc_k(smem_addr, 512, 2); }

// warpgroup-wide (128 threads, converged): order register writes before the async MMAs, close / wait a group
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int N>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] += A[64 x 8] * B[8 x N], tf32 in, fp32 accumulate.  A from registers in the m16n8k8 fragment layout of
// each warp's 16 rows (a0 = (g, t), a1 = (g + 8, t), a2 = (g, t + 4), a3 = (g + 8, t + 4); g = lane / 4, t = lane % 4),
// B K-major through a shared-memory descriptor.  D per n8 block i: d[4i..4i+3] = (g, 8i+2t), (g, 8i+2t+1),
// (g + 8, 8i+2t), (g + 8, 8i+2t+1).
__device__ __forceinline__ void wgmma_m64n32k8_tf32_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));
}
__device__ __forceinline__ void wgmma_m64n128k8_tf32_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));
}

__device__ __forceinline__ void sts128(uint32_t addr, float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}

}  // namespace sm90
