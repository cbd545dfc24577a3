// read_probe.cu -- how fast can one H100 read the flagship's series buffer, and with which TMA load pattern?
//
// The buffer has the flagship layout: 1 M rows of t_fit = 1,095 floats at a pitch of 1,096 floats (4.38 GB).  Every TMA
// kernel here mirrors fit_tc_kernel's producer: one CTA per SM persistent over 128-row tiles (tile = blockIdx.x +
// k * gridDim.x), a 160-KB ring, the series seen through a tensor map clipped at (t_fit, n) with the evict-first hint,
// one {32 x 32} design box per chunk (evict-last, an L2 hit).  The consumers only wait on the full barrier and release
// the slot, so each kernel's time is the read pattern's own.
//   C        coalesced float4 read-and-reduce of the whole buffer (the ceiling)
//   P0       one {32 t x 128 rows} box per ring stage (fit_tc's pattern before multi-chunk slots)
//   P1(G)    G consecutive chunks per slot as {32 x 8} boxes, octet-major: octet 0 of chunks k..k+G-1, then octet 1, ...
//   P2(G)    the same with {32 x 32} boxes
//   P0a      P0 on a 1,120-float (128-B aligned) pitch: the price of rows that straddle L2 lines
//   P0_dyn       P0 with tiles claimed through a global atomic counter (one claim ahead) instead of the static stride
//   P0_nodesign  P0 without the design box (diagnostic: what the design's L2 reads cost)
//   P0_bulk      P0 plus fit_tc's forecast store: after each tile four epilogue warps bulk-store (cp.async.bulk,
//                evict-first) a 14-KB staging tile into a 112-MB table
//   P0_warp      the same bytes written by the four epilogue warps as coalesced 16-B evict-first stores from the
//                staging tile (one warp instruction = 512 contiguous bytes)
// Usage: read_probe [rounds]   -- runs the variants alternately and prints one line per launch:
//   <name> <ms> <GB/s of the 4 * n * t_fit series bytes>
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../sm90_ptx.cuh"

using namespace sm90;

namespace {

constexpr int64_t N = 1000000;        // the flagship batch: 7,813 tiles, the last one 64 rows (clipped at n)
constexpr int T_FIT = 1095, PITCH = 1096, PITCH_ALIGNED = 1120;
constexpr int KC = 32, TILE_M = 128, N_CHUNKS = (T_FIT + KC - 1) / KC;
constexpr int Y_CHUNK = TILE_M * KC * 4, AT_CHUNK = 32 * KC * 4;    // 16 KB + 4 KB per chunk
constexpr int RING = 8 * (Y_CHUNK + AT_CHUNK);                       // 160 KB, fit_tc's ring
constexpr int CONSUMER_WARPS = 8, THREADS = 32 * (CONSUMER_WARPS + 1);
constexpr int EPI_WARPS = 4, THREADS_EPI = THREADS + 32 * EPI_WARPS;   // the store variants add fit_tc's epilogue warps
constexpr int N_PRED = 28, OSTAGE = TILE_M * N_PRED * 4;             // 14 KB of forecasts per tile
constexpr int TILE_RING = 4;                                         // P0_dyn: claimed tiles in flight

enum Mode { PLAIN = 0, DYN, NODESIGN, BULK, WARP };

#define CK(x)                                                                                   \
  do {                                                                                          \
    cudaError_t e_ = (x);                                                                       \
    if (e_ != cudaSuccess) {                                                                    \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));        \
      exit(1);                                                                                  \
    }                                                                                           \
  } while (0)

struct Maps {
  CUtensorMap y;      // {32, BOX_ROWS} over (t_fit, n)
  CUtensorMap at;     // {32, 32} over the design's (t_pad, 32)
};

// G chunks per slot, BOX_ROWS rows per y box (128: one box per chunk).  Slot layout: [row block][chunk][BOX_ROWS][128 B]
// then the G design boxes.  MODE (enum Mode) selects the P0 variants; ctr / ctr_next are P0_dyn's claim counters (this
// launch's and the next one's, which this launch zeroes), out the store variants' forecast table.
template <int G, int BOX_ROWS, int MODE = PLAIN>
__global__ void __launch_bounds__(THREADS_EPI, 1) tma_read_kernel(const __grid_constant__ Maps m, int n_tiles,
                                                                  uint32_t* ctr, uint32_t* ctr_next, float* out) {
  constexpr bool STORE = MODE == BULK || MODE == WARP;
  constexpr int SLOT = G * (Y_CHUNK + AT_CHUNK);
  constexpr int SLOTS = RING / SLOT;
  constexpr int BOX_BYTES = BOX_ROWS * KC * 4;
  constexpr int N_BLOCKS = TILE_M / BOX_ROWS;
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  const uint32_t s_ring = smem_u32(smem);
  float* s_ostage = reinterpret_cast<float*>(smem + RING);
  const uint32_t s_bars = s_ring + RING + OSTAGE;
  int* s_tiles = reinterpret_cast<int*>(smem + RING + OSTAGE + 8 * (2 * SLOTS + 2 * TILE_RING + 4));
  auto bar_full = [&](int s) { return s_bars + 8u * s; };
  auto bar_empty = [&](int s) { return s_bars + 8u * (SLOTS + s); };
  auto bar_tfull = [&](int s) { return s_bars + 8u * (2 * SLOTS + s); };              // P0_dyn's tile ring
  auto bar_tempty = [&](int s) { return s_bars + 8u * (2 * SLOTS + TILE_RING + s); };
  auto bar_done = [&](int b) { return s_bars + 8u * (2 * SLOTS + 2 * TILE_RING + b); };   // store variants: tile
  auto bar_free = [&](int b) { return s_bars + 8u * (2 * SLOTS + 2 * TILE_RING + 2 + b); };  // consumed / hand-off read
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < SLOTS; ++s) {
      mbar_init(bar_full(s), 1);
      mbar_init(bar_empty(s), CONSUMER_WARPS);
    }
    for (int s = 0; s < TILE_RING; ++s) {
      mbar_init(bar_tfull(s), 1);
      mbar_init(bar_tempty(s), CONSUMER_WARPS);
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(bar_done(b), CONSUMER_WARPS);
      mbar_init(bar_free(b), EPI_WARPS);
    }
    fence_mbar_init();
    prefetch_tensormap(&m.y);
    prefetch_tensormap(&m.at);
    if (MODE == DYN && blockIdx.x == 0) *ctr_next = 0u;
  }
  __syncthreads();
  if (warp == CONSUMER_WARPS) {
    int slot = 0;
    uint32_t phase = 0;
    int tile = blockIdx.x, lt = 0;
    auto publish = [&](int t) {            // P0_dyn: hand the claimed tile to the consumers
      const int s = lt % TILE_RING;
      mbar_wait(bar_tempty(s), ((lt / TILE_RING) & 1) ^ 1u);
      if (lane == 0) {
        s_tiles[s] = t;
        mbar_arrive(bar_tfull(s));
      }
      __syncwarp();
    };
    for (; tile < n_tiles; ++lt) {
      uint32_t claim = 0;
      if (MODE == DYN) {
        if (lane == 0) claim = atomicAdd(ctr, 1u);     // one claim ahead: its latency hides under this tile
        publish(tile);
      }
      for (int k = 0; k < N_CHUNKS; k += G) {
        const int g = N_CHUNKS - k < G ? N_CHUNKS - k : G;
        mbar_wait(bar_empty(slot), phase ^ 1u);
        const uint32_t base = s_ring + slot * SLOT;
        mbar_expect_tx_elect(bar_full(slot), static_cast<uint32_t>(g) * (Y_CHUNK + (MODE == NODESIGN ? 0 : AT_CHUNK)));
        if (MODE != NODESIGN)
          for (int j = 0; j < g; ++j)
            tma_issue_2d_elect(bar_full(slot), base + G * Y_CHUNK + j * AT_CHUNK, &m.at, (k + j) * KC, 0, L2_EVICT_LAST);
        for (int b = 0; b < N_BLOCKS; ++b)
          for (int j = 0; j < g; ++j)
            tma_issue_2d_elect(bar_full(slot), base + (b * G + j) * BOX_BYTES, &m.y, (k + j) * KC,
                               tile * TILE_M + b * BOX_ROWS, L2_EVICT_FIRST);
        if (++slot == SLOTS) { slot = 0; phase ^= 1u; }
      }
      tile = MODE == DYN ? static_cast<int>(gridDim.x + __shfl_sync(0xffffffffu, claim, 0)) : tile + static_cast<int>(gridDim.x);
    }
    if (MODE == DYN) publish(-1);
  } else if (warp < CONSUMER_WARPS) {
    int slot = 0;
    uint32_t phase = 0;
    int tile = blockIdx.x;
    for (int lt = 0;; ++lt) {
      if (MODE == DYN) {
        const int s = lt % TILE_RING;
        mbar_wait(bar_tfull(s), (lt / TILE_RING) & 1);
        tile = *reinterpret_cast<volatile int*>(s_tiles + s);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_tempty(s));
        if (tile < 0) break;
      } else if (lt > 0) {
        tile += gridDim.x;
      }
      if (tile >= n_tiles) break;
      for (int k = 0; k < N_CHUNKS; k += G) {
        mbar_wait(bar_full(slot), phase);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty(slot));
        if (++slot == SLOTS) { slot = 0; phase ^= 1u; }
      }
      if (STORE) {                         // hand the finished tile to the epilogue (double-buffered, as fit_tc)
        mbar_wait(bar_free(lt & 1), ((lt >> 1) & 1) ^ 1u);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_done(lt & 1));
      }
    }
  } else if (STORE) {
    // epilogue warps: stage a 128 x 28 forecast tile (each thread its row, as fit_tc), then store it
    const int r = threadIdx.x - (CONSUMER_WARPS + 1) * 32;
    const uint64_t pol = l2_evict_first_policy();
    const uint32_t s_ostage_u32 = smem_u32(s_ostage);
    int lt = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++lt) {
      mbar_wait(bar_done(lt & 1), (lt >> 1) & 1);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_free(lt & 1));
      const int64_t left = N - (int64_t)tile * TILE_M;
      const int nrows = left >= TILE_M ? TILE_M : static_cast<int>(left);
      if (MODE == BULK && r < 32) bulk_wait_read_elect();
      named_bar_sync(1, 128);
      float* srow = s_ostage + r * N_PRED;
      for (int k = 0; k < N_PRED; k += 4) *reinterpret_cast<float4*>(srow + k) = make_float4(1.f, 2.f, 3.f, 4.f);
      if (MODE == BULK) fence_proxy_async_smem();
      named_bar_sync(1, 128);
      float* dst = out + (int64_t)tile * TILE_M * N_PRED;
      if (MODE == BULK) {
        if (r < 32) {
          bulk_store_hint_elect(reinterpret_cast<uint64_t>(dst), s_ostage_u32, static_cast<uint32_t>(nrows) * N_PRED * 4u,
                                L2_EVICT_FIRST);
          bulk_commit_elect();
        }
      } else {
        for (int i = r; i < nrows * (N_PRED / 4); i += 128)
          stg128_hint(reinterpret_cast<float4*>(dst) + i, lds128(s_ostage_u32 + 16u * i), pol);
      }
    }
    if (MODE == BULK && r < 32) bulk_wait_all_elect();
  }
}

__global__ void read_reduce_kernel(const float4* __restrict__ p, int64_t n4, float* __restrict__ out) {
  float s = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = __ldcs(p + i);
    s += (v.x + v.y) + (v.z + v.w);
  }
  if (s == 12345.f) *out = s;      // never true for the zero-filled buffer; keeps the loads
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

CUtensorMap encode(const void* p, uint64_t inner, uint64_t outer, uint64_t pitch_bytes, uint32_t box_outer) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* q = nullptr;
    cudaDriverEntryPointQueryResult r;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &q, cudaEnableDefault, &r));
    if (r != cudaDriverEntryPointSuccess) { fprintf(stderr, "cuTensorMapEncodeTiled not available\n"); exit(1); }
    fn = reinterpret_cast<EncodeTiledFn>(q);
  }
  CUtensorMap m;
  cuuint64_t dims[2] = {inner, outer}, strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {KC, box_outer}, estr[2] = {1, 1};
  CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(p), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { fprintf(stderr, "cuTensorMapEncodeTiled failed: %d\n", (int)r); exit(1); }
  return m;
}

struct Bufs {
  uint32_t* ctr;      // two claim counters: launch i claims through ctr[i & 1] and zeroes the other
  float* out;         // the forecast table of the store variants, n x N_PRED
};

struct Variant {
  const char* name;
  void (*launch)(const Maps&, const Bufs&, int, int, cudaStream_t);
  int box_rows;
  bool aligned;
};

template <int G, int BOX_ROWS, int MODE = PLAIN>
void launch_tma(const Maps& m, const Bufs& b, int grid, int n_tiles, cudaStream_t s) {
  const int smem = RING + OSTAGE + 1024 + 64 * 8;
  static bool set = false;
  static int parity = 0;
  if (!set) {
    CK(cudaFuncSetAttribute(tma_read_kernel<G, BOX_ROWS, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    set = true;
  }
  const int threads = MODE == BULK || MODE == WARP ? THREADS_EPI : THREADS;
  tma_read_kernel<G, BOX_ROWS, MODE><<<grid, threads, smem, s>>>(m, n_tiles, b.ctr + parity, b.ctr + (parity ^ 1), b.out);
  if (MODE == DYN) parity ^= 1;
}

}  // namespace

int main(int argc, char** argv) {
  const int rounds = argc > 1 ? atoi(argv[1]) : 7;
  int dev = 0, sms = 0;
  CK(cudaSetDevice(dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const size_t buf_bytes = (size_t)N * PITCH_ALIGNED * 4;          // big enough for either pitch
  float* y = nullptr;
  float* at = nullptr;
  float* sink = nullptr;
  CK(cudaMalloc(&y, buf_bytes));
  CK(cudaMemset(y, 0, buf_bytes));
  const int t_pad = N_CHUNKS * KC;
  CK(cudaMalloc(&at, (size_t)32 * t_pad * 4));
  CK(cudaMemset(at, 0, (size_t)32 * t_pad * 4));
  CK(cudaMalloc(&sink, 4));
  Bufs bufs{};
  CK(cudaMalloc(&bufs.ctr, 2 * sizeof(uint32_t)));
  CK(cudaMemset(bufs.ctr, 0, 2 * sizeof(uint32_t)));
  CK(cudaMalloc(&bufs.out, (size_t)N * N_PRED * 4));
  const int n_tiles = (int)((N + TILE_M - 1) / TILE_M);
  const int grid = n_tiles < sms ? n_tiles : sms;

  Maps m128, m8, m32, m128a;
  const CUtensorMap mat = encode(at, t_pad, 32, (uint64_t)t_pad * 4, 32);
  m128 = Maps{encode(y, T_FIT, N, (uint64_t)PITCH * 4, 128), mat};
  m8 = Maps{encode(y, T_FIT, N, (uint64_t)PITCH * 4, 8), mat};
  m32 = Maps{encode(y, T_FIT, N, (uint64_t)PITCH * 4, 32), mat};
  m128a = Maps{encode(y, T_FIT, N, (uint64_t)PITCH_ALIGNED * 4, 128), mat};

  const Variant vs[] = {
      {"C", nullptr, 0, false},
      {"P0", launch_tma<1, 128>, 128, false},
      {"P1_G2", launch_tma<2, 8>, 8, false},
      {"P1_G4", launch_tma<4, 8>, 8, false},
      {"P2_G2", launch_tma<2, 32>, 32, false},
      {"P2_G4", launch_tma<4, 32>, 32, false},
      {"P0_aligned", launch_tma<1, 128>, 128, true},
      {"P0_dyn", launch_tma<1, 128, DYN>, 128, false},
      {"P0_nodesign", launch_tma<1, 128, NODESIGN>, 128, false},
      {"P0_bulk", launch_tma<1, 128, BULK>, 128, false},
      {"P0_warp", launch_tma<1, 128, WARP>, 128, false},
  };
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  const double bytes = 4.0 * (double)N * T_FIT;       // the series values a fit reads
  const double bytes_c = 4.0 * (double)N * PITCH;     // C also reads the padding column
  const int64_t n4 = N * PITCH / 4;
  auto run = [&](const Variant& v) {
    if (v.launch == nullptr) {
      read_reduce_kernel<<<sms * 8, 512>>>(reinterpret_cast<const float4*>(y), n4, sink);
    } else {
      const Maps& m = v.aligned ? m128a : (v.box_rows == 8 ? m8 : v.box_rows == 32 ? m32 : m128);
      v.launch(m, bufs, grid, n_tiles, 0);
    }
  };
  for (const Variant& v : vs) { run(v); run(v); }        // warm-up: module load, first-touch of every map
  CK(cudaDeviceSynchronize());
  CK(cudaGetLastError());
  printf("# sms %d grid %d n %lld t_fit %d pitch %d bytes %.0f\n", sms, grid, (long long)N, T_FIT, PITCH, bytes);
  for (int r = 0; r < rounds; ++r)
    for (const Variant& v : vs) {
      CK(cudaEventRecord(e0));
      const int reps = 5;
      for (int i = 0; i < reps; ++i) run(v);
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      CK(cudaGetLastError());
      float ms = 0.f;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      ms /= reps;
      printf("%s %.4f %.1f\n", v.name, ms, (v.launch ? bytes : bytes_c) / (ms * 1e-3) / 1e9);
      fflush(stdout);
    }
  CK(cudaFree(y));
  CK(cudaFree(at));
  CK(cudaFree(sink));
  CK(cudaFree(bufs.ctr));
  CK(cudaFree(bufs.out));
  return 0;
}
