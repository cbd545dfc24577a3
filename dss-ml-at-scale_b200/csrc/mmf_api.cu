// mmf_api.cu -- the C ABI of libmmf.so (include/mmf.h): context, design plan (float64 calendar
// whitening on the host), kernel dispatch, and the pipelined host-buffer path.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include <sched.h>
#include <thread>

#include "mmf_internal.cuh"

using namespace mmf;

// host_narrow.cpp: exact float32 -> uint16 narrowing of a chunk on a few host threads
namespace mmf {
class NarrowPool;
NarrowPool* narrow_pool_create(int n_threads, bool pin);
void narrow_pool_destroy(NarrowPool* p);
int narrow_pool_size(const NarrowPool* p);
bool narrow_f32_to_u16(NarrowPool* p, const float* src, int64_t ld_src, uint16_t* dst, int64_t ld_dst, int64_t n, int32_t t,
                       bool stream_stores);
void narrow_pool_begin_call(NarrowPool* p);
void narrow_pool_end_call(NarrowPool* p);
}  // namespace mmf

namespace {

thread_local std::string g_err;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

#define CU_TRY(expr)                                                                              \
  do {                                                                                            \
    cudaError_t e__ = (expr);                                                                     \
    if (e__ != cudaSuccess)                                                                       \
      return fail(MMF_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// 2-D fp32 tensor map: dims {inner, outer}, row pitch in bytes, box {box_inner, box_outer}, 128-B swizzle
int encode_2d(void* out128, const void* gptr, uint64_t inner, uint64_t outer, uint64_t pitch_bytes,
              uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(MMF_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(reinterpret_cast<CUtensorMap*>(out128), CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                  const_cast<void*>(gptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MMF_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return MMF_OK;
}

struct Plan {
  bool valid = false;
  int32_t n_rows = 0, n_rows_pad = 0, t_fit = 0, t_pad = 0, has_constant = 0;
  uint32_t kept_mask = 0;
  double W[P * P];
  float4* d_a4 = nullptr;
  float* d_at = nullptr;
  float* d_apred = nullptr;
  float* d_w = nullptr;
  float* d_ap_hi = nullptr;   // [n_rows][P] tf32-hi / tf32-lo of A: B operand of predict_tc_kernel
  float* d_ap_lo = nullptr;
  alignas(64) unsigned char tmap_at[128];
  alignas(64) unsigned char tmap_bhi[128];
  alignas(64) unsigned char tmap_blo[128];
};

// Ragged plan: the whitened designs of many calendars stacked (DESIGN.md 4.8)
struct MultiPlan {
  bool valid = false;
  int32_t n_cal = 0, n_pred = 0, has_constant = 0, t_fit_max = 0, t_pad_max = 0, min_chunks = 0;
  std::vector<CalMeta> cals;           // host copy of d_cals
  std::vector<size_t> a4_off;          // float4 offset of every calendar's a4 block
  CalMeta* d_cals = nullptr;
  float* d_at = nullptr;               // [n_cal * 32][t_pad_max]: hi / lo of A^T per calendar (TMA B operand)
  float* d_apred = nullptr;            // [sum n_rows][P]
  float4* d_a4 = nullptr;              // per-calendar column-blocked blocks (general pass)
  float* d_w = nullptr;                // zeros (beta is not offered for ragged batches)
  uint32_t* d_pending_by_cal = nullptr;
  alignas(64) unsigned char tmap_at[128];
  // requests with many / per-calendar numbers of prediction rows (holdout: a value for every date of every calendar):
  // fit kernels hand gamma / c to predict_tc_kernel<true>
  bool many_pred = false;
  int32_t n_pred_max = 0;
  float* d_ap_hi = nullptr;            // [sum n_rows][P] tf32-hi / lo of the stacked whitened designs (B operand)
  float* d_ap_lo = nullptr;
  alignas(64) unsigned char tmap_bhi[128];
  alignas(64) unsigned char tmap_blo[128];
  PredUnit* d_units = nullptr;  size_t units_cap = 0;  int64_t n_units = 0;
  unsigned char* d_tmaps_out = nullptr;
  const void* key_out = nullptr;  int64_t key_ld_out = -1;
  // per-call tables, kept while the same buffer / row layout is fit again
  TileRec* d_tiles = nullptr;  size_t tiles_cap = 0;  int32_t n_tiles = 0;
  unsigned char* d_tmaps_y = nullptr;
  const void* key_y = nullptr;  int64_t key_n = -1, key_ld = -1;  std::vector<int64_t> key_rows;
};

constexpr int NBUF = 3;

struct Staging {
  float* d_y = nullptr;      size_t y_cap = 0;        // bytes
  void* d_yraw = nullptr;    size_t yraw_cap = 0;     // integer chunk as it left the host (mmf_fit_forecast_int)
  float* d_out = nullptr;    size_t out_cap = 0;
  float* d_beta = nullptr;   size_t beta_cap = 0;
  int32_t* d_status = nullptr; size_t status_cap = 0;
  cudaEvent_t ev_h2d = nullptr, ev_comp = nullptr, ev_d2h = nullptr;
};

// Page-locked HOST slots the narrowed (uint16) sub-chunks are written to and copied from (host_narrow.cpp): the
// narrowing of sub-chunk k+1 runs while the copy of sub-chunk k is in flight.
constexpr int NHOST = 4;
struct HostSlot {
  uint16_t* p = nullptr; size_t cap = 0;
  cudaEvent_t ev = nullptr;              // the copy out of the slot has completed
};

}  // namespace

struct mmf_ctx {
  int device = 0;
  int sm_count = 0;
  mmf_config cfg{};
  cudaStream_t stream = nullptr;       // compute stream (owned or borrowed)
  bool own_stream = false;
  cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
  cudaEvent_t ev_a = nullptr, ev_b = nullptr, ev_k0 = nullptr, ev_k1 = nullptr;
  uint32_t* d_pending = nullptr;       // 3 counter sets of CTR_WORDS words {rows left PENDING, solve records queued,
                                       // claimed, CTAs finished, producer done, ...}: 0/1 ping-pong between
                                       // eager calls, 2 belongs to captured CUDA graphs (zeroed by a node of the graph)
  int counter_set = 0;                 // set the next eager call uses
  bool set_clean[2] = {true, true};    // the set is known to be zero (cudaMemset at create, or zeroed by the previous
                                       // eager call's tensor-core kernel); anything else makes the call memset its set
  int last_set = 0;                    // set the last enqueued call used (stats read n_pending from it)
  int pinned = 0;                      // > 0: a captured CUDA graph holds pointers into the scratch below and into the plan
  bool status_scratch_captured = false;   // some capture ran without a caller-provided status buffer
  SolveRec* d_recs = nullptr;          // deferred masked series (grown on demand, capped)
  size_t recs_cap_bytes = 0;
  int64_t* d_rec_rows = nullptr;
  size_t rec_rows_cap_bytes = 0;
  bool rec_rows_clean = false;         // every entry is -1 (what the streaming solve needs to find; its kernels restore it)
  float* d_gamma = nullptr;            // [n][P] + d_c[n]: hand-off from the fit kernels to predict_tc_kernel
  size_t gamma_cap_bytes = 0;
  float* d_c = nullptr;
  size_t c_cap_bytes = 0;
  int32_t* d_status_scratch = nullptr;
  size_t status_scratch_cap = 0;
  void* d_pack_scratch = nullptr;      // sort / scan work space of the packer (grown on demand, kept)
  size_t pack_scratch_cap = 0;
  Plan plan;
  MultiPlan multi;
  Staging st[NBUF];
  NarrowPool* narrow_pool = nullptr;   // created on the first host-buffer call that narrows
  HostSlot hslot[NHOST];
  uint64_t hslot_uses = 0;
};

namespace {

void free_multi(MultiPlan& m) {
  cudaFree(m.d_cals); cudaFree(m.d_at); cudaFree(m.d_apred); cudaFree(m.d_a4); cudaFree(m.d_w);
  cudaFree(m.d_pending_by_cal); cudaFree(m.d_tiles); cudaFree(m.d_tmaps_y);
  cudaFree(m.d_ap_hi); cudaFree(m.d_ap_lo); cudaFree(m.d_units); cudaFree(m.d_tmaps_out);
  m = MultiPlan{};
}

void free_plan(Plan& p) {
  cudaFree(p.d_a4); cudaFree(p.d_at); cudaFree(p.d_apred); cudaFree(p.d_w); cudaFree(p.d_ap_hi); cudaFree(p.d_ap_lo);
  p = Plan{};
}

// Scratch that a captured CUDA graph points into must not move: while ctx->pinned > 0 a reallocation is refused.
thread_local const mmf_ctx* g_grow_ctx = nullptr;
int grow(void** ptr, size_t* cap, size_t need) {
  if (*cap >= need) return MMF_OK;
  if (g_grow_ctx && g_grow_ctx->pinned > 0)
    return fail(MMF_E_UNSUPPORTED, "a captured CUDA graph holds this context's scratch (%zu B) and the call needs %zu B: "
                "release the graph (mmf_pin_scratch(ctx, -1)) or use another context for larger batches", *cap, need);
  if (*ptr) cudaFree(*ptr);
  *ptr = nullptr; *cap = 0;
  cudaError_t e = cudaMalloc(ptr, need);
  if (e != cudaSuccess) return fail(MMF_E_NOMEM, "cudaMalloc(%zu) failed: %s", need, cudaGetErrorString(e));
  *cap = need;
  return MMF_OK;
}

bool is_device_ptr(const void* p) {
  if (!p) return false;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

DesignView view_of(const Plan& p) {
  DesignView d;
  d.a4 = p.d_a4; d.at = p.d_at; d.apred = p.d_apred; d.w = p.d_w;
  d.n_rows = p.n_rows; d.n_rows_pad = p.n_rows_pad; d.t_fit = p.t_fit; d.t_pad = p.t_pad;
  d.kept_mask = p.kept_mask; d.has_constant = p.has_constant;
  return d;
}


// float64 calendar Gram over the fit rows, in-order Cholesky with aliasing, W = L^-T on the kept columns
// (oracle/mmf_oracle.py: whiten), A = X W in float32.  Shared by the single-calendar and the ragged plan.
void whiten_calendar(const double* X, int32_t n_rows, int32_t p, int32_t t_fit, double* W /*[P*P]*/, uint32_t* kept_mask,
                     std::vector<float>& A /*[n_rows*P]*/) {
  double G[P][P] = {}, L[P][P] = {};
  for (int32_t t = 0; t < t_fit; ++t) {
    const double* x = X + (int64_t)t * p;
    for (int i = 0; i < p; ++i)
      for (int j = 0; j <= i; ++j) G[i][j] += x[i] * x[j];
  }
  for (int i = 0; i < P; ++i)
    for (int j = 0; j < i; ++j) G[j][i] = G[i][j];
  bool kept[P] = {};
  for (int j = 0; j < P; ++j) {
    double dsum = G[j][j];
    for (int k = 0; k < j; ++k) dsum -= L[j][k] * L[j][k];
    if (G[j][j] <= 0.0 || dsum <= MMF_CAL_TOL * G[j][j]) continue;
    kept[j] = true;
    L[j][j] = std::sqrt(dsum);
    for (int i = j + 1; i < P; ++i) {
      double sacc = G[i][j];
      for (int k = 0; k < j; ++k) sacc -= L[i][k] * L[j][k];
      L[i][j] = sacc / L[j][j];
    }
  }
  int idx[P], nk = 0;
  for (int j = 0; j < P; ++j) if (kept[j]) idx[nk++] = j;
  double M[P][P] = {};
  for (int c = 0; c < nk; ++c) {
    for (int r = 0; r < nk; ++r) {
      double sacc = (r == c) ? 1.0 : 0.0;
      for (int k = 0; k < r; ++k) sacc -= L[idx[r]][idx[k]] * M[k][c];
      M[r][c] = sacc / L[idx[r]][idx[r]];
    }
  }
  for (int i = 0; i < P * P; ++i) W[i] = 0.0;
  for (int a = 0; a < nk; ++a)
    for (int b = 0; b < nk; ++b) W[idx[a] * P + idx[b]] = M[b][a];
  *kept_mask = 0;
  for (int j = 0; j < P; ++j) if (kept[j]) *kept_mask |= 1u << j;
  A.assign((size_t)n_rows * P, 0.f);
  for (int32_t t = 0; t < n_rows; ++t) {
    const double* x = X + (int64_t)t * p;
    for (int q = 0; q < P; ++q) {
      double sacc = 0.0;
      for (int i = 0; i < p; ++i) sacc += x[i] * W[i * P + q];
      A[(size_t)t * P + q] = (float)sacc;
    }
  }
}

inline void split_tf32(float v, float* hi, float* lo) {
  uint32_t hb; memcpy(&hb, &v, 4); hb &= 0xFFFFE000u;
  memcpy(hi, &hb, 4);
  float l = v - *hi;
  uint32_t lb; memcpy(&lb, &l, 4); lb &= 0xFFFFE000u; memcpy(lo, &lb, 4);
}

// Enqueue the fit of ONE slab of device-resident rows on `s`.  status must be non-null.
int run_device_slab(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t pred_start, int32_t n_pred,
                    float* out, int64_t ld_out, float* beta, int32_t* status, cudaStream_t s, int* launches,
                    int* kernel_used, float* const* out_more, int n_out, int multimem, const SelectArgs* sel) {
  const DesignView d = view_of(ctx->plan);
  FitArgs a{};
  a.y = y; a.n = n; a.ld_y = ld_y; a.pred_start = pred_start; a.n_pred = n_pred;
  a.out = out; a.ld_out = ld_out; a.out_beta = beta; a.status = status;
  a.n_out = n_out; a.out_multimem = multimem;
  for (int i = 0; i + 1 < n_out && i < MAX_OUT - 1; ++i) a.out_more[i] = out_more[i];
  a.only_pending = 0; a.pending_count = nullptr;
  const char* why = nullptr;
  int kernel = ctx->cfg.kernel;
  // Many prediction rows (the reference's "Demand_Fitted for every date", 02:484-494): fit kernels hand
  // gamma/c to predict_tc_kernel, which writes the [n, n_pred] table with TMA stores.
  const bool predict_ok = n_out == 1 && !multimem && ld_out % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0 &&
                          n <= (int64_t)0x7fffffff - 128;
  if (sel != nullptr && !predict_ok)
    return fail(MMF_E_UNSUPPORTED, "model selection needs a 16-B aligned output with ld_out %% 4 == 0");
  const bool many_pred = sel != nullptr || (n_pred > 64 && kernel != MMF_KERNEL_WARP && predict_ok);
  if (many_pred) {
    int rc = grow((void**)&ctx->d_gamma, &ctx->gamma_cap_bytes, (size_t)n * P * sizeof(float));
    if (rc == MMF_OK) rc = grow((void**)&ctx->d_c, &ctx->c_cap_bytes, (size_t)n * sizeof(float));
    if (rc != MMF_OK) return rc;
    a.out_gamma = ctx->d_gamma;
    a.out_c = ctx->d_c;
    a.skip_pred = 1;
  }
  const bool tc_ok = fit_tc_supported(d, a, &why);
  if (kernel == MMF_KERNEL_TC && !tc_ok) return fail(MMF_E_UNSUPPORTED, "tensor-core kernel not applicable: %s", why);
  if (kernel == MMF_KERNEL_AUTO) kernel = tc_ok ? MMF_KERNEL_TC : MMF_KERNEL_WARP;
  const bool may_mask = !ctx->cfg.assume_finite;
  if (may_mask) {
    // scratch for the series with gaps: one 256-B record per row (filled only for rows that have gaps) and the
    // work list of rows whose record is ready for solve_rows_kernel
    const int64_t cap = n;
    int rc = grow((void**)&ctx->d_recs, &ctx->recs_cap_bytes, (size_t)cap * sizeof(SolveRec));
    const int64_t* rows_before = ctx->d_rec_rows;
    if (rc == MMF_OK) rc = grow((void**)&ctx->d_rec_rows, &ctx->rec_rows_cap_bytes, (size_t)cap * sizeof(int64_t));
    if (rc != MMF_OK) return rc;
    if (ctx->d_rec_rows != rows_before) ctx->rec_rows_clean = false;
    a.recs = ctx->d_recs;
    a.rec_rows = ctx->d_rec_rows;
    a.rec_cap = (uint32_t)cap;
  }
  // counters: an eager call uses ping-pong set `cs`; its tensor-core kernel zeroes the other set for the next eager
  // call, so the common path has no memset node.  A set that is not known to be zero (first use after a warp-only
  // call, after an error, ...) is cleared explicitly.  Under stream capture the launches become a graph that is
  // replayed any number of times, interleaved with eager calls: it gets set 2, zeroed by a memset node of its own,
  // and leaves the ping-pong state alone.
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  CU_TRY(cudaStreamIsCapturing(s, &cap));
  const bool capturing = cap != cudaStreamCaptureStatusNone;
  const int cs = capturing ? 2 : ctx->counter_set;
  uint32_t* counters = ctx->d_pending + CTR_WORDS * cs;
  if (may_mask) a.rec_count = counters + 1;
  if (capturing || !ctx->set_clean[cs]) CU_TRY(cudaMemsetAsync(counters, 0, CTR_WORDS * sizeof(uint32_t), s));
  if (!capturing) ctx->set_clean[cs] = false;             // dirty from here on, whatever happens below
  if (kernel == MMF_KERNEL_TC && !capturing) a.zero_next = ctx->d_pending + CTR_WORDS * (cs ^ 1);
  // Streaming solve (opt-in, mmf_config.stream_solve = 1): the series with gaps are solved WHILE the tensor-core kernel is
  // still streaming (solve_stream_kernel launched right behind it with programmatic stream serialisation) instead of in
  // a pass of their own afterwards.  The work list starts out as -1; the producer publishes row indices into it.  It
  // only overlaps when a consumer block fits beside the fit CTA on an SM, which the fit kernel's register and shared
  // memory use (one CTA per SM) does not leave room for, so it is off by default.
  const bool stream_solve = kernel == MMF_KERNEL_TC && may_mask && !capturing && n >= 32768 && ctx->cfg.stream_solve == 1;
  if (stream_solve) {
    if (!ctx->rec_rows_clean) CU_TRY(cudaMemsetAsync(ctx->d_rec_rows, 0xFF, ctx->rec_rows_cap_bytes, s));
    ctx->rec_rows_clean = true;                            // the call's closing solve_rows pass resets what it consumed
    a.stream_ctl = counters + 2;
  } else if (may_mask) {
    ctx->rec_rows_clean = false;
  }
  if (kernel == MMF_KERNEL_TC) {
    TcLaunch tl;
    int rc = encode_2d(tl.tmap_y, y, (uint64_t)d.t_fit, (uint64_t)n, (uint64_t)ld_y * 4, 32, 128);
    if (rc == MMF_OK && fit_tc_balanced_rows(n, ctx->sm_count, ctx->cfg.tc_variant) > 0)
      rc = encode_2d(tl.tmap_y8, y, (uint64_t)d.t_fit, (uint64_t)n, (uint64_t)ld_y * 4, 32, 8);
    if (rc != MMF_OK) return rc;
    memcpy(tl.tmap_at, ctx->plan.tmap_at, 128);
    CU_TRY(launch_fit_tc(d, a, tl, counters, ctx->sm_count, s, ctx->cfg.tc_variant));
    ++*launches;
    if (may_mask) {
      FitArgs m = a;
      m.only_pending = 1;
      m.pending_count = counters;
      if (stream_solve) {
        CU_TRY(launch_solve_stream(d, m, ctx->sm_count, s));
        ++*launches;
      }
      CU_TRY(launch_fit_warp(d, m, ctx->sm_count, s));
      CU_TRY(launch_solve_rows(d, m, ctx->sm_count, s));    // records the general pass queued (and, without the
      *launches += 2;                                        // streaming solve, all of them)
    }
  } else {
    CU_TRY(launch_fit_warp(d, a, ctx->sm_count, s));
    ++*launches;
    if (may_mask) {
      CU_TRY(launch_solve_rows(d, a, ctx->sm_count, s));
      ++*launches;
    }
  }
  if (sel != nullptr) {
    CU_TRY(launch_select(d, a, *sel, ctx->sm_count, s));
    ++*launches;
  }
  if (many_pred) {
    PredictLaunch pl;
    memcpy(pl.tmap_bhi, ctx->plan.tmap_bhi, 128);
    memcpy(pl.tmap_blo, ctx->plan.tmap_blo, 128);
    int rc = encode_2d(pl.tmap_out, out, (uint64_t)n_pred, (uint64_t)n, (uint64_t)ld_out * 4, 32, 64);   // one box per warpgroup half
    if (rc != MMF_OK) return rc;
    CU_TRY(launch_predict_tc(d, a, pl, ctx->sm_count, s));
    ++*launches;
  }
  *kernel_used = kernel;
  ctx->last_set = cs;
  if (!capturing) {                                       // toggle only once every launch of the call is enqueued
    ctx->set_clean[cs ^ 1] = (kernel == MMF_KERNEL_TC);   // zeroed by this call's tensor-core kernel
    ctx->counter_set = cs ^ 1;
  }
  return MMF_OK;
}

// Enqueue the fit for device-resident buffers on `s`: slab by slab, so that the per-row scratch (a 256-B record and a
// work-list entry per row for the series with gaps, gamma / c for the many-rows predict kernel) is proportional to a
// slab, not to the batch.  One slab for batches up to a million rows; beyond that the slab is sized so the scratch
// stays under ~5 % of the input (10 M x 365: 4 slabs, 0.7 GB instead of 2.6 GB).  Slabs run back to back on the
// stream; the scratch of slab i is free again when slab i+1 starts (stream order).
int run_device(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t pred_start, int32_t n_pred,
               float* out, int64_t ld_out, float* beta, int32_t* status, cudaStream_t s, int* launches,
               int* kernel_used, float* const* out_more = nullptr, int n_out = 1, int multimem = 0,
               const SelectArgs* sel = nullptr) {
  int64_t slab = n;
  if (n > (int64_t)1 << 20) {
    const double input_bytes = (double)n * (double)ctx->plan.t_fit * 4.0;
    slab = std::max<int64_t>((int64_t)1 << 20, (int64_t)(0.05 * input_bytes / (double)(sizeof(SolveRec) + sizeof(int64_t))));
    slab = std::min(n, (slab + 127) & ~(int64_t)127);                 // whole 128-row tiles
    const int64_t n_slabs = (n + slab - 1) / slab;
    slab = (((n + n_slabs - 1) / n_slabs) + 127) & ~(int64_t)127;     // equal slabs
  }
  for (int64_t off = 0; off < n; off += slab) {
    const int64_t m = std::min(slab, n - off);
    float* more[MAX_OUT - 1] = {};
    for (int i = 0; i + 1 < n_out && i < MAX_OUT - 1; ++i) more[i] = out_more[i] + off * ld_out;
    SelectArgs sel_slab;
    if (sel != nullptr) {
      sel_slab = *sel;
      if (sel_slab.out_choice) sel_slab.out_choice += off;
      if (sel_slab.out_mse) sel_slab.out_mse += off;
    }
    const int rc = run_device_slab(ctx, y + off * ld_y, m, ld_y, pred_start, n_pred, out + off * ld_out, ld_out,
                                   beta ? beta + off * P : nullptr, status + off, s, launches, kernel_used, more, n_out,
                                   multimem, sel != nullptr ? &sel_slab : nullptr);
    if (rc != MMF_OK) return rc;
  }
  return MMF_OK;
}

// The status scratch is only referenced by a graph whose capture passed out_status == NULL; otherwise it may move.
int grow_status_scratch(mmf_ctx* ctx, int64_t n, cudaStream_t s) {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &cap) == cudaSuccess && cap != cudaStreamCaptureStatusNone) ctx->status_scratch_captured = true;
  const mmf_ctx* saved = g_grow_ctx;
  if (!ctx->status_scratch_captured) g_grow_ctx = nullptr;
  const int rc = grow((void**)&ctx->d_status_scratch, &ctx->status_scratch_cap, (size_t)n * sizeof(int32_t));
  g_grow_ctx = saved;
  return rc;
}

struct GrowScope {                                        // entry points that may reallocate scratch name their ctx
  explicit GrowScope(const mmf_ctx* c) { g_grow_ctx = c; }
  ~GrowScope() { g_grow_ctx = nullptr; }
};

}  // namespace

// =============================================================================
extern "C" {

int mmf_version(void) { return MMF_VERSION; }

const char* mmf_last_error(void) { return g_err.c_str(); }

int mmf_device_count(int32_t* count) {
  if (!count) return fail(MMF_E_INVALID, "count is NULL");
  int c = 0;
  cudaError_t e = cudaGetDeviceCount(&c);
  if (e != cudaSuccess) { cudaGetLastError(); c = 0; }
  *count = c;
  return MMF_OK;
}

int mmf_create(const mmf_config* cfg, mmf_ctx** out) {
  if (!out) return fail(MMF_E_INVALID, "out is NULL");
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(MMF_E_CUDA, "no CUDA device available (%s); libmmf has no CPU path",
                e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
  }
  mmf_ctx* ctx = new mmf_ctx();
  if (cfg) ctx->cfg = *cfg;
  else { ctx->cfg.device = -1; ctx->cfg.kernel = MMF_KERNEL_AUTO; }
  int dev = ctx->cfg.device;
  if (dev < 0) { if (cudaGetDevice(&dev) != cudaSuccess) dev = 0; }
  if (dev >= ndev) { delete ctx; return fail(MMF_E_INVALID, "device %d out of range (%d devices)", dev, ndev); }
  ctx->device = dev;
  auto bail = [&](cudaError_t ee, const char* what) {
    int rc = fail(MMF_E_CUDA, "%s failed: %s", what, cudaGetErrorString(ee));
    delete ctx;
    return rc;
  };
  if ((e = cudaSetDevice(dev)) != cudaSuccess) return bail(e, "cudaSetDevice");
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, dev)) != cudaSuccess) return bail(e, "cudaGetDeviceProperties");
  ctx->sm_count = prop.multiProcessorCount;
  if (prop.major != 9 || prop.minor != 0) {
    int rc = fail(MMF_E_UNSUPPORTED, "device %d is sm_%d%d; libmmf is built for sm_90a (H100) only", dev, prop.major,
                  prop.minor);
    delete ctx;
    return rc;
  }
  if (ctx->cfg.stream) { ctx->stream = (cudaStream_t)ctx->cfg.stream; ctx->own_stream = false; }
  else {
    if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail(e, "cudaStreamCreate");
    ctx->own_stream = true;
  }
  if ((e = cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking)) != cudaSuccess) return bail(e, "cudaStreamCreate");
  if ((e = cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking)) != cudaSuccess) return bail(e, "cudaStreamCreate");
  cudaEventCreate(&ctx->ev_a); cudaEventCreate(&ctx->ev_b); cudaEventCreate(&ctx->ev_k0); cudaEventCreate(&ctx->ev_k1);
  for (int i = 0; i < NBUF; ++i) {
    cudaEventCreateWithFlags(&ctx->st[i].ev_h2d, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ctx->st[i].ev_comp, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ctx->st[i].ev_d2h, cudaEventDisableTiming);
  }
  if ((e = cudaMalloc(&ctx->d_pending, 3 * CTR_WORDS * sizeof(uint32_t))) != cudaSuccess) return bail(e, "cudaMalloc");
  cudaMemset(ctx->d_pending, 0, 3 * CTR_WORDS * sizeof(uint32_t));
  *out = ctx;
  return MMF_OK;
}

int mmf_destroy(mmf_ctx* ctx) {
  if (!ctx) return MMF_OK;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  free_plan(ctx->plan);
  free_multi(ctx->multi);
  for (int i = 0; i < NBUF; ++i) {
    Staging& s = ctx->st[i];
    cudaFree(s.d_y); cudaFree(s.d_yraw); cudaFree(s.d_out); cudaFree(s.d_beta); cudaFree(s.d_status);

    if (s.ev_h2d) cudaEventDestroy(s.ev_h2d);
    if (s.ev_comp) cudaEventDestroy(s.ev_comp);
    if (s.ev_d2h) cudaEventDestroy(s.ev_d2h);
  }
  if (ctx->narrow_pool) narrow_pool_destroy(ctx->narrow_pool);
  for (int i = 0; i < NHOST; ++i) {
    if (ctx->hslot[i].p) cudaFreeHost(ctx->hslot[i].p);
    if (ctx->hslot[i].ev) cudaEventDestroy(ctx->hslot[i].ev);
  }
  cudaFree(ctx->d_pending);
  cudaFree(ctx->d_recs);
  cudaFree(ctx->d_rec_rows);
  cudaFree(ctx->d_gamma);
  cudaFree(ctx->d_c);
  cudaFree(ctx->d_status_scratch);
  cudaFree(ctx->d_pack_scratch);
  if (ctx->ev_a) cudaEventDestroy(ctx->ev_a);
  if (ctx->ev_b) cudaEventDestroy(ctx->ev_b);
  if (ctx->ev_k0) cudaEventDestroy(ctx->ev_k0);
  if (ctx->ev_k1) cudaEventDestroy(ctx->ev_k1);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->s_h2d) cudaStreamDestroy(ctx->s_h2d);
  if (ctx->s_d2h) cudaStreamDestroy(ctx->s_d2h);
  delete ctx;
  return MMF_OK;
}

int mmf_set_stream(mmf_ctx* ctx, void* cuda_stream) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (ctx->own_stream && ctx->stream) { cudaStreamSynchronize(ctx->stream); cudaStreamDestroy(ctx->stream); }
  ctx->stream = (cudaStream_t)cuda_stream;      // NULL = legacy default stream
  ctx->own_stream = false;
  return MMF_OK;
}

int mmf_synchronize(mmf_ctx* ctx) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  CU_TRY(cudaSetDevice(ctx->device));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  CU_TRY(cudaStreamSynchronize(ctx->s_h2d));
  CU_TRY(cudaStreamSynchronize(ctx->s_d2h));
  return MMF_OK;
}

int mmf_plan_design(mmf_ctx* ctx, const double* X, int32_t n_rows, int32_t p, int32_t t_fit, int32_t has_constant) {
  if (!ctx || !X) return fail(MMF_E_INVALID, "ctx or X is NULL");
  if (p < 1 || p > P) return fail(MMF_E_INVALID, "p=%d outside [1,%d]", p, P);
  if (t_fit < 1 || n_rows < t_fit) return fail(MMF_E_INVALID, "need 1 <= t_fit <= n_rows (t_fit=%d n_rows=%d)", t_fit, n_rows);
  for (int64_t i = 0; i < (int64_t)n_rows * p; ++i)
    if (!std::isfinite(X[i])) return fail(MMF_E_INVALID, "design matrix has a non-finite entry at %lld", (long long)i);
  if (has_constant)
    for (int32_t t = 0; t < n_rows; ++t)
      if (X[(int64_t)t * p] != 1.0) return fail(MMF_E_INVALID, "has_constant=1 but X[%d,0] != 1", t);
  if (ctx->pinned > 0)
    return fail(MMF_E_UNSUPPORTED, "a captured CUDA graph references the current plan: release it (mmf_pin_scratch(ctx, -1)) "
                "before planning another design, or plan it on another context");
  CU_TRY(cudaSetDevice(ctx->device));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  free_plan(ctx->plan);
  Plan& pl = ctx->plan;

  // ---- float64 calendar Gram, in-order Cholesky with aliasing, A = X W (whiten_calendar above)
  pl.n_rows = n_rows;
  pl.n_rows_pad = (n_rows + 31) & ~31;
  pl.t_fit = t_fit;
  pl.t_pad = (t_fit + 31) & ~31;
  pl.has_constant = has_constant ? 1 : 0;
  std::vector<float> A;
  whiten_calendar(X, n_rows, p, t_fit, pl.W, &pl.kept_mask, A);
  std::vector<float> a4((size_t)4 * pl.n_rows_pad * 4, 0.f);
  for (int32_t t = 0; t < n_rows; ++t)
    for (int q = 0; q < P; ++q) a4[(((size_t)(q >> 2) * pl.n_rows_pad) + t) * 4 + (q & 3)] = A[(size_t)t * P + q];
  std::vector<float> at((size_t)2 * P * pl.t_pad, 0.f);
  for (int32_t t = 0; t < t_fit; ++t)
    for (int q = 0; q < P; ++q) {
      const float v = A[(size_t)t * P + q];
      uint32_t hb; memcpy(&hb, &v, 4); hb &= 0xFFFFE000u;
      float hi; memcpy(&hi, &hb, 4);
      float lo = v - hi;
      uint32_t lb; memcpy(&lb, &lo, 4); lb &= 0xFFFFE000u; memcpy(&lo, &lb, 4);
      at[(size_t)q * pl.t_pad + t] = hi;
      at[(size_t)(P + q) * pl.t_pad + t] = lo;
    }
  float w32[P * P];
  for (int i = 0; i < P * P; ++i) w32[i] = (float)pl.W[i];
  std::vector<float> ap_hi(A.size()), ap_lo(A.size());
  for (size_t i = 0; i < A.size(); ++i) {
    const float v = A[i];
    uint32_t hb; memcpy(&hb, &v, 4); hb &= 0xFFFFE000u;
    float hi; memcpy(&hi, &hb, 4);
    float lo = v - hi;
    uint32_t lb; memcpy(&lb, &lo, 4); lb &= 0xFFFFE000u; memcpy(&lo, &lb, 4);
    ap_hi[i] = hi; ap_lo[i] = lo;
  }

  CU_TRY(cudaMalloc(&pl.d_a4, a4.size() * sizeof(float)));
  CU_TRY(cudaMalloc(&pl.d_at, at.size() * sizeof(float)));
  CU_TRY(cudaMalloc(&pl.d_apred, A.size() * sizeof(float)));
  CU_TRY(cudaMalloc(&pl.d_w, sizeof(w32)));
  CU_TRY(cudaMemcpy(pl.d_a4, a4.data(), a4.size() * sizeof(float), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(pl.d_at, at.data(), at.size() * sizeof(float), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(pl.d_apred, A.data(), A.size() * sizeof(float), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(pl.d_w, w32, sizeof(w32), cudaMemcpyHostToDevice));
  CU_TRY(cudaMalloc(&pl.d_ap_hi, A.size() * sizeof(float)));
  CU_TRY(cudaMalloc(&pl.d_ap_lo, A.size() * sizeof(float)));
  CU_TRY(cudaMemcpy(pl.d_ap_hi, ap_hi.data(), A.size() * sizeof(float), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(pl.d_ap_lo, ap_lo.data(), A.size() * sizeof(float), cudaMemcpyHostToDevice));
  int rc = encode_2d(pl.tmap_at, pl.d_at, (uint64_t)pl.t_pad, (uint64_t)(2 * P), (uint64_t)pl.t_pad * 4, 32, 2 * P);
  if (rc != MMF_OK) return rc;
  rc = encode_2d(pl.tmap_bhi, pl.d_ap_hi, (uint64_t)P, (uint64_t)n_rows, (uint64_t)P * 4, P, 128, CU_TENSOR_MAP_SWIZZLE_64B);
  if (rc != MMF_OK) return rc;
  rc = encode_2d(pl.tmap_blo, pl.d_ap_lo, (uint64_t)P, (uint64_t)n_rows, (uint64_t)P * 4, P, 128, CU_TENSOR_MAP_SWIZZLE_64B);
  if (rc != MMF_OK) return rc;
  pl.valid = true;
  return MMF_OK;
}

int mmf_pin_scratch(mmf_ctx* ctx, int32_t delta) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (ctx->pinned + delta < 0) return fail(MMF_E_INVALID, "unbalanced mmf_pin_scratch");
  ctx->pinned += delta;
  return MMF_OK;
}

int mmf_get_whitening(mmf_ctx* ctx, double* W, int32_t* kept) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (!ctx->plan.valid) return fail(MMF_E_NOPLAN, "no design planned");
  if (W) memcpy(W, ctx->plan.W, sizeof(double) * P * P);
  if (kept) for (int j = 0; j < P; ++j) kept[j] = (ctx->plan.kept_mask >> j) & 1u;
  return MMF_OK;
}

static int fit_forecast_impl(mmf_ctx* ctx, const void* y_any, int32_t dtype, int64_t n, int64_t ld_y, int32_t pred_start,
                             int32_t n_pred, float* out_pred, int64_t ld_out, float* out_beta, int32_t* out_status,
                             mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (dtype != MMF_DT_F32 && dtype != MMF_DT_I16 && dtype != MMF_DT_U16 && dtype != MMF_DT_I32)
    return fail(MMF_E_INVALID, "dtype %d is not one of MMF_DT_F32 / I16 / U16 / I32", dtype);
  const float* y = static_cast<const float*>(y_any);           // only dereferenced as float when dtype == MMF_DT_F32
  const size_t esize = (dtype == MMF_DT_I16 || dtype == MMF_DT_U16) ? 2 : 4;
  const bool is_int = dtype != MMF_DT_F32;
  GrowScope grow_scope(ctx);
  if (!ctx->plan.valid) return fail(MMF_E_NOPLAN, "mmf_plan_design has not been called");
  const Plan& pl = ctx->plan;
  if (n < 0) return fail(MMF_E_INVALID, "n < 0");
  if (n > 0 && (!y || !out_pred)) return fail(MMF_E_INVALID, "y or out_pred is NULL");
  if (ld_y < pl.t_fit) return fail(MMF_E_INVALID, "ld_y=%lld < t_fit=%d", (long long)ld_y, pl.t_fit);
  if (n_pred < 1 || pred_start < 0 || (int64_t)pred_start + n_pred > pl.n_rows)
    return fail(MMF_E_INVALID, "prediction rows [%d,%d) outside the planned design (%d rows)", pred_start,
                pred_start + n_pred, pl.n_rows);
  if (ld_out < n_pred) return fail(MMF_E_INVALID, "ld_out=%lld < n_pred=%d", (long long)ld_out, n_pred);
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));

  const bool y_dev = is_device_ptr(y), o_dev = is_device_ptr(out_pred);
  const bool b_dev = out_beta ? is_device_ptr(out_beta) : true;
  const bool s_dev = out_status ? is_device_ptr(out_status) : true;
  int launches = 0, kernel_used = 0;
  int64_t h2d = 0, d2h = 0;

  if (!is_int && y_dev && o_dev && b_dev && s_dev) {
    // ------------------------------------------------ all device: just enqueue
    int32_t* status = out_status;
    if (!status) {
      int rc = grow_status_scratch(ctx, n, ctx->stream);
      if (rc != MMF_OK) return rc;
      status = ctx->d_status_scratch;
    }
    if (stats) CU_TRY(cudaEventRecord(ctx->ev_k0, ctx->stream));
    int rc = run_device(ctx, y, n, ld_y, pred_start, n_pred, out_pred, ld_out, out_beta, status, ctx->stream,
                        &launches, &kernel_used);
    if (rc != MMF_OK) return rc;
    if (stats) {
      CU_TRY(cudaEventRecord(ctx->ev_k1, ctx->stream));
      CU_TRY(cudaEventSynchronize(ctx->ev_k1));
      CU_TRY(cudaEventElapsedTime(&stats->kernel_ms, ctx->ev_k0, ctx->ev_k1));
      stats->total_ms = stats->kernel_ms;
      uint32_t pend = 0;
      CU_TRY(cudaMemcpy(&pend, ctx->d_pending + CTR_WORDS * ctx->last_set, sizeof(pend), cudaMemcpyDeviceToHost));
      stats->n_pending = (kernel_used == MMF_KERNEL_TC) ? pend : 0;
    }
  } else {
    // ------------------------------------------------ host buffers (or an integer series buffer): pipelined chunks
    int64_t chunk = ctx->cfg.chunk_series > 0 ? ctx->cfg.chunk_series : 32768;
    if (chunk > n) chunk = n;
    const int64_t pitch = (pl.t_fit + 3) & ~3;                 // staged row pitch (floats), TMA-friendly
    const int64_t rpitch = (pl.t_fit + 7) & ~7;                // staged row pitch of an integer chunk (16-B rows)
    const int64_t opitch = (n_pred + 3) & ~3;
    const int64_t npitch = (pl.t_fit + 15) & ~15;              // ... of a narrowed uint16 chunk (32-B rows: streaming stores)
    // float32 host input is narrowed to uint16 chunk by chunk on host threads while the previous chunk's copy is in
    // flight (exact or not used: host_narrow.cpp), so half the bytes cross PCIe -- the link is what bounds this path
    // Automatic mode narrows only where it was measured to pay: batches of at least 4 M values on a host where this
    // process sees ONE GPU and at least 32 CPUs.  The narrowing pool and the copy engine share the host's memory
    // controllers; with one process per GPU on a multi-GPU host the plain float32 copies are already bound by host
    // memory rather than by PCIe, and several pools would fight over the same cores (host_narrow = 1 opts in anyway).
    bool narrow = !is_int && !y_dev && ctx->cfg.host_narrow != 2;
    if (narrow && ctx->cfg.host_narrow != 1) {
      int ndev = 1;
      if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) { cudaGetLastError(); ndev = 1; }
      narrow = n * (int64_t)pl.t_fit >= ((int64_t)4 << 20) && ndev == 1 && std::thread::hardware_concurrency() >= 32;
    }
    if (narrow && ctx->narrow_pool == nullptr) {
      int want = ctx->cfg.host_threads;
      if (want <= 0) {
        cpu_set_t set;
        const int have = (sched_getaffinity(0, sizeof(set), &set) == 0) ? CPU_COUNT(&set) : (int)std::thread::hardware_concurrency();
        // past ~16 streaming threads the copy engine's reads of the same memory controllers slow down more than the
        // conversion speeds up
        want = std::max(1, std::min(16, have / 2));
      }
      int ndev_vis = 0;
      if (cudaGetDeviceCount(&ndev_vis) != cudaSuccess) { cudaGetLastError(); ndev_vis = 0; }
      bool pin = ndev_vis == 1;                                // this process has the host's cores to itself
      if (const char* e = getenv("MMF_HOST_PIN")) pin = atoi(e) != 0;
      ctx->narrow_pool = narrow_pool_create(want - 1, pin);    // the calling thread is the last worker
    }
    // rows per narrowed sub-chunk and store flavour: keeping the slots cache resident (small sub-chunks, ordinary stores)
    // does not pay for the extra copies and synchronisations
    int64_t sub_rows = 8192;
    bool stream_stores = true;
    if (const char* e = getenv("MMF_HOST_SUB_ROWS")) sub_rows = std::max<int64_t>(64, atoll(e));   // tuning / experiments
    if (const char* e = getenv("MMF_HOST_STREAM_STORES")) stream_stores = atoi(e) != 0;
    sub_rows = std::min(sub_rows, chunk);
    // every third chunk goes over PCIe as float32 without narrowing: the copy engine and the narrowing threads share the load
    int direct_every = 3;
    if (const char* e = getenv("MMF_HOST_DIRECT_EVERY")) direct_every = atoi(e);
    if (narrow) {
      for (int i = 0; i < NHOST && narrow; ++i) {
        HostSlot& hs = ctx->hslot[i];
        if (!hs.ev && cudaEventCreateWithFlags(&hs.ev, cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); narrow = false; break; }
        const size_t need = (size_t)sub_rows * npitch * 2;
        if (hs.cap >= need) continue;
        if (hs.p) { cudaEventSynchronize(hs.ev); cudaFreeHost(hs.p); }
        hs.p = nullptr; hs.cap = 0;
        if (cudaHostAlloc((void**)&hs.p, need, cudaHostAllocDefault) == cudaSuccess) hs.cap = need;
        else { cudaGetLastError(); narrow = false; }           // cannot pin the slots: plain float32 copies
      }
    }
    struct HotScope {                                           // workers spin between sub-chunks only during this call
      NarrowPool* p;
      explicit HotScope(NarrowPool* q) : p(q) { if (p) narrow_pool_begin_call(p); }
      ~HotScope() { if (p) narrow_pool_end_call(p); }
    } hot_scope(narrow ? ctx->narrow_pool : nullptr);
    const mmf_ctx* pinned_scope = g_grow_ctx;
    g_grow_ctx = nullptr;                                       // staging slots are never part of a captured graph
    for (int i = 0; i < NBUF; ++i) {
      Staging& s = ctx->st[i];
      int rc = MMF_OK;
      if (!y_dev || is_int) rc = grow((void**)&s.d_y, &s.y_cap, (size_t)chunk * pitch * sizeof(float));
      if (rc == MMF_OK && (is_int || narrow) && !y_dev)
        rc = grow(&s.d_yraw, &s.yraw_cap, narrow ? (size_t)chunk * npitch * 2 : (size_t)chunk * rpitch * esize);
      if (rc == MMF_OK && !o_dev) rc = grow((void**)&s.d_out, &s.out_cap, (size_t)chunk * opitch * sizeof(float));
      if (rc == MMF_OK && out_beta && !b_dev) rc = grow((void**)&s.d_beta, &s.beta_cap, (size_t)chunk * P * sizeof(float));
      if (rc == MMF_OK && (!out_status || !s_dev)) rc = grow((void**)&s.d_status, &s.status_cap, (size_t)chunk * sizeof(int32_t));
      if (rc != MMF_OK) { g_grow_ctx = pinned_scope; return rc; }
    }
    g_grow_ctx = pinned_scope;
    CU_TRY(cudaEventRecord(ctx->ev_a, ctx->stream));
    CU_TRY(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_a, 0));
    CU_TRY(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_a, 0));
    int it = 0;
    for (int64_t off = 0; off < n; off += chunk, ++it) {
      const int64_t m = std::min(chunk, n - off);
      Staging& s = ctx->st[it % NBUF];
      const float* yk; int64_t ldk;
      if (is_int) {
        // integer series: stage the chunk as it is (half / all of the float32 bytes), widen it on the device
        const char* src = static_cast<const char*>(y_any) + (size_t)off * ld_y * esize;
        if (it >= NBUF) CU_TRY(cudaStreamWaitEvent(y_dev ? ctx->stream : ctx->s_h2d, s.ev_comp, 0));   // d_y / d_yraw free again
        const void* raw = src;
        int64_t raw_ld = ld_y;
        if (!y_dev) {
          if (ld_y == rpitch)
            CU_TRY(cudaMemcpyAsync(s.d_yraw, src, ((size_t)(m - 1) * rpitch + (size_t)pl.t_fit) * esize,
                                   cudaMemcpyHostToDevice, ctx->s_h2d));
          else
            CU_TRY(cudaMemcpy2DAsync(s.d_yraw, (size_t)rpitch * esize, src, (size_t)ld_y * esize, (size_t)pl.t_fit * esize,
                                     (size_t)m, cudaMemcpyHostToDevice, ctx->s_h2d));
          CU_TRY(cudaEventRecord(s.ev_h2d, ctx->s_h2d));
          CU_TRY(cudaStreamWaitEvent(ctx->stream, s.ev_h2d, 0));
          raw = s.d_yraw; raw_ld = rpitch;
          h2d += m * (int64_t)pl.t_fit * (int64_t)esize;
        }
        CU_TRY(launch_widen(dtype, raw, raw_ld, s.d_y, pitch, m, pl.t_fit, ctx->sm_count, ctx->stream));
        ++launches;
        yk = s.d_y; ldk = pitch;
      } else if (y_dev) { yk = y + off * ld_y; ldk = ld_y; }
      else if ([&]() -> bool {
                 // Every `direct_every`-th chunk crosses as float32 straight from the caller's buffer: the narrowing
                 // threads are the slower of the two resources (they and the copy engine share the memory controllers),
                 // so the link would otherwise idle a third of the time; a float32 chunk costs the link twice the bytes
                 // but the host threads nothing.
                 if (!narrow || (direct_every > 0 && (it % direct_every) == direct_every - 1)) return false;
                 const bool ok = [&]() -> bool {
                 // sub-chunk by sub-chunk: narrow into a page-locked host slot, copy it into the chunk's device staging;
                 // the narrowing of sub-chunk k+1 runs while the copy of sub-chunk k is in flight
                 if (it >= NBUF && cudaStreamWaitEvent(ctx->s_h2d, s.ev_comp, 0) != cudaSuccess) return false;   // device staging free
                 for (int64_t so = 0; so < m; so += sub_rows) {
                   const int64_t ms = std::min(sub_rows, m - so);
                   HostSlot& hs = ctx->hslot[ctx->hslot_uses % NHOST];
                   if (ctx->hslot_uses >= (uint64_t)NHOST && cudaEventSynchronize(hs.ev) != cudaSuccess) return false;
                   if (!narrow_f32_to_u16(ctx->narrow_pool, y + (off + so) * ld_y, ld_y, hs.p, npitch, ms, pl.t_fit, stream_stores))
                     return false;                           // not representable: the whole chunk goes as float32
                   if (cudaMemcpyAsync(static_cast<uint16_t*>(s.d_yraw) + so * npitch, hs.p, (size_t)ms * npitch * 2,
                                       cudaMemcpyHostToDevice, ctx->s_h2d) != cudaSuccess) return false;
                   if (cudaEventRecord(hs.ev, ctx->s_h2d) != cudaSuccess) return false;
                   ++ctx->hslot_uses;
                 }
                 return true;
               }();
                 if (!ok) narrow = false;                   // a value uint16 cannot carry: float32 from here on
                 return ok;
               }()) {
        CU_TRY(cudaEventRecord(s.ev_h2d, ctx->s_h2d));
        CU_TRY(cudaStreamWaitEvent(ctx->stream, s.ev_h2d, 0));
        CU_TRY(launch_widen(MMF_DT_U16, s.d_yraw, npitch, s.d_y, pitch, m, pl.t_fit, ctx->sm_count, ctx->stream));
        ++launches;
        yk = s.d_y; ldk = pitch;
        h2d += m * (int64_t)pl.t_fit * 2;
      } else {
        if (it >= NBUF) CU_TRY(cudaStreamWaitEvent(ctx->s_h2d, s.ev_comp, 0));     // staging buffer free again
        if (ld_y == pitch)        // already pitched on the host: one contiguous copy (pad columns ride along, except
                                  // behind the caller's very last row, which may be the end of its buffer)
          CU_TRY(cudaMemcpyAsync(s.d_y, y + off * ld_y, ((size_t)(m - 1) * pitch + (size_t)pl.t_fit) * 4,
                                 cudaMemcpyHostToDevice, ctx->s_h2d));
        else
          CU_TRY(cudaMemcpy2DAsync(s.d_y, (size_t)pitch * 4, y + off * ld_y, (size_t)ld_y * 4, (size_t)pl.t_fit * 4,
                                   (size_t)m, cudaMemcpyHostToDevice, ctx->s_h2d));
        CU_TRY(cudaEventRecord(s.ev_h2d, ctx->s_h2d));
        CU_TRY(cudaStreamWaitEvent(ctx->stream, s.ev_h2d, 0));
        yk = s.d_y; ldk = pitch;
        h2d += m * (int64_t)pl.t_fit * 4;
      }
      float* ok = o_dev ? out_pred + off * ld_out : s.d_out;
      const int64_t ldo = o_dev ? ld_out : opitch;
      float* bk = out_beta ? (b_dev ? out_beta + off * P : s.d_beta) : nullptr;
      int32_t* sk = (out_status && s_dev) ? out_status + off : s.d_status;
      if (it >= NBUF) CU_TRY(cudaStreamWaitEvent(ctx->stream, s.ev_d2h, 0));        // output staging drained
      int rc = run_device(ctx, yk, m, ldk, pred_start, n_pred, ok, ldo, bk, sk, ctx->stream, &launches, &kernel_used);
      if (rc != MMF_OK) return rc;
      CU_TRY(cudaEventRecord(s.ev_comp, ctx->stream));
      bool any_d2h = false;
      if (!o_dev) {
        CU_TRY(cudaStreamWaitEvent(ctx->s_d2h, s.ev_comp, 0));
        if (ld_out == opitch && n_pred == opitch)
          CU_TRY(cudaMemcpyAsync(out_pred + off * ld_out, s.d_out, (size_t)m * opitch * 4, cudaMemcpyDeviceToHost, ctx->s_d2h));
        else
          CU_TRY(cudaMemcpy2DAsync(out_pred + off * ld_out, (size_t)ld_out * 4, s.d_out, (size_t)opitch * 4,
                                   (size_t)n_pred * 4, (size_t)m, cudaMemcpyDeviceToHost, ctx->s_d2h));
        d2h += m * (int64_t)n_pred * 4; any_d2h = true;
      }
      if (out_beta && !b_dev) {
        if (!any_d2h) CU_TRY(cudaStreamWaitEvent(ctx->s_d2h, s.ev_comp, 0));
        CU_TRY(cudaMemcpyAsync(out_beta + off * P, s.d_beta, (size_t)m * P * 4, cudaMemcpyDeviceToHost, ctx->s_d2h));
        d2h += m * (int64_t)P * 4; any_d2h = true;
      }
      if (out_status && !s_dev) {
        if (!any_d2h) CU_TRY(cudaStreamWaitEvent(ctx->s_d2h, s.ev_comp, 0));
        CU_TRY(cudaMemcpyAsync(out_status + off, s.d_status, (size_t)m * 4, cudaMemcpyDeviceToHost, ctx->s_d2h));
        d2h += m * 4; any_d2h = true;
      }
      CU_TRY(cudaEventRecord(s.ev_d2h, ctx->s_d2h));
    }
    // join: compute stream waits for the copies, then the host waits for everything
    CU_TRY(cudaEventRecord(ctx->ev_b, ctx->s_d2h));
    CU_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ev_b, 0));
    CU_TRY(cudaEventRecord(ctx->ev_b, ctx->stream));
    CU_TRY(cudaEventSynchronize(ctx->ev_b));
    if (stats) {
      CU_TRY(cudaEventElapsedTime(&stats->total_ms, ctx->ev_a, ctx->ev_b));
      stats->kernel_ms = 0.f;   // kernels overlap the copies here; use a device-pointer call to time them
    }
  }
  if (stats) {
    stats->n_series = n;
    stats->h2d_bytes = h2d;
    stats->d2h_bytes = d2h;
    stats->kernel_launches = launches;
    stats->kernel_used = kernel_used;
  }
  return MMF_OK;
}

int mmf_fit_forecast_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t pred_start, int32_t n_pred,
                         float* out_pred, int64_t ld_out, float* out_beta, int32_t* out_status, mmf_stats* stats) {
  return fit_forecast_impl(ctx, y, MMF_DT_F32, n, ld_y, pred_start, n_pred, out_pred, ld_out, out_beta, out_status, stats);
}

int mmf_fit_forecast_int(mmf_ctx* ctx, const void* y, int32_t dtype, int64_t n, int64_t ld_y, int32_t pred_start,
                         int32_t n_pred, float* out_pred, int64_t ld_out, float* out_beta, int32_t* out_status,
                         mmf_stats* stats) {
  if (dtype == MMF_DT_F32) return fail(MMF_E_INVALID, "mmf_fit_forecast_int takes MMF_DT_I16 / U16 / I32; use mmf_fit_forecast_f32");
  return fit_forecast_impl(ctx, y, dtype, n, ld_y, pred_start, n_pred, out_pred, ld_out, out_beta, out_status, stats);
}


// ---- ragged batches: many calendars, one launch ------------------------------------------------------------------
int mmf_plan_calendars(mmf_ctx* ctx, const double* X_all, int32_t n_cal, const int32_t* n_rows, const int32_t* t_fit,
                       const int32_t* pred_start, const int32_t* n_pred_cal, int32_t p, int32_t has_constant) {
  if (!ctx || !X_all || !n_rows || !t_fit || !pred_start || !n_pred_cal) return fail(MMF_E_INVALID, "NULL argument");
  if (n_cal < 1 || n_cal > 65535) return fail(MMF_E_INVALID, "n_cal=%d outside [1,65535]", n_cal);
  if (p < 1 || p > P) return fail(MMF_E_INVALID, "p=%d outside [1,%d]", p, P);
  // one common number of prediction rows <= 64: the forecasts are written by the fit kernel's own epilogue; anything
  // else (holdout: every date of every calendar) goes through the tensor-core predict kernel
  bool many = false;
  int32_t n_pred = n_pred_cal[0], n_pred_max = 0;
  for (int c = 0; c < n_cal; ++c) {
    if (n_pred_cal[c] < 1) return fail(MMF_E_INVALID, "calendar %d: n_pred=%d < 1", c, n_pred_cal[c]);
    many = many || n_pred_cal[c] != n_pred || n_pred_cal[c] > 64;
    n_pred_max = std::max(n_pred_max, n_pred_cal[c]);
  }
  if (ctx->pinned > 0) return fail(MMF_E_UNSUPPORTED, "a captured CUDA graph pins this context");
  size_t total_rows = 0;
  int32_t tmax = 0, tmin = INT32_MAX;
  for (int c = 0; c < n_cal; ++c) {
    if (t_fit[c] < 33 || t_fit[c] > 65535 || n_rows[c] < t_fit[c])
      return fail(MMF_E_UNSUPPORTED, "calendar %d: need 33 <= t_fit <= 65535 and n_rows >= t_fit (t_fit=%d n_rows=%d)", c, t_fit[c], n_rows[c]);
    if (pred_start[c] < 0 || pred_start[c] + n_pred_cal[c] > n_rows[c])
      return fail(MMF_E_INVALID, "calendar %d: prediction rows [%d,%d) outside its %d design rows", c, pred_start[c],
                  pred_start[c] + n_pred_cal[c], n_rows[c]);
    total_rows += (size_t)n_rows[c];
    tmax = std::max(tmax, t_fit[c]);
    tmin = std::min(tmin, t_fit[c]);
  }
  for (size_t i = 0; i < total_rows * (size_t)p; ++i)
    if (!std::isfinite(X_all[i])) return fail(MMF_E_INVALID, "design matrix has a non-finite entry at %zu", i);
  CU_TRY(cudaSetDevice(ctx->device));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  free_multi(ctx->multi);
  MultiPlan& m = ctx->multi;
  m.n_cal = n_cal; m.n_pred = many ? 1 : n_pred; m.has_constant = has_constant ? 1 : 0;
  m.many_pred = many; m.n_pred_max = n_pred_max;
  m.t_fit_max = tmax; m.t_pad_max = (tmax + 31) & ~31; m.min_chunks = (tmin + 31) / 32;
  m.cals.resize(n_cal);
  m.a4_off.resize(n_cal);
  std::vector<float> at((size_t)n_cal * 2 * P * m.t_pad_max, 0.f), apred(total_rows * P);
  size_t a4_total = 0;
  for (int c = 0; c < n_cal; ++c) { m.a4_off[c] = a4_total; a4_total += (size_t)4 * ((n_rows[c] + 31) & ~31); }
  std::vector<float> a4(a4_total * 4, 0.f);
  size_t row_off = 0;
  std::vector<float> A;
  double W[P * P];
  for (int c = 0; c < n_cal; ++c) {
    const double* X = X_all + row_off * (size_t)p;
    if (has_constant)
      for (int32_t t = 0; t < n_rows[c]; ++t)
        if (X[(size_t)t * p] != 1.0) return fail(MMF_E_INVALID, "has_constant=1 but calendar %d has X[%d,0] != 1", c, t);
    CalMeta& cm = m.cals[c];
    whiten_calendar(X, n_rows[c], p, t_fit[c], W, &cm.kept_mask, A);
    cm.t_fit = t_fit[c]; cm.n_chunks = (t_fit[c] + 31) / 32; cm.n_rows = n_rows[c];
    cm.row_off = (int32_t)row_off; cm.pred_start = pred_start[c]; cm.n_pred = n_pred_cal[c]; cm.n_rows_pad = (n_rows[c] + 31) & ~31;
    memcpy(apred.data() + row_off * P, A.data(), A.size() * sizeof(float));
    float* atc = at.data() + (size_t)c * 2 * P * m.t_pad_max;
    for (int32_t t = 0; t < t_fit[c]; ++t)
      for (int q = 0; q < P; ++q) split_tf32(A[(size_t)t * P + q], atc + (size_t)q * m.t_pad_max + t, atc + (size_t)(P + q) * m.t_pad_max + t);
    float* a4c = a4.data() + m.a4_off[c] * 4;
    for (int32_t t = 0; t < n_rows[c]; ++t)
      for (int q = 0; q < P; ++q) a4c[(((size_t)(q >> 2) * cm.n_rows_pad) + t) * 4 + (q & 3)] = A[(size_t)t * P + q];
    row_off += (size_t)n_rows[c];
  }
  if (row_off > (size_t)INT32_MAX) return fail(MMF_E_UNSUPPORTED, "too many design rows in one ragged plan");
  CU_TRY(cudaMalloc(&m.d_cals, (size_t)n_cal * sizeof(CalMeta)));
  CU_TRY(cudaMalloc(&m.d_at, at.size() * sizeof(float)));
  CU_TRY(cudaMalloc(&m.d_apred, apred.size() * sizeof(float)));
  CU_TRY(cudaMalloc(&m.d_a4, a4.size() * sizeof(float)));
  CU_TRY(cudaMalloc(&m.d_w, P * P * sizeof(float)));
  CU_TRY(cudaMalloc(&m.d_pending_by_cal, (size_t)n_cal * sizeof(uint32_t)));
  CU_TRY(cudaMalloc(&m.d_tmaps_y, (size_t)n_cal * 128));
  CU_TRY(cudaMemcpy(m.d_cals, m.cals.data(), (size_t)n_cal * sizeof(CalMeta), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(m.d_at, at.data(), at.size() * sizeof(float), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(m.d_apred, apred.data(), apred.size() * sizeof(float), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(m.d_a4, a4.data(), a4.size() * sizeof(float), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemset(m.d_w, 0, P * P * sizeof(float)));
  int rc = encode_2d(m.tmap_at, m.d_at, (uint64_t)m.t_pad_max, (uint64_t)n_cal * 2 * P, (uint64_t)m.t_pad_max * 4, 32, 2 * P);
  if (rc != MMF_OK) return rc;
  if (many) {
    // B operand of predict_tc_kernel: tf32-hi / lo of every calendar's whitened rows, stacked (+128 zero rows: the last
    // chunk of the last calendar reads a full box)
    std::vector<float> hi((total_rows + 128) * P, 0.f), lo((total_rows + 128) * P, 0.f);
    for (size_t i = 0; i < total_rows * P; ++i) split_tf32(apred[i], &hi[i], &lo[i]);
    CU_TRY(cudaMalloc(&m.d_ap_hi, hi.size() * sizeof(float)));
    CU_TRY(cudaMalloc(&m.d_ap_lo, lo.size() * sizeof(float)));
    CU_TRY(cudaMemcpy(m.d_ap_hi, hi.data(), hi.size() * sizeof(float), cudaMemcpyHostToDevice));
    CU_TRY(cudaMemcpy(m.d_ap_lo, lo.data(), lo.size() * sizeof(float), cudaMemcpyHostToDevice));
    rc = encode_2d(m.tmap_bhi, m.d_ap_hi, (uint64_t)P, (uint64_t)(total_rows + 128), (uint64_t)P * 4, P, 128, CU_TENSOR_MAP_SWIZZLE_64B);
    if (rc != MMF_OK) return rc;
    rc = encode_2d(m.tmap_blo, m.d_ap_lo, (uint64_t)P, (uint64_t)(total_rows + 128), (uint64_t)P * 4, P, 128, CU_TENSOR_MAP_SWIZZLE_64B);
    if (rc != MMF_OK) return rc;
    CU_TRY(cudaMalloc(&m.d_tmaps_out, (size_t)n_cal * 128));
  }
  m.valid = true;
  return MMF_OK;
}

int mmf_fit_forecast_ragged_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, const int64_t* cal_row_start,
                                float* out_pred, int64_t ld_out, int32_t* out_status, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  MultiPlan& m = ctx->multi;
  if (!m.valid) return fail(MMF_E_NOPLAN, "mmf_plan_calendars has not been called");
  if (n < 0 || !cal_row_start || (n > 0 && (!y || !out_pred))) return fail(MMF_E_INVALID, "bad y / out_pred / cal_row_start / n");
  if (cal_row_start[0] != 0 || cal_row_start[m.n_cal] != n) return fail(MMF_E_INVALID, "cal_row_start must run from 0 to n");
  for (int c = 0; c < m.n_cal; ++c)
    if (cal_row_start[c + 1] < cal_row_start[c]) return fail(MMF_E_INVALID, "cal_row_start must be non-decreasing");
  if (ld_y < m.t_fit_max) return fail(MMF_E_INVALID, "ld_y=%lld < the longest calendar's t_fit=%d", (long long)ld_y, m.t_fit_max);
  if (!m.many_pred && ld_out < m.n_pred) return fail(MMF_E_INVALID, "ld_out=%lld < n_pred=%d", (long long)ld_out, m.n_pred);
  if (m.many_pred && (ld_out < m.n_pred_max || ld_out % 4 != 0))
    return fail(MMF_E_INVALID, "this plan evaluates up to %d rows per series: ld_out must be >= that and a multiple of 4 (TMA stores)",
                m.n_pred_max);
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  if (n > (int64_t)0x7fffffff - 128) return fail(MMF_E_UNSUPPORTED, "n too large for 32-bit TMA coordinates");
  CU_TRY(cudaSetDevice(ctx->device));
  if (!is_device_ptr(y) || !is_device_ptr(out_pred) || (out_status && !is_device_ptr(out_status)))
    return fail(MMF_E_INVALID, "the ragged entry point takes device buffers only");
  if (ld_y % 4 != 0 || (reinterpret_cast<uintptr_t>(y) & 15u) != 0 || (reinterpret_cast<uintptr_t>(out_pred) & 15u) != 0)
    return fail(MMF_E_UNSUPPORTED, "ragged batches need 16-B aligned y / out_pred and ld_y %% 4 == 0 (TMA)");
  cudaStream_t s = ctx->stream;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  CU_TRY(cudaStreamIsCapturing(s, &cap));
  if (cap != cudaStreamCaptureStatusNone) return fail(MMF_E_UNSUPPORTED, "ragged batches cannot be captured into a CUDA graph");
  int32_t* status = out_status;
  if (!status) {
    int rc = grow_status_scratch(ctx, n, s);
    if (rc != MMF_OK) return rc;
    status = ctx->d_status_scratch;
  }
  // ---- per-call tables: tiles of 128 rows inside one calendar, the y buffer clipped at every calendar's t_fit
  const bool same = m.key_y == y && m.key_n == n && m.key_ld == ld_y && m.key_rows.size() == (size_t)m.n_cal + 1 &&
                    memcmp(m.key_rows.data(), cal_row_start, sizeof(int64_t) * ((size_t)m.n_cal + 1)) == 0;
  if (!same) {
    std::vector<TileRec> tiles;
    tiles.reserve((size_t)(n / 128 + m.n_cal + 1));
    for (int c = 0; c < m.n_cal; ++c)
      for (int64_t r = cal_row_start[c]; r < cal_row_start[c + 1]; r += 128)
        tiles.push_back(TileRec{(int32_t)r, (int32_t)std::min<int64_t>(128, cal_row_start[c + 1] - r), c, m.cals[c].n_chunks});
    int rc = grow((void**)&m.d_tiles, &m.tiles_cap, tiles.size() * sizeof(TileRec));
    if (rc != MMF_OK) return rc;
    std::vector<unsigned char> maps((size_t)m.n_cal * 128);
    for (int c = 0; c < m.n_cal; ++c) {
      rc = encode_2d(maps.data() + (size_t)c * 128, y, (uint64_t)m.cals[c].t_fit, (uint64_t)n, (uint64_t)ld_y * 4, 32, 128);
      if (rc != MMF_OK) return rc;
    }
    CU_TRY(cudaStreamSynchronize(s));                      // a previous call may still read the old tables
    CU_TRY(cudaMemcpy(m.d_tiles, tiles.data(), tiles.size() * sizeof(TileRec), cudaMemcpyHostToDevice));
    CU_TRY(cudaMemcpy(m.d_tmaps_y, maps.data(), maps.size(), cudaMemcpyHostToDevice));
    m.n_tiles = (int32_t)tiles.size();
    m.key_y = y; m.key_n = n; m.key_ld = ld_y;
    m.key_rows.assign(cal_row_start, cal_row_start + m.n_cal + 1);
  }
  if (m.many_pred && (m.key_out != out_pred || m.key_ld_out != ld_out || !same)) {
    // work units of the predict kernel ((tile, chunk) pairs, a tile's chunks next to each other) and every calendar's
    // view of the output table: its rows only, its n_pred columns only
    std::vector<PredUnit> units;
    std::vector<unsigned char> omaps((size_t)m.n_cal * 128);
    for (int c = 0; c < m.n_cal; ++c) {
      const CalMeta& cm = m.cals[c];
      const int64_t r0 = cal_row_start[c], nr = cal_row_start[c + 1] - r0;
      if (nr <= 0) { memset(omaps.data() + (size_t)c * 128, 0, 128); continue; }
      int rc = encode_2d(omaps.data() + (size_t)c * 128, out_pred + r0 * ld_out, (uint64_t)cm.n_pred, (uint64_t)nr,
                         (uint64_t)ld_out * 4, 32, 64);
      if (rc != MMF_OK) return rc;
      const int n_ch = (cm.n_pred + 127) / 128;
      for (int64_t r = r0; r < r0 + nr; r += 128)
        for (int ch = 0; ch < n_ch; ++ch)
          units.push_back(PredUnit{(int32_t)r, (int32_t)std::min<int64_t>(128, r0 + nr - r), c, ch,
                                   cm.row_off + cm.pred_start + ch * 128, (int32_t)(r - r0), {0, 0}});
    }
    int rc = grow((void**)&m.d_units, &m.units_cap, std::max<size_t>(1, units.size()) * sizeof(PredUnit));
    if (rc != MMF_OK) return rc;
    CU_TRY(cudaStreamSynchronize(s));
    if (!units.empty()) CU_TRY(cudaMemcpy(m.d_units, units.data(), units.size() * sizeof(PredUnit), cudaMemcpyHostToDevice));
    CU_TRY(cudaMemcpy(m.d_tmaps_out, omaps.data(), omaps.size(), cudaMemcpyHostToDevice));
    m.n_units = (int64_t)units.size();
    m.key_out = out_pred; m.key_ld_out = ld_out;
  }
  // ---- scratch, counters
  const bool may_mask = !ctx->cfg.assume_finite;
  FitArgs a{};
  a.y = y; a.n = n; a.ld_y = ld_y; a.pred_start = 0; a.n_pred = m.n_pred; a.out = out_pred; a.ld_out = ld_out;
  a.status = status; a.n_out = 1;
  if (m.many_pred) {
    int rc = grow((void**)&ctx->d_gamma, &ctx->gamma_cap_bytes, (size_t)n * P * sizeof(float));
    if (rc == MMF_OK) rc = grow((void**)&ctx->d_c, &ctx->c_cap_bytes, (size_t)n * sizeof(float));
    if (rc != MMF_OK) return rc;
    a.out_gamma = ctx->d_gamma; a.out_c = ctx->d_c; a.skip_pred = 1;
  }
  if (may_mask) {
    int rc = grow((void**)&ctx->d_recs, &ctx->recs_cap_bytes, (size_t)n * sizeof(SolveRec));
    if (rc == MMF_OK) rc = grow((void**)&ctx->d_rec_rows, &ctx->rec_rows_cap_bytes, (size_t)n * sizeof(int64_t));
    if (rc != MMF_OK) return rc;
    a.recs = ctx->d_recs; a.rec_rows = ctx->d_rec_rows; a.rec_cap = (uint32_t)n;
    ctx->rec_rows_clean = false;                           // ragged launches use the work list without the streaming solve
  }
  const int cs = ctx->counter_set;
  uint32_t* counters = ctx->d_pending + CTR_WORDS * cs;
  ctx->set_clean[cs] = false;
  CU_TRY(cudaMemsetAsync(counters, 0, CTR_WORDS * sizeof(uint32_t), s));
  CU_TRY(cudaMemsetAsync(m.d_pending_by_cal, 0, (size_t)m.n_cal * sizeof(uint32_t), s));
  if (may_mask) a.rec_count = counters + 1;
  DesignView d{};
  d.a4 = m.d_a4; d.at = m.d_at; d.apred = m.d_apred; d.w = m.d_w;
  d.n_rows = m.cals[0].n_rows; d.n_rows_pad = m.cals[0].n_rows_pad;
  d.t_fit = m.t_fit_max; d.t_pad = m.t_pad_max; d.kept_mask = 0xFFFFu; d.has_constant = m.has_constant;
  MultiView mv{};
  mv.cals = m.d_cals; mv.tiles = m.d_tiles; mv.tmaps_y = m.d_tmaps_y; mv.pending_by_cal = m.d_pending_by_cal;
  mv.n_cal = m.n_cal; mv.n_tiles = m.n_tiles;
  TcLaunch tl;
  int rc = encode_2d(tl.tmap_y, y, (uint64_t)m.cals[0].t_fit, (uint64_t)n, (uint64_t)ld_y * 4, 32, 128);   // unused by ragged tiles
  if (rc != MMF_OK) return rc;
  memcpy(tl.tmap_at, m.tmap_at, 128);
  if (stats) CU_TRY(cudaEventRecord(ctx->ev_k0, s));
  int launches = 0;
  CU_TRY(launch_fit_tc(d, a, tl, counters, ctx->sm_count, s, 0, &mv));
  ++launches;
  uint32_t pend = 0;
  if (may_mask) {
    // rows the streaming pass could not finish (first 8 values missing, too many gaps): the general pass runs once
    // per calendar that has any -- the one host round trip of a ragged call
    CU_TRY(cudaMemcpyAsync(&pend, counters, sizeof(pend), cudaMemcpyDeviceToHost, s));
    CU_TRY(cudaStreamSynchronize(s));
    if (pend > 0) {
      std::vector<uint32_t> by_cal(m.n_cal);
      CU_TRY(cudaMemcpy(by_cal.data(), m.d_pending_by_cal, (size_t)m.n_cal * sizeof(uint32_t), cudaMemcpyDeviceToHost));
      for (int c = 0; c < m.n_cal; ++c) {
        if (by_cal[c] == 0) continue;
        const CalMeta& cm = m.cals[c];
        const int64_t r0 = cal_row_start[c], nr = cal_row_start[c + 1] - r0;
        DesignView dc = d;
        dc.a4 = m.d_a4 + m.a4_off[c]; dc.apred = m.d_apred + (size_t)cm.row_off * P;
        dc.n_rows = cm.n_rows; dc.n_rows_pad = cm.n_rows_pad; dc.t_fit = cm.t_fit; dc.t_pad = (cm.t_fit + 31) & ~31;
        dc.kept_mask = cm.kept_mask;
        FitArgs ac = a;
        ac.y = y + r0 * ld_y; ac.n = nr; ac.out = out_pred + r0 * ld_out; ac.status = status + r0;
        ac.pred_start = cm.pred_start; ac.recs = a.recs + r0; ac.row_base = r0; ac.cal_id = c;
        if (a.out_gamma != nullptr) { ac.out_gamma = a.out_gamma + r0 * P; ac.out_c = a.out_c + r0; }
        ac.only_pending = 1; ac.pending_count = nullptr;
        CU_TRY(launch_fit_warp(dc, ac, ctx->sm_count, s));
        ++launches;
      }
    }
    CU_TRY(launch_solve_rows(d, a, ctx->sm_count, s, m.d_cals));
    ++launches;
  }
  if (m.many_pred) {
    PredictLaunch pl;
    memcpy(pl.tmap_bhi, m.tmap_bhi, 128);
    memcpy(pl.tmap_blo, m.tmap_blo, 128);
    memcpy(pl.tmap_out, m.tmap_bhi, 128);                  // unused by the ragged kernel (per-calendar maps instead)
    CU_TRY(launch_predict_tc(d, a, pl, ctx->sm_count, s, m.d_units, m.n_units, m.d_tmaps_out));
    ++launches;
  }
  ctx->last_set = cs;
  if (stats) {
    CU_TRY(cudaEventRecord(ctx->ev_k1, s));
    CU_TRY(cudaEventSynchronize(ctx->ev_k1));
    CU_TRY(cudaEventElapsedTime(&stats->kernel_ms, ctx->ev_k0, ctx->ev_k1));
    stats->total_ms = stats->kernel_ms;
    stats->n_series = n; stats->n_pending = pend; stats->kernel_launches = launches; stats->kernel_used = MMF_KERNEL_TC;
  }
  return MMF_OK;
}

int mmf_fit_forecast_bcast_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t pred_start,
                               int32_t n_pred, const uint64_t* out_ptrs, int32_t n_out, int32_t multimem,
                               int64_t ld_out, float* out_beta, int32_t* out_status) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  if (!ctx->plan.valid) return fail(MMF_E_NOPLAN, "mmf_plan_design has not been called");
  const Plan& pl = ctx->plan;
  if (n < 0 || (n > 0 && (!y || !out_ptrs))) return fail(MMF_E_INVALID, "bad y / out_ptrs / n");
  if (n_out < 1 || n_out > MAX_OUT) return fail(MMF_E_INVALID, "n_out=%d outside [1,%d]", n_out, MAX_OUT);
  if (multimem < 0 || multimem > 2) return fail(MMF_E_INVALID, "multimem must be 0, 1 (multimem.st) or 2 (bulk stores to the multicast address)");
  if (multimem && n_out != 1) return fail(MMF_E_INVALID, "multimem=1 takes exactly one (multicast) pointer");
  if (ld_y < pl.t_fit) return fail(MMF_E_INVALID, "ld_y=%lld < t_fit=%d", (long long)ld_y, pl.t_fit);
  if (n_pred < 1 || pred_start < 0 || (int64_t)pred_start + n_pred > pl.n_rows)
    return fail(MMF_E_INVALID, "prediction rows [%d,%d) outside the planned design (%d rows)", pred_start,
                pred_start + n_pred, pl.n_rows);
  if (ld_out < n_pred) return fail(MMF_E_INVALID, "ld_out=%lld < n_pred=%d", (long long)ld_out, n_pred);
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));
  if (!is_device_ptr(y)) return fail(MMF_E_INVALID, "the broadcast variant takes device buffers only");
  int32_t* status = out_status;
  if (!status) {
    int rc = grow_status_scratch(ctx, n, ctx->stream);
    if (rc != MMF_OK) return rc;
    status = ctx->d_status_scratch;
  }
  float* more[MAX_OUT - 1] = {};
  for (int i = 1; i < n_out; ++i) more[i - 1] = reinterpret_cast<float*>(out_ptrs[i]);
  int launches = 0, kernel_used = 0;
  return run_device(ctx, y, n, ld_y, pred_start, n_pred, reinterpret_cast<float*>(out_ptrs[0]), ld_out, out_beta,
                    status, ctx->stream, &launches, &kernel_used, more, n_out, multimem);
}

int mmf_fit_select_forecast_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                                const int32_t* candidates, int32_t n_cand, int32_t pred_start, int32_t n_pred,
                                float* out_pred, int64_t ld_out, int32_t* out_choice, float* out_mse,
                                int32_t* out_status) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  if (!ctx->plan.valid) return fail(MMF_E_NOPLAN, "mmf_plan_design has not been called");
  const Plan& pl = ctx->plan;
  if (n < 0 || (n > 0 && (!y || !out_pred))) return fail(MMF_E_INVALID, "bad y / out_pred / n");
  if (!candidates || n_cand < 1 || n_cand > MMF_MAX_CAND) return fail(MMF_E_INVALID, "need 1..%d candidates", MMF_MAX_CAND);
  for (int i = 0; i < n_cand; ++i)
    if (candidates[i] < 1 || candidates[i] > P || (i > 0 && candidates[i] <= candidates[i - 1]))
      return fail(MMF_E_INVALID, "candidates must be ascending column counts in [1,%d]", P);
  if (n_hold < 1 || pl.t_fit + n_hold > pl.n_rows) return fail(MMF_E_INVALID, "held-out rows exceed the planned design");
  if (n_hold > MMF_SELECT_MAX_HOLD)
    return fail(MMF_E_UNSUPPORTED, "n_hold=%d: select_kernel stages the held-out design rows in shared memory, at most %d",
                n_hold, MMF_SELECT_MAX_HOLD);
  if (ld_y < pl.t_fit + n_hold) return fail(MMF_E_INVALID, "y must hold the fit rows and the held-out rows");
  if (n_pred < 1 || pred_start < 0 || (int64_t)pred_start + n_pred > pl.n_rows)
    return fail(MMF_E_INVALID, "prediction rows outside the planned design");
  if (ld_out < n_pred) return fail(MMF_E_INVALID, "ld_out < n_pred");
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));
  if (!is_device_ptr(y) || !is_device_ptr(out_pred)) return fail(MMF_E_INVALID, "device buffers only");
  int32_t* status = out_status;
  if (!status) {
    int rc = grow_status_scratch(ctx, n, ctx->stream);
    if (rc != MMF_OK) return rc;
    status = ctx->d_status_scratch;
  }
  SelectArgs sel{};
  sel.n_hold = n_hold;
  sel.n_cand = n_cand;
  for (int i = 0; i < n_cand; ++i) sel.cand[i] = candidates[i];
  sel.out_choice = out_choice;
  sel.out_mse = out_mse;
  int launches = 0, kernel_used = 0;
  return run_device(ctx, y, n, ld_y, pred_start, n_pred, out_pred, ld_out, nullptr, status, ctx->stream, &launches,
                    &kernel_used, nullptr, 1, 0, &sel);
}

// ---- device-side packer (pack.cu): every pointer is a device pointer, work is enqueued on the ctx stream
#define PACK_PROLOGUE()                                              \
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");               \
  if (n < 0) return fail(MMF_E_INVALID, "n < 0");                    \
  CU_TRY(cudaSetDevice(ctx->device));

int mmf_pack_hash_utf8(mmf_ctx* ctx, const int32_t* offsets, const uint8_t* data, int64_t n, uint64_t* hash,
                       int32_t first) {
  PACK_PROLOGUE();
  CU_TRY(pack_hash_utf8(offsets, data, n, hash, first, ctx->sm_count, ctx->stream));
  return MMF_OK;
}

int mmf_pack_hash_i32(mmf_ctx* ctx, const int32_t* values, int64_t n, uint64_t* hash, int32_t first) {
  PACK_PROLOGUE();
  CU_TRY(pack_hash_i32(values, n, hash, first, ctx->sm_count, ctx->stream));
  return MMF_OK;
}

int mmf_pack_group_codes(mmf_ctx* ctx, const uint64_t* hash, int64_t n, int32_t* gid, int32_t* first_row,
                         int32_t* n_groups) {
  PACK_PROLOGUE();
  if (!n_groups) return fail(MMF_E_INVALID, "n_groups is NULL");
  if (n > 0x7fffffff) return fail(MMF_E_UNSUPPORTED, "more than 2^31-1 rows in one pack call");
  size_t need = 0;
  CU_TRY(pack_group_codes_scratch_bytes(n, &need));
  GrowScope grow_scope(ctx);
  if (int rc = grow(&ctx->d_pack_scratch, &ctx->pack_scratch_cap, need)) return rc;
  CU_TRY(pack_group_codes(hash, n, gid, first_row, n_groups, ctx->d_pack_scratch, ctx->sm_count, ctx->stream));
  return MMF_OK;
}

int mmf_pack_verify_utf8(mmf_ctx* ctx, const int32_t* offsets, const uint8_t* data, int64_t n, const int32_t* gid,
                         const int32_t* first_row, uint64_t* mismatches) {
  PACK_PROLOGUE();
  if (!mismatches) return fail(MMF_E_INVALID, "mismatches is NULL");
  CU_TRY(pack_verify_utf8(offsets, data, n, gid, first_row, mismatches, ctx->sm_count, ctx->stream));
  return MMF_OK;
}

int mmf_pack_verify_i32(mmf_ctx* ctx, const int32_t* values, int64_t n, const int32_t* gid, const int32_t* first_row,
                        uint64_t* mismatches) {
  PACK_PROLOGUE();
  if (!mismatches) return fail(MMF_E_INVALID, "mismatches is NULL");
  CU_TRY(pack_verify_i32(values, n, gid, first_row, mismatches, ctx->sm_count, ctx->stream));
  return MMF_OK;
}

int mmf_pack_minmax(mmf_ctx* ctx, const int32_t* gid, const int32_t* day, int64_t n, int32_t n_groups,
                    int32_t* gmin, int32_t* gmax) {
  PACK_PROLOGUE();
  CU_TRY(pack_minmax(gid, day, n, n_groups, gmin, gmax, ctx->sm_count, ctx->stream));
  return MMF_OK;
}

int mmf_pack_scatter_f32(mmf_ctx* ctx, const int32_t* gid, const int32_t* day, const float* val, int64_t n,
                         const int64_t* row_of_group, const int32_t* gstart, int32_t step, float* y, int64_t n_rows,
                         int64_t ld_y, int32_t t_len, uint64_t* duplicates) {
  PACK_PROLOGUE();
  if (step < 1 || ld_y % 4 != 0 || ld_y < t_len || (reinterpret_cast<uintptr_t>(y) & 15u) != 0)
    return fail(MMF_E_INVALID, "need step >= 1, a 16-B aligned y and ld_y >= t_len, ld_y %% 4 == 0");
  CU_TRY(pack_scatter(gid, day, val, n, row_of_group, gstart, step, y, n_rows, ld_y, t_len,
                      reinterpret_cast<unsigned long long*>(duplicates), ctx->sm_count, ctx->stream));
  return MMF_OK;
}

int mmf_alloc_pinned(size_t bytes, void** out) {
  if (!out) return fail(MMF_E_INVALID, "out is NULL");
  CU_TRY(cudaHostAlloc(out, bytes, cudaHostAllocDefault));
  return MMF_OK;
}

int mmf_free_pinned(void* p) {
  if (p) CU_TRY(cudaFreeHost(p));
  return MMF_OK;
}

int mmf_host_register(void* p, size_t bytes) {
  if (!p) return fail(MMF_E_INVALID, "pointer is NULL");
  CU_TRY(cudaHostRegister(p, bytes, cudaHostRegisterDefault));
  return MMF_OK;
}

int mmf_host_unregister(void* p) {
  if (p) CU_TRY(cudaHostUnregister(p));
  return MMF_OK;
}

}  // extern "C"
