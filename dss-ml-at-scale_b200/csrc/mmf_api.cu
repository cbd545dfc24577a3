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
#include <initializer_list>
#include <optional>
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
  uint32_t* d_nz = nullptr;    // [n_rows] non-zero masks of the whitened rows (AR calls: the used columns of the dof rule)
  int32_t x_cols = 0;          // mmf_plan_design: columns and 64-bit hash of the raw X (host side; a (p, d) selection
  uint64_t x_hash = 0;         // refuses an ARIMA plan built from another X)
  float* d_sfac = nullptr;    // [n_rows] sqrt(1 + |a_t|^2) (float64 on the host): se of gap-free rows / sigma
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

// Backtest plan (DESIGN.md section 4.12): the longest window [0, t_K) is the basis the tensor-core kernel accumulates in;
// origin k is calendar k of a stacked plan (its own whitening, t_fit = t_k), which the general passes use as they are.
struct BtPlan {
  bool valid = false;
  int32_t n_origin = 0, horizon = 0;
  int32_t origin[MMF_BT_MAX_ORIGINS] = {};
  Plan common;
  MultiPlan cals;
  float* d_pred = nullptr;             // [K][horizon][P] origin k's prediction rows in the common basis, T_k a^(k)_t
  float* d_tmat = nullptr;             // [K][P][P] T_k = W^-1 W_k
};

// ARIMA plan (DESIGN.md section 4.15): the differenced designs D_d, d = 1 .. max_diff, each planned by build_plan as
// mmf_plan_design would plan it (no centring); n_rows / t_fit are the level rows of the calendar
struct ArimaPlan {
  bool valid = false;
  int32_t max_diff = 0, n_rows = 0, t_fit = 0;
  int32_t x_cols = 0;                  // columns and 64-bit hash of the raw X the designs were differenced from
  uint64_t x_hash = 0;
  Plan diff[MMF_DIFF_MAX];
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
  cudaEvent_t ev_switch = nullptr;     // mmf_set_stream: the new stream waits for what the old one holds
  uint32_t* d_pending = nullptr;       // 3 counter sets of CTR_WORDS words {rows left PENDING, solve records queued,
                                       // ...}: 0/1 ping-pong between eager calls, 2 belongs to captured CUDA graphs
                                       // (zeroed by a node of the graph)
  int counter_set = 0;                 // set the next eager call uses
  bool set_clean[2] = {true, true};    // the set is known to be zero (cudaMemset at create, or zeroed by the previous
                                       // eager call's tensor-core kernel); anything else makes the call memset its set
  int last_set = 0;                    // set the last enqueued call used (stats read n_pending from it)
  uint32_t* d_slab_pending = nullptr;  // n_pending of every slab of a multi-slab call with stats (grown on demand)
  size_t slab_pending_cap = 0;
  int pinned = 0;                     // > 0: a captured CUDA graph holds pointers into the scratch below and into the plan
  bool status_scratch_captured = false;   // some capture ran without a caller-provided status buffer
  SolveRec* d_recs = nullptr;          // deferred masked series (grown on demand, capped)
  size_t recs_cap_bytes = 0;
  int64_t* d_rec_rows = nullptr;
  size_t rec_rows_cap_bytes = 0;
  float* d_gamma = nullptr;            // [n][P] + d_c[n]: hand-off from the fit kernels to predict_tc_kernel
  size_t gamma_cap_bytes = 0;
  float* d_c = nullptr;
  size_t c_cap_bytes = 0;
  float* d_sigma_scratch = nullptr;    // sigma of a standard-error call that did not ask for it (the holdout se rows need it)
  size_t sigma_scratch_cap = 0;
  int32_t* d_status_scratch = nullptr;
  size_t status_scratch_cap = 0;
  void* d_pack_scratch = nullptr;      // sort / scan work space of the packer (grown on demand, kept)
  size_t pack_scratch_cap = 0;
  Plan plan;
  MultiPlan multi;
  BtPlan bt;
  ArimaPlan arima;
  float* d_z = nullptr;  size_t z_cap_bytes = 0;           // ARIMA calls: z' of one slab, round4(t_fit - d) per row
  ArimaSelBest* d_asel_best = nullptr;  size_t asel_best_cap = 0;   // (p, d) selection, per slab: running best,
  int32_t* d_asel_status = nullptr;  size_t asel_status_cap = 0;    // and the status of the fit of the current d
  float* d_hsel_q0 = nullptr;  size_t hsel_q0_cap = 0;     // (p, d, q) selection, per slab: the q = 0 scores
  float* d_css_hr = nullptr;  size_t css_hr_cap = 0;       // CSS calls, per slab: the HR phi / theta / ma_order the
                                                           // caller did not ask for
  int32_t* d_refit = nullptr;  size_t refit_cap = 0;       // selection refits, per slab: the winner's outputs the caller
                                                           // did not ask for, the row list and its length
  float* d_bt_mom = nullptr;  size_t bt_mom_cap = 0;   // backtest scratch, per slab: moments at the earlier origins,
  SolveRec* d_bt_recs = nullptr;  size_t bt_recs_cap = 0;   // [K][slab] records, [K][slab] work lists,
  int64_t* d_bt_rows = nullptr;  size_t bt_rows_cap = 0;
  uint32_t* d_bt_ctr = nullptr;  size_t bt_ctr_cap = 0;     // {records queued[K], rows left to the general pass[K]},
  float* d_bt_pred = nullptr;  size_t bt_pred_cap = 0;      // forecasts when the caller did not ask for them
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
  cudaFree(p.d_sfac); cudaFree(p.d_nz);
  p = Plan{};
}

void free_arima(ArimaPlan& m) {
  for (Plan& p : m.diff) free_plan(p);
  m = ArimaPlan{};
}

void free_bt(BtPlan& b) {
  free_plan(b.common);
  free_multi(b.cals);
  cudaFree(b.d_pred); cudaFree(b.d_tmat);
  b = BtPlan{};
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

// FNV-1a over the bytes of a planned X: plans built from the same X carry the same hash
uint64_t hash_x(const double* X, int64_t count) {
  const unsigned char* b = reinterpret_cast<const unsigned char*>(X);
  uint64_t h = 14695981039346656037ull;
  for (int64_t i = 0; i < count * (int64_t)sizeof(double); ++i) h = (h ^ b[i]) * 1099511628211ull;
  return h;
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

// the stacked designs of a ragged plan (or of a backtest plan's origins), as the kernels that take every calendar see them
DesignView view_of(const MultiPlan& m) {
  DesignView d{};
  d.a4 = m.d_a4; d.at = m.d_at; d.apred = m.d_apred; d.w = m.d_w;
  d.n_rows = m.cals[0].n_rows; d.n_rows_pad = m.cals[0].n_rows_pad;
  d.t_fit = m.t_fit_max; d.t_pad = m.t_pad_max; d.kept_mask = 0xFFFFu; d.has_constant = m.has_constant;
  return d;
}

// calendar c of a ragged plan on its own (the general pass of its rows)
DesignView view_of(const MultiPlan& m, int c) {
  const CalMeta& cm = m.cals[c];
  DesignView d = view_of(m);
  d.a4 = m.d_a4 + m.a4_off[c]; d.apred = m.d_apred + (size_t)cm.row_off * P;
  d.n_rows = cm.n_rows; d.n_rows_pad = cm.n_rows_pad; d.t_fit = cm.t_fit; d.t_pad = (cm.t_fit + 31) & ~31;
  d.kept_mask = cm.kept_mask;
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

// The device tables of one calendar (mmf_plan_design; the common basis of a backtest plan).  X is validated.
int build_plan(Plan& pl, const double* X, int32_t n_rows, int32_t p, int32_t t_fit, int32_t has_constant) {

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
  // leverage of a gap-free series (G_i = I): h_t = |a_t|^2 over the kept columns (the others are zero in A)
  std::vector<float> sfac(n_rows);
  for (int32_t t = 0; t < n_rows; ++t) {
    double h = 0.0;
    for (int q = 0; q < P; ++q) h += (double)A[(size_t)t * P + q] * (double)A[(size_t)t * P + q];
    sfac[t] = (float)std::sqrt(1.0 + h);
  }
  CU_TRY(cudaMalloc(&pl.d_sfac, sfac.size() * sizeof(float)));
  CU_TRY(cudaMemcpy(pl.d_sfac, sfac.data(), sfac.size() * sizeof(float), cudaMemcpyHostToDevice));
  std::vector<uint32_t> nz(n_rows, 0u);
  for (int32_t t = 0; t < n_rows; ++t)
    for (int q = 0; q < P; ++q) nz[t] |= (A[(size_t)t * P + q] != 0.f ? 1u : 0u) << q;
  CU_TRY(cudaMalloc(&pl.d_nz, nz.size() * sizeof(uint32_t)));
  CU_TRY(cudaMemcpy(pl.d_nz, nz.data(), nz.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  int rc = encode_2d(pl.tmap_at, pl.d_at, (uint64_t)pl.t_pad, (uint64_t)(2 * P), (uint64_t)pl.t_pad * 4, 32, 2 * P);
  if (rc != MMF_OK) return rc;
  rc = encode_2d(pl.tmap_bhi, pl.d_ap_hi, (uint64_t)P, (uint64_t)n_rows, (uint64_t)P * 4, P, 128, CU_TENSOR_MAP_SWIZZLE_64B);
  if (rc != MMF_OK) return rc;
  rc = encode_2d(pl.tmap_blo, pl.d_ap_lo, (uint64_t)P, (uint64_t)n_rows, (uint64_t)P * 4, P, 128, CU_TENSOR_MAP_SWIZZLE_64B);
  if (rc != MMF_OK) return rc;
  pl.valid = true;
  return MMF_OK;
}

// Stack the whitened designs of n_cal calendars (mmf_plan_calendars; the origins of a backtest plan).  Validates the
// calendars, then waits for the stream `sync` before it frees the previous tables of `m`.
int build_multi(MultiPlan& m, const double* X_all, int32_t n_cal, const int32_t* n_rows, const int32_t* t_fit,
                const int32_t* pred_start, const int32_t* n_pred_cal, int32_t p, int32_t has_constant, bool many,
                int32_t n_pred, int32_t n_pred_max, cudaStream_t sync) {
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
  if (total_rows > (size_t)INT32_MAX) return fail(MMF_E_UNSUPPORTED, "too many design rows in one ragged plan");
  for (size_t i = 0; i < total_rows * (size_t)p; ++i)
    if (!std::isfinite(X_all[i])) return fail(MMF_E_INVALID, "design matrix has a non-finite entry at %zu", i);
  if (has_constant) {                                      // every argument check comes before the previous plan is freed
    size_t off = 0;
    for (int c = 0; c < n_cal; off += (size_t)n_rows[c], ++c)
      for (int32_t t = 0; t < n_rows[c]; ++t)
        if (X_all[(off + t) * (size_t)p] != 1.0) return fail(MMF_E_INVALID, "has_constant=1 but calendar %d has X[%d,0] != 1", c, t);
  }
  CU_TRY(cudaStreamSynchronize(sync));
  free_multi(m);
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

// Launch and kernel-choice bookkeeping of one call (mmf_stats.kernel_launches / kernel_used)
struct Tally {
  int launches = 0;
  int kernel_used = 0;
};

// One call of the device path: the plain fit and the model stages behind it, each present or not.  ARIMA calls (arima,
// with ar): y / ld_y are the levels; diff_kernel writes z' into the context's scratch first, and the fit passes and
// arima_kernel read z' with the plan of D_d.  (p, d) selections (asel) run one call per listed d and end in
// arima_select_kernel; their d = 0 call (arima->d == 0) fits y itself with the mmf_plan_design plan; (p, d, q) selections
// (hsel, with asel) add arma_select_kernel behind it.  ARMA calls (arma, with ar) run arma_kernel behind ar_kernel
// (d = 0, no arima) or arima_kernel; CSS calls (css, with arma) add arma_css_kernel behind arma_kernel, joint calls (joint,
// with css) arma_joint_kernel in its place, ML calls (ml, with css) arma_ml_kernel behind arma_css_kernel, Kalman-predictor
// calls (kf, with ml) arma_kf_kernel behind arma_ml_kernel.  Refit stages of a (p, d, q) selection (refit, with ar, arima, arma and css)
// run the fit of their d, refit_list_kernel and arma_css_list_kernel (joint: arma_joint_list_kernel); with ml they add
// refit_ml_cols_kernel and arma_ml_list_kernel, with kf arma_kf_list_kernel (kf_list), and se_pass runs arima_se_kernel
// over the slab with the per-series d behind them; kf_only stages run the fit, the list and arma_kf_list_kernel alone.
struct Call {
  const float* y = nullptr;
  int64_t ld_y = 0;
  int32_t pred_start = 0, n_pred = 0;
  float* out = nullptr;
  int64_t ld_out = 0;
  float* beta = nullptr;
  int32_t* status = nullptr;
  float* out_more[MAX_OUT - 1] = {};
  int n_out = 1, multimem = 0;
  std::optional<SelectArgs> sel;
  std::optional<SeArgs> se;
  std::optional<ArArgs> ar;
  std::optional<ArSelArgs> arsel;
  std::optional<ArimaArgs> arima;
  std::optional<ArimaSelArgs> asel;
  std::optional<ArmaArgs> arma;
  std::optional<ArmaSelArgs> hsel;
  std::optional<CssArgs> css;
  std::optional<JointArgs> joint;
  std::optional<MlArgs> ml;
  std::optional<KfArgs> kf;
  std::optional<RefitArgs> refit;
  bool kf_list = false, se_pass = false, kf_only = false;   // refit stages of the ML + Kalman call (DESIGN.md 4.25)

  // the same call on the rows from `off` on: every per-row output advanced by `off` rows (null stays null)
  Call slice(int64_t off) const {
    auto at = [off](auto* p, int64_t width) { return p ? p + off * width : p; };
    Call c = *this;
    c.y = y + off * ld_y;
    c.out = out + off * ld_out;
    c.beta = at(beta, P);
    if (!asel && !refit) c.status = status + off;   // selection and refit fits write the per-slab scratch
    for (int i = 0; i + 1 < n_out && i < MAX_OUT - 1; ++i) c.out_more[i] = out_more[i] + off * ld_out;
    if (sel) { c.sel->out_choice = at(sel->out_choice, 1); c.sel->out_mse = at(sel->out_mse, 1); }
    if (se) { c.se->out_se = at(se->out_se, se->ld_se); c.se->sigma = at(se->sigma, 1); c.se->dof = at(se->dof, 1); }
    if (ar) { c.ar->phi = at(ar->phi, MMF_AR_MAX); c.ar->order = at(ar->order, 1); c.ar->sigma = at(ar->sigma, 1); }
    if (arsel) {
      c.arsel->choice = at(arsel->choice, 1);
      c.arsel->mse = at(arsel->mse, 1);
      c.arsel->cand_mse = at(arsel->cand_mse, arsel->n_cand);
    }
    if (asel) {
      c.asel->choice_p = at(asel->choice_p, 1);
      c.asel->choice_d = at(asel->choice_d, 1);
      c.asel->mse = at(asel->mse, 1);
      c.asel->status = at(asel->status, 1);
      // (p, d, q) selections: arima_select_kernel's scores go to scratch, arma_select_kernel copies them into the q = 0
      // slice of hsel->cand_mse
      if (!hsel) c.asel->cand_mse = at(asel->cand_mse, (int64_t)asel->n_diffs * asel->n_cand);
    }
    if (arma) { c.arma->theta = at(arma->theta, MMF_MA_MAX); c.arma->ma_order = at(arma->ma_order, 1); }
    if (hsel) {
      c.hsel->choice_q = at(hsel->choice_q, 1);
      c.hsel->theta = at(hsel->theta, MMF_MA_MAX);
      c.hsel->ma_order = at(hsel->ma_order, 1);
      c.hsel->cand_mse = at(hsel->cand_mse, (int64_t)asel->n_diffs * hsel->n_mas * asel->n_cand);
    }
    if (css) {
      c.css->css_start = at(css->css_start, 1);
      c.css->css = at(css->css, 1);
      c.css->css_stop = at(css->css_stop, 1);
      c.css->iters = at(css->iters, 1);
    }
    if (joint) c.joint->beta = at(joint->beta, P);
    if (ml) {
      c.ml->loglik_start = at(ml->loglik_start, 1);
      c.ml->loglik = at(ml->loglik, 1);
      c.ml->stop = at(ml->stop, 1);
      c.ml->iters = at(ml->iters, 1);
    }
    if (kf) c.kf->se = at(kf->se, kf->ld_se);
    if (refit) { c.refit->choice_d = at(refit->choice_d, 1); c.refit->choice_q = at(refit->choice_q, 1); }
    return c;
  }
};

// Enqueue the fit of ONE slab of n device-resident rows on the context's stream, against `plan` (ctx->plan, or the
// differenced plan of an ARIMA call).  c.status must be non-null.
int run_device_slab(mmf_ctx* ctx, const Plan& plan, const Call& c, int64_t n, Tally& t) {
  const cudaStream_t s = ctx->stream;
  const DesignView d = view_of(plan);
  const float* y = c.y;
  int64_t ld_y = c.ld_y;
  ArimaArgs ma{};
  if (c.arima) {
    ma = *c.arima;
    ma.y = y;
  }
  if (c.arima && ma.d > 0) {
    const int64_t ld_z = (plan.t_fit + 3) & ~3;              // 16-B row pitch: fit_tc's TMA path
    int rc = grow((void**)&ctx->d_z, &ctx->z_cap_bytes, (size_t)n * ld_z * sizeof(float));
    if (rc != MMF_OK) return rc;
    CU_TRY(launch_diff(ma, ctx->d_z, ld_z, n, ctx->sm_count, s));
    ++t.launches;
    y = ctx->d_z;
    ld_y = ld_z;
  }
  FitArgs a{};
  a.y = y; a.n = n; a.ld_y = ld_y; a.pred_start = c.pred_start; a.n_pred = c.n_pred;
  a.out = c.out; a.ld_out = c.ld_out; a.out_beta = c.beta; a.status = c.status;
  a.n_out = c.n_out; a.out_multimem = c.multimem;
  for (int i = 0; i + 1 < c.n_out && i < MAX_OUT - 1; ++i) a.out_more[i] = c.out_more[i];
  a.only_pending = 0; a.pending_count = nullptr;
  const char* why = nullptr;
  int kernel = ctx->cfg.kernel;
  // Many prediction rows (the reference's "Demand_Fitted for every date", 02:484-494): fit kernels hand
  // gamma/c to predict_tc_kernel, which writes the [n, n_pred] table with TMA stores.
  const bool predict_ok = c.n_out == 1 && !c.multimem && c.ld_out % 4 == 0 &&
                          (reinterpret_cast<uintptr_t>(c.out) & 15u) == 0 && n <= (int64_t)0x7fffffff - 128;
  if (c.sel && !predict_ok)
    return fail(MMF_E_UNSUPPORTED, "model selection needs a 16-B aligned output with ld_out %% 4 == 0");
  // AR calls (ar) hand gamma / c to ar_kernel, which writes the table itself: no predict_tc requirement
  const bool many_pred = !c.ar && (c.sel || (c.n_pred > 64 && kernel != MMF_KERNEL_WARP && predict_ok));
  if (many_pred || c.ar) {
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
    if (rc == MMF_OK) rc = grow((void**)&ctx->d_rec_rows, &ctx->rec_rows_cap_bytes, (size_t)cap * sizeof(int64_t));
    if (rc != MMF_OK) return rc;
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
  const SeArgs* se = c.se ? &*c.se : nullptr;
  if (kernel == MMF_KERNEL_TC) {
    TcLaunch tl;
    int rc = encode_2d(tl.tmap_y, y, (uint64_t)d.t_fit, (uint64_t)n, (uint64_t)ld_y * 4, 32, 128);
    if (rc != MMF_OK) return rc;
    memcpy(tl.tmap_at, plan.tmap_at, 128);
    if (se != nullptr) {
      CU_TRY(launch_fit_tc_se(d, a, tl, counters, ctx->sm_count, s, *se));
      ++t.launches;
      if (many_pred) {          // se rows of the rows fit_tc finished, before the passes behind it change any status
        CU_TRY(launch_se_outer(a, *se, ctx->sm_count, s));
        ++t.launches;
      }
    } else {
      CU_TRY(launch_fit_tc(d, a, tl, counters, ctx->sm_count, s, ctx->cfg.tc_variant));
      ++t.launches;
    }
    if (may_mask) {
      FitArgs m = a;
      m.only_pending = 1;
      m.pending_count = counters;
      CU_TRY(launch_fit_warp(d, m, ctx->sm_count, s, se));
      CU_TRY(launch_solve_rows(d, m, ctx->sm_count, s, nullptr, se));   // the records both passes queued
      t.launches += 2;
    }
  } else {
    CU_TRY(launch_fit_warp(d, a, ctx->sm_count, s, se));
    ++t.launches;
    if (may_mask) {
      CU_TRY(launch_solve_rows(d, a, ctx->sm_count, s, nullptr, se));
      ++t.launches;
    }
  }
  if (c.sel) {
    CU_TRY(launch_select(d, a, *c.sel, ctx->sm_count, s));
    ++t.launches;
  }
  if (c.refit) {
    // the winners of this d: refit_list_kernel lists them (and writes the refit outputs of the rows the list leaves
    // out), then the list kernel refits them from the winner's outputs.  ma is this d's (ma.y = a.y for d = 0)
    CU_TRY(cudaMemsetAsync(c.refit->count, 0, sizeof(uint32_t), s));
    const JointArgs jt = c.joint ? *c.joint : JointArgs{};
    CU_TRY(launch_refit_list(d, a, ma, *c.css, jt, *c.refit, s));
    ++t.launches;
    if (!c.kf_only) {
      CU_TRY(c.joint ? launch_arma_joint_list(d, a, *c.ar, ma, *c.arma, *c.css, jt, *c.refit, s)
                     : launch_arma_css_list(d, a, *c.ar, ma, *c.arma, *c.css, *c.refit, s));
      ++t.launches;
    }
    if (c.ml && !c.kf_only) {       // the ML refit from the CSS refit's estimate; the ML columns of the other rows
      CU_TRY(launch_refit_ml_cols(a, ma, *c.ml, *c.refit, s));
      CU_TRY(launch_arma_ml_list(d, a, *c.ar, ma, *c.arma, *c.ml, *c.refit, s));
      t.launches += 2;
    }
    if (c.se_pass) {                // every row's se of the library's predictor, each row at its own d, once every d's
      ArimaSeArgs sa{};             // ML refit has run; the Kalman stages behind overwrite the rows they cover
      sa.y = c.y; sa.ld_y = c.ld_y; sa.t_fit = ma.t_fit; sa.diffs = c.refit->choice_d;
      sa.phi = c.ar->phi; sa.order = c.ar->order; sa.theta = c.arma->theta; sa.ma_order = c.arma->ma_order;
      sa.sigma = c.ar->sigma; sa.pred_start = c.pred_start; sa.n_pred = c.n_pred;
      sa.out = c.kf->se; sa.ld_se = c.kf->ld_se; sa.n = n;
      CU_TRY(launch_arima_se(sa, ctx->sm_count, s));
      ++t.launches;
    }
    if (c.kf_list) {
      CU_TRY(launch_arma_kf_list(d, a, *c.ar, ma, *c.arma, *c.kf, *c.refit, s));
      ++t.launches;
    }
  } else if (c.ar) {
    CU_TRY(c.asel    ? launch_arima_select(d, a, *c.ar, ma, *c.asel, s)
           : c.arima ? launch_arima(d, a, *c.ar, ma, s)
           : c.arsel ? launch_ar_select(d, a, *c.ar, *c.arsel, s) : launch_ar(d, a, *c.ar, s));
    ++t.launches;
    if (c.hsel) {
      CU_TRY(launch_arma_select(d, a, *c.ar, ma, *c.asel, *c.hsel, s));
      ++t.launches;
    }
    if (c.arma) {
      ArimaArgs mh = ma;
      if (!c.arima) { mh.y = a.y; mh.ld_y = a.ld_y; mh.t_fit = d.t_fit; mh.d = 0; }
      CU_TRY(launch_arma(d, a, *c.ar, mh, *c.arma, s));
      ++t.launches;
      if (c.css) {
        CU_TRY(c.joint ? launch_arma_joint(d, a, *c.ar, mh, *c.arma, *c.css, *c.joint, s)
                       : launch_arma_css(d, a, *c.ar, mh, *c.arma, *c.css, s));
        ++t.launches;
        if (c.ml) {
          CU_TRY(launch_arma_ml(d, a, *c.ar, mh, *c.arma, *c.ml, s));
          ++t.launches;
        }
        if (c.kf) {
          if (c.kf->se) {            // every row's se of the library's predictor; arma_kf_kernel overwrites its rows
            ArimaSeArgs sa{};
            sa.y = c.y; sa.ld_y = c.ld_y; sa.t_fit = mh.t_fit; sa.diff_order = mh.d;
            sa.phi = c.ar->phi; sa.order = c.ar->order; sa.theta = c.arma->theta; sa.ma_order = c.arma->ma_order;
            sa.sigma = c.ar->sigma; sa.pred_start = c.pred_start; sa.n_pred = c.n_pred;
            sa.out = c.kf->se; sa.ld_se = c.kf->ld_se; sa.n = n;
            CU_TRY(launch_arima_se(sa, ctx->sm_count, s));
            ++t.launches;
          }
          CU_TRY(launch_arma_kf(d, a, *c.ar, mh, *c.arma, *c.kf, s));
          ++t.launches;
        }
      }
    }
  }
  if (many_pred) {
    PredictLaunch pl;
    memcpy(pl.tmap_bhi, plan.tmap_bhi, 128);
    memcpy(pl.tmap_blo, plan.tmap_blo, 128);
    // the map stops at the last whole 16 B of a row (TMA clips with 16-B granularity); the kernel stores the
    // n_pred % 4 columns behind it itself, so the caller's columns from n_pred on are never written
    pl.n_tma = c.n_pred & ~3;
    int rc = encode_2d(pl.tmap_out, c.out, (uint64_t)(pl.n_tma > 0 ? pl.n_tma : c.n_pred), (uint64_t)n,
                       (uint64_t)c.ld_out * 4, 32, 64);   // one box per warpgroup half
    if (rc != MMF_OK) return rc;
    CU_TRY(launch_predict_tc(d, a, pl, ctx->sm_count, s));
    ++t.launches;
  }
  t.kernel_used = kernel;
  ctx->last_set = cs;
  if (!capturing) {                                       // toggle only once every launch of the call is enqueued
    ctx->set_clean[cs ^ 1] = (kernel == MMF_KERNEL_TC);   // zeroed by this call's tensor-core kernel
    ctx->counter_set = cs ^ 1;
  }
  return MMF_OK;
}

// Enqueue the fit for device-resident buffers: slab by slab, so that the per-row scratch (a 256-B record and a
// work-list entry per row for the series with gaps, gamma / c for the many-rows predict kernel) is proportional to a
// slab, not to the batch.  One slab for batches up to a million rows; beyond that the slab is sized so the scratch
// stays under ~5 % of the input (10 M x 365: 4 slabs, 0.7 GB instead of 2.6 GB).  Slabs run back to back on the
// stream; the scratch of slab i is free again when slab i+1 starts (stream order).
int64_t slab_rows(const Plan& plan, int64_t n) {
  int64_t slab = n;
  if (n > (int64_t)1 << 20) {
    const double input_bytes = (double)n * (double)plan.t_fit * 4.0;
    slab = std::max<int64_t>((int64_t)1 << 20, (int64_t)(0.05 * input_bytes / (double)(sizeof(SolveRec) + sizeof(int64_t))));
    slab = std::min(n, (slab + 127) & ~(int64_t)127);                 // whole 128-row tiles
    const int64_t n_slabs = (n + slab - 1) / slab;
    slab = (((n + n_slabs - 1) / n_slabs) + 127) & ~(int64_t)127;     // equal slabs
  }
  return slab;
}

// One fit a call runs in every slab, against `plan`.  Single-model calls have one stage; the (p, d) and (p, d, q)
// selections one per listed d.
struct Stage {
  const Plan* plan;
  Call call;
};

// The slabs are cut by `slab_plan` (the plan of the call's one stage, or a selection's level plan: the plain fit of the
// level rows would cut them so), and every slab runs each stage in turn.  slab_pending (nullable, one word per slab
// and stage): each fit's count of rows handed to the general pass is copied there before the next fit's tensor-core
// kernel zeroes the counter set it was kept in (0 for a fit by the warp kernel).
int run_device(mmf_ctx* ctx, const Plan& slab_plan, const std::vector<Stage>& stages, int64_t n, Tally& t,
               uint32_t* slab_pending = nullptr) {
  const cudaStream_t s = ctx->stream;
  const int64_t slab = slab_rows(slab_plan, n);
  // CSS and joint calls read the HR (phi, theta, ma_order) back: what the caller did not ask for goes to per-slab scratch;
  // Kalman-predictor calls with standard errors also read order and sigma back
  const Call& c0 = stages[0].call;
  const bool kf_se = c0.kf && c0.kf->se != nullptr;
  float* hr = nullptr;
  if (c0.css && (c0.ar->phi == nullptr || c0.arma->theta == nullptr || c0.arma->ma_order == nullptr ||
                 (kf_se && (c0.ar->order == nullptr || c0.ar->sigma == nullptr)))) {
    const size_t per_row = (MMF_AR_MAX + MMF_MA_MAX + 1 + (kf_se ? 2 : 0)) * sizeof(float);
    int rc = grow((void**)&ctx->d_css_hr, &ctx->css_hr_cap, (size_t)slab * per_row);
    if (rc != MMF_OK) return rc;
    hr = ctx->d_css_hr;
  }
  // selections with refit stages: the refit reads the winner back (phi, theta, order, ma_order, choice_d, choice_q), so
  // what the caller did not ask for goes to per-slab scratch in every stage; the row list and its length live there too.
  // The ML + Kalman refit with standard errors also reads sigma back (the se pass and arma_kf_list_kernel)
  int32_t* rs = nullptr;
  const bool sig_slot = stages.back().call.kf && stages.back().call.kf->se != nullptr && stages[0].call.ar->sigma == nullptr;
  if (stages.back().call.refit) {
    const size_t words = (size_t)slab * (MMF_AR_MAX + MMF_MA_MAX + 5 + (sig_slot ? 1 : 0)) + 1;
    int rc = grow((void**)&ctx->d_refit, &ctx->refit_cap, words * sizeof(int32_t));
    if (rc != MMF_OK) return rc;
    rs = ctx->d_refit;
  }
  for (int64_t off = 0, i = 0; off < n; off += slab, ++i) {
    const int64_t m = std::min(slab, n - off);
    for (size_t k = 0; k < stages.size(); ++k) {
      Call c = stages[k].call.slice(off);
      if (hr != nullptr) {
        if (!c.ar->phi) c.ar->phi = hr;
        if (!c.arma->theta) c.arma->theta = hr + (size_t)slab * MMF_AR_MAX;
        if (!c.arma->ma_order) c.arma->ma_order = reinterpret_cast<int32_t*>(hr + (size_t)slab * (MMF_AR_MAX + MMF_MA_MAX));
        if (kf_se && !c.ar->order)
          c.ar->order = reinterpret_cast<int32_t*>(hr + (size_t)slab * (MMF_AR_MAX + MMF_MA_MAX + 1));
        if (kf_se && !c.ar->sigma) c.ar->sigma = hr + (size_t)slab * (MMF_AR_MAX + MMF_MA_MAX + 2);
      }
      if (rs != nullptr) {
        auto or_scratch = [](auto*& p, int32_t* w) { if (!p) p = reinterpret_cast<decltype(p + 0)>(w); };
        int32_t* w = rs;
        int32_t* phi = w;       w += (size_t)slab * MMF_AR_MAX;
        int32_t* theta = w;     w += (size_t)slab * MMF_MA_MAX;
        int32_t* order = w;     w += slab;
        int32_t* ma_order = w;  w += slab;
        int32_t* choice_d = w;  w += slab;
        int32_t* choice_q = w;  w += slab;
        int32_t* rows = w;      w += slab;
        if (sig_slot) { or_scratch(c.ar->sigma, w); w += slab; }
        or_scratch(c.ar->phi, phi);
        or_scratch(c.ar->order, order);
        if (c.hsel) {
          or_scratch(c.hsel->theta, theta);
          or_scratch(c.hsel->ma_order, ma_order);
          or_scratch(c.hsel->choice_q, choice_q);
          or_scratch(c.asel->choice_d, choice_d);
        }
        if (c.refit) {
          or_scratch(c.arma->theta, theta);
          or_scratch(c.arma->ma_order, ma_order);
          or_scratch(c.refit->choice_d, choice_d);
          or_scratch(c.refit->choice_q, choice_q);
          c.refit->rows = rows;
          c.refit->count = reinterpret_cast<uint32_t*>(w);
        }
      }
      const int rc = run_device_slab(ctx, *stages[k].plan, c, m, t);
      if (rc != MMF_OK) return rc;
      if (slab_pending != nullptr) {
        uint32_t* dst = slab_pending + i * (int64_t)stages.size() + k;
        if (t.kernel_used == MMF_KERNEL_TC)
          CU_TRY(cudaMemcpyAsync(dst, ctx->d_pending + CTR_WORDS * ctx->last_set, sizeof(uint32_t),
                                 cudaMemcpyDeviceToDevice, s));
        else
          CU_TRY(cudaMemsetAsync(dst, 0, sizeof(uint32_t), s));
      }
    }
  }
  return MMF_OK;
}

// grow() for scratch no captured CUDA graph refers to: it may move while one is pinned
int grow_unpinned(void** ptr, size_t* cap, size_t need) {
  const mmf_ctx* saved = g_grow_ctx;
  g_grow_ctx = nullptr;
  const int rc = grow(ptr, cap, need);
  g_grow_ctx = saved;
  return rc;
}

// The status scratch is only referenced by a graph whose capture passed out_status == NULL; otherwise it may move.
int grow_status_scratch(mmf_ctx* ctx, int64_t n) {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(ctx->stream, &cap) == cudaSuccess && cap != cudaStreamCaptureStatusNone)
    ctx->status_scratch_captured = true;
  const size_t need = (size_t)n * sizeof(int32_t);
  return ctx->status_scratch_captured ? grow((void**)&ctx->d_status_scratch, &ctx->status_scratch_cap, need)
                                      : grow_unpinned((void**)&ctx->d_status_scratch, &ctx->status_scratch_cap, need);
}

// a call without a status buffer writes the context's status scratch (n words)
int status_or_scratch(mmf_ctx* ctx, int32_t** status, int64_t n) {
  if (*status != nullptr) return MMF_OK;
  const int rc = grow_status_scratch(ctx, n);
  if (rc == MMF_OK) *status = ctx->d_status_scratch;
  return rc;
}

// A call with stats times its kernels from here (before its first launch) to stats_tail.
int stats_begin(mmf_ctx* ctx, const mmf_stats* stats) {
  if (stats) CU_TRY(cudaEventRecord(ctx->ev_k0, ctx->stream));
  return MMF_OK;
}

// The stats of a call that ran stats_begin: waits for the stream, then the kernel time, the rows handed to the general
// pass (`pend`, plus the n_pend words at `pend_dev`, read once the stream is done) and the launch bookkeeping.  Nothing
// without stats.
int stats_tail(mmf_ctx* ctx, mmf_stats* stats, int64_t n, const Tally& t, const uint32_t* pend_dev = nullptr,
               size_t n_pend = 0, uint32_t pend = 0) {
  if (!stats) return MMF_OK;
  CU_TRY(cudaEventRecord(ctx->ev_k1, ctx->stream));
  CU_TRY(cudaEventSynchronize(ctx->ev_k1));
  CU_TRY(cudaEventElapsedTime(&stats->kernel_ms, ctx->ev_k0, ctx->ev_k1));
  stats->total_ms = stats->kernel_ms;
  std::vector<uint32_t> words(n_pend);
  if (n_pend > 0) CU_TRY(cudaMemcpy(words.data(), pend_dev, n_pend * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  stats->n_pending = pend;
  for (uint32_t v : words) stats->n_pending += v;
  stats->n_series = n;
  stats->kernel_launches = t.launches;
  stats->kernel_used = t.kernel_used;
  return MMF_OK;
}

// The device path of a fit call, its arguments checked (n > 0, device set): status or its scratch, the slab-pending
// scratch when stats need it, the enqueue of every slab, the stats.
int enqueue(mmf_ctx* ctx, const Plan& slab_plan, std::vector<Stage> stages, int64_t n, mmf_stats* stats) {
  for (Stage& st : stages)
    if (int rc = status_or_scratch(ctx, &st.call.status, n)) return rc;
  // Several fits: every fit's tensor-core kernel zeroes the counter set the fit before it used, so the pending count
  // of each is copied aside as it completes and summed at the end.  A call with stats synchronises and so is never
  // captured: this scratch is not part of any graph and may grow while one is pinned.
  const int64_t slab = slab_rows(slab_plan, n);
  const size_t n_fits = (size_t)((n + slab - 1) / slab) * stages.size();
  uint32_t* slab_pending = nullptr;
  if (stats && n_fits > 1) {
    if (int rc = grow_unpinned((void**)&ctx->d_slab_pending, &ctx->slab_pending_cap, n_fits * sizeof(uint32_t))) return rc;
    slab_pending = ctx->d_slab_pending;
  }
  Tally t;
  if (int rc = stats_begin(ctx, stats)) return rc;
  if (int rc = run_device(ctx, slab_plan, stages, n, t, slab_pending)) return rc;
  if (slab_pending != nullptr) return stats_tail(ctx, stats, n, t, slab_pending, n_fits);
  return stats_tail(ctx, stats, n, t, ctx->d_pending + CTR_WORDS * ctx->last_set, t.kernel_used == MMF_KERNEL_TC ? 1 : 0);
}

// ---- argument checks shared by the entry points
// the prediction rows [pred_start, pred_start + n_pred) inside the n_rows planned rows, and ld_out >= n_pred
int check_window(int32_t pred_start, int32_t n_pred, int32_t n_rows, int64_t ld_out) {
  if (n_pred < 1 || pred_start < 0 || (int64_t)pred_start + n_pred > n_rows)
    return fail(MMF_E_INVALID, "prediction rows [%d,%d) outside the planned design (%d rows)", pred_start,
                pred_start + n_pred, n_rows);
  if (ld_out < n_pred) return fail(MMF_E_INVALID, "ld_out=%lld < n_pred=%d", (long long)ld_out, n_pred);
  return MMF_OK;
}

// v[first .. count) ascending and distinct in [0, hi]
int check_ascending(const char* name, const int32_t* v, int32_t count, int32_t hi, int first = 0) {
  for (int j = first; j < count; ++j)
    if (v[j] < 0 || v[j] > hi || (j > 0 && v[j] <= v[j - 1]))
      return fail(MMF_E_INVALID, "%s must be ascending and distinct in [0,%d] (%s[%d]=%d)", name, hi, name, j, v[j]);
  return MMF_OK;
}

// every pointer of `need`, and every non-null pointer of `opt`, is device (or managed) memory
bool on_device(std::initializer_list<const void*> need, std::initializer_list<const void*> opt) {
  for (const void* p : need)
    if (!is_device_ptr(p)) return false;
  for (const void* p : opt)
    if (p && !is_device_ptr(p)) return false;
  return true;
}

// Hannan-Rissanen long AR order for long_order = 0: min(32, max(2 max(p, q), floor(ln(t_fit - d)^2))), where lmax is
// the largest p or q the call fits
int32_t hr_long_order(int32_t lmax, int32_t t_fit_d) {
  const double lt = std::log((double)t_fit_d);
  return std::min<int32_t>(MMF_HR_LONG_MAX, std::max<int32_t>(2 * lmax, (int32_t)std::floor(lt * lt)));
}

// the plain-fit fields of a call
Call plain_call(const float* y, int64_t ld_y, int32_t pred_start, int32_t n_pred, float* out, int64_t ld_out,
                int32_t* status) {
  Call c;
  c.y = y; c.ld_y = ld_y; c.pred_start = pred_start; c.n_pred = n_pred; c.out = out; c.ld_out = ld_out; c.status = status;
  return c;
}

ArArgs ar_args(int32_t p, float* phi, int32_t* order, float* sigma, const Plan& plan) {
  ArArgs ar{};
  ar.p = p; ar.phi = phi; ar.order = order; ar.sigma = sigma; ar.nz = plan.d_nz;
  return ar;
}

// the levels' row pitch and fit rows of an ARIMA call (its y is the slab's), d = 0 .. MMF_DIFF_MAX
ArimaArgs arima_args(int64_t ld_y, int32_t t_fit, int32_t d) {
  ArimaArgs ma{};
  ma.ld_y = ld_y; ma.t_fit = t_fit; ma.d = d;
  return ma;
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
  if ((e = cudaEventCreateWithFlags(&ctx->ev_switch, cudaEventDisableTiming)) != cudaSuccess) return bail(e, "cudaEventCreate");
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
  free_bt(ctx->bt);
  free_arima(ctx->arima);
  cudaFree(ctx->d_z);
  cudaFree(ctx->d_asel_best); cudaFree(ctx->d_asel_status); cudaFree(ctx->d_hsel_q0); cudaFree(ctx->d_css_hr);
  cudaFree(ctx->d_refit);
  cudaFree(ctx->d_bt_mom); cudaFree(ctx->d_bt_recs); cudaFree(ctx->d_bt_rows); cudaFree(ctx->d_bt_ctr); cudaFree(ctx->d_bt_pred);
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
  cudaFree(ctx->d_slab_pending);
  cudaFree(ctx->d_recs);
  cudaFree(ctx->d_rec_rows);
  cudaFree(ctx->d_gamma);
  cudaFree(ctx->d_c);
  cudaFree(ctx->d_sigma_scratch);
  cudaFree(ctx->d_status_scratch);
  cudaFree(ctx->d_pack_scratch);
  if (ctx->ev_a) cudaEventDestroy(ctx->ev_a);
  if (ctx->ev_b) cudaEventDestroy(ctx->ev_b);
  if (ctx->ev_k0) cudaEventDestroy(ctx->ev_k0);
  if (ctx->ev_k1) cudaEventDestroy(ctx->ev_k1);
  if (ctx->ev_switch) cudaEventDestroy(ctx->ev_switch);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->s_h2d) cudaStreamDestroy(ctx->s_h2d);
  if (ctx->s_d2h) cudaStreamDestroy(ctx->s_d2h);
  delete ctx;
  return MMF_OK;
}

int mmf_set_stream(mmf_ctx* ctx, void* cuda_stream) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  cudaStream_t next = (cudaStream_t)cuda_stream;  // NULL = legacy default stream
  if (next == ctx->stream) return MMF_OK;         // the common case: nothing to order
  if (ctx->own_stream && ctx->stream) {
    cudaStreamSynchronize(ctx->stream);
    cudaStreamDestroy(ctx->stream);
  } else {
    // Every call shares the context's counter sets and scratch, and the host's record of which counter set is zero
    // assumes the calls run in the order they were made: the new stream waits for the work enqueued on the old one.
    // Not when either stream is capturing: an event recorded in a capture cannot order work outside it, and
    // torch.cuda.graph synchronises the device before a capture begins.  The new stream is asked first: querying the
    // legacy stream during a global-mode capture would invalidate that capture.
    CU_TRY(cudaSetDevice(ctx->device));
    cudaStreamCaptureStatus cap_next = cudaStreamCaptureStatusNone, cap_prev = cudaStreamCaptureStatusNone;
    CU_TRY(cudaStreamIsCapturing(next, &cap_next));
    if (cap_next == cudaStreamCaptureStatusNone) {
      CU_TRY(cudaStreamIsCapturing(ctx->stream, &cap_prev));
      if (cap_prev == cudaStreamCaptureStatusNone) {
        CU_TRY(cudaEventRecord(ctx->ev_switch, ctx->stream));
        CU_TRY(cudaStreamWaitEvent(next, ctx->ev_switch, 0));
      }
    }
  }
  ctx->stream = next;
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
  const int rc = build_plan(ctx->plan, X, n_rows, p, t_fit, has_constant);
  if (rc == MMF_OK) {
    ctx->plan.x_cols = p;
    ctx->plan.x_hash = hash_x(X, (int64_t)n_rows * p);
  }
  return rc;
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
  if (int rc = check_window(pred_start, n_pred, pl.n_rows, ld_out)) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));

  const bool y_dev = is_device_ptr(y), o_dev = is_device_ptr(out_pred);
  const bool b_dev = out_beta ? is_device_ptr(out_beta) : true;
  const bool s_dev = out_status ? is_device_ptr(out_status) : true;
  Call c = plain_call(y, ld_y, pred_start, n_pred, out_pred, ld_out, out_status);
  c.beta = out_beta;
  if (!is_int && y_dev && o_dev && b_dev && s_dev) {
    // ------------------------------------------------ all device: just enqueue
    return enqueue(ctx, pl, {{&pl, c}}, n, stats);
  } else {
    // ------------------------------------------------ host buffers (or an integer series buffer): pipelined chunks
    Tally t;
    int64_t h2d = 0, d2h = 0;
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
    for (int i = 0; i < NBUF; ++i) {                           // staging slots are never part of a captured graph
      Staging& s = ctx->st[i];
      int rc = MMF_OK;
      if (!y_dev || is_int) rc = grow_unpinned((void**)&s.d_y, &s.y_cap, (size_t)chunk * pitch * sizeof(float));
      if (rc == MMF_OK && (is_int || narrow) && !y_dev)
        rc = grow_unpinned(&s.d_yraw, &s.yraw_cap, narrow ? (size_t)chunk * npitch * 2 : (size_t)chunk * rpitch * esize);
      if (rc == MMF_OK && !o_dev) rc = grow_unpinned((void**)&s.d_out, &s.out_cap, (size_t)chunk * opitch * sizeof(float));
      if (rc == MMF_OK && out_beta && !b_dev)
        rc = grow_unpinned((void**)&s.d_beta, &s.beta_cap, (size_t)chunk * P * sizeof(float));
      if (rc == MMF_OK && (!out_status || !s_dev))
        rc = grow_unpinned((void**)&s.d_status, &s.status_cap, (size_t)chunk * sizeof(int32_t));
      if (rc != MMF_OK) return rc;
    }
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
        ++t.launches;
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
        ++t.launches;
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
      c.y = yk; c.ld_y = ldk;
      c.out = o_dev ? out_pred + off * ld_out : s.d_out;
      c.ld_out = o_dev ? ld_out : opitch;
      c.beta = out_beta ? (b_dev ? out_beta + off * P : s.d_beta) : nullptr;
      c.status = (out_status && s_dev) ? out_status + off : s.d_status;
      if (it >= NBUF) CU_TRY(cudaStreamWaitEvent(ctx->stream, s.ev_d2h, 0));        // output staging drained
      if (int rc = run_device(ctx, pl, {{&pl, c}}, m, t)) return rc;
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
      stats->n_series = n;
      stats->h2d_bytes = h2d;
      stats->d2h_bytes = d2h;
      stats->kernel_launches = t.launches;
      stats->kernel_used = t.kernel_used;
    }
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

int mmf_fit_forecast_se_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t pred_start, int32_t n_pred,
                            float* out_pred, int64_t ld_out, float* out_se, int64_t ld_se, float* out_sigma,
                            int32_t* out_dof, int32_t* out_status, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  if (!ctx->plan.valid) return fail(MMF_E_NOPLAN, "mmf_plan_design has not been called");
  const Plan& pl = ctx->plan;
  if (n < 0) return fail(MMF_E_INVALID, "n < 0");
  if (n > 0 && (!y || !out_pred)) return fail(MMF_E_INVALID, "y or out_pred is NULL");
  if (!out_se && !out_sigma && !out_dof)
    return fail(MMF_E_INVALID, "out_se, out_sigma and out_dof are all NULL: use mmf_fit_forecast_f32");
  if (ld_y < pl.t_fit) return fail(MMF_E_INVALID, "ld_y=%lld < t_fit=%d", (long long)ld_y, pl.t_fit);
  if (int rc = check_window(pred_start, n_pred, pl.n_rows, ld_out)) return rc;
  if (out_se && ld_se < n_pred) return fail(MMF_E_INVALID, "ld_se=%lld < n_pred=%d", (long long)ld_se, n_pred);
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));
  if (!on_device({y, out_pred}, {out_se, out_sigma, out_dof, out_status}))
    return fail(MMF_E_UNSUPPORTED, "mmf_fit_forecast_se_f32 takes device buffers only");
  Call c = plain_call(y, ld_y, pred_start, n_pred, out_pred, ld_out, out_status);
  if (int rc = status_or_scratch(ctx, &c.status, n)) return rc;
  SeArgs se{};
  se.out_se = out_se; se.ld_se = ld_se; se.sigma = out_sigma; se.dof = out_dof; se.sfac = pl.d_sfac;
  if (!se.sigma) {
    int rc = grow((void**)&ctx->d_sigma_scratch, &ctx->sigma_scratch_cap, (size_t)n * sizeof(float));
    if (rc != MMF_OK) return rc;
    se.sigma = ctx->d_sigma_scratch;
  }
  c.se = se;
  return enqueue(ctx, pl, {{&pl, c}}, n, stats);
}

int mmf_fit_forecast_ar_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order, int32_t pred_start,
                            int32_t n_pred, float* out_pred, int64_t ld_out, float* out_phi, int32_t* out_order,
                            float* out_sigma, int32_t* out_status, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  if (!ctx->plan.valid) return fail(MMF_E_NOPLAN, "mmf_plan_design has not been called");
  const Plan& pl = ctx->plan;
  if (n < 0) return fail(MMF_E_INVALID, "n < 0");
  if (n > 0 && (!y || !out_pred)) return fail(MMF_E_INVALID, "y or out_pred is NULL");
  if (ar_order < 1 || ar_order > MMF_AR_MAX) return fail(MMF_E_INVALID, "ar_order=%d outside [1,%d]", ar_order, MMF_AR_MAX);
  if (ld_y < pl.t_fit) return fail(MMF_E_INVALID, "ld_y=%lld < t_fit=%d", (long long)ld_y, pl.t_fit);
  if (int rc = check_window(pred_start, n_pred, pl.n_rows, ld_out)) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));
  if (!on_device({y, out_pred}, {out_phi, out_order, out_sigma, out_status}))
    return fail(MMF_E_UNSUPPORTED, "mmf_fit_forecast_ar_f32 takes device buffers only");
  Call c = plain_call(y, ld_y, pred_start, n_pred, out_pred, ld_out, out_status);
  c.ar = ar_args(ar_order, out_phi, out_order, out_sigma, pl);
  return enqueue(ctx, pl, {{&pl, c}}, n, stats);
}

int mmf_fit_select_ar_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                          const int32_t* orders, int32_t n_orders, int32_t pred_start, int32_t n_pred,
                          float* out_pred, int64_t ld_out, int32_t* out_choice, float* out_mse, float* out_cand_mse,
                          float* out_phi, int32_t* out_order, float* out_sigma, int32_t* out_status, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  if (!ctx->plan.valid) return fail(MMF_E_NOPLAN, "mmf_plan_design has not been called");
  const Plan& pl = ctx->plan;
  if (n < 0) return fail(MMF_E_INVALID, "n < 0");
  if (n > 0 && (!y || !out_pred)) return fail(MMF_E_INVALID, "y or out_pred is NULL");
  if (!orders || n_orders < 1 || n_orders > MMF_ARSEL_MAX_CAND)
    return fail(MMF_E_INVALID, "n_orders=%d outside [1,%d] (or orders is NULL)", n_orders, MMF_ARSEL_MAX_CAND);
  if (int rc = check_ascending("orders", orders, n_orders, MMF_AR_MAX)) return rc;
  if (n_hold < 1 || (int64_t)pl.t_fit + n_hold > pl.n_rows)
    return fail(MMF_E_INVALID, "held-out rows [%d,%lld) outside the planned design (%d rows)", pl.t_fit,
                (long long)pl.t_fit + n_hold, pl.n_rows);
  if (ld_y < (int64_t)pl.t_fit + n_hold)
    return fail(MMF_E_INVALID, "ld_y=%lld < t_fit + n_hold=%lld", (long long)ld_y, (long long)pl.t_fit + n_hold);
  if (int rc = check_window(pred_start, n_pred, pl.n_rows, ld_out)) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));
  if (!on_device({y, out_pred}, {out_choice, out_mse, out_cand_mse, out_phi, out_order, out_sigma, out_status}))
    return fail(MMF_E_UNSUPPORTED, "mmf_fit_select_ar_f32 takes device buffers only");
  Call c = plain_call(y, ld_y, pred_start, n_pred, out_pred, ld_out, out_status);
  c.ar = ar_args(orders[n_orders - 1], out_phi, out_order, out_sigma, pl);
  ArSelArgs sel{};
  sel.n_hold = n_hold; sel.n_cand = n_orders;
  for (int j = 0; j < n_orders; ++j) sel.cand[j] = orders[j];
  sel.choice = out_choice; sel.mse = out_mse; sel.cand_mse = out_cand_mse;
  c.arsel = sel;
  return enqueue(ctx, pl, {{&pl, c}}, n, stats);
}

// ---- regression with ARIMA(p, d, 0) errors (DESIGN.md section 2 item 11) ------------------------------------------
int mmf_plan_arima(mmf_ctx* ctx, const double* X, int32_t n_rows, int32_t p, int32_t t_fit, int32_t max_diff) {
  if (!ctx || !X) return fail(MMF_E_INVALID, "ctx or X is NULL");
  if (p < 1 || p > P) return fail(MMF_E_INVALID, "p=%d outside [1,%d]", p, P);
  if (max_diff < 1 || max_diff > MMF_DIFF_MAX)
    return fail(MMF_E_INVALID, "max_diff=%d outside [1,%d]", max_diff, MMF_DIFF_MAX);
  if (t_fit - max_diff < 1 || n_rows < t_fit)
    return fail(MMF_E_INVALID, "need 1 <= t_fit - max_diff and t_fit <= n_rows (t_fit=%d n_rows=%d max_diff=%d)", t_fit,
                n_rows, max_diff);
  for (int64_t i = 0; i < (int64_t)n_rows * p; ++i)
    if (!std::isfinite(X[i])) return fail(MMF_E_INVALID, "design matrix has a non-finite entry at %lld", (long long)i);
  // every argument check comes before the previous ARIMA plan is freed (the mmf_plan_calendars rule).
  // D_d row s = Delta^d x_{s+d} in float64.  A column whose differences on the fit rows are cancellation residue of the
  // raw column (largest |value| <= 1e-12 x the raw column's there) is zeroed, so the whitening drops it instead of
  // scaling rounding noise up to unit norm (Delta^2 of a linear trend).
  std::vector<double> raw_max(p, 0.0);
  for (int32_t t = 0; t < t_fit; ++t)
    for (int j = 0; j < p; ++j) raw_max[j] = std::max(raw_max[j], std::fabs(X[(int64_t)t * p + j]));
  std::vector<std::vector<double>> D(max_diff);
  for (int d = 1; d <= max_diff; ++d) {
    const double* prev = d == 1 ? X : D[d - 2].data();
    std::vector<double>& Dd = D[d - 1];
    Dd.resize((size_t)(n_rows - d) * p);
    for (int32_t s = 0; s < n_rows - d; ++s)
      for (int j = 0; j < p; ++j) Dd[(size_t)s * p + j] = prev[(size_t)(s + 1) * p + j] - prev[(size_t)s * p + j];
  }
  for (int d = 1; d <= max_diff; ++d) {
    std::vector<double>& Dd = D[d - 1];
    for (int j = 0; j < p; ++j) {
      double mx = 0.0;
      for (int32_t s = 0; s < t_fit - d; ++s) mx = std::max(mx, std::fabs(Dd[(size_t)s * p + j]));
      if (mx <= 1e-12 * raw_max[j])
        for (int32_t s = 0; s < n_rows - d; ++s) Dd[(size_t)s * p + j] = 0.0;
    }
  }
  CU_TRY(cudaSetDevice(ctx->device));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  free_arima(ctx->arima);
  for (int d = 1; d <= max_diff; ++d) {
    const int rc = build_plan(ctx->arima.diff[d - 1], D[d - 1].data(), n_rows - d, p, t_fit - d, 0);
    if (rc != MMF_OK) { free_arima(ctx->arima); return rc; }
  }
  ctx->arima.max_diff = max_diff;
  ctx->arima.n_rows = n_rows;
  ctx->arima.t_fit = t_fit;
  ctx->arima.x_cols = p;
  ctx->arima.x_hash = hash_x(X, (int64_t)n_rows * p);
  ctx->arima.valid = true;
  return MMF_OK;
}

int mmf_fit_forecast_arima_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                               int32_t diff_order, int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                               float* out_phi, int32_t* out_order, float* out_sigma, int32_t* out_status,
                               mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  if (!ctx->arima.valid) return fail(MMF_E_NOPLAN, "mmf_plan_arima has not been called");
  const ArimaPlan& ap = ctx->arima;
  if (n < 0) return fail(MMF_E_INVALID, "n < 0");
  if (n > 0 && (!y || !out_pred)) return fail(MMF_E_INVALID, "y or out_pred is NULL");
  if (ar_order < 0 || ar_order > MMF_AR_MAX) return fail(MMF_E_INVALID, "ar_order=%d outside [0,%d]", ar_order, MMF_AR_MAX);
  if (diff_order < 1 || diff_order > ap.max_diff)
    return fail(MMF_E_INVALID, "diff_order=%d outside [1,%d] (the planned max_diff)", diff_order, ap.max_diff);
  if (ld_y < ap.t_fit) return fail(MMF_E_INVALID, "ld_y=%lld < t_fit=%d", (long long)ld_y, ap.t_fit);
  if (int rc = check_window(pred_start, n_pred, ap.n_rows, ld_out)) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));
  if (!on_device({y, out_pred}, {out_phi, out_order, out_sigma, out_status}))
    return fail(MMF_E_UNSUPPORTED, "mmf_fit_forecast_arima_f32 takes device buffers only");
  const Plan& pl = ap.diff[diff_order - 1];
  Call c = plain_call(y, ld_y, pred_start, n_pred, out_pred, ld_out, out_status);
  c.ar = ar_args(ar_order, out_phi, out_order, out_sigma, pl);
  c.arima = arima_args(ld_y, ap.t_fit, diff_order);
  return enqueue(ctx, pl, {{&pl, c}}, n, stats);
}

// ---- regression with ARIMA(p, d, q) errors (DESIGN.md section 2 items 13, 16, 17) ----------------------------------------
// The HR call (css == nullptr), the CSS call, the joint call (joint != nullptr, with css) and the ML call (ml != nullptr,
// with css): the same checks, plans and launches; the CSS call adds arma_css_kernel behind arma_kernel in every slab, the
// joint call arma_joint_kernel, the ML call arma_ml_kernel behind arma_css_kernel.
static int arma_call(mmf_ctx* ctx, const char* name, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                     int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t pred_start, int32_t n_pred,
                     float* out_pred, int64_t ld_out, float* out_phi, float* out_theta, int32_t* out_order,
                     int32_t* out_ma_order, float* out_sigma, int32_t* out_status, mmf_stats* stats,
                     const CssArgs* css, const JointArgs* joint = nullptr, const MlArgs* ml = nullptr,
                     const KfArgs* kf = nullptr) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  if (n < 0) return fail(MMF_E_INVALID, "n < 0");
  if (n > 0 && (!y || !out_pred)) return fail(MMF_E_INVALID, "y or out_pred is NULL");
  if (ar_order < 0 || ar_order > MMF_AR_MAX) return fail(MMF_E_INVALID, "ar_order=%d outside [0,%d]", ar_order, MMF_AR_MAX);
  if (ma_order < 1 || ma_order > MMF_MA_MAX) return fail(MMF_E_INVALID, "ma_order=%d outside [1,%d]", ma_order, MMF_MA_MAX);
  if (diff_order < 0 || diff_order > MMF_DIFF_MAX)
    return fail(MMF_E_INVALID, "diff_order=%d outside [0,%d]", diff_order, MMF_DIFF_MAX);
  // d = 0 models y with the mmf_plan_design plan; d >= 1 models z' with the mmf_plan_arima plan
  const ArimaPlan& ap = ctx->arima;
  if (diff_order == 0 && !ctx->plan.valid) return fail(MMF_E_NOPLAN, "mmf_plan_design has not been called");
  if (diff_order >= 1 && !ap.valid) return fail(MMF_E_NOPLAN, "mmf_plan_arima has not been called");
  if (diff_order > (diff_order == 0 ? 0 : ap.max_diff))
    return fail(MMF_E_INVALID, "diff_order=%d above the planned max_diff=%d", diff_order, ap.max_diff);
  const Plan& pl = diff_order == 0 ? ctx->plan : ap.diff[diff_order - 1];
  const int32_t T = diff_order == 0 ? pl.t_fit : ap.t_fit;          // level fit rows
  const int32_t n_rows = diff_order == 0 ? pl.n_rows : ap.n_rows;
  const int32_t lmin = std::max(ar_order, ma_order);
  if (long_order != 0 && (long_order < lmin || long_order > MMF_HR_LONG_MAX))
    return fail(MMF_E_INVALID, "long_order=%d outside {0} and [%d,%d]", long_order, lmin, MMF_HR_LONG_MAX);
  if (ld_y < T) return fail(MMF_E_INVALID, "ld_y=%lld < t_fit=%d", (long long)ld_y, T);
  if (int rc = check_window(pred_start, n_pred, n_rows, ld_out)) return rc;
  if (kf && kf->se && kf->ld_se < n_pred)
    return fail(MMF_E_INVALID, "ld_se=%lld < n_pred=%d", (long long)kf->ld_se, n_pred);
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));
  if (!on_device({y, out_pred}, {out_phi, out_theta, out_order, out_ma_order, out_sigma, out_status,
                                 css ? css->css_start : nullptr, css ? css->css : nullptr, css ? css->css_stop : nullptr,
                                 css ? css->iters : nullptr, joint ? joint->beta : nullptr,
                                 ml ? ml->loglik_start : nullptr, ml ? ml->loglik : nullptr, ml ? ml->stop : nullptr,
                                 ml ? ml->iters : nullptr, kf ? kf->se : nullptr}))
    return fail(MMF_E_UNSUPPORTED, "%s takes device buffers only", name);
  Call c = plain_call(y, ld_y, pred_start, n_pred, out_pred, ld_out, out_status);
  c.ar = ar_args(ar_order, out_phi, out_order, out_sigma, pl);
  ArmaArgs hr{};
  hr.q = ma_order;
  hr.m = long_order != 0 ? long_order : hr_long_order(lmin, T - diff_order);
  hr.theta = out_theta; hr.ma_order = out_ma_order;
  c.arma = hr;
  if (diff_order > 0) c.arima = arima_args(ld_y, ap.t_fit, diff_order);
  if (css) c.css = *css;
  if (joint) c.joint = *joint;
  if (ml) c.ml = *ml;
  if (kf) c.kf = *kf;
  return enqueue(ctx, pl, {{&pl, c}}, n, stats);
}

int mmf_fit_forecast_arma_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                              int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t pred_start,
                              int32_t n_pred, float* out_pred, int64_t ld_out, float* out_phi, float* out_theta,
                              int32_t* out_order, int32_t* out_ma_order, float* out_sigma, int32_t* out_status,
                              mmf_stats* stats) {
  return arma_call(ctx, "mmf_fit_forecast_arma_f32", y, n, ld_y, ar_order, diff_order, ma_order, long_order, pred_start,
                   n_pred, out_pred, ld_out, out_phi, out_theta, out_order, out_ma_order, out_sigma, out_status, stats,
                   nullptr);
}

int mmf_fit_forecast_arma_css_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                                  int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t max_iter,
                                  int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out, float* out_phi,
                                  float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                                  int32_t* out_status, float* out_css_start, float* out_css, int32_t* out_css_stop,
                                  int32_t* out_iters, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (max_iter < 0 || max_iter > MMF_CSS_ITER_MAX)
    return fail(MMF_E_INVALID, "max_iter=%d outside [0,%d]", max_iter, MMF_CSS_ITER_MAX);
  CssArgs css{};
  css.max_iter = max_iter == 0 ? MMF_CSS_ITER_DEFAULT : max_iter;
  css.css_start = out_css_start; css.css = out_css; css.css_stop = out_css_stop; css.iters = out_iters;
  return arma_call(ctx, "mmf_fit_forecast_arma_css_f32", y, n, ld_y, ar_order, diff_order, ma_order, long_order,
                   pred_start, n_pred, out_pred, ld_out, out_phi, out_theta, out_order, out_ma_order, out_sigma,
                   out_status, stats, &css);
}

int mmf_fit_forecast_arma_joint_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                                    int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t max_iter,
                                    int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out, float* out_beta,
                                    float* out_phi, float* out_theta, int32_t* out_order, int32_t* out_ma_order,
                                    float* out_sigma, int32_t* out_status, float* out_css_start, float* out_css,
                                    int32_t* out_css_stop, int32_t* out_iters, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (max_iter < 0 || max_iter > MMF_CSS_ITER_MAX)
    return fail(MMF_E_INVALID, "max_iter=%d outside [0,%d]", max_iter, MMF_CSS_ITER_MAX);
  CssArgs css{};
  css.max_iter = max_iter == 0 ? MMF_CSS_ITER_DEFAULT : max_iter;
  css.css_start = out_css_start; css.css = out_css; css.css_stop = out_css_stop; css.iters = out_iters;
  JointArgs joint{};
  joint.beta = out_beta;
  return arma_call(ctx, "mmf_fit_forecast_arma_joint_f32", y, n, ld_y, ar_order, diff_order, ma_order, long_order,
                   pred_start, n_pred, out_pred, ld_out, out_phi, out_theta, out_order, out_ma_order, out_sigma,
                   out_status, stats, &css, &joint);
}

int mmf_fit_forecast_arma_ml_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                                 int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t max_iter,
                                 int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out, float* out_phi,
                                 float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                                 int32_t* out_status, float* out_loglik_start, float* out_loglik, int32_t* out_ml_stop,
                                 int32_t* out_iters, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (max_iter < 0 || max_iter > MMF_CSS_ITER_MAX)
    return fail(MMF_E_INVALID, "max_iter=%d outside [0,%d]", max_iter, MMF_CSS_ITER_MAX);
  CssArgs css{};                           // the CSS call's start, its own columns unwritten
  css.max_iter = max_iter == 0 ? MMF_CSS_ITER_DEFAULT : max_iter;
  MlArgs ml{};
  ml.max_iter = css.max_iter;
  ml.loglik_start = out_loglik_start; ml.loglik = out_loglik; ml.stop = out_ml_stop; ml.iters = out_iters;
  return arma_call(ctx, "mmf_fit_forecast_arma_ml_f32", y, n, ld_y, ar_order, diff_order, ma_order, long_order,
                   pred_start, n_pred, out_pred, ld_out, out_phi, out_theta, out_order, out_ma_order, out_sigma,
                   out_status, stats, &css, nullptr, &ml);
}

int mmf_fit_forecast_arma_ml_kf_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                                    int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t max_iter,
                                    int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out, float* out_phi,
                                    float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                                    int32_t* out_status, float* out_loglik_start, float* out_loglik,
                                    int32_t* out_ml_stop, int32_t* out_iters, float* out_se, int64_t ld_se,
                                    mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (max_iter < 0 || max_iter > MMF_CSS_ITER_MAX)
    return fail(MMF_E_INVALID, "max_iter=%d outside [0,%d]", max_iter, MMF_CSS_ITER_MAX);
  CssArgs css{};                           // the ML call's stages, then the predictor
  css.max_iter = max_iter == 0 ? MMF_CSS_ITER_DEFAULT : max_iter;
  MlArgs ml{};
  ml.max_iter = css.max_iter;
  ml.loglik_start = out_loglik_start; ml.loglik = out_loglik; ml.stop = out_ml_stop; ml.iters = out_iters;
  KfArgs kf{};
  kf.se = out_se; kf.ld_se = ld_se;
  return arma_call(ctx, "mmf_fit_forecast_arma_ml_kf_f32", y, n, ld_y, ar_order, diff_order, ma_order, long_order,
                   pred_start, n_pred, out_pred, ld_out, out_phi, out_theta, out_order, out_ma_order, out_sigma,
                   out_status, stats, &css, nullptr, &ml, &kf);
}

// ---- standard errors of the ARIMA-family forecasts (DESIGN.md section 2 item 15) ---------------------------------------
int mmf_arima_se_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t t_fit, int32_t diff_order,
                     const int32_t* diffs, const float* phi, const int32_t* order, const float* theta,
                     const int32_t* ma_order, const float* sigma, int32_t pred_start, int32_t n_pred, float* out_se,
                     int64_t ld_se, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  if (n < 0) return fail(MMF_E_INVALID, "n < 0");
  if (n > 0 && (!y || !phi || !order || !sigma || !out_se))
    return fail(MMF_E_INVALID, "y, phi, order, sigma or out_se is NULL");
  if ((theta == nullptr) != (ma_order == nullptr))
    return fail(MMF_E_INVALID, "theta and ma_order must both be given or both be NULL");
  if (!diffs && (diff_order < 0 || diff_order > MMF_DIFF_MAX))
    return fail(MMF_E_INVALID, "diff_order=%d outside [0,%d]", diff_order, MMF_DIFF_MAX);
  if (t_fit < 1) return fail(MMF_E_INVALID, "t_fit=%d < 1", t_fit);
  if (ld_y < t_fit) return fail(MMF_E_INVALID, "ld_y=%lld < t_fit=%d", (long long)ld_y, t_fit);
  if (n_pred < 1 || pred_start < 0 || (int64_t)pred_start + n_pred > INT32_MAX)
    return fail(MMF_E_INVALID, "prediction rows [%d,%lld) outside [0,%d]", pred_start,
                (long long)pred_start + n_pred, INT32_MAX);
  if (ld_se < n_pred) return fail(MMF_E_INVALID, "ld_se=%lld < n_pred=%d", (long long)ld_se, n_pred);
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));
  if (!on_device({y, phi, order, sigma, out_se}, {diffs, theta, ma_order}))
    return fail(MMF_E_UNSUPPORTED, "mmf_arima_se_f32 takes device buffers only");
  ArimaSeArgs a{};
  a.y = y; a.ld_y = ld_y; a.t_fit = t_fit; a.diff_order = diff_order; a.diffs = diffs;
  a.phi = phi; a.order = order; a.theta = theta; a.ma_order = ma_order; a.sigma = sigma;
  a.pred_start = pred_start; a.n_pred = n_pred; a.out = out_se; a.ld_se = ld_se; a.n = n;
  if (int rc = stats_begin(ctx, stats)) return rc;
  CU_TRY(launch_arima_se(a, ctx->sm_count, ctx->stream));
  return stats_tail(ctx, stats, n, Tally{1, MMF_KERNEL_WARP});
}

// ---- (p, d) and (p, d, q) selection by hold-out MSE on levels (DESIGN.md section 2 items 12, 14, 18, 21) ----------------
// The MA arguments (mas .. out_ma_order) are those of mmf_fit_select_arma_f32 (with_q); mmf_fit_select_arima_f32 passes
// none and launches no arma_select_kernel.  The refit calls (css, with_q; joint with css; ml with css, kf with ml) add one
// refit stage per listed d behind the selection's stages.  The ML + Kalman call with standard errors (kf->se) cannot run
// the predictor inside those stages: the se pass must see every d's ML refit first, and arma_kf_list_kernel then
// overwrites the rows it covers.  So the last refit stage runs the se pass (per-series d), and one Kalman stage per listed
// d follows (that d's fit again, its list, arma_kf_list_kernel).  Without se the predictor runs in the refit stage.
static int select_arima_call(mmf_ctx* ctx, const char* name, bool with_q, const float* y, int64_t n, int64_t ld_y,
                             int32_t n_hold, const int32_t* orders, int32_t n_orders, const int32_t* diffs,
                             int32_t n_diffs, const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t pred_start,
                             int32_t n_pred, float* out_pred, int64_t ld_out, int32_t* out_choice_p,
                             int32_t* out_choice_d, int32_t* out_choice_q, float* out_mse, float* out_cand_mse,
                             float* out_phi, float* out_theta, int32_t* out_order, int32_t* out_ma_order,
                             float* out_sigma, int32_t* out_status, mmf_stats* stats, const CssArgs* css = nullptr,
                             const JointArgs* joint = nullptr, const MlArgs* ml = nullptr, const KfArgs* kf = nullptr) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  if (n < 0) return fail(MMF_E_INVALID, "n < 0");
  if (n > 0 && (!y || !out_pred)) return fail(MMF_E_INVALID, "y or out_pred is NULL");
  if (!orders || n_orders < 1 || n_orders > MMF_ARSEL_MAX_CAND)
    return fail(MMF_E_INVALID, "n_orders=%d outside [1,%d] (or orders is NULL)", n_orders, MMF_ARSEL_MAX_CAND);
  if (int rc = check_ascending("orders", orders, n_orders, MMF_AR_MAX)) return rc;
  if (!diffs || n_diffs < 1 || n_diffs > MMF_DIFF_MAX + 1)
    return fail(MMF_E_INVALID, "n_diffs=%d outside [1,%d] (or diffs is NULL)", n_diffs, MMF_DIFF_MAX + 1);
  if (int rc = check_ascending("diffs", diffs, n_diffs, MMF_DIFF_MAX)) return rc;
  if (with_q) {
    if (!mas || n_mas < 1 || n_mas > MMF_MA_MAX + 1)
      return fail(MMF_E_INVALID, "n_mas=%d outside [1,%d] (or mas is NULL)", n_mas, MMF_MA_MAX + 1);
    if (mas[0] != 0) return fail(MMF_E_INVALID, "mas[0]=%d: the MA orders must start with 0", mas[0]);
    if (int rc = check_ascending("mas", mas, n_mas, MMF_MA_MAX, 1)) return rc;
    if (n_orders * (n_mas - 1) > MMF_ARMASEL_MAX_PQ)
      return fail(MMF_E_INVALID, "%d x %d (p, q >= 1) pairs above MMF_ARMASEL_MAX_PQ=%d", n_orders, n_mas - 1,
                  MMF_ARMASEL_MAX_PQ);
    const int32_t lmin = std::max(orders[n_orders - 1], mas[n_mas - 1]);
    if (long_order != 0 && (long_order < lmin || long_order > MMF_HR_LONG_MAX))
      return fail(MMF_E_INVALID, "long_order=%d outside {0} and [%d,%d]", long_order, lmin, MMF_HR_LONG_MAX);
  }
  // a listed d = 0 fits y with the mmf_plan_design plan; a listed d >= 1 fits z' with the mmf_plan_arima plan
  const bool use_plain = diffs[0] == 0, use_arima = diffs[n_diffs - 1] >= 1;
  const Plan& pl = ctx->plan;
  const ArimaPlan& ap = ctx->arima;
  if (use_plain && !pl.valid) return fail(MMF_E_NOPLAN, "diffs lists 0 and mmf_plan_design has not been called");
  if (use_arima && !ap.valid) return fail(MMF_E_NOPLAN, "diffs lists d >= 1 and mmf_plan_arima has not been called");
  if (use_arima && diffs[n_diffs - 1] > ap.max_diff)
    return fail(MMF_E_INVALID, "diffs lists d=%d above the planned max_diff=%d", diffs[n_diffs - 1], ap.max_diff);
  if (use_plain && use_arima &&
      (pl.n_rows != ap.n_rows || pl.t_fit != ap.t_fit || pl.x_cols != ap.x_cols || pl.x_hash != ap.x_hash))
    return fail(MMF_E_INVALID, "the mmf_plan_design and mmf_plan_arima plans were built from different designs "
                "(rows %d / %d, t_fit %d / %d, columns %d / %d)", pl.n_rows, ap.n_rows, pl.t_fit, ap.t_fit, pl.x_cols,
                ap.x_cols);
  const int32_t T = use_plain ? pl.t_fit : ap.t_fit;
  const int32_t n_rows = use_plain ? pl.n_rows : ap.n_rows;
  if (n_hold < 1 || (int64_t)T + n_hold > n_rows)
    return fail(MMF_E_INVALID, "held-out rows [%d,%lld) outside the planned design (%d rows)", T, (long long)T + n_hold,
                n_rows);
  if (ld_y < (int64_t)T + n_hold)
    return fail(MMF_E_INVALID, "ld_y=%lld < t_fit + n_hold=%lld", (long long)ld_y, (long long)T + n_hold);
  if (int rc = check_window(pred_start, n_pred, n_rows, ld_out)) return rc;
  if (kf && kf->se && kf->ld_se < n_pred)
    return fail(MMF_E_INVALID, "ld_se=%lld < n_pred=%d", (long long)kf->ld_se, n_pred);
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));
  if (!on_device({y, out_pred}, {out_choice_p, out_choice_d, out_mse, out_cand_mse, out_phi, out_order, out_sigma,
                                 out_status, out_choice_q, out_theta, out_ma_order, css ? css->css_start : nullptr,
                                 css ? css->css : nullptr, css ? css->css_stop : nullptr, css ? css->iters : nullptr,
                                 joint ? joint->beta : nullptr, ml ? ml->loglik_start : nullptr,
                                 ml ? ml->loglik : nullptr, ml ? ml->stop : nullptr, ml ? ml->iters : nullptr,
                                 kf ? kf->se : nullptr}))
    return fail(MMF_E_UNSUPPORTED, "%s takes device buffers only", name);

  // (p, d, q) selection: the (p, q >= 1) pairs q-major, and their row sets R(q, L = max(p, q)) in order of appearance
  ArmaSelArgs hs{};
  if (with_q) {
    hs.n_mas = n_mas;
    for (int qi = 1; qi < n_mas; ++qi)
      for (int j = 0; j < n_orders; ++j) {
        const int p = orders[j], q = mas[qi], L = std::max(p, q);
        int r = 0;
        while (r < hs.n_rs && !(hs.rs_q[r] == q && hs.rs_L[r] == L)) ++r;
        if (r == hs.n_rs) { hs.rs_q[r] = q; hs.rs_L[r] = L; hs.rs_pmax[r] = 0; ++hs.n_rs; }
        hs.rs_pmax[r] = std::max(hs.rs_pmax[r], p);
        const int c = hs.n_pq++;
        hs.pq_p[c] = p; hs.pq_q[c] = q; hs.pq_j[c] = j; hs.pq_qi[c] = qi; hs.pq_rs[c] = r;
      }
    for (int r = 0; r < hs.n_rs; ++r) {
      const int nd = hs.rs_pmax[r] + hs.rs_q[r] + 1;
      hs.rs_off[r] = hs.n_ent;
      hs.n_ent += nd * (nd + 1) / 2 - 1;
    }
  }

  // slabs as the plain fit of the level rows would cut them; per slab, one fit and one arima_select_kernel per listed d
  // (their status goes to per-slab scratch, arima_select_kernel writes the caller's)
  const Plan& level_plan = use_plain ? pl : ap.diff[0];
  const int64_t slab = slab_rows(level_plan, n);
  int rc = grow((void**)&ctx->d_asel_best, &ctx->asel_best_cap, (size_t)slab * sizeof(ArimaSelBest));
  if (rc == MMF_OK) rc = grow((void**)&ctx->d_asel_status, &ctx->asel_status_cap, (size_t)slab * sizeof(int32_t));
  if (rc == MMF_OK && with_q)
    rc = grow((void**)&ctx->d_hsel_q0, &ctx->hsel_q0_cap, (size_t)slab * n_diffs * n_orders * sizeof(float));
  if (rc != MMF_OK) return rc;
  std::vector<Stage> stages;
  for (int k = 0; k < n_diffs; ++k) {
    const int dd = diffs[k];
    const Plan& plan = dd == 0 ? pl : ap.diff[dd - 1];
    Call c = plain_call(y, ld_y, pred_start, n_pred, out_pred, ld_out, ctx->d_asel_status);
    c.ar = ar_args(orders[n_orders - 1], out_phi, out_order, out_sigma, plan);
    c.arima = arima_args(ld_y, T, dd);
    ArimaSelArgs sel{};
    sel.n_hold = n_hold; sel.n_cand = n_orders;
    for (int j = 0; j < n_orders; ++j) sel.cand[j] = orders[j];
    sel.d_index = k; sel.n_diffs = n_diffs;
    sel.best = ctx->d_asel_best;
    sel.choice_p = out_choice_p; sel.choice_d = out_choice_d; sel.mse = out_mse; sel.cand_mse = out_cand_mse;
    sel.status = out_status;
    if (with_q) {
      // arima_select_kernel's scores go to scratch: arma_select_kernel copies them into the q = 0 slice
      sel.cand_mse = ctx->d_hsel_q0;
      ArmaSelArgs hsd = hs;
      hsd.cand_q0 = ctx->d_hsel_q0;
      hsd.cand_mse = out_cand_mse; hsd.choice_q = out_choice_q; hsd.theta = out_theta; hsd.ma_order = out_ma_order;
      hsd.m = long_order != 0 ? long_order : hr_long_order(std::max(orders[n_orders - 1], mas[n_mas - 1]), T - dd);
      c.hsel = hsd;
    }
    c.asel = sel;
    stages.push_back({&plan, c});
  }
  // the refit of the winners: per listed d, that d's fit again (the selection's z', gamma / c and status scratch hold the
  // last d's by then; the status goes to scratch), then the list of the winners with this d and q >= 1 and their refit
  // at the winner's (p, q) with long order m_d.  ar.p / hr.q: the largest listed orders (read by no product kernel)
  for (int k = 0; css && k < n_diffs; ++k) {
    const int dd = diffs[k];
    const Plan& plan = dd == 0 ? pl : ap.diff[dd - 1];
    Call c = plain_call(y, ld_y, pred_start, n_pred, out_pred, ld_out, ctx->d_asel_status);
    c.ar = ar_args(orders[n_orders - 1], out_phi, out_order, out_sigma, plan);
    c.arima = arima_args(ld_y, T, dd);
    ArmaArgs hr{};
    hr.q = mas[n_mas - 1];
    hr.m = long_order != 0 ? long_order : hr_long_order(std::max(orders[n_orders - 1], mas[n_mas - 1]), T - dd);
    hr.theta = out_theta; hr.ma_order = out_ma_order;
    c.arma = hr;
    c.css = *css;
    if (joint) c.joint = *joint;
    if (ml) c.ml = *ml;
    if (kf) {
      c.kf = *kf;
      c.kf_list = kf->se == nullptr;
      c.se_pass = kf->se != nullptr && k == n_diffs - 1;
    }
    RefitArgs rf{};
    rf.choice_d = out_choice_d; rf.choice_q = out_choice_q; rf.first = k == 0;
    c.refit = rf;
    stages.push_back({&plan, c});
  }
  // the Kalman stages of a call with standard errors: per listed d, the refit stage's fit and list again (the scratch
  // holds the last d's), then arma_kf_list_kernel over the ML refit's outputs
  for (int k = 0; kf && kf->se && k < n_diffs; ++k) {
    Stage st = stages[n_diffs + k];
    st.call.ml.reset();
    st.call.kf_list = true; st.call.se_pass = false; st.call.kf_only = true;
    st.call.refit->first = 0;
    stages.push_back(st);
  }
  return enqueue(ctx, level_plan, std::move(stages), n, stats);
}

int mmf_fit_select_arima_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                             const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                             int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                             int32_t* out_choice_p, int32_t* out_choice_d, float* out_mse, float* out_cand_mse,
                             float* out_phi, int32_t* out_order, float* out_sigma, int32_t* out_status,
                             mmf_stats* stats) {
  return select_arima_call(ctx, "mmf_fit_select_arima_f32", false, y, n, ld_y, n_hold, orders, n_orders, diffs, n_diffs,
                           nullptr, 0, 0, pred_start, n_pred, out_pred, ld_out, out_choice_p, out_choice_d, nullptr,
                           out_mse, out_cand_mse, out_phi, nullptr, out_order, nullptr, out_sigma, out_status, stats);
}

int mmf_fit_select_arma_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                            const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                            const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t pred_start, int32_t n_pred,
                            float* out_pred, int64_t ld_out, int32_t* out_choice_p, int32_t* out_choice_d,
                            int32_t* out_choice_q, float* out_mse, float* out_cand_mse, float* out_phi,
                            float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                            int32_t* out_status, mmf_stats* stats) {
  return select_arima_call(ctx, "mmf_fit_select_arma_f32", true, y, n, ld_y, n_hold, orders, n_orders, diffs, n_diffs, mas,
                           n_mas, long_order, pred_start, n_pred, out_pred, ld_out, out_choice_p, out_choice_d,
                           out_choice_q, out_mse, out_cand_mse, out_phi, out_theta, out_order, out_ma_order, out_sigma,
                           out_status, stats);
}

int mmf_fit_select_arma_css_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                                const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                                const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t max_iter,
                                int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                                int32_t* out_choice_p, int32_t* out_choice_d, int32_t* out_choice_q, float* out_mse,
                                float* out_cand_mse, float* out_phi, float* out_theta, int32_t* out_order,
                                int32_t* out_ma_order, float* out_sigma, int32_t* out_status, float* out_css_start,
                                float* out_css, int32_t* out_css_stop, int32_t* out_iters, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (max_iter < 0 || max_iter > MMF_CSS_ITER_MAX)
    return fail(MMF_E_INVALID, "max_iter=%d outside [0,%d]", max_iter, MMF_CSS_ITER_MAX);
  CssArgs css{};
  css.max_iter = max_iter == 0 ? MMF_CSS_ITER_DEFAULT : max_iter;
  css.css_start = out_css_start; css.css = out_css; css.css_stop = out_css_stop; css.iters = out_iters;
  return select_arima_call(ctx, "mmf_fit_select_arma_css_f32", true, y, n, ld_y, n_hold, orders, n_orders, diffs,
                           n_diffs, mas, n_mas, long_order, pred_start, n_pred, out_pred, ld_out, out_choice_p,
                           out_choice_d, out_choice_q, out_mse, out_cand_mse, out_phi, out_theta, out_order,
                           out_ma_order, out_sigma, out_status, stats, &css);
}

int mmf_fit_select_arma_joint_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                                  const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                                  const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t max_iter,
                                  int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out, float* out_beta,
                                  int32_t* out_choice_p, int32_t* out_choice_d, int32_t* out_choice_q, float* out_mse,
                                  float* out_cand_mse, float* out_phi, float* out_theta, int32_t* out_order,
                                  int32_t* out_ma_order, float* out_sigma, int32_t* out_status, float* out_css_start,
                                  float* out_css, int32_t* out_css_stop, int32_t* out_iters, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (max_iter < 0 || max_iter > MMF_CSS_ITER_MAX)
    return fail(MMF_E_INVALID, "max_iter=%d outside [0,%d]", max_iter, MMF_CSS_ITER_MAX);
  CssArgs css{};
  css.max_iter = max_iter == 0 ? MMF_CSS_ITER_DEFAULT : max_iter;
  css.css_start = out_css_start; css.css = out_css; css.css_stop = out_css_stop; css.iters = out_iters;
  JointArgs joint{};
  joint.beta = out_beta;
  return select_arima_call(ctx, "mmf_fit_select_arma_joint_f32", true, y, n, ld_y, n_hold, orders, n_orders, diffs,
                           n_diffs, mas, n_mas, long_order, pred_start, n_pred, out_pred, ld_out, out_choice_p,
                           out_choice_d, out_choice_q, out_mse, out_cand_mse, out_phi, out_theta, out_order,
                           out_ma_order, out_sigma, out_status, stats, &css, &joint);
}

int mmf_fit_select_arma_ml_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                               const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                               const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t max_iter,
                               int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                               int32_t* out_choice_p, int32_t* out_choice_d, int32_t* out_choice_q, float* out_mse,
                               float* out_cand_mse, float* out_phi, float* out_theta, int32_t* out_order,
                               int32_t* out_ma_order, float* out_sigma, int32_t* out_status, float* out_loglik_start,
                               float* out_loglik, int32_t* out_ml_stop, int32_t* out_iters, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (max_iter < 0 || max_iter > MMF_CSS_ITER_MAX)
    return fail(MMF_E_INVALID, "max_iter=%d outside [0,%d]", max_iter, MMF_CSS_ITER_MAX);
  CssArgs css{};                           // the CSS refit's start, its own columns unwritten
  css.max_iter = max_iter == 0 ? MMF_CSS_ITER_DEFAULT : max_iter;
  MlArgs ml{};
  ml.max_iter = css.max_iter;
  ml.loglik_start = out_loglik_start; ml.loglik = out_loglik; ml.stop = out_ml_stop; ml.iters = out_iters;
  return select_arima_call(ctx, "mmf_fit_select_arma_ml_f32", true, y, n, ld_y, n_hold, orders, n_orders, diffs,
                           n_diffs, mas, n_mas, long_order, pred_start, n_pred, out_pred, ld_out, out_choice_p,
                           out_choice_d, out_choice_q, out_mse, out_cand_mse, out_phi, out_theta, out_order,
                           out_ma_order, out_sigma, out_status, stats, &css, nullptr, &ml);
}

int mmf_fit_select_arma_ml_kf_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                                  const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                                  const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t max_iter,
                                  int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                                  int32_t* out_choice_p, int32_t* out_choice_d, int32_t* out_choice_q, float* out_mse,
                                  float* out_cand_mse, float* out_phi, float* out_theta, int32_t* out_order,
                                  int32_t* out_ma_order, float* out_sigma, int32_t* out_status,
                                  float* out_loglik_start, float* out_loglik, int32_t* out_ml_stop, int32_t* out_iters,
                                  float* out_se, int64_t ld_se, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  if (max_iter < 0 || max_iter > MMF_CSS_ITER_MAX)
    return fail(MMF_E_INVALID, "max_iter=%d outside [0,%d]", max_iter, MMF_CSS_ITER_MAX);
  CssArgs css{};                           // the ML refit's stages, then the predictor
  css.max_iter = max_iter == 0 ? MMF_CSS_ITER_DEFAULT : max_iter;
  MlArgs ml{};
  ml.max_iter = css.max_iter;
  ml.loglik_start = out_loglik_start; ml.loglik = out_loglik; ml.stop = out_ml_stop; ml.iters = out_iters;
  KfArgs kf{};
  kf.se = out_se; kf.ld_se = ld_se;
  return select_arima_call(ctx, "mmf_fit_select_arma_ml_kf_f32", true, y, n, ld_y, n_hold, orders, n_orders, diffs,
                           n_diffs, mas, n_mas, long_order, pred_start, n_pred, out_pred, ld_out, out_choice_p,
                           out_choice_d, out_choice_q, out_mse, out_cand_mse, out_phi, out_theta, out_order,
                           out_ma_order, out_sigma, out_status, stats, &css, nullptr, &ml, &kf);
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
  CU_TRY(cudaSetDevice(ctx->device));
  return build_multi(ctx->multi, X_all, n_cal, n_rows, t_fit, pred_start, n_pred_cal, p, has_constant, many, n_pred,
                     n_pred_max, ctx->stream);
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
  if (!on_device({y, out_pred}, {out_status})) return fail(MMF_E_INVALID, "the ragged entry point takes device buffers only");
  if (ld_y % 4 != 0 || (reinterpret_cast<uintptr_t>(y) & 15u) != 0 || (reinterpret_cast<uintptr_t>(out_pred) & 15u) != 0)
    return fail(MMF_E_UNSUPPORTED, "ragged batches need 16-B aligned y / out_pred and ld_y %% 4 == 0 (TMA)");
  cudaStream_t s = ctx->stream;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  CU_TRY(cudaStreamIsCapturing(s, &cap));
  if (cap != cudaStreamCaptureStatusNone) return fail(MMF_E_UNSUPPORTED, "ragged batches cannot be captured into a CUDA graph");
  int32_t* status = out_status;
  if (int rc = status_or_scratch(ctx, &status, n)) return rc;
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
  }
  const int cs = ctx->counter_set;
  uint32_t* counters = ctx->d_pending + CTR_WORDS * cs;
  ctx->set_clean[cs] = false;
  CU_TRY(cudaMemsetAsync(counters, 0, CTR_WORDS * sizeof(uint32_t), s));
  CU_TRY(cudaMemsetAsync(m.d_pending_by_cal, 0, (size_t)m.n_cal * sizeof(uint32_t), s));
  if (may_mask) a.rec_count = counters + 1;
  const DesignView d = view_of(m);
  MultiView mv{};
  mv.cals = m.d_cals; mv.tiles = m.d_tiles; mv.tmaps_y = m.d_tmaps_y; mv.pending_by_cal = m.d_pending_by_cal;
  mv.n_cal = m.n_cal; mv.n_tiles = m.n_tiles;
  TcLaunch tl;
  int rc = encode_2d(tl.tmap_y, y, (uint64_t)m.cals[0].t_fit, (uint64_t)n, (uint64_t)ld_y * 4, 32, 128);   // unused by ragged tiles
  if (rc != MMF_OK) return rc;
  memcpy(tl.tmap_at, m.tmap_at, 128);
  if (int rc = stats_begin(ctx, stats)) return rc;
  Tally t{0, MMF_KERNEL_TC};
  CU_TRY(launch_fit_tc(d, a, tl, counters, ctx->sm_count, s, 0, &mv));
  ++t.launches;
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
        FitArgs ac = a;
        ac.y = y + r0 * ld_y; ac.n = nr; ac.out = out_pred + r0 * ld_out; ac.status = status + r0;
        ac.pred_start = cm.pred_start; ac.recs = a.recs + r0; ac.row_base = r0; ac.cal_id = c;
        if (a.out_gamma != nullptr) { ac.out_gamma = a.out_gamma + r0 * P; ac.out_c = a.out_c + r0; }
        ac.only_pending = 1; ac.pending_count = nullptr;
        CU_TRY(launch_fit_warp(view_of(m, c), ac, ctx->sm_count, s));
        ++t.launches;
      }
    }
    CU_TRY(launch_solve_rows(d, a, ctx->sm_count, s, m.d_cals));
    ++t.launches;
  }
  if (m.many_pred) {
    PredictLaunch pl;
    memcpy(pl.tmap_bhi, m.tmap_bhi, 128);
    memcpy(pl.tmap_blo, m.tmap_blo, 128);
    memcpy(pl.tmap_out, m.tmap_bhi, 128);                  // unused by the ragged kernel (per-calendar maps instead)
    pl.n_tma = 0;                                          // unused as well: each calendar's map clips its own block
    CU_TRY(launch_predict_tc(d, a, pl, ctx->sm_count, s, m.d_units, m.n_units, m.d_tmaps_out));
    ++t.launches;
  }
  ctx->last_set = cs;
  return stats_tail(ctx, stats, n, t, nullptr, 0, pend);
}

// ---- rolling-origin backtest: K origins in one pass (DESIGN.md sections 2 item 8, 4.12) -------------------------
int mmf_plan_backtest(mmf_ctx* ctx, const double* X, int32_t n_rows, int32_t p, int32_t has_constant, int32_t n_origin,
                      const int32_t* origin, int32_t horizon) {
  if (!ctx || !X || !origin) return fail(MMF_E_INVALID, "ctx, X or origin is NULL");
  if (p < 1 || p > P) return fail(MMF_E_INVALID, "p=%d outside [1,%d]", p, P);
  if (n_origin < 1 || n_origin > MMF_BT_MAX_ORIGINS)
    return fail(MMF_E_INVALID, "n_origin=%d outside [1,%d]", n_origin, MMF_BT_MAX_ORIGINS);
  if (horizon < 1 || horizon > 64) return fail(MMF_E_INVALID, "horizon=%d outside [1,64]", horizon);
  for (int k = 0; k < n_origin; ++k)
    if (origin[k] < 33 || (k > 0 && origin[k] <= origin[k - 1]))
      return fail(MMF_E_INVALID, "origins must be increasing and at least 33 (origin[%d]=%d)", k, origin[k]);
  const int32_t t_k = origin[n_origin - 1];
  if (t_k > 65535) return fail(MMF_E_UNSUPPORTED, "the last origin %d exceeds 65535", t_k);
  if ((int64_t)t_k + horizon > n_rows)
    return fail(MMF_E_INVALID, "the last origin + horizon = %d exceeds the %d design rows", t_k + horizon, n_rows);
  for (int64_t i = 0; i < (int64_t)n_rows * p; ++i)
    if (!std::isfinite(X[i])) return fail(MMF_E_INVALID, "design matrix has a non-finite entry at %lld", (long long)i);
  if (has_constant)
    for (int32_t t = 0; t < n_rows; ++t)
      if (X[(int64_t)t * p] != 1.0) return fail(MMF_E_INVALID, "has_constant=1 but X[%d,0] != 1", t);
  if (ctx->pinned > 0) return fail(MMF_E_UNSUPPORTED, "a captured CUDA graph pins this context");
  // origin k as calendar k: the first t_k + horizon rows of X, fit on [0, t_k), evaluated on [t_k, t_k + horizon)
  std::vector<int32_t> rows(n_origin), tfit(n_origin), pstart(n_origin), npred(n_origin, horizon);
  std::vector<double> X_all;
  for (int k = 0; k < n_origin; ++k) {
    rows[k] = origin[k] + horizon; tfit[k] = origin[k]; pstart[k] = origin[k];
    X_all.insert(X_all.end(), X, X + (size_t)rows[k] * p);
  }
  // the change of basis, float64: x_t = a_t W^-1 on the columns the longest window keeps, so a^(k)_t = a_t T_k with
  // T_k = W^-1 W_k.  W is upper triangular on its kept columns (W = L^-T): T_k by back substitution.
  double W[P * P];
  uint32_t kept = 0;
  std::vector<float> A;
  whiten_calendar(X, t_k + horizon, p, t_k, W, &kept, A);
  std::vector<float> tmat((size_t)n_origin * P * P, 0.f), pred((size_t)n_origin * horizon * P, 0.f);
  for (int k = 0; k < n_origin; ++k) {
    float* tk = tmat.data() + (size_t)k * P * P;
    float* pk = pred.data() + (size_t)k * horizon * P;
    if (k == n_origin - 1) {                               // the longest window itself: T = I, its own rows exactly
      for (int j = 0; j < P; ++j) tk[j * P + j] = ((kept >> j) & 1u) ? 1.f : 0.f;
      memcpy(pk, A.data() + (size_t)t_k * P, (size_t)horizon * P * sizeof(float));
      continue;
    }
    double Wk[P * P];
    uint32_t kept_k = 0;
    std::vector<float> Ak;
    whiten_calendar(X, rows[k], p, tfit[k], Wk, &kept_k, Ak);
    if ((kept_k & ~kept) != 0u)
      return fail(MMF_E_UNSUPPORTED, "origin %d keeps a column the longest window drops (kept 0x%x, longest 0x%x)",
                  origin[k], kept_k, kept);
    double T[P][P] = {};
    for (int c = 0; c < P; ++c)
      for (int r = P - 1; r >= 0; --r) {
        if (!((kept >> r) & 1u)) continue;
        double s = Wk[r * P + c];
        for (int q = r + 1; q < P; ++q) s -= W[r * P + q] * T[q][c];
        T[r][c] = s / W[r * P + r];
      }
    for (int r = 0; r < P; ++r)
      for (int c = 0; c < P; ++c) tk[r * P + c] = (float)T[r][c];
    // prediction rows in the common basis: T_k a^(k)_t, a^(k)_t = x_t W_k, all in float64
    for (int h = 0; h < horizon; ++h) {
      const double* x = X + (size_t)(origin[k] + h) * p;
      double ak[P];
      for (int c = 0; c < P; ++c) {
        double s = 0.0;
        for (int i = 0; i < p; ++i) s += x[i] * Wk[i * P + c];
        ak[c] = s;
      }
      for (int r = 0; r < P; ++r) {
        double s = 0.0;
        for (int c = 0; c < P; ++c) s += T[r][c] * ak[c];
        pk[(size_t)h * P + r] = (float)s;
      }
    }
  }
  CU_TRY(cudaSetDevice(ctx->device));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  free_bt(ctx->bt);
  BtPlan& b = ctx->bt;
  int rc = build_plan(b.common, X, t_k + horizon, p, t_k, has_constant);
  if (rc == MMF_OK)
    rc = build_multi(b.cals, X_all.data(), n_origin, rows.data(), tfit.data(), pstart.data(), npred.data(), p, has_constant,
                     false, horizon, horizon, ctx->stream);
  if (rc != MMF_OK) { free_bt(ctx->bt); return rc; }
  CU_TRY(cudaMalloc(&b.d_pred, pred.size() * sizeof(float)));
  CU_TRY(cudaMalloc(&b.d_tmat, tmat.size() * sizeof(float)));
  CU_TRY(cudaMemcpy(b.d_pred, pred.data(), pred.size() * sizeof(float), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy(b.d_tmat, tmat.data(), tmat.size() * sizeof(float), cudaMemcpyHostToDevice));
  b.n_origin = n_origin; b.horizon = horizon;
  for (int k = 0; k < n_origin; ++k) b.origin[k] = origin[k];
  b.valid = true;
  return MMF_OK;
}

int mmf_backtest_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, float* out_pred, int64_t ld_out,
                     float* out_metrics, int32_t* out_count, int32_t* out_status, mmf_stats* stats) {
  if (!ctx) return fail(MMF_E_INVALID, "ctx is NULL");
  GrowScope grow_scope(ctx);
  const BtPlan& b = ctx->bt;
  if (!b.valid) return fail(MMF_E_NOPLAN, "mmf_plan_backtest has not been called");
  const int K = b.n_origin, H = b.horizon, t_K = b.origin[K - 1];
  if (n < 0 || (n > 0 && !y)) return fail(MMF_E_INVALID, "bad y / n");
  if (!out_pred && !out_metrics) return fail(MMF_E_INVALID, "out_pred and out_metrics are both NULL");
  if (ld_y < (int64_t)t_K + H)
    return fail(MMF_E_INVALID, "ld_y=%lld < last origin + horizon = %d (the actual values are read)", (long long)ld_y, t_K + H);
  if (out_pred && ld_out < H) return fail(MMF_E_INVALID, "ld_out=%lld < horizon=%d", (long long)ld_out, H);
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n == 0) return MMF_OK;
  if (n > (int64_t)0x7fffffff - 128) return fail(MMF_E_UNSUPPORTED, "n too large for 32-bit TMA coordinates");
  if (ld_y % 4 != 0 || (reinterpret_cast<uintptr_t>(y) & 15u) != 0)
    return fail(MMF_E_UNSUPPORTED, "backtests need a 16-B aligned y with ld_y %% 4 == 0 (TMA)");
  CU_TRY(cudaSetDevice(ctx->device));
  if (!on_device({y}, {out_pred, out_metrics, out_count, out_status}))
    return fail(MMF_E_UNSUPPORTED, "mmf_backtest_f32 takes device buffers only");
  cudaStream_t s = ctx->stream;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  CU_TRY(cudaStreamIsCapturing(s, &cap));
  if (cap != cudaStreamCaptureStatusNone) return fail(MMF_E_UNSUPPORTED, "backtests cannot be captured into a CUDA graph");
  // slabs (section 4.10) over the K * n output rows: at most 2^20 of them per slab, whole 128-row tiles, equal slabs
  int64_t slab = n;
  if ((int64_t)K * n > ((int64_t)1 << 20)) {
    slab = std::max<int64_t>(128, (((int64_t)1 << 20) / K) & ~(int64_t)127);
    const int64_t n_slabs = (n + slab - 1) / slab;
    slab = (((n + n_slabs - 1) / n_slabs) + 127) & ~(int64_t)127;
  }
  const int64_t n_slabs = (n + slab - 1) / slab;
  const bool may_mask = !ctx->cfg.assume_finite;
  int32_t* status = out_status;
  int rc = status_or_scratch(ctx, &status, (int64_t)K * n);
  if (rc == MMF_OK) rc = grow((void**)&ctx->d_bt_ctr, &ctx->bt_ctr_cap, 2 * MMF_BT_MAX_ORIGINS * sizeof(uint32_t));
  if (rc == MMF_OK && K > 1) rc = grow((void**)&ctx->d_bt_mom, &ctx->bt_mom_cap, (size_t)(K - 1) * 2 * slab * P * sizeof(float));
  if (rc == MMF_OK && may_mask) rc = grow((void**)&ctx->d_bt_recs, &ctx->bt_recs_cap, (size_t)K * slab * sizeof(SolveRec));
  if (rc == MMF_OK && may_mask) rc = grow((void**)&ctx->d_bt_rows, &ctx->bt_rows_cap, (size_t)K * slab * sizeof(int64_t));
  const int64_t ld_scr = (H + 3) & ~3;
  if (rc == MMF_OK && !out_pred) rc = grow((void**)&ctx->d_bt_pred, &ctx->bt_pred_cap, (size_t)K * slab * ld_scr * sizeof(float));
  uint32_t* slab_pending = nullptr;
  if (rc == MMF_OK && stats) {
    rc = grow_unpinned((void**)&ctx->d_slab_pending, &ctx->slab_pending_cap, (size_t)n_slabs * sizeof(uint32_t));
    slab_pending = ctx->d_slab_pending;
  }
  if (rc != MMF_OK) return rc;
  const int cs = ctx->counter_set;
  uint32_t* counters = ctx->d_pending + CTR_WORDS * cs;
  ctx->set_clean[cs] = false;
  const DesignView d = view_of(b.common);
  const DesignView dm = view_of(b.cals);                   // the origins' stacked designs, as a ragged plan's
  uint32_t* rec_count = ctx->d_bt_ctr;
  uint32_t* pend_by_origin = ctx->d_bt_ctr + MMF_BT_MAX_ORIGINS;
  if (int rc = stats_begin(ctx, stats)) return rc;
  Tally t{0, MMF_KERNEL_TC};
  for (int64_t off = 0, si = 0; off < n; off += slab, ++si) {
    const int64_t m = std::min(slab, n - off);
    float* obase = out_pred ? out_pred + off * ld_out : ctx->d_bt_pred;
    const int64_t ldo = out_pred ? ld_out : ld_scr;
    const int64_t okstride = out_pred ? n : m;
    CU_TRY(cudaMemsetAsync(counters, 0, CTR_WORDS * sizeof(uint32_t), s));
    CU_TRY(cudaMemsetAsync(ctx->d_bt_ctr, 0, 2 * MMF_BT_MAX_ORIGINS * sizeof(uint32_t), s));
    FitArgs a{};
    a.y = y + off * ld_y; a.n = m; a.ld_y = ld_y; a.pred_start = t_K; a.n_pred = H;
    a.out = obase; a.ld_out = ldo; a.status = status + off; a.n_out = 1;
    if (may_mask) {
      a.recs = ctx->d_bt_recs + (int64_t)(K - 1) * m;       // the consumers record gap positions in the last origin's block
      a.rec_rows = ctx->d_bt_rows + (int64_t)(K - 1) * m;
      a.rec_count = rec_count + (K - 1);
      a.rec_cap = (uint32_t)m;
    }
    BtArgs bt{};
    bt.cals = b.cals.d_cals; bt.pred = b.d_pred; bt.tmat = b.d_tmat; bt.mom = ctx->d_bt_mom;
    bt.recs = ctx->d_bt_recs; bt.rec_rows = ctx->d_bt_rows; bt.rec_count = rec_count; bt.pending = pend_by_origin;
    bt.out_kstride = okstride; bt.st_kstride = n; bt.n_origin = K;
    for (int k = 0; k < MMF_BT_MAX_ORIGINS - 1; ++k) bt.t_orig[k] = k < K - 1 ? b.origin[k] : INT32_MAX;
    TcLaunch tl;
    rc = encode_2d(tl.tmap_y, a.y, (uint64_t)t_K, (uint64_t)m, (uint64_t)ld_y * 4, 32, 128);
    if (rc != MMF_OK) return rc;
    memcpy(tl.tmap_at, b.common.tmap_at, 128);
    CU_TRY(launch_fit_tc_bt(d, a, tl, counters, ctx->sm_count, s, bt));
    ++t.launches;
    if (may_mask) {
      // per origin: the general pass for the rows the fast path left to it (exits at once when there are none), then
      // the solve of the queued records, calendar = origin
      for (int k = 0; k < K; ++k) {
        const CalMeta& cm = b.cals.cals[k];
        FitArgs ak = a;
        ak.out = obase + (int64_t)k * okstride * ldo; ak.status = status + (int64_t)k * n + off;
        ak.pred_start = cm.pred_start; ak.recs = ctx->d_bt_recs + (int64_t)k * m; ak.rec_rows = ctx->d_bt_rows + (int64_t)k * m;
        ak.rec_count = rec_count + k; ak.row_base = 0; ak.cal_id = k;
        ak.only_pending = 1; ak.pending_count = pend_by_origin + k;
        CU_TRY(launch_fit_warp(view_of(b.cals, k), ak, ctx->sm_count, s));
        ak.pending_count = nullptr;
        CU_TRY(launch_solve_rows(dm, ak, ctx->sm_count, s, b.cals.d_cals));
        t.launches += 2;
      }
    }
    ScoreArgs sa{};
    sa.pred = obase; sa.ld_pred = ldo; sa.pred_kstride = okstride; sa.y = a.y; sa.ld_y = ld_y; sa.cals = b.cals.d_cals;
    sa.metrics = out_metrics ? out_metrics + off * MMF_BT_NMETRIC : nullptr; sa.count = out_count ? out_count + off : nullptr;
    sa.out_kstride = n; sa.n = m; sa.n_origin = K; sa.horizon = H;
    if (sa.metrics || sa.count) {
      CU_TRY(launch_bt_score(sa, ctx->sm_count, s));
      ++t.launches;
    }
    if (slab_pending != nullptr)
      CU_TRY(cudaMemcpyAsync(slab_pending + si, counters, sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  }
  ctx->last_set = cs;
  return stats_tail(ctx, stats, n, t, slab_pending, (size_t)n_slabs);
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
  if (int rc = check_window(pred_start, n_pred, pl.n_rows, ld_out)) return rc;
  if (n == 0) return MMF_OK;
  CU_TRY(cudaSetDevice(ctx->device));
  if (!is_device_ptr(y)) return fail(MMF_E_INVALID, "the broadcast variant takes device buffers only");
  Call c = plain_call(y, ld_y, pred_start, n_pred, reinterpret_cast<float*>(out_ptrs[0]), ld_out, out_status);
  c.beta = out_beta;
  c.n_out = n_out; c.multimem = multimem;
  for (int i = 1; i < n_out; ++i) c.out_more[i - 1] = reinterpret_cast<float*>(out_ptrs[i]);
  return enqueue(ctx, pl, {{&pl, c}}, n, nullptr);
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
  if (!on_device({y, out_pred}, {})) return fail(MMF_E_INVALID, "device buffers only");
  SelectArgs sel{};
  sel.n_hold = n_hold;
  sel.n_cand = n_cand;
  for (int i = 0; i < n_cand; ++i) sel.cand[i] = candidates[i];
  sel.out_choice = out_choice;
  sel.out_mse = out_mse;
  Call c = plain_call(y, ld_y, pred_start, n_pred, out_pred, ld_out, out_status);
  c.sel = sel;
  return enqueue(ctx, pl, {{&pl, c}}, n, nullptr);
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
