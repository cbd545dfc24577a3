// Internal declarations shared by the C-ABI translation unit and the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/mmf.h"

namespace mmf {

constexpr int P = MMF_P;                 // design columns
constexpr int NPAIR = P * (P + 1) / 2;   // packed symmetric Gram entries (136)

// ---- device-side view of a planned design --------------------------------
// A = X W (whitened, float32).  Three layouts of the same numbers:
//  a4   : column-blocked float4, a4[j*n_rows_pad + t] = A[t][4j..4j+3]   (warp kernel: conflict-free LDS.128)
//  at   : [2P][t_pad] K-major rows for the tensor-core B operand: row n<P is tf32-hi of column n,
//         row P+n is the tf32 residual (lo); columns t >= t_fit are zero            (tensor-core kernel)
//  apred: [n_rows][P] row-major                                                     (wgmma epilogue)
struct DesignView {
  const float4* a4;
  const float*  at;
  const float*  apred;
  const float*  w;          // [P][P] row-major float32 whitening matrix (beta = W gamma)
  int32_t n_rows;
  int32_t n_rows_pad;       // multiple of 32
  int32_t t_fit;
  int32_t t_pad;            // t_fit rounded up to 32
  uint32_t kept_mask;       // bit j set: whitened column j retained on the calendar
  int32_t has_constant;
};

// ---- ragged batches: groups on MANY calendars in one launch ---------------------------------------------
// The reference re-indexes every group on its own calendar (02:422-423); a batch can therefore hold groups with
// different first dates and lengths.  A ragged plan stacks the whitened designs of all calendars (A operand rows,
// prediction rows) and a launch carries a table of 128-row tiles, each inside one calendar: the kernels read the
// tile's calendar from the table instead of from launch constants.
struct CalMeta {                           // one calendar of a ragged plan (32 B)
  int32_t t_fit;
  int32_t n_chunks;                        // ceil(t_fit / 32): 32-step chunks of the tensor-core kernel
  int32_t n_rows;                          // design rows planned (fit + forecast rows)
  uint32_t kept_mask;                      // whitened columns retained on this calendar
  int32_t row_off;                         // first row of this calendar in the stacked apred / ap_hi / ap_lo / a4 tables
  int32_t pred_start;                      // first prediction row, relative to the calendar's own rows
  int32_t n_pred;                          // prediction rows
  int32_t n_rows_pad;                      // rows of this calendar's a4 block (multiple of 32)
};
static_assert(sizeof(CalMeta) == 32, "CalMeta is two 16-B loads");
struct TileRec {                           // one 128-row tile of a ragged launch (16 B)
  int32_t row0;                            // first series row
  int32_t nrows;                           // rows of the tile that belong to the calendar (1..128)
  int32_t cal;
  int32_t n_chunks;                        // == cals[cal].n_chunks
};
struct MultiView {                         // all null / 0 for an ordinary single-calendar launch
  const CalMeta* cals;
  const TileRec* tiles;
  const unsigned char* tmaps_y;            // [n_cal][128]: the y buffer clipped at each calendar's t_fit (CUtensorMap)
  uint32_t* pending_by_cal;                // [n_cal]: rows per calendar the fast path left to the general pass
  int32_t n_cal;
  int32_t n_tiles;
  int32_t bal_rows;                        // balanced single-calendar launch: rows per CTA (multiple of 8), else 0
};

// One series with gaps, handed to the thread-per-series solve kernel (256 B, indexed by row).
// Missing grid positions come in two segments so that two producers (the two transform groups of the
// tensor-core kernel) can append without atomics: segment g holds nm[g] entries at miss_t[g*SOLVE_SEG ...].
// Segments are a multiple of 4 entries and 8-B aligned: the solve kernel reads the positions four at a time.
constexpr int SOLVE_SEG = 44;
constexpr int SOLVE_MISS_CAP = 2 * SOLVE_SEG;
struct SolveRec {
  float b[P];                              // moments A_fit^T (y - c) over the observed rows
  float c;                                 // centring constant
  uint16_t nm[2];                          // entries in each segment
  uint16_t miss_t[SOLVE_MISS_CAP];         // grid positions of the missing fit rows (byte offset 72)
  int32_t cal;                             // ragged launches: the series' calendar (index into MultiView::cals)
  uint16_t pad_[2];
};
static_assert(sizeof(SolveRec) == 256, "SolveRec is one 256-B record");
static_assert(SOLVE_SEG % 4 == 0 && offsetof(SolveRec, miss_t) % 8 == 0, "position groups are aligned 8-B words");
constexpr int MMF_STATUS_DEFERRED = -2;    // internal: the row's SolveRec is queued for solve_rows_kernel

constexpr int MAX_OUT = 8;               // replicas of the forecast table one launch can write (one per GPU)

struct FitArgs {
  const float* y;
  int64_t n;
  int64_t ld_y;
  int32_t pred_start;
  int32_t n_pred;
  float* out;               // forecast rows [n, ld_out]; with n_out > 1 the same rows also go to out_more[]
  int64_t ld_out;
  float* out_more[MAX_OUT - 1];   // peer-mapped copies of the table slice (NVLink P2P stores), n_out - 1 valid
  int32_t n_out;            // 1 = local only
  int32_t out_multimem;     // `out` is an NVLS multicast address: 1 -> multimem.st per row, 2 -> bulk (TMA) stores to it
  float* out_gamma;         // nullable [n][P]: whitened coefficients (+ out_c[n]) for predict_tc_kernel
  float* out_c;
  int32_t skip_pred;        // 1: fit only (gamma/c out); predictions come from predict_tc_kernel
  float* out_beta;          // nullable [n][P]
  int32_t* status;          // never null inside the library (scratch if caller passed NULL)
  SolveRec* recs;           // nullable: [n] records by row; series with gaps are deferred to solve_rows_kernel
  int64_t* rec_rows;        //   [n] work list: rows whose record is ready
  uint32_t* rec_count;      //   length of the work list (device counter)
  uint32_t rec_cap;         //   == n
  int32_t only_pending;     // 1: process only rows whose status == MMF_STATUS_PENDING
  const uint32_t* pending_count;  // nullable; if non-null and *pending_count == 0 the kernel exits at once
  uint32_t* zero_next;      // nullable: 2 counters of the NEXT call's set, zeroed by the tensor-core kernel (no memset node)
  uint32_t* stream_ctl;     // nullable: {claimed, CTAs finished, producer done} of the streaming solve (solve_stream_kernel
                            // consumes the queued records WHILE the tensor-core kernel is still producing them)
  int64_t row_base;         // ragged fallback launches cover one calendar's rows: absolute row of this launch's row 0
  int32_t cal_id;           //   ... and that calendar's index (written into the records the launch queues)
};

// warp-per-series CUDA-core kernel (general path)
cudaError_t launch_fit_warp(const DesignView& d, const FitArgs& a, int sm_count, cudaStream_t s);
size_t fit_warp_smem_bytes(const DesignView& d, int* smem_rows);

// thread-per-series normal equations for the deferred masked rows: Gram downdate, in-order Cholesky with
// pivot dropping and both triangular solves entirely in registers, then the forecasts
cudaError_t launch_solve_rows(const DesignView& d, const FitArgs& a, int sm_count, cudaStream_t s,
                              const CalMeta* cals = nullptr);
// the same solve as a CONSUMER that runs beside fit_tc_kernel (launched right behind it with programmatic stream
// serialisation; fit_tc_kernel releases it once all its CTAs are resident): records are solved as the epilogue
// publishes them, the kernel retires when the producer has finished and the work list is drained
cudaError_t launch_solve_stream(const DesignView& d, const FitArgs& a, int sm_count, cudaStream_t s);
constexpr int CTR_WORDS = 8;             // one counter set: {pending, records queued, claimed, CTAs finished, producer done, -, -, -}

// fitted values + forecasts for MANY prediction rows (the reference's "Demand_Fitted for every date"
// contract, 02:484-494): out[n, n_pred] = c + gamma A_pred^T as a wgmma GEMM with TMA-stored tiles
struct PredictLaunch {
  alignas(64) unsigned char tmap_bhi[128];
  alignas(64) unsigned char tmap_blo[128];
  alignas(64) unsigned char tmap_out[128];
};
struct PredUnit {                          // one (tile, chunk) work unit of a ragged predict launch (32 B)
  int32_t row0, nrows;                     // series rows of the tile inside one calendar
  int32_t cal;                             // calendar: selects the output tensor map
  int32_t ch;                              // 128-row chunk of that calendar's prediction rows
  int32_t b_row;                           // first row of the chunk in the stacked (hi / lo) design tables
  int32_t row_in_map;                      // row0 relative to the calendar's first row (outer coordinate of its map)
  int32_t pad_[2];
};
static_assert(sizeof(PredUnit) == 32, "PredUnit is two 16-B loads");
cudaError_t launch_predict_tc(const DesignView& d, const FitArgs& a, const PredictLaunch& pl, int sm_count,
                              cudaStream_t s, const PredUnit* units = nullptr, int64_t n_units_multi = 0,
                              const unsigned char* tmaps_out = nullptr);

// TMA + wgmma kernel (fully observed fast path).  `tmap_y` / `tmap_at` are CUtensorMap blobs.
struct TcLaunch {
  alignas(64) unsigned char tmap_y[128];    // box {32 t, 128 series}
  alignas(64) unsigned char tmap_at[128];
  alignas(64) unsigned char tmap_y8[128];   // box {32 t, 8 series}: the short last tile of a balanced launch's CTA
};
// variant: 0 / 1 = <10 smem stages, 1 forecast staging tile>, tiles dealt round robin (the product), 2 = <8 stages,
// 2 staging tiles>, 3 = balanced row ranges per CTA (both experiments that did not pay, kept for the record)
int fit_tc_balanced_rows(int64_t n, int sm_count, int variant);
cudaError_t launch_fit_tc(const DesignView& d, const FitArgs& a, const TcLaunch& tl,
                          uint32_t* pending_count, int sm_count, cudaStream_t s, int variant = 0,
                          const MultiView* multi = nullptr);
bool fit_tc_supported(const DesignView& d, const FitArgs& a, const char** why);

// per-series model selection by hold-out MSE over nested whitened designs (select.cu)
constexpr int MMF_MAX_CAND = 8;
struct SelectArgs {
  int32_t n_hold;                 // held-out rows: design rows [t_fit, t_fit + n_hold), y columns likewise
  int32_t n_cand;
  int32_t cand[MMF_MAX_CAND];     // ascending numbers of leading whitened columns, last == full model
  int32_t* out_choice;            // nullable [n]: chosen number of columns (0 for empty series)
  float* out_mse;                 // nullable [n]: hold-out MSE of the chosen model
};
cudaError_t launch_select(const DesignView& d, const FitArgs& a, const SelectArgs& sel, int sm_count, cudaStream_t s);

// integer series -> float32 staging rows, sentinel -> NaN (widen.cu); dtype = MMF_DT_I16 / U16 / I32
cudaError_t launch_widen(int dtype, const void* src, int64_t ld_src, float* dst, int64_t ld_dst, int64_t n, int32_t t,
                         int sm_count, cudaStream_t s);

// device-side packer (pack.cu)
cudaError_t pack_hash_utf8(const int32_t* offsets, const uint8_t* data, int64_t n, uint64_t* h, int first, int sm,
                           cudaStream_t s);
cudaError_t pack_hash_i32(const int32_t* v, int64_t n, uint64_t* h, int first, int sm, cudaStream_t s);
cudaError_t pack_verify_utf8(const int32_t* offsets, const uint8_t* data, int64_t n, const int32_t* gid,
                             const int32_t* first_row, uint64_t* mismatches, int sm, cudaStream_t s);
cudaError_t pack_verify_i32(const int32_t* v, int64_t n, const int32_t* gid, const int32_t* first_row,
                            uint64_t* mismatches, int sm, cudaStream_t s);
cudaError_t pack_group_codes_scratch_bytes(int64_t n, size_t* bytes);
cudaError_t pack_group_codes(const uint64_t* h, int64_t n, int32_t* gid, int32_t* first_row, int32_t* n_groups_host,
                             void* scratch, int sm, cudaStream_t s);
cudaError_t pack_minmax(const int32_t* gid, const int32_t* day, int64_t n, int32_t n_groups, int32_t* gmin,
                        int32_t* gmax, int sm, cudaStream_t s);
cudaError_t pack_scatter(const int32_t* gid, const int32_t* day, const float* val, int64_t n,
                         const int64_t* row_of_group, const int32_t* gstart, int32_t step, float* y, int64_t n_rows,
                         int64_t ld_y, int32_t t_len, unsigned long long* dups, int sm, cudaStream_t s);

#ifdef __CUDACC__
// Forecast stores: plain, NVSwitch multicast (multimem.st) or fan-out over peer-mapped pointers.
__device__ __forceinline__ void store_out1(const FitArgs& a, int64_t off, float v) {
  if (a.out_multimem) {
    asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(a.out + off), "f"(v) : "memory");
  } else {
    __stcs(a.out + off, v);
    for (int i = 0; i + 1 < a.n_out; ++i) __stcs(a.out_more[i] + off, v);
  }
}
__device__ __forceinline__ void store_out4(const FitArgs& a, int64_t off, float4 v) {   // off: 16-B aligned element offset
  if (a.out_multimem) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a.out + off), "f"(v.x), "f"(v.y),
                 "f"(v.z), "f"(v.w)
                 : "memory");
  } else {
    __stcs(reinterpret_cast<float4*>(a.out + off), v);
    for (int i = 0; i + 1 < a.n_out; ++i) __stcs(reinterpret_cast<float4*>(a.out_more[i] + off), v);
  }
}
#endif

}  // namespace mmf
