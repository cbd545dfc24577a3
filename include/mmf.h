/*
 * mmf.h -- C ABI of libmmf.so, the H100-native many-models fit+forecast engine.
 *
 * This is the drop-in boundary for ONE hot path of sebrahimi1988/dss-ml-at-scale:
 * the per-(Product,SKU) fit + predict that the reference fans out with
 *     enriched_df.repartition(n_tasks,"Product","SKU").groupBy("Product","SKU")
 *                .applyInPandas(build_tune_and_score_model, schema=tuning_schema)
 * (group_apply/02_Fine_Grained_Demand_Forecasting.py:523-528, UDF body 417-494).
 * The reference has no FFI of its own (it is pure Python on Spark); the binding a
 * maintainer adds is the ctypes stub in INTEGRATION.md.  Every entry point below
 * names the reference lines it replaces.
 *
 * Conventions
 *  - plain C, no CUDA/torch types: device and host pointers are both `float*`;
 *    the library classifies them with cudaPointerGetAttributes.
 *  - every function returns 0 on success or a negative MMF_E_* code; the text is
 *    available from mmf_last_error() (thread local).  Nothing throws across the ABI.
 *  - per-series numerical outcomes go to `out_status`, never to the return code.
 *  - a ctx is single-caller; separate ctxs (one per process / per GPU) are
 *    independent.  Missing observations are NaN (any non-finite value) in `y`.
 *  - series are rows: y[i*ld_y + t], t = 0..t_fit-1 on the shared regular grid
 *    (the packed form of `sort_values("Date").set_index("Date").asfreq(freq)`,
 *    reference 02:422-423).
 */
#ifndef MMF_H_
#define MMF_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MMF_VERSION 102          /* 0.1.2 */
#define MMF_P 16                 /* design columns (zero-pad narrower designs) */
#define MMF_PIVOT_TOL 1e-3f      /* per-series relative Cholesky pivot threshold */
#define MMF_CAL_TOL 1e-10        /* aliasing threshold on the float64 calendar Gram */
#define MMF_SELECT_MAX_HOLD 3500 /* held-out rows mmf_fit_select_forecast_f32 accepts (64 B of shared memory each) */

/* return codes */
#define MMF_OK 0
#define MMF_E_INVALID (-1)
#define MMF_E_CUDA (-2)
#define MMF_E_UNSUPPORTED (-3)
#define MMF_E_NOPLAN (-4)
#define MMF_E_NOMEM (-5)

/* per-series status (out_status) */
#define MMF_STATUS_OK 0          /* fit on all requested rows */
#define MMF_STATUS_EMPTY 1       /* no observed fit row: outputs are NaN */
#define MMF_STATUS_RANKDEF 2     /* ok, but a whitened column was dropped for this series' mask */
#define MMF_STATUS_PENDING (-1)  /* internal: fast path saw a non-finite value, masked pass owes a result */

/* element types of the series buffer (mmf_fit_forecast_int) and the value that means "missing" in each */
#define MMF_DT_F32 0             /* float32, NaN / Inf = missing (mmf_fit_forecast_f32)  */
#define MMF_DT_I16 1             /* int16,   -32768      = missing                        */
#define MMF_DT_U16 2             /* uint16,  65535       = missing                        */
#define MMF_DT_I32 3             /* int32,   INT32_MIN   = missing; exact for |v| < 2^24  */

/* kernel selection */
#define MMF_KERNEL_AUTO 0        /* tensor-core fast path + masked fix-up where eligible, else warp kernel */
#define MMF_KERNEL_WARP 1        /* warp-per-series CUDA-core kernel (general: masks, any ld, any n_pred) */
#define MMF_KERNEL_TC 2          /* TMA + wgmma kernel (fully observed rows; others -> masked pass) */

typedef struct mmf_ctx mmf_ctx;

typedef struct mmf_config {
  int32_t device;          /* CUDA device ordinal, -1 = current device */
  int32_t kernel;          /* MMF_KERNEL_* */
  int32_t assume_finite;   /* 1: caller guarantees y has no NaN/Inf, skip the masked fix-up pass */
  int32_t tc_variant;      /* tuning of the tensor-core kernel, same results whichever: 0 / 1 = the product (128-row tiles dealt
                              round robin over the SMs), 2 = the experimental <6-stage, 2 staging tiles> instantiation,
                              3 = the experimental balanced launch (one row range per SM) */
  int64_t chunk_series;    /* host-buffer path: series per pipelined chunk (0 = library default) */
  void*   stream;          /* cudaStream_t to enqueue on (NULL = library-owned stream) */
  int32_t host_narrow;     /* host-buffer path: 0 = automatic, 1 = always try, 2 = never: narrow float32 chunks to
                              uint16 on host threads when every value is an integer in [0, 65534] (exactly, or the
                              chunk goes as float32), so that half the bytes cross PCIe; widened back on the device */
  int32_t host_threads;    /* threads of that narrowing pool (0 = half of the process's cores, at most 16) */
  int32_t stream_solve;    /* series with gaps: 0 = solved in a pass of their own after the tensor-core kernel (default), 1 = by a
                              consumer kernel launched BESIDE it (experimental: pays only with a register-capped build) */
  int32_t reserved1;
} mmf_config;

typedef struct mmf_stats {
  float   kernel_ms;       /* device time of the fit kernels (CUDA events) */
  float   total_ms;        /* device time of the whole call incl. copies */
  int64_t n_series;
  int64_t n_pending;       /* rows the fast path handed to the masked pass */
  int64_t h2d_bytes;
  int64_t d2h_bytes;
  int32_t kernel_launches; /* kernels of this library launched by the call */
  int32_t kernel_used;     /* MMF_KERNEL_WARP or MMF_KERNEL_TC (dominant kernel) */
} mmf_stats;

/* ---- lifecycle ---------------------------------------------------------- */
int mmf_version(void);
const char* mmf_last_error(void);
int mmf_device_count(int32_t* count);
/* replaces: the Spark Python worker that hosts the UDF (one ctx per worker process) */
int mmf_create(const mmf_config* cfg, mmf_ctx** out);
int mmf_destroy(mmf_ctx* ctx);
int mmf_set_stream(mmf_ctx* ctx, void* cuda_stream);   /* borrow e.g. torch's current stream */
int mmf_synchronize(mmf_ctx* ctx);

/* ---- design plan --------------------------------------------------------
 * X: [n_rows, p] row-major float64 design rows on the shared calendar; rows
 * [0,t_fit) are the fit window, later rows are forecast rows.  p <= MMF_P.
 * has_constant: 1 iff X[:,0] == 1 for every row (enables per-series centring).
 * The library whitens the calendar Gram in float64 (in-order Cholesky, aliased
 * columns dropped), uploads A = X W in the layouts the kernels use.
 * replaces: the design the reference builds per row in add_exo_variables
 * (02:343-358) and hands to SARIMAX as exog= (02:441-449, 472-480).           */
int mmf_plan_design(mmf_ctx* ctx, const double* X, int32_t n_rows, int32_t p,
                    int32_t t_fit, int32_t has_constant);
/* CUDA-graph capture support.  A device-pointer call enqueued on a capturing stream records the library's kernels
 * into the caller's graph; the graph then holds raw pointers to the context's scratch and to the planned design.
 * mmf_pin_scratch(ctx, +1) after a capture makes every later call that would have to move that memory (a larger
 * batch, mmf_plan_design) fail with MMF_E_UNSUPPORTED instead of leaving the graph with dangling pointers;
 * mmf_pin_scratch(ctx, -1) when the graph is destroyed.  Counted: one +1 per live graph.
 * replaces: nothing in the reference (Spark re-launches a Python task per group, 02:523-528); it is the H100
 * answer to that per-task launch overhead for small batches.                                                   */
int mmf_pin_scratch(mmf_ctx* ctx, int32_t delta);
/* W [MMF_P*MMF_P] row-major (beta = W gamma), kept[MMF_P] 0/1; either may be NULL */
int mmf_get_whitening(mmf_ctx* ctx, double* W, int32_t* kept);

/* ---- the hot path -------------------------------------------------------
 * Fit every series on rows [0,t_fit) of the planned design and evaluate rows
 * [pred_start, pred_start+n_pred):
 *   holdout / drop-in mode : pred_start = 0,     n_pred = T      (Demand_Fitted for every date)
 *   future mode            : pred_start = t_fit, n_pred = horizon
 * y        [n, ld_y]   float32, host or device, NaN = missing
 * out_pred [n, ld_out] float32, host or device (same side as y not required)
 * out_beta [n, MMF_P]  nullable: coefficients on the raw X columns
 * out_status [n]       nullable
 * Device-pointer calls are enqueued on the ctx stream and return without
 * synchronising unless `stats` is non-NULL.  Host-pointer calls pipeline
 * H2D / kernel / D2H in chunks and return when the results are in host memory.
 * replaces: model.fit + predict + output assembly of build_tune_and_score_model
 * (02:435-494) for ALL groups of the applyInPandas fan-out (02:523-528).      */
int mmf_fit_forecast_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y,
                         int32_t pred_start, int32_t n_pred,
                         float* out_pred, int64_t ld_out,
                         float* out_beta, int32_t* out_status, mmf_stats* stats);

/* Same contract for an INTEGER series buffer y[n, ld_y] of element type `dtype` (MMF_DT_I16 / U16 / I32; ld_y in
 * elements; host or device).  The reference's demand is integer valued (01-data-generator.py:304) and an int16 /
 * uint16 value column halves the bytes that cross PCIe, which is what bounds the host-buffer path.  Chunks are
 * staged as they are, widened to float32 on the device (sentinel -> missing) and fit by the same kernels: the
 * results are bit-equal to mmf_fit_forecast_f32 on the float32 copy of the same values.
 * replaces: the same lines as mmf_fit_forecast_f32, for a Demand column that arrives as ShortType / IntegerType. */
int mmf_fit_forecast_int(mmf_ctx* ctx, const void* y, int32_t dtype, int64_t n, int64_t ld_y,
                         int32_t pred_start, int32_t n_pred,
                         float* out_pred, int64_t ld_out,
                         float* out_beta, int32_t* out_status, mmf_stats* stats);

/* ---- ragged batches: groups on MANY calendars in one launch ---------------------------------------------
 * The reference re-indexes every group on its own calendar (sort_values + asfreq per group, 02:422-423), so one
 * batch may hold groups with different first dates and lengths.  Planning and fitting them calendar by calendar
 * costs a launch sequence per distinct calendar; a ragged plan whitens all calendars in one host call and ONE pass
 * of the tensor-core kernel fits every group, each 128-row tile against its own calendar's design.
 *   X_all        the calendars' design matrices back to back: calendar c contributes n_rows[c] rows of p doubles
 *   t_fit[c]     fit rows of calendar c (33 .. 65535); rows [pred_start[c], pred_start[c] + n_pred[c]) are evaluated
 *   n_pred[c]    per calendar.  One common value <= 64 (future mode: pred_start[c] = t_fit[c], n_pred[c] = horizon): the fit
 *                kernel's own epilogue writes the forecasts.  Anything else (holdout, the reference's contract: pred_start[c]
 *                = 0, n_pred[c] = every date of calendar c, 02:484-494): the fit hands gamma / c to the tensor-core predict
 *                kernel, which writes each calendar's block of the table through that calendar's own tensor map.
 * mmf_fit_forecast_ragged_f32: y [n, ld_y] device, rows grouped by calendar: calendar c owns rows
 * [cal_row_start[c], cal_row_start[c+1]) (host array of n_cal + 1 entries, 0 .. n); columns >= t_fit[c] of a row
 * are ignored; out_pred [n, ld_out] device, ld_out >= the largest n_pred[c] (and a multiple of 4 when the predict kernel
 * writes it); columns from the next multiple of 4 behind a row's own n_pred[c] on are left untouched (TMA stores clip with 16-byte granularity).  Enqueues on the ctx stream and synchronises
 * once (rows the streaming pass leaves to the general pass are counted per calendar on the host).
 * replaces: the same reference lines as mmf_plan_design / mmf_fit_forecast_f32, for all calendars of a batch.   */
int mmf_plan_calendars(mmf_ctx* ctx, const double* X_all, int32_t n_cal, const int32_t* n_rows, const int32_t* t_fit,
                       const int32_t* pred_start, const int32_t* n_pred, int32_t p, int32_t has_constant);
int mmf_fit_forecast_ragged_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, const int64_t* cal_row_start,
                                float* out_pred, int64_t ld_out, int32_t* out_status, mmf_stats* stats);

/* ---- multi-GPU: fit + write the forecast rows into every GPU's copy of the table ----------
 * Same fit as above (device buffers only, enqueue-only), but each forecast row is stored to
 * n_out destinations in ONE kernel: out_ptrs[0] is this GPU's own slice, out_ptrs[1..] the same slice
 * of the peers' tables (peer-mapped pointers, NVLink P2P stores).  With multimem=1, n_out must be 1 and
 * out_ptrs[0] is an NVLS multicast address: the kernel issues multimem.st and the NVSwitch replicates the
 * store to every GPU.  The "single all-gather of the forecast table" (reference analogue: the shuffle
 * back from the per-group tasks, 02:523-528) thereby rides under the fit; the caller only needs a
 * cross-GPU barrier before reading peers' rows.                                                   */
int mmf_fit_forecast_bcast_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y,
                               int32_t pred_start, int32_t n_pred,
                               const uint64_t* out_ptrs, int32_t n_out, int32_t multimem, int64_t ld_out,
                               float* out_beta, int32_t* out_status);

/* ---- per-series model selection on the device ------------------------------------------------------
 * GPU analogue of the per-group hyperopt loop (02:435-469) + final refit/predict (02:472-488): the planned design
 * is fit on rows [0,t_fit); the candidates are the nested models made of the first candidates[k] whitened columns;
 * each is scored by its MSE over the held-out rows [t_fit, t_fit+n_hold) of y; the best one (first minimum) produces
 * out_pred for rows [pred_start, pred_start+n_pred).  Device buffers only, enqueue-only.
 * out_choice[n] (nullable): chosen number of columns; out_mse[n] (nullable): its hold-out MSE.                  */
int mmf_fit_select_forecast_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                                const int32_t* candidates, int32_t n_cand, int32_t pred_start, int32_t n_pred,
                                float* out_pred, int64_t ld_out, int32_t* out_choice, float* out_mse,
                                int32_t* out_status);

/* ---- device-side packer: long-format rows -> padded series on the GPU ------------------------------
 * replaces the hash shuffle of repartition(n_tasks,"Product","SKU") + groupBy (02:525-526) and the per-group
 * sort_values("Date") + set_index("Date").asfreq(freq) (02:422-423).  All pointers are DEVICE pointers holding
 * the Arrow column buffers as they are; rows may arrive in any order.
 *   hash_utf8 / hash_i32 : chain a utf8 (offsets+bytes) or dictionary-index key column into a 64-bit FNV-1a row
 *                          hash (first != 0 starts a new hash, 0 continues `hash`; first = 1 is the standard
 *                          FNV basis, first = 2, 3, ... other bases for a re-hash after a collision)
 *   group_codes          : dense group code per row (groups numbered in hash order), the first row of every
 *                          group (to read its key values back) and the number of groups (host int, synchronises)
 *   verify_utf8 / _i32   : adds to *mismatches (device uint64, caller zeroes it) the rows whose key differs from
 *                          the key of their group's first row, i.e. rows merged by a 64-bit hash collision
 *   minmax               : first / last day of every group
 *   scatter_f32          : y[row_of_group[g], (day - gstart[g]) / step] = value after a NaN fill; rows of groups with
 *                          row_of_group < 0 (other calendar buckets) and off-grid dates are skipped.  `duplicates`
 *                          (nullable device uint64, caller zeroes it) counts rows that landed on a (group, date)
 *                          cell another row had already written: the reference's asfreq raises on those (02:423)  */
int mmf_pack_hash_utf8(mmf_ctx* ctx, const int32_t* offsets, const uint8_t* data, int64_t n, uint64_t* hash,
                       int32_t first);
int mmf_pack_hash_i32(mmf_ctx* ctx, const int32_t* values, int64_t n, uint64_t* hash, int32_t first);
int mmf_pack_group_codes(mmf_ctx* ctx, const uint64_t* hash, int64_t n, int32_t* gid, int32_t* first_row,
                         int32_t* n_groups);
int mmf_pack_verify_utf8(mmf_ctx* ctx, const int32_t* offsets, const uint8_t* data, int64_t n, const int32_t* gid,
                         const int32_t* first_row, uint64_t* mismatches);
int mmf_pack_verify_i32(mmf_ctx* ctx, const int32_t* values, int64_t n, const int32_t* gid, const int32_t* first_row,
                        uint64_t* mismatches);
int mmf_pack_minmax(mmf_ctx* ctx, const int32_t* gid, const int32_t* day, int64_t n, int32_t n_groups,
                    int32_t* gmin, int32_t* gmax);
int mmf_pack_scatter_f32(mmf_ctx* ctx, const int32_t* gid, const int32_t* day, const float* val, int64_t n,
                         const int64_t* row_of_group, const int32_t* gstart, int32_t step, float* y, int64_t n_rows,
                         int64_t ld_y, int32_t t_len, uint64_t* duplicates);

/* ---- host memory helpers (Arrow buffers -> one cudaMemcpyAsync) ---------- */
int mmf_alloc_pinned(size_t bytes, void** out);
int mmf_free_pinned(void* p);
int mmf_host_register(void* p, size_t bytes);     /* pin an existing (Arrow/NumPy) buffer */
int mmf_host_unregister(void* p);

#ifdef __cplusplus
}
#endif
#endif /* MMF_H_ */
