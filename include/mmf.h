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

#define MMF_VERSION 117          /* 0.1.17 */
#define MMF_P 16                 /* design columns (zero-pad narrower designs) */
#define MMF_PIVOT_TOL 1e-3f      /* per-series relative Cholesky pivot threshold */
#define MMF_CAL_TOL 1e-10        /* aliasing threshold on the float64 calendar Gram */
#define MMF_SELECT_MAX_HOLD 3500 /* held-out rows mmf_fit_select_forecast_f32 accepts (64 B of shared memory each) */
#define MMF_BT_MAX_ORIGINS 8     /* backtest origins per call (mmf_plan_backtest) */
#define MMF_BT_NMETRIC 4         /* backtest metrics per (origin, series): MSE, MAE, bias, MAPE */
#define MMF_AR_MAX 8             /* largest AR order of mmf_fit_forecast_ar_f32 */
#define MMF_AR_KAPPA_MAX 0.999   /* Levinson-Durbin stops before a partial autocorrelation |kappa| >= this */
#define MMF_ARSEL_MAX_CAND 9     /* candidate AR orders per mmf_fit_select_ar_f32 call (0 .. MMF_AR_MAX) */
#define MMF_DIFF_MAX 2           /* largest differencing order of mmf_fit_forecast_arima_f32 */
#define MMF_MA_MAX 4             /* largest MA order of mmf_fit_forecast_arma_f32 */
#define MMF_HR_LONG_MAX 32       /* largest long AR order of the Hannan-Rissanen step 1 (one lag per lane of a warp) */
#define MMF_HR_PIVOT_TOL 1e-5    /* a Hannan-Rissanen Cholesky pivot must exceed this x its Gram diagonal */
#define MMF_ARMASEL_MAX_PQ 32    /* (p, q >= 1) candidate pairs per mmf_fit_select_arma_f32 call (one per lane of a warp) */
#define MMF_CSS_LAMBDA0 1e-3     /* mmf_fit_forecast_arma_css_f32: the Levenberg-Marquardt damping of the first step */
#define MMF_CSS_LAMBDA_MAX 1e10  /* ... a series stops (stalled) once its damping exceeds this */
#define MMF_CSS_RTOL 1e-6        /* ... and (converged) when an accepted pass lowers S by at most this x S */
#define MMF_CSS_ITER_DEFAULT 20  /* ... passes per series for max_iter = 0 */
#define MMF_CSS_ITER_MAX 64      /* ... the largest max_iter accepted */

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
  int32_t tc_variant;      /* tuning of the tensor-core kernel, same results whichever: 2 = the <6-stage, 2 staging tiles>
                              instantiation, any other value = the product (<8 stages, 1 staging tile>) */
  int64_t chunk_series;    /* host-buffer path: series per pipelined chunk (0 = library default) */
  void*   stream;          /* cudaStream_t to enqueue on (NULL = library-owned stream) */
  int32_t host_narrow;     /* host-buffer path: 0 = automatic, 1 = always try, 2 = never: narrow float32 chunks to
                              uint16 on host threads when every value is an integer in [0, 65534] (exactly, or the
                              chunk goes as float32), so that half the bytes cross PCIe; widened back on the device */
  int32_t host_threads;    /* threads of that narrowing pool (0 = half of the process's cores, at most 16) */
  int32_t stream_solve;    /* accepted and ignored: series with gaps are always solved in a pass of their own after
                              the tensor-core kernel */
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
/* Borrow a stream, e.g. torch's current one; NULL = the legacy default stream.  The context's calls share its counter
 * sets and scratch, so they must run on the device in the order they were made.  When `cuda_stream` differs from the
 * stream in use, the new stream waits (an event, no host synchronisation) for everything already enqueued on the old
 * one.  Setting the stream in use again costs nothing.  No wait is added while either stream is capturing: a capture
 * cannot order work outside it (torch.cuda.graph synchronises the device before it begins).  A borrowed stream must
 * stay valid until the next mmf_set_stream or mmf_destroy. */
int mmf_set_stream(mmf_ctx* ctx, void* cuda_stream);
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
 * A replay does not pass through mmf_set_stream, and every graph of a context shares one counter set and the scratch
 * with the eager calls: replay on the stream the context's calls use, or order it with them yourself.  Replays
 * running concurrently with each other, or with eager calls on another stream, are not supported.
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
 * Only columns [0, n_pred) of each out_pred row are written: columns [n_pred, ld_out) keep what the caller left
 * there, whatever the kernel (any ld_out >= n_pred and any base pointer; 16-B aligned tables with ld_out % 4 == 0
 * take the tensor-core store path, others the CUDA-core kernels).
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

/* The same fit with prediction standard errors for forecast intervals (DESIGN.md section 2 item 7).  For series i,
 * with n_obs its finite fit values, k the whitened columns its fit uses and S = sum over them of (y_t - c_i)^2:
 *   out_sigma[i] = sqrt(RSS / dof), RSS = S - b'gamma (clamped at 0), out_dof[i] = dof = n_obs - k;
 *                  NaN (and dof <= 0) when dof <= 0, in particular for empty series (status 1: dof = 0)
 *   out_se[i, j] = sigma_i * sqrt(1 + h_t), h_t = a_t' G_i^-1 a_t over the used columns, t = pred_start + j:
 *                  the least-squares standard error of a new observation at design row t (leverage included)
 * out_pred and out_status are bit-equal to mmf_fit_forecast_f32 on the same inputs.  out_se [n, ld_se] (ld_se >=
 * n_pred; only columns [0, n_pred) of a row are written), out_sigma [n], out_dof [n] are each nullable, but not all
 * three.  Device buffers only (host pointers: MMF_E_UNSUPPORTED); enqueue-only unless `stats` is non-NULL.  The
 * call always runs the product tensor-core configuration, whatever mmf_config.tc_variant says; mmf_config.kernel is
 * honoured.
 * replaces: the forecast variance / conf_int() the reference's per-group SARIMAX model offers beside the mean. */
int mmf_fit_forecast_se_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y,
                            int32_t pred_start, int32_t n_pred,
                            float* out_pred, int64_t ld_out,
                            float* out_se, int64_t ld_se,
                            float* out_sigma, int32_t* out_dof,
                            int32_t* out_status, mmf_stats* stats);

/* Regression with AR(p) errors (DESIGN.md section 2 item 9): the plain fit (gamma, c, kept columns and out_status bit-equal
 * to mmf_fit_forecast_f32 on the same inputs), then per series, from the residuals e_t = y_t - c - a_t.gamma of the observed
 * fit rows:
 *   r_k = (1/n_obs) sum e_t e_{t-k} over the pairs with both rows observed (k = 0..ar_order, float64, not demeaned);
 *   order p_i = 0 when dof = n_obs - used columns <= ar_order, else the last order float64 Levinson-Durbin completes
 *   before r_0 <= 0 or |kappa_j| >= MMF_AR_KAPPA_MAX; phi_1..phi_{p_i} Yule-Walker, sigma_eps^2 = r_0 prod (1 - kappa_j^2);
 *   filled residuals u_s = e_s (observed) or sum_j phi_j u_{s-j} (missing, and every s >= t_fit), u_s = 0 for s < 0;
 *   out_pred[i, t - pred_start] = c + a_t.gamma + sum_j phi_j u_{t-j}: one-step-ahead in sample, the dynamic forecast
 *   from origin t_fit beyond it.  y is never read at or beyond t_fit.
 * A row's prediction does not depend on the requested window, to the bit: the recursion may restart at the latest row
 * s <= min(pred_start, t_fit) whose p predecessors are all observed (their u are plain residuals), and that restart
 * changes no bit of any requested row.
 * 1 <= ar_order <= MMF_AR_MAX.  out_phi [n][MMF_AR_MAX] (zero beyond the series' order), out_order [n] and out_sigma [n]
 * (sqrt(sigma_eps^2)) are nullable; empty series (status 1) get order 0, phi 0, sigma NaN and NaN predictions.  Device
 * buffers only (host pointers: MMF_E_UNSUPPORTED); any ld_out >= n_pred and any base pointer, only columns [0, n_pred)
 * written; enqueue-only unless `stats` is non-NULL; mmf_config.kernel and assume_finite are honoured.  Refused arguments
 * write nothing.  The kernel rule of every ARIMA-family call: each fit the call runs picks its kernel by the buffer it
 * reads.  A fit of y itself (d = 0) needs a 16-B aligned y with ld_y % 4 == 0 for the tensor-core kernel; otherwise
 * MMF_KERNEL_AUTO runs the warp kernel and MMF_KERNEL_TC refuses the call (MMF_E_UNSUPPORTED, "tensor-core kernel not
 * applicable", nothing written).  A fit of z' (d >= 1) reads the context's 16-B-pitch scratch, so it runs the
 * tensor-core kernel under AUTO and TC whatever y's layout.  A selection that lists d = 0 and d >= 1 on such a y thus
 * mixes the kernels under AUTO, and stats->n_pending counts the rows of its tensor-core fits only.
 * replaces: SARIMAX(p, 0, 0) + exog fit and predict of the reference's per-group model (02:441-450, 472-488 with p > 0),
 * for a caller-fixed order and the two-step (OLS, then Yule-Walker on the residuals) estimator. */
int mmf_fit_forecast_ar_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                            int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                            float* out_phi, int32_t* out_order, float* out_sigma,
                            int32_t* out_status, mmf_stats* stats);

/* Regression with AR(p) errors, the order p chosen per series by hold-out MSE (DESIGN.md section 2 item 10).  The fit rows
 * are [0, t_fit) of the planned design, the held-out rows [t_fit, t_fit + n_hold) of the design and of y.
 *   candidate m >= 1 is mmf_fit_forecast_ar_f32 with ar_order = m (the same residuals, r_k, dof rule, Levinson-Durbin,
 *   phi, sigma and fill); candidate 0 is the plain regression c + a_t.gamma (phi 0, order 0, sigma = sqrt(r_0));
 *   score of m: the MSE of the dynamic forecast from origin t_fit over the held-out rows (the predictions of
 *   mmf_fit_forecast_ar_f32(ar_order = m, pred_start = t_fit, n_pred = n_hold)) against y[t_fit, t_fit + n_hold), over
 *   the points where both are finite, summed in float64, stored as float32, NaN where no point is scored.  Held-out y
 *   never enters the recursion: the score is multi-step, not one-step-ahead;
 *   choice: the first minimum of the float64 MSE in list order (equal models go to the smaller order); the last listed
 *   candidate when no point is scored.
 * out_pred[i, t - pred_start] is then the prediction of the chosen candidate: bit-equal to mmf_fit_forecast_ar_f32
 * (ar_order = choice) for choice >= 1 (pred, phi, order, sigma, status), c + a_t.gamma for choice 0.  y is read on
 * [0, t_fit + n_hold) only; held-out values reach the output only through the choice.
 * orders [n_orders] is a host array of 1 .. MMF_ARSEL_MAX_CAND ascending distinct orders in [0, MMF_AR_MAX];
 * 1 <= n_hold, t_fit + n_hold <= the planned rows, ld_y >= t_fit + n_hold.  out_choice [n] (the chosen order, -1 for
 * empty series), out_mse [n] (its hold-out MSE), out_cand_mse [n][n_orders] (every candidate's), out_phi [n][MMF_AR_MAX],
 * out_order [n] (the effective order, <= the choice), out_sigma [n] and out_status [n] are nullable.  Empty series
 * (status 1) get choice -1, order 0, phi 0 and NaN sigma, MSEs and predictions.  Otherwise the contract of
 * mmf_fit_forecast_ar_f32: device buffers only, any ld_out >= n_pred and any base pointer, enqueue-only unless `stats`
 * is non-NULL, mmf_config.kernel and assume_finite honoured, refused arguments write nothing.
 * replaces: the reference's per-group tuning loop over p (02:435-488: SARIMAX candidates fit on the train rows, scored by
 * the MSE of their forecast over the last FORECAST_HORIZON rows, 02:453-459, the best order refit and predicted,
 * 02:472-488) as an exhaustive search over p with d = q = 0, not TPE over (p, d, q). */
int mmf_fit_select_ar_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                          const int32_t* orders, int32_t n_orders, int32_t pred_start, int32_t n_pred,
                          float* out_pred, int64_t ld_out,
                          int32_t* out_choice, float* out_mse, float* out_cand_mse,
                          float* out_phi, int32_t* out_order, float* out_sigma,
                          int32_t* out_status, mmf_stats* stats);

/* ---- regression with ARIMA(p, d, 0) errors (DESIGN.md section 2 item 11) ----------------------------------------------
 * mmf_plan_arima: X [n_rows, p] float64 as for mmf_plan_design, 1 <= max_diff <= MMF_DIFF_MAX, t_fit - max_diff >= 1.
 * For d = 1 .. max_diff it plans the differenced design D_d, row s = Delta^d x_{s+d} (float64, s in [0, n_rows - d)), as
 * mmf_plan_design(D_d, n_rows - d, p, t_fit - d, has_constant = 0) would: a differenced column whose largest |value| on
 * the fit rows is at most 1e-12 x the largest |value| of the raw column there is set to 0 first (cancellation residue).
 * A plan of its own: the mmf_plan_design, mmf_plan_calendars and mmf_plan_backtest plans stay in force.  Every argument
 * is checked before the previous ARIMA plan is freed, so a refused plan keeps it.
 * mmf_fit_forecast_arima_f32: for series i and d = diff_order (1 <= d <= the planned max_diff), 0 <= ar_order <= MMF_AR_MAX:
 *   z_t = y_t - y_{t-1} (d = 1) or (y_t - y_{t-1}) - (y_{t-1} - y_{t-2}) (d = 2) in that fp32 order, for d <= t < t_fit,
 *   missing when any of y_{t-d} .. y_t is; z'_s = z_{s+d};
 *   zhat_t: mmf_fit_forecast_ar_f32(ar_order) on z' with the plan D_d (ar_order = 0: the plain fit, phi 0, sigma =
 *   sqrt(r_0)), the prediction of z'_{t-d}: one step ahead in sample, the dynamic forecast from t_fit beyond it;
 *   levels: ytilde_s = y_s for s < t_fit with y_s finite, else yhat_s (NaN for s < d);
 *   yhat_t = zhat_t + ytilde_{t-1} (d = 1), yhat_t = (zhat_t + 2 ytilde_{t-1}) - ytilde_{t-2} (d = 2), each sum rounded
 *   once in fp32 in that order (2 ytilde_{t-1} is exact); yhat_t = NaN for t < d.
 * out_pred[i, t - pred_start] = yhat_t for the rows [pred_start, pred_start + n_pred) of the planned design: one step
 * ahead in sample, the integrated dynamic forecast beyond t_fit.  y is read on [0, t_fit) only.  A missing fit value
 * is replaced by its prediction, so later rows integrate from the filled level; a missing value before the first
 * observed one makes the predictions NaN until an observed level restarts the chain.  A row's prediction does not
 * depend on the requested window, to the bit: the recursion may restart at the latest z' row s <= min(pred_start,
 * t_fit) - d whose max(p, 1) predecessors in z' are all observed (so are the levels the integration of row s + d reads),
 * and that restart changes no bit of any requested row.
 * out_phi [n][MMF_AR_MAX], out_order [n], out_sigma [n] are those of the AR part on z'; out_status [n] is the status of
 * the fit on z' (1 when z' has no observed fit row: NaN predictions, order 0, phi 0, sigma NaN).  All nullable except
 * out_pred.  Otherwise the contract of mmf_fit_forecast_ar_f32: device buffers only, any ld_out >= n_pred and any base
 * pointer with only columns [0, n_pred) written, enqueue-only unless `stats` is non-NULL, mmf_config.kernel and
 * assume_finite honoured, refused arguments write nothing.  Scratch: one slab of rows x round4(t_fit - d) floats for z'.
 * replaces: SARIMAX(p, d, 0) + exog fit and predict of the reference's per-group model (02:441-450, 472-488 with d > 0),
 * for caller-fixed orders and the two-step estimator on the differenced series. */
int mmf_plan_arima(mmf_ctx* ctx, const double* X, int32_t n_rows, int32_t p, int32_t t_fit, int32_t max_diff);
int mmf_fit_forecast_arima_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                               int32_t diff_order, int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                               float* out_phi, int32_t* out_order, float* out_sigma, int32_t* out_status,
                               mmf_stats* stats);

/* ---- regression with ARIMA(p, d, q) errors (DESIGN.md section 2 item 13) ------------------------------------------------
 * mmf_fit_forecast_arma_f32: for series i, 0 <= ar_order = p <= MMF_AR_MAX, 1 <= ma_order = q <= MMF_MA_MAX and
 * 0 <= diff_order = d <= MMF_DIFF_MAX (d = 0 needs the mmf_plan_design plan; d >= 1 the mmf_plan_arima plan with
 * max_diff >= d; missing: MMF_E_NOPLAN, max_diff too small: MMF_E_INVALID).  The series modelled is y (d = 0) or z' of
 * mmf_fit_forecast_arima_f32 (d >= 1); e_t is the residual of its plain fit on the observed fit rows t < T = t_fit - d
 * (0 elsewhere), and the status is that fit's.  Hannan-Rissanen, no likelihood optimisation and no re-estimation of beta
 * (it is not SARIMAX's Kalman-filter MLE):
 *   long order m = long_order (max(p, q) <= m <= MMF_HR_LONG_MAX), or for long_order = 0
 *   min(MMF_HR_LONG_MAX, max(2 max(p, q), floor(ln(T)^2)));
 *   step 1: mmf_fit_forecast_ar_f32's estimator with order m (r_0..r_m over n_obs, the dof rule, Levinson-Durbin with the
 *   kappa stop) gives psi and the completed order m_i; the filled long-AR residuals u^L (e on observed fit rows, the AR
 *   prediction sum_j psi_j u^L_{s-j} elsewhere, 0 before row 0) give eps^_s = e_s - sum_{j<=m_i} psi_j u^L_{s-j} on the
 *   observed fit rows;
 *   step 2: the rows R = { t in [m + q, T) : e observed at t, t-1, .., t-max(p, q) } regress e_t on (e_{t-1..t-p},
 *   eps^_{t-1..t-q}) by float64 normal equations and an in-order Cholesky: (phi_1..phi_p, theta_1..theta_q), with the
 *   sign convention u_t = sum phi_j u_{t-j} + eps_t + sum theta_j eps_{t-j};
 *   gate: m_i >= 1, |R| > p + q, every Cholesky pivot > MMF_HR_PIVOT_TOL x its Gram diagonal, and the step-down recursion
 *   of 1 - sum phi_j z^j and of 1 + sum theta_j z^j gives every |kappa| < MMF_AR_KAPPA_MAX (stationary AR part,
 *   invertible MA part);
 *   fallback: a series that fails the gate gets, bit for bit, mmf_fit_forecast_ar_f32(p) (d = 0, p >= 1), the plain
 *   regression of mmf_fit_select_ar_f32 with orders (0) (d = 0, p = 0) or mmf_fit_forecast_arima_f32(p, d) (d >= 1) in
 *   out_pred, out_phi, out_order, out_sigma and out_status, with ma_order 0 and theta 0;
 *   forecast (gated series): from s = 0, with u_s = eps~_s = 0 for s < 0, pr_s = sum phi_j u_{s-j} + sum theta_j eps~_{s-j};
 *   on an observed fit row u_s = e_s and eps~_s = e_s - pr_s, elsewhere u_s = pr_s and eps~_s = 0.  The prediction is
 *   c + a_s.gamma + pr_s, for d >= 1 integrated to levels as mmf_fit_forecast_arima_f32 does (NaN for t < d).
 *   sigma = sqrt(mean of eps~_t^2 over R); order = p, ma_order = q.
 * out_pred[i, t - pred_start]: one step ahead in sample, the dynamic forecast from t_fit beyond it; y is read on
 * [0, t_fit) only.  The recursion never restarts: a row's prediction does not depend on the requested window.
 * out_phi [n][MMF_AR_MAX], out_theta [n][MMF_MA_MAX], out_order [n], out_ma_order [n], out_sigma [n], out_status [n] are
 * nullable (empty series: status 1, NaN predictions and sigma, orders 0, phi and theta 0).  Otherwise the contract of
 * mmf_fit_forecast_arima_f32: device buffers only, any ld_out >= n_pred and any base pointer with only columns
 * [0, n_pred) written, enqueue-only unless `stats` is non-NULL, mmf_config.kernel and assume_finite honoured, refused
 * arguments write nothing.
 * replaces: SARIMAX(p, d, q) + exog fit and predict of the reference's per-group model (02:441-450, 472-488 with q > 0),
 * e.g. its order (1, 2, 1) (02:226-229), for caller-fixed orders. */
int mmf_fit_forecast_arma_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                              int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t pred_start,
                              int32_t n_pred, float* out_pred, int64_t ld_out, float* out_phi, float* out_theta,
                              int32_t* out_order, int32_t* out_ma_order, float* out_sigma, int32_t* out_status,
                              mmf_stats* stats);

/* ---- ARIMA(p, d, q) errors by conditional least squares (DESIGN.md section 2 item 16) ---------------------------------
 * mmf_fit_forecast_arma_css_f32: mmf_fit_forecast_arma_f32, then Levenberg-Marquardt refinement of every gated series'
 * (phi, theta) on the conditional sum of squares (R's arima(method = "CSS") conditioning, with the gap rule above):
 *   S(x) = sum over C = { s in [p, T) : e observed at s } of eps~_s(x)^2, eps~ the forecast recursion of
 *   mmf_fit_forecast_arma_f32 from s = 0 (zero pre-sample, missing rows filled), evaluated in float64 from the fp32
 *   residuals e; the Jacobian d eps~ / dx is exact, gaps included (a filled value depends on x);
 *   start: x0 = the (phi, theta) the HR call ships (fp32).  One pass over the fit window evaluates S, g = J' eps~ and
 *   H = J'J at an fp32 point (float64 sums); the first pass is at x0;
 *   step: (H + lambda diag H) delta = -g by an in-order float64 Cholesky, lambda starting at MMF_CSS_LAMBDA0; the trial
 *   point is x' = fp32(x + delta).  A pivot <= MMF_HR_PIVOT_TOL x its diagonal, or an x' whose 1 - sum phi_j z^j or
 *   1 + sum theta_j z^j fails the HR gate's step-down test, sets lambda <- 10 lambda and solves again (no pass);
 *   accept: the next pass evaluates S(x'); S(x') < S(x) accepts x' (lambda <- lambda / 10, H and g of x'), otherwise
 *   lambda <- 10 lambda with H and g kept;
 *   stop (out_css_stop): 1 converged (an accepted pass lowered S by <= MMF_CSS_RTOL x S), 2 stalled (lambda >
 *   MMF_CSS_LAMBDA_MAX), 3 budget (max_iter passes run; max_iter = 0: MMF_CSS_ITER_DEFAULT, at most MMF_CSS_ITER_MAX).
 *   So S(shipped) <= S(x0) for every gated series.
 * Outputs: a series that accepted no step keeps the HR call's pred, phi, theta, order, ma_order and status bit for bit;
 * one that did gets the recursion and level integration of the HR call with the shipped (phi, theta).  For every gated
 * series sigma = sqrt(S / |C|) at the shipped point (the conditional MLE).  Series that fail the HR gate and empty
 * series get the HR call's outputs bit for bit.  out_css_start [n] (S(x0)), out_css [n] (S shipped), out_css_stop [n]
 * and out_iters [n] (passes run) are nullable; NaN, NaN, 0, 0 for fallback and empty series.  beta is not re-estimated;
 * this is not the exact (Kalman) likelihood (mmf_fit_forecast_arma_ml_f32 refines this call's estimate to it).  Otherwise the contract of mmf_fit_forecast_arma_f32 (plans, device buffers
 * only, any ld_out, enqueue-only unless `stats` is non-NULL, mmf_config.kernel and assume_finite honoured, refused
 * arguments write nothing); max_iter outside [0, MMF_CSS_ITER_MAX] is MMF_E_INVALID.  Scratch: per slab, 52 B per row
 * when out_phi, out_theta or out_ma_order is NULL.
 * replaces: SARIMAX(p, d, q) + exog fit of the reference's per-group model (02:441-450, 472-481) by likelihood
 * optimisation, with the conditional likelihood in place of the exact one. */
int mmf_fit_forecast_arma_css_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                                  int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t max_iter,
                                  int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out, float* out_phi,
                                  float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                                  int32_t* out_status, float* out_css_start, float* out_css, int32_t* out_css_stop,
                                  int32_t* out_iters, mmf_stats* stats);

/* ---- ARIMA(p, d, q) errors with beta estimated jointly (DESIGN.md section 2 item 17) ---------------------------------
 * mmf_fit_forecast_arma_joint_f32: mmf_fit_forecast_arma_css_f32 with the regression coefficients added to the
 * parameter vector (R's arima(xreg =, method = "CSS")): x = (phi_1..phi_p, theta_1..theta_q, gamma_j for j in J), J the
 * series' used columns of the dof rule (kept by the plan, non-zero on an observed fit row, not dropped for the series'
 * mask), gamma the whitened coefficients of the plan the call fits (mmf_plan_design's for d = 0, D_d's for d >= 1), c
 * (the fit's centring constant, 0 for d >= 1) held fixed.  The residual of a pass is e_s = z'_s - (c + a_s . gamma) in
 * fp32 at the pass's gamma; S, the gap rule, the exact Jacobian (the gamma columns through the same recursion: d u~_s =
 * -a_{s,j} and d eps~_s = -a_{s,j} - d pr_s on an observed row, d u~_s = d pr_s and d eps~_s = 0 on a missing one), the
 * step, its constants and the stops are the CSS call's, on the (n_x + 1)-square system, n_x = p + q + |J| <= 28; the
 * step-down tests apply to (phi, theta) only.  Start: x0 = (the HR (phi, theta), the fit's gamma on J), so out_css_start
 * is the CSS call's bit for bit.
 * Outputs: as mmf_fit_forecast_arma_css_f32's, a series that accepted a step getting the recursion at the shipped
 * (gamma, phi, theta): c + a_s . gamma + pr_s, integrated to levels for d >= 1.  out_beta [n][MMF_P] (nullable) = W gamma
 * (+ c on the intercept when the plan has a constant) of the gamma each series ships, in the fp32 order of
 * mmf_fit_forecast_f32's out_beta (so a d = 0 series that kept the fit's gamma gets its out_beta bit for bit); for d >= 1
 * the coefficients of Delta^d X.  NaN for empty series.  With J empty every output is mmf_fit_forecast_arma_css_f32's bit
 * for bit.  Otherwise the contract of mmf_fit_forecast_arma_css_f32 (plans, refusals, device buffers only, scratch).
 * replaces: SARIMAX(p, d, q) + exog fit with the exog coefficients estimated jointly (02:441-450, 472-481), by the
 * conditional likelihood. */
int mmf_fit_forecast_arma_joint_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                                    int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t max_iter,
                                    int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out, float* out_beta,
                                    float* out_phi, float* out_theta, int32_t* out_order, int32_t* out_ma_order,
                                    float* out_sigma, int32_t* out_status, float* out_css_start, float* out_css,
                                    int32_t* out_css_stop, int32_t* out_iters, mmf_stats* stats);

/* ---- ARIMA(p, d, q) errors by exact Gaussian likelihood (DESIGN.md section 2 item 19) ---------------------------------
 * mmf_fit_forecast_arma_ml_f32: mmf_fit_forecast_arma_css_f32 with the same arguments and max_iter, then
 * Levenberg-Marquardt refinement of every gated series' (phi, theta) on the exact Gaussian likelihood of its residuals
 * (R's arima(method = "CSS-ML") on the differenced series):
 *   model: e_s, s < T, the residual the CSS call models (y for d = 0, z' for d >= 1; beta not re-estimated) is a zero-mean
 *   ARMA(p, q) in Harvey's state-space form: r = max(p, q + 1), T with phi in its first column and I on its
 *   superdiagonal, R = (1, theta_1 .. theta_{r-1})', Z = (1, 0 .. 0), no observation noise, sigma^2 concentrated out;
 *   start of the filter: a = 0 and P_{0|-1} the stationary state covariance, vec P = (I - T (x) T)^-1 vec(R R'), solved in
 *   float64 on the r (r + 1) / 2 symmetric unknowns by Gaussian elimination with partial pivoting; a pivot |u_kk| <=
 *   MMF_HR_PIVOT_TOL x max |A| fails the solve.  This is Gardner's start on the differenced series, not SARIMAX's
 *   approximate-diffuse start over the levels;
 *   filter over s in [0, T) in float64 from the fp32 residuals: on an observed row v_s = e_s - a_1, F_s = P_11, K = T P Z'
 *   / F_s, a <- T a + K v_s, P <- T P T' + R R' - K K' F_s; on a missing row a <- T a, P <- T P T' + R R' (no steady-state
 *   shortcut).  With n the number of observed rows (none conditioned on), S_w = sum v_s^2 / F_s:
 *   L = n log(S_w / n) + sum log F_s, loglik = -(L + n (1 + log 2 pi)) / 2, sigma = sqrt(S_w / n);
 *   optimiser: the CSS call's Levenberg-Marquardt (start, step, constants, accept, stops) on the scaled innovations r_s =
 *   G v_s / sqrt(F_s), G = exp(sum log F_s / (2 n)), so that sum r_s^2 = G^2 S_w = n exp(L / n) is the objective and
 *   MMF_CSS_RTOL applies to it.  The Jacobian is exact (forward-mode derivatives of a, P, K and P_0); G enters H and g
 *   as a rank-2 correction.  The first pass is at x0 = the (phi, theta) the CSS call ships; a trial point whose P_0
 *   solve fails counts as one that fails the step-down test (lambda <- 10 lambda, no pass).
 * Outputs: a gated series that accepted no step keeps the CSS call's pred, phi, theta, order, ma_order and status bit for
 * bit; one that did gets the recursion and level integration of the HR call with the shipped (phi, theta) (the library's
 * predictor, not the Kalman filter's, so mmf_arima_se_f32 applies unchanged; mmf_fit_forecast_arma_ml_kf_f32 predicts with
 * the filter).  For every gated series sigma = sigma at
 * the shipped point.  out_loglik_start [n] (loglik at x0), out_loglik [n] (at the shipped point, >= out_loglik_start),
 * out_ml_stop [n] (the CSS call's codes, 0 not refined) and out_iters [n] (passes run) are nullable.  A gated series whose
 * x0 fails the P_0 solve keeps every CSS output, with NaN, NaN, 0, 0.  Series that fail the HR gate and empty series get
 * the HR call's outputs and NaN, NaN, 0, 0.  Otherwise the contract of mmf_fit_forecast_arma_css_f32 (plans, refusals
 * with max_iter checked first, device buffers only, any ld_out, enqueue-only unless `stats`, mmf_config.kernel and
 * assume_finite, scratch).
 * replaces: SARIMAX(p, d, q) + exog fit of the reference's per-group model (02:441-450, 472-481), which maximises the
 * exact likelihood. */
int mmf_fit_forecast_arma_ml_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                                 int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t max_iter,
                                 int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out, float* out_phi,
                                 float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                                 int32_t* out_status, float* out_loglik_start, float* out_loglik, int32_t* out_ml_stop,
                                 int32_t* out_iters, mmf_stats* stats);

/* ---- the Kalman predictor of the exact-likelihood fit (DESIGN.md section 2 item 20) -----------------------------------
 * mmf_fit_forecast_arma_ml_kf_f32: mmf_fit_forecast_arma_ml_f32 with the same arguments, then the predictions of every
 * covered series (a gated series whose P_0 solves at the shipped (phi, theta), including one that accepted no ML step)
 * from the Kalman filter of that call's model, evaluated in float64 at the shipped fp32 (phi, theta):
 *   e: a_s the filter's predicted state of z-row s (the residual of y for d = 0, of z' for d >= 1), from a = 0 and P_0;
 *   for s < T it uses the observed rows before s only (a missing row predicted and not updated, as in the likelihood),
 *   for s >= T it is the dynamic forecast a_{T+h} = T^h a_T.  The prediction of e_s is a_{s,1};
 *   levels: zhat_s = fitted_s + a_{s,1} (fp32), integrated to levels as mmf_fit_forecast_arma_f32 integrates its zhat
 *   (a missing level filled with its prediction).  This is the ML call's pred with the recursion's prediction replaced;
 *   out_se [n, ld_se] (nullable; ld_se >= n_pred): se_t = sigma sqrt(Var(y_t - yhat_t)) with the fitted model taken as
 *   true and no estimation uncertainty (mmf_arima_se_f32's definition applied to this predictor).  The error state is
 *   (alpha_s - a_s, the errors of the d previous filled levels); its alpha block is the filter's P, and its full
 *   covariance moves with the filter (alpha - a <- (T - K Z)(alpha - a) + R eps on an update, T (alpha - a) + R eps on a
 *   missing row; the level error of row t is Z (alpha_s - a_s) plus the integration of the previous level errors, 0
 *   where y_t is observed).  On a gap-free fit window se = sigma sqrt(F_s) in sample.  NaN where mmf_arima_se_f32 gives
 *   NaN (rows t < d, a level chain without an anchor), +Inf where the float64 variance overflowed.
 * Every other output (phi, theta, order, ma_order, sigma, status, loglik_start, loglik, ml_stop, iters) is the ML call's
 * bit for bit on every row.  Series the predictor does not cover (HR-gate fallbacks, empty series, a P_0 that fails at
 * the shipped point) keep every output of the ML call bit for bit, and their out_se is mmf_arima_se_f32 of the call's
 * outputs bit for bit.  Otherwise the contract of mmf_fit_forecast_arma_ml_f32 (plans, refusals with max_iter checked
 * first, device buffers only, any ld_out, enqueue-only unless `stats`, mmf_config.kernel and assume_finite); ld_se <
 * n_pred with out_se given is MMF_E_INVALID.  Scratch: per slab, 60 B per row when out_se is given and out_phi,
 * out_theta, out_order, out_ma_order or out_sigma is NULL (52 B as the CSS call otherwise).
 * replaces: SARIMAX predict() / get_forecast() of the reference's fitted per-group model (02:453-457, 484-488): the
 * Kalman filter's one-step predictions in sample, its dynamic forecast beyond, and their standard errors. */
int mmf_fit_forecast_arma_ml_kf_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t ar_order,
                                    int32_t diff_order, int32_t ma_order, int32_t long_order, int32_t max_iter,
                                    int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out, float* out_phi,
                                    float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                                    int32_t* out_status, float* out_loglik_start, float* out_loglik,
                                    int32_t* out_ml_stop, int32_t* out_iters, float* out_se, int64_t ld_se,
                                    mmf_stats* stats);

/* ---- (p, d) selection by hold-out MSE on levels (DESIGN.md section 2 item 12) -----------------------------------------
 * mmf_fit_select_arima_f32: orders [n_orders] (1 .. MMF_ARSEL_MAX_CAND ascending distinct values in [0, MMF_AR_MAX]) and
 * diffs [n_diffs] (1 .. MMF_DIFF_MAX + 1 ascending distinct values in [0, MMF_DIFF_MAX]) are host arrays; the candidates
 * are every pair (p, d) in d-major list order (d ascending, then p ascending).  Fit rows [0, t_fit), held-out rows
 * [t_fit, t_fit + n_hold) of the level design and of y.
 *   candidate (p, 0) is candidate p of mmf_fit_select_ar_f32 (the plain regression for p = 0, AR(p) on y otherwise, with
 *   the mmf_plan_design plan); candidate (p, d >= 1) is mmf_fit_forecast_arima_f32(ar_order = p, diff_order = d) with
 *   the mmf_plan_arima plan;
 *   score: the MSE on levels of the candidate's dynamic forecast from origin t_fit over the held-out rows (the predictions
 *   of its single call with pred_start = t_fit, n_pred = n_hold) against y[t_fit, t_fit + n_hold), over the points
 *   where both are finite, summed in float64, stored as float32, NaN where no point is scored.  Held-out y never enters
 *   a z-space history or a level chain;
 *   eligible: the fit the candidate builds on (on y for d = 0, on z' of its d otherwise) is not empty;
 *   choice: the first minimum of the float64 MSE over the eligible candidates in list order (ties go to the smaller d,
 *   then the smaller p); the last eligible candidate when none scores a point; (-1, -1) when none is eligible.
 * out_pred[i, t - pred_start] is the prediction of the chosen candidate, bit-equal to its single call (pred, phi, order,
 * sigma, status): mmf_fit_select_ar_f32 with orders (p) for d = 0, mmf_fit_forecast_arima_f32(p, d) otherwise (NaN on
 * the rows t < d).  For d >= 1 the status is that of the fit on z'.  With diffs = (0) the call is mmf_fit_select_ar_f32.
 * A row with no eligible candidate gets choice (-1, -1), status 1, order 0, phi 0 and NaN sigma, MSEs and predictions.
 * y is read on [0, t_fit + n_hold) only.  out_choice_p [n], out_choice_d [n], out_mse [n] (the winner's MSE),
 * out_cand_mse [n][n_diffs][n_orders], out_phi [n][MMF_AR_MAX], out_order [n], out_sigma [n], out_status [n] are
 * nullable.
 * Plans: a listed d = 0 needs the mmf_plan_design plan, a listed d >= 1 the mmf_plan_arima plan with max_diff >= max(diffs)
 * (missing: MMF_E_NOPLAN; max_diff too small: MMF_E_INVALID).  A call that uses both needs them built from the same X (the
 * same rows, columns, t_fit and bytes; otherwise MMF_E_INVALID).  1 <= n_hold, t_fit + n_hold <= the planned rows,
 * ld_y >= t_fit + n_hold.  Otherwise the contract of mmf_fit_select_ar_f32: device buffers only, any ld_out >= n_pred and
 * any base pointer with only columns [0, n_pred) written, enqueue-only unless `stats` is non-NULL (n_pending sums the
 * fits of every listed d), mmf_config.kernel and assume_finite honoured, refused arguments write nothing.  Scratch: per
 * slab, z' as mmf_fit_forecast_arima_f32, 20 B per row.
 * replaces: the reference's per-group tuning loop over p and d (02:435-488, search space 02:461-465) as an exhaustive
 * search over (p, d) with q = 0; mmf_fit_select_arma_f32 adds q. */
int mmf_fit_select_arima_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                             const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                             int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                             int32_t* out_choice_p, int32_t* out_choice_d, float* out_mse,
                             float* out_cand_mse /* [n][n_diffs][n_orders] */, float* out_phi, int32_t* out_order,
                             float* out_sigma, int32_t* out_status, mmf_stats* stats);

/* ---- (p, d, q) selection by hold-out MSE on levels (DESIGN.md section 2 item 14) -----------------------------------------
 * mmf_fit_select_arma_f32: the arguments of mmf_fit_select_arima_f32, and mas [n_mas] (a host array of 1 .. MMF_MA_MAX + 1
 * ascending distinct values in [0, MMF_MA_MAX], mas[0] = 0) and long_order.  The candidates are every triple (p, d, q),
 * in list order d ascending, then q ascending, then p ascending: for each d the q = 0 block comes first and is
 * mmf_fit_select_arima_f32's candidates.  At most MMF_ARMASEL_MAX_PQ pairs (p, q >= 1), n_orders x (n_mas - 1).
 *   candidate (p, d, 0) is mmf_fit_select_arima_f32's candidate (p, d), its score bit-equal to that call's cand_mse;
 *   candidate (p, d, q >= 1) is mmf_fit_forecast_arma_f32(p, d, q, long_order = m_d), with one long order per d and call:
 *   m_d = long_order (max(orders, mas) <= long_order <= MMF_HR_LONG_MAX), or for long_order = 0
 *   min(MMF_HR_LONG_MAX, max(2 max(orders, mas), floor(ln(t_fit - d)^2))).  This is the single call's default whenever
 *   t_fit - d >= 55 (floor(ln(t_fit - d)^2) >= 16 >= 2 max(p, q) then); below that it may be a larger m.  A candidate that
 *   fails the Hannan-Rissanen gate forecasts as (p, d, 0), so its score is (p, d, 0)'s bit for bit and, (p, d, 0) coming
 *   first, it never wins;
 *   score, eligibility and choice are mmf_fit_select_arima_f32's: the MSE on levels of the dynamic forecast from t_fit over
 *   the held-out rows, summed in float64; eligible when the fit the candidate builds on is not empty; the first minimum
 *   over the eligible candidates in list order.  A q >= 1 candidate wins only with a scored point: with none anywhere the
 *   choice is mmf_fit_select_arima_f32's (the last eligible q = 0 candidate); (-1, -1, -1) when none is eligible.
 * Outputs: a winner with q >= 1 gets its single call's pred, phi, theta, order, ma_order, sigma and status bit for bit; a
 * winner with q = 0 gets mmf_fit_select_arima_f32's outputs bit for bit, with theta 0, ma_order 0 and choice_q 0.  With
 * mas = (0) the call is mmf_fit_select_arima_f32 in every shared output.  y is read on [0, t_fit + n_hold) only, and
 * held-out y enters no recursion and no level chain.  out_choice_q [n], out_theta [n][MMF_MA_MAX], out_ma_order [n] and
 * out_cand_mse [n][n_diffs][n_mas][n_orders] are nullable, as is every output of mmf_fit_select_arima_f32 but out_pred.
 * Otherwise the contract of mmf_fit_select_arima_f32 (plans, device buffers, ld_out, enqueue-only unless `stats`, refused
 * arguments write nothing).  Scratch: per slab, that of mmf_fit_select_arima_f32 and 4 B per row and candidate (p, d, 0).
 * replaces: the reference's per-group tuning loop over p, d and q (02:435-488, search space 02:461-465), exhaustively
 * rather than by TPE. */
int mmf_fit_select_arma_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                            const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                            const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t pred_start, int32_t n_pred,
                            float* out_pred, int64_t ld_out, int32_t* out_choice_p, int32_t* out_choice_d,
                            int32_t* out_choice_q, float* out_mse,
                            float* out_cand_mse /* [n][n_diffs][n_mas][n_orders] */, float* out_phi, float* out_theta,
                            int32_t* out_order, int32_t* out_ma_order, float* out_sigma, int32_t* out_status,
                            mmf_stats* stats);

/* ---- the (p, d, q) selection's winner refit by conditional least squares (DESIGN.md section 2 item 18) -----------------
 * mmf_fit_select_arma_css_f32: mmf_fit_select_arma_f32, then every series' winner refit at its own (p, d, q) by
 * mmf_fit_forecast_arma_css_f32's Levenberg-Marquardt, from the winner's Hannan-Rissanen (phi, theta).  The arguments are
 * mmf_fit_select_arma_f32's, with max_iter and the nullable out_css_start, out_css, out_css_stop and out_iters [n] of
 * mmf_fit_forecast_arma_css_f32.  Per row:
 *   a winner with q >= 1 gets every output (pred, phi, theta, order, ma_order, sigma, status, css_start, css, css_stop,
 *   iters) of mmf_fit_forecast_arma_css_f32 at its (p, d, q) with long_order = m_d (the selection's long order of its d),
 *   the same max_iter and the same prediction window, bit for bit (such a winner passed the Hannan-Rissanen gate);
 *   a winner with q = 0 keeps every output of mmf_fit_select_arma_f32 bit for bit, with css_start and css NaN and
 *   css_stop and iters 0; so does a row with no eligible candidate.
 * choice_p, choice_d, choice_q, mse and cand_mse are mmf_fit_select_arma_f32's bit for bit: the refit does not choose
 * again, and mse stays the score of the Hannan-Rissanen winner.  max_iter outside [0, MMF_CSS_ITER_MAX] is MMF_E_INVALID,
 * checked first; every other refusal is mmf_fit_select_arma_f32's, with its code and text.  Otherwise the contract of
 * mmf_fit_select_arma_f32 (plans, device buffers only, any ld_out, enqueue-only unless `stats` is non-NULL, whose n_pending
 * then also counts the refit's fits, mmf_config.kernel and assume_finite honoured, refused arguments write nothing).
 * Scratch: per slab, that of mmf_fit_select_arma_f32 and 68 B per row (the winner's phi, theta, order, ma_order,
 * choice_d and choice_q, written there when the caller passes NULL for them, and the list of the rows refit).
 * replaces: the reference's final model (02:472-481), SARIMAX(order = the tuned order, exog) fitted on the training rows
 * after the tuning loop, by the conditional likelihood. */
int mmf_fit_select_arma_css_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                                const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                                const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t max_iter,
                                int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                                int32_t* out_choice_p, int32_t* out_choice_d, int32_t* out_choice_q, float* out_mse,
                                float* out_cand_mse /* [n][n_diffs][n_mas][n_orders] */, float* out_phi,
                                float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                                int32_t* out_status, float* out_css_start, float* out_css, int32_t* out_css_stop,
                                int32_t* out_iters, mmf_stats* stats);

/* mmf_fit_select_arma_joint_f32: mmf_fit_select_arma_css_f32 with each q >= 1 winner refit by
 * mmf_fit_forecast_arma_joint_f32 (beta jointly with (phi, theta)) instead, every output of that call at the winner's
 * (p, d, q), long_order = m_d, bit for bit; and the nullable out_beta [n][MMF_P]: the joint call's for a q >= 1 winner;
 * for a q = 0 winner W gamma (+ c on the intercept) of the plain fit the winner builds on, in arma_joint's fp32 order
 * (for d = 0 mmf_fit_forecast_f32's out_beta bit for bit; for d >= 1 the coefficients of Delta^d X); NaN for a row with
 * no eligible candidate.  Otherwise mmf_fit_select_arma_css_f32's contract. */
int mmf_fit_select_arma_joint_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                                  const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                                  const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t max_iter,
                                  int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out, float* out_beta,
                                  int32_t* out_choice_p, int32_t* out_choice_d, int32_t* out_choice_q, float* out_mse,
                                  float* out_cand_mse /* [n][n_diffs][n_mas][n_orders] */, float* out_phi,
                                  float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                                  int32_t* out_status, float* out_css_start, float* out_css, int32_t* out_css_stop,
                                  int32_t* out_iters, mmf_stats* stats);

/* ---- the (p, d, q) selection's winner refit by exact likelihood, and its Kalman predictor (DESIGN.md section 2 item 21)
 * mmf_fit_select_arma_ml_f32: mmf_fit_select_arma_css_f32, then every q >= 1 winner refined by
 * mmf_fit_forecast_arma_ml_f32's maximum likelihood from the CSS refit's (phi, theta).  The arguments are
 * mmf_fit_select_arma_css_f32's with that call's four CSS columns replaced by the nullable out_loglik_start, out_loglik,
 * out_ml_stop and out_iters [n] of mmf_fit_forecast_arma_ml_f32 (the CSS columns are not returned).  Per row:
 *   a winner with q >= 1 gets every output (pred, phi, theta, order, ma_order, sigma, status, loglik_start, loglik,
 *   ml_stop, iters) of mmf_fit_forecast_arma_ml_f32 at its (p, d, q) with long_order = m_d, the same max_iter and the
 *   same prediction window, bit for bit;
 *   a winner with q = 0, and a row with no eligible candidate, keeps every output of mmf_fit_select_arma_f32 bit for bit,
 *   with loglik_start and loglik NaN and ml_stop and iters 0 (q = 0 winners are not refit).
 * choice_p, choice_d, choice_q, mse and cand_mse are mmf_fit_select_arma_f32's bit for bit.  max_iter outside [0,
 * MMF_CSS_ITER_MAX] is MMF_E_INVALID, checked first; every other refusal is mmf_fit_select_arma_f32's, with its code and
 * text.  Otherwise mmf_fit_select_arma_css_f32's contract, scratch included (68 B per row).
 * replaces: the reference's final model (02:472-481), SARIMAX(order = the tuned order, exog) fitted on the training rows
 * after the tuning loop, by the exact likelihood. */
int mmf_fit_select_arma_ml_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                               const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                               const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t max_iter,
                               int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                               int32_t* out_choice_p, int32_t* out_choice_d, int32_t* out_choice_q, float* out_mse,
                               float* out_cand_mse /* [n][n_diffs][n_mas][n_orders] */, float* out_phi,
                               float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                               int32_t* out_status, float* out_loglik_start, float* out_loglik, int32_t* out_ml_stop,
                               int32_t* out_iters, mmf_stats* stats);

/* mmf_fit_select_arma_ml_kf_f32: mmf_fit_select_arma_ml_f32 with the same arguments and out_se / ld_se of
 * mmf_fit_forecast_arma_ml_kf_f32.  Per row:
 *   a winner with q >= 1 gets every output of mmf_fit_forecast_arma_ml_kf_f32 at its (p, d, q) with long_order = m_d,
 *   the same max_iter and the same prediction window, out_se included, bit for bit;
 *   every other row keeps mmf_fit_select_arma_ml_f32's outputs, and its out_se is mmf_arima_se_f32 of the call's outputs
 *   with the per-series d (diffs = choice_d) bit for bit (NaN for a row with no eligible candidate).
 * ld_se < n_pred with out_se given is MMF_E_INVALID.  Otherwise mmf_fit_select_arma_ml_f32's contract.  With out_se the
 * call runs each listed d's fit once more (the predictor follows the se pass over every row), so n_pending counts
 * 3 n_diffs fits per row; without it 2 n_diffs.  Scratch: per slab, 72 B per row when out_se is given and out_sigma is
 * NULL (the winner's sigma as well), 68 B otherwise.
 * replaces: the reference's final model and its predict() (02:472-488): SARIMAX fitted at the tuned order by exact
 * likelihood, then the Kalman filter's predictions in sample, its dynamic forecast beyond, and their standard errors. */
int mmf_fit_select_arma_ml_kf_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t n_hold,
                                  const int32_t* orders, int32_t n_orders, const int32_t* diffs, int32_t n_diffs,
                                  const int32_t* mas, int32_t n_mas, int32_t long_order, int32_t max_iter,
                                  int32_t pred_start, int32_t n_pred, float* out_pred, int64_t ld_out,
                                  int32_t* out_choice_p, int32_t* out_choice_d, int32_t* out_choice_q, float* out_mse,
                                  float* out_cand_mse /* [n][n_diffs][n_mas][n_orders] */, float* out_phi,
                                  float* out_theta, int32_t* out_order, int32_t* out_ma_order, float* out_sigma,
                                  int32_t* out_status, float* out_loglik_start, float* out_loglik,
                                  int32_t* out_ml_stop, int32_t* out_iters, float* out_se, int64_t ld_se,
                                  mmf_stats* stats);

/* ---- standard errors of the ARIMA-family forecasts (DESIGN.md section 2 item 15) ----------------------------------------
 * mmf_arima_se_f32: a post-pass over the outputs of any ARIMA-family call (mmf_fit_forecast_ar_f32, _arima_f32, _arma_f32,
 * mmf_fit_select_ar_f32, _select_arima_f32, _select_arma_f32): se[i, j] = sqrt(Var(y_t - yhat_t)), t = pred_start + j,
 * for the predictor those calls ship (one step ahead in sample, the dynamic forecast from t_fit beyond it, missing values
 * filled with predictions), taking the fitted model as true: u_s = sum phi_j u_{s-j} + eps_s + sum theta_j eps_{s-j} on
 * y (d = 0) or z' (d >= 1), eps iid with variance sigma^2, u_s = eps_s = 0 for s < 0, and beta, phi, theta, sigma known
 * (no estimation uncertainty).  The covariance of the predictor's error state is propagated in float64 over rows
 * [0, pred_start + n_pred); rows whose z' value (t < t_fit and y_{t-d} .. y_t finite) and level (t < t_fit and y_t
 * finite) are observed reset their error components.  On a gap-free fit window se = sigma in sample and
 * sigma sqrt(sum_{j<h} psi*_j^2) beyond (h = t - t_fit + 1, psi* the psi-weights of (phi, theta) summed d times).
 *   y [n, ld_y]: levels, read on [0, t_fit) only, and only for whether each value is finite (1 <= t_fit <= ld_y);
 *   diffs [n] (nullable): per-row d, e.g. out_choice_d of a selection; NULL: diff_order (0 .. MMF_DIFF_MAX) for every row;
 *   phi [n][MMF_AR_MAX], order [n], sigma [n]: the call's outputs (phi read up to the row's order);
 *   theta [n][MMF_MA_MAX], ma_order [n]: both given or both NULL (NULL: q = 0);
 *   out_se [n, ld_se] (ld_se >= n_pred, any base pointer): only columns [0, n_pred) of a row are written, float32 of
 *   sigma sqrt(1 + c'Pc).  NaN for rows t < d, rows whose level chain is NaN in the predictor (a missing level before
 *   the first observed one), and every row of a series whose sigma is not finite (status 1, choice -1) or whose order,
 *   ma_order or d is out of range; +Inf where the float64 variance overflows (explosive parameters).
 * No plan is needed and none is changed.  Device buffers only (host pointers: MMF_E_UNSUPPORTED); enqueue-only unless
 * `stats` is non-NULL; refused arguments write nothing.
 * replaces: SARIMAX's get_forecast().se_mean / conf_int() beside the reference's forecast (02:453-457, 484-488). */
int mmf_arima_se_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y, int32_t t_fit,
                     int32_t diff_order, const int32_t* diffs, const float* phi, const int32_t* order,
                     const float* theta, const int32_t* ma_order, const float* sigma, int32_t pred_start,
                     int32_t n_pred, float* out_se, int64_t ld_se, mmf_stats* stats);

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

/* ---- rolling-origin backtest: K forecast origins in one pass over the data -------------------------------------
 * Origin k (0 <= k < n_origin <= MMF_BT_MAX_ORIGINS, 33 <= origin[0] < ... < origin[n_origin-1]) is exactly the plain
 * model of mmf_plan_design(X, t_fit = origin[k]) evaluated on design rows [origin[k], origin[k] + horizon): the same
 * whitening, kept columns, centring constant, pivot rule and status codes (DESIGN.md section 2 item 8).
 * mmf_plan_backtest: X [n_rows, p] float64 as for mmf_plan_design, 1 <= horizon <= 64,
 * origin[n_origin-1] + horizon <= n_rows, origin[n_origin-1] <= 65535.  A plan of its own: the mmf_plan_design and
 * mmf_plan_calendars plans stay in force.
 * mmf_backtest_f32: y [n, ld_y] device, ld_y >= origin[n_origin-1] + horizon (the actual values are read), 16-B
 * aligned with ld_y % 4 == 0.  Outputs, each nullable (but not out_pred and out_metrics both), device:
 *   out_pred    [n_origin][n][ld_out]  forecasts of origin k for series i (ld_out >= horizon)
 *   out_metrics [n_origin][n][MMF_BT_NMETRIC]  MSE, MAE, bias = mean(forecast - actual), MAPE = mean |e| / |y| over
 *               the points with y != 0; only points where the forecast and y are both finite are scored, in float64;
 *               NaN where nothing is averaged
 *   out_count   [n_origin][n]  scored points
 *   out_status  [n_origin][n]  MMF_STATUS_* of origin k's fit
 * Enqueued on the ctx stream; the call synchronises only when `stats` is non-NULL.  Refused arguments write nothing.
 * replaces: the reference's single train / score split (split_train_score_data, 02:372-380) and its hold-out MSE
 * (02:453-459), at several origins. */
int mmf_plan_backtest(mmf_ctx* ctx, const double* X, int32_t n_rows, int32_t p, int32_t has_constant,
                      int32_t n_origin, const int32_t* origin, int32_t horizon);
int mmf_backtest_f32(mmf_ctx* ctx, const float* y, int64_t n, int64_t ld_y,
                     float* out_pred, int64_t ld_out,
                     float* out_metrics, int32_t* out_count,
                     int32_t* out_status, mmf_stats* stats);

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
