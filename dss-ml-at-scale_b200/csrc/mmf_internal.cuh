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
  float ss;                                // standard-error calls: S = sum over the observed rows of (y - c)^2
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
  uint32_t* zero_next;      // nullable: the NEXT call's counter set (CTR_WORDS words), zeroed by the tensor-core kernel
                            // (no memset node)
  int64_t row_base;         // ragged fallback launches cover one calendar's rows: absolute row of this launch's row 0
  int32_t cal_id;           //   ... and that calendar's index (written into the records the launch queues)
};

// Outputs of a standard-error call (mmf_fit_forecast_se_f32, DESIGN.md section 2 item 7).  Kernels take it as their
// last parameter and read it only in their SE instantiation, so the plain instantiations are unchanged.
struct SeArgs {
  float* out_se;            // nullable [n, ld_se]: sigma * sqrt(1 + h_t) for the requested rows
  int64_t ld_se;
  float* sigma;             // [n] residual scale (never null inside the library: scratch if the caller passed NULL)
  int32_t* dof;             // nullable [n]: n_obs - used columns
  const float* sfac;        // [n_rows] sqrt(1 + |a_t|^2) of the planned design (gap-free rows: G_i = I)
};

// Backtest calls (mmf_backtest_f32, DESIGN.md section 2 item 8): one pass of fit_tc_kernel over [0, t_K) captures the
// moments at every origin t_0 < ... < t_{K-1} = t_K in the basis of the longest window.  Origin k is calendar k of the
// backtest plan's stacked designs (its own whitening, t_fit = t_k, prediction rows [t_k, t_k + n_pred)).
struct BtArgs {
  const CalMeta* cals;      // [K] the origins as calendars of the stacked plan
  const float* pred;        // [K][n_pred][P] origin k's prediction rows in the common basis, T_k a^(k)_t (float64 -> fp32)
  const float* tmat;        // [K][P][P] T_k = W^-1 W_k, row-major: b^(k) = T_k^T b_k
  float* mom;               // [K-1][2 consumer groups][n][P] partial moments at the earlier origins
  SolveRec* recs;           // [K][n] records by origin, then row (FitArgs::recs is block K-1)
  int64_t* rec_rows;        // [K][n] work lists
  uint32_t* rec_count;      // [K]
  uint32_t* pending;        // [K] rows of each origin left to the general pass
  int64_t out_kstride;      // rows between the origin blocks of FitArgs::out
  int64_t st_kstride;       // ... and of FitArgs::status
  int32_t n_origin;
  int32_t t_orig[MMF_BT_MAX_ORIGINS - 1];   // t_k of the earlier origins; INT32_MAX from n_origin - 1 on
};

// warp-per-series CUDA-core kernel (general path)
cudaError_t launch_fit_warp(const DesignView& d, const FitArgs& a, int sm_count, cudaStream_t s,
                            const SeArgs* se = nullptr);
size_t fit_warp_smem_bytes(const DesignView& d, int* smem_rows);

// thread-per-series normal equations for the deferred masked rows: Gram downdate, in-order Cholesky with
// pivot dropping and both triangular solves entirely in registers, then the forecasts
cudaError_t launch_solve_rows(const DesignView& d, const FitArgs& a, int sm_count, cudaStream_t s,
                              const CalMeta* cals = nullptr, const SeArgs* se = nullptr);
// se rows of the gap-free rows of a fit + predict_tc call: out_se[i, k] = sigma_i * sfac[pred_start + k] for every row
// whose status is MMF_STATUS_OK right after fit_tc_kernel (launched before the passes that finish the other rows)
cudaError_t launch_se_outer(const FitArgs& a, const SeArgs& se, int sm_count, cudaStream_t s);
constexpr int CTR_WORDS = 8;             // one counter set: {rows left pending, solve records queued, tiles claimed by
                                         // fit_tc beyond its first wave, 5 unused words}
constexpr int CTR_TILE_CLAIM = 2;

// fitted values + forecasts for MANY prediction rows (the reference's "Demand_Fitted for every date"
// contract, 02:484-494): out[n, n_pred] = c + gamma A_pred^T as a wgmma GEMM with TMA-stored tiles
struct PredictLaunch {
  alignas(64) unsigned char tmap_bhi[128];
  alignas(64) unsigned char tmap_blo[128];
  alignas(64) unsigned char tmap_out[128];
  int32_t n_tma;                           // single calendar: columns [0, n_tma) leave through tmap_out, [n_tma, n_pred)
                                           // through plain stores (TMA clips with 16-B granularity, n_tma = n_pred & ~3)
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
};
// variant: 2 = <6 smem stages, 2 forecast staging tiles>, anything else = <8 stages, 1 staging tile> (the product);
// 128-row tiles dealt round robin over the SMs either way
cudaError_t launch_fit_tc(const DesignView& d, const FitArgs& a, const TcLaunch& tl,
                          uint32_t* pending_count, int sm_count, cudaStream_t s, int variant = 0,
                          const MultiView* multi = nullptr);
// the product configuration <8, 1> with the standard-error outputs (SE instantiation)
cudaError_t launch_fit_tc_se(const DesignView& d, const FitArgs& a, const TcLaunch& tl, uint32_t* pending_count,
                             int sm_count, cudaStream_t s, const SeArgs& se);
// the product configuration <8, 1> capturing the moments at every backtest origin (BT instantiation)
cudaError_t launch_fit_tc_bt(const DesignView& d, const FitArgs& a, const TcLaunch& tl, uint32_t* pending_count,
                             int sm_count, cudaStream_t s, const BtArgs& bt);
bool fit_tc_supported(const DesignView& d, const FitArgs& a, const char** why);

// Forecast errors of a backtest (backtest.cu): one warp per (series, origin) scores pred[k][i][0, H) against
// y[i][t_k, t_k + H) and writes {MSE, MAE, bias, MAPE} and the number of scored points.
struct ScoreArgs {
  const float* pred;        // origin k, row i: pred + (k * pred_kstride + i) * ld_pred
  int64_t ld_pred, pred_kstride;
  const float* y;           // row i: y + i * ld_y
  int64_t ld_y;
  const CalMeta* cals;      // t_fit of calendar k = origin t_k
  float* metrics;           // nullable: (k * out_kstride + i) * MMF_BT_NMETRIC
  int32_t* count;           // nullable: k * out_kstride + i
  int64_t out_kstride;
  int64_t n;                // rows
  int32_t n_origin, horizon;
};
cudaError_t launch_bt_score(const ScoreArgs& sa, int sm_count, cudaStream_t s);

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

// regression with AR(p) errors (ar.cu, DESIGN.md section 2 item 9): runs behind the fit passes of a gamma / c hand-off
// call, reads a.status / a.out_gamma / a.out_c, writes out[row, 0 .. n_pred) itself (any ld_out, any base pointer)
struct ArArgs {
  int32_t p;                      // 1 .. MMF_AR_MAX (selection: the largest candidate, 0 .. MMF_AR_MAX), one per call
  float* phi;                     // nullable [n][MMF_AR_MAX]: Yule-Walker coefficients, 0 beyond the series' order
  int32_t* order;                 // nullable [n]: the series' order p_i
  float* sigma;                   // nullable [n]: innovation standard deviation
  const uint32_t* nz;             // [n_rows] of the planned design: bit q set when whitened column q is non-zero on row t
};
cudaError_t launch_ar(const DesignView& d, const FitArgs& a, const ArArgs& ar, cudaStream_t s);

// per-series AR order selection by hold-out MSE (ar.cu, DESIGN.md section 2 item 10): the ar_kernel passes with
// ArArgs::p = the largest candidate, a scoring walk over the held-out rows [t_fit, t_fit + n_hold) per candidate, and
// pass B with the winner's order
struct ArSelArgs {
  int32_t n_hold;                           // held-out rows: design rows [t_fit, t_fit + n_hold), y columns likewise
  int32_t n_cand;                           // 1 .. MMF_ARSEL_MAX_CAND
  int32_t cand[MMF_ARSEL_MAX_CAND];         // ascending distinct orders in [0, MMF_AR_MAX], last == ArArgs::p
  int32_t* choice;                          // nullable [n]: the chosen order (-1 for empty series)
  float* mse;                               // nullable [n]: hold-out MSE of the chosen order
  float* cand_mse;                          // nullable [n][n_cand]: hold-out MSE of every candidate
};
cudaError_t launch_ar_select(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArSelArgs& sel,
                             cudaStream_t s);

// regression with ARIMA(p, d, 0) errors (arima.cu, DESIGN.md section 2 item 11).  The fit passes and arima_kernel run on
// the differenced series z' (FitArgs::y, ld_y: the pitched scratch diff_kernel writes) with the plan of D_d;
// FitArgs::pred_start / n_pred / out / ld_out are the LEVEL rows of the caller's window, which the fit passes ignore
// (gamma / c hand-off, skip_pred)
struct ArimaArgs {
  const float* y;                 // levels [n, ld_y] (row 0 of the slab)
  int64_t ld_y;
  int32_t t_fit;                  // level fit rows; z' has t_fit - d
  int32_t d;                      // 1 .. MMF_DIFF_MAX (selection calls: 0 for the candidates on y itself)
};
// z'[i, s] = Delta^d y[i, s + d] for s in [0, t_fit - d) (NaN when any of its d + 1 levels is missing), rows of ld_z floats
cudaError_t launch_diff(const ArimaArgs& ma, float* z, int64_t ld_z, int64_t n, int sm_count, cudaStream_t s);
cudaError_t launch_arima(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma, cudaStream_t s);

// per-series (p, d) selection by hold-out MSE on levels (arima.cu, DESIGN.md section 2 item 12): one launch per listed d,
// in list order, behind that d's fit (on y for d = 0, ArimaArgs::d = 0; on z' otherwise).  Each launch scores its d's
// candidates and compares its first minimum with the running best the earlier d's left in `best`.
struct ArimaSelBest {                     // one row's running best over the d's launched so far (16 B)
  double mse;                             // float64 hold-out MSE of the leader (valid when flags & SCORED)
  int16_t p, d;                           // the leader
  int32_t flags;                          // ARIMASEL_SCORED: some eligible candidate scored a point; ARIMASEL_ELIGIBLE
};
static_assert(sizeof(ArimaSelBest) == 16, "ArimaSelBest is one 16-B record");
constexpr int32_t ARIMASEL_SCORED = 1, ARIMASEL_ELIGIBLE = 2;
struct ArimaSelArgs {
  int32_t n_hold;                         // held-out level rows [t_fit, t_fit + n_hold)
  int32_t n_cand;                         // orders: 1 .. MMF_ARSEL_MAX_CAND
  int32_t cand[MMF_ARSEL_MAX_CAND];       // ascending distinct orders in [0, MMF_AR_MAX], last == ArArgs::p
  int32_t d_index;                        // position of this d in the call's list; 0 writes every output of every row
  int32_t n_diffs;
  ArimaSelBest* best;                     // [n] running best (scratch)
  int32_t* choice_p;                      // nullable [n]: the chosen order (-1: no eligible candidate)
  int32_t* choice_d;                      // nullable [n]: the chosen d (-1 likewise)
  float* mse;                             // nullable [n]: the winner's hold-out MSE
  float* cand_mse;                        // nullable [n][n_diffs][n_cand]
  int32_t* status;                        // nullable [n]: the winner's fit status (FitArgs::status is this d's scratch)
};
cudaError_t launch_arima_select(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                                const ArimaSelArgs& sel, cudaStream_t s);

// regression with ARIMA(p, d, q) errors (arma.cu, DESIGN.md section 2 item 13): arma_kernel runs behind ar_kernel
// (d = 0) or arima_kernel (d >= 1) with order p, which write every row's fallback outputs, and overwrites the outputs of
// the rows whose Hannan-Rissanen estimate passes the gate.  ArimaArgs::d = 0 with ArimaArgs::y = FitArgs::y for d = 0.
struct ArmaArgs {
  int32_t q;                              // 1 .. MMF_MA_MAX
  int32_t m;                              // long AR order, max(p, q) .. MMF_HR_LONG_MAX (resolved: never 0)
  float* theta;                           // nullable [n][MMF_MA_MAX]
  int32_t* ma_order;                      // nullable [n]
};
cudaError_t launch_arma(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                        const ArmaArgs& hr, cudaStream_t s);

// ARIMA(p, d, q) errors by conditional least squares (arma_css.cu, DESIGN.md section 2 item 16): arma_css_kernel runs
// behind arma_kernel in the same slab (same fit hand-off, z'), reads the HR (phi, theta) from ArArgs::phi /
// ArmaArgs::theta and the gated rows from ArmaArgs::ma_order (caller buffers or scratch: never null for this kernel), and
// overwrites the outputs of the rows that accepted a step
struct CssArgs {
  int32_t max_iter;                       // passes per series, 1 .. MMF_CSS_ITER_MAX (resolved: never 0)
  float* css_start;                       // nullable [n]: S at the HR estimate
  float* css;                             // nullable [n]: S at the shipped estimate
  int32_t* css_stop;                      // nullable [n]: 1 converged, 2 stalled, 3 budget, 0 not refined
  int32_t* iters;                         // nullable [n]: passes run
};
cudaError_t launch_arma_css(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                            const ArmaArgs& hr, const CssArgs& cs, cudaStream_t s);

// ARIMA(p, d, q) errors with beta estimated jointly by conditional least squares (arma_joint.cu, DESIGN.md section 2
// item 17): arma_joint_kernel runs where arma_css_kernel runs for the CSS call, with the same CssArgs, and adds the
// whitened coefficients of the series' used columns to the parameter vector
struct JointArgs {
  float* beta;                            // nullable [n][P]: W gamma (+ c on the intercept) of the shipped gamma
};
cudaError_t launch_arma_joint(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                              const ArmaArgs& hr, const CssArgs& cs, const JointArgs& jt, cudaStream_t s);

// ARIMA(p, d, q) errors by exact Gaussian likelihood (arma_ml.cu, DESIGN.md section 2 item 19): arma_ml_kernel runs
// behind arma_css_kernel in the same slab, reads the CSS (phi, theta) from ArArgs::phi / ArmaArgs::theta and the gated
// rows from ArmaArgs::ma_order (never null for this kernel), and overwrites the outputs of the rows that accepted a step
struct MlArgs {
  int32_t max_iter;                       // passes per series, 1 .. MMF_CSS_ITER_MAX (resolved: never 0)
  float* loglik_start;                    // nullable [n]: the exact log-likelihood at the CSS estimate
  float* loglik;                          // nullable [n]: ... at the shipped estimate
  int32_t* stop;                          // nullable [n]: 1 converged, 2 stalled, 3 budget, 0 not refined
  int32_t* iters;                         // nullable [n]: passes run
};
cudaError_t launch_arma_ml(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                           const ArmaArgs& hr, const MlArgs& ml, cudaStream_t s);

// the Kalman predictor of the ML fit (arma_kf.cu, DESIGN.md section 2 item 20): arma_kf_kernel runs behind arma_ml_kernel
// in the same slab (and behind arima_se_kernel over the slab's rows when se is given), reads the shipped (phi, theta)
// and the gated rows as arma_ml_kernel does, and overwrites pred (and se) of every gated row whose P_0 solves there
struct KfArgs {
  float* se;                              // nullable [n, ld_se]: the standard errors of the predictions
  int64_t ld_se;
};
cudaError_t launch_arma_kf(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                           const ArmaArgs& hr, const KfArgs& kf, cudaStream_t s);

// the refit of a (p, d, q) selection's winners (DESIGN.md section 2 item 18): one stage per listed d behind the
// selection's stages, on that d's fit.  refit_list_kernel lists the slab's rows whose winner is (p, d, q >= 1) and writes
// the refit outputs of the rows no refit kernel touches; arma_css_list_kernel / arma_joint_list_kernel run the fixed-order
// kernels over the list, p and q of each row read from ArArgs::order / ArmaArgs::ma_order (the winner's).  ArArgs::p and
// ArmaArgs::q are the call's largest listed orders there.
struct RefitArgs {
  const int32_t* choice_d;                // [n] the selection's winner (caller buffers or scratch: never null here)
  const int32_t* choice_q;
  int32_t first;                          // the call's first refit stage: it also writes the rows with no eligible candidate
  int32_t* rows;                          // [n] per-slab scratch: the list (any order), and its length
  uint32_t* count;
};
cudaError_t launch_refit_list(const DesignView& d, const FitArgs& a, const ArimaArgs& ma, const CssArgs& cs,
                              const JointArgs& jt, const RefitArgs& rf, cudaStream_t s);
cudaError_t launch_arma_css_list(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                                 const ArmaArgs& hr, const CssArgs& cs, const RefitArgs& rf, cudaStream_t s);
cudaError_t launch_arma_joint_list(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                                   const ArmaArgs& hr, const CssArgs& cs, const JointArgs& jt, const RefitArgs& rf,
                                   cudaStream_t s);
// the ML refit and its Kalman predictor (arma_ml.cu, arma_kf.cu, DESIGN.md section 2 item 21): arma_ml_list_kernel and
// arma_kf_list_kernel run arma_ml_kernel / arma_kf_kernel over the refit stage's list as arma_css_list_kernel runs
// arma_css_kernel; refit_ml_cols_kernel writes the ML columns of the rows refit_list_kernel leaves out, by its rule
cudaError_t launch_arma_ml_list(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                                const ArmaArgs& hr, const MlArgs& ml, const RefitArgs& rf, cudaStream_t s);
cudaError_t launch_refit_ml_cols(const FitArgs& a, const ArimaArgs& ma, const MlArgs& ml, const RefitArgs& rf,
                                 cudaStream_t s);
cudaError_t launch_arma_kf_list(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                                const ArmaArgs& hr, const KfArgs& kf, const RefitArgs& rf, cudaStream_t s);

// per-series (p, d, q) selection by hold-out MSE on levels (arma_select.cu, DESIGN.md section 2 item 14): one launch per
// listed d, right behind that d's arima_select_kernel (same fit, z', gamma / c and running best), for the q >= 1 blocks.
// Candidate lane c is the pair (pq_p[c], pq_q[c]), q-major; its normal equations are those of row set pq_rs[c], the rows
// R(q, L = max(p, q)), shared by every candidate with the same (q, L).
struct ArmaSelArgs {
  int32_t m;                                        // long AR order of this d (resolved)
  int32_t n_mas;                                    // listed MA orders, mas[0] = 0
  int32_t n_pq;                                     // candidate lanes: the (p, q >= 1) pairs (0: the q outputs only)
  int32_t n_rs;                                     // distinct row sets
  int32_t n_ent;                                    // normal-equation entries of all row sets
  int32_t pq_p[MMF_ARMASEL_MAX_PQ], pq_q[MMF_ARMASEL_MAX_PQ];
  int32_t pq_j[MMF_ARMASEL_MAX_PQ];                 // index of p in the orders
  int32_t pq_qi[MMF_ARMASEL_MAX_PQ];                // index of q in the MA orders
  int32_t pq_rs[MMF_ARMASEL_MAX_PQ];
  int32_t rs_q[MMF_ARMASEL_MAX_PQ], rs_L[MMF_ARMASEL_MAX_PQ];
  int32_t rs_pmax[MMF_ARMASEL_MAX_PQ];              // largest p of the row set's candidates: its e lags
  int32_t rs_off[MMF_ARMASEL_MAX_PQ];               // first entry; (pmax + q + 1)(pmax + q + 2) / 2 - 1 entries
  const float* cand_q0;                             // [n][n_diffs][n_orders]: arima_select_kernel's scores (scratch)
  float* cand_mse;                                  // nullable [n][n_diffs][n_mas][n_orders]
  int32_t* choice_q;                                // nullable [n]: the chosen q (-1: no eligible candidate)
  float* theta;                                     // nullable [n][MMF_MA_MAX]
  int32_t* ma_order;                                // nullable [n]
};
size_t arma_select_smem_bytes(int n_ent);          // dynamic shared memory of a launch
cudaError_t launch_arma_select(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                               const ArimaSelArgs& sel, const ArmaSelArgs& hs, cudaStream_t s);

// standard errors of the ARIMA-family forecasts (arima_se.cu, DESIGN.md section 2 item 15): one warp per series, no plan
struct ArimaSeArgs {
  const float* y;                 // [n, ld_y] levels, read on [0, t_fit) for finiteness only
  int64_t ld_y;
  int32_t t_fit;
  int32_t diff_order;             // d of every row when diffs is null
  const int32_t* diffs;           // nullable [n]: per-row d
  const float* phi;               // [n][MMF_AR_MAX]
  const int32_t* order;           // [n]
  const float* theta;             // nullable [n][MMF_MA_MAX] (with ma_order)
  const int32_t* ma_order;        // nullable [n]: q = 0 when null
  const float* sigma;             // [n]
  int32_t pred_start, n_pred;
  float* out;                     // [n, ld_se]
  int64_t ld_se;
  int64_t n;
};
cudaError_t launch_arima_se(const ArimaSeArgs& a, int sm_count, cudaStream_t s);

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
