"""GPU (-m gpu): paths of the C ABI that the other GPU modules leave untested.  Each one is checked against the
float64 oracle, or against a property that must hold exactly.

A. Batches of more than 2^20 rows, which run_device (csrc/mmf_api.cu) fits slab by slab.  Every row is compared with
   the oracle.  Forecasts, holdout tables, coefficients, statuses, model selection, broadcast stores and CUDA-graph
   replays must be bit-equal to the same rows fitted as separate calls of at most 2^20 rows.
   stats.n_pending must count the rows of every slab.
B. Model selection (csrc/select.cu) against a vectorised float64 selection oracle, row by row: the choice is optimal
   up to fp32 noise on every row.  Also the edges: one candidate, eight, rejected lists, n_hold = 1 and 3,500, exact
   ties, non-finite and unobserved held-out windows.
C. tc_variant = 2, the <6 stages, 2 staging tiles> instantiation of fit_tc_kernel, is bit-equal to the product variant.
D. Exact scale and sign equivariance: multiplying a series by 2^k or negating it scales its forecast bit for bit.
   Centring, the mask-based tf32 hi / lo split, fp32 rounding and the pivot tests (which see only the mask) are all
   exponent-relative, so any difference would be a scale dependence inside a kernel."""
import numpy as np
import pytest

import mmf
from conftest import forecast_leverage, record_err, tolerance
from oracle import mmf_oracle as O

pytestmark = pytest.mark.gpu

SLAB_ROWS = 1 << 20                # run_device fits batches of MORE than this many rows slab by slab
N_BIG, T_BIG = 3 * SLAB_ROWS + 1001, 100
CANDS = (1, 3, 9, 13, 16)


def _le(err, tol, what=""):
    """assert err <= tol, leaving the measured error in the scratch log of conftest.record_err"""
    import os
    name = os.environ.get("PYTEST_CURRENT_TEST", "?").split("::")[-1].split(" ")[0]
    record_err(name, err, tol, what=str(what))
    assert err <= tol, (what, float(err), float(tol))


def _design(start, t, h, mode="future"):
    """(X, t_fit, pred_start, n_pred) of a daily calendar: future = fit all t rows, forecast h; holdout = fit t - h,
    evaluate every date"""
    if mode == "holdout":
        return O.design_matrix(O.calendar_grid(start, t, "D"), t - h), t - h, 0, t
    return O.design_matrix(O.calendar_grid(start, t + h, "D"), t), t, t, h


def _bits(t):
    import torch
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same_bits(a, b):
    """bit-for-bit equality of two CUDA tensors (equal NaNs count as equal)"""
    import torch
    return tuple(a.shape) == tuple(b.shape) and torch.equal(_bits(a), _bits(b))


def _row_tol(y, leverage=1.0):
    """conftest.tolerance evaluated with every row's own max|y|: [n]"""
    return np.array([tolerance(r, leverage) for r in y])


def _ill_conditioning(ratio):
    """factor 1/min(1, min_pivot_ratio/0.25) of test_parity_masked_series (empty rows, ratio 0, get inf)"""
    r = np.asarray(ratio, dtype=np.float64)
    return np.where(r > 0, 1.0 / np.minimum(1.0, np.where(r > 0, r, 1.0) / 0.25), np.inf)


def _mask_factor(y, X, t_fit, ps, npred, ratio):
    """Tolerance factor of every row of y for its mask: 1/min(1, ratio/0.25) (test_parity_masked_series) or, where
    larger, the forward-error amplification of the row's own normal equations G_i = A_obs^T A_obs on the columns the
    oracle keeps: (leverage of the prediction rows in G_i's metric / the calendar's) / sqrt(min(1, lambda_min/0.25)).
    The pivot ratio alone misses masks such as the first 9 of 72 fit days missing: pivot ratio 0.08, but
    lambda_min(G_i) ~ 1e-4 and the leverage grows from 38 to 89 -- a plain float32 Cholesky of those rows is off by
    ~5x the ratio-scaled tolerance.  Gap-free rows get 1."""
    W, _ = O.whiten(np.asarray(X, dtype=np.float64)[:t_fit])
    A = np.asarray(X, dtype=np.float64) @ W
    a_fit, a_pred = A[:t_fit], A[ps:ps + npred]
    lev = max(1.0, forecast_leverage(X, t_fit, ps, npred))
    out = _ill_conditioning(ratio)
    cache = {}
    for i, row in enumerate(np.asarray(y)[:, :t_fit]):
        obs = np.isfinite(row)
        if obs.all() or not obs.any():
            continue
        key = obs.tobytes()
        if key not in cache:
            G = a_fit[obs].T @ a_fit[obs]
            keep, L = [], np.zeros((O.P, O.P))
            for j in range(O.P):                             # the oracle's in-order pivot dropping (O.solve_series)
                d = G[j, j] - L[j, :j] @ L[j, :j] if G[j, j] > 0 else 0.0
                if G[j, j] <= 0 or d <= O.PIVOT_TOL * G[j, j]:
                    continue
                keep.append(j)
                L[j, j] = np.sqrt(d)
                L[j + 1:, j] = (G[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
            Gk = G[np.ix_(keep, keep)]
            lam = max(float(np.linalg.eigvalsh(Gk)[0]), 1e-300)
            ak = a_pred[:, keep]
            lev_i = float(np.sqrt(np.einsum("ij,ij->i", ak @ np.linalg.inv(Gk), ak)).max())
            cache[key] = max(1.0, lev_i / lev) / np.sqrt(min(1.0, lam / 0.25))
        out[i] = max(out[i], cache[key])
    return out


def _mostly_missing_cols(t_fit, t, n_obs_fit, n_obs_rest, seed=0):
    """missing columns of a row that has only n_obs_fit observed values in [0, t_fit) and n_obs_rest in [t_fit, t)"""
    rng = np.random.default_rng(seed)
    obs = np.zeros(t, dtype=bool)
    obs[rng.choice(np.arange(t_fit), n_obs_fit, replace=False)] = True
    obs[rng.choice(np.arange(t_fit, t), n_obs_rest, replace=False)] = True
    return np.flatnonzero(~obs)


# ---- selection oracle ----------------------------------------------------------------------------------------------
def select_oracle(y, X, t_fit, n_hold, cands, pred_start, n_pred):
    """Vectorised float64 model selection, the rule of O.select_forecast_packed: gamma from the oracle's full fit on
    the observed rows of [0, t_fit); candidate m keeps gamma[:m]; its score is the mean squared residual over the
    observed held-out rows; the first minimum wins (no observed held-out row: the last candidate; empty series: 0).
    Returns a dict with mse_all [n, n_cand] (NaN where a row has no score), choice, mse, pred, status, gamma, ratio, A."""
    y = np.asarray(y, dtype=np.float64)
    X = np.asarray(X, dtype=np.float64)
    n = y.shape[0]
    _, status, gamma, ratio = O.fit_forecast_packed(y[:, :t_fit], X, t_fit, 0, 1, return_gamma=True)
    W, _ = O.whiten(X[:t_fit])
    A = X @ W
    a_hold = A[t_fit:t_fit + n_hold]
    yh = y[:, t_fit:t_fit + n_hold]
    obs = np.isfinite(yh)
    n_obs = obs.sum(axis=1)
    g = np.where(np.isfinite(gamma), gamma, 0.0)
    # running sums over the columns, in column order: a column that is exactly zero leaves the prediction -- and so
    # the score -- bit-identical, as it does on the device (a matrix product may reassociate and break such ties)
    prefix = np.cumsum(a_hold[None, :, :] * g[:, None, :], axis=2)
    mse_all = np.empty((n, len(cands)))
    for k, m in enumerate(cands):
        e = np.where(obs, yh - prefix[:, :, m - 1], 0.0)
        mse_all[:, k] = (e * e).sum(axis=1) / np.maximum(n_obs, 1)
    live = status != 1
    scored = live & (n_obs > 0)
    mse_all[~scored] = np.nan
    k = np.full(n, len(cands) - 1)
    k[scored] = np.argmin(mse_all[scored], axis=1)
    choice = np.where(live, np.asarray(cands)[k], 0).astype(np.int32)
    mse = np.where(scored, mse_all[np.arange(n), k], np.nan)
    return dict(mse_all=mse_all, choice=choice, mse=mse, status=status, gamma=gamma, ratio=ratio, A=A,
                pred=_predict_with(A, gamma, choice, pred_start, n_pred))


def _predict_with(A, gamma, choice, pred_start, n_pred):
    """float64 prediction of every row from its first choice[i] whitened columns (NaN for choice 0)"""
    a_pred = A[pred_start:pred_start + n_pred]
    out = np.full((gamma.shape[0], n_pred), np.nan)
    for m in np.unique(choice):
        if m > 0:
            r = choice == m
            out[r] = gamma[r, :m] @ a_pred[:, :m].T
    return out


def check_selection(got, y, X, t_fit, n_hold, cands, pred_start, n_pred, what="", orc=None):
    """Per-row checks of a device selection {pred, choice, mse, status} (numpy) against the float64 oracle.
    tol = the conftest formula with the row's own max|y| and the leverage of the held-out rows (times _mask_factor for
    rows with gaps); each held-out residual is then off by at most tol, which bounds
      the choice:  mse_o[m_gpu] <= min_m mse_o[m] + 2 (2 sqrt(min_m mse_o[m]) tol + tol^2)
      the MSE:     |mse_gpu - mse_o[m_gpu]| <= 2 sqrt(mse_o[m_gpu]) tol + tol^2 + 1e-5 mse_o[m_gpu]
    and the prediction must match the oracle's prediction FOR THE GPU'S OWN CHOICE on every non-empty row."""
    y = np.asarray(y)
    orc = orc if orc is not None else select_oracle(y, X, t_fit, n_hold, cands, pred_start, n_pred)
    pred, choice, mse, status = (np.asarray(got[k]) for k in ("pred", "choice", "mse", "status"))
    assert np.array_equal(status, orc["status"]), what
    live = orc["status"] != 1
    assert (choice[~live] == 0).all() and np.isnan(pred[~live]).all() and np.isnan(mse[~live]).all(), what
    assert np.isin(choice[live], cands).all(), what
    scored = live & np.isfinite(orc["mse"])
    unscored = live & ~scored
    assert (choice[unscored] == cands[-1]).all() and np.isnan(mse[unscored]).all(), what
    assert np.isfinite(mse[scored]).all(), what
    yw = np.asarray(y, dtype=np.float64)[:, :t_fit + n_hold]
    tol_h = _row_tol(yw, forecast_leverage(X, t_fit, t_fit, n_hold)) * _mask_factor(y, X, t_fit, t_fit, n_hold, orc["ratio"])
    tol_p = (_row_tol(yw, forecast_leverage(X, t_fit, pred_start, n_pred))
             * _mask_factor(y, X, t_fit, pred_start, n_pred, orc["ratio"]))
    if scored.any():
        kk = np.searchsorted(np.asarray(cands), choice)
        rows = np.flatnonzero(scored)
        mo = orc["mse_all"][rows, kk[rows]]
        best = orc["mse"][rows]
        th = tol_h[rows]
        slack = 2.0 * (2.0 * np.sqrt(best) * th + th * th)
        _le(float(((mo - best) / slack).max()), 1.0, f"{what}: choice optimality (excess held-out MSE / fp32 bound)")
        bound = 2.0 * np.sqrt(mo) * th + th * th + 1e-5 * mo
        _le(float((np.abs(mse[rows] - mo) / bound).max()), 1.0, f"{what}: |mse - oracle mse of the choice| / bound")
    if live.any():
        want = _predict_with(orc["A"], orc["gamma"], np.where(live, choice, 0), pred_start, n_pred)
        err = np.abs(pred[live] - want[live]).max(axis=1) / tol_p[live]
        _le(float(err.max()), 1.0, f"{what}: prediction of the chosen model, worst row error / row tolerance")
    return orc


def _select(eng, yd, n_hold, cands, pred_start, n_pred):
    import torch
    res = eng.fit_select_forecast(yd, n_hold, cands, pred_start, n_pred)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in res.items()}


# =====================================================================================================================
# A. batches of more than one slab
# =====================================================================================================================
KINDS = ("gaps", "leading", "mostly_missing", "empty", "inf")


def _planted_rows(n):
    """rows that get a special pattern: the first and last row, both sides of every multiple of 2^19, and every 997th
    row (so every slab, wherever its edges fall, holds each kind many times); kind = position in that list mod 5"""
    edges = [0, n - 1]
    for k in range(1, (n - 1) // (1 << 19) + 1):
        edges += [k * (1 << 19) - 1, k * (1 << 19)]
    spread = np.arange(3, n, 997)
    rows = np.concatenate([np.array(edges), spread])
    kinds = np.concatenate([np.arange(len(edges)) % len(KINDS), np.arange(len(spread)) % len(KINDS)])
    rows, first = np.unique(rows, return_index=True)
    return rows, kinds[first]


def _plant(yd, rows, kinds):
    """in place, on a [n, 100] CUDA tensor.  Holdout fits columns [0, 72), future mode all 100."""
    import torch
    nan, inf = float("nan"), float("inf")
    cols = {"gaps": [10, 37, 61, 85],                                   # isolated gaps: the queued solve
            "leading": list(range(9)),                                  # first 9 values missing: the general pass
            "mostly_missing": _mostly_missing_cols(72, 100, 30, 8).tolist(),   # > half of either fit window missing:
            "empty": list(range(100))}                                  # the direct Gram of the general pass
    for ki, kind in enumerate(KINDS):
        r = torch.as_tensor(rows[kinds == ki], device=yd.device, dtype=torch.long)[:, None]
        if kind == "inf":
            yd[r, torch.tensor([[20, 50, 90]], device=yd.device)] = inf  # +Inf == missing (90: a held-out value)
        else:
            yd[r, torch.tensor([cols[kind]], device=yd.device)] = nan


@pytest.fixture(scope="module")
def big():
    """3 * 2^20 + 1001 daily series x 100 days on the device (several slabs and a short last tile), special rows
    planted in every slab"""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 8e9:
        pytest.skip("needs 8 GB of free device memory")
    assert N_BIG > SLAB_ROWS                              # more than 2^20 rows: at least two slabs
    yd, start = mmf.synth.daily_store_item_demand_torch(N_BIG, T_BIG, seed=2024)
    rows, kinds = _planted_rows(N_BIG)
    _plant(yd, rows, kinds)
    torch.cuda.synchronize()
    return dict(yd=yd, y=yd.cpu().numpy(), start=start, rows=rows, kinds=kinds)


def _pieces(n):
    """separate calls of at most 2^20 rows, each starting at a multiple of 128"""
    edges = list(range(0, n, SLAB_ROWS)) + [n]
    return list(zip(edges[:-1], edges[1:]))


def _check_big_against_oracle(pred_t, status_t, y, X, t_fit, ps, npred, planted, what):
    """every row against O.fit_forecast_packed_c: equal statuses, NaN rows for empty series, the stated tolerance
    (scaled on the planted rows by their mask's factor, _mask_factor, ratio from the NumPy oracle on those rows only)"""
    n = y.shape[0]
    tol = tolerance(y, forecast_leverage(X, t_fit, ps, npred))
    _, _, _, ratio = O.fit_forecast_packed(y[planted], X, t_fit, ps, npred, return_gamma=True)
    row_tol = np.full(n, tol)
    row_tol[planted] = tol * _mask_factor(y[planted], X, t_fit, ps, npred, ratio)
    worst = 0.0
    for b0 in range(0, n, 1 << 19):
        b1 = min(n, b0 + (1 << 19))
        want, wst = O.fit_forecast_packed_c(y[b0:b1], X, t_fit, ps, npred)
        got, st = pred_t[b0:b1].cpu().numpy(), status_t[b0:b1].cpu().numpy()
        assert np.array_equal(st, wst), (what, (b0 + np.flatnonzero(st != wst))[:8])
        ok = wst != 1
        assert np.isnan(got[~ok]).all(), what
        worst = max(worst, float((np.abs(got[ok] - want[ok]).max(axis=1) / row_tol[b0:b1][ok]).max()))
    _le(worst, 1.0, f"{what}: worst row error / row tolerance")


@pytest.mark.parametrize("mode", ["future", "holdout"])
def test_slabbed_batch_matches_oracle_and_pieces(big, mode):
    """future (h = 28: the fit kernel's bulk-store epilogue) and holdout (100 values per row: predict_tc_kernel), every
    kernel: all rows against the oracle, and pred / status / beta bit-equal to separate calls of <= 2^20 rows (rows do
    not depend on their launch position: test_gappy_rows_do_not_depend_on_their_position_in_the_launch)."""
    import torch
    yd, y, start = big["yd"], big["y"], big["start"]
    X, t_fit, ps, npred = _design(start, T_BIG, 28, mode)
    for kernel in ("auto", "tc", "warp"):
        eng = mmf.ForecastEngine(kernel=kernel)
        eng.plan(X, t_fit, True)
        whole = eng.fit_forecast(yd, ps, npred, want_beta=True, want_status=True)
        pred = torch.empty_like(whole["pred"])
        beta = torch.empty_like(whole["beta"])
        status = torch.empty_like(whole["status"])
        for a, b in _pieces(N_BIG):
            eng.fit_forecast(yd[a:b], ps, npred, out=pred[a:b], beta=beta[a:b], status=status[a:b])
        torch.cuda.synchronize()
        assert _same_bits(whole["status"], status), kernel
        assert _same_bits(whole["pred"], pred), kernel
        assert _same_bits(whole["beta"], beta), kernel
        del pred, beta, status
        _check_big_against_oracle(whole["pred"], whole["status"], y, X, t_fit, ps, npred, big["rows"],
                                  f"{mode} {kernel}")
        eng.close()


@pytest.mark.parametrize("kernel", ["auto", "tc"])
def test_slabbed_n_pending_counts_every_slab(big, kernel):
    """stats.n_pending of a several-slab call = the sum over separate calls of <= 2^20 rows.  Each slab's tensor-core
    kernel zeroes the counter set the slab before it used, so a count read from the last set covers the last slab only."""
    yd, start = big["yd"], big["start"]
    eng = mmf.ForecastEngine(kernel=kernel)
    _, ps, npred = eng.plan_calendar(start, T_BIG, "D", 28, "future")
    whole = eng.fit_forecast(yd, ps, npred, want_stats=True)["stats"]
    parts = [eng.fit_forecast(yd[a:b], ps, npred, want_stats=True)["stats"].n_pending for a, b in _pieces(N_BIG)]
    assert whole.kernel_used == "tc"
    assert min(parts) > 0                                 # leading-gap / mostly-missing rows in every piece
    assert whole.n_pending == sum(parts), (whole.n_pending, parts)
    eng.close()


def test_slabbed_selection_matches_pieces_and_oracle(big):
    """fit_select_forecast on the several-slab batch (holdout plan, 28 held-out days): pred / choice / mse / status
    bit-equal to separate calls of <= 2^20 rows; 20,000 sampled rows, the planted ones included, against the float64
    selection oracle."""
    import torch
    yd, y, start = big["yd"], big["y"], big["start"]
    eng = mmf.ForecastEngine()
    _, ps, npred = eng.plan_calendar(start, T_BIG, "D", 28, "holdout")
    whole = eng.fit_select_forecast(yd, 28, CANDS, ps, npred)
    parts = [eng.fit_select_forecast(yd[a:b], 28, CANDS, ps, npred) for a, b in _pieces(N_BIG)]
    torch.cuda.synchronize()
    for k in ("pred", "choice", "mse", "status"):
        assert _same_bits(whole[k], torch.cat([p[k] for p in parts])), k
    del parts
    rng = np.random.default_rng(11)
    idx = np.unique(np.concatenate([big["rows"], rng.choice(N_BIG, 20_000 - len(big["rows"]), replace=False)]))
    ti = torch.as_tensor(idx, device="cuda")
    got = {k: whole[k][ti].cpu().numpy() for k in ("pred", "choice", "mse", "status")}
    X, t_fit, _, _ = _design(start, T_BIG, 28, "holdout")
    check_selection(got, y[idx], X, t_fit, 28, CANDS, ps, npred, "slabbed selection, sampled rows")
    eng.close()


def test_slabbed_bcast_replicas_equal_fit_forecast(big):
    """fit_forecast_bcast on the several-slab batch, three local replicas: each slab offsets every replica pointer"""
    import torch
    yd, start = big["yd"], big["start"]
    eng = mmf.ForecastEngine()
    _, ps, npred = eng.plan_calendar(start, T_BIG, "D", 28, "future")
    want = eng.fit_forecast(yd, ps, npred)
    reps = [torch.zeros((N_BIG, npred), device="cuda") for _ in range(3)]
    eng.fit_forecast_bcast(yd, ps, npred, [r.data_ptr() for r in reps], npred)
    torch.cuda.synchronize()
    for i, r in enumerate(reps):
        assert _same_bits(r, want), i
    eng.close()


def test_slabbed_capture_replays_equal_eager_calls(big):
    """capture() of the several-slab batch: replay() = the eager call, also after y changes in place"""
    import torch
    yd, start = big["yd"].clone(), big["start"]
    eng = mmf.ForecastEngine()
    _, ps, npred = eng.plan_calendar(start, T_BIG, "D", 28, "future")
    status = torch.empty(N_BIG, dtype=torch.int32, device="cuda")
    graph, out = eng.capture(yd, ps, npred, status=status)
    for rep in range(2):
        if rep:
            yd[:, 40:60] += 3.0                           # new data in the same buffer (NaN stays NaN)
            yd[SLAB_ROWS + 5, :9] = float("nan")          # one more row for the general pass
        graph.replay()
        want = eng.fit_forecast(yd, ps, npred, want_status=True)
        torch.cuda.synchronize()
        assert _same_bits(out, want["pred"]), rep
        assert _same_bits(status, want["status"]), rep
    graph.close()
    eng.close()


# =====================================================================================================================
# B. model selection against float64
# =====================================================================================================================
def _selection_batch(n=1200, t=400, h=28, seed=61):
    """the daily generator plus series that favour small models and every kind of mask: gaps in the fit window, rows
    for the general pass, rank-deficient masks (status 2), held-out windows with +Inf / -Inf / nothing observed, an
    empty row"""
    rng = np.random.default_rng(seed)
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=seed)
    tt = np.arange(t)
    y[:150] = np.round(5000 + rng.normal(0, 30, (150, t)))                         # level + noise
    y[150:300] = np.round(3000 + 4.0 * tt[None, :] + rng.normal(0, 20, (150, t)))  # level + trend
    t_fit = t - h
    wd = np.array([d.weekday() for d in O.calendar_grid(start, t, "D")])
    y[300:320, 50:80] = np.nan                                                     # gaps in the fit window
    y[320:330, :9] = np.nan                                                        # general pass
    for r in range(330, 340):                                                      # every Tuesday of the fit window
        y[r, np.flatnonzero(wd[:t_fit] == 1)] = np.nan                             # missing: dow1 dropped, status 2
    y[340:350, t - 10:t - 3] = np.nan                                              # gaps in the held-out window
    y[350:360, t - 5] = np.inf
    y[360:370, t - 20] = -np.inf
    y[370:375, t_fit:] = np.nan                                                    # nothing held out observed
    y[375, :] = np.nan                                                             # empty
    y[376:380, 100] = -np.inf                                                      # -Inf in the fit window
    return y.astype(np.float32), start


def test_model_selection_every_row_against_the_float64_oracle():
    """every row: the choice is optimal up to fp32 noise, the MSE and the prediction of the chosen model match the
    float64 oracle.  The vectorised oracle is pinned to O.select_forecast_packed on a few hundred rows first."""
    n, t, h = 1200, 400, 28
    y, start = _selection_batch(n, t, h)
    X, t_fit, ps, npred = _design(start, t, h, "holdout")
    orc = select_oracle(y, X, t_fit, h, CANDS, ps, npred)
    pin = np.r_[0:40, 150:190, 290:400]
    w_pred, w_choice, w_mse, w_st = O.select_forecast_packed(y[pin], X, t_fit, h, CANDS, ps, npred)
    assert np.array_equal(orc["choice"][pin], w_choice) and np.array_equal(orc["status"][pin], w_st)
    assert np.allclose(orc["mse"][pin], w_mse, rtol=1e-12, equal_nan=True)
    assert np.allclose(orc["pred"][pin], w_pred, rtol=1e-12, atol=1e-9, equal_nan=True)
    assert (orc["status"] == 2).sum() >= 10 and (orc["status"] == 1).sum() == 1
    for kernel in ("auto", "warp"):
        eng = mmf.ForecastEngine(kernel=kernel)
        eng.plan_calendar(start, t, "D", h, "holdout")
        got = _select(eng, mmf.device_packed(y), h, CANDS, ps, npred)
        check_selection(got, y, X, t_fit, h, CANDS, ps, npred, kernel, orc=orc)
        eng.close()


def test_select_full_model_only_is_bit_equal_to_the_holdout_fit():
    """candidates = (16,): the fit kernels, the select kernel (which keeps every column) and predict_tc_kernel must give
    exactly the plain holdout fit (fit kernels + predict_tc_kernel) -- T > 64, so both write through the predict kernel"""
    import torch
    n, t, h = 1000, 200, 28
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=8, nan_frac=0.01)
    y[3, :9] = np.nan
    y[4, :] = np.nan
    yd = mmf.device_packed(y)
    eng = mmf.ForecastEngine()
    _, ps, npred = eng.plan_calendar(start, t, "D", h, "holdout")
    sel = eng.fit_select_forecast(yd, h, (16,), ps, npred)
    plain = eng.fit_forecast(yd, ps, npred, want_status=True)
    torch.cuda.synchronize()
    assert _same_bits(sel["status"], plain["status"])
    assert _same_bits(sel["pred"], plain["pred"])
    live = plain["status"] != 1
    assert bool((sel["choice"][live] == 16).all()) and bool((sel["choice"][~live] == 0).all())
    eng.close()


def test_select_mean_model_predicts_the_mean_of_the_fit_window():
    """candidates = (1,) on gap-free rows: the intercept-only model predicts the mean of the fit window on every date
    (closed form, whatever the whitening)"""
    n, t, h = 700, 300, 28
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=19)
    eng = mmf.ForecastEngine()
    _, ps, npred = eng.plan_calendar(start, t, "D", h, "holdout")
    got = _select(eng, mmf.device_packed(y), h, (1,), ps, npred)
    assert (got["status"] == 0).all() and (got["choice"] == 1).all()
    want = y[:, :t - h].astype(np.float64).mean(axis=1)
    err = np.abs(got["pred"] - want[:, None]).max(axis=1) / _row_tol(y)
    _le(float(err.max()), 1.0, "mean model: worst row error / row tolerance")
    eng.close()


def test_select_eight_candidates_work_and_bad_lists_are_rejected():
    n, t, h = 500, 300, 28
    y, start = _selection_batch(n, t, h, seed=3)
    X, t_fit, ps, npred = _design(start, t, h, "holdout")
    eng = mmf.ForecastEngine()
    eng.plan_calendar(start, t, "D", h, "holdout")
    yd = mmf.device_packed(y)
    eight = (1, 2, 3, 5, 9, 12, 13, 16)
    check_selection(_select(eng, yd, h, eight, ps, npred), y, X, t_fit, h, eight, ps, npred, "eight candidates")
    for bad in (tuple(range(1, 10)), (3, 3), (9, 3), (0, 16), (1, 17)):
        with pytest.raises(mmf.MmfError) as e:
            eng.fit_select_forecast(yd, h, bad, ps, npred)
        assert e.value.code == -1, bad
    eng.close()


@pytest.mark.parametrize("n_hold", [1, 3500])
def test_select_held_out_window_extremes(n_hold):
    """n_hold = 1, and n_hold = MMF_SELECT_MAX_HOLD = 3,500 (224,000 B of opt-in shared memory for the held-out design
    rows, just under the H100's 232,448 B); 3,501 is refused"""
    n, t_fit = 200, 100
    t = t_fit + n_hold
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=40 + n_hold, nan_frac=0.01)
    y[5, :9] = np.nan
    y[6, :] = np.nan
    y[7, t_fit:] = np.nan
    X, _, ps, npred = _design(start, t, n_hold, "holdout")
    eng = mmf.ForecastEngine()
    eng.plan_calendar(start, t, "D", n_hold, "holdout")
    got = _select(eng, mmf.device_packed(y), n_hold, CANDS, ps, npred)
    check_selection(got, y, X, t_fit, n_hold, CANDS, ps, npred, f"n_hold={n_hold}")
    if n_hold == 3500:
        y2, start2 = mmf.synth.daily_store_item_demand(8, t + 1, seed=1)
        eng.plan_calendar(start2, t + 1, "D", n_hold + 1, "holdout")
        with pytest.raises(mmf.MmfError) as e:
            eng.fit_select_forecast(mmf.device_packed(y2), n_hold + 1, CANDS, 0, t + 1)
        assert e.value.code == -3 and "n_hold" in str(e.value)
    eng.close()


def test_select_exact_ties_keep_the_first_minimum():
    """Weekly calendar (W-MON): every date is a Monday, so the day-of-week columns are aliased and whitened columns 3-8
    are exactly zero.  Candidates 3 and 9 then have bit-identical held-out SSE; the first minimum (3) must win, as in the
    oracle, never 9."""
    df = mmf.synth.reference_weekly_demand(n_skus=1)
    b = mmf.pack_groups(df, freq="W-MON", pinned=False)[0]
    t, h = b.y.shape[1], 40
    rng = np.random.default_rng(4)
    y = np.concatenate([b.y, np.round(5000 + rng.normal(0, 40, (300, t))),
                        np.round(2000 + 6.0 * np.arange(t)[None, :] + rng.normal(0, 30, (100, t)))]).astype(np.float32)
    grid = O.calendar_grid(b.start, t, "W-MON")
    X = O.design_matrix(grid, t - h)
    W, kept = O.whiten(X[:t - h])
    assert not kept[3:9].any() and not (X @ W)[:, 3:9].any()
    cands = (3, 9, 16)
    eng = mmf.ForecastEngine()
    eng.plan_calendar(b.start, t, "W-MON", h, "holdout")
    got = _select(eng, mmf.device_packed(y), h, cands, 0, t)
    orc = check_selection(got, y, X, t - h, h, cands, 0, t, "weekly ties")
    assert np.array_equal(orc["mse_all"][:, 0], orc["mse_all"][:, 1])
    assert (orc["choice"] == 3).sum() >= 10               # the tie is the minimum on many rows
    assert not (got["choice"] == 9).any(), np.flatnonzero(got["choice"] == 9)[:10]
    eng.close()


# =====================================================================================================================
# C. tc_variant = 2
# =====================================================================================================================
_VARIANT_CASES = [("future", 1), ("future", 7), ("future", 28), ("future", 30), ("future", 64), ("future", 13),
                  ("holdout", 28)]


def _variant_batch(n, t, seed):
    import torch
    yd, start = mmf.synth.daily_store_item_demand_torch(n, t, seed=seed)
    yd[::7, torch.tensor([17, 90, 151], device="cuda")] = float("nan")      # queued solve
    yd[3::11, :9] = float("nan")                                              # general pass
    if n > 2:
        yd[2, :] = float("nan")                                               # empty
    return yd, start


@pytest.mark.parametrize("n", [1, 129, 132 * 128 + 5, 70_000])
def test_tc_variant_2_is_bit_equal_to_the_product_variant(n):
    """fit_tc_kernel<6, 2, false> (two staging tiles used in turn by the bulk-store epilogue) against the product
    instantiation: pred, status and beta bit-equal for horizons 1 .. 64 (28: the bulk path), an odd one and holdout;
    both against the oracle"""
    import torch
    t = 200
    yd, start = _variant_batch(n, t, seed=900 + n)
    y = yd.cpu().numpy()
    engs = {v: mmf.ForecastEngine(kernel="tc", tc_variant=v) for v in (0, 2)}
    for mode, h in _VARIANT_CASES:
        got = {}
        for v, eng in engs.items():
            got[v] = mmf.forecast_packed(yd, start, "D", h, mode, engine=eng, want_status=True, want_beta=True)
        torch.cuda.synchronize()
        for k in ("pred", "status", "beta"):
            assert _same_bits(got[0][k], got[2][k]), (mode, h, k)
        X, t_fit, ps, npred = _design(start, t, h, mode)
        want, wst = O.fit_forecast_packed_c(y, X, t_fit, ps, npred)
        st = got[2]["status"].cpu().numpy()
        assert np.array_equal(st, wst), (mode, h)
        ok = wst != 1
        if ok.any():
            # two fixed gap patterns (3 isolated days, the first 9 days): their pivot ratios bound every row's
            sample = [r for r in (0, 3) if r < n]
            _, _, _, ratio = O.fit_forecast_packed(y[sample], X, t_fit, ps, npred, return_gamma=True)
            tol = tolerance(y, forecast_leverage(X, t_fit, ps, npred)) / min(1.0, float(ratio.min()) / 0.25)
            _le(np.abs(got[2]["pred"].cpu().numpy()[ok] - want[ok]).max(), tol, (n, mode, h))
    for eng in engs.values():
        eng.close()


def test_tc_variant_2_broadcast_stores_match_the_product_variant():
    """fit_forecast_bcast with three replicas through tc_variant = 2: every replica bit-equal to tc_variant = 0"""
    import torch
    n, t = 70_000, 200
    yd, start = _variant_batch(n, t, seed=5)
    engs = {v: mmf.ForecastEngine(kernel="tc", tc_variant=v) for v in (0, 2)}
    for h in (28, 30, 7):
        for eng in engs.values():
            eng.plan_calendar(start, t, "D", h, "future")
        want = engs[0].fit_forecast(yd, t, h)
        reps = [torch.zeros((n, h), device="cuda") for _ in range(3)]
        engs[2].fit_forecast_bcast(yd, t, h, [r.data_ptr() for r in reps], h)
        torch.cuda.synchronize()
        for i, r in enumerate(reps):
            assert _same_bits(r, want), (h, i)
    for eng in engs.values():
        eng.close()


# =====================================================================================================================
# D. exact scale and sign equivariance
# =====================================================================================================================
SCALES = (-12, -4, 0, 6, 14)                # 2^k: every value of the batch stays a normal float


def _equivariant_batch(t=150):
    """64 base rows (gap-free, gappy, leading gap, mostly missing) -> 6 copies each, interleaved (row 6 i + c = copy c of
    base row i, so copies share tiles): 2^k * base for k in SCALES, then -base"""
    base, start = mmf.synth.daily_store_item_demand(64, t, seed=33)
    base[1::4, [20, 77, 121]] = np.nan
    base[2::4, :9] = np.nan
    base[3::4, _mostly_missing_cols(t - 28, t, 40, 10, seed=1)] = np.nan
    copies = [base * np.float32(2.0 ** k) for k in SCALES] + [-base]
    return np.stack(copies, axis=1).reshape(-1, t).astype(np.float32), start, len(copies)


def _assert_equivariant(pred, status, n_copies, what, power=1):
    """rows of the interleaved batch: copy c = 2^(power k_c) x the k = 0 copy, the negated copy = (-1)^power x it"""
    p = pred.reshape(-1, n_copies, *pred.shape[1:])
    s = status.reshape(-1, n_copies)
    ref = SCALES.index(0)
    for c in range(n_copies):
        assert np.array_equal(s[:, c], s[:, ref]), (what, c)
        f = (-1.0) ** power if c == len(SCALES) else 2.0 ** (power * SCALES[c])
        want = p[:, ref] * np.float32(f)
        bad = ~((p[:, c] == want) | (np.isnan(p[:, c]) & np.isnan(want)))
        assert not bad.any(), (what, c, np.argwhere(bad)[:5].tolist())


@pytest.mark.parametrize("kernel,variant", [("auto", 0), ("tc", 0), ("warp", 0), ("tc", 2)])
def test_forecasts_scale_exactly_with_the_series(kernel, variant):
    import torch
    t = 150
    y, start, nc = _equivariant_batch(t)
    yd = mmf.device_packed(y)
    eng = mmf.ForecastEngine(kernel=kernel, tc_variant=variant)
    for mode, h in (("future", 28), ("future", 30), ("holdout", 28)):
        res = mmf.forecast_packed(yd, start, "D", h, mode, engine=eng, want_status=True)
        torch.cuda.synchronize()
        pred, status = res["pred"].cpu().numpy(), res["status"].cpu().numpy()
        assert (status[::nc] != 1).all()
        _assert_equivariant(pred, status, nc, (kernel, variant, mode, h))
    eng.close()


def test_selection_scales_exactly_with_the_series():
    """fit_select_forecast: the same choice for every copy, mse scaled by 4^k and pred by 2^k exactly"""
    t, h = 150, 28
    y, start, nc = _equivariant_batch(t)
    eng = mmf.ForecastEngine()
    eng.plan_calendar(start, t, "D", h, "holdout")
    got = _select(eng, mmf.device_packed(y), h, CANDS, 0, t)
    _assert_equivariant(got["pred"], got["status"], nc, "selection pred")
    _assert_equivariant(got["mse"], got["status"], nc, "selection mse", power=2)
    c = got["choice"].reshape(-1, nc)
    assert (c == c[:, :1]).all()
    eng.close()
