"""float64 oracle of AR order selection by hold-out MSE (DESIGN.md section 2 item 10), on top of ``ar_oracle``.

Candidate m >= 1 is ``ar_oracle.fit_forecast_ar_packed`` with p = m; candidate 0 is the plain regression of
``oracle.mmf_oracle`` (phi 0, order 0, sigma = sqrt(r_0)).  Candidate m's score is the MSE of its dynamic forecast from
origin t_fit over the held-out rows [t_fit, t_fit + n_hold) (``fit_forecast_ar_packed(y, X, t_fit, t_fit, n_hold, m)``)
against y there, over the points where both are finite; NaN where none is.  The first minimum in list order wins; the
last candidate when no point is scored; -1 for empty series.  The predictions are the chosen candidate's.

``mse_bound`` is the first-order bound on |MSE_gpu - MSE_oracle| of every candidate that the GPU tests hold the library to
(DESIGN.md section 6).
"""
from __future__ import annotations

import numpy as np

from ar_oracle import AR_MAX, FP32_EPS, ar_bound, degenerate_bound, fit_forecast_ar_packed
from oracle import mmf_oracle as O


def holdout_mse(pred, y_hold):
    """(mse [n] float64, count [n]) over the points where the forecast and y are both finite; NaN where none is"""
    pred = np.asarray(pred, dtype=np.float64)
    y_hold = np.asarray(y_hold, dtype=np.float64)
    ok = np.isfinite(pred) & np.isfinite(y_hold)
    d = np.where(ok, y_hold - np.where(ok, pred, 0.0), 0.0)
    cnt = ok.sum(axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        mse = np.where(cnt > 0, (d * d).sum(axis=1) / np.maximum(cnt, 1), np.nan)
    return mse, cnt


def first_minimum(cand_mse):
    """index of the first minimum of each row (NaN never wins); the last index where every entry is NaN"""
    cand_mse = np.asarray(cand_mse, dtype=np.float64)
    n, k = cand_mse.shape
    out = np.full(n, k - 1, dtype=np.int64)
    for i in range(n):
        best = None
        for j in range(k):
            v = cand_mse[i, j]
            if not np.isnan(v) and (best is None or v < best):
                best, out[i] = v, j
    return out


def candidate(y, X, t_fit: int, pred_start: int, n_pred: int, m: int):
    """the model of candidate m as a dict of fit_forecast_ar_packed's keys (m = 0: the plain regression)"""
    if m >= 1:
        return fit_forecast_ar_packed(y, X, t_fit, pred_start, n_pred, m)
    res = fit_forecast_ar_packed(y, X, t_fit, pred_start, n_pred, 1)
    n = len(res["status"])
    pred = res["fitted"][:, pred_start:pred_start + n_pred].copy()
    pred[res["status"] == 1] = np.nan
    sigma = np.where(res["status"] != 1, np.sqrt(res["r"][:, 0]), np.nan)
    return dict(res, pred=pred, phi=np.zeros((n, AR_MAX)), order=np.zeros(n, dtype=np.int32), sigma=sigma,
                ar=np.zeros_like(pred), kappas=[[] for _ in range(n)], r=res["r"][:, :1])


def select_ar_packed(y, X, t_fit: int, n_hold: int, orders, pred_start: int, n_pred: int):
    """-> dict(pred, choice, mse, cand_mse [n, k], count [n], phi, order, sigma, status, hold [k] (candidate m's
    future-mode result over the held-out rows), idx [n] (the chosen position in ``orders``))"""
    y = np.asarray(y, dtype=np.float64)
    orders = [int(m) for m in orders]
    y_hold = y[:, t_fit:t_fit + n_hold]
    hold = [candidate(y[:, :t_fit], X, t_fit, t_fit, n_hold, m) for m in orders]
    scores = [holdout_mse(h["pred"], y_hold) for h in hold]
    cand_mse = np.stack([s[0] for s in scores], axis=1)
    count = scores[0][1]
    status = hold[0]["status"]
    idx = first_minimum(cand_mse)
    n = y.shape[0]
    final = {m: candidate(y[:, :t_fit], X, t_fit, pred_start, n_pred, m) for m in sorted(set(orders[j] for j in idx))}
    pred = np.full((n, n_pred), np.nan)
    phi = np.zeros((n, AR_MAX))
    order = np.zeros(n, dtype=np.int32)
    sigma = np.full(n, np.nan)
    for i in range(n):
        r = final[orders[idx[i]]]
        pred[i], phi[i], order[i], sigma[i] = r["pred"][i], r["phi"][i], r["order"][i], r["sigma"][i]
    empty = status == 1
    choice = np.where(empty, -1, np.array(orders)[idx])
    mse = cand_mse[np.arange(n), idx]
    return dict(pred=pred, choice=choice, mse=mse, cand_mse=cand_mse, count=count, phi=phi, order=order, sigma=sigma,
                status=status, hold=hold, idx=idx, final=final)


def mse_bound(sel, y, tau_fit, tau_hold, t_fit: int, n_hold: int, orders, phi_gpu=None):
    """First-order bound on |MSE_gpu - MSE_oracle| per series and candidate [n, k] (DESIGN.md section 6):
      |dMSE_m| <= (1/N) sum_s (2 |e_s| b_s + b_s^2) + 2 eps |MSE_m|   (float32 storage)
    e_s = y_s - the oracle's forecast, b_s = ar_bound of candidate m on the held-out rows (candidate 0: tau_hold, the
    plain tolerance x the leverage of the held-out rows), N the scored points.  tau_fit / tau_hold are per series.
    With phi_gpu (one [n, AR_MAX] array per candidate: the GPU's coefficients of candidate m), b_s is
    ar_oracle.degenerate_bound instead, which also holds on degenerate rows."""
    y_hold = np.asarray(y, dtype=np.float64)[:, t_fit:t_fit + n_hold]
    out = np.zeros(sel["cand_mse"].shape)
    for j, m in enumerate(orders):
        h = sel["hold"][j]
        if m >= 1 and phi_gpu is not None:
            b = degenerate_bound(h, phi_gpu[j], tau_fit, tau_hold, t_fit, t_fit, n_hold)
        elif m >= 1:
            b = ar_bound(h, tau_fit, tau_hold, t_fit, t_fit, n_hold)
        else:
            b = np.repeat(np.asarray(tau_hold, dtype=np.float64)[:, None], n_hold, axis=1)
        ok = np.isfinite(h["pred"]) & np.isfinite(y_hold)
        e = np.where(ok, y_hold - np.where(ok, h["pred"], 0.0), 0.0)
        term = np.where(ok, 2.0 * np.abs(e) * b + b * b, 0.0).sum(axis=1)
        cnt = ok.sum(axis=1)
        out[:, j] = term / np.maximum(cnt, 1) + 2 * FP32_EPS * np.nan_to_num(np.abs(sel["cand_mse"][:, j]))
    return out
