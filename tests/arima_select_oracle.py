"""float64 oracle of (p, d) selection by hold-out MSE on levels (DESIGN.md section 2 item 12), on top of
``ar_select_oracle`` and ``arima_oracle``.

Candidate (p, 0) is ``ar_select_oracle.candidate`` p (the plain regression for p = 0, AR(p) on y otherwise); candidate
(p, d >= 1) is ``arima_oracle.fit_forecast_arima_packed`` with (p, d).  The candidates run d-major: d ascending, then p
ascending.  A candidate's score is the MSE of its dynamic level forecast from origin t_fit over the held-out rows
[t_fit, t_fit + n_hold) against y there, over the points where both are finite; NaN where none is.  A candidate is
eligible when the fit it builds on (y for d = 0, z' of its d otherwise) is not empty.  Among the eligible candidates the
first minimum in list order wins; the last eligible one when none scores a point; (-1, -1) when none is eligible.  The
predictions, phi, order, sigma and status are the winner's.

``mse_bound`` is ``ar_select_oracle.mse_bound`` for the d = 0 candidates and the same first-order bound with
``arima_bound`` on the held-out rows for d >= 1 (DESIGN.md section 6).
"""
from __future__ import annotations

import numpy as np

from ar_oracle import AR_MAX, FP32_EPS
from ar_select_oracle import candidate, holdout_mse
from ar_select_oracle import mse_bound as ar_mse_bound
from arima_oracle import arima_bound, fit_forecast_arima_packed


def model(y, X, t_fit: int, pred_start: int, n_pred: int, p: int, d: int):
    """candidate (p, d) as a dict with pred / phi / order / sigma / status (y: fit rows only are read)"""
    y = np.asarray(y, dtype=np.float64)[:, :t_fit]
    if d == 0:
        return candidate(y, X, t_fit, pred_start, n_pred, p)
    return fit_forecast_arima_packed(y, X, t_fit, pred_start, n_pred, p, d)


def choose(cand_mse, eligible):
    """(k [n], j [n]) positions of the winner in (diffs, orders) for cand_mse [n, n_diffs, n_orders] and eligible
    [n, n_diffs]: the first minimum over the eligible candidates in d-major order, the last eligible candidate when none
    is scored, (-1, -1) when none is eligible"""
    cand_mse = np.asarray(cand_mse, dtype=np.float64)
    n, nd, no = cand_mse.shape
    kk = np.full(n, -1, dtype=np.int64)
    jj = np.full(n, -1, dtype=np.int64)
    for i in range(n):
        best = None
        last = None
        for k in range(nd):
            if not eligible[i, k]:
                continue
            for j in range(no):
                last = (k, j)
                v = cand_mse[i, k, j]
                if not np.isnan(v) and (best is None or v < best[0]):
                    best = (v, k, j)
        if best is not None:
            kk[i], jj[i] = best[1], best[2]
        elif last is not None:
            kk[i], jj[i] = last
    return kk, jj


def select_arima_packed(y, X, t_fit: int, n_hold: int, orders, diffs, pred_start: int, n_pred: int):
    """-> dict(pred, choice_p, choice_d, mse, cand_mse [n, n_diffs, n_orders], eligible [n, n_diffs], phi, order, sigma,
    status, hold [n_diffs][n_orders] (each candidate's future-mode result over the held-out rows), k, j (the winner's
    positions, -1 when none is eligible))"""
    y = np.asarray(y, dtype=np.float64)
    orders = [int(p) for p in orders]
    diffs = [int(d) for d in diffs]
    n = y.shape[0]
    y_hold = y[:, t_fit:t_fit + n_hold]
    hold = [[model(y, X, t_fit, t_fit, n_hold, p, d) for p in orders] for d in diffs]
    cand_mse = np.stack([np.stack([holdout_mse(h["pred"], y_hold)[0] for h in row], axis=1) for row in hold], axis=1)
    eligible = np.stack([row[0]["status"] != 1 for row in hold], axis=1)
    kk, jj = choose(cand_mse, eligible)
    pred = np.full((n, n_pred), np.nan)
    phi = np.zeros((n, AR_MAX))
    order = np.zeros(n, dtype=np.int32)
    sigma = np.full(n, np.nan)
    status = np.ones(n, dtype=np.int32)
    mse = np.full(n, np.nan)
    won = kk >= 0
    for k, j in sorted(set(zip(kk[won].tolist(), jj[won].tolist()))):
        r = model(y, X, t_fit, pred_start, n_pred, orders[j], diffs[k])
        sel = won & (kk == k) & (jj == j)
        pred[sel], phi[sel], order[sel] = r["pred"][sel], r["phi"][sel], r["order"][sel]
        sigma[sel], status[sel] = r["sigma"][sel], r["status"][sel]
        mse[sel] = cand_mse[sel, k, j]
    choice_p = np.where(won, np.array(orders)[np.maximum(jj, 0)], -1)
    choice_d = np.where(won, np.array(diffs)[np.maximum(kk, 0)], -1)
    return dict(pred=pred, choice_p=choice_p, choice_d=choice_d, mse=mse, cand_mse=cand_mse, eligible=eligible,
                phi=phi, order=order, sigma=sigma, status=status, hold=hold, k=kk, j=jj)


def mse_bound(sel, y, taus, t_fit: int, n_hold: int, orders, diffs):
    """First-order bound on |MSE_gpu - MSE_oracle| per series and candidate [n, n_diffs, n_orders] (DESIGN.md section 6).
    taus[d] = (tau_fit, tau_hold), per series: for d = 0 those of ar_select_oracle.mse_bound; for d >= 1 the tau_fit /
    tau_pred of arima_bound (the fit on z' of that d).  For d >= 1, b_s = arima_bound of the candidate on the held-out rows
    and, as there, |dMSE| <= (1/N) sum_s (2 |e_s| b_s + b_s^2) + 2 eps |MSE| (float32 storage)."""
    y_hold = np.asarray(y, dtype=np.float64)[:, t_fit:t_fit + n_hold]
    out = np.zeros(sel["cand_mse"].shape)
    for k, d in enumerate(diffs):
        tf, th = taus[d]
        if d == 0:
            out[:, k, :] = ar_mse_bound({"cand_mse": sel["cand_mse"][:, k, :], "hold": sel["hold"][k]}, y, tf, th,
                                        t_fit, n_hold, orders)
            continue
        for j in range(len(orders)):
            h = sel["hold"][k][j]
            b = arima_bound(h, tf, th, t_fit, t_fit, n_hold)
            ok = np.isfinite(h["pred"]) & np.isfinite(y_hold)
            e = np.where(ok, y_hold - np.where(ok, h["pred"], 0.0), 0.0)
            with np.errstate(over="ignore"):                 # a bound beyond the float64 range is unbounded (inf)
                term = np.where(ok, 2.0 * np.abs(e) * b + b * b, 0.0).sum(axis=1)
            cnt = ok.sum(axis=1)
            out[:, k, j] = term / np.maximum(cnt, 1) + 2 * FP32_EPS * np.nan_to_num(np.abs(sel["cand_mse"][:, k, j]))
    return out
