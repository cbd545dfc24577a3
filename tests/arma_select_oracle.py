"""float64 oracle of (p, d, q) selection by hold-out MSE on levels (DESIGN.md section 2 item 14), on top of
``arima_select_oracle`` and ``arma_oracle``.

Candidate (p, d, 0) is ``arima_select_oracle.model`` (p, d); candidate (p, d, q >= 1) is
``arma_oracle.fit_forecast_arma_packed`` with (p, q, d) and the long order m_d of its d (the caller's, or
``default_long_order``).  The candidates run d ascending, then q ascending, then p ascending.  A candidate's score is the
MSE of its dynamic level forecast from origin t_fit over the held-out rows [t_fit, t_fit + n_hold) against y there,
over the points where both are finite; NaN where none is.  A candidate is eligible when the fit it builds on is not
empty.  Among the eligible candidates the first minimum in list order wins; a q >= 1 candidate wins only with a scored
point, so with none scored anywhere the winner is ``arima_select_oracle``'s (the last eligible q = 0 candidate); (-1, -1,
-1) when none is eligible.  The predictions, phi, theta, order, ma_order, sigma and status are the winner's.

``mse_bound`` is ``arima_select_oracle.mse_bound`` for the q = 0 candidates and for the q >= 1 candidates that fall
back; for the gated q >= 1 candidates the same first-order bound with ``arma_oracle.pred_bound`` on the held-out rows.
"""
from __future__ import annotations

import math

import numpy as np

from ar_oracle import AR_MAX, FP32_EPS
from ar_select_oracle import holdout_mse
from arima_select_oracle import model as arima_model
from arima_select_oracle import mse_bound as arima_mse_bound
from arma_oracle import HR_LONG_MAX, MA_MAX, fit_forecast_arma_packed, pred_bound

MAX_PQ = 32                                     # MMF_ARMASEL_MAX_PQ
DELTA, COND0 = 2e-6, 1e3                        # test_gpu_arma's beta tolerance: DELTA max(COND0, cond(G)) (1 + |beta|)


def default_long_order(t_fit: int, d: int, orders, mas) -> int:
    """m_d = min(32, max(2 max(orders, mas), floor(ln(t_fit - d)^2))): one long order per d for every candidate"""
    lt = math.log(t_fit - d)
    return min(HR_LONG_MAX, max(2 * max(max(orders), max(mas)), int(math.floor(lt * lt))))


def model(y, X, t_fit: int, pred_start: int, n_pred: int, p: int, d: int, q: int, m: int = 0):
    """candidate (p, d, q) as a dict with pred / phi / theta / order / ma_order / sigma / status"""
    if q == 0:
        r = dict(arima_model(y, X, t_fit, pred_start, n_pred, p, d))
        n = len(r["status"])
        r["theta"], r["ma_order"] = np.zeros((n, MA_MAX)), np.zeros(n, dtype=np.int32)
        return r
    return fit_forecast_arma_packed(y, X, t_fit, pred_start, n_pred, p, q, d, m)


def choose(cand_mse, eligible):
    """(k [n], l [n], j [n]) positions of the winner in (diffs, mas, orders) for cand_mse [n, n_diffs, n_mas, n_orders]
    and eligible [n, n_diffs]: the first minimum over the eligible scored candidates in list order; with none scored,
    the last eligible q = 0 candidate; (-1, -1, -1) when none is eligible"""
    cand_mse = np.asarray(cand_mse, dtype=np.float64)
    n, nd, nq, no = cand_mse.shape
    out = np.full((3, n), -1, dtype=np.int64)
    for i in range(n):
        best = last = None
        for k in range(nd):
            if not eligible[i, k]:
                continue
            last = (k, 0, no - 1)
            for l in range(nq):
                for j in range(no):
                    v = cand_mse[i, k, l, j]
                    if not np.isnan(v) and (best is None or v < best[0]):
                        best = (v, k, l, j)
        if best is not None:
            out[:, i] = best[1:]
        elif last is not None:
            out[:, i] = last
    return out[0], out[1], out[2]


def select_arma_packed(y, X, t_fit: int, n_hold: int, orders, diffs, mas, pred_start: int, n_pred: int,
                       long_order: int = 0):
    """-> dict(pred, choice_p, choice_d, choice_q, mse, cand_mse [n, n_diffs, n_mas, n_orders], eligible [n, n_diffs],
    phi, theta, order, ma_order, sigma, status, hold [n_diffs][n_mas][n_orders] (each candidate's future-mode result),
    m [n_diffs] (the long orders), k, l, j (the winner's positions, -1 when none is eligible))"""
    y = np.asarray(y, dtype=np.float64)
    orders, diffs, mas = [int(p) for p in orders], [int(d) for d in diffs], [int(q) for q in mas]
    assert mas[0] == 0 and len(orders) * (len(mas) - 1) <= MAX_PQ
    n = y.shape[0]
    y_hold = y[:, t_fit:t_fit + n_hold]
    ms = [long_order or default_long_order(t_fit, d, orders, mas) for d in diffs]
    hold = [[[model(y, X, t_fit, t_fit, n_hold, p, d, q, ms[k]) for p in orders] for q in mas]
            for k, d in enumerate(diffs)]
    cand_mse = np.array([[[holdout_mse(h["pred"], y_hold)[0] for h in row] for row in blk] for blk in hold])
    cand_mse = np.moveaxis(cand_mse.reshape(len(diffs), len(mas), len(orders), n), 3, 0)
    eligible = np.stack([blk[0][0]["status"] != 1 for blk in hold], axis=1)
    kk, ll, jj = choose(cand_mse, eligible)
    pred = np.full((n, n_pred), np.nan)
    phi, theta = np.zeros((n, AR_MAX)), np.zeros((n, MA_MAX))
    order, ma_order = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    sigma, mse = np.full(n, np.nan), np.full(n, np.nan)
    status = np.ones(n, dtype=np.int32)
    won = kk >= 0
    for k, l, j in sorted(set(zip(kk[won].tolist(), ll[won].tolist(), jj[won].tolist()))):
        r = model(y, X, t_fit, pred_start, n_pred, orders[j], diffs[k], mas[l], ms[k])
        s = won & (kk == k) & (ll == l) & (jj == j)
        for key, dst in (("pred", pred), ("phi", phi), ("theta", theta), ("order", order), ("ma_order", ma_order),
                         ("sigma", sigma), ("status", status)):
            dst[s] = r[key][s]
        mse[s] = cand_mse[s, k, l, j]
    pick = lambda v, idx: np.where(won, np.array(v)[np.maximum(idx, 0)], -1)
    return dict(pred=pred, choice_p=pick(orders, jj), choice_d=pick(diffs, kk), choice_q=pick(mas, ll), mse=mse,
                cand_mse=cand_mse, eligible=eligible, phi=phi, theta=theta, order=order, ma_order=ma_order,
                sigma=sigma, status=status, hold=hold, m=ms, k=kk, l=ll, j=jj)


def beta_tol(res):
    """DELTA max(COND0, cond(G)) (1 + |beta|) per gated row (0 elsewhere): test_gpu_arma's bound on the GPU's (phi,
    theta), the fitted values' relative fp32 error carried through the normal equations"""
    out = np.zeros(len(res["status"]))
    for i, h in enumerate(res["hr"]):
        if h is not None and res["gated"][i]:
            out[i] = DELTA * max(COND0, float(np.linalg.cond(h["G"]))) * (1.0 + np.linalg.norm(h["beta"]))
    return out


def mse_bound(sel, y, taus, t_fit: int, n_hold: int, orders, diffs, mas):
    """First-order bound on |MSE_gpu - MSE_oracle| per series and candidate [n, n_diffs, n_mas, n_orders].  taus[d] =
    (tau_fit, tau_hold) as in arima_select_oracle.mse_bound.  q = 0, and q >= 1 rows that fall back: that bound; gated
    q >= 1 rows: b_s = arma_oracle.pred_bound on the held-out rows with |dbeta| <= beta_tol, and |dMSE| <= (1/N) sum_s
    (2 |e_s| b_s + b_s^2) + 2 eps |MSE| (float32 storage)."""
    y_hold = np.asarray(y, dtype=np.float64)[:, t_fit:t_fit + n_hold]
    cm = sel["cand_mse"]
    q0 = arima_mse_bound({"cand_mse": cm[:, :, 0, :], "hold": [blk[0] for blk in sel["hold"]]}, y, taus, t_fit, n_hold,
                         orders, diffs)
    out = np.repeat(q0[:, :, None, :], len(mas), axis=2)
    for k, d in enumerate(diffs):
        tf, th = taus[d]
        for l in range(1, len(mas)):
            for j in range(len(orders)):
                h = sel["hold"][k][l][j]
                if not h["gated"].any():
                    continue
                b, _ = pred_bound(h, beta_tol(h), tf, th, t_fit, n_hold)
                ok = np.isfinite(h["pred"]) & np.isfinite(y_hold)
                e = np.where(ok, y_hold - np.where(ok, h["pred"], 0.0), 0.0)
                with np.errstate(over="ignore", invalid="ignore"):
                    term = np.where(ok, 2.0 * np.abs(e) * b + b * b, 0.0).sum(axis=1)
                cnt = ok.sum(axis=1)
                g = h["gated"]
                out[g, k, l, j] = (term / np.maximum(cnt, 1) + 2 * FP32_EPS * np.nan_to_num(np.abs(cm[:, k, l, j])))[g]
    return out
