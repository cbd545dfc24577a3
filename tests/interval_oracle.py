"""float64 oracle of the prediction standard errors (DESIGN.md section 2 item 7), beside ``oracle.mmf_oracle``'s fit.

For series i: n_obs finite fit values, k whitened columns its fit uses (the calendar's kept columns less those the
in-order pivot dropping of ``mmf_oracle.solve_series`` drops for its mask), RSS = sum_obs (y - yhat)^2 computed from the
residuals themselves (not through S - b'gamma, the library's shortcut), dof = n_obs - k, sigma = sqrt(RSS / dof) (NaN
when dof <= 0), se_t = sigma * sqrt(1 + h_t) with h_t = a_t' G_i^-1 a_t over the used columns.  S = sum_obs (y - c)^2
with the library's centring constant c (first finite fit value; 0 without a constant) is returned as the scale the
cancellation bound of the GPU tests is stated against.
"""
from __future__ import annotations

import numpy as np

from oracle import mmf_oracle as O


def _factor(G):
    """in-order Cholesky with the oracle's pivot dropping -> (L, kept index list)"""
    p = G.shape[0]
    L = np.zeros((p, p))
    keep = []
    for j in range(p):
        if G[j, j] <= 0.0:
            continue
        d = G[j, j] - L[j, :j] @ L[j, :j]
        if d <= O.PIVOT_TOL * G[j, j]:
            continue
        keep.append(j)
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (G[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L, keep


def fit_forecast_se_packed(y, X, t_fit: int, pred_start: int, n_pred: int, has_constant: bool = True):
    """-> dict(pred, status, se, sigma, dof, S, rss, h, ratio) in float64 (int32 status / dof; ratio: the oracle's
    smallest pivot ratio per row)."""
    y = np.asarray(y, dtype=np.float64)[:, :t_fit]
    X = np.asarray(X, dtype=np.float64)
    pred, status, gamma, ratio = O.fit_forecast_packed(y, X, t_fit, pred_start, n_pred, return_gamma=True)
    W, kept = O.whiten(X[:t_fit])
    A = X @ W
    a_fit, a_pred = A[:t_fit], A[pred_start:pred_start + n_pred]
    n = y.shape[0]
    obs = np.isfinite(y)
    n_obs = obs.sum(axis=1)
    resid = np.where(obs, y - gamma @ a_fit.T, 0.0)
    rss = (resid ** 2).sum(axis=1)
    first = np.where(obs.any(axis=1), y[np.arange(n), np.argmax(obs, axis=1)], 0.0)
    c = first if has_constant else np.zeros(n)
    S = np.where(obs, (y - c[:, None]) ** 2, 0.0).sum(axis=1)
    k = np.full(n, int(kept.sum()))
    h = np.broadcast_to((a_pred ** 2).sum(axis=1), (n, n_pred)).copy()      # gap-free rows: G_i = I
    cache = {}
    for i in np.flatnonzero(~obs.all(axis=1) & obs.any(axis=1)):
        key = obs[i].tobytes()
        if key not in cache:
            G = a_fit[obs[i]].T @ a_fit[obs[i]]
            L, keep = _factor(G)
            if keep:
                Lk = L[np.ix_(keep, keep)]
                w = np.linalg.solve(Lk, a_pred[:, keep].T)
                cache[key] = (len(keep), (w ** 2).sum(axis=0))
            else:
                cache[key] = (0, np.zeros(n_pred))
        k[i], h[i] = cache[key]
    dof = np.where(obs.any(axis=1), n_obs - k, 0).astype(np.int32)
    with np.errstate(invalid="ignore", divide="ignore"):
        sigma = np.where(dof > 0, np.sqrt(rss / np.maximum(dof, 1)), np.nan)
    se = sigma[:, None] * np.sqrt(1.0 + h)
    return dict(pred=pred, status=status, se=se, sigma=sigma, dof=dof, S=S, rss=rss, h=h, ratio=ratio)
