"""float64 oracle of regression with ARIMA(p, d, 0) errors (DESIGN.md section 2 item 11), on top of ``ar_oracle``.

For series i: the differenced series z'_s = Delta^d y_{s+d} (missing when any of its d + 1 levels is), the differenced
design D_d (``diff_design``: float64 differences of the raw rows, cancellation residue zeroed), the AR(p) oracle
``fit_forecast_ar_packed`` on z' and D_d (p = 0: the plain fit), and the integration of its predictions zhat back to
levels with the filled levels ytilde (observed y on the fit rows, the prediction elsewhere, NaN before row d).

``arima_bound`` is the first-order bound the GPU tests hold the library's level predictions to (DESIGN.md section 6).
"""
from __future__ import annotations

import numpy as np

from ar_oracle import FP32_EPS, ar_bound, fit_forecast_ar_packed

DIFF_MAX = 2
RESIDUE = 1e-12


def diff_series(y, d: int):
    """z' [n, t - d] of y [n, t] (float64, NaN where any of the d + 1 levels is not finite)"""
    y = np.asarray(y, dtype=np.float64)
    y = np.where(np.isfinite(y), y, np.nan)
    return np.diff(y, d, axis=1)


def diff_design(X, t_fit: int, d: int):
    """D_d [n_rows - d, p]: row s = Delta^d x_{s+d}; a column whose largest |value| on the fit rows [0, t_fit - d) is at
    most RESIDUE x the raw column's largest |value| on [0, t_fit) is set to 0"""
    X = np.asarray(X, dtype=np.float64)
    D = np.diff(X, d, axis=0)
    raw = np.abs(X[:t_fit]).max(axis=0)
    res = np.abs(D[:t_fit - d]).max(axis=0) <= RESIDUE * raw
    D[:, res] = 0.0
    return D


def fit_forecast_arima_packed(y, X, t_fit: int, pred_start: int, n_pred: int, p: int, d: int):
    """-> dict(pred [n, n_pred], status, phi, order, sigma (those of the AR part on z'), z [n, t_fit - d], D (D_d),
    zres (the ar_oracle result on z' for every z' row), zhat [n, end] (zhat_t at level row t, NaN for t < d),
    ytilde [n, end] the filled levels, obs [n, t_fit], d)"""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)[:, :t_fit]
    n, n_rows = y.shape[0], X.shape[0]
    end = pred_start + n_pred
    z = diff_series(y, d)
    D = diff_design(X, t_fit, d)
    zres = fit_forecast_ar_packed(z, D, t_fit - d, 0, n_rows - d, p)
    obs = np.isfinite(y)
    zhat = np.full((n, end), np.nan)
    if end > d:
        zhat[:, d:end] = zres["pred"][:, :end - d]
    yt = np.full((n, end), np.nan)
    yh = np.full((n, end), np.nan)
    for t in range(end):
        if t >= d:
            yh[:, t] = zhat[:, t] + yt[:, t - 1] if d == 1 else zhat[:, t] + 2.0 * yt[:, t - 1] - yt[:, t - 2]
        keep = obs[:, t] if t < t_fit else np.zeros(n, dtype=bool)
        yt[:, t] = np.where(keep, y[:, t] if t < t_fit else 0.0, yh[:, t])
    pred = yh[:, pred_start:end].copy()
    st = zres["status"]
    pred[st == 1] = np.nan
    return dict(pred=pred, status=st, phi=zres["phi"], order=zres["order"], sigma=zres["sigma"], z=z, D=D, zres=zres,
                zhat=zhat, ytilde=yt, obs=obs, d=d)


def z_tau(res, leverage=1.0):
    """conftest.tolerance of every row's z' (its own max|z|), times the leverage: [n]"""
    z = res["z"]
    mz = np.nanmax(np.abs(np.where(np.isfinite(z), z, 0.0)), axis=1, initial=0.0)
    return (5e-6 * mz + 1e-3) * max(1.0, float(leverage))


def arima_bound(res, tau_fit, tau_pred, t_fit: int, pred_start: int, n_pred: int):
    """First-order bound on |pred_gpu - pred_oracle| per element (DESIGN.md section 6).  tau_fit / tau_pred: the bounds of
    ar_oracle.ar_bound for the fit on z' (the tolerance with max|z|, x the mask factor; on the requested rows also x
    their leverage).  b_s = ar_bound of zhat at z' row s (already x 2).  A level prediction builds on the filled levels
    before it: B_t = b_{t-d} + B~_{t-1} (d = 1) or b_{t-d} + 2 B~_{t-1} + B~_{t-2} (d = 2), with B~_s = 0 for an
    observed fit level and B_s otherwise -- over a dynamic stretch that is sum_j b_j (d = 1) and
    sum_j (h - j + 1) b_j (d = 2) -- plus 2 x the fp32 rounding of each step, 2 eps (|zhat| + 2 |ytilde_{t-1}| +
    |ytilde_{t-2}|)."""
    d = res["d"]
    zr = res["zres"]
    n = zr["pred"].shape[0]
    end = pred_start + n_pred
    tz = t_fit - d
    nz = max(end - d, 0)
    bz = np.zeros((n, end))
    if nz > 0:
        bz[:, d:end] = ar_bound(zr, tau_fit, tau_pred, tz, 0, nz)
    zh = np.nan_to_num(np.abs(res["zhat"]))
    yt = np.nan_to_num(np.abs(res["ytilde"]))
    obs = res["obs"]
    B = np.zeros((n, end))
    Bt = np.zeros((n, end))
    for t in range(d, end):
        if d == 1:
            prop = Bt[:, t - 1]
            rnd = 2 * FP32_EPS * (zh[:, t] + yt[:, t - 1])
        else:
            prop = 2.0 * Bt[:, t - 1] + Bt[:, t - 2]
            rnd = 2 * FP32_EPS * (zh[:, t] + 2.0 * yt[:, t - 1] + yt[:, t - 2])
        B[:, t] = bz[:, t] + prop + 2.0 * rnd
        keep = obs[:, t] if t < t_fit else np.zeros(n, dtype=bool)
        Bt[:, t] = np.where(keep, 0.0, B[:, t])
    return B[:, pred_start:end]
