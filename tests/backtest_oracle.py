"""Float64 oracle of the rolling-origin backtest (DESIGN.md section 2 item 8).

Origin k is, by definition, the plain model fit on rows [0, t_k) of the design and evaluated on rows
[t_k, t_k + horizon): ``oracle/mmf_oracle.py``'s whitening and fit, called once per origin.  The metrics are computed
from scratch in float64.  ``change_of_basis`` states the library's route (one moment in the longest window's basis,
mapped to each origin by T_k = W^-1 W_k) so that tests can check it and size the error bound by ||T_k||_2.  This module
sits beside the tests so that the parity oracle in ``oracle/`` stays unchanged.
"""
import numpy as np

from oracle import mmf_oracle as O

NMETRIC = 4            # MSE, MAE, bias, MAPE


def origins(t_len, horizon, n_origins, step=None):
    """t_k = t_len - horizon - (K-1-k) * step; the last origin is the reference's train / score split (02:372-380)."""
    step = horizon if step is None else step
    return np.array([t_len - horizon - (n_origins - 1 - k) * step for k in range(n_origins)], dtype=np.int64)


def backtest_packed(y, X, origin, horizon, return_ratio=False):
    """-> pred [K, n, horizon] float64, status [K, n] int32 (and the oracle's min pivot ratio [K, n])."""
    X = np.asarray(X, dtype=np.float64)
    preds, sts, ratios = [], [], []
    for t in origin:
        t = int(t)
        pred, st, _, ratio = O.fit_forecast_packed(y, X[:t + horizon], t, t, horizon, return_gamma=True)
        preds.append(pred); sts.append(st); ratios.append(ratio)
    out = (np.stack(preds), np.stack(sts))
    return out + (np.stack(ratios),) if return_ratio else out


def metrics(pred, actual):
    """pred, actual [..., H] -> (metrics [..., 4] float64 = MSE, MAE, bias, MAPE; count [...] int).  Only points where
    both are finite are scored; MAPE averages |e| / |y| over the scored points with y != 0; NaN where nothing is averaged."""
    pred = np.asarray(pred, dtype=np.float64)
    actual = np.asarray(actual, dtype=np.float64)
    ok = np.isfinite(pred) & np.isfinite(actual)
    e = np.where(ok, pred - actual, 0.0)
    cnt = ok.sum(axis=-1)
    nz = ok & (actual != 0)
    cnz = nz.sum(axis=-1)
    with np.errstate(invalid="ignore", divide="ignore"):
        mse = np.where(cnt > 0, (e * e).sum(axis=-1) / cnt, np.nan)
        mae = np.where(cnt > 0, np.abs(e).sum(axis=-1) / cnt, np.nan)
        bias = np.where(cnt > 0, e.sum(axis=-1) / cnt, np.nan)
        ape = np.where(nz, np.abs(e) / np.where(nz, np.abs(actual), 1.0), 0.0)
        mape = np.where(cnz > 0, ape.sum(axis=-1) / cnz, np.nan)
    return np.stack([mse, mae, bias, mape], axis=-1), cnt


def actuals(y, origin, horizon):
    """y[:, t_k : t_k + horizon] for every origin -> [K, n, horizon]"""
    y = np.asarray(y)
    return np.stack([y[:, int(t):int(t) + horizon] for t in origin])


def change_of_basis(X, origin, horizon):
    """The library's route in float64: W of the longest window [0, t_K), W_k of origin k, T_k = W^-1 W_k on the columns
    the longest window keeps.  Returns (T [K, P, P], kappa [K] = ||T_k||_2, leverage [K] = the largest 2-norm of origin
    k's whitened prediction rows)."""
    X = np.asarray(X, dtype=np.float64)
    t_last = int(origin[-1])
    W, kept = O.whiten(X[:t_last])
    idx = np.flatnonzero(kept)
    Winv = np.zeros_like(W)
    Winv[np.ix_(idx, idx)] = np.linalg.inv(W[np.ix_(idx, idx)])
    Ts, kappa, lev = [], [], []
    for t in origin:
        t = int(t)
        Wk, kept_k = O.whiten(X[:t])
        assert not (kept_k & ~kept).any(), "a column aliased on the longest window is aliased on every prefix"
        T = Winv @ Wk
        Ts.append(T)
        kappa.append(float(np.linalg.norm(T, 2)))
        lev.append(float(np.linalg.norm((X @ Wk)[t:t + horizon], axis=1).max()))
    return np.stack(Ts), np.array(kappa), np.array(lev)
