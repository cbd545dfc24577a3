"""float64 oracle of the Kalman predictor of the exact-likelihood ARIMA(p, d, q) fit (DESIGN.md section 2 item 20), on top
of ``arma_ml_oracle``.

For a covered series (gated, P_0 solves at the shipped point x): the model of ``arma_ml_oracle`` (Harvey's form, r =
max(p, q + 1), dense T and R here), the filter from a = 0 and the stationary P_0 = (I - T (x) T)^-1 vec(R R') (a dense
Kronecker solve, not the kernel's folded system):
  prediction   ehat_s = a_{s,1}: s < T the filter's prediction from the observed rows before s (a missing row predicted,
               not updated), s >= T the dynamic forecast a <- T a;
  levels       zhat_s = fitted_s + ehat_s, integrated to levels by ``arma_oracle._integrate`` (missing levels filled);
  variance     the dense covariance C of xi = (alpha - a, the d previous level errors), C' = A C A' + b b' with
               A = [[T - K Z, 0], [lambda row or 0], [shift]], b = (R, 0): the level error of row t is lambda = Z (alpha -
               a) + L . (level errors), L = (1) or (2, -1), and is 0 where y_t is observed.  var_t = c' C c (units of
               sigma^2) before the row's update; NaN for t < d and where arima_se's level-chain flags are set.
``gain_p0`` and ``no_cross`` restate the two negative-control builds.
"""
from __future__ import annotations

import numpy as np
from scipy.signal import lfilter

from arma_ml_oracle import p0_solve, state_dim
from arma_oracle import _integrate


def model(x, p: int, q: int):
    """-> (r, T [r, r], R [r]) of the library's sign convention"""
    r = state_dim(p, q)
    x = np.asarray(x, dtype=np.float64)
    Tm = np.zeros((r, r))
    Tm[:p, 0] = x[:p]
    Tm[np.arange(r - 1), np.arange(1, r)] = 1.0
    R = np.zeros(r)
    R[0] = 1.0
    R[1:q + 1] = x[p:p + q]
    return r, Tm, R


def stationary_p0(Tm, R):
    r = len(R)
    return np.linalg.solve(np.eye(r * r) - np.kron(Tm, Tm), np.outer(R, R).ravel()).reshape(r, r)


def covered(x, p: int, q: int) -> bool:
    """the kernel's cover rule: the folded P_0 system passes its pivot test at x"""
    return p0_solve(np.asarray(x, dtype=np.float64), p, q) is not None


def kf_forecast(e, obs, T: int, p: int, q: int, x, fitted, y, t_fit: int, d: int, end: int,
                gain_p0: bool = False, no_cross: bool = False):
    """level predictions yhat [end] (NaN for t < d), their error variances var [end] (units of sigma^2, NaN for t < d and
    flagged rows) and ehat [max(end - d, T)].  e, obs: the residual rows [0, T); fitted: z-space fitted values, at least
    max(end - d, T) long; y: the levels [0, t_fit) (NaN missing)"""
    r, Tm, R = model(x, p, q)
    k = r + d
    endz = end - d
    endB = max(endz, T)
    y = np.asarray(y, dtype=np.float64)
    lobs = lambda t: t < t_fit and bool(np.isfinite(y[t]))   # noqa: E731
    C = np.zeros((k, k))
    C[:r, :r] = stationary_p0(Tm, R)
    K0 = Tm @ C[:r, 0] / C[0, 0]
    cv = np.zeros(k)
    cv[0] = 1.0
    cv[r:] = [1.0] if d == 1 else [2.0, -1.0] if d == 2 else []
    b = np.zeros(k)
    b[:r] = R
    flag = {t: not lobs(t) for t in range(d)}
    a = np.zeros(r)
    ehat = np.zeros(endB)
    var = np.full(end, np.nan)
    for s in range(endB):
        t = s + d
        flagged = any(flag[t - 1 - j] for j in range(d))
        ehat[s] = a[0]
        if t < end and not flagged:
            var[t] = cv @ C @ cv
        flag[t] = not lobs(t) and flagged
        o = s < T and bool(obs[s])
        K = (K0 if gain_p0 else Tm @ C[:r, 0] / C[0, 0]) if o else np.zeros(r)
        A = np.zeros((k, k))
        A[:r, :r] = Tm
        A[:r, 0] -= K
        if d >= 1 and not lobs(t):
            A[r] = cv
        if d == 2:
            A[r + 1, r] = 1.0
        C = A @ C @ A.T + np.outer(b, b)
        if no_cross:
            C[:r, r:] = 0.0
            C[r:, :r] = 0.0
        a = Tm @ a + (K * (float(e[s]) - a[0]) if o else 0.0)
    zhat = np.full(end, np.nan)
    zhat[d:end] = np.asarray(fitted, dtype=np.float64)[:endz] + ehat[:endz]
    if d == 0:
        yhat = zhat
    else:
        yl = np.full((1, max(t_fit, end)), np.nan)
        yl[0, :t_fit] = y[:t_fit]
        yhat = _integrate(zhat[None], yl, np.isfinite(yl), t_fit, d, end)[0][0]
    return yhat, var, ehat


def acov(x, p: int, q: int, n: int, n_psi: int = 200000):
    """the autocovariances gamma_0 .. gamma_{n-1} of the ARMA(p, q) process (units of sigma^2), from its psi-weights
    (``arma_ml_oracle.dense_loglik``'s construction)"""
    x = np.asarray(x, dtype=np.float64)
    imp = np.zeros(n_psi)
    imp[0] = 1.0
    psi = lfilter(np.r_[1.0, x[p:p + q]], np.r_[1.0, -x[:p]], imp)
    return np.array([psi[:n_psi - h] @ psi[h:] for h in range(n)])


def conditional_mean(e, obs, T: int, g, endB: int):
    """E[e_s | the observed e before min(s, T)] for s < endB, from the Toeplitz autocovariance g (at least endB long)"""
    out = np.zeros(endB)
    for s in range(endB):
        idx = np.flatnonzero(np.asarray(obs[:min(s, T)], dtype=bool))
        if len(idx) == 0:
            continue
        S = g[np.abs(idx[:, None] - idx[None, :])]
        out[s] = g[s - idx] @ np.linalg.solve(S, np.asarray(e, dtype=np.float64)[idx])
    return out


def error_map(lmask, T: int, p: int, q: int, x, t_fit: int, d: int, end: int):
    """W [end, endz]: the level error y_t - yhat_t of the predictor as a linear map of the true z' (d observed zero
    anchors), found by running ``kf_forecast`` on basis vectors.  lmask: the observed levels [t_fit]."""
    endz = end - d
    W = np.zeros((end, endz))
    for j in range(endz):
        z = np.zeros(endz)
        z[j] = 1.0
        lev = np.zeros(end)
        for t in range(d, end):
            lev[t] = z[t - d] + (lev[t - 1] if d == 1 else 2.0 * lev[t - 1] - lev[t - 2] if d == 2 else 0.0)
        yo = np.where(lmask, lev[:t_fit], np.nan)
        zobs = np.array([all(lmask[s:s + d + 1]) if s + d < t_fit else False for s in range(T)])
        yhat, _, _ = kf_forecast(np.where(zobs, z[:T], 0.0), zobs, T, p, q, x, np.zeros(max(endz, T)), yo, t_fit, d,
                                 end)
        W[:, j] = lev - yhat
    return W


__all__ = ["model", "stationary_p0", "covered", "kf_forecast", "acov", "conditional_mean", "error_map"]
