"""Float64 oracle of the ARIMA-family forecast standard errors (mmf_arima_se_f32, DESIGN.md section 2 item 15).

The error of the predictor the ARIMA-family calls ship, y_t - yhat_t, is linear in the innovations when the fitted model
is taken as true.  Its variance is propagated as the covariance P (units of sigma^2) of the predictor's error state
x = (du_{s-1..s-8}, deps_{s-1..s-4}, dy_{t-1..t-2}) -- the largest state, zero-padded, so every series shares one layout
-- from row 0 with no shortcut: P' = A P A' + b b' with A built in full, vectorised over the series."""
import numpy as np

AR_MAX, MA_MAX, DIFF_MAX = 8, 4, 2
KM = AR_MAX + MA_MAX + DIFF_MAX
IU, IE, IY = 0, AR_MAX, AR_MAX + MA_MAX          # heads of the three blocks

_SHIFT = np.zeros((KM, KM))
for _lo, _hi in ((IU, IE), (IE, IY), (IY, KM)):
    for _r in range(_lo + 1, _hi):
        _SHIFT[_r, _r - 1] = 1.0


def arima_se(y, t_fit: int, phi, order, sigma, pred_start: int, n_pred: int, diff_order: int = 0, diffs=None,
             theta=None, ma_order=None, no_gaps: bool = False):
    """-> se [n, n_pred] float64: sigma sqrt(1 + c'Pc) of rows [pred_start, pred_start + n_pred); NaN for t < d, for
    rows whose used level lag is NaN in the predictor's level chain and for rows with an invalid order, d or sigma; +Inf
    where the variance overflows.  ``no_gaps``: every fit row counts as observed (the negative control's rule)."""
    y = np.asarray(y, dtype=np.float64)[:, :t_fit]
    n = y.shape[0]
    end = pred_start + n_pred
    p = np.asarray(order, dtype=np.int64)
    q = np.zeros(n, dtype=np.int64) if ma_order is None else np.asarray(ma_order, dtype=np.int64)
    d = np.full(n, int(diff_order), dtype=np.int64) if diffs is None else np.asarray(diffs, dtype=np.int64)
    sig = np.asarray(sigma, dtype=np.float64)
    valid = (p >= 0) & (p <= AR_MAX) & (q >= 0) & (q <= MA_MAX) & (d >= 0) & (d <= DIFF_MAX) & np.isfinite(sig)
    obs = np.ones_like(y, dtype=bool) if no_gaps else np.isfinite(y)
    a = np.zeros((n, KM))
    a[:, IU:IE] = np.where(np.arange(AR_MAX)[None, :] < p[:, None], np.asarray(phi, dtype=np.float64)[:, :AR_MAX], 0.0)
    if theta is not None:
        a[:, IE:IY] = np.where(np.arange(MA_MAX)[None, :] < q[:, None], np.asarray(theta, dtype=np.float64), 0.0)
    c = a.copy()
    c[:, IY] = np.where(d == 1, 1.0, np.where(d == 2, 2.0, 0.0))
    c[:, IY + 1] = np.where(d == 2, -1.0, 0.0)
    P = np.zeros((n, KM, KM))
    f0, f1 = np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
    run = np.zeros(n, dtype=np.int64)
    out = np.full((n, n_pred), np.nan)
    with np.errstate(over="ignore", invalid="ignore"):
        for t in range(end):
            lobs = obs[:, t] if t < t_fit else np.zeros(n, dtype=bool)
            run = np.where(lobs, run + 1, 0)
            pre = t < d
            v = np.einsum("ni,nij,nj->n", c, P, c)
            flagged = ((d >= 1) & f0) | ((d == 2) & f1)
            if t >= pred_start:
                se = sig * np.sqrt(1.0 + v)
                se = np.where(np.isnan(se), np.inf, se)
                out[:, t - pred_start] = np.where(pre | flagged | ~valid, np.nan, se)
            zobs = run >= d + 1
            A = np.broadcast_to(_SHIFT, (n, KM, KM)).copy()
            b = np.zeros((n, KM))
            A[:, IU] = np.where(zobs[:, None], 0.0, a)
            b[:, IU] = np.where(zobs, 0.0, 1.0)
            A[:, IE] = np.where(zobs[:, None], -a, 0.0)
            b[:, IE] = np.where(zobs, 0.0, 1.0)
            A[:, IY] = np.where(lobs[:, None], 0.0, c)
            b[:, IY] = np.where(lobs, 0.0, 1.0)
            Pn = A @ P @ np.swapaxes(A, 1, 2) + b[:, :, None] * b[:, None, :]
            P = np.where(pre[:, None, None], P, Pn)
            nf = np.where(pre, ~lobs, ~lobs & flagged)
            f1, f0 = f0, nf
    return out


def psi_star(phi, theta, d: int, length: int):
    """psi-weights of (phi, theta), summed d times, from scipy's impulse response (independent of the recursion)"""
    from scipy.signal import lfilter
    imp = np.zeros(length)
    imp[0] = 1.0
    psi = lfilter(np.r_[1.0, np.asarray(theta, dtype=np.float64)], np.r_[1.0, -np.asarray(phi, dtype=np.float64)], imp)
    for _ in range(d):
        psi = np.cumsum(psi)
    return psi


def simulate(phi, theta, d: int, length: int, n: int, rng):
    """n paths of levels from a zero pre-sample (u_s = eps_s = 0 for s < 0), sigma = 1; levels y_0 .. y_{d-1} N(0, 1)"""
    p, q = len(phi), len(theta)
    L = length - d
    eps = rng.standard_normal((n, L))
    u = np.zeros((n, L))
    for s in range(L):
        u[:, s] = eps[:, s]
        for j in range(p):
            if s - 1 - j >= 0:
                u[:, s] += phi[j] * u[:, s - 1 - j]
        for j in range(q):
            if s - 1 - j >= 0:
                u[:, s] += theta[j] * eps[:, s - 1 - j]
    if d == 0:
        return u
    y = np.zeros((n, length))
    y[:, :d] = rng.standard_normal((n, d))
    for t in range(d, length):
        y[:, t] = u[:, t - d] + (y[:, t - 1] if d == 1 else 2.0 * y[:, t - 1] - y[:, t - 2])
    return y


def predict(y, obs, t_fit: int, phi, theta, d: int, end: int):
    """the shipped predictor with the regression known (0), every path sharing one observation pattern: the ARMA
    recursion of arma_oracle.recursion on z' and the level integration of arma_oracle._integrate, vectorised over
    paths -> yhat [n, end]"""
    n = y.shape[0]
    p, q = len(phi), len(theta)
    lev = np.where(obs[None, :t_fit], y[:, :t_fit], np.nan)
    z = lev.copy()
    for _ in range(d):
        z = np.diff(z, axis=1)
    T, endz = t_fit - d, end - d
    U, E, pr = np.zeros((n, endz)), np.zeros((n, endz)), np.zeros((n, endz))
    for s in range(endz):
        g = np.zeros(n)
        for j in range(p):
            if s - 1 - j >= 0:
                g += phi[j] * U[:, s - 1 - j]
        for j in range(q):
            if s - 1 - j >= 0:
                g += theta[j] * E[:, s - 1 - j]
        pr[:, s] = g
        if s < T and np.isfinite(z[0, s]):
            U[:, s] = z[:, s]
            E[:, s] = z[:, s] - g
        else:
            U[:, s] = g
    if d == 0:
        return pr
    yt, yh = np.full((n, end), np.nan), np.full((n, end), np.nan)
    for t in range(end):
        if t >= d:
            yh[:, t] = pr[:, t - d] + yt[:, t - 1] if d == 1 else pr[:, t - d] + 2.0 * yt[:, t - 1] - yt[:, t - 2]
        yt[:, t] = y[:, t] if (t < t_fit and obs[t]) else yh[:, t]
    return yh
