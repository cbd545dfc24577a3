"""float64 oracle of ARIMA(p, d, q) errors by conditional least squares (DESIGN.md section 2 item 16), on top of
``arma_oracle``.

For a gated series (``arma_oracle.hannan_rissanen`` passed its gate): x = (phi, theta), and
  objective  S(x) = sum over C = {s in [p, T): e observed at s} of eps~_s(x)^2, eps~ the forecast recursion of
             ``arma_oracle.recursion`` (zero pre-sample, missing rows filled with their prediction);
  Jacobian   J = d eps~ / dx, exact: on an observed row d u~ = 0 and d eps~ = -d pr, on a missing row d u~ = d pr and
             d eps~ = 0 (``gap_jacobian=False``: the gap-free two-filter form on every row, the control build's rule);
  LM         one pass evaluates S, g = J' eps~, H = J'J at an fp32 point; (H + lam diag H) delta = -g by an in-order
             Cholesky (pivot > PIVOT_TOL x diagonal), x' = fp32(x + delta) must pass the step-down tests, else lam x 10
             with no pass; S(x') < S(x) accepts (lam / 10), otherwise lam x 10; stop 1 converged (an accepted pass lowered
             S by <= RTOL x S), 2 stalled (lam > LAMBDA_MAX), 3 budget (max_iter passes, the first at x0).
Outputs as the library's: the HR row when no step was accepted, otherwise the recursion with the shipped x; sigma =
sqrt(S / |C|) for every gated row.
"""
from __future__ import annotations

import numpy as np

from ar_oracle import AR_MAX, FP32_EPS, KAPPA_MAX
from arma_oracle import MA_MAX, PIVOT_TOL, _integrate, fit_forecast_arma_packed, recursion, step_down

LAMBDA0 = 1e-3
LAMBDA_MAX = 1e10
RTOL = 1e-6
ITER_DEFAULT = 20
ITER_MAX = 64


def css_eval(e, obs, T: int, p: int, q: int, x, gap_jacobian: bool = True):
    """-> (S, J [T, p + q], eps~ [T], C [T] bool) of one series at x = (phi_1..phi_p, theta_1..theta_q)"""
    x = np.asarray(x, dtype=np.float64)
    phi, th = x[:p], x[p:p + q]
    n = p + q
    u = np.zeros(T + AR_MAX)
    ep = np.zeros(T + MA_MAX)
    du = np.zeros((T + AR_MAX, n))
    de = np.zeros((T + MA_MAX, n))
    J = np.zeros((T, n))
    for s in range(T):
        ul = u[AR_MAX + s - 1 - np.arange(p)] if p else np.zeros(0)
        el = ep[MA_MAX + s - 1 - np.arange(q)] if q else np.zeros(0)
        pr = phi @ ul + th @ el
        dpr = np.concatenate([ul, el])
        if p:
            dpr = dpr + phi @ du[AR_MAX + s - 1 - np.arange(p)]
        if q:
            dpr = dpr + th @ de[MA_MAX + s - 1 - np.arange(q)]
        if obs[s]:
            u[AR_MAX + s] = e[s]
            ep[MA_MAX + s] = e[s] - pr
            de[MA_MAX + s] = -dpr
        else:
            u[AR_MAX + s] = pr
            if gap_jacobian:
                du[AR_MAX + s] = dpr
            else:
                de[MA_MAX + s] = -dpr
        J[s] = de[MA_MAX + s]
    eps = ep[MA_MAX:]
    C = np.asarray(obs[:T], dtype=bool).copy()
    C[:p] = False
    return float(eps[C] @ eps[C]), J, eps, C


def two_filter_jacobian(e, obs, T: int, p: int, q: int, x):
    """J_s = (-v_{s-1..s-p}, -w_{s-1..s-q}), v = (1 + theta(B))^-1 u~, w = (1 + theta(B))^-1 eps~ (exact before the
    first missing row)"""
    x = np.asarray(x, dtype=np.float64)
    th = x[p:p + q]
    _, u, eps = recursion(e, obs, T, x[:p], th, T)
    v, w = np.zeros(T), np.zeros(T)
    for s in range(T):
        v[s] = u[s] - sum(th[k] * v[s - 1 - k] for k in range(q) if s - 1 - k >= 0)
        w[s] = eps[s] - sum(th[k] * w[s - 1 - k] for k in range(q) if s - 1 - k >= 0)
    J = np.zeros((T, p + q))
    for s in range(T):
        for j in range(p):
            J[s, j] = -v[s - 1 - j] if s - 1 - j >= 0 else 0.0
        for k in range(q):
            J[s, p + k] = -w[s - 1 - k] if s - 1 - k >= 0 else 0.0
    return J


def _step(H, g, x, p: int, q: int, lam: float):
    """(trial x' or None, lam) of the step rule: lam x 10 until a pivot-safe, step-down-valid fp32 trial point"""
    n = p + q
    while lam <= LAMBDA_MAX:
        A = H + lam * np.diag(np.diag(H))
        L = np.zeros((n, n))
        ok = True
        for j in range(n):
            dj = A[j, j] - L[j, :j] @ L[j, :j]
            if not dj > PIVOT_TOL * A[j, j]:
                ok = False
                break
            L[j, j] = np.sqrt(dj)
            L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
        if ok:
            delta = np.linalg.solve(L.T, np.linalg.solve(L, -g))
            xt = (x.astype(np.float64) + delta).astype(np.float32)
            ks = step_down(xt[:p].astype(np.float64)) + step_down(-xt[p:].astype(np.float64))
            if all(abs(k) < KAPPA_MAX for k in ks):
                return xt, lam
        lam *= 10.0
    return None, lam


def lm(e, obs, T: int, p: int, q: int, x0, max_iter: int = 0, gap_jacobian: bool = True):
    """LM of section 2 item 16 from the fp32 point x0 -> dict(x (fp32), S0, S, stop, iters, n_acc, path (S after every
    pass), n_C)"""
    max_iter = max_iter or ITER_DEFAULT
    x = np.asarray(x0, dtype=np.float32).copy()
    xt = x
    lam, S, S0, passes, n_acc, stop = LAMBDA0, 0.0, np.nan, 0, 0, 0
    H = g = None
    path = []
    n_C = 0
    while True:
        Sn, J, eps, C = css_eval(e, obs, T, p, q, xt, gap_jacobian)
        n_C = int(C.sum())
        passes += 1
        conv = False
        if passes == 1:
            take, S0 = True, Sn
        else:
            take = Sn < S
            conv = take and S - Sn <= RTOL * S
        if take:
            if passes > 1:
                n_acc += 1
                lam /= 10.0
                x = xt
            S = Sn
            H, g = J[C].T @ J[C], J[C].T @ eps[C]
        else:
            lam *= 10.0
        path.append(S)
        if conv:
            stop = 1
        elif lam > LAMBDA_MAX:
            stop = 2
        elif passes >= max_iter:
            stop = 3
        if not stop:
            xt, lam = _step(H, g, x, p, q, lam)
            if xt is None:
                stop = 2
        if stop:
            return dict(x=x, S0=S0, S=S, stop=stop, iters=passes, n_acc=n_acc, path=path, n_C=n_C)


def css_bound(e, obs, T: int, p: int, q: int, x, tau):
    """first-order bound on |S_gpu - S_oracle| at the same x from a per-row error tau of e (the fp32 residuals): eps~
    moves by at most be_s = sum_k |h_k| (tau + sum |phi_j| bu_{s-j}) with h the impulse response of 1 / (1 + theta(z))
    (bu = tau on observed rows, the filled value's bound elsewhere), so |dS| <= sum over C of 2 |eps~_s| be_s + be_s^2,
    plus the float64 rounding of the recursion and the sum; x 2"""
    x = np.asarray(x, dtype=np.float64)
    phi, th = np.abs(x[:p]), np.abs(x[p:p + q])
    _, u, eps = recursion(e, obs, T, x[:p], x[p:p + q], T)
    bu = np.zeros(T + AR_MAX)
    be = np.zeros(T + MA_MAX)
    for s in range(T):
        ar_b = sum(phi[j] * bu[AR_MAX + s - 1 - j] for j in range(p))
        ma_b = sum(th[j] * be[MA_MAX + s - 1 - j] for j in range(q))
        if obs[s]:
            be[MA_MAX + s] = tau + ar_b + ma_b
            bu[AR_MAX + s] = tau
        else:
            bu[AR_MAX + s] = ar_b + ma_b
    be = be[MA_MAX:]
    C = np.asarray(obs[:T], dtype=bool).copy()
    C[:p] = False
    S = float(eps[C] @ eps[C])
    return 2.0 * float(np.sum(2.0 * np.abs(eps[C]) * be[C] + be[C] ** 2)) + 64 * 2.0 ** -52 * T * S


def fit_forecast_arma_css_packed(y, X, t_fit: int, pred_start: int, n_pred: int, p: int, q: int, d: int = 0,
                                 long_order: int = 0, max_iter: int = 0, gap_jacobian: bool = True, hr=None):
    """``arma_oracle.fit_forecast_arma_packed`` (or ``hr``, its result), then LM on every gated row from fp32 of its
    HR estimate -> that dict with pred / phi / theta / sigma replaced on the refined rows and css_start, css, css_stop,
    iters, refined [n], lm [n] (per-row ``lm`` results, None elsewhere)"""
    res = hr if hr is not None else fit_forecast_arma_packed(y, X, t_fit, pred_start, n_pred, p, q, d, long_order)
    res = dict(res)
    y = np.asarray(y, dtype=np.float64)[:, :t_fit]
    n = len(res["status"])
    T, end = res["T"], pred_start + n_pred
    endz = max(end - d, 0)
    pred, phi, theta, sigma = (np.array(res[k], dtype=np.float64) for k in ("pred", "phi", "theta", "sigma"))
    css_start, css, stop, iters = np.full(n, np.nan), np.full(n, np.nan), np.zeros(n, np.int32), np.zeros(n, np.int32)
    refined = np.zeros(n, dtype=bool)
    lms = [None] * n
    zhat = np.array(res["zhat"], dtype=np.float64)
    for i in np.flatnonzero(res["gated"]):
        x0 = np.r_[res["phi"][i, :p], res["theta"][i, :q]].astype(np.float32)
        r = lm(res["e"][i], res["obs"][i], T, p, q, x0, max_iter, gap_jacobian)
        lms[i] = r
        css_start[i], css[i], stop[i], iters[i] = r["S0"], r["S"], r["stop"], r["iters"]
        sigma[i] = np.sqrt(r["S"] / r["n_C"])
        if r["n_acc"] == 0:
            continue
        refined[i] = True
        x = r["x"].astype(np.float64)
        phi[i] = 0.0
        phi[i, :p] = x[:p]
        theta[i] = 0.0
        theta[i, :q] = x[p:]
        pr, _, _ = recursion(res["e"][i], res["obs"][i], T, x[:p], x[p:], endz)
        zhat[i, d:end] = res["fitted"][i, :endz] + pr
    if refined.any():
        if d == 0:
            pred[refined] = zhat[refined, pred_start:end]
        else:
            yh, _ = _integrate(zhat[refined], y[refined], np.isfinite(y[refined]), t_fit, d, end)
            pred[refined] = yh[:, pred_start:end]
    res.update(pred=pred, phi=phi, theta=theta, sigma=sigma, css_start=css_start, css=css, css_stop=stop, iters=iters,
               refined=refined, lm=lms, zhat=zhat)
    return res


def optimality_gap(e, obs, T: int, p: int, q: int, x):
    """relative decrease of S that SciPy's least_squares finds when started at x: (S(x) - S(x*)) / S(x), with x* kept
    inside the stationary / invertible region by the step-down test (0 when it leaves it)"""
    from scipy.optimize import least_squares

    x = np.asarray(x, dtype=np.float64)
    S0, _, _, C = css_eval(e, obs, T, p, q, x)

    def resid(z):
        _, _, eps, _ = css_eval(e, obs, T, p, q, z)
        return eps[C]

    def jac(z):
        _, J, _, _ = css_eval(e, obs, T, p, q, z)
        return J[C]

    sol = least_squares(resid, x, jac=jac, method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=400)
    ks = step_down(sol.x[:p]) + step_down(-sol.x[p:])
    if not all(abs(k) < KAPPA_MAX for k in ks):
        return 0.0
    S1 = float(sol.fun @ sol.fun)
    return max(S0 - S1, 0.0) / S0 if S0 > 0 else 0.0


__all__ = ["LAMBDA0", "LAMBDA_MAX", "RTOL", "ITER_DEFAULT", "ITER_MAX", "FP32_EPS", "css_eval", "two_filter_jacobian",
           "lm", "css_bound", "fit_forecast_arma_css_packed", "optimality_gap"]
