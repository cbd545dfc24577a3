"""float64 oracle of regression with ARIMA(p, d, q) errors, beta estimated jointly with (phi, theta) by conditional least
squares (DESIGN.md section 2 item 17), on top of ``arma_oracle`` (HR, the recursion, integration), ``arma_css_oracle``
(the step rules and constants) and ``mmf_oracle`` (the plain fit).

For a gated series: A the whitened design of the plan the call fits (X W for d = 0, D_d W_D for d >= 1), gamma0 the
plain fit's whitened coefficients, J the used columns (kept, non-zero on an observed fit row), and
  x          (phi_1..phi_p, theta_1..theta_q, gamma_j for j in J), gamma off J held at gamma0;
  residual   e_s(gamma) = z_s - A_s gamma on the observed fit rows;
  objective  S(x) = sum over C = {s in [p, T): observed} of eps~_s(x)^2, eps~ the recursion of ``arma_css_oracle``;
  Jacobian   the (phi, theta) columns as ``arma_css_oracle.css_eval``; a gamma_j column through the same recursion:
             d pr_s = sum phi_k d u~_{s-k} + sum theta_k d eps~_{s-k}, on an observed row d u~_s = -A_{s,j} and
             d eps~_s = -A_{s,j} - d pr_s, on a missing row d u~_s = d pr_s and d eps~_s = 0.  ``white_beta=True`` is the
             negative control's rule: d eps~_s = -A_{s,j} on observed rows and 0 elsewhere, no recursion;
  LM         ``arma_css_oracle.lm``'s rules on the (n_x + 1)-square system, the step-down tests on (phi, theta) only.
The library's gamma carries a centring constant c next to it (fitted = c + a . gamma); c lies in the span of the
intercept column, so the optimum over the used columns, S and beta are the same either way.
"""
from __future__ import annotations

import numpy as np

from ar_oracle import AR_MAX, KAPPA_MAX
from arma_css_oracle import ITER_DEFAULT, LAMBDA0, LAMBDA_MAX, RTOL
from arma_oracle import MA_MAX, PIVOT_TOL, _integrate, fit_forecast_arma_packed, recursion, step_down
from oracle import mmf_oracle as O


def used_cols(A_fit, obs, kept):
    """J: kept columns non-zero on an observed fit row"""
    nz = (np.asarray(A_fit)[np.asarray(obs, dtype=bool)] != 0.0).any(axis=0)
    return np.flatnonzero(np.asarray(kept, dtype=bool) & nz)


def residuals(z, obs, A_fit, gamma):
    """e [T] of one series: z - A gamma on the observed rows, 0 elsewhere"""
    T = len(obs)
    return np.where(obs, np.where(obs, z[:T], 0.0) - A_fit[:T] @ gamma, 0.0)


def joint_eval(z, obs, A_fit, T: int, p: int, q: int, x, g0, cols, white_beta: bool = False):
    """-> (S, J [T, p + q + |cols|], eps~ [T], C [T] bool) of one series at x; gamma = g0 with x[p + q:] on cols.  The
    (phi, theta) columns are ``arma_css_oracle.css_eval``'s, computed by the same operations"""
    x = np.asarray(x, dtype=np.float64)
    nreg, ng = p + q, len(cols)
    phi, th = x[:p], x[p:nreg]
    gamma = np.array(g0, dtype=np.float64)
    gamma[cols] = x[nreg:]
    e = residuals(z, obs, A_fit, gamma)
    u = np.zeros(T + AR_MAX)
    ep = np.zeros(T + MA_MAX)
    du = np.zeros((T + AR_MAX, nreg))
    de = np.zeros((T + MA_MAX, nreg))
    dug = np.zeros((T + AR_MAX, ng))
    deg = np.zeros((T + MA_MAX, ng))
    J = np.zeros((T, nreg + ng))
    for s in range(T):
        ul = u[AR_MAX + s - 1 - np.arange(p)] if p else np.zeros(0)
        el = ep[MA_MAX + s - 1 - np.arange(q)] if q else np.zeros(0)
        pr = phi @ ul + th @ el
        dpr = np.concatenate([ul, el])
        dprg = np.zeros(ng)
        if p:
            dpr = dpr + phi @ du[AR_MAX + s - 1 - np.arange(p)]
            dprg = dprg + phi @ dug[AR_MAX + s - 1 - np.arange(p)]
        if q:
            dpr = dpr + th @ de[MA_MAX + s - 1 - np.arange(q)]
            dprg = dprg + th @ deg[MA_MAX + s - 1 - np.arange(q)]
        a = A_fit[s, cols]
        if obs[s]:
            u[AR_MAX + s] = e[s]
            ep[MA_MAX + s] = e[s] - pr
            de[MA_MAX + s] = -dpr
            if white_beta:
                deg[MA_MAX + s] = -a
            else:
                dug[AR_MAX + s] = -a
                deg[MA_MAX + s] = -a - dprg
        else:
            u[AR_MAX + s] = pr
            du[AR_MAX + s] = dpr
            if not white_beta:
                dug[AR_MAX + s] = dprg
        J[s, :nreg] = de[MA_MAX + s]
        J[s, nreg:] = deg[MA_MAX + s]
    eps = ep[MA_MAX:]
    C = np.asarray(obs[:T], dtype=bool).copy()
    C[:p] = False
    return float(eps[C] @ eps[C]), J, eps, C


def _step(H, g, x, p: int, q: int, lam: float):
    """``arma_css_oracle._step`` with the step-down tests on (phi, theta) only"""
    n = len(g)
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
            ks = step_down(xt[:p].astype(np.float64)) + step_down(-xt[p:p + q].astype(np.float64))
            if all(abs(k) < KAPPA_MAX for k in ks):
                return xt, lam
        lam *= 10.0
    return None, lam


def lm_joint(z, obs, A_fit, T: int, p: int, q: int, x0, g0, cols, max_iter: int = 0, white_beta: bool = False):
    """LM of section 2 item 17 from the fp32 point x0 -> dict(x (fp32), S0, S, stop, iters, n_acc, path, acc, n_C),
    ``arma_css_oracle.lm``'s fields"""
    max_iter = max_iter or ITER_DEFAULT
    x = np.asarray(x0, dtype=np.float32).copy()
    xt = x
    lam, S, S0, passes, n_acc, stop = LAMBDA0, 0.0, np.nan, 0, 0, 0
    H = g = None
    path, acc = [], []
    n_C = 0
    while True:
        Sn, J, eps, C = joint_eval(z, obs, A_fit, T, p, q, xt, g0, cols, white_beta)
        n_C = int(C.sum())
        passes += 1
        conv = False
        if passes == 1:
            take, S0 = True, Sn
        else:
            take = Sn < S
            conv = take and S - Sn <= RTOL * S
            acc.append(bool(take))
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
            return dict(x=x, S0=S0, S=S, stop=stop, iters=passes, n_acc=n_acc, path=path, acc=acc, n_C=n_C)


def optimality_gap(z, obs, A_fit, T: int, p: int, q: int, x, g0, cols):
    """relative decrease of S that SciPy's least_squares finds when started at x over the full vector (phi, theta,
    gamma_J): (S(x) - S(x*)) / S(x), x* kept inside the stationary / invertible region (0 when it leaves it)"""
    from scipy.optimize import least_squares

    x = np.asarray(x, dtype=np.float64)
    S0, _, _, C = joint_eval(z, obs, A_fit, T, p, q, x, g0, cols)

    def resid(v):
        return joint_eval(z, obs, A_fit, T, p, q, v, g0, cols)[2][C]

    def jac(v):
        return joint_eval(z, obs, A_fit, T, p, q, v, g0, cols)[1][C]

    sol = least_squares(resid, x, jac=jac, method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=400)
    ks = step_down(sol.x[:p]) + step_down(-sol.x[p:p + q])
    if not all(abs(k) < KAPPA_MAX for k in ks):
        return 0.0
    S1 = float(sol.fun @ sol.fun)
    return max(S0 - S1, 0.0) / S0 if S0 > 0 else 0.0


def plan_of(y, X, t_fit: int, d: int):
    """(z [n, T] the modelled series, Dm [rows - d, P] its design, W, kept, A_fit [T, P], gamma0 [n, P]) of the plan a
    call with differencing order d fits"""
    y = np.asarray(y, dtype=np.float64)[:, :t_fit]
    X = np.asarray(X, dtype=np.float64)
    if d == 0:
        z, Dm = y, X
    else:
        from arima_oracle import diff_design
        z = y.copy()
        for _ in range(d):
            z = z[:, 1:] - z[:, :-1]
        Dm = diff_design(X, t_fit, d)
    T = t_fit - d
    W, kept = O.whiten(Dm[:T])
    A = Dm @ W
    _, _, gamma0, _ = O.fit_forecast_packed(z, Dm, T, 0, 1, return_gamma=True)
    return z, Dm, W, kept, A, gamma0


def fit_forecast_arma_joint_packed(y, X, t_fit: int, pred_start: int, n_pred: int, p: int, q: int, d: int = 0,
                                   long_order: int = 0, max_iter: int = 0, white_beta: bool = False, hr=None):
    """``arma_oracle.fit_forecast_arma_packed`` (or ``hr``), then ``lm_joint`` on every gated row from (its HR (phi,
    theta), gamma0 on J), fp32 -> that dict with pred / phi / theta / sigma replaced on the refined rows, and css_start,
    css, css_stop, iters, refined [n], beta [n, P] (W gamma of the shipped gamma; NaN for empty rows), gamma [n, P],
    cols [n] (J), lm [n]"""
    res = hr if hr is not None else fit_forecast_arma_packed(y, X, t_fit, pred_start, n_pred, p, q, d, long_order)
    res = dict(res)
    yl = np.asarray(y, dtype=np.float64)[:, :t_fit]
    z, Dm, W, kept, A, gamma0 = plan_of(y, X, t_fit, d)
    n = len(res["status"])
    T, end = res["T"], pred_start + n_pred
    endz = max(end - d, 0)
    obs_all = np.isfinite(z)
    pred, phi, theta, sigma = (np.array(res[k], dtype=np.float64) for k in ("pred", "phi", "theta", "sigma"))
    css_start, css, stop, iters = np.full(n, np.nan), np.full(n, np.nan), np.zeros(n, np.int32), np.zeros(n, np.int32)
    refined = np.zeros(n, dtype=bool)
    gamma = gamma0.copy()
    lms, colss = [None] * n, [np.zeros(0, dtype=np.int64)] * n
    zhat = np.array(res["zhat"], dtype=np.float64)
    for i in np.flatnonzero(res["gated"]):
        obs = obs_all[i, :T]
        cols = used_cols(A[:T], obs, kept)
        colss[i] = cols
        x0 = np.r_[res["phi"][i, :p], res["theta"][i, :q], gamma0[i, cols]].astype(np.float32)
        g0 = gamma0[i]
        r = lm_joint(z[i], obs, A[:T], T, p, q, x0, g0, cols, max_iter, white_beta)
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
        theta[i, :q] = x[p:p + q]
        gamma[i, cols] = x[p + q:]
        e = residuals(z[i], obs, A[:T], gamma[i])
        pr, _, _ = recursion(e, obs, T, x[:p], x[p:p + q], endz)
        zhat[i, d:end] = A[:endz] @ gamma[i] + pr
    if refined.any():
        if d == 0:
            pred[refined] = zhat[refined, pred_start:end]
        else:
            yh, _ = _integrate(zhat[refined], yl[refined], np.isfinite(yl[refined]), t_fit, d, end)
            pred[refined] = yh[:, pred_start:end]
    beta = gamma @ W.T
    beta[np.asarray(res["status"]) == 1] = np.nan
    res.update(pred=pred, phi=phi, theta=theta, sigma=sigma, css_start=css_start, css=css, css_stop=stop, iters=iters,
               refined=refined, lm=lms, zhat=zhat, beta=beta, gamma=gamma, gamma0=gamma0, cols=colss, A=A, W=W, z=z)
    return res


__all__ = ["used_cols", "residuals", "joint_eval", "lm_joint", "optimality_gap", "plan_of",
           "fit_forecast_arma_joint_packed"]
