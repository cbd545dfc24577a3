"""float64 oracle of ARIMA(p, d, q) errors by exact Gaussian likelihood (DESIGN.md section 2 item 19), on top of
``arma_css_oracle``.

For a gated series: e_s, s < T, the residual of the plain fit (z' for d >= 1), x = (phi, theta) in the library's sign
convention, and the ARMA(p, q) model of e in Harvey's state-space form: r = max(p, q + 1), T with phi in its first
column and I on its superdiagonal, R = (1, theta_1 .. theta_{r-1}), Z = (1, 0 .. 0), no observation noise, sigma^2
concentrated out.
  start      P_{0|-1} the stationary covariance, (I - T (x) T) vec P = vec(R R') solved on the r (r + 1) / 2 symmetric
             unknowns by Gaussian elimination with partial pivoting; a pivot |u_kk| <= PIVOT_TOL x max |A| fails the
             solve.  d P_0 / dx solves the same system with the right-hand sides d(R R') + dT P T' + T P dT';
  filter     observed row: v = e - a_1, F = P_11, K = T P Z' / F, a <- T a + K v, P <- T P T' + R R' - K K' F;
             missing row: a <- T a, P <- T P T' + R R'; forward-mode derivatives of a, P, K by every parameter;
  objective  L = n log(S_w / n) + sum log F over the n observed rows, S_w = sum v^2 / F; loglik = -(L + n (1 + log
             2 pi)) / 2; sigma = sqrt(S_w / n);
  LM         on r_s = G v_s / sqrt(F_s), G = exp(sum log F / (2 n)): with D~ = d(v / sqrt F) and gamma = sum dF / F / (2 n),
             g = sum D~' v~ + S_w gamma and H = sum D~' D~ + gamma b' + b gamma' + S_w gamma gamma' (b = sum D~' v~): the
             Gauss-Newton system of r divided by G^2.  The objective is G^2 S_w = n exp(L / n).  The step rule is the
             CSS call's, and a trial point whose P_0 solve fails counts as a failed step-down (lam x 10, no pass).
``no_logdet`` and ``gap_as_zero`` restate the two negative-control builds.
"""
from __future__ import annotations

import numpy as np
from scipy.signal import lfilter

from ar_oracle import KAPPA_MAX
from arma_oracle import PIVOT_TOL, _integrate, recursion, step_down
from arma_css_oracle import ITER_DEFAULT, LAMBDA0, LAMBDA_MAX, RTOL, _step, fit_forecast_arma_css_packed

LOG2PI1 = 1.0 + np.log(2.0 * np.pi)


def state_dim(p: int, q: int) -> int:
    return max(p, q + 1)


def _pad(x, p: int, q: int):
    r = state_dim(p, q)
    x = np.asarray(x, dtype=np.float64)
    phi = np.zeros(r)
    phi[:p] = x[:p]
    R = np.zeros(r)
    R[0] = 1.0
    R[1:q + 1] = x[p:p + q]
    return r, phi, R


def _packed(r: int):
    """(i, j), i <= j, in the kernel's column-major packed order"""
    return [(i, j) for j in range(r) for i in range(j + 1)]


def _fold(r: int, phi):
    """the r (r + 1) / 2 square matrix of P - T P T' on the packed symmetric unknowns"""
    idx = {}
    for k, (i, j) in enumerate(_packed(r)):
        idx[(i, j)] = idx[(j, i)] = k
    N = r * (r + 1) // 2
    A = np.zeros((N, N))
    for k, (i, j) in enumerate(_packed(r)):
        A[k, k] += 1.0
        A[k, idx[(0, 0)]] -= phi[i] * phi[j]
        if j + 1 < r:
            A[k, idx[(0, j + 1)]] -= phi[i]
        if i + 1 < r:
            A[k, idx[(i + 1, 0)]] -= phi[j]
        if i + 1 < r and j + 1 < r:
            A[k, idx[(i + 1, j + 1)]] -= 1.0
    return A, idx


def _lu_ok(A):
    """partial-pivoting elimination of A: False when a pivot |u_kk| <= PIVOT_TOL x max |A|"""
    U = A.copy()
    N = len(U)
    amax = np.abs(A).max()
    for k in range(N):
        piv = k + int(np.argmax(np.abs(U[k:, k])))
        if not abs(U[piv, k]) > PIVOT_TOL * amax:
            return False
        U[[k, piv]] = U[[piv, k]]
        U[k + 1:, k:] -= np.outer(U[k + 1:, k] / U[k, k], U[k, k:])
    return True


def p0_solve(x, p: int, q: int):
    """-> (P0 [r, r], dP0 [p + q, r, r]) or None when the solve fails"""
    r, phi, R = _pad(x, p, q)
    A, idx = _fold(r, phi)
    if not _lu_ok(A):
        return None
    pk = _packed(r)
    unf = lambda u: np.array([[u[idx[(i, j)]] for j in range(r)] for i in range(r)])
    P0 = unf(np.linalg.solve(A, np.array([R[i] * R[j] for i, j in pk])))
    M = phi * P0[0, 0] + np.r_[P0[1:, 0], 0.0]                 # T P Z'
    n = p + q
    dP0 = np.zeros((n, r, r))
    for l in range(n):
        dphi, dR = np.zeros(r), np.zeros(r)
        if l < p:
            dphi[l] = 1.0
        else:
            dR[l - p + 1] = 1.0
        rhs = np.array([dR[i] * R[j] + R[i] * dR[j] + dphi[i] * M[j] + M[i] * dphi[j] for i, j in pk])
        dP0[l] = unf(np.linalg.solve(A, rhs))
    return P0, dP0


def ml_eval(e, obs, T: int, p: int, q: int, x, no_logdet: bool = False, gap_as_zero: bool = False):
    """-> dict(ok, L, loglik, obj (G^2 S_w), S_w, sum_logF, n, sigma, g, H, r (the scaled innovations), Jr (d r / dx))
    at x; ok False (and nothing else) when the P_0 solve fails"""
    sol = p0_solve(x, p, q)
    if sol is None:
        return dict(ok=False)
    P, dP = sol
    r, phi, R = _pad(x, p, q)
    n = p + q
    Tm = np.zeros((r, r))
    Tm[:, 0] = phi
    Tm[np.arange(r - 1), np.arange(1, r)] = 1.0
    dT, dR = np.zeros((n, r, r)), np.zeros((n, r))
    for l in range(n):
        if l < p:
            dT[l, l, 0] = 1.0
        else:
            dR[l, l - p + 1] = 1.0
    a, da = np.zeros(r), np.zeros((n, r))
    Sw, slf, nobs = 0.0, 0.0, 0
    dlf = np.zeros(n)
    vt, Dt = [], []
    RR = np.outer(R, R)
    dRR = np.einsum("li,j->lij", dR, R) + np.einsum("i,lj->lij", R, dR)
    for s in range(T):
        o = bool(obs[s]) or gap_as_zero
        es = float(e[s]) if obs[s] else 0.0
        TPT = Tm @ P @ Tm.T
        dTPT = (np.einsum("lik,kj->lij", dT, P @ Tm.T) + np.einsum("ik,lkj->lij", Tm @ P, dT.transpose(0, 2, 1))
                + np.einsum("ik,lkm,jm->lij", Tm, dP, Tm))
        if o:
            F = P[0, 0]
            dF = dP[:, 0, 0]
            M = Tm @ P[:, 0]
            dM = np.einsum("lik,k->li", dT, P[:, 0]) + np.einsum("ik,lk->li", Tm, dP[:, :, 0])
            K = M / F
            dK = (dM - np.outer(dF, K)) / F
            v = es - a[0]
            dv = -da[:, 0]
            sF = np.sqrt(F)
            vt.append(v / sF)
            Dt.append(dv / sF - (v / sF) * dF / (2.0 * F))
            Sw += v * v / F
            slf += np.log(F)
            dlf += dF / F
            nobs += 1
            a_n = Tm @ a + K * v
            da_n = np.einsum("lik,k->li", dT, a) + da @ Tm.T + np.outer(dv, K) + dK * v
            P_n = TPT + RR - F * np.outer(K, K)
            dP_n = (dTPT + dRR - F * (np.einsum("li,j->lij", dK, K) + np.einsum("i,lj->lij", K, dK))
                    - dF[:, None, None] * np.outer(K, K)[None])
        else:
            a_n = Tm @ a
            da_n = np.einsum("lik,k->li", dT, a) + da @ Tm.T
            P_n, dP_n = TPT + RR, dTPT + dRR
        a, da, P, dP = a_n, da_n, P_n, dP_n
    vt, Dt = np.array(vt), np.array(Dt).reshape(len(vt), n)
    if no_logdet:
        slf, dlf = 0.0, np.zeros(n)
    L = nobs * np.log(Sw / nobs) + slf
    gam = dlf / (2.0 * nobs)
    b = Dt.T @ vt
    H = Dt.T @ Dt + np.outer(gam, b) + np.outer(b, gam) + Sw * np.outer(gam, gam)
    g = b + Sw * gam
    G = np.exp(slf / (2.0 * nobs))
    return dict(ok=True, L=L, loglik=-0.5 * (L + nobs * LOG2PI1), obj=G * G * Sw, S_w=Sw, sum_logF=slf, n=nobs,
                sigma=np.sqrt(Sw / nobs), g=g, H=H, r=G * vt, Jr=G * (Dt + np.outer(vt, gam)))


def lm(e, obs, T: int, p: int, q: int, x0, max_iter: int = 0, no_logdet: bool = False, gap_as_zero: bool = False):
    """LM of section 2 item 19 from the fp32 point x0 -> dict(x (fp32), ok (P_0 at x0 solved), L0, L, loglik0, loglik,
    sigma, stop, iters, n_acc, path (L of the accepted point after every pass))"""
    max_iter = max_iter or ITER_DEFAULT
    x = np.asarray(x0, dtype=np.float32).copy()
    xt = x
    lam, passes, n_acc, stop = LAMBDA0, 0, 0, 0
    cur = first = None
    path = []
    while True:
        ev = ml_eval(e, obs, T, p, q, xt, no_logdet, gap_as_zero)
        if not ev["ok"]:
            if passes == 0:
                return dict(x=x, ok=False, L0=np.nan, L=np.nan, loglik0=np.nan, loglik=np.nan, sigma=np.nan, stop=0,
                            iters=0, n_acc=0, path=[])
            lam *= 10.0                        # a failed step-down: no pass
            xt = None
            if lam <= LAMBDA_MAX:
                xt, lam = _step(cur["H"], cur["g"], x, p, q, lam)
            if xt is None:
                stop = 2
                break
            continue
        passes += 1
        conv = False
        if passes == 1:
            take = True
            first = ev
        else:
            take = ev["obj"] < cur["obj"]
            conv = take and cur["obj"] - ev["obj"] <= RTOL * cur["obj"]
        if take:
            if passes > 1:
                n_acc += 1
                lam /= 10.0
                x = xt
            cur = ev
        else:
            lam *= 10.0
        path.append(cur["L"])
        if conv:
            stop = 1
        elif lam > LAMBDA_MAX:
            stop = 2
        elif passes >= max_iter:
            stop = 3
        if not stop:
            xt, lam = _step(cur["H"], cur["g"], x, p, q, lam)
            if xt is None:
                stop = 2
        if stop:
            break
    return dict(x=x, ok=True, L0=first["L"], L=cur["L"], loglik0=first["loglik"], loglik=cur["loglik"],
                sigma=cur["sigma"], stop=stop, iters=passes, n_acc=n_acc, path=path)


def dense_loglik(e, obs, T: int, p: int, q: int, x, n_psi: int = 200000):
    """the exact Gaussian log-likelihood of the observed rows with sigma^2 concentrated out, from the Toeplitz
    autocovariance of the psi-weights (independent of P_0 and of the filter)"""
    x = np.asarray(x, dtype=np.float64)
    imp = np.zeros(n_psi)
    imp[0] = 1.0
    psi = lfilter(np.r_[1.0, x[p:p + q]], np.r_[1.0, -x[:p]], imp)
    acov = np.array([psi[:n_psi - h] @ psi[h:] for h in range(T)])
    idx = np.flatnonzero(np.asarray(obs[:T], dtype=bool))
    Sig = acov[np.abs(idx[:, None] - idx[None, :])]
    ev = np.asarray(e, dtype=np.float64)[idx]
    Lc = np.linalg.cholesky(Sig)
    w = np.linalg.solve(Lc, ev)
    n = len(idx)
    L = n * np.log(w @ w / n) + 2.0 * np.log(np.diag(Lc)).sum()
    return -0.5 * (L + n * LOG2PI1)


def fit_forecast_arma_ml_packed(y, X, t_fit: int, pred_start: int, n_pred: int, p: int, q: int, d: int = 0,
                                long_order: int = 0, max_iter: int = 0, css=None):
    """``arma_css_oracle.fit_forecast_arma_css_packed`` (or ``css``, its result), then ML on every gated row from fp32 of
    its CSS estimate -> that dict with pred / phi / theta / sigma replaced where section 2 item 19 says, and
    loglik_start, loglik, ml_stop, ml_iters, ml_refined [n], ml [n] (per-row ``lm`` results)"""
    res = css if css is not None else fit_forecast_arma_css_packed(y, X, t_fit, pred_start, n_pred, p, q, d, long_order,
                                                                   max_iter)
    res = dict(res)
    y = np.asarray(y, dtype=np.float64)[:, :t_fit]
    n = len(res["status"])
    T, end = res["T"], pred_start + n_pred
    endz = max(end - d, 0)
    pred, phi, theta, sigma = (np.array(res[k], dtype=np.float64) for k in ("pred", "phi", "theta", "sigma"))
    ll0, ll = np.full(n, np.nan), np.full(n, np.nan)
    stop, iters = np.zeros(n, np.int32), np.zeros(n, np.int32)
    refined = np.zeros(n, dtype=bool)
    mls = [None] * n
    zhat = np.array(res["zhat"], dtype=np.float64)
    for i in np.flatnonzero(res["gated"]):
        x0 = np.r_[res["phi"][i, :p], res["theta"][i, :q]].astype(np.float32)
        r = lm(res["e"][i], res["obs"][i], T, p, q, x0, max_iter)
        mls[i] = r
        if not r["ok"]:
            continue
        ll0[i], ll[i], stop[i], iters[i] = r["loglik0"], r["loglik"], r["stop"], r["iters"]
        sigma[i] = r["sigma"]
        if r["n_acc"] == 0:
            continue
        refined[i] = True
        xs = r["x"].astype(np.float64)
        phi[i] = 0.0
        phi[i, :p] = xs[:p]
        theta[i] = 0.0
        theta[i, :q] = xs[p:]
        pr, _, _ = recursion(res["e"][i], res["obs"][i], T, xs[:p], xs[p:], endz)
        zhat[i, d:end] = res["fitted"][i, :endz] + pr
    if refined.any():
        if d == 0:
            pred[refined] = zhat[refined, pred_start:end]
        else:
            yh, _ = _integrate(zhat[refined], y[refined], np.isfinite(y[refined]), t_fit, d, end)
            pred[refined] = yh[:, pred_start:end]
    res.update(pred=pred, phi=phi, theta=theta, sigma=sigma, loglik_start=ll0, loglik=ll, ml_stop=stop, ml_iters=iters,
               ml_refined=refined, ml=mls, zhat=zhat)
    return res


def optimum(e, obs, T: int, p: int, q: int, x):
    """the smallest L SciPy's Nelder-Mead and BFGS find from x inside the stationary / invertible region -> (L*, x*)"""
    from scipy.optimize import minimize

    def f(z):
        ks = step_down(z[:p]) + step_down(-z[p:])
        if not all(abs(k) < KAPPA_MAX for k in ks):
            return np.inf
        ev = ml_eval(e, obs, T, p, q, z)
        return ev["L"] if ev["ok"] else np.inf

    x = np.asarray(x, dtype=np.float64)
    best, bx = f(x), x
    for method in ("Nelder-Mead", "BFGS"):
        opts = dict(xatol=1e-10, fatol=1e-12, maxiter=4000) if method == "Nelder-Mead" else dict(gtol=1e-10)
        sol = minimize(f, bx, method=method, options=opts)
        if np.isfinite(sol.fun) and sol.fun < best:
            best, bx = float(sol.fun), sol.x
    return best, bx


__all__ = ["state_dim", "p0_solve", "ml_eval", "lm", "dense_loglik", "fit_forecast_arma_ml_packed", "optimum"]
