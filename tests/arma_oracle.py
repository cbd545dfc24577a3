"""float64 oracle of regression with ARIMA(p, d, q) errors (DESIGN.md section 2 item 13), on top of ``ar_oracle`` and
``arima_oracle``.

For series i: the fit the ARIMA(p, d, 0) oracle builds (d = 0: ``ar_oracle.fit_forecast_ar_packed`` on y; d >= 1:
``arima_oracle.fit_forecast_arima_packed`` on z'), its residuals e on the observed fit rows t < T, and Hannan-Rissanen:
  step 1  r_0..r_m over n_obs, the dof rule with order m, Levinson-Durbin with the kappa stop -> psi, m_i; the filled
          long-AR residuals u^L (e where observed, the AR prediction elsewhere, 0 before row 0); eps^ = e - psi . u^L lags;
  step 2  rows R = {t in [m + q, T): e observed at t .. t - max(p, q)}, e_t on (e_{t-1..t-p}, eps^_{t-1..t-q}) by the
          normal equations and an in-order Cholesky;
  gate    m_i >= 1, |R| > p + q, pivots > PIVOT_TOL x diagonal, step-down |kappa| < KAPPA_MAX for 1 - phi(z) and 1 + theta(z);
  forecast the recursion from s = 0 (pr_s = phi . u lags + theta . eps~ lags; observed fit rows u = e, eps~ = e - pr;
          elsewhere u = pr, eps~ = 0), c + a.gamma + pr, integrated to levels as ``arima_oracle`` does for d >= 1.
A series that fails the gate is the ARIMA(p, d, 0) oracle's row, with ma_order 0 and theta 0.

``coef_bound`` and ``pred_bound`` are the first-order bounds the GPU tests hold the library's gated rows to (DESIGN.md
section 6).
"""
from __future__ import annotations

import math

import numpy as np

from ar_oracle import AR_MAX, FP32_EPS, KAPPA_MAX, autocov, fit_forecast_ar_packed
from arima_oracle import fit_forecast_arima_packed

MA_MAX = 4
HR_LONG_MAX = 32
PIVOT_TOL = 1e-5


def default_long_order(t_fit_z: int, p: int, q: int) -> int:
    """min(32, max(2 max(p, q), floor(ln(T)^2))), T the fit rows of the modelled series"""
    lt = math.log(t_fit_z)
    return min(HR_LONG_MAX, max(2 * max(p, q), int(math.floor(lt * lt))))


def levinson_long(r, m: int):
    """Levinson-Durbin on r_0..r_m with the kappa stop -> (psi [m], completed order, kappas reached)"""
    psi = np.zeros(max(m, 1))
    kappas = []
    var = float(r[0])
    if not r[0] > 0.0:
        return psi, 0, kappas
    order = 0
    for j in range(1, m + 1):
        kap = (r[j] - psi[:j - 1] @ r[j - 1:0:-1]) / var
        kappas.append(float(kap))
        if abs(kap) >= KAPPA_MAX:
            break
        prev = psi[:j - 1].copy()
        psi[:j - 1] = prev - kap * prev[::-1]
        psi[j - 1] = kap
        var *= 1.0 - kap * kap
        order = j
    return psi, order, kappas


def step_down(a):
    """kappas of the step-down (reverse Levinson) recursion of 1 - sum_j a_j z^j, highest stage first; it stops after
    the first |kappa| >= KAPPA_MAX"""
    a = [float(v) for v in a]
    ks = []
    for j in range(len(a), 0, -1):
        kap = a[j - 1]
        ks.append(kap)
        if not abs(kap) < KAPPA_MAX:
            break
        den = 1.0 - kap * kap
        a = [(a[i] + kap * a[j - 2 - i]) / den for i in range(j - 1)]
    return ks


def cholesky_in_order(G):
    """in-order Cholesky -> (L or None, the smallest pivot / diagonal ratio reached)"""
    n = G.shape[0]
    L = np.zeros((n, n))
    worst = np.inf
    for j in range(n):
        d = G[j, j] - L[j, :j] @ L[j, :j]
        ratio = d / G[j, j] if G[j, j] > 0 else -np.inf
        worst = min(worst, ratio)
        if not d > PIVOT_TOL * G[j, j]:
            return None, worst
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (G[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L, worst


def hr_rows(e, obs, T: int, m: int, p: int, q: int, gappy: bool = False):
    """the rows R as a boolean [T] (gappy: every observed t >= m + q, the control build's rule)"""
    L = max(p, q)
    R = np.zeros(T, dtype=bool)
    for t in range(m + q, T):
        R[t] = obs[t] if gappy else bool(obs[t - L:t + 1].all())
    return R


def hannan_rissanen(e, obs, T: int, dof: int, p: int, q: int, m: int, gappy: bool = False):
    """Hannan-Rissanen on one series' residuals e [T] (0 where missing) -> dict(ok, beta, psi, m_i, r, kappas_long,
    uL, eps_hat, R, G, b, n_R, pivot, kappas_step)"""
    e = np.asarray(e, dtype=np.float64)[:T]
    obs = np.asarray(obs, dtype=bool)[:T]
    r = autocov(e, obs, T, m)
    res = dict(ok=False, beta=np.zeros(p + q), psi=np.zeros(m), m_i=0, r=r, kappas_long=[], uL=None, eps_hat=None,
               R=None, G=None, b=None, n_R=0, pivot=np.inf, kappas_step=[])
    if dof <= m:
        return res
    psi, m_i, kl = levinson_long(r, m)
    res.update(psi=psi[:m], m_i=m_i, kappas_long=kl)
    if m_i < 1:
        return res
    uL = np.zeros(T + m)                                   # uL[m + s] = u^L_s; the first m entries are s < 0
    eh = np.zeros(T)
    for s in range(T):
        lag = uL[m + s - 1::-1][:m] if m + s - 1 >= 0 else np.zeros(m)
        a = psi[:m] @ lag[:m]
        if obs[s]:
            uL[m + s] = e[s]
            eh[s] = e[s] - a
        else:
            uL[m + s] = a
    R = hr_rows(e, obs, T, m, p, q, gappy)
    ts = np.flatnonzero(R)
    n = p + q
    Xr = np.zeros((len(ts), n))
    for j in range(p):
        Xr[:, j] = e[ts - 1 - j]
    for j in range(q):
        Xr[:, p + j] = eh[ts - 1 - j]
    yr = e[ts]
    G = Xr.T @ Xr
    b = Xr.T @ yr
    res.update(uL=uL[m:], eps_hat=eh, R=R, G=G, b=b, n_R=len(ts), X=Xr, target=yr)
    if len(ts) <= n:
        return res
    Lc, piv = cholesky_in_order(G)
    res["pivot"] = piv
    if Lc is None:
        return res
    beta = np.linalg.solve(Lc.T, np.linalg.solve(Lc, b))
    ks = step_down(beta[:p]) + step_down(-beta[p:])
    res.update(beta=beta, kappas_step=ks, ok=all(abs(k) < KAPPA_MAX for k in ks))
    return res


def recursion(e, obs, T: int, phi, theta, end: int):
    """pr [end], u [end], eps~ [end] of the ARMA recursion from s = 0 (never restarted)"""
    p, q = len(phi), len(theta)
    u = np.zeros(end + AR_MAX)
    ep = np.zeros(end + MA_MAX)
    pr = np.zeros(end)
    for s in range(end):
        a = sum(phi[j] * u[AR_MAX + s - 1 - j] for j in range(p)) + sum(theta[j] * ep[MA_MAX + s - 1 - j]
                                                                        for j in range(q))
        pr[s] = a
        if s < T and obs[s]:
            u[AR_MAX + s] = e[s]
            ep[MA_MAX + s] = e[s] - a
        else:
            u[AR_MAX + s] = a
    return pr, u[AR_MAX:], ep[MA_MAX:]


def _integrate(zhat, y, obs, t_fit: int, d: int, end: int):
    """levels from zhat at level rows (NaN for t < d), the filled levels of arima_oracle"""
    n = zhat.shape[0]
    yt = np.full((n, end), np.nan)
    yh = np.full((n, end), np.nan)
    for t in range(end):
        if t >= d:
            yh[:, t] = zhat[:, t] + yt[:, t - 1] if d == 1 else zhat[:, t] + 2.0 * yt[:, t - 1] - yt[:, t - 2]
        keep = obs[:, t] if t < t_fit else np.zeros(n, dtype=bool)
        yt[:, t] = np.where(keep, y[:, t] if t < t_fit else 0.0, yh[:, t])
    return yh, yt


def fit_forecast_arma_packed(y, X, t_fit: int, pred_start: int, n_pred: int, p: int, q: int, d: int = 0,
                             long_order: int = 0, gappy: bool = False):
    """-> dict(pred [n, n_pred], status, phi [n, AR_MAX], theta [n, MA_MAX], order, ma_order, sigma, hr [n] per-series
    Hannan-Rissanen results, base (the ARIMA(p, d, 0) oracle's result), e [n, T], obs [n, T], fitted [n, rows of the
    modelled series], T, m, d, and for the gated rows pr / u / eps [n, end - d])"""
    y = np.asarray(y, dtype=np.float64)[:, :t_fit]
    end = pred_start + n_pred
    if d == 0:
        base = fit_forecast_ar_packed(y, X, t_fit, pred_start, n_pred, p)
        zr = base
    else:
        base = fit_forecast_arima_packed(y, X, t_fit, pred_start, n_pred, p, d)
        zr = base["zres"]
    T = t_fit - d
    m = long_order or default_long_order(T, p, q)
    n = y.shape[0]
    e, zobs, status, dof, fitted = zr["e"], zr["obs"], zr["status"], zr["dof"], zr["fitted"]
    pred = np.array(base["pred"], dtype=np.float64)
    phi = np.array(base["phi"], dtype=np.float64)
    theta = np.zeros((n, MA_MAX))
    order = np.array(base["order"], dtype=np.int32)
    ma_order = np.zeros(n, dtype=np.int32)
    sigma = np.array(base["sigma"], dtype=np.float64)
    endz = max(end - d, 0)
    hr, prs, us, eps = [None] * n, np.zeros((n, endz)), np.zeros((n, endz)), np.zeros((n, endz))
    gated = np.zeros(n, dtype=bool)
    zhat = np.full((n, end), np.nan)
    for i in range(n):
        if status[i] == 1:
            continue
        h = hannan_rissanen(e[i], zobs[i], T, int(dof[i]), p, q, m, gappy)
        hr[i] = h
        if not h["ok"]:
            continue
        gated[i] = True
        ph, th = h["beta"][:p], h["beta"][p:]
        prs[i], us[i], eps[i] = recursion(e[i], zobs[i], T, ph, th, endz)
        phi[i] = 0.0
        phi[i, :p] = ph
        theta[i, :q] = th
        order[i], ma_order[i] = p, q
        sigma[i] = np.sqrt(np.mean(eps[i][:T][h["R"]] ** 2))
        zhat[i, d:end] = fitted[i, :endz] + prs[i]
    if gated.any():
        if d == 0:
            pred[gated] = zhat[gated, pred_start:end]
        else:
            yh, _ = _integrate(zhat[gated], y[gated], np.isfinite(y[gated]), t_fit, d, end)
            pred[gated] = yh[:, pred_start:end]
    yt = None
    if d >= 1:
        zh_all = np.where(gated[:, None], zhat, base["zhat"])
        _, yt = _integrate(zh_all, y, np.isfinite(y), t_fit, d, end)
    return dict(pred=pred, status=status, phi=phi, theta=theta, order=order, ma_order=ma_order, sigma=sigma, hr=hr,
                gated=gated, base=base, zres=zr, e=e, obs=zobs, fitted=fitted, T=T, m=m, d=d, p=p, q=q, pr=prs, u=us,
                eps=eps, zhat=zhat, ytilde=yt, lobs=np.isfinite(y))


def near_threshold(res, kappa_margin: float = 1e-3):
    """rows whose gate decision may go either way under a first-order perturbation: a long-AR or step-down kappa within
    kappa_margin of the limit, a pivot ratio within 10x of the tolerance, or |R| at the boundary"""
    n = len(res["status"])
    out = np.zeros(n, dtype=bool)
    nreg = res["p"] + res["q"]
    for i, h in enumerate(res["hr"]):
        if h is None:
            continue
        ks = list(h["kappas_long"]) + list(h["kappas_step"])
        out[i] = (any(abs(abs(k) - KAPPA_MAX) < kappa_margin for k in ks) or
                  (np.isfinite(h["pivot"]) and h["pivot"] < 10 * PIVOT_TOL) or h["n_R"] in (nreg, nreg + 1))
    return out


def _impulse_inv_ma(theta, length: int):
    """h_k of 1 / (1 + sum_j theta_j z^j), k < length"""
    h = np.zeros(length)
    h[0] = 1.0
    for k in range(1, length):
        h[k] = -sum(theta[j] * h[k - 1 - j] for j in range(len(theta)) if k - 1 - j >= 0)
    return h


def coef_bound(res, tau_fit):
    """First-order bound on |beta_gpu - beta_oracle|_2 = |(dphi, dtheta)|_2 per gated series from the fitted-value error
    tau_fit, x 2 (DESIGN.md section 6):
      e moves by tau; r_k by 2 tau sqrt(r_0); psi by |dpsi|_1 <= m_i |dr| (1 + |psi|_1) / lambda_min(R_m);
      eps^ by tau (1 + |psi|_1) + |dpsi|_1 max|u^L|; so every entry of [X y] on R moves by at most delta and
      |d[X y]|_F <= delta sqrt(|R| (p + q + 1)) = D;  |dG|, |db| <= 2 |[X y]|_2 D + D^2;
      |dbeta| <= |G^-1|_2 (|db| + |dG| |beta|);
    plus the fp32 rounding of the stored values, 4 eps |beta|_2.  0 for rows that are not gated."""
    n = len(res["status"])
    out = np.zeros(n)
    for i, h in enumerate(res["hr"]):
        if h is None or not res["gated"][i]:
            continue
        r, m_i = h["r"], h["m_i"]
        tau = float(tau_fit[i])
        dr = 2.0 * tau * np.sqrt(r[0])
        psi = h["psi"][:m_i]
        a1 = np.abs(psi).sum()
        Rm = np.array([[r[abs(a - b)] for b in range(m_i)] for a in range(m_i)])
        lam = max(float(np.linalg.eigvalsh(Rm)[0]), 1e-300)
        dpsi = m_i * dr * (1.0 + a1) / lam
        dv = tau * (1.0 + a1) + dpsi * np.abs(h["uL"]).max()
        delta = max(tau, dv)
        Xa = np.column_stack([h["X"], h["target"]])
        D = delta * np.sqrt(Xa.size)
        dG = 2.0 * np.linalg.norm(Xa, 2) * D + D * D
        ginv = 1.0 / max(float(np.linalg.eigvalsh(h["G"])[0]), 1e-300)
        beta = h["beta"]
        out[i] = 2.0 * ginv * (dG + dG * np.linalg.norm(beta)) + 4 * FP32_EPS * np.linalg.norm(beta)
    return out


def pred_bound(res, dbeta, tau_fit, tau_pred, pred_start: int, n_pred: int):
    """First-order bounds of the gated rows (0 elsewhere), x 2 (DESIGN.md section 6) -> (|pred_gpu - pred_oracle| per
    element [n, n_pred], |sigma_gpu - sigma_oracle| [n]).  Along the recursion: bu_s bounds the error of u_s (tau on an
    observed fit row, bpr_s elsewhere) and be_s that of eps~_s (0 on the other rows, where eps~ = 0 exactly).  On an
    observed stretch starting at a the error of eps~ solves (1 + theta(z)) deps = f, so be_s <= sum_k |h_k| bf_{s-k} with h
    the impulse response of the invertible MA part (it decays; the tail beyond the first K terms is added as
    sum_{k>K} |h_k| max bf) and bf_s = tau + sum |phi_j| bu_{s-j} + |dbeta| (|u lags|_1 + |eps~ lags|_1) + rounding
    + sum_{j: s-j < a} |theta_j| be_{s-j} (eps~ from before a gap shorter than q).  bpr_s = sum |phi_j| bu_{s-j}
    + sum |theta_j| be_{s-j} + |dbeta| (|u lags|_1 + |eps~ lags|_1) + rounding.  The prediction adds tau_pred, and for
    d >= 1 it is carried to levels as arima_oracle.arima_bound does.  sigma is an RMS over R, so it moves by at most
    max_R be_s, plus 4 eps sigma."""
    n = len(res["status"])
    d, T, p, q = res["d"], res["T"], res["p"], res["q"]
    end = pred_start + n_pred
    endz = max(end - d, 0)
    bz = np.zeros((n, end))
    sig = np.zeros(n)
    for i in np.flatnonzero(res["gated"]):
        ph, th = res["phi"][i, :p], res["theta"][i, :q]
        aph, ath = np.abs(ph), np.abs(th)
        db = float(dbeta[i])
        tau = float(tau_fit[i])
        obs = res["obs"][i]
        R = res["hr"][i]["R"]
        n_all = max(endz, T)
        _, u_, e_ = recursion(res["e"][i], obs, T, ph, th, n_all)
        u, ep = np.abs(u_), np.abs(e_)
        h = np.abs(_impulse_inv_ma(th, n_all))
        tail = np.cumsum(h[::-1])[::-1]                              # tail[k] = sum_{k' >= k} |h_k'|
        K = int(np.searchsorted(-tail, -1e-13 * tail[0])) if n_all else 0
        K = max(min(K, n_all), 1)
        tail_K = float(tail[K]) if K < n_all else 0.0
        hK = h[:K]
        bu = np.zeros(n_all + AR_MAX)
        be = np.zeros(n_all + MA_MAX)
        bf = np.zeros(n_all)
        start, bfmax = 0, 0.0
        for s in range(n_all):
            ul = u[max(s - p, 0):s][::-1]
            el = ep[max(s - q, 0):s][::-1]
            coef = db * (ul.sum() + el.sum())
            rnd = 16 * FP32_EPS * (aph[:len(ul)] @ ul + ath[:len(el)] @ el)
            ar_b = sum(aph[j] * bu[AR_MAX + s - 1 - j] for j in range(p))
            ma_b = sum(ath[j] * be[MA_MAX + s - 1 - j] for j in range(q))
            bpr = ar_b + ma_b + coef + rnd
            if s < T and obs[s]:
                if s == 0 or not obs[s - 1]:
                    start, bfmax = s, 0.0
                pre = sum(ath[j] * be[MA_MAX + s - 1 - j] for j in range(q) if s - 1 - j < start)
                bf[s] = tau + ar_b + coef + rnd + pre
                bfmax = max(bfmax, bf[s])
                k = min(K, s - start + 1)
                be[MA_MAX + s] = hK[:k] @ bf[s - k + 1:s + 1][::-1] + tail_K * bfmax
                bu[AR_MAX + s] = tau
            else:
                bu[AR_MAX + s] = bpr
            if s < endz:
                bz[i, s + d] = bpr
        sig[i] = 2.0 * be[MA_MAX:MA_MAX + T][R].max(initial=0.0) + 4 * FP32_EPS * res["sigma"][i]
    bz = 2.0 * (bz + np.asarray(tau_pred, dtype=np.float64)[:, None])
    if d == 0:
        return bz[:, pred_start:end], sig
    zh = np.nan_to_num(np.abs(res["zhat"]))
    yt = np.nan_to_num(np.abs(res["ytilde"]))
    lobs = res["lobs"]
    t_fit = T + d
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
        keep = lobs[:, t] if t < t_fit else np.zeros(n, dtype=bool)
        Bt[:, t] = np.where(keep, 0.0, B[:, t])
    return B[:, pred_start:end], sig
