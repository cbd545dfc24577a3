"""float64 oracle of regression with AR(p) errors (DESIGN.md section 2 item 9), on top of ``oracle.mmf_oracle``'s fit.

For series i: the plain fit's gamma, status and fitted values (``O.fit_forecast_packed`` over every design row), the
residuals e_t = y_t - yhat_t of the observed fit rows (0 elsewhere), r_k = (1/n_obs) sum_t e_t e_{t-k} (k = 0..p), the
order rule and Levinson-Durbin of item 4, the filled residuals u of item 5 and the predictions of item 6.  The used
columns k of the dof rule are those of section 2 item 7: the columns the in-order pivoted solve of ``O.solve_series``
retains for the series' mask (``used_columns`` restates its pivot rule; all kept columns for a gap-free series).

``ar_bound`` is the first-order forward-error bound of the predictions and ``coef_bounds`` that of phi and sigma, which
the GPU tests hold the library to (DESIGN.md section 6).
"""
from __future__ import annotations

import numpy as np

from oracle import mmf_oracle as O

AR_MAX = 8
KAPPA_MAX = 0.999
FP32_EPS = 2.0 ** -24


def levinson(r, p: int, kappa_max: float = KAPPA_MAX):
    """Levinson-Durbin on r_0..r_p (float64) -> (phi [AR_MAX], order, innovation variance, kappas of every stage it
    reached, including the one it stopped at).  Stops before the first j with r_0 <= 0 or |kappa_j| >= kappa_max."""
    phi = np.zeros(AR_MAX)
    kappas = []
    var = float(r[0])
    if not r[0] > 0.0:
        return phi, 0, var, kappas
    order = 0
    for j in range(1, p + 1):
        kap = (r[j] - phi[:j - 1] @ r[j - 1:0:-1]) / var
        kappas.append(float(kap))
        if abs(kap) >= kappa_max:
            break
        prev = phi[:j - 1].copy()
        phi[:j - 1] = prev - kap * prev[::-1]
        phi[j - 1] = kap
        var *= 1.0 - kap * kap
        order = j
    return phi, order, var, kappas


def used_columns(obs_row, A_fit, kept):
    """number of whitened columns the pivoted solve of O.solve_series retains for one series' observed fit rows"""
    if obs_row.all():
        return int(kept.sum())
    Ao = A_fit[obs_row]
    G = Ao.T @ Ao
    p = G.shape[0]
    L = np.zeros((p, p))
    k = 0
    for j in range(p):
        if G[j, j] <= 0.0:
            continue
        d = G[j, j] - L[j, :j] @ L[j, :j]
        if d <= O.PIVOT_TOL * G[j, j]:
            continue
        k += 1
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (G[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return k


def autocov(e, obs, t_fit: int, p: int):
    """r_0..r_p of one series: e residuals (0 where missing), the divisor n_obs for every lag"""
    n_obs = int(obs[:t_fit].sum())
    r = np.array([e[k:t_fit] @ e[:t_fit - k] for k in range(p + 1)]) / max(n_obs, 1)
    return r


def fit_forecast_ar_packed(y, X, t_fit: int, pred_start: int, n_pred: int, p: int):
    """-> dict(pred [n, n_pred], status, phi [n, AR_MAX], order, sigma, fitted [n, n_rows], e [n, t_fit],
    u [n, end] filled residuals, r [n, p+1], dof, kappas (list per series), ar [n, n_pred] the AR part of pred)."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)[:, :t_fit]
    n_rows = X.shape[0]
    end = pred_start + n_pred
    fitted, status, gamma, _ = O.fit_forecast_packed(y, X, t_fit, 0, n_rows, return_gamma=True)
    W, kept = O.whiten(X[:t_fit])
    A_fit = X[:t_fit] @ W
    n = y.shape[0]
    obs = np.isfinite(y)
    n_obs = obs.sum(axis=1)
    e = np.where(obs, y - fitted[:, :t_fit], 0.0)
    k_used = np.array([used_columns(obs[i], A_fit, kept) if status[i] != 1 else 0 for i in range(n)])
    dof = np.where(status != 1, n_obs - k_used, 0)
    phi = np.zeros((n, AR_MAX))
    order = np.zeros(n, dtype=np.int32)
    sigma = np.full(n, np.nan)
    r_all = np.zeros((n, p + 1))
    kappas = [[] for _ in range(n)]
    for i in range(n):
        if status[i] == 1:
            continue
        r = autocov(e[i], obs[i], t_fit, p)
        r_all[i] = r
        if dof[i] <= p:
            sigma[i] = np.sqrt(r[0])
            continue
        phi[i], order[i], var, kappas[i] = levinson(r, p)
        sigma[i] = np.sqrt(var)
    u = np.zeros((n, end + AR_MAX))                 # u[:, AR_MAX + s] = u_s; the first AR_MAX columns are s < 0
    ar = np.zeros((n, end))
    for s in range(end):
        a = (phi * u[:, s + AR_MAX - 1::-1][:, :AR_MAX] if s + AR_MAX - 1 >= 0 else 0).sum(axis=1)
        ar[:, s] = a
        keep = obs[:, s] if s < t_fit else np.zeros(n, dtype=bool)
        u[:, AR_MAX + s] = np.where(keep, e[:, s] if s < t_fit else 0.0, a)
    pred = fitted[:, pred_start:end] + ar[:, pred_start:end]
    pred[status == 1] = np.nan
    return dict(pred=pred, status=status, phi=phi, order=order, sigma=sigma, fitted=fitted, e=e,
                u=u[:, AR_MAX:], r=r_all, dof=dof, kappas=kappas, ar=ar[:, pred_start:end], obs=obs)


def kappa_margin(res):
    """per series: the smallest distance of a reached |kappa_j| to the limit (inf where none was computed)"""
    return np.array([min((abs(abs(k) - KAPPA_MAX) for k in ks), default=np.inf) for ks in res["kappas"]])


def _coef_terms(res, tau_fit):
    """first-order |dphi|_1 and |dsigma| per series, before the factor 2 and the fp32 rounding of coef_bounds"""
    n = len(res["order"])
    phi, order, r = res["phi"], res["order"], res["r"]
    dphi = np.zeros(n)
    dsig = np.zeros(n)
    for i in range(n):
        if res["status"][i] == 1 or not r[i, 0] > 0:
            continue
        p_i = int(order[i])
        dr = 2.0 * tau_fit[i] * np.sqrt(r[i, 0])
        a1 = np.abs(phi[i]).sum()
        if p_i > 0:
            R = np.array([[r[i, abs(a - b)] for b in range(p_i)] for a in range(p_i)])
            lam = max(float(np.linalg.eigvalsh(R)[0]), 1e-300)
            dphi[i] = p_i * dr * (1.0 + a1) / lam
        dvar = dr * (1.0 + a1) + dphi[i] * np.abs(r[i, :p_i + 1]).max()
        sig = res["sigma"][i]
        dsig[i] = min(dvar / sig, np.sqrt(dvar)) if sig > 0 else np.sqrt(dvar)
    return dphi, dsig


def coef_bounds(res, tau_fit):
    """First-order bounds on |phi_gpu - phi_oracle|_1 and |sigma_gpu - sigma_oracle| per series from the fitted-value
    error tau_fit (DESIGN.md section 6), x 2:
      |dr_k|  <= 2 tau_fit sqrt(r_0)                         (Cauchy-Schwarz over the n_obs pairs)
      |dphi|_1 <= p_i |dr|_inf (1 + |phi|_1) / lambda_min(R)  (perturbed Yule-Walker system R phi = r, R p_i x p_i)
      sigma^2 = r_0 - phi . r_{1..p_i}:  |dsigma^2| <= |dr|_inf (1 + |phi|_1) + |dphi|_1 max_k |r_k|,
      |dsigma| <= min(|dsigma^2| / sigma, sqrt |dsigma^2|)     (|sqrt a - sqrt b| <= |a - b| / sqrt a, sqrt |a - b|);
    plus the fp32 rounding of the stored values (4 eps |phi|_1, 4 eps sigma).  Rows of order 0: phi is compared exactly
    (dphi = 0)."""
    dphi, dsig = _coef_terms(res, tau_fit)
    return (2.0 * dphi + 4 * FP32_EPS * np.abs(res["phi"]).sum(axis=1),
            2.0 * dsig + 4 * FP32_EPS * np.nan_to_num(res["sigma"]))


DEGENERATE_TAU = 4.0


def degenerate_rows(res, tau_fit):
    """Rows where the first-order bounds (coef_bounds, ar_bound) do not apply: the oracle's RMS residual sqrt(r_0) is at
    most DEGENERATE_TAU x tau_fit, so |dr_k| <= 2 tau_fit sqrt(r_0) is not small next to r_0 (it is >= r_0 / 2).  This is
    a series the regression fits to rounding level -- all zero, constant, an exact line or level plus weekly pattern in
    the design's span: the GPU's residuals are fp32 noise of size ~tau_fit, the oracle's float64 noise, and the two run
    Levinson-Durbin on unrelated noise.  Status-1 rows are never degenerate."""
    return (np.asarray(res["status"]) != 1) & (np.sqrt(np.maximum(res["r"][:, 0], 0.0)) <= DEGENERATE_TAU * tau_fit)


def impulse(phi, length: int):
    """c [n, length, AR_MAX]: inside a dynamic stretch of the recursion u_s = sum_j phi_j u_{s-j} entered at position a,
    u_{a+h} = sum_k c[:, h, k-1] u_{a-k} (k = 1..AR_MAX).  Signed, so for a stable phi it decays with h."""
    phi = np.asarray(phi, dtype=np.float64)
    n = phi.shape[0]
    c = np.zeros((n, length, AR_MAX))
    for h in range(length):
        acc = np.zeros((n, AR_MAX))
        if h < AR_MAX:
            acc[:, :AR_MAX - h] = phi[:, h:]                        # phi_{h+k}: a state value reached directly
        for j in range(1, min(h, AR_MAX) + 1):
            acc += phi[:, j - 1:j] * c[:, h - j]
        c[:, h] = acc
    return c


def _ar_magnitude(phi, obs, e_max, t_fit: int, pred_start: int, n_pred: int):
    """bound on |AR part| of every requested row when every observed fit residual is at most e_max.  B_s bounds |u_s|:
    e_max on an observed fit row; in a stretch of unobserved rows entered at a, sum_k |c_{s-a,k}| B_{a-k} with c the
    signed impulse coefficients of phi (u before row 0 is 0).  The AR part is u_s itself on an unobserved row and
    sum_j phi_j u_{s-j} (<= sum_j |phi_j| B_{s-j}, one step) on an observed one."""
    phi = np.asarray(phi, dtype=np.float64)
    n = phi.shape[0]
    end = pred_start + n_pred
    aphi = np.abs(phi)
    c = np.abs(impulse(phi, max(end, 1)))
    B = np.zeros((n, end + AR_MAX))                                  # B[:, AR_MAX + s]; columns < AR_MAX are s < 0
    rows = np.arange(n)
    lag = np.arange(1, AR_MAX + 1)
    entry = np.zeros(n, dtype=np.int64)
    out = np.zeros((n, n_pred))
    for s in range(end):
        if 0 < s <= t_fit:
            entry = np.where(obs[:, s - 1], s, entry)
        o = obs[:, s] if s < t_fit else np.zeros(n, dtype=bool)
        state = B[rows[:, None], AR_MAX + entry[:, None] - lag[None, :]]
        dyn = (c[rows, s - entry] * state).sum(axis=1)
        one = (aphi * B[:, AR_MAX + s - lag]).sum(axis=1)
        B[:, AR_MAX + s] = np.where(o, e_max, dyn)
        if s >= pred_start:
            out[:, s - pred_start] = np.where(o, one, dyn)
    return out


def degenerate_bound(res, phi_gpu, tau_fit, tau_pred, t_fit: int, pred_start: int, n_pred: int):
    """Bound on |pred_gpu - pred_oracle| per element that holds on every row, degenerate ones included (DESIGN.md
    section 6): the fitted values differ by at most tau_pred; each side's AR part is at most what its own phi -- through
    the signed impulse coefficients, which decay for a stable phi -- makes of residuals of at most max|e_oracle|
    (+ tau_fit on the GPU's side, whose residuals carry its fitted-value error).  No first-order term: it does not need
    r_0 to be large next to tau.  Returned x 2, plus fp32 rounding."""
    obs = res["obs"]
    e_max = np.abs(res["e"]).max(axis=1)
    a_gpu = _ar_magnitude(phi_gpu, obs, e_max + tau_fit, t_fit, pred_start, n_pred)
    a_orc = _ar_magnitude(res["phi"], obs, e_max, t_fit, pred_start, n_pred)
    rnd = 16 * FP32_EPS * np.nan_to_num(np.abs(res["pred"]))
    return 2.0 * (tau_pred[:, None] + a_gpu + a_orc + rnd)


def ar_bound(res, tau_fit, tau_pred, t_fit: int, pred_start: int, n_pred: int):
    """First-order bound on |pred_gpu - pred_oracle| per element (DESIGN.md section 6).
    tau_fit[i]: bound on the error of a plain fitted value on the fit rows (the parity tolerance x mask factor);
    tau_pred[i]: the same on the requested rows (x their leverage).  Errors of the fitted values reach
      the residuals:       |de_t| <= tau_fit
      the autocovariances: |dr_k| <= 2 tau_fit sqrt(r_0)  (Cauchy-Schwarz over the n_obs pairs)
      the coefficients:    |dphi|_1 <= p |dr|_inf (1 + |phi|_1) / lambda_min(R)  (perturbed Yule-Walker system R phi = r)
    and travel through the recursion: b_s = tau_fit for an observed fit row, else |dphi|_1 max_j |u_{s-j}| + sum_j |phi_j|
    b_{s-j}; the prediction adds its own fitted-value error, the AR sum's |dphi| and fp32 rounding terms.  Returned x 2."""
    n = res["pred"].shape[0]
    end = pred_start + n_pred
    phi, order, u, r, obs = res["phi"], res["order"], res["u"], res["r"], res["obs"]
    dphi = _coef_terms(res, tau_fit)[0]
    aphi = np.abs(phi)
    b = np.zeros((n, end + AR_MAX))
    out = np.zeros((n, n_pred))
    ua = np.abs(np.pad(u, ((0, 0), (AR_MAX, 0))))
    for s in range(end):
        lag_u = ua[:, s + AR_MAX - 1::-1][:, :AR_MAX] if s + AR_MAX - 1 >= 0 else np.zeros((n, AR_MAX))
        lag_b = b[:, s + AR_MAX - 1::-1][:, :AR_MAX]
        prop = dphi * lag_u.max(axis=1) + (aphi * lag_b).sum(axis=1)
        rnd = 16 * FP32_EPS * (aphi * lag_u).sum(axis=1)
        fit_row = obs[:, s] if s < t_fit else np.zeros(n, dtype=bool)
        b[:, AR_MAX + s] = np.where(fit_row, tau_fit, prop + rnd)
        if s >= pred_start:
            out[:, s - pred_start] = tau_pred + prop + rnd
    return 2.0 * out
