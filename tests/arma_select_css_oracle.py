"""float64 oracle of the (p, d, q) selection's winner refit (DESIGN.md section 2 item 18): arma_select_oracle's
selection, then every winner with q >= 1 refit at its own (p, d, q) and long order m_d by the CSS oracle
(arma_css_oracle) or the joint oracle (arma_joint_oracle), as the reference fits its final model on the tuned order.
A winner with q = 0 and a row with no eligible candidate keep the selection's outputs, with css_start, css NaN and
css_stop, iters 0; beta of a q = 0 winner is W gamma of the plain fit its d builds on, NaN without a winner."""
import numpy as np

from arma_css_oracle import fit_forecast_arma_css_packed
from arma_joint_oracle import fit_forecast_arma_joint_packed, plan_of
from arma_select_oracle import select_arma_packed

REFIT_KEYS = ("pred", "phi", "theta", "order", "ma_order", "sigma", "status", "css_start", "css", "css_stop", "iters")


def select_arma_refit_packed(y, X, t_fit: int, n_hold: int, orders, diffs, mas, pred_start: int, n_pred: int,
                             long_order: int = 0, max_iter: int = 0, joint: bool = False):
    """-> select_arma_packed's dict with the refit's pred, phi, theta, order, ma_order, sigma, status on the q >= 1
    winners, and css_start, css, css_stop, iters [n], refit [n] (the q >= 1 winners), beta [n, P] (joint only) and
    fixed {(p, d, q): the fixed-order oracle's result of that class}"""
    sel = select_arma_packed(y, X, t_fit, n_hold, orders, diffs, mas, pred_start, n_pred, long_order)
    res = {k: np.array(v) for k, v in sel.items() if k not in ("hold", "m")}
    res.update(hold=sel["hold"], m=sel["m"])
    n = len(res["status"])
    res["pred"] = res["pred"].astype(np.float64)
    for k in ("phi", "theta", "sigma"):
        res[k] = res[k].astype(np.float64)
    res["css_start"], res["css"] = np.full(n, np.nan), np.full(n, np.nan)
    res["css_stop"], res["iters"] = np.zeros(n, np.int32), np.zeros(n, np.int32)
    cp, cd, cq = res["choice_p"], res["choice_d"], res["choice_q"]
    refit = cq >= 1
    res["refit"] = refit
    m_of = dict(zip([int(d) for d in diffs], sel["m"]))
    if joint:
        beta = np.full((n, 16), np.nan)
        for d in set(cd[cq == 0].tolist()):
            _, _, W, _, _, gamma0 = plan_of(y, X, t_fit, d)
            s = (cd == d) & (cq == 0)
            beta[s] = (gamma0 @ W.T)[s]
        res["beta"] = beta
    fixed = {}
    fit = fit_forecast_arma_joint_packed if joint else fit_forecast_arma_css_packed
    for p, d, q in sorted(set(zip(cp[refit].tolist(), cd[refit].tolist(), cq[refit].tolist()))):
        r = fit(y, X, t_fit, pred_start, n_pred, p, q, d, long_order=m_of[d], max_iter=max_iter)
        fixed[(p, d, q)] = r
        s = (cp == p) & (cd == d) & (cq == q)
        for k in REFIT_KEYS + (("beta",) if joint else ()):
            res[k][s] = np.asarray(r[k])[s]
    res["fixed"] = fixed
    return res


__all__ = ["REFIT_KEYS", "select_arma_refit_packed"]
