"""CPU: the float64 oracle of tests/arma_joint_oracle.py (DESIGN.md section 2 item 17): the gamma columns of its Jacobian
against central differences, its LM against the CSS oracle's with J empty, a non-increasing objective, optimality against
SciPy over the full vector, the dummy coefficients' RMSE against OLS on simulated regression-with-ARMA-errors rows, the
negative control's failure of the optimality check, and the frame layer's joint_beta= argument."""
import numpy as np
import pytest

import arma_css_oracle as S
import arma_joint_oracle as JO
import arma_oracle as A
from oracle import mmf_oracle as O
from test_arma_css_oracle import OPT_RTOL, _CssOracleEngine, _arma_series

DUMMY_ROWS = (60, 112)
BETA_TRUE = np.array([50.0, 10.0, 15.0, -12.0])


def joint_rows(n, T, phi, theta, seed, n_pred=8, sd=1.0):
    """n series of T weekly rows: intercept + trend + two one-week dummies (DUMMY_ROWS) with BETA_TRUE, ARMA(phi,
    theta) errors -> (y [n, T] float32, X [T + n_pred, 16])"""
    rows = T + n_pred
    X = np.zeros((rows, 16))
    X[:, 0] = 1.0
    X[:, 1] = np.arange(rows) / T
    X[DUMMY_ROWS[0], 2] = 1.0
    X[DUMMY_ROWS[1], 3] = 1.0
    y = np.empty((n, T))
    for i in range(n):
        e, _ = _arma_series(T, phi, theta, seed=seed * 100003 + i, sd=sd)
        y[i] = X[:T, :4] @ BETA_TRUE + e
    return y.astype(np.float32), X


def _case(obs, p, q, seed=5):
    """one series with its plan: z, obs, A_fit, gamma0, cols"""
    T = len(obs)
    X = np.zeros((T, 16))
    X[:, 0] = 1.0
    X[:, 1] = np.arange(T) / T
    X[30, 2] = 1.0
    X[T - 20, 3] = 1.0
    X[:, 4] = np.sin(2 * np.pi * np.arange(T) / 13)
    e, _ = _arma_series(T, [0.5, -0.2][:p], [0.4, 0.2][:q], seed=seed)
    y = (X[:, :5] @ np.array([5.0, 2.0, 3.0, -2.0, 1.0]) + e)[None]
    y = np.where(obs[None], y, np.nan)
    z, Dm, W, kept, Af, g0 = JO.plan_of(y, X, T, 0)
    cols = JO.used_cols(Af, obs, kept)
    return z[0], obs, Af, g0[0], cols


def _gap_cases():
    base = np.ones(120, dtype=bool)
    iso = base.copy(); iso[[20, 47, 90]] = False
    long = base.copy(); long[31:39] = False; long[80:86] = False
    early = base.copy(); early[1] = False; early[60] = False
    return {"gap-free": base, "isolated": iso, "longer than q": long, "before p": early}


@pytest.mark.parametrize("d", [0, 1, 2])
@pytest.mark.parametrize("case", list(_gap_cases()))
def test_gamma_columns_match_central_differences(case, d):
    obs0 = _gap_cases()[case]
    T0 = len(obs0)
    X = np.zeros((T0, 16))
    X[:, 0] = 1.0
    X[:, 1] = np.arange(T0) / T0
    X[30, 2] = 1.0
    X[:, 4] = np.sin(2 * np.pi * np.arange(T0) / 13)
    e, _ = _arma_series(T0, [0.5], [0.4, 0.2], seed=d + 1)
    y = np.where(obs0, X[:, :5] @ np.array([5.0, 2.0, 3.0, 0.0, 1.0]) + np.cumsum(e) * (d > 0) + e, np.nan)[None]
    z, Dm, W, kept, Af, g0 = JO.plan_of(y, X, T0, d)
    T = T0 - d
    obs = np.isfinite(z[0, :T])
    cols = JO.used_cols(Af[:T], obs, kept)
    assert len(cols) >= 2
    p, q = 1, 2
    x = np.r_[0.3, 0.4, 0.15, g0[0, cols] + 0.1]
    _, J, _, _ = JO.joint_eval(z[0], obs, Af[:T], T, p, q, x, g0[0], cols)
    h = 1e-6
    for k in range(p + q + len(cols)):
        xp, xm = x.copy(), x.copy()
        xp[k] += h
        xm[k] -= h
        fd = (JO.joint_eval(z[0], obs, Af[:T], T, p, q, xp, g0[0], cols)[2]
              - JO.joint_eval(z[0], obs, Af[:T], T, p, q, xm, g0[0], cols)[2]) / (2 * h)
        sc = max(1.0, np.abs(fd).max())
        assert np.allclose(J[:, k], fd, rtol=1e-6, atol=1e-7 * sc), (case, d, k, np.abs(J[:, k] - fd).max())
    # the control's gamma columns differ from the exact ones
    _, Jw, _, _ = JO.joint_eval(z[0], obs, Af[:T], T, p, q, x, g0[0], cols, white_beta=True)
    assert np.abs(Jw[:, p + q:] - J[:, p + q:]).max() > 1e-3


@pytest.mark.parametrize("p,q", [(0, 1), (1, 1), (2, 2)])
@pytest.mark.parametrize("case", ["gap-free", "longer than q"])
def test_with_j_empty_lm_joint_is_the_css_oracles_lm(case, p, q):
    obs = _gap_cases()[case]
    z, obs, Af, g0, _ = _case(obs, p, q)
    T = len(obs)
    e = JO.residuals(z, obs, Af, g0)
    h = A.hannan_rissanen(e, obs, T, T - 5, p, q, A.default_long_order(T, p, q))
    x0 = (h["beta"] if h["ok"] else np.r_[np.full(p, 0.2), np.full(q, 0.2)]).astype(np.float32)
    want = S.lm(e, obs, T, p, q, x0)
    got = JO.lm_joint(z, obs, Af, T, p, q, x0, g0, np.zeros(0, dtype=np.int64))
    assert got["stop"] == want["stop"] and got["iters"] == want["iters"] and got["n_acc"] == want["n_acc"]
    assert got["x"].tobytes() == want["x"].tobytes() and got["path"] == want["path"]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_objective_never_increases_and_converged_rows_are_optimal(seed):
    obs = _gap_cases()["isolated" if seed == 2 else "gap-free"]
    z, obs, Af, g0, cols = _case(obs, 1, 1, seed=seed)
    T = len(obs)
    x0 = np.r_[0.1, 0.1, g0[cols]].astype(np.float32)
    r = JO.lm_joint(z, obs, Af, T, 1, 1, x0, g0, cols, max_iter=64)
    assert all(b <= a for a, b in zip(r["path"], r["path"][1:]))
    assert r["S"] < r["S0"] and r["n_acc"] >= 1
    if r["stop"] == 1:
        assert JO.optimality_gap(z, obs, Af, T, 1, 1, r["x"], g0, cols) <= OPT_RTOL


def _gate_set(phi, theta, seed, n=200):
    y, X = joint_rows(n, 157, phi, theta, seed)
    res = JO.fit_forecast_arma_joint_packed(y, X, 157, 157, 8, 1, 1, 0, max_iter=64)
    _, _, g_ols, _ = O.fit_forecast_packed(y, X, 157, 157, 8, return_gamma=True)
    b_ols = O.beta_from_gamma(g_ols, X[:157])
    return y, X, res, b_ols


@pytest.mark.parametrize("phi,theta,seed", [([0.8], [0.4], 11), ([0.9], [], 12)])
def test_dummy_beta_rmse_beats_ols_and_joint_s_is_not_above_css(phi, theta, seed):
    """200 series of 157 weekly rows, ARMA(1, 1) errors (0.8, 0.4) and AR(1) errors (0.9): the dummies' beta RMSE of the
    joint fit <= 0.6 x OLS's (measured: 0.27-0.36); on rows both fits converged, S_joint <= S_css (1 + OPT_RTOL)"""
    y, X, res, b_ols = _gate_set(phi, theta, seed)
    g = res["gated"]
    assert g.sum() >= 150
    ratios = []
    for k in (2, 3):
        rj = np.sqrt(np.mean((res["beta"][g, k] - BETA_TRUE[k]) ** 2))
        ro = np.sqrt(np.mean((b_ols[g, k] - BETA_TRUE[k]) ** 2))
        ratios.append(rj / ro)
    print(f"dummy beta RMSE joint / OLS: {ratios[0]:.3f} {ratios[1]:.3f}")
    assert max(ratios) <= 0.6, ratios
    css = S.fit_forecast_arma_css_packed(y, X, 157, 157, 8, 1, 1, 0, max_iter=64)
    both = g & (res["css_stop"] == 1) & (css["css_stop"] == 1)
    assert both.sum() >= 50
    assert (res["css"][both] <= css["css"][both] * (1 + OPT_RTOL)).all()


def test_white_beta_control_fails_the_optimality_check():
    """the control's converged rows: at least half fail the optimality check; the product's pass it"""
    y, X = joint_rows(30, 157, [0.8], [0.4], 11)
    hr = A.fit_forecast_arma_packed(y, X, 157, 157, 8, 1, 1, 0)
    good = JO.fit_forecast_arma_joint_packed(y, X, 157, 157, 8, 1, 1, 0, max_iter=64, hr=hr)
    bad = JO.fit_forecast_arma_joint_packed(y, X, 157, 157, 8, 1, 1, 0, max_iter=64, white_beta=True, hr=hr)
    z, A_fit = good["z"], good["A"][:157]
    fails, rows = 0, 0
    for i in np.flatnonzero(hr["gated"]):
        obs = np.isfinite(z[i])
        cols = good["cols"][i]
        if good["css_stop"][i] == 1:
            xg = np.r_[good["phi"][i, :1], good["theta"][i, :1], good["gamma"][i, cols]]
            assert JO.optimality_gap(z[i], obs, A_fit, 157, 1, 1, xg, good["gamma0"][i], cols) <= OPT_RTOL, i
        if bad["css_stop"][i] == 1:
            rows += 1
            xb = np.r_[bad["phi"][i, :1], bad["theta"][i, :1], bad["gamma"][i, cols]]
            fails += JO.optimality_gap(z[i], obs, A_fit, 157, 1, 1, xb, bad["gamma0"][i], cols) > OPT_RTOL
    assert rows >= 10 and fails >= 0.5 * rows, (fails, rows)


class _JointOracleEngine(_CssOracleEngine):
    """ForecastEngine stand-in answering fit_forecast_arma(..., joint_beta=True) with the joint oracle"""

    def fit_forecast_arma(self, y, p, q, d, ps, npred, estimator="hr", joint_beta=False):
        if not joint_beta:
            return super().fit_forecast_arma(y, p, q, d, ps, npred, estimator=estimator)
        assert estimator == "css"
        self.arma_calls.append((p, q, d, "joint"))
        res = JO.fit_forecast_arma_joint_packed(np.asarray(y), self.X, self.t_fit, ps, npred, p, q, d)
        return {"pred": res["pred"].astype(np.float32)}


@pytest.mark.parametrize("diff", [None, 1])
def test_forecast_groups_with_the_joint_oracle_engine(diff):
    import mmf
    from test_arima_oracle import _frame
    pdf = _frame()
    eng = _JointOracleEngine()
    out = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=eng, ar=1, diff=diff, ma=1,
                              estimator="css", joint_beta=True)
    assert eng.arma_calls == [(1, 1, diff or 0, "joint")] * 2
    for (prod, sku), g in out.groupby(["Product", "SKU"], sort=True):
        src = pdf[(pdf["Product"] == prod) & (pdf["SKU"] == sku)].sort_values("Date")
        y = src["Demand"].to_numpy(dtype=np.float32)[None, :]
        t_len, t_fit = y.shape[1], y.shape[1] - 14
        X = O.design_matrix(O.calendar_grid(np.datetime64(src["Date"].min(), "D"), t_len, "D"), t_fit)
        want = JO.fit_forecast_arma_joint_packed(y, X, t_fit, 0, t_len, 1, 1, diff or 0)
        got = g["Demand_Fitted"].to_numpy(dtype=np.float32)
        assert np.array_equal(got, want["pred"][0].astype(np.float32), equal_nan=True), (prod, sku)
    tbl = mmf.forecast_table(pdf, freq="D", horizon=14, mode="holdout", engine=_JointOracleEngine(), ar=1, diff=diff,
                             ma=1, estimator="css", joint_beta=True)
    assert np.array_equal(tbl.column("Demand_Fitted").to_numpy(zero_copy_only=False).astype(np.float32),
                          out["Demand_Fitted"].to_numpy(dtype=np.float32), equal_nan=True)


def test_joint_beta_argument_checks():
    import mmf
    pdf = mmf.synth.reference_weekly_demand(2)
    for fg in (mmf.frames.forecast_groups, mmf.frames.forecast_table):
        for kw, msg in ((dict(ar=1, ma=1, joint_beta=True), "joint_beta=True needs estimator='css'"),
                        (dict(ar=1, ma=1, estimator="hr", joint_beta=True), "joint_beta=True needs estimator='css'"),
                        (dict(ar=1, joint_beta=True, estimator="css"), "estimator= needs one MA order"),
                        (dict(ar=1, ma=1, estimator="mle", joint_beta=True), "estimator must be 'hr' or 'css'")):
            with pytest.raises(ValueError, match=msg):
                fg(pdf, freq="W-MON", horizon=40, mode="holdout", engine=object(), **kw)
