"""CPU: the float64 ARIMA(p, d, q) oracle of tests/arma_oracle.py (DESIGN.md section 2 item 13) against independent
restatements (scipy's Toeplitz solve and lfilter, numpy's lstsq and roots), its gate rules on constructed rows, known
answers on simulated MA(1) and ARMA(1, 1) errors, and the frame layer's ma= argument."""
import numpy as np
import pytest
from scipy.linalg import solve_toeplitz
from scipy.signal import lfilter

import arma_oracle as A
from ar_oracle import KAPPA_MAX, autocov
from oracle import mmf_oracle as O
from test_arima_oracle import _OracleEngine as _ArimaOracleEngine


def _daily(n, t, p_true=0.0, theta=0.6, seed=0, gaps=0.0):
    rng = np.random.default_rng(seed)
    X = O.design_matrix(O.calendar_grid("2019-01-01", t + 28, "D"), t)
    eps = rng.normal(0, 5, (n, t + 1))
    u = np.zeros((n, t))
    for k in range(t):
        u[:, k] = eps[:, k + 1] + theta * eps[:, k] + (p_true * u[:, k - 1] if k else 0.0)
    y = 400.0 + rng.normal(0, 20, (n, X.shape[1])) @ X[:t].T + u
    if gaps:
        for i in range(n):
            y[i, rng.choice(np.arange(2, t - 1), size=int(gaps * t), replace=False)] = np.nan
    return y, X


def test_step_one_and_step_two_against_independent_solves():
    y, X = _daily(4, 600, p_true=0.5, theta=0.4, seed=1)
    res = A.fit_forecast_arma_packed(y, X, 600, 600, 28, 1, 1, 0, 12)
    for i in range(4):
        h = res["hr"][i]
        r = h["r"]
        psi = solve_toeplitz(r[:12], r[1:13])
        assert h["m_i"] == 12 and np.allclose(h["psi"], psi, rtol=1e-9, atol=1e-12)
        beta = np.linalg.lstsq(h["X"], h["target"], rcond=None)[0]
        assert np.allclose(h["beta"], beta, rtol=1e-9)


def test_recursion_against_lfilter_and_a_loop_with_gaps():
    rng = np.random.default_rng(2)
    e = rng.normal(0, 1, 300)
    obs = np.ones(300, dtype=bool)
    phi, th = np.array([0.5, -0.2]), np.array([0.4, 0.1])
    pr, u, ep = A.recursion(e, obs, 300, phi, th, 300)
    assert np.allclose(ep[:300], lfilter(np.r_[1.0, -phi], np.r_[1.0, th], e), rtol=1e-12, atol=1e-12)
    obs[[10, 11, 50, 299]] = False
    pr, u, ep = A.recursion(e, obs, 300, phi, th, 320)
    U, E, P = [0.0] * 2, [0.0] * 2, []
    for s in range(320):
        a = phi[0] * U[-1] + phi[1] * U[-2] + th[0] * E[-1] + th[1] * E[-2]
        P.append(a)
        o = s < 300 and obs[s]
        U.append(e[s] if o else a)
        E.append(e[s] - a if o else 0.0)
    assert np.allclose(pr, P, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("seed", range(20))
def test_step_down_against_roots(seed):
    rng = np.random.default_rng(seed)
    a = rng.uniform(-1.2, 1.2, rng.integers(1, 5))
    ks = A.step_down(a)
    stable = np.all(np.abs(np.roots(np.r_[-a[::-1], 1.0])) > 1.0)
    assert (all(abs(k) < KAPPA_MAX for k in ks) and len(ks) == len(a)) == stable or \
        np.min(np.abs(np.abs(np.roots(np.r_[-a[::-1], 1.0])) - 1.0)) < 1e-3


def test_gate_rules_on_constructed_rows(monkeypatch):
    """every rule of the gate reached through hannan_rissanen, with the field that decides it"""
    t = 400
    obs = np.ones(t, dtype=bool)
    rng = np.random.default_rng(3)
    zero = A.hannan_rissanen(np.zeros(t), obs, t, t - 5, 1, 1, 10)          # r_0 = 0: m_i = 0
    assert not zero["ok"] and zero["m_i"] == 0 and zero["G"] is None
    e = rng.normal(0, 1, t)
    few = np.zeros(t, dtype=bool)
    few[::3] = True                                                          # no two consecutive observations
    few[-2:] = True                                                          # one row of R for p = q = 1
    h = A.hannan_rissanen(np.where(few, e, 0.0), few, t, t - 5, 1, 1, 10)
    assert h["m_i"] >= 1 and h["n_R"] <= 2 and not h["ok"] and h["kappas_step"] == []
    # psi = 0 makes eps^ = e, so the regressors e_{t-1} and eps^_{t-1} are the same column: the pivot rule fails
    monkeypatch.setattr(A, "levinson_long", lambda r, m: (np.r_[1e-300, np.zeros(m - 1)], 1, [1e-300]))
    h = A.hannan_rissanen(e, obs, t, t - 5, 1, 1, 10)
    assert h["n_R"] > 2 and h["pivot"] <= A.PIVOT_TOL and not h["ok"] and h["kappas_step"] == []
    monkeypatch.undo()
    # an explosive AR(1), x_t = 1.02 x_{t-1} + noise: the estimate phi ~ 1.02 passes the pivots and fails the step-down
    rng = np.random.default_rng(3)
    x = np.zeros(t)
    for k in range(1, t):
        x[k] = 1.02 * x[k - 1] + rng.normal()
    h = A.hannan_rissanen(x, obs, t, t - 5, 1, 1, 4)
    assert h["m_i"] >= 1 and h["n_R"] > 2 and h["pivot"] > A.PIVOT_TOL
    assert not h["ok"] and any(abs(k) >= KAPPA_MAX for k in h["kappas_step"]), h["kappas_step"]
    assert A.step_down([-1.5]) == [-1.5]                                     # theta = 1.5: stops at the first stage


def test_known_answers_and_a_better_one_step_fit_than_ar1():
    y, X = _daily(40, 1095, theta=0.6, seed=4)
    res = A.fit_forecast_arma_packed(y, X, 1095, 0, 1095, 0, 1, 0)
    th = res["theta"][res["gated"], 0]
    assert res["gated"].all() and abs(th.mean() - 0.6) < 0.02 and th.std() < 0.06
    ar1 = A.fit_forecast_ar_packed(y, X, 1095, 0, 1095, 1)
    mse_ma = np.mean((res["pred"][:, 1:] - y[:, 1:]) ** 2)
    mse_ar = np.mean((ar1["pred"][:, 1:] - y[:, 1:]) ** 2)
    assert mse_ma < mse_ar
    y, X = _daily(40, 1095, p_true=0.5, theta=0.4, seed=5)
    res = A.fit_forecast_arma_packed(y, X, 1095, 1095, 28, 1, 1, 0)
    assert abs(res["phi"][:, 0].mean() - 0.5) < 0.03 and abs(res["theta"][:, 0].mean() - 0.4) < 0.03


def test_fallback_rows_are_the_arima_oracle_rows():
    y, X = _daily(6, 300, seed=6)
    y[0] = 5.0                                                               # constant: r_0 = 0, falls back
    res = A.fit_forecast_arma_packed(y, X, 300, 300, 28, 1, 1, 1)
    assert not res["gated"][0] and res["ma_order"][0] == 0 and not res["theta"][0].any()
    assert np.array_equal(res["pred"][0], res["base"]["pred"][0], equal_nan=True)


class _OracleEngine(_ArimaOracleEngine):
    """ForecastEngine stand-in of tests/test_arima_oracle.py, answering fit_forecast_arma with the oracle"""

    def __init__(self):
        super().__init__()
        self.arma_calls = []

    def fit_forecast_arma(self, y, p, q, d, ps, npred):
        assert d == 0 or (self.max_diff is not None and d <= self.max_diff)
        self.arma_calls.append((p, q, d))
        return {"pred": A.fit_forecast_arma_packed(np.asarray(y), self.X, self.t_fit, ps, npred, p, q, d)["pred"]
                .astype(np.float32)}


@pytest.mark.parametrize("diff", [None, 1, 2])
def test_forecast_groups_with_the_oracle_engine(diff):
    """one call per calendar bucket with (p, d, q); each group's rows are the oracle's on that group's calendar"""
    import mmf
    from test_arima_oracle import _frame
    pdf = _frame()
    eng = _OracleEngine()
    out = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=eng, ar=1, diff=diff, ma=1)
    assert eng.arma_calls == [(1, 1, diff or 0)] * 2 and eng.arima_calls == 0 and eng.plain_calls == 0
    plain = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine())
    assert list(out.columns) == list(plain.columns) and (out.dtypes == plain.dtypes).all()
    assert out[["Product", "SKU", "Date"]].equals(plain[["Product", "SKU", "Date"]])
    for (prod, sku), g in out.groupby(["Product", "SKU"], sort=True):
        src = pdf[(pdf["Product"] == prod) & (pdf["SKU"] == sku)].sort_values("Date")
        y = src["Demand"].to_numpy(dtype=np.float32)[None, :]
        t_len, t_fit = y.shape[1], y.shape[1] - 14
        X = O.design_matrix(O.calendar_grid(np.datetime64(src["Date"].min(), "D"), t_len, "D"), t_fit)
        want = A.fit_forecast_arma_packed(y, X, t_fit, 0, t_len, 1, 1, diff or 0)["pred"][0].astype(np.float32)
        assert np.array_equal(g["Demand_Fitted"].to_numpy(dtype=np.float32), want, equal_nan=True), (prod, sku)
    tbl = mmf.forecast_table(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine(), ar=1, diff=diff, ma=1)
    assert np.array_equal(tbl.column("Demand_Fitted").to_numpy(zero_copy_only=False).astype(np.float32),
                          out["Demand_Fitted"].to_numpy(dtype=np.float32), equal_nan=True)


def test_forecast_groups_ma_argument_checks():
    import mmf
    pdf = mmf.synth.reference_weekly_demand(2)
    fg = mmf.frames.forecast_groups
    for kw in (dict(ar=1, ma=(1, 2)), dict(ar=(0, 1), ma=1), dict(ar=1, ma=5), dict(ar=1, ma=0),
               dict(ar=1, ma=1, select=(1, 3)), dict(ar=1, ma=1, interval=0.9), dict(ar=1, diff=(0, 1), ma=1),
               dict(ar=None, ma=1)):
        with pytest.raises(ValueError):
            fg(pdf, freq="W-MON", horizon=40, mode="holdout", engine=object(), **kw)
