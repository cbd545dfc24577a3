"""CPU: the float64 AR(p)-errors oracle (tests/ar_oracle.py) against independent restatements of DESIGN.md section 2
item 9, and forecast_groups(ar=...) with the oracle standing in for the engine."""
import numpy as np
import pandas as pd
import pytest
from scipy.linalg import solve_toeplitz

import mmf
from ar_oracle import AR_MAX, KAPPA_MAX, fit_forecast_ar_packed, levinson
from oracle import mmf_oracle as O


def _daily(n, t, seed, h=28):
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=seed)
    X = O.design_matrix(O.calendar_grid(start, t + h, "D"), t)
    return y.astype(np.float64), X


@pytest.mark.parametrize("p", [1, 2, 3, 5, 8])
def test_levinson_matches_a_toeplitz_solve(p):
    rng = np.random.default_rng(p)
    x = rng.normal(size=500)
    r = np.array([x[k:] @ x[:len(x) - k] for k in range(p + 1)]) / len(x)
    phi, order, var, _ = levinson(r, p)
    assert order == p
    want = solve_toeplitz(r[:p], r[1:p + 1])
    assert np.allclose(phi[:p], want, rtol=1e-12, atol=1e-14) and not phi[p:].any()
    assert np.isclose(var, r[0] - want @ r[1:p + 1], rtol=1e-12)


def test_estimator_against_an_independent_restatement():
    y, X = _daily(12, 300, seed=5)
    t = 300
    res = fit_forecast_ar_packed(y, X, t, t, 28, 3)
    for i in range(len(y)):
        beta = np.linalg.lstsq(X[:t], y[i], rcond=None)[0]
        e = y[i] - X[:t] @ beta
        r = np.correlate(e, e, "full")[t - 1:t + 3] / t
        phi = solve_toeplitz(r[:3], r[1:4])
        assert np.allclose(res["phi"][i, :3], phi, rtol=1e-9, atol=1e-12), i
        assert res["order"][i] == 3


def test_predictions_against_a_plain_loop():
    y, X = _daily(6, 200, seed=7, h=20)
    t, p = 200, 3
    y[0, t - 1] = np.nan                                   # gap at the origin
    y[1, t - 10:t - 4] = np.nan                            # before it
    y[2, :p] = np.nan                                      # in the first p rows
    y[3, 50:80] = np.nan
    for ps, npred in ((t, 20), (0, t + 20), (70, 90)):
        res = fit_forecast_ar_packed(y, X, t, ps, npred, p)
        for i in range(len(y)):
            phi, fit = res["phi"][i], res["fitted"][i]
            u = {}
            for s in range(ps + npred):
                ar = sum(phi[j - 1] * u.get(s - j, 0.0) for j in range(1, AR_MAX + 1))
                u[s] = y[i, s] - fit[s] if s < t and np.isfinite(y[i, s]) else ar
                if s >= ps:
                    assert np.isclose(res["pred"][i, s - ps], fit[s] + ar, rtol=1e-12, atol=1e-9), (i, s)


def test_order_rule():
    t = 120
    X = O.design_matrix(O.calendar_grid("2020-01-01", t + 10, "D"), t)
    perfect = np.zeros((1, t))                                         # residuals exactly 0: r_0 = 0
    res = fit_forecast_ar_packed(perfect, X, t, t, 10, 2)
    assert res["r"][0, 0] == 0.0 and res["order"][0] == 0 and not res["phi"][0].any()
    hit = 0
    for m in range(3, 40):                                             # the first m values observed: dof = m - used
        few = np.full((1, t), np.nan)
        few[0, :m] = np.arange(m) ** 1.5
        res = fit_forecast_ar_packed(few, X, t, t, 10, 2)
        if res["dof"][0] <= 2:
            hit += res["dof"][0] >= 1
            assert res["order"][0] == 0 and not res["phi"][0].any(), m
    assert hit >= 1
    phi, order, _, ks = levinson(np.array([1.0, 0.9995, 0.999]), 2)      # |kappa_1| past the limit
    assert order == 0 and abs(ks[0]) >= KAPPA_MAX and not phi.any()
    phi, order, _, ks = levinson(np.array([1.0, 0.5, 0.9995]), 2)       # the second stage is cut
    assert order == 1 and abs(ks[1]) >= KAPPA_MAX and phi[0] == 0.5


@pytest.mark.parametrize("phi_true", [(0.9,), (0.5, 0.3)])
def test_recovers_known_coefficients(phi_true):
    rng = np.random.default_rng(11)
    n, t = 200, 1000
    X = O.design_matrix(O.calendar_grid("2018-01-01", t + 5, "D"), t)
    e = rng.normal(0, 1, (n, t))
    u = np.zeros((n, t))
    for s in range(t):
        u[:, s] = e[:, s] + sum(f * u[:, s - j - 1] for j, f in enumerate(phi_true) if s - j - 1 >= 0)
    res = fit_forecast_ar_packed(50 + u, X, t, t, 5, len(phi_true))
    # sampling error of the mean over n series, plus the known O(1/t) downward bias of Yule-Walker on the residuals of a
    # k = 16 column regression (the design absorbs part of the slow AR variation): (k + 2) (1 + |phi|_1) / t
    se = np.sqrt((1 - np.asarray(phi_true) ** 2) / t) / np.sqrt(n)
    bias = 18 * (1 + np.abs(phi_true).sum()) / t
    assert np.all(np.abs(res["phi"][:, :len(phi_true)].mean(0) - phi_true) < 5 * se + bias)
    assert np.all(np.abs(res["phi"][:, :len(phi_true)] - phi_true) < 5 * se * np.sqrt(n) + bias)
    assert abs(res["sigma"].mean() - 1.0) < 0.02


def test_holdout_mse_beats_the_plain_model_on_daily_demand():
    y, X = _daily(40, 760, seed=3, h=0)
    t = 760 - 7
    res = fit_forecast_ar_packed(y, X, t, t, 7, 1)
    plain, _ = O.fit_forecast_packed(y, X, t, t, 7)
    act = y[:, t:t + 7]
    assert np.mean((res["pred"] - act) ** 2) < np.mean((plain - act) ** 2)


class _OracleEngine:
    """stands in for ForecastEngine: plans a calendar, answers fit_forecast / fit_forecast_ar with the oracles"""

    def __init__(self):
        self.ar_calls = 0
        self.plain_calls = 0

    def plan_calendar(self, start, t_len, freq="D", horizon=28, mode="future", design="trend_season_exog"):
        if mode == "holdout":
            self.t_fit, days = t_len - horizon, O.calendar_grid(start, t_len, freq)
            ps, npred = 0, t_len
        else:
            self.t_fit, days = t_len, O.calendar_grid(start, t_len + horizon, freq)
            ps, npred = t_len, horizon
        self.X = O.design_matrix(days, self.t_fit, design)
        return np.array(days, dtype="datetime64[D]")[ps:ps + npred], ps, npred

    def fit_forecast(self, y, ps, npred):
        self.plain_calls += 1
        return O.fit_forecast_packed(np.asarray(y), self.X, self.t_fit, ps, npred)[0].astype(np.float32)

    def fit_forecast_ar(self, y, p, ps, npred):
        self.ar_calls += 1
        return {"pred": fit_forecast_ar_packed(np.asarray(y), self.X, self.t_fit, ps, npred, p)["pred"]
                .astype(np.float32)}


def _frame():
    parts = []
    for j, t in enumerate((200, 180)):
        y, start = mmf.synth.daily_store_item_demand(3, t, seed=30 + j, end=np.datetime64("2021-06-30") - 10 * j)
        days = (np.datetime64(start, "D") + np.arange(t)).astype("datetime64[ns]")
        for i in range(3):
            parts.append(pd.DataFrame({"Product": f"P{j}", "SKU": f"S{i}", "Date": days, "Demand": y[i]}))
    return pd.concat(parts, ignore_index=True)


def test_forecast_groups_with_the_oracle_engine():
    pdf = _frame()
    eng = _OracleEngine()
    out = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="future", engine=eng, ar=2)
    assert eng.ar_calls == 2 and eng.plain_calls == 0                   # one call per calendar bucket
    plain = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="future", engine=_OracleEngine())
    assert list(out.columns) == list(plain.columns) and (out.dtypes == plain.dtypes).all()
    assert out[["Product", "SKU", "Date"]].equals(plain[["Product", "SKU", "Date"]])
    assert not np.allclose(out["Demand_Fitted"], plain["Demand_Fitted"])
    for bad in (dict(ar=2, select=(1, 3)), dict(ar=2, interval=0.9), dict(ar=0), dict(ar=9), dict(ar=1.5)):
        with pytest.raises(ValueError):
            mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine(), **bad)
    one = pdf[pdf["SKU"] == "S0"][pdf["Product"] == "P0"]
    e1 = _OracleEngine()
    mmf.forecast_groups(one, freq="D", horizon=14, mode="future", engine=e1)
    assert e1.plain_calls == 1 and e1.ar_calls == 0                     # ar=None: the plain single-group path
