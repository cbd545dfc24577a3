"""CPU: the float64 ARIMA(p, d, 0)-errors oracle (tests/arima_oracle.py) against an independent restatement of DESIGN.md
section 2 item 11, known answers, the residue rule, and forecast_groups(ar=..., diff=...) with the oracle standing in
for the engine."""
import numpy as np
import pandas as pd
import pytest
from scipy.linalg import solve_toeplitz

import mmf
from arima_oracle import diff_design, fit_forecast_arima_packed
from oracle import mmf_oracle as O


def _restated(y, X, t_fit, ps, npred, p, d):
    """np.diff, lstsq of Delta^d y on np.diff(X, d) over the observed rows, solve_toeplitz on the residuals, and a plain
    Python integration loop"""
    n_rows = X.shape[0]
    D = diff_design(X, t_fit, d)
    tz = t_fit - d
    out = np.full(npred, np.nan)
    z = np.diff(y[:t_fit], d)
    ok = np.isfinite(z)
    beta = np.linalg.lstsq(D[:tz][ok], z[ok], rcond=None)[0]
    e = np.where(ok, z - D[:tz] @ beta, 0.0)
    n_obs = ok.sum()
    r = np.array([e[k:] @ e[:tz - k] for k in range(p + 1)]) / n_obs
    phi = solve_toeplitz(r[:p], r[1:p + 1]) if p else np.zeros(0)
    u = {}
    zh = {}
    for s in range(n_rows - d):
        ar = sum(phi[j - 1] * u.get(s - j, 0.0) for j in range(1, p + 1))
        zh[s] = D[s] @ beta + ar
        u[s] = e[s] if s < tz and ok[s] else ar
    yt, yh = {}, {}
    for t in range(ps + npred):
        yh[t] = np.nan
        if t >= d:
            yh[t] = zh[t - d] + yt[t - 1] if d == 1 else zh[t - d] + 2 * yt[t - 1] - yt[t - 2]
        yt[t] = y[t] if t < t_fit and np.isfinite(y[t]) else yh[t]
        if t >= ps:
            out[t - ps] = yh[t]
    return out, phi


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("p", [0, 1, 3])
def test_oracle_against_an_independent_restatement(p, d):
    rng = np.random.default_rng(10 * p + d)
    t, h = 160, 20
    X = O.design_matrix(O.calendar_grid("2020-01-06", t + h, "D"), t)
    w = np.cumsum(rng.normal(0, 3, (7, t)), axis=1)
    y = 300 + w + rng.normal(0, 1, (7, t)) @ np.eye(t)
    y[0, t - 1] = np.nan                                   # gaps at t_fit - 1
    y[1, t - 2] = np.nan                                   # ... t_fit - 2
    y[2, :d] = np.nan                                      # in the first d rows
    y[3, 0] = np.nan
    y[4, 40:55] = np.nan                                   # a run
    y[5, 20::9] = np.nan                                   # throughout
    for ps, npred in ((t, h), (0, t + h), (50, 70)):
        res = fit_forecast_arima_packed(y, X, t, ps, npred, p, d)
        compared = 0
        for i in range(len(y)):
            if res["status"][i] == 2:                      # the pivot rule dropped a column lstsq keeps: another model
                continue
            compared += 1
            want, phi = _restated(y[i], X, t, ps, npred, p, d)
            got = res["pred"][i]
            assert np.array_equal(np.isnan(got), np.isnan(want)), (i, ps)
            fin = np.isfinite(want)
            scale = np.abs(want[fin]).max()
            assert np.allclose(got[fin], want[fin], rtol=1e-9, atol=1e-9 * scale), (i, ps, npred)
            if p and res["order"][i] == p:
                assert np.allclose(res["phi"][i, :p], phi, rtol=1e-9, atol=1e-12), i
        assert compared >= 5


def test_random_walk_with_drift_known_answer():
    """(0, 1) on [1, t]: the forecast is y_{T-1} + h mean(Delta y)"""
    rng = np.random.default_rng(3)
    t, h = 300, 15
    s = np.arange(t + h, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), s])
    y = np.cumsum(2.5 + rng.normal(0, 1, (4, t)), axis=1)
    res = fit_forecast_arima_packed(y, X, t, t, h, 0, 1)
    mu = np.diff(y, axis=1).mean(axis=1)
    want = y[:, -1:] + np.arange(1, h + 1)[None, :] * mu[:, None]
    assert np.allclose(res["pred"], want, rtol=1e-12, atol=1e-9)
    assert res["D"][:, 0].max() == 0.0 and np.all(res["D"][:, 1] == 1.0)      # Delta(intercept) = 0, drift column


def test_quadratic_continues_exactly():
    t, h = 200, 30
    s = np.arange(t + h, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), s, s * s])
    y = (3.0 + 0.5 * s - 0.01 * s * s)[None, :t].repeat(2, axis=0)
    res = fit_forecast_arima_packed(y, X, t, t, h, 0, 2)
    want = 3.0 + 0.5 * s[t:] - 0.01 * s[t:] ** 2
    assert np.allclose(res["pred"], want[None, :], rtol=1e-10, atol=1e-8)


def test_integrated_ar1_recovers_phi():
    rng = np.random.default_rng(11)
    n, t = 150, 1000
    X = O.design_matrix(O.calendar_grid("2018-01-01", t + 5, "D"), t)
    w = np.zeros((n, t))
    e = rng.normal(0, 1, (n, t))
    for k in range(t):
        w[:, k] = e[:, k] + (0.6 * w[:, k - 1] if k else 0)
    y = 100 + np.cumsum(w, axis=1)
    res = fit_forecast_arima_packed(y, X, t, t, 5, 1, 1)
    se = np.sqrt((1 - 0.36) / t)
    bias = 18 * 1.6 / t
    assert abs(res["phi"][:, 0].mean() - 0.6) < 5 * se / np.sqrt(n) + bias
    assert np.all(np.abs(res["phi"][:, 0] - 0.6) < 5 * se + bias)


def test_residue_rule_zeroes_the_second_difference_of_the_trend():
    t = 400
    X = O.design_matrix(O.calendar_grid("2019-01-01", t + 28, "D"), t)
    trend = 1                                                    # column 1 of the default design: the linear trend
    raw2 = np.diff(X, 2, axis=0)[:, trend]
    assert raw2[:t - 2].any() and np.abs(raw2[:t - 2]).max() <= 1e-12 * np.abs(X[:t, trend]).max()
    D2 = diff_design(X, t, 2)
    assert not D2[:, trend].any() and not D2[:, 0].any()
    D1 = diff_design(X, t, 1)
    assert not D1[:, 0].any() and np.ptp(D1[:t - 1, trend]) <= 1e-12 * np.abs(D1[:, trend]).max()
    W, kept = O.whiten(D2[:t - 2])
    assert not kept[trend] and not kept[0]


class _OracleEngine:
    """stands in for ForecastEngine: plans a calendar, answers fit_forecast / fit_forecast_arima with the oracles"""

    def __init__(self):
        self.arima_calls = 0
        self.plain_calls = 0
        self.max_diff = None

    def plan_calendar(self, start, t_len, freq="D", horizon=28, mode="future", design="trend_season_exog",
                      max_diff=None):
        self.max_diff = max_diff
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

    def fit_forecast_arima(self, y, p, d, ps, npred):
        assert self.max_diff is not None and d <= self.max_diff
        self.arima_calls += 1
        return {"pred": fit_forecast_arima_packed(np.asarray(y), self.X, self.t_fit, ps, npred, p, d)["pred"]
                .astype(np.float32)}


def _frame():
    parts = []
    for j, t in enumerate((200, 180)):
        y, start = mmf.synth.daily_store_item_demand(3, t, seed=30 + j, end=np.datetime64("2021-06-30") - 10 * j)
        days = (np.datetime64(start, "D") + np.arange(t)).astype("datetime64[ns]")
        for i in range(3):
            parts.append(pd.DataFrame({"Product": f"P{j}", "SKU": f"S{i}", "Date": days, "Demand": y[i]}))
    return pd.concat(parts, ignore_index=True)


@pytest.mark.parametrize("d", [1, 2])
def test_forecast_groups_with_the_oracle_engine(d):
    pdf = _frame()
    eng = _OracleEngine()
    out = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=eng, ar=1, diff=d)
    assert eng.arima_calls == 2 and eng.plain_calls == 0                # one call per calendar bucket
    plain = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine())
    assert list(out.columns) == list(plain.columns) and (out.dtypes == plain.dtypes).all()
    assert out[["Product", "SKU", "Date"]].equals(plain[["Product", "SKU", "Date"]])
    first = out.groupby(["Product", "SKU"], sort=True)["Demand_Fitted"].apply(lambda s: s.to_numpy()[:d + 1])
    for v in first:
        assert np.isnan(v[:d]).all() and np.isfinite(v[d])            # the first d dates of every group are NaN
    tbl = mmf.forecast_table(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine(), ar=1, diff=d)
    assert tbl.column("Demand_Fitted").null_count == d * 6
    assert np.allclose(tbl.column("Demand_Fitted").to_numpy(zero_copy_only=False), out["Demand_Fitted"].to_numpy(),
                       equal_nan=True)
    fut = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="future", engine=_OracleEngine(), ar=0, diff=d)
    assert np.isfinite(fut["Demand_Fitted"]).all()


def test_forecast_groups_refusals_and_diff_none_unchanged():
    pdf = _frame()
    for bad in (dict(ar=1, diff=(1,)), dict(ar=(0, 1), diff=1), dict(ar=None, diff=1), dict(ar=1, diff=3),
                dict(ar=1, diff=0), dict(ar=9, diff=1), dict(ar=1, diff=True), dict(ar=1, diff=1, select=(1, 3)),
                dict(ar=1, diff=1, interval=0.9), dict(ar=0)):
        with pytest.raises(ValueError):
            mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine(), **bad)
        with pytest.raises(ValueError):
            mmf.forecast_table(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine(), **bad)
    a = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="future", engine=_OracleEngine(), diff=None)
    b = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="future", engine=_OracleEngine())
    assert a.equals(b)
    one = pdf[(pdf["SKU"] == "S0") & (pdf["Product"] == "P0")]
    e1 = _OracleEngine()
    mmf.forecast_groups(one, freq="D", horizon=14, mode="future", engine=e1, diff=None)
    assert e1.plain_calls == 1 and e1.arima_calls == 0 and e1.max_diff is None
