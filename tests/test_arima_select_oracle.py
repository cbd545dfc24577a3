"""CPU: the float64 oracle of (p, d) selection by hold-out MSE on levels (tests/arima_select_oracle.py, DESIGN.md section 2
item 12): scores against an independent loop, diffs = (0,) against AR order selection, the tie / eligibility /
no-scored-point rules, known answers, and forecast_groups(ar=(...), diff=(...)) with the oracle standing in for the
engine."""
import numpy as np
import pandas as pd
import pytest

import mmf
from ar_oracle import fit_forecast_ar_packed
from ar_select_oracle import select_ar_packed
from arima_oracle import fit_forecast_arima_packed
from arima_select_oracle import choose, select_arima_packed
from oracle import mmf_oracle as O

H = 28


def _daily(n, t, seed, kind, h=H):
    """y [n, t + h] on the default daily design: 'rw' random walks with drift, 'ar1' AR(1) noise (phi 0.5) around the
    design's trend and seasonality"""
    rng = np.random.default_rng(seed)
    X = O.design_matrix(O.calendar_grid("2019-01-01", t + h + 8, "D"), t)
    tt = t + h
    if kind == "rw":
        y = 500.0 + np.cumsum(rng.normal(1.5, 4.0, (n, tt)), axis=1)
    else:
        beta = rng.normal(0, 20, (n, X.shape[1]))
        e = rng.normal(0, 5, (n, tt))
        w = np.zeros((n, tt))
        for k in range(tt):
            w[:, k] = e[:, k] + (0.5 * w[:, k - 1] if k else 0)
        y = 300.0 + beta @ X[:tt].T + w
    return y.astype(np.float32), X, t


def test_scores_match_an_independent_loop():
    y, X, t = _daily(12, 200, 1, "rw")
    y[3, 50:60] = np.nan
    y[4, t + 2:t + 9] = np.nan
    y[5, t:] = np.nan                                                # no scored point
    orders, diffs = (0, 1, 3), (0, 1, 2)
    sel = select_arima_packed(y, X, t, H, orders, diffs, t, H)
    for k, d in enumerate(diffs):
        for j, p in enumerate(orders):
            if d == 0 and p == 0:
                f = O.fit_forecast_packed(y[:, :t].astype(np.float64), X, t, t, H)[0]
            elif d == 0:
                f = fit_forecast_ar_packed(y[:, :t], X, t, t, H, p)["pred"]
            else:
                f = fit_forecast_arima_packed(y[:, :t], X, t, t, H, p, d)["pred"]
            for i in range(len(y)):
                yh = y[i, t:t + H].astype(np.float64)
                ok = np.isfinite(yh) & np.isfinite(f[i])
                want = np.mean((yh[ok] - f[i][ok]) ** 2) if ok.any() else np.nan
                got = sel["cand_mse"][i, k, j]
                assert (np.isnan(want) and np.isnan(got)) or abs(got - want) <= 1e-9 * abs(want), (i, p, d)
    # the chosen candidate is the first minimum of its row and the predictions are its own
    for i in range(len(y)):
        k, j = sel["k"][i], sel["j"][i]
        flat = sel["cand_mse"][i].reshape(-1)
        if np.isfinite(flat).any():
            assert k * len(orders) + j == int(np.nanargmin(flat))
    i = 0
    k, j = sel["k"][i], sel["j"][i]
    r = (fit_forecast_arima_packed(y[:, :t], X, t, t, H, orders[j], diffs[k]) if diffs[k] else
         select_ar_packed(y, X, t, H, (orders[j],), t, H))
    assert np.allclose(sel["pred"][i], r["pred"][i], equal_nan=True)
    assert np.isnan(sel["cand_mse"][5]).all() and sel["choice_d"][5] == 2 and sel["choice_p"][5] == 3


def test_diffs_zero_is_ar_order_selection():
    y, X, t = _daily(16, 180, 2, "ar1")
    y[2, ::2] = np.nan
    y[3] = np.nan
    orders = (0, 1, 2, 4)
    a = select_arima_packed(y, X, t, H, orders, (0,), 0, t + H)
    b = select_ar_packed(y, X, t, H, orders, 0, t + H)
    assert np.array_equal(a["choice_p"], b["choice"]) and np.array_equal(a["choice_d"], np.where(b["choice"] < 0, -1, 0))
    for ka, kb in (("pred", "pred"), ("phi", "phi"), ("order", "order"), ("sigma", "sigma"), ("status", "status"),
                   ("mse", "mse")):
        assert np.array_equal(a[ka], b[kb], equal_nan=True), ka
    assert np.array_equal(a["cand_mse"][:, 0, :], b["cand_mse"], equal_nan=True)


def test_tie_eligibility_and_no_scored_point_rules():
    nan = np.nan
    cm = np.array([
        [[5.0, 3.0], [3.0, 4.0], [3.0, 3.0]],       # tie across d: the smaller d wins, then the smaller p
        [[nan, nan], [2.0, 2.0], [1.0, nan]],       # d = 0 unscored: the d = 2 minimum
        [[nan, nan], [nan, nan], [nan, nan]],       # nothing scored: the last eligible candidate
        [[4.0, 1.0], [0.5, 0.5], [0.1, 0.1]],       # d = 1, 2 not eligible: their scores do not count
        [[nan, nan], [nan, nan], [nan, nan]],       # nothing eligible
        [[nan, nan], [nan, nan], [nan, nan]],       # nothing scored, d = 2 not eligible: the last of d = 1
    ])
    el = np.array([[1, 1, 1], [1, 1, 1], [1, 1, 1], [1, 0, 0], [0, 0, 0], [1, 1, 0]], dtype=bool)
    k, j = choose(cm, el)
    assert k.tolist() == [0, 2, 2, 0, -1, 1] and j.tolist() == [1, 0, 1, 1, -1, 1]


def test_eligibility_of_a_series_with_every_other_value_missing():
    y, X, t = _daily(4, 160, 3, "rw")
    y[1, :t:2] = np.nan                                              # z' of d = 1 and 2 empty, y not
    y[2, :t] = np.nan                                                # empty for every d
    sel = select_arima_packed(y, X, t, H, (0, 1), (0, 1, 2), t, H)
    assert sel["eligible"][1].tolist() == [True, False, False] and sel["choice_d"][1] == 0
    assert np.isnan(sel["cand_mse"][1, 1:]).all()
    assert not sel["eligible"][2].any() and sel["choice_p"][2] == -1 and sel["choice_d"][2] == -1
    assert sel["status"][2] == 1 and np.isnan(sel["pred"][2]).all() and np.isnan(sel["sigma"][2])
    assert np.isnan(sel["mse"][2]) and sel["order"][2] == 0 and not sel["phi"][2].any()


# The two statistical thresholds are set from the oracle on these seeds, over (0..4) x (0, 1, 2) with 56 held-out days.
# A score chosen on one window is noisy: over 28 days the random walks pick d = 1 on 41 % (d = 2 on 33 %) and the AR(1)
# series pick d = 0 on 56 %.  Over 56 days, 200 random walks with drift pick d = 1 on 54 % (d = 0: 18 %, d = 2: 28 %),
# and 200 AR(1) series (phi 0.5) around the design pick d = 0 on 67 % (d = 1: 30 %, d = 2: 3 %).  The tests ask that
# the expected d be the most frequent choice and reach 50 % and 60 %.
def test_random_walks_with_drift_pick_d1():
    y, X, t = _daily(200, 300, 4, "rw", h=56)
    sel = select_arima_packed(y, X, t, 56, (0, 1, 2, 3, 4), (0, 1, 2), t, 56)
    frac = np.bincount(sel["choice_d"] + 1, minlength=4)[1:] / len(y)
    assert frac[1] >= 0.5 and frac.argmax() == 1, frac


def test_ar1_noise_around_the_design_picks_d0():
    y, X, t = _daily(200, 300, 4, "ar1", h=56)
    sel = select_arima_packed(y, X, t, 56, (0, 1, 2, 3, 4), (0, 1, 2), t, 56)
    frac = np.bincount(sel["choice_d"] + 1, minlength=4)[1:] / len(y)
    assert frac[0] >= 0.6 and frac.argmax() == 0, frac


def test_a_quadratic_on_a_t_squared_design_picks_d2():
    """y = a t^2 + b t + c with b != 0 on the caller design [1, t^2]: only d = 2 continues it exactly (d = 0 cannot fit
    the b t term, d = 1 turns it into a constant the differenced design [2t + 1] has no column for)"""
    t, n = 120, 6
    s = np.arange(t + H + 4, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), (s / t) ** 2])
    rng = np.random.default_rng(6)
    a, b, c = rng.uniform(5, 20, n), rng.uniform(3, 9, n), rng.uniform(100, 200, n)
    tt = np.arange(t + H, dtype=np.float64)
    y = a[:, None] * (tt / t) ** 2 + b[:, None] * tt + c[:, None]
    sel = select_arima_packed(y, X, t, H, (0, 1, 2), (0, 1, 2), t, H)
    assert (sel["choice_d"] == 2).all(), sel["choice_d"]
    assert (sel["mse"] <= 1e-12 * np.abs(y).max() ** 2).all()


class _OracleEngine:
    """stands in for ForecastEngine: plans a calendar, answers fit_forecast / fit_select_arima with the oracles"""

    def __init__(self):
        self.select_calls = 0
        self.plain_calls = 0
        self.max_diff = "unset"

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

    def fit_select_arima(self, y, n_hold, orders, diffs, ps, npred):
        assert (max(diffs) == 0 and self.max_diff is None) or self.max_diff == max(diffs)
        self.select_calls += 1
        sel = select_arima_packed(np.asarray(y), self.X, self.t_fit, n_hold, orders, diffs, ps, npred)
        return {"pred": sel["pred"].astype(np.float32)}


def _frame():
    parts = []
    for j, t in enumerate((200, 180)):
        y, start = mmf.synth.daily_store_item_demand(3, t, seed=40 + j, end=np.datetime64("2021-06-30") - 10 * j)
        days = (np.datetime64(start, "D") + np.arange(t)).astype("datetime64[ns]")
        for i in range(3):
            parts.append(pd.DataFrame({"Product": f"P{j}", "SKU": f"S{i}", "Date": days, "Demand": y[i]}))
    return pd.concat(parts, ignore_index=True)


@pytest.mark.parametrize("diffs", [(0, 1, 2), (0,), (1, 2)])
def test_forecast_groups_with_the_oracle_engine(diffs):
    pdf = _frame()
    eng = _OracleEngine()
    out = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=eng, ar=(0, 1, 2, 3, 4), diff=diffs)
    assert eng.select_calls == 2 and eng.plain_calls == 0                # one call per calendar bucket
    plain = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine())
    assert list(out.columns) == list(plain.columns) and (out.dtypes == plain.dtypes).all()
    assert out[["Product", "SKU", "Date"]].equals(plain[["Product", "SKU", "Date"]])
    e2 = _OracleEngine()
    tbl = mmf.forecast_table(pdf, freq="D", horizon=14, mode="holdout", engine=e2, ar=[0, 1, 2, 3, 4], diff=list(diffs))
    assert e2.select_calls == 2
    assert np.allclose(tbl.column("Demand_Fitted").to_numpy(zero_copy_only=False), out["Demand_Fitted"].to_numpy(),
                       equal_nan=True)


def test_forecast_groups_refusals():
    pdf = _frame()
    for bad in (dict(ar=(0, 1), diff=()), dict(ar=(0, 1), diff=(2, 1)), dict(ar=(0, 1), diff=(1, 1)),
                dict(ar=(0, 1), diff=(0, 3)), dict(ar=(0, 1), diff=(-1, 0)), dict(ar=(0, 1), diff=(True,)),
                dict(ar=1, diff=(0, 1)), dict(ar=None, diff=(0, 1)), dict(ar=(1, 0), diff=(0, 1)),
                dict(ar=(0, 9), diff=(0, 1)), dict(ar=(0, 1), diff=(0, 1), select=(1, 3)),
                dict(ar=(0, 1), diff=(0, 1), interval=0.9)):
        with pytest.raises(ValueError):
            mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine(), **bad)
        with pytest.raises(ValueError):
            mmf.forecast_table(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine(), **bad)
    with pytest.raises(ValueError):                                  # holdout mode only
        mmf.forecast_groups(pdf, freq="D", horizon=14, mode="future", engine=_OracleEngine(), ar=(0, 1), diff=(0, 1))
