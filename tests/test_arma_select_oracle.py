"""CPU: the float64 oracle of (p, d, q) selection by hold-out MSE on levels (tests/arma_select_oracle.py, DESIGN.md
section 2 item 14): scores against an independent loop over the single-candidate oracles, mas = (0,) against (p, d)
selection, gate-failing candidates, the eligibility / no-scored-point rules, a known answer, and forecast_groups(ar=(...),
diff=(...), ma=(...)) with the oracle standing in for the engine."""
import numpy as np
import pandas as pd
import pytest

import mmf
from arima_select_oracle import model as arima_model
from arima_select_oracle import select_arima_packed
from arma_oracle import fit_forecast_arma_packed
from arma_select_oracle import choose, default_long_order, select_arma_packed
from oracle import mmf_oracle as O

H = 28


def _daily(n, t, seed, theta=0.6, h=H):
    """y [n, t + h] on the default daily design: MA(1) errors (theta) around the design's trend and seasonality"""
    rng = np.random.default_rng(seed)
    X = O.design_matrix(O.calendar_grid("2019-01-01", t + h + 8, "D"), t)
    tt = t + h
    beta = rng.normal(0, 20, (n, X.shape[1]))
    e = rng.normal(0, 5, (n, tt + 1))
    y = 300.0 + beta @ X[:tt].T + e[:, 1:] + theta * e[:, :-1]
    return y.astype(np.float32), X, t


def test_long_order_per_d():
    assert default_long_order(400, 0, (0, 1, 2, 3, 4), (0, 1, 2, 3, 4)) == 32     # floor(ln(400)^2) = 35
    assert default_long_order(117, 1, (0, 1, 2, 3, 4), (0, 1, 2, 3, 4)) == 22     # floor(ln(116)^2) = 22
    # below 55 fit rows the call's m_d can exceed a single call's default 2 max(p, q)
    assert default_long_order(40, 0, (0, 1), (0, 1, 4)) == 13
    from arma_oracle import default_long_order as single_default
    assert single_default(40, 1, 1) == 13 and single_default(60, 1, 1) == 16


def test_scores_match_an_independent_loop():
    y, X, t = _daily(10, 200, 1)
    y[3, 50:60] = np.nan
    y[4, t + 2:t + 9] = np.nan
    y[5, t:] = np.nan                                                # no scored point
    orders, diffs, mas = (0, 2), (0, 1), (0, 1, 2)
    sel = select_arma_packed(y, X, t, H, orders, diffs, mas, t, H)
    for k, d in enumerate(diffs):
        m = default_long_order(t, d, orders, mas)
        assert sel["m"][k] == m
        for l, q in enumerate(mas):
            for j, p in enumerate(orders):
                if q == 0:
                    f = arima_model(y, X, t, t, H, p, d)["pred"]
                else:
                    f = fit_forecast_arma_packed(y[:, :t], X, t, t, H, p, q, d, m)["pred"]
                for i in range(len(y)):
                    yh = y[i, t:t + H].astype(np.float64)
                    ok = np.isfinite(yh) & np.isfinite(f[i])
                    want = np.mean((yh[ok] - f[i][ok]) ** 2) if ok.any() else np.nan
                    got = sel["cand_mse"][i, k, l, j]
                    assert (np.isnan(want) and np.isnan(got)) or abs(got - want) <= 1e-9 * abs(want), (i, p, d, q)
    # the chosen candidate is the first minimum of its row in list order (d, q, p), its outputs are its own
    for i in range(len(y)):
        flat = sel["cand_mse"][i].reshape(-1)
        if np.isfinite(flat).any():
            no, nq = len(orders), len(mas)
            assert (sel["k"][i] * nq + sel["l"][i]) * no + sel["j"][i] == int(np.nanargmin(flat))
    i = int(np.flatnonzero(sel["choice_q"] > 0)[0])
    k, l, j = sel["k"][i], sel["l"][i], sel["j"][i]
    r = fit_forecast_arma_packed(y[:, :t], X, t, t, H, orders[j], mas[l], diffs[k], sel["m"][k])
    for key in ("pred", "phi", "theta", "order", "ma_order", "sigma", "status"):
        assert np.allclose(sel[key][i], r[key][i], equal_nan=True), key
    assert np.isnan(sel["cand_mse"][5]).all() and sel["choice_q"][5] == 0
    assert sel["choice_d"][5] == 1 and sel["choice_p"][5] == 2                  # the last eligible q = 0 candidate


def test_mas_zero_is_pd_selection():
    y, X, t = _daily(12, 180, 2)
    y[2, ::2] = np.nan
    y[3] = np.nan
    orders, diffs = (0, 1, 2, 4), (0, 1, 2)
    a = select_arma_packed(y, X, t, H, orders, diffs, (0,), 0, t + H)
    b = select_arima_packed(y, X, t, H, orders, diffs, 0, t + H)
    for key in ("pred", "choice_p", "choice_d", "mse", "phi", "order", "sigma", "status"):
        assert np.array_equal(a[key], b[key], equal_nan=True), key
    assert np.array_equal(a["cand_mse"][:, :, 0, :], b["cand_mse"], equal_nan=True)
    assert np.array_equal(a["choice_q"], np.where(b["choice_p"] < 0, -1, 0))
    assert not a["theta"].any() and not a["ma_order"].any()


def test_a_gate_failing_candidate_scores_as_q0_and_never_wins():
    """every other fit value missing: no row t has t - 1 observed, so R is empty and every q >= 1 candidate falls back"""
    y, X, t = _daily(6, 200, 3)
    y[:, 1:t:2] = np.nan
    orders, diffs, mas = (0, 1, 2), (0,), (0, 1, 3)
    sel = select_arma_packed(y, X, t, H, orders, diffs, mas, t, H)
    for l in (1, 2):
        for j in range(len(orders)):
            assert not sel["hold"][0][l][j]["gated"].any()
            assert np.array_equal(sel["cand_mse"][:, 0, l, j], sel["cand_mse"][:, 0, 0, j], equal_nan=True)
    assert (sel["choice_q"] == 0).all() and not sel["theta"].any()


def test_choice_eligibility_and_no_scored_point_rules():
    nan = np.nan
    cm = np.full((5, 2, 2, 2), nan)
    cm[0] = [[[5.0, 3.0], [3.0, 2.0]], [[2.0, 4.0], [nan, nan]]]     # q = 1 of d = 0 ties with (0, 1, 0): d first
    cm[1] = [[[nan, nan], [nan, 7.0]], [[nan, nan], [nan, nan]]]     # only a q >= 1 candidate scores: it wins
    cm[2] = [[[4.0, 1.0], [0.5, 0.5]], [[0.1, 0.1], [0.1, 0.1]]]     # d = 1 not eligible
    el = np.array([[1, 1], [1, 1], [1, 0], [1, 1], [0, 0]], dtype=bool)  # 3: nothing scored; 4: nothing eligible
    k, l, j = choose(cm, el)
    assert k.tolist() == [0, 0, 0, 1, -1] and l.tolist() == [1, 1, 1, 0, -1] and j.tolist() == [1, 1, 0, 1, -1]


def test_eligibility_of_a_series_with_every_other_value_missing():
    y, X, t = _daily(4, 160, 3)
    y[1, :t:2] = np.nan                                              # z' of d = 1 and 2 empty, y not
    y[2, :t] = np.nan                                                # empty for every d
    sel = select_arma_packed(y, X, t, H, (0, 1), (0, 1, 2), (0, 1), t, H)
    assert sel["eligible"][1].tolist() == [True, False, False] and sel["choice_d"][1] == 0
    assert np.isnan(sel["cand_mse"][1, 1:]).all()
    assert not sel["eligible"][2].any() and (sel["choice_p"][2], sel["choice_d"][2], sel["choice_q"][2]) == (-1, -1, -1)
    assert sel["status"][2] == 1 and np.isnan(sel["pred"][2]).all() and np.isnan(sel["sigma"][2])
    assert np.isnan(sel["mse"][2]) and sel["order"][2] == 0 and sel["ma_order"][2] == 0 and not sel["theta"][2].any()


# The threshold is set from the oracle on this seed, over (0, 1, 2) x (0, 1) x (0, 1, 2) with 56 held-out days: 120
# series with MA(1) theta = 0.6 errors around the default design pick q >= 1 on 53 % (q = 1: 24 %, q = 2: 29 %); the
# test asks that q >= 1 win more often than q = 0.  The answer is weak evidence: the same rows with white-noise errors
# (theta = 0) pick q >= 1 on 56 %.  An MA(1) term changes only the first step of a dynamic forecast, so over 56 days the
# candidates' scores differ by less than their sampling noise, and the first minimum over 18 near-equal scores lands on
# a q >= 1 candidate about as often with or without MA errors.  Per-series hold-out selection does not identify q.
def test_ma1_errors_pick_q_at_least_1():
    y, X, t = _daily(120, 300, 4, h=56)
    sel = select_arma_packed(y, X, t, 56, (0, 1, 2), (0, 1), (0, 1, 2), t, 56)
    frac = float((sel["choice_q"] >= 1).mean())
    assert frac > 0.5, frac


class _OracleEngine:
    """stands in for ForecastEngine: plans a calendar, answers fit_forecast / fit_select_arma with the oracles"""

    def __init__(self):
        self.select_calls = 0
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
        return O.fit_forecast_packed(np.asarray(y), self.X, self.t_fit, ps, npred)[0].astype(np.float32)

    def fit_select_arma(self, y, n_hold, orders, diffs, mas, ps, npred):
        assert (max(diffs) == 0 and self.max_diff is None) or self.max_diff == max(diffs)
        self.select_calls += 1
        sel = select_arma_packed(np.asarray(y), self.X, self.t_fit, n_hold, orders, diffs, mas, ps, npred)
        return {"pred": sel["pred"].astype(np.float32)}


def _frame():
    parts = []
    for j, t in enumerate((150, 140)):
        y, start = mmf.synth.daily_store_item_demand(2, t, seed=40 + j, end=np.datetime64("2021-06-30") - 10 * j)
        days = (np.datetime64(start, "D") + np.arange(t)).astype("datetime64[ns]")
        for i in range(2):
            parts.append(pd.DataFrame({"Product": f"P{j}", "SKU": f"S{i}", "Date": days, "Demand": y[i]}))
    return pd.concat(parts, ignore_index=True)


@pytest.mark.parametrize("diffs", [(0, 1), None])
def test_forecast_groups_with_the_oracle_engine(diffs):
    pdf = _frame()
    eng = _OracleEngine()
    out = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=eng, ar=(0, 1), diff=diffs, ma=(0, 1))
    assert eng.select_calls == 2                                     # one call per calendar bucket
    plain = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine())
    assert list(out.columns) == list(plain.columns) and (out.dtypes == plain.dtypes).all()
    assert out[["Product", "SKU", "Date"]].equals(plain[["Product", "SKU", "Date"]])
    e2 = _OracleEngine()
    tbl = mmf.forecast_table(pdf, freq="D", horizon=14, mode="holdout", engine=e2, ar=[0, 1],
                             diff=None if diffs is None else list(diffs), ma=[0, 1])
    assert e2.select_calls == 2
    assert np.allclose(tbl.column("Demand_Fitted").to_numpy(zero_copy_only=False), out["Demand_Fitted"].to_numpy(),
                       equal_nan=True)


def test_forecast_groups_refusals():
    pdf = _frame()
    for bad in (dict(ar=(0, 1), ma=(1, 2)), dict(ar=(0, 1), ma=()), dict(ar=(0, 1), ma=(0, 0)),
                dict(ar=(0, 1), ma=(0, 2, 1)), dict(ar=(0, 1), ma=(0, 5)), dict(ar=(0, 1), ma=(0, True)),
                dict(ar=1, ma=(0, 1)), dict(ar=None, ma=(0, 1)), dict(ar=(0, 1), diff=1, ma=(0, 1)),
                dict(ar=(0, 1), diff=(1, 0), ma=(0, 1)), dict(ar=(0, 1), diff=(0, 3), ma=(0, 1)),
                dict(ar=tuple(range(9)), ma=(0, 1, 2, 3, 4)), dict(ar=(0, 1), ma=(0, 1), select=(1, 3)),
                dict(ar=(0, 1), ma=(0, 1), interval=0.9)):
        with pytest.raises(ValueError):
            mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine(), **bad)
        with pytest.raises(ValueError):
            mmf.forecast_table(pdf, freq="D", horizon=14, mode="holdout", engine=_OracleEngine(), **bad)
    with pytest.raises(ValueError):                                  # holdout mode only
        mmf.forecast_groups(pdf, freq="D", horizon=14, mode="future", engine=_OracleEngine(), ar=(0, 1), ma=(0, 1))
