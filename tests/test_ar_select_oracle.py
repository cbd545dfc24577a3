"""CPU: the float64 oracle of AR order selection by hold-out MSE (tests/ar_select_oracle.py) against an independent
restatement, its choice rules, and ``forecast_groups(ar=(0, 1, 2, 3, 4))`` with the oracle standing in for the engine."""
import numpy as np
import pandas as pd
import pytest

import mmf
from ar_oracle import fit_forecast_ar_packed
from ar_select_oracle import select_ar_packed
from oracle import mmf_oracle as O

ORDERS = (0, 1, 2, 3, 4)


def _ar_noise_case(n=40, t=260, n_hold=28, phi=0.9, seed=5):
    """daily design, y = level + AR(1) noise with coefficient phi; y has t_fit + n_hold columns"""
    rng = np.random.default_rng(seed)
    X = O.design_matrix(O.calendar_grid("2020-01-01", t + n_hold, "D"), t)
    noise = np.zeros((n, t + n_hold))
    eps = rng.normal(0, 5, (n, t + n_hold))
    for k in range(t + n_hold):
        noise[:, k] = eps[:, k] + (phi * noise[:, k - 1] if k else 0)
    y = 100.0 + rng.normal(0, 20, (n, X.shape[1])) @ X.T + noise
    return y.astype(np.float32), X, t


def test_scores_match_an_independent_loop():
    y, X, t_fit = _ar_noise_case(n=12, phi=0.6)
    y[3, t_fit + 5] = np.nan
    y[4, t_fit + 2] = np.inf
    y[5, 100:110] = np.nan
    n_hold = 28
    sel = select_ar_packed(y, X, t_fit, n_hold, ORDERS, t_fit, n_hold)
    plain, _ = O.fit_forecast_packed(y[:, :t_fit].astype(np.float64), X, t_fit, t_fit, n_hold)
    for i in range(len(y)):
        yh = y[i, t_fit:t_fit + n_hold].astype(np.float64)
        want = []
        for m in ORDERS:
            f = plain[i] if m == 0 else fit_forecast_ar_packed(y[i:i + 1, :t_fit], X, t_fit, t_fit, n_hold, m)["pred"][0]
            ok = np.isfinite(yh) & np.isfinite(f)
            want.append(np.mean((yh[ok] - f[ok]) ** 2))
        np.testing.assert_allclose(sel["cand_mse"][i], want, rtol=1e-12)
        assert sel["choice"][i] == ORDERS[int(np.argmin(want))]
        assert sel["mse"][i] == sel["cand_mse"][i].min() and np.isclose(sel["mse"][i], min(want), rtol=1e-12)
    assert sel["count"][3] == n_hold - 1 and sel["count"][4] == n_hold - 1 and sel["count"][0] == n_hold


def test_final_predictions_are_the_winners():
    y, X, t_fit = _ar_noise_case(n=10, phi=0.7)
    sel = select_ar_packed(y, X, t_fit, 28, ORDERS, 0, t_fit + 28)
    for i in range(len(y)):
        m = int(sel["choice"][i])
        if m == 0:
            want = O.fit_forecast_packed(y[i:i + 1, :t_fit].astype(np.float64), X, t_fit, 0, t_fit + 28)[0][0]
        else:
            r = fit_forecast_ar_packed(y[i:i + 1, :t_fit], X, t_fit, 0, t_fit + 28, m)
            want = r["pred"][0]
            assert sel["order"][i] == r["order"][0]
            np.testing.assert_allclose(sel["phi"][i], r["phi"][0], rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(sel["pred"][i], want, rtol=1e-9)


def test_ties_go_to_the_first_candidate():
    """a series with dof <= 1 gets order 0 from every candidate: all forecasts are the plain one, so 0 wins"""
    t_fit, n_hold = 60, 10
    s = np.arange(t_fit + n_hold, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), s / t_fit, np.sin(s / 5)])
    rng = np.random.default_rng(2)
    y = (50 + rng.normal(0, 3, (3, t_fit + n_hold))).astype(np.float32)
    y[:, :t_fit] = np.nan
    y[:, [3, 17, 33, 51]] = (50 + rng.normal(0, 3, (3, 4))).astype(np.float32)     # 4 observations, 3 columns: dof 1
    sel = select_ar_packed(y, X, t_fit, n_hold, (0, 1, 2, 3), t_fit, n_hold)
    assert (sel["cand_mse"] == sel["cand_mse"][:, :1]).all()
    assert (sel["choice"] == 0).all() and (sel["order"] == 0).all()
    sel = select_ar_packed(y, X, t_fit, n_hold, (2, 5), t_fit, n_hold)
    assert (sel["choice"] == 2).all()


def test_no_scored_point_takes_the_last_candidate():
    y, X, t_fit = _ar_noise_case(n=4)
    y[1, t_fit:] = np.nan
    y[2, t_fit:] = np.inf
    y[3, :] = np.nan                                                                  # empty: choice -1
    sel = select_ar_packed(y, X, t_fit, 28, (0, 2, 3), t_fit, 8)
    assert np.isnan(sel["cand_mse"][1:]).all() and np.isnan(sel["mse"][1:]).all()
    assert list(sel["choice"]) == [sel["choice"][0], 3, 3, -1]
    assert sel["status"][3] == 1 and np.isnan(sel["pred"][3]).all() and np.isnan(sel["sigma"][3])


def test_autocorrelated_noise_chooses_an_ar_order():
    """phi = 0.9 AR(1) noise, 28 held-out rows: an AR order wins on about three series in four (0.757 and 0.753 of 300
    series for seeds 5 and 6), not on nine in ten.  The score is multi-step: the AR gain over the plain forecast and
    the noise of that gain both scale with the last fit residual, so a 28-row window does not tell them apart more often.
    The mean hold-out MSE of every AR candidate stays below the plain one's."""
    y, X, t_fit = _ar_noise_case(n=120, phi=0.9)
    sel = select_ar_packed(y, X, t_fit, 28, ORDERS, t_fit, 28)
    share = float((sel["choice"] >= 1).mean())
    assert share >= 2 / 3, share
    mean = np.nanmean(sel["cand_mse"], axis=0)
    assert (mean[1:] < mean[0]).all(), mean


class _OracleSelectEngine:
    """Stands in for ForecastEngine where there is no GPU (test infrastructure only): plan_calendar, fit_forecast and
    fit_select_ar on host arrays, computed by the float64 oracles."""

    def __init__(self):
        self.calls = []

    def plan_calendar(self, start, t_len, freq="D", horizon=28, mode="future", design="trend_season_exog"):
        if mode == "holdout":
            self.t_fit, n_rows, ps, npred = t_len - horizon, t_len, 0, t_len
        else:
            self.t_fit, n_rows, ps, npred = t_len, t_len + horizon, t_len, horizon
        days = mmf.design.calendar_grid(start, n_rows, freq)
        self.X = mmf.design.design_matrix(days, self.t_fit, design)
        return days[ps:ps + npred], ps, npred

    def fit_forecast(self, y, pred_start, n_pred, out=None):
        return O.fit_forecast_packed(np.asarray(y), self.X, self.t_fit, pred_start, n_pred)[0].astype(np.float32)

    def fit_select_ar(self, y, n_hold, orders=ORDERS, pred_start=0, n_pred=None, want_stats=False):
        y = np.asarray(y)
        self.calls.append((y.shape, n_hold, tuple(orders)))
        sel = select_ar_packed(y, self.X, self.t_fit, n_hold, orders, pred_start, n_pred)
        return {"pred": sel["pred"].astype(np.float32), "choice": sel["choice"]}


def _frame():
    """five groups on two weekly calendars, one with gaps"""
    rng = np.random.default_rng(8)
    parts = []
    for k, (start, n) in enumerate((("2019-01-07", 120), ("2019-01-07", 120), ("2019-06-03", 100),
                                    ("2019-06-03", 100), ("2019-06-03", 100))):
        days = np.datetime64(start) + 7 * np.arange(n)
        noise = np.zeros(n)
        for i in range(1, n):
            noise[i] = 0.8 * noise[i - 1] + rng.normal(0, 4)
        v = 80 + 10 * k + 0.2 * np.arange(n) + noise
        keep = np.ones(n, dtype=bool)
        if k == 1:
            keep[[10, 11, 50]] = False
        parts.append(pd.DataFrame({"Product": f"P{k // 2}", "SKU": f"S{k}", "Date": days[keep].astype("datetime64[ns]"),
                                   "Demand": v[keep]}))
    return pd.concat(parts, ignore_index=True)


def test_forecast_groups_with_order_selection():
    pdf = _frame()
    eng = _OracleSelectEngine()
    kw = dict(freq="W-MON", horizon=20, mode="holdout")
    got = mmf.forecast_groups(pdf, ar=ORDERS, engine=eng, **kw)
    plain = mmf.forecast_groups(pdf, engine=_OracleSelectEngine(), **kw)
    assert list(got.columns) == list(plain.columns) and len(got) == len(plain)
    assert got.dtypes.equals(plain.dtypes)
    assert len(eng.calls) == 2 and all(c[1] == 20 and c[2] == ORDERS for c in eng.calls)
    # every group's Demand_Fitted is its own winner's holdout-mode prediction
    for (key, g) in got.groupby(["Product", "SKU"], sort=True):
        src = pdf[(pdf["Product"] == key[0]) & (pdf["SKU"] == key[1])].sort_values("Date")
        d0 = np.datetime64(src["Date"].min(), "D")
        t_len = len(g)
        y = np.full((1, t_len), np.nan)
        pos = (src["Date"].to_numpy().astype("datetime64[D]") - d0).astype(int) // 7
        y[0, pos] = src["Demand"].to_numpy()
        X = O.design_matrix(O.calendar_grid(d0, t_len, "W-MON"), t_len - 20)
        want = select_ar_packed(y.astype(np.float32), X, t_len - 20, 20, ORDERS, 0, t_len)
        np.testing.assert_allclose(g["Demand_Fitted"].to_numpy(), want["pred"][0].astype(np.float32), rtol=1e-6)


@pytest.mark.parametrize("bad, match", [
    ((), "at least one"), ((2, 1), "ascending"), ((1, 1), "ascending"), ((0, 9), r"\[0, 8\]"), ((-1, 2), r"\[0, 8\]"),
])
def test_forecast_groups_refuses_bad_order_lists(bad, match):
    with pytest.raises(ValueError, match=match):
        mmf.forecast_groups(_frame(), ar=bad, engine=_OracleSelectEngine(), freq="W-MON", horizon=20)


def test_forecast_groups_order_selection_needs_holdout_and_no_select_or_interval():
    pdf = _frame()
    eng = _OracleSelectEngine()
    with pytest.raises(ValueError, match="holdout"):
        mmf.forecast_groups(pdf, ar=ORDERS, engine=eng, freq="W-MON", horizon=20, mode="future")
    with pytest.raises(ValueError, match="select="):
        mmf.forecast_groups(pdf, ar=ORDERS, engine=eng, freq="W-MON", horizon=20, select=(4, 16))
    with pytest.raises(ValueError, match="interval="):
        mmf.forecast_groups(pdf, ar=ORDERS, engine=eng, freq="W-MON", horizon=20, interval=0.9)
    import pyarrow as pa
    with pytest.raises(ValueError, match="holdout"):
        mmf.forecast_table(pa.Table.from_pandas(pdf, preserve_index=False), ar=[0, 1], engine=eng, freq="W-MON",
                           horizon=20, mode="future")
    assert not eng.calls


def test_integer_ar_is_unchanged():
    with pytest.raises(ValueError, match=r"AR order in \[1, 8\]"):
        mmf.forecast_groups(_frame(), ar=0, engine=_OracleSelectEngine(), freq="W-MON", horizon=20)
    with pytest.raises(ValueError, match=r"AR order in \[1, 8\]"):
        mmf.forecast_groups(_frame(), ar=9, engine=_OracleSelectEngine(), freq="W-MON", horizon=20)
    from mmf import frames
    assert frames._ar_order(3, None, None, "future") == 3 and frames._ar_order(None, None, None) is None
