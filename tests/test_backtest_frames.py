"""CPU: ``backtest_groups`` / ``backtest_schema`` with the float64 backtest oracle standing in for the engine: schema and
dtypes, (key, Cutoff) order, origins placed per group relative to its own last date, the last origin's MSE equal to the
reference's held-out score (``build_tune_and_score_model``), short groups left out, ``forecast_groups`` unchanged."""
import datetime as dt

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

import mmf
from oracle import mmf_oracle as O
import backtest_oracle as B


class _OracleBacktestEngine:
    """Stands in for ForecastEngine where there is no GPU (test infrastructure only): plan_backtest / backtest and
    plan_calendar / fit_forecast on host arrays, computed by the float64 oracles."""

    def plan_backtest(self, start, t_len, freq="D", horizon=28, n_origins=3, step=None, design="trend_season_exog"):
        self.origin = B.origins(t_len, horizon, n_origins, step)
        days = mmf.design.calendar_grid(start, t_len, freq)
        self.X = mmf.design.design_matrix(days, t_len - horizon, design)
        self.h = horizon
        self.calls = getattr(self, "calls", 0) + 1
        return self.origin.astype(np.int32)

    def backtest(self, y, want_pred=True):
        y = np.asarray(y)
        pred, st = B.backtest_packed(y, self.X, self.origin, self.h)
        m, cnt = B.metrics(pred, B.actuals(y, self.origin, self.h))
        return {"pred": pred.astype(np.float32) if want_pred else None, "metrics": m.astype(np.float32),
                "count": cnt.astype(np.int32), "status": st}

    def plan_calendar(self, start, t_len, freq="D", horizon=28, mode="future", design="trend_season_exog"):
        if mode == "holdout":
            self.t_fit, n_rows, ps, npred = t_len - horizon, t_len, 0, t_len
        else:
            self.t_fit, n_rows, ps, npred = t_len, t_len + horizon, t_len, horizon
        days = mmf.design.calendar_grid(start, n_rows, freq)
        self.Xc = mmf.design.design_matrix(days, self.t_fit, design)
        return days[ps:ps + npred], ps, npred

    def fit_forecast(self, y, pred_start, n_pred, out=None):
        return O.fit_forecast_packed(np.asarray(y), self.Xc, self.t_fit, pred_start, n_pred)[0].astype(np.float32)


def weekly_frame(seed=11):
    """six groups on four calendars (different first and last dates), gaps in one, a zero in another, one group too
    short for any origin and one with room for only some"""
    rng = np.random.default_rng(seed)
    rows = []
    spec = [("P0", "S0", dt.date(2020, 1, 6), 90), ("P0", "S1", dt.date(2020, 1, 6), 90),
            ("P1", "S2", dt.date(2020, 6, 1), 50), ("P1", "S3", dt.date(2020, 1, 6), 90),
            ("P2", "S4", dt.date(2020, 3, 2), 40), ("P2", "S5", dt.date(2020, 6, 1), 70)]
    for k, (p, sku, start, n) in enumerate(spec):
        for i in range(n):
            if sku == "S1" and i in (10, 11, 40, 85):
                continue
            v = float(50 + 10 * k + 0.3 * i + 5 * rng.normal())
            if sku == "S3" and i == 88:
                v = 0.0
            rows.append((p, sku, start + dt.timedelta(weeks=i), v))
    df = pd.DataFrame(rows, columns=["Product", "SKU", "Date", "Demand"])
    return df.sample(frac=1.0, random_state=3).reset_index(drop=True), spec


KW = dict(freq="W-MON", horizon=8, n_origins=3, step=6)


def test_schema_dtypes_and_order():
    df, spec = weekly_frame()
    got = mmf.backtest_groups(df, engine=_OracleBacktestEngine(), **KW)
    assert list(got.columns) == ["Product", "SKU", "Cutoff", "N", "MSE", "MAE", "Bias", "MAPE"]
    assert got["N"].dtype == np.int32 and all(got[m].dtype == np.float32 for m in ("MSE", "MAE", "Bias", "MAPE"))
    assert got["Cutoff"].dtype.kind == "M"
    keyed = got[["Product", "SKU", "Cutoff"]]
    assert keyed.equals(keyed.sort_values(["Product", "SKU", "Cutoff"]).reset_index(drop=True))
    assert mmf.backtest_schema() == pa.schema([("Product", pa.string()), ("SKU", pa.string()), ("Cutoff", pa.date32()),
                                                ("N", pa.int32()), ("MSE", pa.float32()), ("MAE", pa.float32()),
                                                ("Bias", pa.float32()), ("MAPE", pa.float32())])
    pa.Table.from_pandas(got, schema=mmf.backtest_schema(), preserve_index=False)     # the frame fits its schema


def test_origins_per_group_and_short_groups():
    df, spec = weekly_frame()
    got = mmf.backtest_groups(df, engine=_OracleBacktestEngine(), **KW)
    h, K, step = KW["horizon"], KW["n_origins"], KW["step"]
    for p, sku, start, n in spec:
        g = got[got["SKU"] == sku]
        want = [t for t in (n - h - (K - 1 - k) * step for k in range(K)) if t >= 33]
        cut = np.array([np.datetime64(start + dt.timedelta(weeks=int(t)), "ns") for t in want], dtype="datetime64[ns]")
        assert np.array_equal(g["Cutoff"].to_numpy(), cut), sku     # relative to the group's own last date
    assert (got["SKU"] == "S4").sum() == 0                           # 40 weeks: no origin with 33 fit rows
    assert (got["SKU"] == "S2").sum() == 2                           # 50 weeks: origins 30 (left out), 36, 42
    assert set(got["N"][got["SKU"] == "S0"]) == {h}


def test_last_origin_mse_is_the_reference_held_out_score():
    df, spec = weekly_frame()
    got = mmf.backtest_groups(df, engine=_OracleBacktestEngine(), **KW)
    h = KW["horizon"]
    for p, sku, start, n in spec:
        if n - h < 33:
            continue
        out = O.build_tune_and_score_model(df[df["SKU"] == sku], freq="W-MON", horizon=h)
        tail = out.tail(h)
        e = tail["Demand_Fitted"].to_numpy(np.float64) - tail["Demand"].to_numpy(np.float64)
        ok = np.isfinite(e)
        last = got[got["SKU"] == sku].iloc[-1]
        assert last["N"] == ok.sum()
        np.testing.assert_allclose(last["MSE"], np.mean(e[ok] ** 2), rtol=1e-5)
        np.testing.assert_allclose(last["Bias"], np.mean(e[ok]), rtol=1e-4, atol=1e-4)


def test_one_call_per_bucket_and_forecast_groups_unchanged():
    df, spec = weekly_frame()
    eng = _OracleBacktestEngine()
    before = mmf.forecast_groups(df, freq="W-MON", horizon=8, engine=eng)
    mmf.backtest_groups(df, engine=eng, **KW)
    assert eng.calls == 3                    # four calendar buckets; S4's has no origin with 33 fit rows: not planned
    after = mmf.forecast_groups(df, freq="W-MON", horizon=8, engine=eng)
    pd.testing.assert_frame_equal(before, after)
    assert list(after.columns) == ["Product", "SKU", "Date", "Demand", "Demand_Fitted"]


def test_empty_result_has_the_columns():
    df, _ = weekly_frame()
    got = mmf.backtest_groups(df[df["SKU"] == "S4"], engine=_OracleBacktestEngine(), **KW)
    assert len(got) == 0 and list(got.columns) == ["Product", "SKU", "Cutoff", "N", "MSE", "MAE", "Bias", "MAPE"]
