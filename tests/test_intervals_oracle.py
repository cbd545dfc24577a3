"""The float64 oracle of the prediction standard errors (tests/interval_oracle.py, DESIGN.md section 2 item 7), on the
CPU: against an independent raw-basis route, and by Monte-Carlo coverage; and the interval= columns of the DataFrame /
Arrow boundary with the oracle standing in for the engine."""
import numpy as np
import pytest

from interval_oracle import fit_forecast_se_packed
from oracle import mmf_oracle as O


def _raw_route(y, X, t_fit, ps, npred):
    """lstsq on the raw design over the observed rows: sigma^2 = residuals / (n - rank), h = x' pinv(X_o'X_o) x"""
    n = y.shape[0]
    sigma, dof, se = np.full(n, np.nan), np.zeros(n, dtype=np.int64), np.full((n, npred), np.nan)
    Xf, Xp = X[:t_fit], X[ps:ps + npred]
    for i in range(n):
        obs = np.isfinite(y[i, :t_fit])
        if not obs.any():
            continue
        Xo = Xf[obs]
        beta, *_ = np.linalg.lstsq(Xo, y[i, :t_fit][obs], rcond=None)
        rss = float(((y[i, :t_fit][obs] - Xo @ beta) ** 2).sum())
        rank = np.linalg.matrix_rank(Xo)
        dof[i] = obs.sum() - rank
        if dof[i] > 0:
            sigma[i] = np.sqrt(rss / dof[i])
            h = np.einsum("ij,jk,ik->i", Xp, np.linalg.pinv(Xo.T @ Xo), Xp)
            se[i] = sigma[i] * np.sqrt(1.0 + h)
    return sigma, dof, se


def _gaussian(n, X, t_fit, seed, p_live):
    rng = np.random.default_rng(seed)
    beta = rng.normal(0, 1, (n, X.shape[1])) * p_live
    return (X[:t_fit] @ beta.T).T * 5.0 + 100.0 * p_live[0] + rng.normal(0, 2.0, (n, t_fit))


def _cases():
    daily = O.design_matrix(O.calendar_grid("2019-01-01", 228, "D"), 200)
    weekly = O.design_matrix(O.calendar_grid("2018-01-01", 130, "W-MON"), 104)
    exog = O.design_matrix(O.calendar_grid("2019-06-03", 400, "W-MON"), 372, "exog_only")
    rng = np.random.default_rng(1)
    caller = np.zeros((90, 16))
    caller[:, 0] = 1.0
    caller[:, 1:5] = rng.normal(0, 1, (90, 4))
    caller[:, 5] = caller[:, 1] + caller[:, 2]            # aliased with columns 1 and 2
    caller[:, 6] = caller[:, 3]                           # aliased with column 3
    return {"daily": (daily, 200, 200, 28, True), "weekly": (weekly, 104, 104, 26, True),
            "exog_only": (exog, 372, 0, 400, False), "caller_aliased": (caller, 80, 70, 20, True)}


@pytest.mark.parametrize("case", sorted(_cases()))
def test_oracle_matches_the_raw_lstsq_route(case):
    X, t_fit, ps, npred, const = _cases()[case]
    live = (np.abs(X[:t_fit]).sum(axis=0) > 0).astype(float)
    y = _gaussian(40, X, t_fit, seed=3, p_live=live)
    y[1, [5, 17, 60]] = np.nan                            # isolated gaps
    y[2, :8] = np.nan                                     # leading gaps
    y[3, ::3] = np.nan                                    # a third missing
    y[4, :] = np.nan                                      # empty
    y[5, 1:] = np.nan                                     # a single value: dof <= 0
    got = fit_forecast_se_packed(y, X, t_fit, ps, npred, has_constant=const)
    sigma, dof, se = _raw_route(y, X, t_fit, ps, npred)
    assert np.array_equal(got["dof"], np.where(np.isfinite(y[:, :t_fit]).any(axis=1), dof, 0)), case
    if case == "weekly":          # on Mondays the six day-of-week dummies are aliased, before 2020-03 covid as well
        assert got["dof"][0] == t_fit - 9
    ok = got["dof"] > 0
    assert np.isnan(got["sigma"][~ok]).all() and np.isnan(got["se"][~ok]).all()
    np.testing.assert_allclose(got["sigma"][ok], sigma[ok], rtol=1e-9)
    np.testing.assert_allclose(got["se"][ok], se[ok], rtol=1e-9)
    np.testing.assert_allclose(got["rss"][ok], got["sigma"][ok] ** 2 * got["dof"][ok], rtol=1e-12)


def test_monte_carlo_coverage_of_the_t_interval():
    """4,000 Gaussian series x 200 days with known per-series sigma, horizon 28: pred -+ t_{dof,0.95} se covers 90 % of
    the future values within 4 standard errors of the per-series coverage fractions (a series' 28 rows share its
    sigma-hat, so they are not independent)."""
    from scipy import stats
    t_fit, h, n = 200, 28, 4000
    X = O.design_matrix(O.calendar_grid("2019-01-01", t_fit + h, "D"), t_fit)
    rng = np.random.default_rng(7)
    sd = rng.uniform(0.5, 20.0, (n, 1))
    beta = rng.normal(0, 1, (n, X.shape[1]))
    mean = beta @ X.T + 50.0
    y = mean + sd * rng.normal(0, 1, mean.shape)
    got = fit_forecast_se_packed(y[:, :t_fit], X, t_fit, t_fit, h)
    q = stats.t.ppf(0.95, got["dof"])[:, None]
    per_series = (np.abs(y[:, t_fit:] - got["pred"]) <= q * got["se"]).mean(axis=1)
    err = per_series.std(ddof=1) / np.sqrt(n)
    assert abs(per_series.mean() - 0.9) <= 4 * err, (per_series.mean(), err)
    # and sigma-hat is an unbiased-variance estimate of the known sigma
    assert abs(float(np.mean(got["sigma"] ** 2 / sd[:, 0] ** 2)) - 1.0) < 0.02


# ---- the DataFrame / Arrow boundary: forecast_groups / forecast_table(..., interval=level) --------------------------
class _OracleSEEngine:
    """Stands in for ForecastEngine where there is no GPU (test infrastructure only): plan_calendar, fit_forecast and
    fit_forecast_se on host arrays, computed by the float64 oracles."""

    def plan_calendar(self, start, t_len, freq="D", horizon=28, mode="future", design="trend_season_exog"):
        import mmf
        if mode == "holdout":
            self.t_fit, n_rows, ps, npred = t_len - horizon, t_len, 0, t_len
        else:
            self.t_fit, n_rows, ps, npred = t_len, t_len + horizon, t_len, horizon
        days = mmf.design.calendar_grid(start, n_rows, freq)
        self.X = mmf.design.design_matrix(days, self.t_fit, design)
        self.has_constant = design == "trend_season_exog"
        return days[ps:ps + npred], ps, npred

    def fit_forecast(self, y, pred_start, n_pred, out=None):
        return O.fit_forecast_packed(np.asarray(y), self.X, self.t_fit, pred_start, n_pred)[0].astype(np.float32)

    def fit_forecast_se(self, y, pred_start, n_pred):
        r = fit_forecast_se_packed(np.asarray(y), self.X, self.t_fit, pred_start, n_pred, self.has_constant)
        return {"pred": r["pred"].astype(np.float32), "se": r["se"].astype(np.float32),
                "sigma": r["sigma"].astype(np.float32), "dof": r["dof"], "status": r["status"]}


def _weekly_frame():
    """four groups on two calendars (so the batch has two buckets), one with a gap"""
    import datetime as dt
    import pandas as pd
    rng = np.random.default_rng(11)
    rows = []
    for k, (start, n) in enumerate(((dt.date(2020, 1, 6), 80), (dt.date(2020, 1, 6), 80), (dt.date(2020, 6, 1), 60),
                                    (dt.date(2020, 1, 6), 80))):
        for i in range(n):
            if k == 1 and i in (10, 11, 40):
                continue
            rows.append((f"P{k % 2}", f"S{k}", start + dt.timedelta(weeks=i), float(50 + 10 * k + 5 * rng.normal())))
    return pd.DataFrame(rows, columns=["Product", "SKU", "Date", "Demand"])


@pytest.mark.parametrize("mode", ["holdout", "future"])
def test_interval_columns_in_the_frame_path(mode):
    import pandas as pd
    import pyarrow as pa
    from statistics import NormalDist

    import mmf
    df = _weekly_frame()
    eng = _OracleSEEngine()
    kw = dict(freq="W-MON", horizon=12, mode=mode, engine=eng)
    plain = mmf.forecast_groups(df, **kw)
    none = mmf.forecast_groups(df, interval=None, **kw)
    pd.testing.assert_frame_equal(plain, none)
    assert list(plain.columns) == ["Product", "SKU", "Date", "Demand", "Demand_Fitted"]
    got = mmf.forecast_groups(df, interval=0.9, **kw)
    assert list(got.columns) == list(plain.columns) + ["Demand_Lower", "Demand_Upper"]
    assert got["Demand_Lower"].dtype == np.float32 and got["Demand_Upper"].dtype == np.float32
    pd.testing.assert_frame_equal(got[plain.columns], plain)
    lo, fit, hi = (got[c].to_numpy(np.float64) for c in ("Demand_Lower", "Demand_Fitted", "Demand_Upper"))
    assert np.isfinite(lo).all() and (lo <= fit).all() and (fit <= hi).all()
    # the width is 2 z se with the normal quantile, se from the oracle of that group's own calendar
    z = NormalDist().inv_cdf(0.95)
    s0 = got[got["SKU"] == "S0"]
    t_len = 80
    X = O.design_matrix(O.calendar_grid("2020-01-06", t_len + (12 if mode == "future" else 0), "W-MON"),
                        t_len - (12 if mode == "holdout" else 0))
    y0 = df[df["SKU"] == "S0"]["Demand"].to_numpy(np.float32)[None, :]
    t_fit = t_len - (12 if mode == "holdout" else 0)
    ps, npred = (0, t_len) if mode == "holdout" else (t_len, 12)
    ref = fit_forecast_se_packed(y0, X, t_fit, ps, npred)
    np.testing.assert_allclose((s0["Demand_Upper"] - s0["Demand_Lower"]).to_numpy(np.float64), 2 * z * ref["se"][0],
                               rtol=1e-5)
    # the Arrow flavour: same values, schema opt-in
    table = pa.Table.from_pandas(df, preserve_index=False)
    at = mmf.forecast_table(table, interval=0.9, **kw)
    assert at.schema == mmf.frames.tuning_schema(interval=True)
    assert mmf.forecast_table(table, **kw).schema == mmf.frames.tuning_schema()
    assert mmf.frames.tuning_schema().names == ["Product", "SKU", "Date", "Demand", "Demand_Fitted"]
    for c in ("Demand_Fitted", "Demand_Lower", "Demand_Upper"):
        assert np.array_equal(at[c].to_numpy(zero_copy_only=False).astype(np.float32), got[c].to_numpy(), equal_nan=True)
    with pytest.raises(ValueError):
        mmf.forecast_groups(df, interval=1.5, **kw)
