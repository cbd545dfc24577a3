"""The float64 oracle of the ARIMA-family forecast standard errors (tests/arima_se_oracle.py, DESIGN.md section 2 item 15),
on the CPU: Monte-Carlo exactness against the shipped predictor on simulated paths (with power: the no-gaps rule fails
the same test), the textbook psi-weight variance on gap-free windows, the NaN pattern of the model oracles' predictions
on the demand shapes, and the conf_int= columns of the DataFrame / Arrow boundary with a fake engine."""
import numpy as np
import pytest

from arima_se_oracle import arima_se, predict, psi_star, simulate

# (phi, theta, d, gaps as [a, b) level rows of a 150-row fit window); 10 rows beyond it
MC_CASES = {
    "101": ([0.6], [0.4], 0, [(100, 110), (120, 121), (140, 141)]),
    "111": ([0.5], [0.3], 1, [(0, 3), (100, 107), (110, 111)]),
    "221": ([0.4, -0.2], [0.5], 2, [(100, 104), (106, 107)]),
    "011": ([], [0.7], 1, [(60, 61), (100, 102)]),
    "220": ([0.3, 0.2], [], 2, [(100, 102), (120, 121)]),
    "000": ([], [], 0, [(50, 60)]),
    "800": ([0.7, 0.1, -0.1, 0.05, 0.05, -0.05, 0.05, 0.05], [], 0, [(100, 101), (110, 114)]),
    "424": ([0.3, 0.1, -0.1, 0.1], [0.4, 0.2, 0.1, -0.1], 2, [(90, 93), (120, 121)]),
    "111_long_lead": ([0.5], [0.3], 1, [(0, 40)]),
    "221_long_tail": ([0.4, -0.2], [0.5], 2, [(118, 150)]),
}
T_FIT, H, N_PATHS = 150, 10, 40000


def _params(phi, theta):
    ph, th = np.zeros((1, 8)), np.zeros((1, 4))
    ph[0, :len(phi)], th[0, :len(theta)] = phi, theta
    return ph, th


def _mc(case, seed):
    phi, theta, d, gaps = MC_CASES[case]
    obs = np.ones(T_FIT, dtype=bool)
    for a, b in gaps:
        obs[a:b] = False
    rng = np.random.default_rng(seed)
    y = simulate(phi, theta, d, T_FIT + H, N_PATHS, rng)
    err = y - predict(y, obs, T_FIT, phi, theta, d, T_FIT + H)
    ph, th = _params(phi, theta)
    row = np.where(obs, 1.0, np.nan)[None, :]
    kw = dict(theta=th, ma_order=[len(theta)])
    se = arima_se(row, T_FIT, ph, [len(phi)], [1.0], 0, T_FIT + H, d, **kw)[0]
    nogaps = arima_se(row, T_FIT, ph, [len(phi)], [1.0], 0, T_FIT + H, d, no_gaps=True, **kw)[0]
    return obs, err, se, nogaps, gaps


@pytest.mark.parametrize("case", sorted(MC_CASES))
def test_monte_carlo_variance_of_the_shipped_predictor(case):
    """40,000 paths from a zero pre-sample: every row's empirical error variance is within 5 sqrt(2/N) (relative) of
    sigma^2 (1 + c'Pc), and se is NaN exactly where every path's prediction is"""
    obs, err, se, nogaps, gaps = _mc(case, seed=sorted(MC_CASES).index(case))
    fin = np.isfinite(se)
    assert np.array_equal(~fin, np.isnan(err).all(axis=0)), case
    assert not np.isnan(err[:, fin]).any()
    rel = np.abs(err[:, fin].var(axis=0) / se[fin] ** 2 - 1.0)
    assert rel.max() <= 5 * np.sqrt(2.0 / N_PATHS), (case, float(rel.max()))


@pytest.mark.parametrize("case", sorted(c for c in MC_CASES if c not in ("000", "011")))
def test_monte_carlo_rejects_the_no_gaps_rule(case):
    """the plausible wrong rule (every fit row observed) misses the empirical variance by more than 20 % on some row
    within 3 rows after a gap, so the test above has power (ARIMA(0, 0, 0) and the invertible MA(1) walk are
    exempt: their band does not depend on the gaps, or only barely)"""
    obs, err, se, nogaps, gaps = _mc(case, seed=100 + sorted(MC_CASES).index(case))
    after = np.zeros(T_FIT + H, dtype=bool)
    for a, b in gaps:
        after[b:b + 3] = True
    after &= np.isfinite(nogaps) & ~np.isnan(err).any(axis=0)
    assert after.any()
    rel = np.abs(err[:, after].var(axis=0) / nogaps[after] ** 2 - 1.0)
    assert rel.max() > 0.2, (case, float(rel.max()))


@pytest.mark.parametrize("p,d,q", [(0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 1), (2, 2, 1), (4, 2, 4), (8, 0, 4),
                                   (0, 2, 3), (3, 1, 0)])
def test_gap_free_rows_follow_the_psi_weights(p, d, q):
    """on a gap-free fit window se = sigma in sample (NaN for t < d) and sigma sqrt(sum_{j<h} psi*_j^2) beyond, psi*
    from scipy's impulse response summed d times: independent of the covariance recursion"""
    rng = np.random.default_rng(10 * p + 3 * d + q)
    n, t_fit, h = 6, 60, 25
    phi = np.zeros((n, 8))
    theta = np.zeros((n, 4))
    phi[:, :p] = rng.uniform(-0.3, 0.3, (n, p)) / max(p, 1)
    theta[:, :q] = rng.uniform(-0.5, 0.5, (n, q)) / max(q, 1)
    sigma = rng.uniform(0.5, 30.0, n)
    y = rng.normal(size=(n, t_fit))
    se = arima_se(y, t_fit, phi, np.full(n, p), sigma, 0, t_fit + h, d, theta=theta, ma_order=np.full(n, q))
    assert np.isnan(se[:, :d]).all()
    np.testing.assert_array_equal(se[:, d:t_fit], np.broadcast_to(sigma[:, None], (n, t_fit - d)))
    for i in range(n):
        want = sigma[i] * np.sqrt(np.cumsum(psi_star(phi[i, :p], theta[i, :q], d, h) ** 2))
        np.testing.assert_allclose(se[i, t_fit:], want, rtol=1e-12)
    if p == q == d == 0:
        assert (se == sigma[:, None]).all()
    if (p, q, d) == (0, 0, 1):
        np.testing.assert_allclose(se[:, t_fit:], sigma[:, None] * np.sqrt(np.arange(1, h + 1))[None, :], rtol=1e-14)


def test_invalid_rows_and_explosive_parameters():
    n, t_fit = 6, 40
    y = np.ones((n, t_fit))
    phi = np.zeros((n, 8))
    phi[:, 0] = 0.5
    order = np.array([1, 9, 1, 1, -1, 1])
    sigma = np.array([1.0, 1.0, np.nan, np.inf, 1.0, 1.0])
    diffs = np.array([1, 1, 1, 1, 1, -1])
    se = arima_se(y, t_fit, phi, order, sigma, 0, t_fit + 5, diffs=diffs)
    assert np.isfinite(se[0, 1:]).all() and np.isnan(se[1:]).all()
    phi[:, 0] = 3.0
    big = arima_se(y, t_fit, phi, np.ones(n), np.ones(n), t_fit, 1000, 2)
    assert np.isinf(big[:, -1]).all() and np.isfinite(big[:, 0]).all()


@pytest.mark.parametrize("d", [0, 1, 2])
def test_nan_pattern_equals_the_model_oracles_predictions(d):
    """on the demand shapes (launched, discontinued, stocked-out, intermittent), a non-empty series' se is NaN exactly
    where the ARIMA(1, d, 1) oracle's prediction is"""
    from arma_oracle import fit_forecast_arma_packed
    from demand_shapes import calendar, demand_batch
    _, t, _, X = calendar("weekly157", extra=12)
    y, kinds, _ = demand_batch(62, "weekly157", seed=3 + d)
    y[5, :4] = np.nan
    y[6, 10:14] = np.nan
    for ps, npred in ((0, t + 12), (t, 12), (40, t - 28)):
        want = fit_forecast_arma_packed(y, X, t, ps, npred, 1, 1, d)
        se = arima_se(y, t, want["phi"], want["order"], want["sigma"], ps, npred, d, theta=want["theta"],
                      ma_order=want["ma_order"])
        ok = want["status"] != 1
        assert np.array_equal(np.isnan(se[ok]), np.isnan(want["pred"][ok])), (d, ps)
        assert np.isnan(se[~ok]).all()


# ---- the DataFrame / Arrow boundary: forecast_groups / forecast_table(..., conf_int=level) --------------------------
class _FakeArimaEngine:
    """Stands in for ForecastEngine where there is no GPU (test infrastructure only): every ARIMA-family call returns
    predictions and standard errors that encode the row, so the frame's bounds can be checked exactly"""

    def __init__(self):
        self.calls = []

    def plan_calendar(self, start, t_len, freq="D", horizon=28, mode="future", design="trend_season_exog",
                      max_diff=None):
        import mmf
        ps, npred = (0, t_len) if mode == "holdout" else (t_len, horizon)
        return mmf.design.calendar_grid(start, ps + npred, freq)[ps:], ps, npred

    def _res(self, name, y, npred, want_se):
        self.calls.append((name, want_se))
        y = np.asarray(y)
        n = y.shape[0]
        pred = (np.arange(n)[:, None] * 100.0 + np.arange(npred)[None, :]).astype(np.float32)
        res = {"pred": pred}
        if want_se:
            res["se"] = np.full((n, npred), 2.0, dtype=np.float32)
            res["se"][:, 0] = np.nan
        return res

    def fit_forecast_ar(self, y, p, ps, npred, want_se=False):
        return self._res("ar", y, npred, want_se)

    def fit_select_ar(self, y, n_hold, orders, ps, npred, want_se=False):
        return self._res("select_ar", y, npred, want_se)

    def fit_forecast_arima(self, y, p, d, ps, npred, want_se=False):
        return self._res("arima", y, npred, want_se)

    def fit_select_arima(self, y, n_hold, orders, diffs, ps, npred, want_se=False):
        return self._res("select_arima", y, npred, want_se)

    def fit_forecast_arma(self, y, p, q, d, ps, npred, want_se=False):
        return self._res("arma", y, npred, want_se)

    def fit_select_arma(self, y, n_hold, orders, diffs, mas, ps, npred, want_se=False):
        return self._res("select_arma", y, npred, want_se)


FORMS = {"ar": dict(ar=2), "select_ar": dict(ar=(0, 1, 2)), "arima": dict(ar=1, diff=1),
         "select_arima": dict(ar=(0, 1), diff=(0, 1, 2)), "arma": dict(ar=1, diff=2, ma=1),
         "select_arma": dict(ar=(0, 1, 2, 3, 4), diff=(0, 1, 2), ma=(0, 1, 2, 3, 4))}


@pytest.mark.parametrize("form", sorted(FORMS))
def test_conf_int_columns_in_the_frame_path(form):
    import pandas as pd
    import pyarrow as pa
    from statistics import NormalDist

    import mmf
    from test_intervals_oracle import _weekly_frame
    df = _weekly_frame()
    eng = _FakeArimaEngine()
    kw = dict(freq="W-MON", horizon=12, mode="holdout", engine=eng, **FORMS[form])
    plain = mmf.forecast_groups(df, **kw)
    assert eng.calls and all(c == (form, False) for c in eng.calls)
    pd.testing.assert_frame_equal(plain, mmf.forecast_groups(df, conf_int=None, **kw))
    eng.calls.clear()
    got = mmf.forecast_groups(df, conf_int=0.9, **kw)
    assert eng.calls and all(c == (form, True) for c in eng.calls)
    assert list(got.columns) == list(plain.columns) + ["Demand_Lower", "Demand_Upper"]
    assert got["Demand_Lower"].dtype == np.float32 and got["Demand_Upper"].dtype == np.float32
    pd.testing.assert_frame_equal(got[plain.columns], plain)
    z = NormalDist().inv_cdf(0.95)
    fit = got["Demand_Fitted"].to_numpy(np.float64)
    first = got["Date"] == got.groupby("SKU")["Date"].transform("min")
    lo, hi = got["Demand_Lower"].to_numpy(np.float64), got["Demand_Upper"].to_numpy(np.float64)
    assert np.isnan(lo[first.to_numpy()]).all() and np.isnan(hi[first.to_numpy()]).all()
    rest = ~first.to_numpy()
    np.testing.assert_array_equal(lo[rest], (fit[rest] - z * 2.0).astype(np.float32))
    np.testing.assert_array_equal(hi[rest], (fit[rest] + z * 2.0).astype(np.float32))
    table = pa.Table.from_pandas(df, preserve_index=False)
    at = mmf.forecast_table(table, conf_int=0.9, **kw)
    assert at.schema == mmf.frames.tuning_schema(interval=True)
    assert mmf.forecast_table(table, **kw).schema == mmf.frames.tuning_schema()
    for c in ("Demand_Fitted", "Demand_Lower", "Demand_Upper"):
        assert np.array_equal(at[c].to_numpy(zero_copy_only=False).astype(np.float32), got[c].to_numpy(), equal_nan=True)


def test_conf_int_refusals():
    import mmf
    from test_intervals_oracle import _weekly_frame
    df = _weekly_frame()
    eng = _FakeArimaEngine()
    kw = dict(freq="W-MON", horizon=12, mode="holdout", engine=eng)
    for bad in (dict(conf_int=0.9),                                   # no ar=
                dict(conf_int=0.9, diff=1),
                dict(conf_int=0.9, ar=1, interval=0.9),               # the regression band is a different quantity
                dict(conf_int=0.9, ar=1, select=(1, 3)),
                dict(conf_int=0.0, ar=1), dict(conf_int=1.0, ar=1), dict(conf_int=1.5, ar=(0, 1)),
                dict(conf_int=-0.1, ar=1, diff=1, ma=1)):
        with pytest.raises(ValueError):
            mmf.forecast_groups(df, **kw, **bad)
        with pytest.raises(ValueError):
            mmf.forecast_table(df, **kw, **bad)
    assert not eng.calls
    # interval= keeps every refusal it had with the ARIMA family
    for bad in (dict(interval=0.9, ar=1), dict(interval=0.9, ar=1, diff=1), dict(interval=0.9, ar=1, ma=1)):
        with pytest.raises(ValueError):
            mmf.forecast_groups(df, **kw, **bad)
