"""CPU: the float64 CSS oracle of tests/arma_css_oracle.py (DESIGN.md section 2 item 16): its Jacobian against central
finite differences (gap-free, isolated gaps, gaps longer than q, a gap before row p), the two-filter form before the first
gap, a non-increasing objective along the LM path, optimality against SciPy, the theta RMSE against Hannan-Rissanen on
simulated MA(1) rows, the negative control's failure on gappy rows, the header constants and the frame layer's
estimator= argument."""
import os
import re

import numpy as np
import pytest

import arma_css_oracle as S
import arma_oracle as A
from oracle import mmf_oracle as O
from test_arima_oracle import _OracleEngine as _ArimaOracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# relative decrease of S that SciPy's least_squares finds from the oracle's converged answers: at worst 1.0e-6 on the
# rows of test_converged_rows_are_optimal and 2.5e-6 on gappy_rows (RTOL stops at a step that gains <= 1e-6 x S, and
# LM's last steps gain a few times that); the threshold leaves a factor of 4
OPT_RTOL = 1e-5


def _arma_series(T, phi, theta, seed, gaps=0.0, sd=1.0):
    rng = np.random.default_rng(seed)
    eps = rng.normal(0, sd, T + 200)
    u = np.zeros(T + 200)
    for s in range(T + 200):
        u[s] = eps[s] + sum(theta[k] * eps[s - 1 - k] for k in range(len(theta)) if s - 1 - k >= 0) + \
               sum(phi[j] * u[s - 1 - j] for j in range(len(phi)) if s - 1 - j >= 0)
    e = u[200:]
    obs = np.ones(T, dtype=bool)
    if gaps:
        obs[rng.choice(np.arange(T), size=int(gaps * T), replace=False)] = False
    return np.where(obs, e, 0.0), obs


def _gap_cases():
    base = np.ones(120, dtype=bool)
    iso = base.copy(); iso[[20, 47, 90]] = False
    long = base.copy(); long[30:38] = False; long[80:86] = False
    early = base.copy(); early[1] = False; early[60] = False
    return {"gap-free": base, "isolated": iso, "longer than q": long, "before p": early}


@pytest.mark.parametrize("case", list(_gap_cases()))
@pytest.mark.parametrize("p,q", [(1, 1), (2, 2), (0, 3), (3, 1)])
def test_jacobian_matches_central_differences(case, p, q):
    obs = _gap_cases()[case]
    e, _ = _arma_series(len(obs), [0.4, -0.1, 0.05][:p], [0.5, 0.2, -0.1][:q], seed=p * 10 + q)
    e = np.where(obs, e, 0.0)
    x = np.r_[np.array([0.3, -0.1, 0.05])[:p], np.array([0.4, 0.15, -0.1])[:q]]
    _, J, _, _ = S.css_eval(e, obs, len(obs), p, q, x)
    h = 1e-6
    for k in range(p + q):
        xp, xm = x.copy(), x.copy()
        xp[k] += h
        xm[k] -= h
        fd = (S.css_eval(e, obs, len(obs), p, q, xp)[2] - S.css_eval(e, obs, len(obs), p, q, xm)[2]) / (2 * h)
        assert np.allclose(J[:, k], fd, rtol=1e-6, atol=1e-7), (case, k, np.abs(J[:, k] - fd).max())
    if case != "gap-free":    # the control's Jacobian is wrong somewhere after the first gap
        _, Jn, _, _ = S.css_eval(e, obs, len(obs), p, q, x, gap_jacobian=False)
        assert np.abs(Jn - J).max() > 1e-3


@pytest.mark.parametrize("p,q", [(1, 1), (2, 3), (0, 4)])
def test_two_filter_form_equals_the_recursion_before_the_first_gap(p, q):
    obs = _gap_cases()["isolated"]
    e, _ = _arma_series(len(obs), [0.5, -0.2][:p], [0.4, 0.2, 0.1, -0.1][:q], seed=3)
    e = np.where(obs, e, 0.0)
    x = np.r_[np.array([0.45, -0.15])[:p], np.array([0.35, 0.1, 0.05, -0.05])[:q]]
    _, J, _, _ = S.css_eval(e, obs, len(obs), p, q, x)
    J2 = S.two_filter_jacobian(e, obs, len(obs), p, q, x)
    first = int(np.flatnonzero(~obs)[0])
    assert np.allclose(J[:first], J2[:first], rtol=1e-12, atol=1e-12)
    # and the control build's rule is the two-filter form on every row
    _, Jn, _, _ = S.css_eval(e, obs, len(obs), p, q, x, gap_jacobian=False)
    assert np.allclose(Jn, J2, rtol=1e-10, atol=1e-10)


def _hr_start(e, obs, T, p, q):
    m = A.default_long_order(T, p, q)
    h = A.hannan_rissanen(e, obs, T, T, p, q, m)
    return (h["beta"].astype(np.float32) if h["ok"] else None), h


@pytest.mark.parametrize("seed", range(12))
def test_objective_never_increases_and_stop_rules(seed):
    rng = np.random.default_rng(seed)
    p, q = [(1, 1), (0, 1), (2, 1), (1, 2)][seed % 4]
    e, obs = _arma_series(300, [0.5, -0.2][:p], [0.6, 0.2][:q], seed, gaps=0.02 * (seed % 3))
    x0, _ = _hr_start(e, obs, 300, p, q)
    if x0 is None:
        pytest.skip("HR gate failed")
    for mi in (1, 0, 64):
        r = S.lm(e, obs, 300, p, q, x0, mi)
        assert all(b <= a for a, b in zip(r["path"], r["path"][1:]))
        assert r["S"] <= r["S0"] and r["iters"] <= (mi or S.ITER_DEFAULT)
        assert r["stop"] in (1, 2, 3)
        if mi == 1:
            assert r["iters"] == 1 and r["stop"] == 3 and r["n_acc"] == 0 and r["S"] == r["S0"]
        assert rng is not None


def test_converged_rows_are_optimal():
    worst, n_conv = 0.0, 0
    for seed in range(30):
        p, q = [(1, 1), (0, 1), (0, 2)][seed % 3]
        e, obs = _arma_series(240, [0.5][:p], [0.7, 0.2][:q], 100 + seed, gaps=0.01 * (seed % 2))
        x0, _ = _hr_start(e, obs, 240, p, q)
        if x0 is None:
            continue
        r = S.lm(e, obs, 240, p, q, x0, 64)
        if r["stop"] != 1:
            continue
        n_conv += 1
        worst = max(worst, S.optimality_gap(e, obs, 240, p, q, r["x"]))
    assert n_conv >= 20
    assert worst <= OPT_RTOL, worst


def _ma1_rows(n, T, seed, theta=0.8, gaps=0.0):
    """gated MA(1) rows with a calendar regression part, through the HR oracle -> (res, rows)"""
    rng = np.random.default_rng(seed)
    X = O.design_matrix(O.calendar_grid("2019-01-07", T + 4, "W-MON" if T < 300 else "D"), T)
    eps = rng.normal(0, 5, (n, T + 1))
    u = eps[:, 1:] + theta * eps[:, :-1]
    y = 300.0 + rng.normal(0, 10, (n, X.shape[1])) @ X[:T].T + u
    if gaps:
        for i in range(n):
            y[i, rng.choice(np.arange(2, T - 1), size=max(int(gaps * T), 1), replace=False)] = np.nan
    return y, X


@pytest.mark.parametrize("T,n", [(117, 300), (1095, 60)])
def test_theta_rmse_beats_hannan_rissanen(T, n):
    y, X = _ma1_rows(n, T, seed=7)
    res = S.fit_forecast_arma_css_packed(y, X, T, T, 1, 0, 1)
    g = res["gated"]
    assert g.sum() >= 0.8 * n
    th_hr = np.array([res["hr"][i]["beta"][0] for i in np.flatnonzero(g)])
    th_css = res["theta"][g, 0]
    rmse_hr = np.sqrt(np.mean((th_hr - 0.8) ** 2))
    rmse_css = np.sqrt(np.mean((th_css - 0.8) ** 2))
    assert rmse_css <= 0.8 * rmse_hr, (rmse_css, rmse_hr)


NRUN = 20


def gappy_rows(n=40, T=365, seed=23):
    """the negative control's set: MA(2) errors, about 16 % of the values missing in runs of 3 (with 5 % the control's
    optimality gaps straddle the threshold on fewer than half of the rows)"""
    rng = np.random.default_rng(seed)
    X = O.design_matrix(O.calendar_grid("2019-01-01", T + 28, "D"), T)
    eps = rng.normal(0, 5, (n, T + 2))
    u = eps[:, 2:] + 0.7 * eps[:, 1:-1] + 0.3 * eps[:, :-2]
    y = rng.normal(0, 2, (n, X.shape[1])) @ X[:T].T + u           # no level: fp32 residuals stay close to float64
    for i in range(n):
        for s in rng.choice(np.arange(20, T - 4), size=NRUN, replace=False):
            y[i, s:s + 3] = np.nan
    return y, X


def test_negative_control_fails_the_optimality_check_on_gappy_rows():
    y, X = gappy_rows()
    T = y.shape[1]
    hr = A.fit_forecast_arma_packed(y, X, T, T, 1, 1, 2, 0)
    good = S.fit_forecast_arma_css_packed(y, X, T, T, 1, 1, 2, hr=hr)
    bad = S.fit_forecast_arma_css_packed(y, X, T, T, 1, 1, 2, gap_jacobian=False, hr=hr)
    rows = np.flatnonzero(hr["gated"])
    assert len(rows) >= 20
    fails = 0
    for i in rows:
        x_bad = np.r_[bad["phi"][i, :1], bad["theta"][i, :2]]
        x_good = np.r_[good["phi"][i, :1], good["theta"][i, :2]]
        gap_good = S.optimality_gap(hr["e"][i], hr["obs"][i], hr["T"], 1, 2, x_good)
        gap_bad = S.optimality_gap(hr["e"][i], hr["obs"][i], hr["T"], 1, 2, x_bad)
        if good["css_stop"][i] == 1:
            assert gap_good <= OPT_RTOL, (i, gap_good)
        fails += gap_bad > OPT_RTOL
    assert fails >= 0.5 * len(rows), (fails, len(rows))


def test_header_constants_equal_the_oracle():
    from mmf import _native as N
    with open(os.path.join(ROOT, "include", "mmf.h")) as f:
        h = f.read()

    def num(name):
        return float(re.search(rf"#define {name} ([0-9.e+-]+)", h).group(1))

    assert num("MMF_CSS_LAMBDA0") == S.LAMBDA0 == N.CSS_LAMBDA0
    assert num("MMF_CSS_LAMBDA_MAX") == S.LAMBDA_MAX == N.CSS_LAMBDA_MAX
    assert num("MMF_CSS_RTOL") == S.RTOL == N.CSS_RTOL
    assert num("MMF_CSS_ITER_DEFAULT") == S.ITER_DEFAULT == N.CSS_ITER_DEFAULT
    assert num("MMF_CSS_ITER_MAX") == S.ITER_MAX == N.CSS_ITER_MAX


class _CssOracleEngine(_ArimaOracleEngine):
    """ForecastEngine stand-in of tests/test_arima_oracle.py, answering fit_forecast_arma(..., estimator=) with the
    oracles"""

    def __init__(self):
        super().__init__()
        self.arma_calls = []

    def fit_forecast_arma(self, y, p, q, d, ps, npred, estimator="hr"):
        assert d == 0 or (self.max_diff is not None and d <= self.max_diff)
        self.arma_calls.append((p, q, d, estimator))
        f = S.fit_forecast_arma_css_packed if estimator == "css" else A.fit_forecast_arma_packed
        return {"pred": f(np.asarray(y), self.X, self.t_fit, ps, npred, p, q, d)["pred"].astype(np.float32)}


@pytest.mark.parametrize("diff", [None, 1, 2])
def test_forecast_groups_with_the_oracle_engine(diff):
    """one call per calendar bucket with estimator='css'; each group's rows are the CSS oracle's on its calendar"""
    import mmf
    from test_arima_oracle import _frame
    pdf = _frame()
    eng = _CssOracleEngine()
    out = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=eng, ar=1, diff=diff, ma=1,
                              estimator="css")
    assert eng.arma_calls == [(1, 1, diff or 0, "css")] * 2 and eng.arima_calls == 0 and eng.plain_calls == 0
    plain = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=_CssOracleEngine())
    assert list(out.columns) == list(plain.columns) and (out.dtypes == plain.dtypes).all()
    n_diff = 0
    for (prod, sku), g in out.groupby(["Product", "SKU"], sort=True):
        src = pdf[(pdf["Product"] == prod) & (pdf["SKU"] == sku)].sort_values("Date")
        y = src["Demand"].to_numpy(dtype=np.float32)[None, :]
        t_len, t_fit = y.shape[1], y.shape[1] - 14
        X = O.design_matrix(O.calendar_grid(np.datetime64(src["Date"].min(), "D"), t_len, "D"), t_fit)
        want = S.fit_forecast_arma_css_packed(y, X, t_fit, 0, t_len, 1, 1, diff or 0)
        got = g["Demand_Fitted"].to_numpy(dtype=np.float32)
        assert np.array_equal(got, want["pred"][0].astype(np.float32), equal_nan=True), (prod, sku)
        n_diff += bool(want["refined"][0])
    assert n_diff >= 1                      # some group's forecast is not the HR one
    hr_eng = _CssOracleEngine()
    hr = mmf.forecast_groups(pdf, freq="D", horizon=14, mode="holdout", engine=hr_eng, ar=1, diff=diff, ma=1,
                             estimator="hr")
    assert hr_eng.arma_calls == [(1, 1, diff or 0, "hr")] * 2
    tbl = mmf.forecast_table(pdf, freq="D", horizon=14, mode="holdout", engine=_CssOracleEngine(), ar=1, diff=diff,
                             ma=1, estimator="css")
    assert np.array_equal(tbl.column("Demand_Fitted").to_numpy(zero_copy_only=False).astype(np.float32),
                          out["Demand_Fitted"].to_numpy(dtype=np.float32), equal_nan=True)
    assert not np.array_equal(hr["Demand_Fitted"].to_numpy(dtype=np.float32),
                              out["Demand_Fitted"].to_numpy(dtype=np.float32), equal_nan=True)


def test_estimator_argument_checks():
    import mmf
    pdf = mmf.synth.reference_weekly_demand(2)
    for fg in (mmf.frames.forecast_groups, mmf.frames.forecast_table):
        for kw, msg in ((dict(ar=1, estimator="css"), "estimator= needs one MA order"),
                        (dict(ar=1, diff=1, estimator="css"), "estimator= needs one MA order"),
                        (dict(ar=(0, 1), ma=(0, 1), estimator="css"), "not offered with candidate MA orders"),
                        (dict(ar=(0, 1), diff=(0, 1), ma=(0, 1), estimator="hr"), "not offered with candidate MA"),
                        (dict(select=(1, 3), ar=1, ma=1, estimator="css"), "not offered with select= or interval="),
                        (dict(interval=0.9, ar=1, ma=1, estimator="css"), "not offered with select= or interval="),
                        (dict(ar=1, ma=1, estimator="mle"), "estimator must be 'hr' or 'css'")):
            with pytest.raises(ValueError, match=msg):
                fg(pdf, freq="W-MON", horizon=40, mode="holdout", engine=object(), **kw)
