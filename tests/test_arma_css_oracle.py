"""CPU: the float64 CSS oracle of tests/arma_css_oracle.py (DESIGN.md section 2 item 16): its Jacobian against central
finite differences (gap-free, isolated gaps, gaps longer than q, a gap before row p), the two-filter form before the first
gap, a non-increasing objective along the LM path, optimality against SciPy, the theta RMSE against Hannan-Rissanen on
simulated MA(1) rows, the negative control's failure on gappy rows, the header constants and the frame layer's
estimator= argument; the vectorised replay against the scalar LM and its decision margins on constructed rows."""
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


def _replay_rows(p, q, n, T, seed, gaps=0.0):
    """n simulated ARMA(p, q) rows with random stationary, invertible parameters and their HR starts -> (E, OBS, X0) of
    the rows whose HR estimate passed the gate"""
    rng = np.random.default_rng(seed)
    E, OBS, X0 = [], [], []
    for i in range(n):
        ph = _random_poly(rng, p)
        th = -_random_poly(rng, q)
        e, obs = _arma_series(T, ph, th, seed * 1000 + i, gaps=gaps)
        x0, _ = _hr_start(e, obs, T, p, q)
        if x0 is not None:
            E.append(e), OBS.append(obs), X0.append(x0)
    return np.array(E), np.array(OBS), np.array(X0, dtype=np.float32)


def _random_poly(rng, k, rmax=0.85):
    """a_1..a_k of 1 - sum a_j z^j from random reflection coefficients in (-rmax, rmax): stationary (invertible)"""
    a = np.zeros(0)
    for j in range(k):
        kap = rng.uniform(-rmax, rmax)
        a = np.r_[a - kap * a[::-1], kap]
    return a


REPLAY_CASES = [(1, 1, 0.0), (0, 2, 0.05), (2, 1, 0.02), (3, 4, 0.0), (4, 2, 0.1), (8, 4, 0.0)]


def test_vectorised_replay_equals_the_scalar_lm():
    """lm_replay, all rows of a case in lockstep, against lm row by row on every decided row: stop code, pass count,
    acceptance sequence and x bit-equal, S within 1e-12; max_iter 64 so that every stop code can occur.  At least 30
    rows are compared, and every case compares some"""
    n_cmp = 0
    for p, q, gaps in REPLAY_CASES:
        E, OBS, X0 = _replay_rows(p, q, 12, 160, seed=31 + p * 5 + q, gaps=gaps)
        assert len(E) >= 4, (p, q)
        r = S.lm_replay(E, OBS, 160, p, q, X0, max_iter=64)
        case = 0
        for i in np.flatnonzero(~r["ambiguous"]):
            w = S.lm(E[i], OBS[i], 160, p, q, X0[i], 64)
            what = (p, q, int(i))
            assert r["stop"][i] == w["stop"] and r["iters"][i] == w["iters"] and r["n_acc"][i] == w["n_acc"], what
            assert list(r["acc"][i, :w["iters"] - 1]) == w["acc"], what
            assert r["x"][i].tobytes() == np.asarray(w["x"], dtype=np.float32).tobytes(), what
            assert abs(r["S"][i] - w["S"]) <= 1e-12 * w["S"] and abs(r["S0"][i] - w["S0"]) <= 1e-12 * w["S0"], what
            assert r["n_C"][i] == (OBS[i, p:160]).sum(), what
            case += 1
        assert case >= 1, (p, q)
        n_cmp += case
    assert n_cmp >= 30, n_cmp


def test_replay_classifies_a_row_the_same_alone_and_in_a_batch():
    """margins depend on the row's own path only: every row replayed alone gets the batch's margins and outputs"""
    E, OBS, X0 = _replay_rows(3, 4, 8, 160, seed=31 + 15 + 4)
    r = S.lm_replay(E, OBS, 160, 3, 4, X0, max_iter=64)
    for i in range(len(E)):
        a = S.lm_replay(E[i:i + 1], OBS[i:i + 1], 160, 3, 4, X0[i:i + 1], max_iter=64)
        assert a["ambiguous"][0] == r["ambiguous"][i] and a["x"][0].tobytes() == r["x"][i].tobytes(), i
        for m in S.MARGINS:
            assert a["margin"][m][0] == pytest.approx(r["margin"][m][i], rel=1e-9), (i, m)


def test_replay_margins_on_constructed_rows():
    """a convergence threshold placed exactly at a pass's realised gain makes the row ambiguous, and only through the
    conv margin; a value exactly at an fp32 rounding midpoint has margin 0; a trial point equal to the accepted one
    is never ambiguous"""
    E, OBS, X0 = _replay_rows(1, 1, 6, 200, seed=5)
    r = S.lm_replay(E, OBS, 200, 1, 1, X0, max_iter=64)
    assert not r["ambiguous"].any()
    i = int(np.flatnonzero(r["n_acc"] >= 2)[0])
    w = S.lm(E[i], OBS[i], 200, 1, 1, X0[i], 64)
    k = w["acc"].index(True) + 1                      # the first accepted pass after the first one
    gain = (w["path"][k - 1] - w["path"][k]) / w["path"][k - 1]
    at = S.lm_replay(E[i:i + 1], OBS[i:i + 1], 200, 1, 1, X0[i:i + 1], max_iter=64, rtol=gain)
    assert at["ambiguous"][0] and at["margin"]["conv"][0] < 1.0
    assert all(at["margin"][m][0] >= 1.0 for m in S.MARGINS if m != "conv")
    # just above and below the threshold, by far more than the noise: decided, and the stop follows
    hi = S.lm_replay(E[i:i + 1], OBS[i:i + 1], 200, 1, 1, X0[i:i + 1], max_iter=64, rtol=gain * (1 + 1e-6))
    assert not hi["ambiguous"][0] and hi["stop"][0] == 1 and hi["iters"][0] == k + 1
    f = np.float32(1.5)
    mid = 0.5 * (float(f) + float(np.nextafter(f, np.float32(2))))
    assert S.rounding_margin(np.array([mid]), 1e-20)[0] == 0.0
    assert S.rounding_margin(np.array([mid + 1e-12]), 1e-12)[0] == pytest.approx(1.0, rel=1e-3)
    assert S.rounding_margin(np.array([1.5]), 0.0)[0] == np.inf
    # started at its own answer with no convergence rule, the row runs until lam passes LAMBDA_MAX or the budget ends;
    # its trial points round back to x or lower S by less than the noise, and each such pass is marked: a trial point
    # equal to x bit for bit is decided (S is then the same on both sides), any other is held to the accept margin
    one = S.lm_replay(E[i:i + 1], OBS[i:i + 1], 200, 1, 1, r["x"][i:i + 1], max_iter=64, rtol=0.0)
    assert one["stop"][0] in (2, 3)
    assert bool(one["ambiguous"][0]) == any(one["margin"][m][0] < 1.0 for m in S.MARGINS)


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
