"""CPU: the float64 oracle of ARIMA(p, d, q) errors by exact Gaussian likelihood (tests/arma_ml_oracle.py, DESIGN.md
section 2 item 19) against independent restatements: a dense Gaussian log-likelihood from psi-weight autocovariances,
central differences of L and of the scaled innovations, SciPy's optimisers and a statistical gate near the MA unit
circle; the two negative-control rules; the engine's and the frame layer's argument checks."""
import numpy as np
import pytest
from scipy.signal import lfilter

import arma_ml_oracle as ML
import arma_css_oracle as S
from test_arma_css_oracle import _random_poly

ORDERS = [(0, 1), (1, 1), (2, 1), (0, 4), (2, 2), (3, 4), (4, 4), (5, 3), (8, 1), (8, 4)]
OPT_TOL = 2e-6          # (L_shipped - L_scipy) / n_obs; worst measured 6.6e-7 over the cases below


def _series(rng, p, q, T, x=None):
    if x is None:
        x = np.r_[_random_poly(rng, p), -_random_poly(rng, q)]
    e = lfilter(np.r_[1.0, x[p:]], np.r_[1.0, -x[:p]], rng.normal(size=T + 400))[400:]
    return np.asarray(x, dtype=np.float64), e


def _gaps(rng, T, frac):
    obs = np.ones(T, dtype=bool)
    if frac:
        obs[rng.choice(T, size=max(1, int(frac * T)), replace=False)] = False
    return obs


@pytest.mark.parametrize("p,q", ORDERS)
@pytest.mark.parametrize("frac", [0.0, 0.16])
def test_filter_loglik_is_the_dense_gaussian_loglik(p, q, frac):
    rng = np.random.default_rng(100 * p + 10 * q + int(frac * 100))
    T = 60
    x, e = _series(rng, p, q, T)
    obs = _gaps(rng, T, frac)
    ev = ML.ml_eval(e, obs, T, p, q, x)
    want = ML.dense_loglik(e, obs, T, p, q, x, n_psi=20000)
    assert abs(ev["loglik"] - want) <= 1e-10 * abs(want), (ev["loglik"], want)


@pytest.mark.parametrize("frac", [0.0, 0.1])
def test_near_the_stationarity_bound(frac):
    rng = np.random.default_rng(7)
    T = 80
    for x, p, q in (([0.995, 0.3], 1, 1), ([1.6, -0.7, 0.4], 2, 1)):
        x, e = _series(rng, p, q, T, np.array(x))
        obs = _gaps(rng, T, frac)
        ev = ML.ml_eval(e, obs, T, p, q, x)
        want = ML.dense_loglik(e, obs, T, p, q, x, n_psi=200000)
        assert abs(ev["loglik"] - want) <= 1e-10 * abs(want), (x, ev["loglik"], want)


@pytest.mark.parametrize("p,q", [(0, 1), (1, 1), (2, 2), (4, 4), (8, 4)])
def test_gradient_and_gauss_newton_matrix_match_central_differences(p, q):
    """dL/dx = 2 n g / S_w and J'J = G^2 H, J the central differences of the scaled innovations r (rank-2 term in H)"""
    rng = np.random.default_rng(p * 10 + q)
    T = 70
    x, e = _series(rng, p, q, T)
    obs = _gaps(rng, T, 0.1)
    ev = ML.ml_eval(e, obs, T, p, q, x)
    h = 1e-6
    k = p + q
    gL = np.zeros(k)
    J = np.zeros((len(ev["r"]), k))
    for j in range(k):
        a = ML.ml_eval(e, obs, T, p, q, x + h * np.eye(k)[j])
        b = ML.ml_eval(e, obs, T, p, q, x - h * np.eye(k)[j])
        gL[j] = (a["L"] - b["L"]) / (2 * h)
        J[:, j] = (a["r"] - b["r"]) / (2 * h)
    g = 2 * ev["n"] * ev["g"] / ev["S_w"]
    assert np.abs(gL - g).max() <= 1e-5 * np.abs(g).max()
    G2 = ev["obj"] / ev["S_w"]
    assert np.abs(J.T @ J - G2 * ev["H"]).max() <= 1e-5 * np.abs(G2 * ev["H"]).max()
    assert np.allclose(ev["Jr"], J, rtol=0, atol=1e-5 * np.abs(J).max())


def test_the_lm_path_never_raises_L_and_ends_near_scipys_optimum():
    rng = np.random.default_rng(21)
    worst = 0.0
    for p, q in ((0, 1), (1, 1), (2, 2), (1, 3)):
        for frac in (0.0, 0.1):
            T = 115
            x, e = _series(rng, p, q, T)
            obs = _gaps(rng, T, frac)
            r = ML.lm(e, obs, T, p, q, (0.8 * x).astype(np.float32), max_iter=64)
            assert r["ok"] and r["n_acc"] >= 1
            assert all(b <= a for a, b in zip(r["path"], r["path"][1:])), r["path"]
            assert r["loglik"] >= r["loglik0"]
            Lopt, _ = ML.optimum(e, obs, T, p, q, r["x"])
            gap = (r["L"] - Lopt) / obs.sum()
            worst = max(worst, gap)
            assert gap <= OPT_TOL, (p, q, frac, r["L"], Lopt)


def test_ml_beats_css_near_the_ma_unit_circle():
    """MA(1), theta = -0.95, T = 115 (the weekly shape's rows at d = 2), 60 series, CSS from -0.5 then ML from the CSS
    point: theta RMSE of ML <= 0.6 x CSS's (measured 0.033 against 0.074, 0.44x, with this seed)"""
    rng = np.random.default_rng(2026)
    T, th = 115, -0.95
    ec, em = [], []
    for _ in range(60):
        e = lfilter([1.0, th], [1.0], rng.normal(size=T + 1))[1:]
        obs = np.ones(T, dtype=bool)
        c = S.lm(e, obs, T, 0, 1, np.array([-0.5], dtype=np.float32), max_iter=64)
        m = ML.lm(e, obs, T, 0, 1, c["x"], max_iter=64)
        ec.append(float(c["x"][0]) - th)
        em.append(float(m["x"][0]) - th)
    rc, rm = np.sqrt(np.mean(np.square(ec))), np.sqrt(np.mean(np.square(em)))
    assert rm <= 0.6 * rc, (rm, rc)


def test_negative_control_rules_fail_the_dense_check():
    rng = np.random.default_rng(5)
    T = 60
    x, e = _series(rng, 1, 1, T, np.array([0.6, 0.4]))
    obs = _gaps(rng, T, 0.16)
    want = ML.dense_loglik(e, obs, T, 1, 1, x, n_psi=20000)
    assert abs(ML.ml_eval(e, obs, T, 1, 1, x, no_logdet=True)["loglik"] - want) > 1e-3 * abs(want)
    assert abs(ML.ml_eval(e, obs, T, 1, 1, x, gap_as_zero=True)["loglik"] - want) > 1e-3 * abs(want)
    full = np.ones(T, dtype=bool)
    want_full = ML.dense_loglik(e, full, T, 1, 1, x, n_psi=20000)
    assert abs(ML.ml_eval(e, full, T, 1, 1, x, gap_as_zero=True)["loglik"] - want_full) <= 1e-10 * abs(want_full)
    # without the log-determinant the objective still falls along its own path
    r = ML.lm(e, obs, T, 1, 1, np.array([0.3, 0.1], dtype=np.float32), no_logdet=True)
    assert r["ok"] and all(b <= a for a, b in zip(r["path"], r["path"][1:]))


def test_p0_solve_refuses_a_unit_root():
    assert ML.p0_solve(np.array([1.0, 0.3]), 1, 1) is None
    assert ML.p0_solve(np.array([0.5, 0.3]), 1, 1) is not None


def test_engine_and_frame_argument_checks():
    import mmf
    eng = mmf.ForecastEngine.__new__(mmf.ForecastEngine)
    for kw, msg in ((dict(estimator="mle"), r"estimator must be 'hr' or 'css' \(or 'ml' for the exact likelihood\)"),
                    (dict(estimator="ml", joint_beta=True), "joint_beta=True needs estimator='css'"),
                    (dict(estimator="hr", max_iter=3), "max_iter= is the pass budget")):
        with pytest.raises(ValueError, match=msg):
            eng.fit_forecast_arma(None, 1, 1, **kw)
    pdf = mmf.synth.reference_weekly_demand(2)
    for fg in (mmf.frames.forecast_groups, mmf.frames.forecast_table):
        for kw, msg in ((dict(ar=1, estimator="ml"), "estimator= needs one MA order"),
                        (dict(ar=(0, 1), ma=(0, 1), estimator="ml"), "not offered with candidate MA orders"),
                        (dict(select=(1, 3), ar=1, ma=1, estimator="ml"), "not offered with select= or interval="),
                        (dict(ar=1, ma=1, estimator="ml", joint_beta=True), "joint_beta=True needs estimator='css'"),
                        (dict(ar=(0, 1), diff=(0, 1), ma=(0, 1), refit="css", estimator="ml"),
                         "is not offered with"),
                        (dict(ar=1, ma=1, estimator="mle"), "estimator must be 'hr' or 'css'")):
            with pytest.raises(ValueError, match=msg):
                fg(pdf, freq="W-MON", horizon=40, mode="holdout", engine=object(), **kw)
