"""CPU: the float64 composition of tests/arma_select_css_oracle.py (DESIGN.md section 2 item 18): the selection's
choice kept, the CSS / joint refit of each q >= 1 winner from its Hannan-Rissanen start never raising S, the q = 0
winners untouched; the dummy coefficients of the joint refit against the selection's OLS ones on weekly ARIMA(1, 1, 1)
rows; and the refit= argument of the frame layer."""
import numpy as np
import pytest

import arma_oracle as A
from arma_joint_oracle import plan_of
from arma_select_css_oracle import select_arma_refit_packed
from arma_select_oracle import select_arma_packed
from oracle import mmf_oracle as O
from test_arma_css_oracle import _CssOracleEngine, _arma_series
from test_arma_joint_oracle import BETA_TRUE, DUMMY_ROWS

T_FIT, N_HOLD = 117, 40                        # the reference's weekly 157 / 117 / 40
GRID = ((0, 1), (0, 1), (0, 1))


def weekly_arima_rows(n, phi, theta, seed, sd=1.0):
    """n weekly series of T_FIT + N_HOLD rows: intercept + trend + two one-week dummies with BETA_TRUE, ARIMA(1, 1, 1)
    errors (the ARMA(phi, theta) series summed once) -> (y [n, 157] float32, X [157, 16])"""
    rows = T_FIT + N_HOLD
    X = np.zeros((rows, 16))
    X[:, 0] = 1.0
    X[:, 1] = np.arange(rows) / T_FIT
    X[DUMMY_ROWS[0], 2] = 1.0
    X[DUMMY_ROWS[1], 3] = 1.0
    y = np.empty((n, rows))
    for i in range(n):
        e, _ = _arma_series(rows, phi, theta, seed=seed * 100003 + i, sd=sd)
        y[i] = X[:, :4] @ BETA_TRUE + np.cumsum(e)
    return y.astype(np.float32), X


@pytest.mark.parametrize("joint", [False, True])
def test_composition(joint):
    """choice, mse and cand_mse are the selection's; the q >= 1 winners carry their class's fixed-order refit, with
    S(shipped) <= S(HR start); every other row keeps the selection's outputs with NaN, NaN, 0, 0"""
    y, X = weekly_arima_rows(24, [0.6], [0.4], seed=3)
    y[5] = np.nan                                          # no eligible candidate
    y[7, 20:30] = np.nan
    sel = select_arma_packed(y, X, T_FIT, N_HOLD, *GRID, 0, X.shape[0])
    got = select_arma_refit_packed(y, X, T_FIT, N_HOLD, *GRID, 0, X.shape[0], joint=joint)
    for k in ("choice_p", "choice_d", "choice_q", "mse", "cand_mse"):
        assert np.array_equal(got[k], sel[k], equal_nan=True), k
    refit = got["refit"]
    assert refit.sum() >= 3 and (~refit).sum() >= 2
    assert (got["css"][refit] <= got["css_start"][refit]).all()
    assert (got["css_stop"][refit] >= 1).all() and (got["iters"][refit] >= 1).all()
    for k in ("pred", "phi", "theta", "order", "ma_order", "sigma", "status"):
        assert np.array_equal(np.asarray(got[k])[~refit], np.asarray(sel[k])[~refit], equal_nan=True), k
    assert np.isnan(got["css"][~refit]).all() and (got["css_stop"][~refit] == 0).all()
    for (p, d, q), r in got["fixed"].items():
        s = refit & (got["choice_p"] == p) & (got["choice_d"] == d) & (got["choice_q"] == q)
        assert np.array_equal(got["pred"][s], r["pred"][s], equal_nan=True)
    if joint:
        assert np.isnan(got["beta"][5]).all()
        q0 = ~refit & (got["choice_p"] >= 0)
        for d in set(got["choice_d"][q0].tolist()):
            _, _, W, _, _, g0 = plan_of(y, X, T_FIT, d)
            s = q0 & (got["choice_d"] == d)
            assert np.array_equal(got["beta"][s], (g0 @ W.T)[s])


def test_dummy_beta_rmse_of_the_joint_refit_beats_the_selections_ols():
    """120 weekly series with ARIMA(1, 1, 1) errors (0.6, 0.4), selected on (0, 1) x (0, 1) x (0, 1): over the rows whose
    winner is refit, the dummies' beta RMSE of the joint refit <= 0.2 x that of the selection's OLS beta (the plain
    fit the winner builds on; measured 0.081 and 0.074 over 33 rows)"""
    y, X = weekly_arima_rows(120, [0.6], [0.4], seed=7)
    got = select_arma_refit_packed(y, X, T_FIT, N_HOLD, *GRID, T_FIT, N_HOLD, max_iter=64, joint=True)
    refit = got["refit"]
    print(f"refit rows: {int(refit.sum())}")
    assert refit.sum() >= 15
    ols = np.full((len(y), 16), np.nan)
    for d in (0, 1):
        _, _, W, _, _, g0 = plan_of(y, X, T_FIT, d)
        s = got["choice_d"] == d
        ols[s] = (g0 @ W.T)[s]
    ratios = []
    for k in (2, 3):
        rj = np.sqrt(np.mean((got["beta"][refit, k] - BETA_TRUE[k]) ** 2))
        ro = np.sqrt(np.mean((ols[refit, k] - BETA_TRUE[k]) ** 2))
        ratios.append(rj / ro)
    print(f"dummy beta RMSE joint refit / selection OLS: {ratios[0]:.3f} {ratios[1]:.3f} over {int(refit.sum())} rows")
    assert max(ratios) <= 0.2, ratios


class _SelectRecorder(_CssOracleEngine):
    """ForecastEngine stand-in of tests/test_arma_css_oracle.py that records fit_select_arma's refit arguments and
    answers with the selection oracle"""

    def __init__(self):
        super().__init__()
        self.calls = []

    def fit_select_arma(self, y, n_hold, orders, diffs, mas, ps, npred, refit=None, joint_beta=False):
        self.calls.append((refit, joint_beta))
        res = select_arma_packed(np.asarray(y), self.X, self.t_fit, n_hold, orders, diffs, mas, ps, npred)
        return {"pred": res["pred"].astype(np.float32)}


def test_frame_refit_argument_and_refusals():
    import mmf
    from test_arima_oracle import _frame
    pdf = _frame()
    eng = _SelectRecorder()
    kw = dict(freq="D", horizon=14, mode="holdout", engine=eng, ar=(0, 1), diff=(0, 1), ma=(0, 1))
    mmf.forecast_groups(pdf, refit="css", **kw)
    mmf.forecast_groups(pdf, refit="css", joint_beta=True, **kw)
    mmf.forecast_groups(pdf, **kw)
    n_buckets = len(eng.calls) // 3
    assert eng.calls == [("css", False)] * n_buckets + [("css", True)] * n_buckets + [(None, False)] * n_buckets
    for fg in (mmf.frames.forecast_groups, mmf.frames.forecast_table):
        for extra, msg in ((dict(ar=1, ma=1, refit="css"), "refit= needs candidate MA orders"),
                           (dict(ar=1, ma=1, estimator="css", refit="css"), "refit= is not offered with estimator="),
                           (dict(ar=(0, 1), ma=(0, 1), estimator="css", refit="css"),
                            "estimator= is not offered with candidate MA orders"),
                           (dict(ar=(0, 1), ma=(0, 1), refit="mle"), "refit must be None or 'css'"),
                           (dict(ar=(0, 1), ma=(0, 1), refit="css", select=(1, 3)), "is not offered with select="),
                           (dict(refit="css", interval=0.9), "is not offered with select= or interval="),
                           (dict(ar=(0, 1), ma=(0, 1), joint_beta=True), "joint_beta=True needs estimator='css'"),
                           (dict(ar=1, ma=1), None)):
            if msg is None:
                continue
            with pytest.raises(ValueError, match=msg):
                fg(pdf, freq="D", horizon=14, mode="holdout", engine=object(), **extra)
