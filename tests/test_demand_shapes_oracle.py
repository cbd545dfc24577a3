"""CPU: the demand-shape generator (tests/demand_shapes.py) produces what it claims, the float64 oracles give the closed
forms on its degenerate rows, and ar_oracle's degenerate-row rule and degenerate_bound hold."""
import numpy as np
import pytest

from ar_oracle import AR_MAX, autocov, degenerate_bound, degenerate_rows, fit_forecast_ar_packed, impulse, levinson
from arima_oracle import fit_forecast_arima_packed
from conftest import tolerance
from demand_shapes import CALENDARS, EXACT_FIT, KINDS, LEVELS, calendar, demand_batch, kind_rows, landmarks


@pytest.mark.parametrize("cal", sorted(CALENDARS))
def test_generator_shapes(cal):
    y, kinds, level = demand_batch(400, cal, seed=1)
    t = CALENDARS[cal][0]
    assert y.dtype == np.float32 and y.shape[1] == t
    a, b = demand_batch(40, cal, seed=1)[0], demand_batch(40, cal, seed=1)[0]
    assert np.array_equal(a, b, equal_nan=True)                               # seeded
    for kind in ("counts", "counts_sparse"):
        c = y[kind_rows(kinds, (kind,))]
        zf = (c == 0).mean(axis=1)
        assert ((zf >= 0.6) & (zf <= 0.98)).all(), (kind, zf)
        assert (c == np.round(c)).all() and (c >= 0).all()
    st = y[kind_rows(kinds, ("stockout",))]
    nan = y[kind_rows(kinds, ("stockout_nan",))]
    min_run = 7 if CALENDARS[cal][1] == "D" else 2
    for row, hole in ((r, r == 0) for r in st):
        runs = np.diff(np.flatnonzero(np.diff(np.r_[0, hole.astype(int), 0])))[::2]
        assert runs.size and runs.max() >= min_run and runs.max() <= 3 * 60
    assert np.isnan(nan).any(axis=1).all() and not np.isnan(st).any()
    assert np.array_equal(np.isnan(nan), st == 0) and np.array_equal(nan[~np.isnan(nan)], st[st != 0])   # same rows
    covid, xmas = landmarks(cal, t)
    first = np.array([np.argmax(np.isfinite(r)) for r in y])
    last = np.array([t - 1 - np.argmax(np.isfinite(r[::-1])) for r in y])
    early, late = kind_rows(kinds, ("launch_early",)), kind_rows(kinds, ("launch_late",))
    assert (first[early] >= 9).all() and (first[early] <= t // 2).all()
    assert (first[late] > t // 2).all() and (first[late] <= t - 40).all()
    if covid > 40:
        assert (last[kind_rows(kinds, ("discontinued",))] < covid).all()
    assert (first[kind_rows(kinds, ("launch_after_xmas",))] >= min(xmas, t - 40)).all()
    assert (y[kind_rows(kinds, ("returns", "signed"))] < 0).any(axis=1).all()
    sg = y[kind_rows(kinds, ("signed",))].astype(np.float64)
    assert (np.abs(sg.mean(axis=1)) < 0.3 * np.abs(sg).mean(axis=1)).all()
    pr = kind_rows(kinds, ("promo_origin",))
    assert (y[pr, t - 1] >= 20 * level[pr] * 0.5).all()
    assert not y[kind_rows(kinds, ("zeros",))].any()
    assert (y[kind_rows(kinds, ("const65534",))] == 65534).all()
    for i in np.flatnonzero(kind_rows(kinds, ("line", "walk"))):
        assert len(set(np.diff(y[i].astype(np.float64)))) == 1 and (y[i] == np.round(y[i])).all()
    # every 128-row tile mixes levels over at least five decades
    assert len(y) >= 3 * 128
    for lo in range(0, len(y) - 127, 128):
        lv = level[lo:lo + 128]
        assert lv.max() / lv.min() >= 1e5


def _degenerate_case(kind, cal="daily365", h=28):
    start, t, freq, X = calendar(cal, h)
    y, kinds, _ = demand_batch(len(KINDS), cal, seed=3)
    i = kinds.index(kind)
    return y[i:i + 1], X, t, h


def test_all_zero_rows_have_closed_forms():
    y, X, t, h = _degenerate_case("zeros")
    res = fit_forecast_ar_packed(y, X, t, t, h, 8)
    assert (res["r"] == 0).all() and res["order"][0] == 0 and not res["phi"].any()
    assert (res["pred"] == 0).all() and res["sigma"][0] == 0


def test_exact_line_is_continued():
    y, X, t, h = _degenerate_case("line")
    res = fit_forecast_ar_packed(y, X, t, t, h, 2)
    s = np.arange(t, t + h)
    a, b = float(y[0, 0]), float(y[0, 1] - y[0, 0])
    np.testing.assert_allclose(res["pred"][0], a + b * s, rtol=0, atol=1e-9 * (a + b * t))


@pytest.mark.parametrize("p", [0, 2])
def test_constant_step_walk_with_one_difference(p):
    y, X, t, h = _degenerate_case("walk")
    res = fit_forecast_arima_packed(y, X, t, t, h, p, 1)
    step = float(y[0, 1]) - float(y[0, 0])
    want = float(y[0, t - 1]) + step * np.arange(1, h + 1)
    np.testing.assert_allclose(res["pred"][0], want, rtol=0, atol=1e-9 * np.abs(want).max())


def test_degenerate_rule():
    """the exactly fit rows are degenerate, regular and intermittent rows are not, empty rows never"""
    start, t, freq, X = calendar("daily365", 28)
    y, kinds, level = demand_batch(3 * len(KINDS), "daily365", seed=4)
    y[0] = np.nan
    res = fit_forecast_ar_packed(y, X, t, t, 28, 2)
    tau = np.array([tolerance(r) for r in y])
    deg = degenerate_rows(res, tau)
    assert not deg[0]
    ex = kind_rows(kinds, EXACT_FIT)
    ex[0] = False
    assert deg[ex].all()
    # a level-0.1 series with 1 % noise is degenerate too: its noise is the absolute 1e-3 of the tolerance
    assert not deg[kind_rows(kinds, ("regular", "counts", "stockout", "returns", "promo")) & (level >= 1)].any()


def _perturbed_fit(res, delta, t_fit, ps, npred, p=AR_MAX):
    """the AR(p) fit and forecast that ar_oracle's model gives when the fitted values are off by delta [n, rows] (an
    error in the design's span, as an fp32 solve leaves): residuals e - delta, Levinson-Durbin, the recursion"""
    obs = res["obs"]
    n = len(obs)
    e = np.where(obs, res["e"] - delta[:, :t_fit], 0.0)
    phi = np.zeros((n, AR_MAX))
    for i in range(n):
        phi[i] = levinson(autocov(e[i], obs[i], t_fit, p), p)[0]
    end = ps + npred
    u = np.zeros((n, end + AR_MAX))
    ar = np.zeros((n, end))
    for s in range(end):
        ar[:, s] = (phi * u[:, s + AR_MAX - 1::-1][:, :AR_MAX]).sum(axis=1)
        keep = obs[:, s] if s < t_fit else np.zeros(n, dtype=bool)
        u[:, AR_MAX + s] = np.where(keep, e[:, s] if s < t_fit else 0.0, ar[:, s])
    return phi, (res["fitted"] + delta)[:, ps:end] + ar[:, ps:end]


@pytest.mark.parametrize("h", [28, 64])
def test_degenerate_bound_on_a_correlated_fit_error(h):
    """Exactly fit rows (daily 1,095) whose fitted values carry a smooth in-span error of tau / 3: Levinson-Durbin on
    those residuals gives order 8 with |phi|_1 > 1, the regime the GPU reaches on such rows.  The emulated forecast
    stays within degenerate_bound; the bound stays within 20 tau over the whole horizon (the signed impulse
    coefficients of a stable phi decay); and a forecast that amplifies tau over the horizon fails it."""
    start, t, freq, X = calendar("daily1095", h)
    y, kinds, _ = demand_batch(2 * len(KINDS), "daily1095", seed=6)
    rows = np.flatnonzero(kind_rows(kinds, ("line", "walk", "level_weekly", "const65534")))
    y = y[rows]
    n = len(y)
    tau = np.array([tolerance(r) for r in y])
    res = fit_forecast_ar_packed(y, X, t, t, h, AR_MAX)
    assert degenerate_rows(res, tau).all()
    rng = np.random.default_rng(7)
    shape = X @ rng.normal(0, 1, (X.shape[1], n))                    # [rows, n]: in the design's span
    delta = (tau / 3.0)[:, None] * (shape / np.abs(shape[:t]).max(axis=0)).T
    phi, pred = _perturbed_fit(res, delta, t, t, h)
    assert (np.abs(phi).sum(axis=1) > 1.0).any()
    tau_pred = np.maximum(tau, np.abs(delta[:, t:]).max(axis=1))
    b = degenerate_bound(res, phi, tau, tau_pred, t, t, h)
    assert (np.abs(pred - res["pred"]) <= b).all()
    assert (b / tau[:, None]).max() <= 20.0, float((b / tau[:, None]).max())     # 7.6-11.3 measured
    planted = res["pred"] + tau[:, None] * 1.2 ** np.arange(1, h + 1)  # tau amplified to ~160 tau at step 28
    assert (np.abs(planted - res["pred"]) > b).any(axis=1).all()


def test_impulse_coefficients_reproduce_the_recursion():
    rng = np.random.default_rng(8)
    phi = np.zeros((3, AR_MAX))
    phi[0, :2] = (0.5, 0.3)
    phi[1] = rng.uniform(-0.2, 0.2, AR_MAX)
    phi[2, 0] = 0.999
    c = impulse(phi, 40)
    state = rng.normal(size=(3, AR_MAX))                             # u_{a-1} .. u_{a-8}
    u = np.concatenate([state[:, ::-1], np.zeros((3, 40))], axis=1)
    for h in range(40):
        u[:, AR_MAX + h] = (phi * u[:, AR_MAX + h - 1::-1][:, :AR_MAX]).sum(axis=1)
        np.testing.assert_allclose(u[:, AR_MAX + h], (c[:, h] * state).sum(axis=1), rtol=1e-12, atol=1e-12)
