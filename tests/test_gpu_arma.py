"""GPU (-m gpu): regression with ARIMA(p, d, q) errors by Hannan-Rissanen (mmf_fit_forecast_arma_f32, DESIGN.md section 2
item 13).

Two yardsticks:
  - existing code: a row that fails the gate is, bit for bit, mmf_fit_forecast_ar_f32(p) (d = 0, p >= 1), the plain
    regression of mmf_fit_select_ar_f32 with orders (0,) (d = 0, p = 0) or mmf_fit_forecast_arima_f32(p, d), with
    ma_order 0 and theta exactly 0;
  - the float64 oracle of tests/arma_oracle.py on the gated rows: gate decisions equal outside the rows near a threshold
    and the degenerate rows (counted), (phi, theta) within BETA_TOL, sigma and the part the ARMA terms add to the
    fallback's prediction within arma_oracle.pred_bound.
Every batch carries test_gpu_arima.py's row mix (gaps of every kind, empty rows, inf) plus MA(1) rows with theta = 0.9,
rows with 12 % isolated gaps and two degenerate rows (constant, exact line: r_0 = 0, so they fall back)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mmf
from ar_oracle import degenerate_rows
from arma_oracle import MA_MAX, coef_bound, fit_forecast_arma_packed, near_threshold, pred_bound
from arima_oracle import z_tau
from conftest import ROOT, forecast_leverage, record_err
from oracle import mmf_oracle as O
from test_gpu_abi_contract import PATTERN
from test_gpu_arima import _case, _dev, _np, _windows
from test_gpu_edges import _le, _same_bits

pytestmark = pytest.mark.gpu

# (phi, theta) of a gated row: |beta_gpu - beta_oracle|_2 <= DELTA max(COND0, cond(G)) (1 + |beta|_2).  Derivation: the GPU's
# residuals carry the fp32 error of its fitted values, a few 1e-6 of their scale (tests/conftest.py: "~10^3 accumulated
# terms leave a few 1e-6 relative"), so G and b of the normal equations move by a relative DELTA = 2e-6; to first order
# |dbeta| <= cond(G) DELTA (1 + |beta|).  eps^ reaches G through the long AR, whose Toeplitz system amplifies the same
# relative error by its own condition number, which the Gram's does not show: COND0 = 1e3 is the floor for it (the
# order-32 Toeplitz matrices of these rows stay below 1e3).  BETA_TOL = DELTA x COND0.
# The first-order bound arma_oracle.coef_bound is reported beside it in the error log; it carries the tolerance itself
# (1e-3 absolute plus 5e-6 of max|y|, not the fit's actual error) through a Cauchy-Schwarz step on the autocovariances,
# so with m up to 32 it is far above |beta| and cannot tell a wrong estimate from a right one.
DELTA = 2e-6
COND0 = 1e3
BETA_TOL = DELTA * COND0


def _arma_case(cal, n=170, seed=5):
    """test_gpu_arima's rows, with every 5th row an MA(1) theta = 0.9 error on the regression (levels not integrated),
    every 7th row with 12 % isolated gaps, and two degenerate rows (constant, exact line)"""
    y, X, t_fit, has_c = _case(cal, n, seed)
    rng = np.random.default_rng(seed + 100)
    t = t_fit
    eps = rng.normal(0, 4, (n, t + 1))
    ma = eps[:, 1:] + 0.9 * eps[:, :-1]
    base = 300.0 + rng.normal(0, 20, (n, X.shape[1])) @ X[:t].T
    for i in range(0, n, 5):
        y[i] = (base[i] + ma[i]).astype(np.float32)
    for i in range(3, n, 7):
        cols = rng.choice(np.arange(2, t - 1), size=int(0.12 * t), replace=False)
        y[i, cols] = np.nan
    y[1] = 42.0
    y[2] = (7.0 + 0.25 * np.arange(t)).astype(np.float32)
    return y, X, t_fit, has_c


def _cond_factor(want):
    """max(1, cond(G) / COND0) per row: the Gram's condition number amplifies a relative perturbation of the normal
    equations into beta (1 for rows without a regression)"""
    out = np.ones(len(want["status"]))
    for i, h in enumerate(want["hr"]):
        if h is not None and h.get("G") is not None and h["G"].size and want["gated"][i]:
            out[i] = max(1.0, float(np.linalg.cond(h["G"])) / COND0)
    return out


def _engines(X, t_fit, has_c):
    engs = {k: mmf.ForecastEngine(kernel=k) for k in ("auto", "tc", "warp")}
    for e in engs.values():
        e.plan(X, t_fit, has_c)
        e.plan_arima(X, t_fit, 2)
    return engs


def _fallback(eng, yd, p, d, ps, npred, t_fit):
    if d >= 1:
        return _np(eng.fit_forecast_arima(yd[:, :t_fit], p, d, ps, npred))
    if p >= 1:
        return _np(eng.fit_forecast_ar(yd[:, :t_fit], p, ps, npred))
    return _np(eng.fit_select_ar(yd, 1, (0,), ps, npred))


def _check(got, fb, want, y, X, t_fit, ps, npred, what):
    """fallback rows bit-equal to the single call; gated rows against the oracle.  Returns (worst ratio, near count)"""
    gated = got["ma_order"] > 0
    d = want["d"]
    zt = {"z": want["base"]["z"]} if d >= 1 else {"z": np.where(np.isfinite(y), y, np.nan)[:, :t_fit]}
    tau_fit = z_tau(zt)
    # rows the regression fits to rounding level (ar_oracle.degenerate_rows: RMS residual <= 4 tau) carry fp32 noise on
    # the GPU and float64 noise in the oracle, so their gate decisions are unrelated: counted with the near rows
    near = near_threshold(want) | degenerate_rows(want["zres"], tau_fit)
    agree = gated == want["gated"]
    assert (agree | near).all(), (what, np.flatnonzero(~agree & ~near)[:8])
    fbr = ~gated
    for k in ("pred", "phi", "order", "sigma", "status"):
        a, b = np.ascontiguousarray(got[k][fbr]), np.ascontiguousarray(fb[k][fbr])
        assert a.tobytes() == b.tobytes(), (what, k, np.flatnonzero(fbr)[:8])
    assert not got["theta"][fbr].any()
    assert np.array_equal(got["status"], fb["status"]), what
    rows = gated & want["gated"] & ~near
    if not rows.any():
        return 0.0, int(near.sum())
    p, q = want["p"], want["q"]
    assert (got["order"][rows] == p).all() and (got["ma_order"][rows] == q).all(), what
    bg = np.concatenate([got["phi"][:, :p], got["theta"][:, :q]], axis=1).astype(np.float64)
    bw = np.concatenate([want["phi"][:, :p], want["theta"][:, :q]], axis=1)
    db = np.linalg.norm(bg - bw, axis=1)
    lim = BETA_TOL * (1.0 + np.linalg.norm(bw, axis=1)) * _cond_factor(want)
    w_beta = float((db[rows] / lim[rows]).max())
    _le(w_beta, 1.0, f"{what}: |dbeta| / BETA_TOL")
    T = t_fit - d
    Dm = want["base"]["D"] if d >= 1 else X
    lev = forecast_leverage(Dm, T, 0, max(ps + npred - d, 1))
    tau_pred = z_tau(zt, lev)
    pb, sb = pred_bound(want, lim, tau_fit, tau_pred, ps, npred)
    # the part the ARMA terms add to the fallback's prediction, on both sides: it cancels the plain fit's own error (the
    # subject of the ARIMA(p, d, 0) tests), including rows where a design column the series never observes is non-zero
    wp = want["pred"][rows] - want["base"]["pred"][rows]
    gp = got["pred"][rows].astype(np.float64) - fb["pred"][rows].astype(np.float64)
    assert np.array_equal(np.isnan(wp), np.isnan(gp)), what
    fin = np.isfinite(wp)
    err = np.abs(np.where(fin, gp - wp, 0.0)) / np.where(fin, pb[rows], 1.0)
    w_pred = float(err.max())
    _le(w_pred, 1.0, f"{what}: prediction error / pred_bound")
    w_sig = float((np.abs(got["sigma"][rows] - want["sigma"][rows]) / sb[rows]).max())
    _le(w_sig, 1.0, f"{what}: |dsigma| / bound")
    cb = coef_bound(want, tau_fit)
    record_err("test_gpu_arma coef_bound", float((db[rows] / cb[rows]).max()), 1.0, what=what)
    return max(w_beta, w_pred, w_sig), int(near.sum())


@pytest.mark.parametrize("d", [0, 1, 2])
@pytest.mark.parametrize("p,q", [(0, 1), (1, 1), (2, 2), (8, 4)])
@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_arma_matches_existing_code_and_the_oracle(cal, p, q, d):
    """every window is a slice of the holdout window's rows, on the GPU bit for bit (no restart) and in the oracle"""
    y, X, t_fit, has_c = _arma_case(cal, n=60)
    engs = _engines(X, t_fit, has_c)
    yd = _dev(y, t_fit + 1)
    n_rows = X.shape[0]
    worst, near_n, gated_n = 0.0, 0, 0
    for m in (0, max(p, q), 32):
        want = fit_forecast_arma_packed(y, X, t_fit, 0, n_rows, p, q, d, m)
        for k, eng in engs.items():
            full = _np(eng.fit_forecast_arma(yd[:, :t_fit], p, q, d, 0, n_rows, long_order=m))
            fb = _fallback(eng, yd, p, d, 0, n_rows, t_fit)
            w, nn = _check(full, fb, want, y, X, t_fit, 0, n_rows, f"{cal} p={p} q={q} d={d} m={m} {k}")
            worst, near_n = max(worst, w), max(near_n, nn)
            gated_n = max(gated_n, int((full["ma_order"] > 0).sum()))
            g = full["ma_order"] > 0
            for name, (ps, npred) in _windows(t_fit, n_rows).items():
                got = _np(eng.fit_forecast_arma(yd[:, :t_fit], p, q, d, ps, npred, long_order=m))
                fbw = _fallback(eng, yd, p, d, ps, npred, t_fit)
                for key in got:
                    ref = full[key][:, ps:ps + npred] if key == "pred" else full[key]
                    if key == "pred":       # fallback rows restart as their single call does: that call is the yardstick
                        ref = np.where(g[:, None], ref, fbw["pred"])
                    assert np.ascontiguousarray(got[key]).tobytes() == np.ascontiguousarray(ref).tobytes(), \
                        (cal, p, q, d, m, name, k, key)
    for e in engs.values():
        e.close()
    assert gated_n > 0, (cal, p, q, d)
    record_err("test_arma_matches_existing_code_and_the_oracle", worst, 1.0, what=f"{cal} p={p} q={q} d={d}",
               near_threshold=near_n, gated=gated_n)


def test_y_at_and_beyond_t_fit_is_never_read_and_power_of_two_scaling():
    y, X, t_fit, _ = _arma_case("daily")
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, True)
    eng.plan_arima(X, t_fit, 2)
    base = _dev(y, t_fit + 40)
    for d in (0, 1, 2):
        ref = _np(eng.fit_forecast_arma(base[:, :t_fit], 1, 1, d, 0, X.shape[0]))
        assert (ref["ma_order"] > 0).any()
        for fill in (float("nan"), 1e30, -7.0):
            yd = _dev(y, t_fit + 40)
            yd[:, t_fit:] = fill
            got = _np(eng.fit_forecast_arma(yd, 1, 1, d, 0, X.shape[0]))
            for k in ref:
                assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(ref[k]).tobytes(), (fill, d, k)
        a = _np(eng.fit_forecast_arma(base[:, :t_fit], 2, 1, d, t_fit, 28))
        b = _np(eng.fit_forecast_arma(base[:, :t_fit] * 8.0, 2, 1, d, t_fit, 28))
        for k, f in (("pred", 8.0), ("phi", 1.0), ("theta", 1.0), ("order", 1), ("ma_order", 1), ("sigma", 8.0),
                     ("status", 1)):
            w = a[k] * f
            same = (b[k] == w) | (np.isnan(b[k]) & np.isnan(w))
            assert same.all(), (d, k)
    eng.close()


def test_slabs_are_bit_equal_to_per_slab_calls():
    n, t = (1 << 20) + 1001, 48
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=9, nan_frac=0.01)
    X = O.design_matrix(O.calendar_grid(start, t + 8, "D"), t)
    eng = mmf.ForecastEngine()
    eng.plan(X, t, True)
    eng.plan_arima(X, t, 2)
    yd = torch.from_numpy(y).cuda()
    for d in (0, 2):
        whole = eng.fit_forecast_arma(yd, 1, 1, d, t, 8)
        for lo, hi in ((0, 1 << 19), (1 << 19, n)):
            part = eng.fit_forecast_arma(yd[lo:hi], 1, 1, d, t, 8)
            for k in ("pred", "phi", "theta", "order", "ma_order", "sigma", "status"):
                assert _same_bits(whole[k][lo:hi], part[k]), (d, k)
    eng.close()


def test_nullable_outputs_wide_table_and_refusals():
    y, X, t_fit, _ = _arma_case("daily", n=40)
    n = len(y)
    eng = mmf.ForecastEngine()
    lib, h = eng._lib, eng._h
    yd = _dev(y)
    out = torch.full((n, 28), 7.0, device="cuda")
    nulls = (None,) * 7
    assert lib.mmf_fit_forecast_arma_f32(h, yd.data_ptr(), n, yd.stride(0), 1, 0, 1, 0, t_fit, 28, out.data_ptr(), 28,
                                         *nulls) == -4                        # MMF_E_NOPLAN (no design plan)
    eng.plan(X, t_fit, True)
    assert lib.mmf_fit_forecast_arma_f32(h, yd.data_ptr(), n, yd.stride(0), 1, 1, 1, 0, t_fit, 28, out.data_ptr(), 28,
                                         *nulls) == -4                        # no ARIMA plan for d = 1
    eng.plan_arima(X, t_fit, 1)
    for d in (0, 1):
        ref = eng.fit_forecast_arma(yd, 1, 1, d, t_fit, 28)
        wide = torch.full((n, 41), float(np.float32(PATTERN)), device="cuda")
        view = wide[:, 5:33]
        rc = lib.mmf_fit_forecast_arma_f32(h, yd.data_ptr(), n, yd.stride(0), 1, d, 1, 0, t_fit, 28, view.data_ptr(),
                                           41, *nulls)
        assert rc == 0
        torch.cuda.synchronize()
        assert _same_bits(view, ref["pred"])
        assert (wide[:, :5] == float(np.float32(PATTERN))).all() and (wide[:, 33:] == float(np.float32(PATTERN))).all()
    theta = torch.full((n, MA_MAX), 7.0, device="cuda")
    host_out = np.zeros((n, 28), dtype=np.float32)
    bad = [(1, 0, 0, 0), (1, 0, 5, 0), (9, 0, 1, 0), (-1, 0, 1, 0), (1, 3, 1, 0), (1, 2, 1, 0),  # max_diff is 1
           (2, 0, 1, 1), (1, 0, 1, 33), (1, 0, 1, -1)]
    for (p, d, q, m) in bad:
        rc = lib.mmf_fit_forecast_arma_f32(h, yd.data_ptr(), n, yd.stride(0), p, d, q, m, t_fit, 28, out.data_ptr(),
                                           28, None, theta.data_ptr(), None, None, None, None, None)
        assert rc != 0, (p, d, q, m)
    for args in ((-1, 28, out.data_ptr(), 28), (t_fit, 65, out.data_ptr(), 65), (t_fit, 28, out.data_ptr(), 27),
                 (t_fit, 28, None, 28), (t_fit, 28, host_out.ctypes.data, 28)):
        rc = lib.mmf_fit_forecast_arma_f32(h, yd.data_ptr(), n, yd.stride(0), 1, 0, 1, 0, *args, None,
                                           theta.data_ptr(), None, None, None, None, None)
        assert rc != 0, args
    torch.cuda.synchronize()
    assert (out == 7.0).all() and (theta == 7.0).all() and not host_out.any()
    eng.close()


def test_other_calls_unchanged_by_arma_calls_and_a_shared_context_matches_a_fresh_one():
    y, X, t_fit, has_c = _arma_case("daily")
    start = np.datetime64("2019-01-01", "D")
    eng = mmf.ForecastEngine()
    eng.plan_calendars([start, start + 30], [t_fit, t_fit - 30], "D", 28)
    eng.plan_backtest(start, t_fit, "D", 28, 3)
    eng.plan(X, t_fit, has_c)
    eng.plan_arima(X, t_fit, 2)
    yd = _dev(y, t_fit + 28)
    yf = yd[:, :t_fit]

    def calls():
        bt = eng.backtest(yf)
        return (eng.fit_forecast(yf, t_fit, 28).clone(), eng.fit_forecast(yf, 0, t_fit + 64).clone(),
                eng.fit_forecast_ar(yf, 2, t_fit, 28)["pred"].clone(), eng.fit_select_ar(yd, 28, (0, 1, 2))["pred"].clone(),
                eng.fit_forecast_arima(yf, 2, 1, t_fit, 28)["pred"].clone(),
                eng.fit_select_arima(yd, 28, (0, 1), (0, 1), t_fit, 28)["pred"].clone(),
                eng.fit_forecast_ragged(yf, [0, 70, len(y)]).clone(), bt["pred"].clone(), bt["metrics"].clone(),
                bt["status"].clone())

    args = ((1, 1, 0, t_fit, 28, 0), (8, 4, 2, 0, t_fit + 64, 32), (0, 2, 1, 50, 100, 2))
    before = calls()
    shared = [_np(eng.fit_forecast_arma(yf, p, q, d, ps, npred, long_order=m)) for p, q, d, ps, npred, m in args]
    after = calls()
    assert all(_same_bits(a, b) for a, b in zip(before, after))
    fresh = mmf.ForecastEngine()
    fresh.plan(X, t_fit, has_c)
    fresh.plan_arima(X, t_fit, 2)
    for (p, q, d, ps, npred, m), a in zip(args, shared):
        b = _np(fresh.fit_forecast_arma(yf, p, q, d, ps, npred, long_order=m))
        for k in a:
            assert np.ascontiguousarray(a[k]).tobytes() == np.ascontiguousarray(b[k]).tobytes(), (p, q, d, k)
    eng.close()
    fresh.close()


def test_long_hourly_series():
    """70,001 fit rows, a 400-row gap and isolated gaps, d = 0, 1, 2: the limits x sqrt(t_fit / 1095)"""
    t, h = 70001, 48
    s_ = np.arange(t + h, dtype=np.float64)
    X = np.column_stack([np.ones_like(s_), (s_ - t / 2) / t, np.sin(2 * np.pi * s_ / 24), np.cos(2 * np.pi * s_ / 24)])
    rng = np.random.default_rng(4)
    n = 8
    eps = rng.normal(0, 3, (n, t + 1))
    u = np.zeros((n, t))
    phi = np.array([0.5, 0.0, 0.6, 0.3, 0.8, 0.2, 0.5, 0.0])
    theta = np.array([0.4, 0.9, 0.3, -0.5, 0.2, 0.6, 0.4, 0.7])
    for k in range(t):
        u[:, k] = eps[:, k + 1] + theta * eps[:, k] + (phi * u[:, k - 1] if k else 0.0)
    y = 2000 + 10 * X[:t, 2] + u
    y[4:] = 2000 + np.cumsum(u[4:], axis=1) / 20                     # integrated rows: d >= 1 has work to do
    y = y.astype(np.float32)
    y[1, t - 3:] = np.nan
    y[2, 1000:1400] = np.nan
    y[3, rng.choice(np.arange(2, t - 1), size=t // 20, replace=False)] = np.nan
    eng = mmf.ForecastEngine()
    eng.plan(X, t, True)
    eng.plan_arima(X, t, 2)
    sc = np.sqrt(t / 1095)
    yd = _dev(y)
    for d in (0, 1, 2):
        got = _np(eng.fit_forecast_arma(yd, 1, 1, d, t, h))
        fb = _fallback(eng, yd, 1, d, t, h, t)
        want = fit_forecast_arma_packed(y, X, t, t, h, 1, 1, d)
        zt = {"z": want["base"]["z"]} if d >= 1 else {"z": y}
        near = near_threshold(want) | degenerate_rows(want["zres"], z_tau(zt) * sc)
        assert ((got["ma_order"] > 0) == want["gated"])[~near].all(), (d, got["ma_order"], want["gated"], near)
        fbr = got["ma_order"] == 0
        for k in ("pred", "phi", "order", "sigma", "status"):
            assert np.ascontiguousarray(got[k][fbr]).tobytes() == np.ascontiguousarray(fb[k][fbr]).tobytes(), (d, k)
        gated = (got["ma_order"] > 0) & want["gated"] & ~near
        assert gated.sum() >= 4, (d, gated)
        Dm = want["base"]["D"] if d >= 1 else X
        tau_fit = z_tau(zt) * sc
        tau_pred = z_tau(zt, forecast_leverage(Dm, t - d, 0, t + h - d)) * sc
        bg = np.column_stack([got["phi"][:, 0], got["theta"][:, 0]]).astype(np.float64)
        bw = np.column_stack([want["phi"][:, 0], want["theta"][:, 0]])
        lim = BETA_TOL * (1.0 + np.linalg.norm(bw, axis=1)) * _cond_factor(want) * sc
        w_beta = float((np.linalg.norm(bg - bw, axis=1)[gated] / lim[gated]).max())
        pb, sb = pred_bound(want, lim, tau_fit, tau_pred, t, h)
        wp = want["pred"][gated] - want["base"]["pred"][gated]
        gp = got["pred"][gated].astype(np.float64) - fb["pred"][gated].astype(np.float64)
        w_pred = float((np.abs(gp - wp) / pb[gated]).max())
        w_sig = float((np.abs(got["sigma"][gated] - want["sigma"][gated]) / sb[gated]).max())
        record_err("test_gpu_arma long hourly", max(w_beta, w_pred, w_sig), 1.0, what=f"d={d}")
        _le(w_beta, 1.0, f"hourly 70,001 d={d}: |dbeta| / limit")
        _le(w_pred, 1.0, f"hourly 70,001 d={d}: prediction error / pred_bound")
        _le(w_sig, 1.0, f"hourly 70,001 d={d}: |dsigma| / bound")
    eng.close()


_NEGCTL = r"""
import json, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import numpy as np, torch, mmf
from test_gpu_arma import _gappy_rows
y, X, t = _gappy_rows()
eng = mmf.ForecastEngine()
eng.plan(X, t, True)
yd = torch.full((y.shape[0], (t + 3) & ~3), float("nan"), device="cuda")
yd[:, :t] = torch.from_numpy(y).cuda()
r = eng.fit_forecast_arma(yd[:, :t], 1, 2, 0, t, 28)
print(json.dumps({{"lib": mmf._native.LIB_PATH, "phi": r["phi"][:, 0].tolist(), "theta": r["theta"][:, :2].tolist(),
                   "ma": r["ma_order"].tolist()}}))
"""


def _gappy_rows(n=64, t=730, seed=31):
    """ARMA(1, 1) errors with phi = 0.5, theta = 0.4 and 12 % isolated gaps on the daily design"""
    rng = np.random.default_rng(seed)
    X = O.design_matrix(O.calendar_grid("2019-01-01", t + 28, "D"), t)
    eps = rng.normal(0, 5, (n, t + 1))
    u = np.zeros((n, t))
    for k in range(t):
        u[:, k] = eps[:, k + 1] + 0.4 * eps[:, k] + (0.5 * u[:, k - 1] if k else 0.0)
    y = (400.0 + rng.normal(0, 20, (n, X.shape[1])) @ X[:t].T + u).astype(np.float32)
    for i in range(n):
        y[i, rng.choice(np.arange(2, t - 1), size=int(0.12 * t), replace=False)] = np.nan
    return y, X, t


@pytest.mark.parametrize("lib", ["product", "gappyreg"])
def test_negative_control_regression_rows_with_gaps(lib):
    """on rows with 12 % isolated gaps the build whose regression step takes every observed row, a missing lag entering
    as 0 (tests/_build/libmmf_arma_gappyreg.so), must exceed BETA_TOL on at least half of the rows; the product stays
    within it"""
    env = dict(os.environ)
    env.pop("MMF_LIB", None)
    if lib == "gappyreg":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_arma_gappyreg.so")
        assert os.path.exists(env["MMF_LIB"]), "negative-control library missing: run __graft_entry__.build()"
    r = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    y, X, t = _gappy_rows()
    want = fit_forecast_arma_packed(y, X, t, t, 28, 1, 2, 0)
    rows = want["gated"] & (np.array(got["ma"]) > 0)
    bw = np.column_stack([want["phi"][:, 0], want["theta"][:, :2]])
    bg = np.column_stack([got["phi"], got["theta"]])
    ratio = np.linalg.norm(bg - bw, axis=1) / (BETA_TOL * (1.0 + np.linalg.norm(bw, axis=1)) * _cond_factor(want))
    over = int((ratio[rows] > 1.0).sum())
    record_err("test_negative_control_regression_rows_with_gaps", float(ratio[rows].max()), 1.0, what=lib,
               rows_over=over, rows=int(rows.sum()))
    assert rows.sum() >= len(y) // 2, rows.sum()
    if lib == "product":
        assert over == 0, ratio[rows].max()
    else:
        assert got["lib"].endswith("libmmf_arma_gappyreg.so") and over >= rows.sum() // 2, (over, rows.sum())


@pytest.mark.parametrize("frame", ["daily", "weekly"])
def test_forecast_groups_with_arma(frame):
    """each group of forecast_groups(ar=1, diff=d, ma=1) against the oracle on that group's own calendar: the part the
    MA terms add to forecast_groups(ar=1, diff=d)'s prediction within pred_bound, and groups that fall back bit-equal"""
    import pandas as pd
    if frame == "weekly":
        pdf = mmf.synth.reference_weekly_demand(4)
        kw = dict(freq="W-MON", horizon=40, mode="holdout")
        f = "W-MON"
    else:
        parts = []
        for j, (t, end) in enumerate(((400, "2021-06-30"), (380, "2021-06-10"))):
            y, start = mmf.synth.daily_store_item_demand(6, t, seed=20 + j, end=np.datetime64(end))
            y[1, 100:110] = np.nan
            days = np.datetime64(start, "D") + np.arange(t)
            for i in range(len(y)):
                parts.append(pd.DataFrame({"Product": f"P{j}", "SKU": f"S{i}", "Date": days.astype("datetime64[ns]"),
                                           "Demand": y[i]}))
        pdf = pd.concat(parts, ignore_index=True)
        pdf = pdf[np.isfinite(pdf["Demand"])]
        kw = dict(freq="D", horizon=28, mode="holdout")
        f = "D"
    plain = mmf.forecast_groups(pdf, **kw)
    worst, n_gated = 0.0, 0
    for diff in (2, None):
        out = mmf.forecast_groups(pdf, ar=1, diff=diff, ma=1, **kw)
        base = mmf.forecast_groups(pdf, ar=1, diff=diff, **kw) if diff else mmf.forecast_groups(pdf, ar=1, **kw)
        assert list(out.columns) == list(plain.columns) and len(out) == len(plain)
        assert out[["Product", "SKU", "Date"]].equals(plain[["Product", "SKU", "Date"]])
        d = diff or 0
        gb = dict(tuple(base.groupby(["Product", "SKU"], sort=True)))
        for key, g in out.groupby(["Product", "SKU"], sort=True):
            src = pdf[(pdf["Product"] == key[0]) & (pdf["SKU"] == key[1])].sort_values("Date")
            d0, d1 = np.datetime64(src["Date"].min(), "D"), np.datetime64(src["Date"].max(), "D")
            step = O.FREQ_DAYS[f]
            t_len = int((d1 - d0).astype(int) // step + 1)
            y = np.full((1, t_len), np.nan, dtype=np.float32)
            pos = ((src["Date"].to_numpy().astype("datetime64[D]") - d0).astype(int) // step)
            y[0, pos] = src["Demand"].to_numpy()
            t_fit = t_len - kw["horizon"]
            X = O.design_matrix(O.calendar_grid(d0, t_len, f), t_fit)
            want = fit_forecast_arma_packed(y, X, t_fit, 0, t_len, 1, 1, d)
            got = g["Demand_Fitted"].to_numpy().astype(np.float64)
            fbp = gb[key]["Demand_Fitted"].to_numpy().astype(np.float64)
            zt = {"z": want["base"]["z"]} if d >= 1 else {"z": y[:, :t_fit]}
            tau_fit = z_tau(zt)
            if not want["gated"][0] or (near_threshold(want) | degenerate_rows(want["zres"], tau_fit))[0]:
                continue
            n_gated += 1
            Dm = want["base"]["D"] if d >= 1 else X
            tau_pred = z_tau(zt, forecast_leverage(Dm, t_fit - d, 0, t_len - d))
            lim = BETA_TOL * (1.0 + np.linalg.norm([want["phi"][0, 0], want["theta"][0, 0]])) * _cond_factor(want)
            pb, _ = pred_bound(want, lim, tau_fit, tau_pred, 0, t_len)
            wp = want["pred"][0] - want["base"]["pred"][0]
            gp = got - fbp
            assert np.array_equal(np.isnan(wp), np.isnan(gp)), key
            fin = np.isfinite(wp)
            err = float((np.abs(gp[fin] - wp[fin]) / pb[0][fin]).max())
            worst = max(worst, err)
            _le(err, 1.0, f"forecast_groups {frame} diff={diff} {key}: error / pred_bound")
    assert n_gated > 0
    record_err("test_forecast_groups_with_arma", worst, 1.0, what=frame, gated=n_gated)
