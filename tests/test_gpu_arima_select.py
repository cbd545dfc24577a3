"""GPU (-m gpu): (p, d) selection by hold-out MSE on levels (mmf_fit_select_arima_f32, DESIGN.md section 2 item 12).

Candidate (p, 0) is, by definition, mmf_fit_select_ar_f32 with orders (p,) and candidate (p, d >= 1)
mmf_fit_forecast_arima_f32(p, d), so every series' pred, phi, order, sigma and status must be bit-equal to the single
call of its winner, and every candidate's score must be the float64 MSE of that call's own future-mode predictions.
With diffs = (0,) the call is mmf_fit_select_ar_f32, bit for bit.  Against the float64 oracle of
tests/arima_select_oracle.py the scores must lie within mse_bound and the choice must be optimal up to the bounds.
Batches carry test_gpu_arima.py's row mix (ARIMA_KINDS: z' empty for d = 1 but not y, first values missing, gaps at the
origin) plus gaps, +Inf and fully missing held-out windows and rows empty for every d."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mmf
from ar_oracle import AR_MAX, kappa_margin
from arima_oracle import z_tau
from arima_select_oracle import choose, mse_bound, select_arima_packed
from conftest import ROOT, forecast_leverage, record_err
from oracle import mmf_oracle as O
from test_gpu_abi_contract import PATTERN, _mask_factor
from test_gpu_ar import KAPPA_MARGIN
from test_gpu_arima import ARIMA_KINDS, _cols
from test_gpu_edges import _le, _row_tol, _same_bits

pytestmark = pytest.mark.gpu

N_HOLD = 28
GRIDS = (((0, 1, 2, 3, 4), (0, 1, 2)), (tuple(range(9)), (0, 1, 2)), ((0,), (1,)), ((8,), (2,)), ((1, 3), (0, 2)),
         ((0,), (0, 1, 2)))
HOLD_KINDS = ("hold_gaps", "hold_inf", "hold_missing", "none")


def _case(cal, n=170, seed=5, n_hold=N_HOLD):
    """(y [n, t_fit + n_hold] float32, X [t_fit + 64, p], t_fit, has_constant): a regression on X plus an integrated
    AR(1) error with drift on half the rows and AR(1) noise on the other half, so both d = 0 and d >= 1 win somewhere;
    test_gpu_arima's row mix on the fit rows, the held-out kinds on the held-out rows, and the last row empty"""
    rng = np.random.default_rng(seed)
    t = {"daily": 400, "weekly": 117, "exog_only": 300, "caller": 250}[cal]
    n_rows = t + 64 if cal != "weekly" else 157
    if cal == "daily":
        X = O.design_matrix(O.calendar_grid("2019-01-01", n_rows, "D"), t)
    elif cal == "weekly":                                            # the reference's 157 / 117 / 40 weeks
        X = O.design_matrix(O.calendar_grid("2018-01-01", n_rows, "W-MON"), t)
    elif cal == "exog_only":
        X = O.design_matrix(O.calendar_grid("2019-06-03", n_rows, "D"), t, "exog_only")
    else:
        s = np.arange(n_rows, dtype=np.float64)
        X = np.column_stack([np.ones_like(s), (s - t / 2) / t, np.sqrt(s / t), np.sin(2 * np.pi * s / 30.5),
                             np.cos(2 * np.pi * s / 30.5)])
    has_c = cal != "exog_only"
    tt = t + n_hold
    beta = rng.normal(0, 20, (n, X.shape[1]))
    phi = rng.uniform(0.1, 0.8, n)
    w = np.zeros((n, tt))
    eps = rng.normal(0, 4, (n, tt))
    for k in range(tt):
        w[:, k] = eps[:, k] + (phi * w[:, k - 1] if k else 0)
    walk = np.cumsum(w + rng.normal(0, 0.5, (n, 1)), axis=1)
    integrated = (np.arange(n) // 2) % 2 == 0
    y = 500.0 + beta @ X[:tt].T + np.where(integrated[:, None], walk, 3 * w)
    y = y.astype(np.float32)
    for i in range(n):
        kind = ARIMA_KINDS[i % len(ARIMA_KINDS)]
        y[i, _cols(kind, t)] = np.inf if kind == "inf" else np.nan
        hk = HOLD_KINDS[(i // len(ARIMA_KINDS)) % len(HOLD_KINDS)]
        if hk == "hold_gaps":
            y[i, [t, t + 3, t + 4, t + n_hold - 1]] = np.nan
        elif hk == "hold_inf":
            y[i, [t + 1, t + 9]] = np.inf
        elif hk == "hold_missing":
            y[i, t:] = np.nan
    y[-1, :t] = np.nan                                               # empty for every d
    y[-2, :t:2] = np.nan                                             # z' empty for d = 1, 2; y not
    return y, X, t, has_c


def _device(y, extra=0):
    n, tt = y.shape
    full = torch.full((n, (tt + extra + 3) & ~3), float("nan"), device="cuda")
    full[:, :tt] = torch.from_numpy(y).cuda()
    return full, full[:, :tt + extra]


def _np(r):
    return {k: v.cpu().numpy() for k, v in r.items() if k != "stats"}


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _windows(t_fit, n_rows):
    return {"future": (t_fit, n_rows - t_fit), "holdout": (0, t_fit + N_HOLD), "mid": (t_fit // 3, t_fit // 2 + 20)}


def _engine(kernel, X, t_fit, has_c):
    eng = mmf.ForecastEngine(kernel=kernel)
    eng.plan(X, t_fit, has_c)
    eng.plan_arima(X, t_fit, 2)
    return eng


def _single(eng, yd, p, d, ps, npred):
    """the single call of candidate (p, d)"""
    if d == 0:
        return _np(eng.fit_select_ar(yd, N_HOLD, (p,), ps, npred))
    return _np(eng.fit_forecast_arima(yd, p, d, ps, npred))


def _scores(fut, y, t_fit, orders, diffs):
    """[n, n_diffs, n_orders] float64 MSE of every candidate's own future-mode predictions over the held-out rows"""
    yh = y[:, t_fit:t_fit + N_HOLD].astype(np.float64)
    out = np.full((len(y), len(diffs), len(orders)), np.nan)
    for k, d in enumerate(diffs):
        for j, p in enumerate(orders):
            f = fut[p, d]["pred"][:, :N_HOLD].astype(np.float64)
            ok = np.isfinite(f) & np.isfinite(yh)
            cnt = ok.sum(axis=1)
            e = np.where(ok, yh - np.where(ok, f, 0), 0)
            with np.errstate(invalid="ignore"):
                out[:, k, j] = np.where(cnt > 0, (e * e).sum(axis=1) / np.maximum(cnt, 1), np.nan)
    return out


def _ambiguous(scores, eligible):
    """rows whose two smallest eligible scores differ but lie within 1e-6 relative (equal scores come from candidates
    with bit-equal forecasts, whose GPU scores are equal too, so the first-minimum rule is checked on them)"""
    s = np.where(eligible[:, :, None], scores, np.nan).reshape(len(scores), -1)
    s = np.sort(np.where(np.isnan(s), np.inf, s), axis=1)
    if s.shape[1] < 2:
        return np.zeros(len(s), dtype=bool)
    a, b = s[:, 0], s[:, 1]
    with np.errstate(invalid="ignore"):
        return np.isfinite(b) & (b != a) & (b - a <= 1e-6 * np.abs(b))


def _check_against_single_calls(got, runs, fut_scores, eligible, orders, diffs, what):
    """checks 2-4 of the module docstring; returns the number of ambiguous rows"""
    n = len(got["choice_p"])
    cm = got["cand_mse"].astype(np.float64)
    assert np.array_equal(np.isnan(cm), np.isnan(fut_scores)), what
    ok = ~np.isnan(fut_scores)
    rel = np.abs(cm[ok] - fut_scores[ok]) / np.maximum(np.abs(fut_scores[ok]), 1e-30)
    _le(float(rel.max()) if rel.size else 0.0, 1e-6, f"{what}: cand_mse against the single calls")
    kk, jj = choose(fut_scores, eligible)
    amb = _ambiguous(fut_scores, eligible)
    cp, cd = got["choice_p"], got["choice_d"]
    want_p = np.where(kk >= 0, np.array(orders)[np.maximum(jj, 0)], -1)
    want_d = np.where(kk >= 0, np.array(diffs)[np.maximum(kk, 0)], -1)
    bad = np.flatnonzero(((cp != want_p) | (cd != want_d)) & ~amb)
    assert bad.size == 0, (what, bad[:8], cp[bad[:8]], cd[bad[:8]], want_p[bad[:8]], want_d[bad[:8]])
    assert np.isin(cp[cp >= 0], orders).all() and np.isin(cd[cd >= 0], diffs).all() and ((cp < 0) == (cd < 0)).all()
    none = cp < 0
    assert (none == ~eligible.any(axis=1)).all(), what
    for key in ("pred", "phi", "order", "sigma", "status"):
        want = np.empty_like(got[key])
        for (p, d), r in runs.items():
            sel = (cp == p) & (cd == d)
            want[sel] = r[key][sel]
        if none.any():
            want[none] = {"pred": np.nan, "phi": 0.0, "order": 0, "sigma": np.nan, "status": 1}[key]
        bad = np.flatnonzero((_bits(got[key]) != _bits(want)).reshape(n, -1).any(axis=1))
        assert bad.size == 0, (what, key, bad[:8], cp[bad[:8]], cd[bad[:8]])
    k_of = {d: k for k, d in enumerate(diffs)}
    j_of = {p: j for j, p in enumerate(orders)}
    rows = np.flatnonzero(~none)
    win = got["cand_mse"][rows, [k_of[d] for d in cd[rows]], [j_of[p] for p in cp[rows]]]
    assert np.array_equal(_bits(got["mse"][rows]), _bits(win)) and np.isnan(got["mse"][none]).all(), what
    return int(amb.sum())


@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_diffs_zero_is_bit_equal_to_ar_order_selection(cal):
    y, X, t_fit, has_c = _case(cal)
    _, yd = _device(y)
    for kernel in ("auto", "tc", "warp"):
        eng = _engine(kernel, X, t_fit, has_c)
        for name, (ps, npred) in _windows(t_fit, X.shape[0]).items():
            for orders in ((0, 1, 2, 3, 4), tuple(range(9)), (0,), (8,), (1, 3)):
                got = _np(eng.fit_select_arima(yd, N_HOLD, orders, (0,), ps, npred))
                ref = _np(eng.fit_select_ar(yd, N_HOLD, orders, ps, npred))
                what = f"{cal} {kernel} {name} {orders}"
                assert np.array_equal(got["choice_p"], ref["choice"]), what
                assert np.array_equal(got["choice_d"], np.where(ref["choice"] < 0, -1, 0)), what
                assert _bits(got["cand_mse"][:, 0, :]).tobytes() == _bits(ref["cand_mse"]).tobytes(), what
                for k in ("pred", "mse", "phi", "order", "sigma", "status"):
                    assert _bits(got[k]).tobytes() == _bits(ref[k]).tobytes(), (what, k)
        eng.close()


@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_bit_equal_to_the_winners_single_call(cal):
    y, X, t_fit, has_c = _case(cal)
    _, yd = _device(y)
    amb_total = checked = 0
    for kernel in ("auto", "tc", "warp"):
        eng = _engine(kernel, X, t_fit, has_c)
        fut = {(p, d): _single(eng, yd, p, d, t_fit, N_HOLD) for p in range(AR_MAX + 1) for d in (0, 1, 2)}
        eligible_d = {d: fut[0, d]["status"] != 1 for d in (0, 1, 2)}
        for name, (ps, npred) in _windows(t_fit, X.shape[0]).items():
            runs = {(p, d): _single(eng, yd, p, d, ps, npred) for p in range(AR_MAX + 1) for d in (0, 1, 2)}
            for orders, diffs in GRIDS:
                got = _np(eng.fit_select_arima(yd, N_HOLD, orders, diffs, ps, npred))
                sc = _scores(fut, y, t_fit, orders, diffs)
                el = np.stack([eligible_d[d] for d in diffs], axis=1)
                amb_total += _check_against_single_calls(got, runs, sc, el, orders, diffs,
                                                         f"{cal} {kernel} {name} {orders} x {diffs}")
                checked += 1
        eng.close()
    record_err("arima_select_ambiguous_rows", float(amb_total), float(checked * len(y)), what=cal)


def _taus(y, X, t_fit, want, diffs, n_hold=N_HOLD, scale=1.0):
    """per d, the (tau_fit, tau_hold) of mse_bound: the plain tolerances for d = 0 (test_gpu_ar_select), those of
    test_gpu_arima's arima_bound on z' for d >= 1, each x its mask factor and x ``scale``"""
    n = len(y)
    out = {}
    for k, d in enumerate(diffs):
        if d == 0:
            lev = forecast_leverage(X, t_fit, t_fit, n_hold)
            tf = _row_tol(y[:, :t_fit]) * _mask_factor(y[:, :t_fit], X, t_fit, 0, t_fit, np.ones(n))
            th = _row_tol(y[:, :t_fit], lev) * _mask_factor(y[:, :t_fit], X, t_fit, t_fit, n_hold, np.ones(n))
        else:
            h = want["hold"][k][0]
            z, D = h["z"], h["D"]
            tz, nz = t_fit - d, t_fit + n_hold - d
            lev = forecast_leverage(D, tz, 0, nz)
            tf = z_tau(h) * _mask_factor(z, D, tz, 0, tz, np.ones(n))
            th = z_tau(h, lev) * _mask_factor(z, D, tz, 0, nz, np.ones(n))
        out[d] = (np.where(np.isfinite(tf), tf * scale, 0.0), np.where(np.isfinite(th), th * scale, 0.0))
    return out


@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_scores_and_choice_against_the_oracle(cal):
    y, X, t_fit, has_c = _case(cal)
    n = len(y)
    orders, diffs = (0, 1, 2, 3, 4), (0, 1, 2)
    _, yd = _device(y)
    eng = _engine("auto", X, t_fit, has_c)
    got = _np(eng.fit_select_arima(yd, N_HOLD, orders, diffs, t_fit, N_HOLD))
    eng.close()
    want = select_arima_packed(y, X, t_fit, N_HOLD, orders, diffs, t_fit, N_HOLD)
    bound = mse_bound(want, y, _taus(y, X, t_fit, want, diffs), t_fit, N_HOLD, orders, diffs)
    near = np.zeros(n, dtype=bool)
    for row in want["hold"]:
        for h in row:
            near |= kappa_margin(h.get("zres", h)) < KAPPA_MARGIN
    live = want["eligible"].any(axis=1) & ~near
    record_err("arima_select_near_limit_rows", float(near.sum()), float(n), what=cal)
    assert np.array_equal(got["choice_p"] < 0, ~want["eligible"].any(axis=1)), cal
    cm = got["cand_mse"].astype(np.float64)
    assert np.array_equal(np.isnan(cm[live]), np.isnan(want["cand_mse"][live])), cal
    ok = live[:, None, None] & ~np.isnan(want["cand_mse"])
    err = np.abs(cm - np.where(ok, want["cand_mse"], 0))
    ratio = np.where(ok, err / np.where(bound > 0, bound, np.inf), 0)
    _le(float(ratio.max()), 1.0, f"{cal}: |cand_mse - oracle| / mse_bound")
    # the oracle MSE of the GPU's choice lies within both bounds of the oracle's minimum; differing choices are counted
    k_of = {d: k for k, d in enumerate(diffs)}
    j_of = {p: j for j, p in enumerate(orders)}
    rows = np.flatnonzero(live & ~np.isnan(want["cand_mse"]).all(axis=(1, 2)))
    gk = np.array([k_of[d] for d in got["choice_d"][rows]])
    gj = np.array([j_of[p] for p in got["choice_p"][rows]])
    ok_, oj = want["k"][rows], want["j"][rows]
    o_mse = want["cand_mse"]
    slack = bound[rows, gk, gj] + bound[rows, ok_, oj]
    over = o_mse[rows, gk, gj] > o_mse[rows, ok_, oj] + slack
    assert not over.any(), (cal, rows[over][:8])
    record_err("arima_select_choice_differs", float(((gk != ok_) | (gj != oj)).sum()), float(rows.size), what=cal)
    hist = {f"{p},{d}": int(((got["choice_p"] == p) & (got["choice_d"] == d)).sum()) for d in diffs for p in orders}
    record_err("arima_select_choice_histogram", 0.0, 1.0, what=cal, hist=hist)


def test_y_beyond_the_held_out_window_is_never_read():
    y, X, t_fit, has_c = _case("daily")
    eng = _engine("auto", X, t_fit, has_c)
    full, yd = _device(y, extra=40)
    ref = _np(eng.fit_select_arima(yd, N_HOLD, (0, 1, 2), (0, 1, 2), 0, t_fit + 64))
    full[:, t_fit + N_HOLD:] = 3.0e38
    other = _np(eng.fit_select_arima(yd, N_HOLD, (0, 1, 2), (0, 1, 2), 0, t_fit + 64))
    for k in ref:
        assert _bits(ref[k]).tobytes() == _bits(other[k]).tobytes(), k
    eng.close()


def test_exact_power_of_two_scaling():
    y, X, t_fit, has_c = _case("daily")
    eng = _engine("auto", X, t_fit, has_c)
    _, yd = _device(y)
    a = _np(eng.fit_select_arima(yd, N_HOLD, (0, 1, 3), (0, 1, 2), t_fit, 28))
    b = _np(eng.fit_select_arima(yd * 8.0, N_HOLD, (0, 1, 3), (0, 1, 2), t_fit, 28))
    for k, f in (("pred", 8.0), ("phi", 1.0), ("order", 1), ("sigma", 8.0), ("status", 1), ("mse", 64.0),
                 ("cand_mse", 64.0), ("choice_p", 1), ("choice_d", 1)):
        w = a[k] * f
        same = (b[k] == w) | (np.isnan(b[k]) & np.isnan(w))
        assert same.all(), (k, np.flatnonzero(~same.reshape(len(y), -1).all(axis=1))[:6])
    eng.close()


def test_slabs_are_bit_equal_to_per_slab_calls():
    n, t = (1 << 20) + 1001, 48
    y, start = mmf.synth.daily_store_item_demand(n, t + 8, seed=9, nan_frac=0.01)
    X = O.design_matrix(O.calendar_grid(start, t + 8, "D"), t)
    eng = _engine("auto", X, t, True)
    yd = torch.from_numpy(y).cuda()
    whole = eng.fit_select_arima(yd, 8, (0, 1, 2), (0, 1, 2), t, 8)
    for lo, hi in ((0, 1 << 19), (1 << 19, n)):
        part = eng.fit_select_arima(yd[lo:hi], 8, (0, 1, 2), (0, 1, 2), t, 8)
        for k in whole:
            assert _same_bits(whole[k][lo:hi], part[k]), k
    eng.close()


def test_long_hourly_series():
    """70,001 fit rows: bounds x sqrt(t_fit / 1095)"""
    t, h = 70001, 48
    s = np.arange(t + h + 8, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), (s - t / 2) / t, np.sin(2 * np.pi * s / 24), np.cos(2 * np.pi * s / 24)])
    rng = np.random.default_rng(4)
    n = 24
    w = np.zeros((n, t + h))
    eps = rng.normal(0, 3, (n, t + h))
    for k in range(1, t + h):
        w[:, k] = 0.6 * w[:, k - 1] + eps[:, k]
    y = 2000 + 10 * X[:t + h, 2] + np.where(np.arange(n)[:, None] % 2 == 0, np.cumsum(w, axis=1) / 20, w)
    y = y.astype(np.float32)
    y[1, t - 3:t] = np.nan
    y[2, 1000:1400] = np.nan
    eng = _engine("auto", X, t, True)
    orders, diffs = (0, 1, 2), (0, 1, 2)
    _, yd = _device(y)
    got = _np(eng.fit_select_arima(yd, h, orders, diffs, t, h))
    eng.close()
    want = select_arima_packed(y, X, t, h, orders, diffs, t, h)
    bound = mse_bound(want, y, _taus(y, X, t, want, diffs, h, np.sqrt(t / 1095)), t, h, orders, diffs)
    ok = ~np.isnan(want["cand_mse"])
    ratio = np.abs(got["cand_mse"].astype(np.float64)[ok] - want["cand_mse"][ok]) / bound[ok]
    _le(float(ratio.max()), 1.0, "hourly 70,001: |cand_mse - oracle| / mse_bound")
    assert np.array_equal(np.isnan(got["cand_mse"]), ~ok)


def test_nullable_outputs_and_a_wide_table():
    y, X, t_fit, has_c = _case("daily")
    n = len(y)
    eng = _engine("auto", X, t_fit, has_c)
    lib, h = eng._lib, eng._h
    _, yd = _device(y)
    orders, diffs = (0, 2), (0, 1, 2)
    ref = eng.fit_select_arima(yd, N_HOLD, orders, diffs, t_fit, 28)
    wide = torch.full((n, 41), float(np.float32(PATTERN)), device="cuda")
    view = wide[:, 5:33]
    c = (ctypes.c_int32 * 2)(*orders)
    dl = (ctypes.c_int32 * 3)(*diffs)
    rc = lib.mmf_fit_select_arima_f32(h, yd.data_ptr(), n, yd.stride(0), N_HOLD, c, 2, dl, 3, t_fit, 28,
                                      view.data_ptr(), 41, None, None, None, None, None, None, None, None, None)
    assert rc == 0
    torch.cuda.synchronize()
    assert _same_bits(view, ref["pred"])
    assert (wide[:, :5] == float(np.float32(PATTERN))).all() and (wide[:, 33:] == float(np.float32(PATTERN))).all()
    cd = torch.full((n,), 7, device="cuda", dtype=torch.int32)
    rc = lib.mmf_fit_select_arima_f32(h, yd.data_ptr(), n, yd.stride(0), N_HOLD, c, 2, dl, 3, t_fit, 28,
                                      view.data_ptr(), 41, None, cd.data_ptr(), None, None, None, None, None, None, None)
    assert rc == 0
    torch.cuda.synchronize()
    assert _same_bits(cd, ref["choice_d"]) and _same_bits(view, ref["pred"])
    eng.close()


def test_refused_calls_write_nothing():
    y, X, t_fit, has_c = _case("daily", n=40)
    n = len(y)
    eng = mmf.ForecastEngine()
    lib, h = eng._lib, eng._h
    _, yd = _device(y)
    ld = yd.stride(0)
    bufs = [torch.full((n, 28), 7.0, device="cuda"), torch.full((n,), 7, device="cuda", dtype=torch.int32),
            torch.full((n,), 7, device="cuda", dtype=torch.int32), torch.full((n,), 7.0, device="cuda"),
            torch.full((n, 27), 7.0, device="cuda"), torch.full((n, AR_MAX), 7.0, device="cuda"),
            torch.full((n,), 7, device="cuda", dtype=torch.int32), torch.full((n,), 7.0, device="cuda"),
            torch.full((n,), 7, device="cuda", dtype=torch.int32)]
    host_out = np.zeros((n, 28), dtype=np.float32)

    def call(orders=(1,), diffs=(0, 1), n_hold=N_HOLD, ps=t_fit, npred=28, optr=None, ldo=28, ld_y=ld, ctx=h):
        c = (ctypes.c_int32 * max(len(orders), 1))(*orders) if orders is not None else None
        dl = (ctypes.c_int32 * max(len(diffs), 1))(*diffs) if diffs is not None else None
        return lib.mmf_fit_select_arima_f32(ctx, yd.data_ptr(), n, ld_y, n_hold, c, len(orders or ()), dl,
                                            len(diffs or ()), ps, npred, bufs[0].data_ptr() if optr is None else optr,
                                            ldo, *[b.data_ptr() for b in bufs[1:]], None)
    assert call(diffs=(0,)) == -4 and call(diffs=(1,)) == -4                   # MMF_E_NOPLAN: no plan at all
    eng.plan(X, t_fit, has_c)
    assert call(diffs=(0, 1)) == -4 and call(diffs=(1,)) == -4                 # no ARIMA plan
    eng.plan_arima(X, t_fit, 1)
    refused = [dict(orders=()), dict(orders=None), dict(orders=(2, 1)), dict(orders=(1, 1)), dict(orders=(0, 9)),
               dict(orders=(-1, 2)), dict(orders=tuple(range(9)) + (8,)), dict(diffs=()), dict(diffs=None),
               dict(diffs=(1, 0)), dict(diffs=(1, 1)), dict(diffs=(0, 3)), dict(diffs=(-1, 0)),
               dict(diffs=(0, 1, 2, 2)), dict(diffs=(0, 2)), dict(diffs=(2,)),                     # max_diff is 1
               dict(n_hold=0), dict(n_hold=X.shape[0] - t_fit + 1), dict(ld_y=t_fit + N_HOLD - 1), dict(ps=-1),
               dict(npred=X.shape[0] + 1), dict(ldo=27), dict(optr=host_out.ctypes.data), dict(ctx=None)]
    for kw in refused:
        assert call(**kw) != 0, kw
    Xo = X.copy()
    Xo[5, 1] += 1e-9                                                           # the same shape, other bytes
    eng.plan_arima(Xo, t_fit, 2)
    assert call(diffs=(0, 1)) == -1                                            # MMF_E_INVALID: plans of different X
    eng.plan_arima(X[:-1], t_fit, 2)
    assert call(diffs=(0, 1)) == -1                                            # ... and of other rows
    eng.plan_arima(X, t_fit - 1, 2)
    assert call(diffs=(0, 1)) == -1                                            # ... and of another t_fit
    torch.cuda.synchronize()
    assert all((b == 7).all() for b in bufs)
    assert not host_out.any()
    eng.close()


def test_other_calls_unchanged_and_a_shared_context_matches_a_fresh_one():
    y, X, t_fit, has_c = _case("daily")
    start = np.datetime64("2019-01-01", "D")
    eng = mmf.ForecastEngine()
    eng.plan_calendars([start, start + 30], [t_fit, t_fit - 30], "D", 28)
    eng.plan_backtest(start, t_fit, "D", 28, 3)
    eng.plan(X, t_fit, has_c)
    eng.plan_arima(X, t_fit, 2)
    _, yd = _device(y)
    yf = yd[:, :t_fit]

    def calls():
        bt = eng.backtest(yf)
        return (eng.fit_forecast(yf, t_fit, 28).clone(), eng.fit_forecast(yf, 0, t_fit + 64).clone(),
                eng.fit_forecast_ar(yf, 2, t_fit, 28)["pred"].clone(), eng.fit_select_ar(yd, 28, (0, 1, 2))["pred"].clone(),
                eng.fit_forecast_arima(yf, 2, 1, t_fit, 28)["pred"].clone(),
                eng.fit_forecast_ragged(yf, [0, 70, len(y)]).clone(), bt["pred"].clone(), bt["metrics"].clone(),
                bt["status"].clone())

    args = (((0, 1, 2, 3, 4), (0, 1, 2), t_fit, 28), ((8,), (2,), 0, t_fit + 64), ((1, 3), (0, 2), 50, 100))
    before = calls()
    shared = [_np(eng.fit_select_arima(yd, N_HOLD, o, d, ps, npred)) for o, d, ps, npred in args]
    after = calls()
    assert all(_same_bits(a, b) for a, b in zip(before, after))
    fresh_eng = mmf.ForecastEngine()
    fresh_eng.plan(X, t_fit, has_c)
    fresh_eng.plan_arima(X, t_fit, 2)
    fresh = [_np(fresh_eng.fit_select_arima(yd, N_HOLD, o, d, ps, npred)) for o, d, ps, npred in args]
    for a, b in zip(shared, fresh):
        for k in a:
            assert _bits(a[k]).tobytes() == _bits(b[k]).tobytes(), k
    eng.close()
    fresh_eng.close()


_NEGCTL = """
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np, torch
import mmf
import test_gpu_arima_select as T
from arima_select_oracle import mse_bound, select_arima_packed
from oracle import mmf_oracle as O
n, t, h = 300, 400, 28
rng = np.random.default_rng(8)
X = O.design_matrix(O.calendar_grid("2019-01-01", t + h, "D"), t)
y = (1000 + np.cumsum(rng.normal(2.0, 5.0, (n, t + h)), axis=1)).astype(np.float32)
orders, diffs = (0, 1, 2), (0, 1, 2)
eng = T._engine("auto", X, t, True)
_, yd = T._device(y)
got = T._np(eng.fit_select_arima(yd, h, orders, diffs, t, h))
want = select_arima_packed(y, X, t, h, orders, diffs, t, h)
b = mse_bound(want, y, T._taus(y, X, t, want, diffs), t, h, orders, diffs)
r = np.abs(got["cand_mse"].astype(np.float64) - want["cand_mse"]) / b
over = (r[:, 1:, :] > 1).reshape(-1)
print(json.dumps({{"worst_d0": float(r[:, 0, :].max()), "worst": float(r[:, 1:, :].max()), "over": int(over.sum()),
                  "cands": int(over.size), "lib": mmf.LIB_PATH}}))
"""


@pytest.mark.parametrize("lib", ["product", "onestep"])
def test_negative_control_with_a_leaky_one_step_score(lib):
    """random walks with drift: the build that feeds each observed held-out level into the candidates' level chains
    (tests/_build/libmmf_arimasel_onestep.so) must exceed mse_bound on at least half of the d >= 1 candidates' rows;
    the product library stays within it"""
    env = dict(os.environ)
    env.pop("MMF_LIB", None)
    if lib == "onestep":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_arimasel_onestep.so")
        assert os.path.exists(env["MMF_LIB"]), "negative-control library missing: run __graft_entry__.build()"
    r = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    record_err("test_negative_control_with_a_leaky_one_step_score", got["worst"], 1.0, what=lib, over=got["over"],
               cands=got["cands"])
    if lib == "product":
        assert got["worst"] <= 1.0 and got["worst_d0"] <= 1.0, got
    else:
        assert got["lib"].endswith("libmmf_arimasel_onestep.so") and got["over"] >= got["cands"] // 2, got


@pytest.mark.parametrize("frame", ["daily", "weekly"])
def test_forecast_groups_with_pd_selection(frame):
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
    orders, diffs = (0, 1, 2, 3, 4), (0, 1, 2)
    out = mmf.forecast_groups(pdf, ar=orders, diff=diffs, **kw)
    plain = mmf.forecast_groups(pdf, **kw)
    assert list(out.columns) == list(plain.columns) and len(out) == len(plain)
    worst, amb = 0.0, 0
    for key, g in out.groupby(["Product", "SKU"], sort=True):
        src = pdf[(pdf["Product"] == key[0]) & (pdf["SKU"] == key[1])].sort_values("Date")
        d0, d1 = np.datetime64(src["Date"].min(), "D"), np.datetime64(src["Date"].max(), "D")
        step = O.FREQ_DAYS[f]
        t_len = int((d1 - d0).astype(int) // step + 1)
        y = np.full((1, t_len), np.nan, dtype=np.float32)
        pos = ((src["Date"].to_numpy().astype("datetime64[D]") - d0).astype(int) // step)
        y[0, pos] = src["Demand"].to_numpy()
        h = kw["horizon"]
        t_fit = t_len - h
        X = O.design_matrix(O.calendar_grid(d0, t_len, f), t_fit)
        want = select_arima_packed(y, X, t_fit, h, orders, diffs, 0, t_len)
        b = mse_bound(want, y, _taus(y, X, t_fit, want, diffs, h), t_fit, h, orders, diffs)
        # the hold-out MSE of the group's forecast lies within two bounds (its winner's and the oracle's winner's, each
        # at most the largest of the group) of the oracle's minimum; groups whose score is closest to another
        # candidate's oracle score than to the minimum's took another winner (two candidates within the bounds), counted
        got = g["Demand_Fitted"].to_numpy().astype(np.float64)
        fut = _score_of(got[t_fit:t_fit + h], y[0, t_fit:t_fit + h])
        best = want["cand_mse"][0, want["k"][0], want["j"][0]]
        if not np.isnan(best):
            worst = max(worst, float((fut - best) / max(2 * b[0].max(), 1e-30)))
            flat = want["cand_mse"][0].reshape(-1)
            near = int(np.nanargmin(np.abs(flat - fut)))
            amb += int(flat[near] != best)
    record_err("arima_select_frames_ambiguous_groups", float(amb), float(out.groupby(["Product", "SKU"]).ngroups),
               what=frame)
    _le(worst, 1.0, f"forecast_groups(ar=(0..4), diff=(0, 1, 2)) {frame}: hold-out MSE over the oracle's minimum / bound")


def _score_of(pred, yh):
    ok = np.isfinite(pred) & np.isfinite(yh)
    return float(np.mean((yh[ok].astype(np.float64) - pred[ok]) ** 2)) if ok.any() else np.nan

