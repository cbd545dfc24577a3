"""GPU (-m gpu): AR order selection by hold-out MSE (mmf_fit_select_ar_f32, DESIGN.md section 2 item 10).

Candidate m >= 1 is, by definition, mmf_fit_forecast_ar_f32 with ar_order = m, so every series' pred, phi, order, sigma
and status must be bit-equal to that call with ar_order = its choice, and every candidate's hold-out MSE must be the
float64 MSE of that call's own future-mode predictions.  Against the float64 oracle of tests/ar_select_oracle.py the
scores must lie within mse_bound and the choice must be optimal up to the bounds.  Batches carry the row mix of
test_gpu_ar.py (AR_KINDS) plus rows with gaps and +Inf inside the held-out window and rows whose held-out window is
fully missing."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mmf
from ar_oracle import AR_MAX, ar_bound, kappa_margin
from ar_select_oracle import mse_bound, select_ar_packed
from conftest import ROOT, forecast_leverage, record_err
from oracle import mmf_oracle as O
from test_gpu_abi_contract import PATTERN, _mask_factor
from test_gpu_ar import AR_KINDS, KAPPA_MARGIN, _plant
from test_gpu_edges import _le, _row_tol, _same_bits

pytestmark = pytest.mark.gpu

N_HOLD = 28
ORDER_LISTS = ((0, 1, 2, 3, 4), (0,), (8,), (1, 3, 8), tuple(range(9)))
HOLD_KINDS = ("hold_gaps", "hold_inf", "hold_missing", "none")


def _hold_kind(i):
    return HOLD_KINDS[(i // len(AR_KINDS)) % len(HOLD_KINDS)]


def _case(cal, n=150, seed=3, n_hold=N_HOLD, phi=None):
    """(y [n, t_fit + n_hold] float32, X, t_fit, has_constant): test_gpu_ar's calendars and row mix on the fit rows,
    the held-out rows continue each series; phi None: AR(1) noise with phi ~ U(0.1, 0.9) per series"""
    rng = np.random.default_rng(seed)
    t = {"daily": 400, "weekly": 130, "exog_only": 300, "caller": 250}[cal]
    tt = t + n_hold
    if cal == "daily":
        X = O.design_matrix(O.calendar_grid("2019-01-01", t + 64, "D"), t)
    elif cal == "weekly":
        X = O.design_matrix(O.calendar_grid("2018-01-01", t + 64, "W-MON"), t)
    elif cal == "exog_only":
        X = O.design_matrix(O.calendar_grid("2019-06-03", t + 64, "D"), t, "exog_only")
    else:
        s = np.arange(t + 64, dtype=np.float64)
        X = np.column_stack([np.ones_like(s), (s - t / 2) / t, np.sqrt(s / t), np.sin(2 * np.pi * s / 30.5),
                             np.cos(2 * np.pi * s / 30.5)])
    has_c = cal != "exog_only"
    beta = rng.normal(0, 20, (n, X.shape[1]))
    base = 100.0 + beta @ X[:tt].T if has_c else 100.0 * (1 + X[:tt, :3].sum(1)) + beta @ X[:tt].T
    ph = rng.uniform(0.1, 0.9, n) if phi is None else np.full(n, phi)
    eps = rng.normal(0, 5, (n, tt))
    noise = np.zeros((n, tt))
    for k in range(tt):
        noise[:, k] = eps[:, k] + (ph * noise[:, k - 1] if k else 0)
    y = (base + noise).astype(np.float32)
    if phi is None:
        _plant(y[:, :t], t)
        for i in range(n):
            kind = _hold_kind(i)
            if kind == "hold_gaps":
                y[i, [t, t + 3, t + 4, t + n_hold - 1]] = np.nan
            elif kind == "hold_inf":
                y[i, [t + 1, t + 9]] = np.inf
            elif kind == "hold_missing":
                y[i, t:] = np.nan
    return y, X, t, has_c


def _device(y, extra=0):
    """y on the GPU with a 16-B row pitch (the tensor-core kernel) and ``extra`` further columns of NaN"""
    n, tt = y.shape
    full = torch.full((n, (tt + extra + 3) & ~3), float("nan"), device="cuda")
    full[:, :tt] = torch.from_numpy(y).cuda()
    return full, full[:, :tt + extra]


def _np(r):
    return {k: v.cpu().numpy() for k, v in r.items() if k != "stats"}


def _windows(t_fit, n_rows):
    return {"future": (t_fit, min(64, n_rows - t_fit)), "holdout": (0, t_fit + N_HOLD),
            "mid": (t_fit // 3, t_fit // 2 + 40)}


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _gather(runs, choice, orders, key):
    """per row, runs[m][key][row] for m = the row's choice (empty rows, choice -1: the last listed order)"""
    m = np.where(choice < 0, orders[-1], choice)
    out = np.empty_like(runs[orders[0]][key])
    for o in set(m.tolist()):
        out[m == o] = runs[o][key][m == o]
    return out


def _scores(runs_future, y, t_fit, orders):
    """float64 MSE of every order's own future-mode predictions over the held-out rows, NaN where nothing is scored"""
    yh = y[:, t_fit:t_fit + N_HOLD].astype(np.float64)
    out = []
    for m in orders:
        f = runs_future[m]["pred"][:, :N_HOLD].astype(np.float64)
        ok = np.isfinite(f) & np.isfinite(yh)
        cnt = ok.sum(axis=1)
        d = np.where(ok, yh - np.where(ok, f, 0), 0)
        with np.errstate(invalid="ignore"):
            out.append(np.where(cnt > 0, (d * d).sum(axis=1) / np.maximum(cnt, 1), np.nan))
    return np.stack(out, axis=1)


def _fixed_runs(eng, yd, ps, npred):
    """order 0 through a one-candidate selection, orders 1..8 through mmf_fit_forecast_ar_f32"""
    runs = {0: _np(eng.fit_select_ar(yd, N_HOLD, (0,), ps, npred))}
    for m in range(1, AR_MAX + 1):
        runs[m] = _np(eng.fit_forecast_ar(yd, m, ps, npred))
    return runs


@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_selection_is_bit_equal_to_the_fixed_order_call(cal):
    y, X, t_fit, has_c = _case(cal)
    n = len(y)
    _, yd = _device(y)
    checked = 0
    for kernel in ("auto", "tc", "warp"):
        eng = mmf.ForecastEngine(kernel=kernel)
        eng.plan(X, t_fit, has_c)
        fut = _fixed_runs(eng, yd, t_fit, N_HOLD)
        for name, (ps, npred) in _windows(t_fit, X.shape[0]).items():
            runs = _fixed_runs(eng, yd, ps, npred)
            plain = eng.fit_forecast(yd, ps, npred).cpu().numpy()
            lev = forecast_leverage(X, t_fit, ps, npred)
            tau = _row_tol(y[:, :t_fit], lev) * _mask_factor(y[:, :t_fit], X, t_fit, ps, npred, np.ones(n))
            for orders in ORDER_LISTS:
                what = f"{cal} {kernel} {name} {orders}"
                got = _np(eng.fit_select_ar(yd, N_HOLD, orders, ps, npred))
                ch = got["choice"]
                st = got["status"]
                assert np.array_equal(st, runs[1]["status"]), what
                assert ((ch == -1) == (st == 1)).all() and np.isin(ch[st != 1], orders).all(), what
                for k in ("pred", "phi", "order", "sigma", "status"):
                    want = _gather(runs, ch, orders, k)
                    bad = np.flatnonzero((_bits(got[k]) != _bits(want)).reshape(n, -1).any(axis=1))
                    assert bad.size == 0, (what, k, bad[:8], ch[bad[:8]])
                zero = ch == 0
                assert not got["phi"][zero].any() and not got["order"][zero].any(), what
                err = np.abs(got["pred"][zero].astype(np.float64) - plain[zero])
                _le(float((err / (2 * tau[zero, None])).max()) if zero.any() else 0.0, 1.0,
                    f"{what}: order-0 rows against the plain call / 2 tol")
                # scores: the float64 MSE of every order's own future-mode predictions, and the choice among them
                want = _scores(fut, y, t_fit, orders)
                cm = got["cand_mse"].astype(np.float64)
                assert np.array_equal(np.isnan(cm), np.isnan(want)), what
                ok = ~np.isnan(want)
                rel = np.abs(cm[ok] - want[ok]) / np.maximum(np.abs(want[ok]), 1e-30)
                _le(float(rel.max()) if rel.size else 0.0, 1e-6, f"{what}: cand_mse against the fixed-order calls")
                idx = np.array([orders.index(c) if c >= 0 else len(orders) - 1 for c in ch])
                assert np.array_equal(_bits(got["mse"]), _bits(got["cand_mse"][np.arange(n), idx])), what
                with np.errstate(invalid="ignore"):
                    assert not (got["cand_mse"] < got["mse"][:, None]).any(), what
                unscored = (st != 1) & np.isnan(got["cand_mse"]).all(axis=1)
                assert (idx[unscored] == len(orders) - 1).all(), what
                checked += 1
        eng.close()
    record_err("test_selection_is_bit_equal_to_the_fixed_order_call", 0.0, 1.0, what=cal, combos=checked)


@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_scores_and_choice_against_the_oracle(cal):
    y, X, t_fit, has_c = _case(cal)
    n = len(y)
    orders = tuple(range(9))
    _, yd = _device(y)
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    got = _np(eng.fit_select_ar(yd, N_HOLD, orders, t_fit, N_HOLD))
    eng.close()
    want = select_ar_packed(y, X, t_fit, N_HOLD, orders, t_fit, N_HOLD)
    lev = forecast_leverage(X, t_fit, t_fit, N_HOLD)
    tau_fit = _row_tol(y[:, :t_fit]) * _mask_factor(y[:, :t_fit], X, t_fit, 0, t_fit, np.ones(n))
    tau_hold = _row_tol(y[:, :t_fit], lev) * _mask_factor(y[:, :t_fit], X, t_fit, t_fit, N_HOLD, np.ones(n))
    tau_fit = np.where(np.isfinite(tau_fit), tau_fit, 0)
    tau_hold = np.where(np.isfinite(tau_hold), tau_hold, 0)
    bound = mse_bound(want, y, tau_fit, tau_hold, t_fit, N_HOLD, orders)
    near = np.zeros(n, dtype=bool)
    for h in want["hold"]:
        near |= kappa_margin(h) < KAPPA_MARGIN
    live = (want["status"] != 1) & ~near
    record_err("ar_select_near_limit_rows", float(near.sum()), float(n), what=cal)
    cm = got["cand_mse"].astype(np.float64)
    assert np.array_equal(np.isnan(cm[live]), np.isnan(want["cand_mse"][live])), cal
    ok = live[:, None] & ~np.isnan(want["cand_mse"])
    err = np.abs(cm - np.where(ok, want["cand_mse"], 0))
    ratio = np.where(ok, err / np.where(bound > 0, bound, np.inf), 0)
    _le(float(ratio.max()), 1.0, f"{cal}: |cand_mse - oracle| / mse_bound")
    # the GPU's choice is optimal up to the bounds; rows where two candidates lie within them are counted
    rows = np.arange(n)
    gidx = np.array([orders.index(c) if c >= 0 else len(orders) - 1 for c in got["choice"]])
    scored = live & ~np.isnan(want["cand_mse"]).all(axis=1)
    o_mse = want["cand_mse"]
    oi = want["idx"]
    slack = bound[rows, gidx] + bound[rows, oi]
    over = scored & (o_mse[rows, gidx] > o_mse[rows, oi] + slack)
    assert not over.any(), (cal, np.flatnonzero(over)[:8])
    close = scored & (gidx != oi)
    record_err("ar_select_ambiguous_rows", float(close.sum()), float(scored.sum()), what=cal)
    unscored = live & np.isnan(want["cand_mse"]).all(axis=1)
    assert unscored.any() and (got["choice"][unscored] == orders[-1]).all(), cal


def test_y_beyond_the_held_out_window_is_never_read():
    y, X, t_fit, has_c = _case("daily")
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    full, yd = _device(y, extra=40)
    ref = eng.fit_select_ar(yd, N_HOLD, (0, 1, 2, 3, 4), 0, t_fit + 64)
    full[:, t_fit + N_HOLD:] = 3.0e38
    other = eng.fit_select_ar(yd, N_HOLD, (0, 1, 2, 3, 4), 0, t_fit + 64)
    for k in ref:
        assert _same_bits(ref[k], other[k]), k
    eng.close()


def test_nullable_outputs_and_a_wide_table():
    y, X, t_fit, has_c = _case("daily")
    n = len(y)
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    lib, h = eng._lib, eng._h
    _, yd = _device(y)
    orders = (0, 2, 5)
    ref = eng.fit_select_ar(yd, N_HOLD, orders, t_fit, 28)
    wide = torch.full((n, 41), float(np.float32(PATTERN)), device="cuda")
    view = wide[:, 5:33]
    import ctypes
    cand = (ctypes.c_int32 * 3)(*orders)
    rc = lib.mmf_fit_select_ar_f32(h, yd.data_ptr(), n, yd.stride(0), N_HOLD, cand, 3, t_fit, 28, view.data_ptr(), 41,
                                   None, None, None, None, None, None, None, None)
    assert rc == 0
    torch.cuda.synchronize()
    assert _same_bits(view, ref["pred"])
    assert (wide[:, :5] == float(np.float32(PATTERN))).all() and (wide[:, 33:] == float(np.float32(PATTERN))).all()
    ch = torch.full((n,), 7, device="cuda", dtype=torch.int32)
    rc = lib.mmf_fit_select_ar_f32(h, yd.data_ptr(), n, yd.stride(0), N_HOLD, cand, 3, t_fit, 28, view.data_ptr(), 41,
                                   ch.data_ptr(), None, None, None, None, None, None, None)
    assert rc == 0
    torch.cuda.synchronize()
    assert _same_bits(ch, ref["choice"]) and _same_bits(view, ref["pred"])
    eng.close()


def test_refused_arguments_write_nothing():
    import ctypes
    y, X, t_fit, has_c = _case("daily", n=40)
    n = len(y)
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    lib, h = eng._lib, eng._h
    _, yd = _device(y)
    ld = yd.stride(0)
    bufs = [torch.full((n, 28), 7.0, device="cuda"), torch.full((n,), 7, device="cuda", dtype=torch.int32),
            torch.full((n,), 7.0, device="cuda"), torch.full((n, 9), 7.0, device="cuda"),
            torch.full((n, AR_MAX), 7.0, device="cuda"), torch.full((n,), 7, device="cuda", dtype=torch.int32),
            torch.full((n,), 7.0, device="cuda"), torch.full((n,), 7, device="cuda", dtype=torch.int32)]
    host_out = np.zeros((n, 28), dtype=np.float32)

    def call(orders, n_hold=N_HOLD, ps=t_fit, npred=28, optr=None, ldo=28, ld_y=ld, ctx=h):
        c = (ctypes.c_int32 * max(len(orders), 1))(*orders) if orders is not None else None
        return lib.mmf_fit_select_ar_f32(ctx, yd.data_ptr(), n, ld_y, n_hold, c, len(orders or ()), ps, npred,
                                         bufs[0].data_ptr() if optr is None else optr, ldo,
                                         *[b.data_ptr() for b in bufs[1:]], None)
    refused = [dict(orders=()), dict(orders=None), dict(orders=(2, 1)), dict(orders=(1, 1)), dict(orders=(0, 9)),
               dict(orders=(-1, 2)), dict(orders=tuple(range(9)) + (8,)), dict(orders=(1,), n_hold=0),
               dict(orders=(1,), n_hold=X.shape[0] - t_fit + 1), dict(orders=(1,), ld_y=t_fit + N_HOLD - 1),
               dict(orders=(1,), ps=-1), dict(orders=(1,), npred=X.shape[0] + 1), dict(orders=(1,), ldo=27),
               dict(orders=(1,), optr=host_out.ctypes.data), dict(orders=(1,), ctx=None)]
    for kw in refused:
        assert call(**kw) != 0, kw
    torch.cuda.synchronize()
    assert all((b == 7).all() for b in bufs)
    assert not host_out.any()
    eng.close()


def test_slabs_are_bit_equal_to_per_slab_calls():
    n, t = (1 << 20) + 1001, 48
    y, start = mmf.synth.daily_store_item_demand(n, t + 8, seed=9, nan_frac=0.01)
    X = O.design_matrix(O.calendar_grid(start, t + 8, "D"), t)
    eng = mmf.ForecastEngine()
    eng.plan(X, t, True)
    yd = torch.from_numpy(y).cuda()
    whole = eng.fit_select_ar(yd, 8, (0, 1, 2), 0, t + 8)
    for lo, hi in ((0, 1 << 19), (1 << 19, n)):
        part = eng.fit_select_ar(yd[lo:hi], 8, (0, 1, 2), 0, t + 8)
        for k in whole:
            assert _same_bits(whole[k][lo:hi], part[k]), k
    eng.close()


def test_exact_power_of_two_scaling():
    y, X, t_fit, has_c = _case("daily")
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    _, yd = _device(y)
    a = _np(eng.fit_select_ar(yd, N_HOLD, (0, 1, 2, 3, 4), t_fit, 28))
    b = _np(eng.fit_select_ar(yd * 8.0, N_HOLD, (0, 1, 2, 3, 4), t_fit, 28))
    for k, f in (("pred", 8.0), ("mse", 64.0), ("cand_mse", 64.0), ("phi", 1.0), ("sigma", 8.0), ("choice", 1),
                 ("order", 1), ("status", 1)):
        w = a[k] * f
        same = (b[k] == w) | (np.isnan(b[k]) & np.isnan(w))
        assert same.all(), (k, np.flatnonzero(~same.reshape(len(y), -1).any(axis=1))[:8])
    eng.close()


def test_long_hourly_series():
    """70,001 fit rows and 48 held-out rows: bounds x sqrt(t_fit / 1095); predictions bit-equal to the fixed-order call"""
    t, hold = 70001, 48
    s = np.arange(t + hold, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), (s - t / 2) / t, np.sin(2 * np.pi * s / 24), np.cos(2 * np.pi * s / 24)])
    rng = np.random.default_rng(4)
    n = 24
    noise = np.zeros((n, t + hold))
    eps = rng.normal(0, 3, (n, t + hold))
    for k in range(1, t + hold):
        noise[:, k] = 0.7 * noise[:, k - 1] + eps[:, k]
    y = (200 + 10 * X[:, 2] + noise).astype(np.float32)
    y[1, t - 3:t] = np.nan
    y[2, 1000:1400] = np.nan
    y[3, t + 5:t + 9] = np.nan
    eng = mmf.ForecastEngine()
    eng.plan(X, t, True)
    orders = (0, 1, 2, 3)
    yd = torch.from_numpy(y).cuda()
    got = _np(eng.fit_select_ar(yd, hold, orders, t, hold))
    for m in (1, 2, 3):
        r = _np(eng.fit_forecast_ar(yd, m, t, hold))
        rows = got["choice"] == m
        assert np.array_equal(_bits(got["pred"][rows]), _bits(r["pred"][rows])), m
    want = select_ar_packed(y, X, t, hold, orders, t, hold)
    sc = np.sqrt(t / 1095)
    lev = forecast_leverage(X, t, t, hold)
    b = mse_bound(want, y, _row_tol(y[:, :t]) * sc, _row_tol(y[:, :t], lev) * sc, t, hold, orders)
    _le(float(np.nanmax(np.abs(got["cand_mse"] - want["cand_mse"]) / b)), 1.0, "hourly 70,001: |dMSE| / scaled bound")
    eng.close()


def test_other_calls_unchanged_by_a_selection_call():
    y, X, t_fit, has_c = _case("daily")
    start = np.datetime64("2019-01-01", "D")
    eng = mmf.ForecastEngine()
    eng.plan_calendars([start, start + 30], [t_fit, t_fit - 30], "D", 28)
    eng.plan_backtest(start, t_fit, "D", 28, 3)
    eng.plan(X, t_fit, has_c)
    _, yd = _device(y)
    yf = yd[:, :t_fit]

    def calls():
        bt = eng.backtest(yf)
        ar = eng.fit_forecast_ar(yd, 3, t_fit, 28)
        return (eng.fit_forecast(yf, t_fit, 28).clone(), eng.fit_forecast(yf, 0, t_fit + 64).clone(),
                eng.fit_forecast_ragged(yf, [0, 70, len(y)]).clone(), bt["pred"].clone(), bt["metrics"].clone(),
                bt["status"].clone(), ar["pred"].clone(), ar["phi"].clone())

    before = calls()
    eng.fit_select_ar(yd, N_HOLD, tuple(range(9)), 0, t_fit + 64)
    eng.fit_select_ar(yd, N_HOLD, (0, 1, 2), t_fit, 28)
    after = calls()
    assert all(_same_bits(a, b) for a, b in zip(before, after))
    eng.close()


_NEGCTL = """
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np, torch
import test_gpu_ar_select as T
from ar_select_oracle import select_ar_packed, mse_bound
from conftest import forecast_leverage
from test_gpu_edges import _row_tol
import mmf
y, X, t_fit, has_c = T._case("daily", n=96, seed=12, phi=0.9)
orders = (0, 1, 2, 3, 4)
eng = mmf.ForecastEngine()
eng.plan(X, t_fit, has_c)
got = T._np(eng.fit_select_ar(torch.from_numpy(y).cuda(), T.N_HOLD, orders, t_fit, T.N_HOLD))
want = select_ar_packed(y, X, t_fit, T.N_HOLD, orders, t_fit, T.N_HOLD)
lev = forecast_leverage(X, t_fit, t_fit, T.N_HOLD)
b = mse_bound(want, y, _row_tol(y[:, :t_fit]), _row_tol(y[:, :t_fit], lev), t_fit, T.N_HOLD, orders)
r = np.abs(got["cand_mse"] - want["cand_mse"]) / b
print(json.dumps({{"worst": float(r.max()), "over": [int((r[:, j] > 1).sum()) for j in range(len(orders))],
                   "rows": len(y), "lib": mmf.LIB_PATH}}))
"""


@pytest.mark.parametrize("lib", ["product", "onestep"])
def test_negative_control_one_step_score(lib):
    """the build that feeds observed held-out residuals into the candidates' histories
    (tests/_build/libmmf_arsel_onestep.so) must exceed mse_bound on at least half of the rows for every order >= 1;
    the product library stays within it"""
    env = dict(os.environ)
    env.pop("MMF_LIB", None)
    if lib == "onestep":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_arsel_onestep.so")
        assert os.path.exists(env["MMF_LIB"]), "negative-control library missing: run __graft_entry__.build()"
    r = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    record_err("test_negative_control_one_step_score", got["worst"], 1.0, what=lib, over=got["over"])
    if lib == "product":
        assert got["worst"] <= 1.0, got
    else:
        assert got["lib"].endswith("libmmf_arsel_onestep.so"), got
        assert all(o >= got["rows"] // 2 for o in got["over"][1:]), got


@pytest.mark.parametrize("frame", ["daily", "weekly"])
def test_forecast_groups_with_order_selection(frame):
    import pandas as pd
    orders = (0, 1, 2, 3, 4)
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
    out = mmf.forecast_groups(pdf, ar=orders, **kw)
    plain = mmf.forecast_groups(pdf, **kw)
    assert list(out.columns) == list(plain.columns) and len(out) == len(plain)
    worst, ambiguous = 0.0, 0
    for (key, g) in out.groupby(["Product", "SKU"], sort=True):
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
        want = select_ar_packed(y, X, t_fit, h, orders, 0, t_len)
        lev_h = forecast_leverage(X, t_fit, t_fit, h)
        tf = _row_tol(y[:, :t_fit]) * _mask_factor(y[:, :t_fit], X, t_fit, 0, t_fit, np.ones(1))
        mb = mse_bound(want, y, tf, _row_tol(y[:, :t_fit], lev_h) * _mask_factor(y[:, :t_fit], X, t_fit, t_fit, h,
                                                                                 np.ones(1)), t_fit, h, orders)[0]
        cm, oi = want["cand_mse"][0], int(want["idx"][0])
        rivals = [j for j in range(len(orders)) if j != oi and cm[j] <= cm[oi] + mb[j] + mb[oi]]
        if rivals:                                       # two candidates within the bounds: either may win
            ambiguous += 1
            continue
        m = orders[oi]
        r = want["final"][m]
        lev = forecast_leverage(X, t_fit, 0, t_len)
        tp = _row_tol(y[:, :t_fit], lev) * _mask_factor(y[:, :t_fit], X, t_fit, 0, t_len, np.ones(1))
        b = ar_bound(r, tf, tp, t_fit, 0, t_len) if m >= 1 else np.repeat(tp[:, None], t_len, axis=1)
        got = g["Demand_Fitted"].to_numpy().astype(np.float64)
        worst = max(worst, float((np.abs(got - want["pred"][0]) / b[0]).max()))
    record_err("ar_select_frames_ambiguous_groups", float(ambiguous), float(out.groupby(["Product", "SKU"]).ngroups),
               what=frame)
    _le(worst, 1.0, f"forecast_groups(ar={orders}) {frame}: error / bound")
