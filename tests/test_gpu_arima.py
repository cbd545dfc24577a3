"""GPU (-m gpu): regression with ARIMA(p, d, 0) errors (mmf_plan_arima + mmf_fit_forecast_arima_f32, DESIGN.md section 2
item 11).

Two yardsticks:
  - existing code: z' formed in fp32 and D_d planned with mmf_plan_design (the oracle's float64 differencing and residue
    rule) give, through mmf_fit_forecast_ar_f32(p) (p = 0: mmf_fit_select_ar_f32 with orders (0,)) under the same forced
    kernel, phi / order / sigma / status bit-equal to the ARIMA call's, and predictions whose fp32 integration in the
    order include/mmf.h states is bit-equal to the ARIMA call's predictions;
  - the float64 oracle of tests/arima_oracle.py: predictions within arima_bound (x the mask factor), statuses equal,
    orders exact outside the kappa margin, phi / sigma within ar_oracle.coef_bounds.
Every batch carries test_gpu_ar.py's row mix plus rows with alternate values missing (z' empty), y_0 or y_1 missing and
gaps exactly at t_fit - 1 and t_fit - 2."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mmf
from ar_oracle import AR_MAX, coef_bounds, kappa_margin
from arima_oracle import arima_bound, diff_design, fit_forecast_arima_packed, z_tau
from conftest import ROOT, forecast_leverage, record_err
from oracle import mmf_oracle as O
from test_gpu_abi_contract import PATTERN, _mask_factor
from test_gpu_ar import AR_KINDS, KAPPA_MARGIN, _ar_cols, _ratio
from test_gpu_edges import _le, _same_bits

pytestmark = pytest.mark.gpu

ARIMA_KINDS = AR_KINDS + ("alternate", "first0", "first1", "origin2only")


def _cols(kind, t_fit):
    c = np.arange(t_fit)
    if kind == "alternate":
        return c[1::2]
    if kind == "first0":
        return np.array([0])
    if kind == "first1":
        return np.array([1])
    if kind == "origin2only":
        return np.array([t_fit - 2])
    return _ar_cols(kind, t_fit)


def _plant(y, t_fit):
    for i in range(y.shape[0]):
        kind = ARIMA_KINDS[i % len(ARIMA_KINDS)]
        y[i, _cols(kind, t_fit)] = np.inf if kind == "inf" else np.nan
    return y


def _case(cal, n=170, seed=5):
    """(y [n, t_fit] float32 with the row mix, X [n_rows, p], t_fit, has_constant): a regression on X plus an integrated
    AR(1) error with drift, so the levels wander"""
    rng = np.random.default_rng(seed)
    if cal == "daily":
        t, n_rows = 400, 464
        X = O.design_matrix(O.calendar_grid("2019-01-01", n_rows, "D"), t)
    elif cal == "weekly":                                            # the reference's 157 / 117 / 40 weeks
        t, n_rows = 117, 157
        X = O.design_matrix(O.calendar_grid("2018-01-01", n_rows, "W-MON"), t)
    elif cal == "exog_only":
        t, n_rows = 300, 364
        X = O.design_matrix(O.calendar_grid("2019-06-03", n_rows, "D"), t, "exog_only")
    else:                                                            # a caller design with a constant, 5 columns
        t, n_rows = 250, 314
        s = np.arange(n_rows, dtype=np.float64)
        X = np.column_stack([np.ones_like(s), (s - t / 2) / t, np.sqrt(s / t), np.sin(2 * np.pi * s / 30.5),
                             np.cos(2 * np.pi * s / 30.5)])
    has_c = cal != "exog_only"
    beta = rng.normal(0, 20, (n, X.shape[1]))
    phi = rng.uniform(0.1, 0.8, n)
    w = np.zeros((n, t))
    eps = rng.normal(0, 4, (n, t))
    for k in range(t):
        w[:, k] = eps[:, k] + (phi * w[:, k - 1] if k else 0)
    y = 500.0 + beta @ X[:t].T + np.cumsum(w + rng.normal(0, 0.5, (n, 1)), axis=1)
    return _plant(y.astype(np.float32), t), X, t, has_c


def _windows(t_fit, n_rows):
    return {"future": (t_fit, min(64, n_rows - t_fit)), "holdout": (0, n_rows), "mid": (t_fit // 3, t_fit // 2 + 40)}


def _dev(y, cols=None):
    """y on the device with a 16-B row pitch (the tensor-core kernel); `cols` columns, NaN beyond y's"""
    n, t = y.shape
    cols = t if cols is None else cols
    full = torch.full((n, (cols + 3) & ~3), float("nan"), device="cuda")
    full[:, :t] = torch.from_numpy(np.ascontiguousarray(y, dtype=np.float32)).cuda()
    return full[:, :cols]


def _np(r):
    return {k: v.cpu().numpy() for k, v in r.items() if k != "stats"}


def _z32(y, d):
    """z' in fp32, in the order the library forms it"""
    y = np.asarray(y, dtype=np.float32)
    return y[:, 1:] - y[:, :-1] if d == 1 else (y[:, 2:] - y[:, 1:-1]) - (y[:, 1:-1] - y[:, :-2])


def _integrate32(zh, y, t_fit, d, end):
    """fp32 levels from zhat at z' rows [0, end - d): the order include/mmf.h states, row t = z' row t - d"""
    n = y.shape[0]
    yt = np.full((n, end), np.nan, dtype=np.float32)
    yh = np.full((n, end), np.nan, dtype=np.float32)
    two = np.float32(2.0)
    for t in range(end):
        if t >= d:
            z = zh[:, t - d].astype(np.float32)
            yh[:, t] = z + yt[:, t - 1] if d == 1 else (z + two * yt[:, t - 1]) - yt[:, t - 2]
        if t < t_fit:
            yt[:, t] = np.where(np.isfinite(y[:, t]), y[:, t], yh[:, t])
        else:
            yt[:, t] = yh[:, t]
    return yh


def _anchor(kernel, y, X, t_fit, p, d, ps, npred, got):
    """the ARIMA call's results against mmf_fit_forecast_ar_f32 / mmf_fit_select_ar_f32 on z' and D_d (bit for bit)"""
    end = ps + npred
    D = diff_design(X, t_fit, d)
    tz = t_fit - d
    eng = mmf.ForecastEngine(kernel=kernel)
    eng.plan(D, tz, False)
    zd = _dev(_z32(y[:, :t_fit], d), tz + 1)                        # one NaN held-out column for the p = 0 call
    nz = end - d
    if p >= 1:
        ref = _np(eng.fit_forecast_ar(zd[:, :tz], p, 0, nz))
    else:
        ref = _np(eng.fit_select_ar(zd, 1, (0,), 0, nz))
    eng.close()
    for k in ("phi", "order", "sigma", "status"):
        a, b = np.ascontiguousarray(got[k]), np.ascontiguousarray(ref[k])
        assert a.tobytes() == b.tobytes(), (kernel, p, d, k, np.flatnonzero((a != b).reshape(len(a), -1).any(1))[:6])
    lv = _integrate32(ref["pred"], y, t_fit, d, end)[:, ps:end]
    ok = (lv.view(np.uint32) == got["pred"].view(np.uint32)) | (np.isnan(lv) & np.isnan(got["pred"]))
    bad = np.flatnonzero(~ok.all(axis=1))
    assert bad.size == 0, (kernel, p, d, ps, npred, bad[:6], [ARIMA_KINDS[i % len(ARIMA_KINDS)] for i in bad[:6]])


def _compare(got, want, t_fit, ps, npred, what):
    """statuses equal, orders exact outside the kappa margin, predictions within arima_bound x the mask factor, phi and
    sigma within coef_bounds; returns the worst ratio"""
    d = want["d"]
    st = want["status"]
    assert np.array_equal(got["status"], st), what
    zr = want["zres"]
    near = kappa_margin(zr) < KAPPA_MARGIN
    live = (st != 1) & ~near
    bad = np.flatnonzero(live & (got["order"] != want["order"]))
    assert bad.size == 0, (what, bad[:8], got["order"][bad[:8]], want["order"][bad[:8]])
    assert np.isnan(got["pred"][st == 1]).all() and np.isnan(got["sigma"][st == 1]).all(), what
    assert (got["order"][st == 1] == 0).all() and not got["phi"][st == 1].any(), what
    end = ps + npred
    tz, nz = t_fit - d, max(end - d, 1)
    z, D = want["z"], want["D"]
    lev = forecast_leverage(D, tz, 0, nz)
    ones = np.ones(len(z))
    mf_fit = _mask_factor(z, D, tz, 0, tz, ones)
    mf_pred = _mask_factor(z, D, tz, 0, nz, ones)
    tau_fit = np.where(np.isfinite(mf_fit), z_tau(want) * mf_fit, 0.0)
    tau_pred = np.where(np.isfinite(mf_pred), z_tau(want, lev) * mf_pred, 0.0)
    bound = arima_bound(want, tau_fit, tau_pred, t_fit, ps, npred)
    wp, gp = want["pred"][live], got["pred"][live].astype(np.float64)
    assert np.array_equal(np.isnan(wp), np.isnan(gp)), what
    fin = np.isfinite(wp)
    err = _ratio(np.abs(np.where(fin, gp - wp, 0.0)), np.where(fin, bound[live], 1.0))
    worst = float(err.max()) if err.size else 0.0
    _le(worst, 1.0, f"{what}: prediction error / arima_bound")
    dphi, dsig = coef_bounds(zr, tau_fit)
    pos = live & (want["order"] > 0)
    e_phi = _ratio(np.abs(got["phi"][pos].astype(np.float64) - want["phi"][pos]).sum(axis=1), dphi[pos])
    w_phi = float(e_phi.max()) if e_phi.size else 0.0
    _le(w_phi, 1.0, f"{what}: |dphi|_1 / coef_bounds")
    e_sig = _ratio(np.abs(got["sigma"][live].astype(np.float64) - want["sigma"][live]), dsig[live])
    w_sig = float(e_sig.max()) if e_sig.size else 0.0
    _le(w_sig, 1.0, f"{what}: |dsigma| / coef_bounds")
    return max(worst, w_phi, w_sig)


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("p", [0, 1, 2, 8])
@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_arima_matches_existing_code_and_the_oracle(cal, p, d):
    y, X, t_fit, has_c = _case(cal)
    engs = {k: mmf.ForecastEngine(kernel=k) for k in ("auto", "tc", "warp")}
    for e in engs.values():
        e.plan_arima(X, t_fit, 2)
    yd = _dev(y)
    worst = 0.0
    for name, (ps, npred) in _windows(t_fit, X.shape[0]).items():
        want = fit_forecast_arima_packed(y, X, t_fit, ps, npred, p, d)
        for k, eng in engs.items():
            got = _np(eng.fit_forecast_arima(yd, p, d, ps, npred))
            _anchor(k, y, X, t_fit, p, d, ps, npred, got)
            worst = max(worst, _compare(got, want, t_fit, ps, npred, f"{cal} p={p} d={d} {name} {k}"))
    for e in engs.values():
        e.close()
    record_err("test_arima_matches_existing_code_and_the_oracle", worst, 1.0, what=f"{cal} p={p} d={d}")


def test_y_at_and_beyond_t_fit_is_never_read():
    y, X, t_fit, _ = _case("daily")
    eng = mmf.ForecastEngine()
    eng.plan_arima(X, t_fit, 2)
    base = _dev(y, t_fit + 40)
    ref = {d: _np(eng.fit_forecast_arima(base[:, :t_fit], 2, d, 0, X.shape[0])) for d in (1, 2)}
    for fill in (float("nan"), 1e30, -7.0):
        yd = _dev(y, t_fit + 40)
        yd[:, t_fit:] = fill
        for d in (1, 2):
            got = _np(eng.fit_forecast_arima(yd, 2, d, 0, X.shape[0]))
            for k in ref[d]:
                assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(ref[d][k]).tobytes(), (fill, d, k)
    eng.close()


def test_exact_power_of_two_scaling():
    y, X, t_fit, _ = _case("daily")
    eng = mmf.ForecastEngine()
    eng.plan_arima(X, t_fit, 2)
    yd = _dev(y)
    for d in (1, 2):
        a = _np(eng.fit_forecast_arima(yd, 3, d, t_fit, 28))
        b = _np(eng.fit_forecast_arima(yd * 8.0, 3, d, t_fit, 28))
        for k, f in (("pred", 8.0), ("phi", 1.0), ("order", 1), ("sigma", 8.0), ("status", 1)):
            w = a[k] * f
            same = (b[k] == w) | (np.isnan(b[k]) & np.isnan(w))
            assert same.all(), (d, k, np.flatnonzero(~same.reshape(len(y), -1).all(axis=1))[:6])
    eng.close()


def test_slabs_are_bit_equal_to_per_slab_calls():
    n, t = (1 << 20) + 1001, 48
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=9, nan_frac=0.01)
    X = O.design_matrix(O.calendar_grid(start, t + 8, "D"), t)
    eng = mmf.ForecastEngine()
    eng.plan_arima(X, t, 2)
    yd = torch.from_numpy(y).cuda()
    for d in (1, 2):
        whole = eng.fit_forecast_arima(yd, 2, d, t, 8)
        for lo, hi in ((0, 1 << 19), (1 << 19, n)):
            part = eng.fit_forecast_arima(yd[lo:hi], 2, d, t, 8)
            for k in ("pred", "phi", "order", "sigma", "status"):
                assert _same_bits(whole[k][lo:hi], part[k]), (d, k)
    eng.close()


def test_long_hourly_series():
    """70,001 fit rows: bounds x sqrt(t_fit / 1095)"""
    t = 70001
    s = np.arange(t + 48, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), (s - t / 2) / t, np.sin(2 * np.pi * s / 24), np.cos(2 * np.pi * s / 24)])
    rng = np.random.default_rng(4)
    n = 24
    w = np.zeros((n, t))
    eps = rng.normal(0, 3, (n, t))
    for k in range(1, t):
        w[:, k] = 0.6 * w[:, k - 1] + eps[:, k]
    y = (2000 + 10 * X[:t, 2] + np.cumsum(w, axis=1) / 20).astype(np.float32)
    y[1, t - 3:] = np.nan
    y[2, 1000:1400] = np.nan
    eng = mmf.ForecastEngine()
    eng.plan_arima(X, t, 2)
    sc = np.sqrt(t / 1095)
    for d in (1, 2):
        got = _np(eng.fit_forecast_arima(_dev(y), 2, d, t, 48))
        want = fit_forecast_arima_packed(y, X, t, t, 48, 2, d)
        lev = forecast_leverage(want["D"], t - d, 0, t + 48 - d)
        bound = arima_bound(want, z_tau(want) * sc, z_tau(want, lev) * sc, t, t, 48)
        assert np.array_equal(got["order"], want["order"]) and np.array_equal(got["status"], want["status"])
        _le(float((np.abs(got["pred"] - want["pred"]) / bound).max()), 1.0, f"hourly 70,001 d={d}: error / bound")
    eng.close()


def test_nullable_outputs_and_a_wide_table():
    y, X, t_fit, _ = _case("daily")
    n = len(y)
    eng = mmf.ForecastEngine()
    eng.plan_arima(X, t_fit, 2)
    lib, h = eng._lib, eng._h
    yd = _dev(y)
    ref = eng.fit_forecast_arima(yd, 2, 1, t_fit, 28)
    wide = torch.full((n, 41), float(np.float32(PATTERN)), device="cuda")
    view = wide[:, 5:33]                                           # any base pointer, ld_out = 41
    rc = lib.mmf_fit_forecast_arima_f32(h, yd.data_ptr(), n, yd.stride(0), 2, 1, t_fit, 28, view.data_ptr(), 41,
                                        None, None, None, None, None)
    assert rc == 0
    torch.cuda.synchronize()
    assert _same_bits(view, ref["pred"])
    assert (wide[:, :5] == float(np.float32(PATTERN))).all() and (wide[:, 33:] == float(np.float32(PATTERN))).all()
    eng.close()


def test_refused_plans_and_calls_write_nothing_and_keep_the_plan():
    y, X, t_fit, _ = _case("daily", n=40)
    n = len(y)
    eng = mmf.ForecastEngine()
    lib, h = eng._lib, eng._h
    yd = _dev(y)
    out = torch.full((n, 28), 7.0, device="cuda")
    assert lib.mmf_fit_forecast_arima_f32(h, yd.data_ptr(), n, yd.stride(0), 1, 1, t_fit, 28, out.data_ptr(), 28,
                                          None, None, None, None, None) == -4          # MMF_E_NOPLAN
    eng.plan_arima(X, t_fit, 1)
    ref = _np(eng.fit_forecast_arima(yd, 2, 1, t_fit, 28))
    Xc = np.ascontiguousarray(X)
    Xbad = Xc.copy()
    Xbad[3, 2] = np.nan
    for args in ((Xc.ctypes.data, X.shape[0], X.shape[1], t_fit, 0), (Xc.ctypes.data, X.shape[0], X.shape[1], t_fit, 3),
                 (Xc.ctypes.data, X.shape[0], 17, t_fit, 1), (Xc.ctypes.data, X.shape[0], X.shape[1], 2, 2),
                 (Xc.ctypes.data, t_fit - 1, X.shape[1], t_fit, 1), (Xbad.ctypes.data, X.shape[0], X.shape[1], t_fit, 2),
                 (None, X.shape[0], X.shape[1], t_fit, 1)):
        assert lib.mmf_plan_arima(h, *args) != 0, args
    phi = torch.full((n, AR_MAX), 7.0, device="cuda")
    order = torch.full((n,), 7, device="cuda", dtype=torch.int32)
    sig = torch.full((n,), 7.0, device="cuda")
    status = torch.full((n,), 7, device="cuda", dtype=torch.int32)
    host_out = np.zeros((n, 28), dtype=np.float32)
    calls = [(-1, 1, t_fit, 28, out.data_ptr(), 28), (9, 1, t_fit, 28, out.data_ptr(), 28),
             (2, 0, t_fit, 28, out.data_ptr(), 28), (2, 2, t_fit, 28, out.data_ptr(), 28),      # max_diff is 1
             (2, 1, -1, 28, out.data_ptr(), 28), (2, 1, t_fit, 65, out.data_ptr(), 65),
             (2, 1, t_fit, 28, out.data_ptr(), 27), (2, 1, t_fit, 28, None, 28),
             (2, 1, t_fit, 28, host_out.ctypes.data, 28)]
    for p, d, ps, npred, optr, ld in calls:
        rc = lib.mmf_fit_forecast_arima_f32(h, yd.data_ptr(), n, yd.stride(0), p, d, ps, npred, optr, ld,
                                            phi.data_ptr(), order.data_ptr(), sig.data_ptr(), status.data_ptr(), None)
        assert rc != 0, (p, d, ps, npred, ld)
    assert lib.mmf_fit_forecast_arima_f32(h, yd.data_ptr(), n, t_fit - 1, 2, 1, t_fit, 28, out.data_ptr(), 28,
                                          None, None, None, None, None) != 0             # ld_y < t_fit
    torch.cuda.synchronize()
    assert (out == 7).all() and (phi == 7).all() and (order == 7).all() and (sig == 7).all() and (status == 7).all()
    assert not host_out.any()
    got = _np(eng.fit_forecast_arima(yd, 2, 1, t_fit, 28))                 # the refused plans kept the previous one
    for k in ref:
        assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(ref[k]).tobytes(), k
    eng.close()


def test_other_calls_unchanged_and_a_shared_context_matches_a_fresh_one():
    """plain, AR, selection, ragged and backtest calls give the same bits before and after an ARIMA plan and call on one
    context; an ARIMA call on that context is bit-equal to the same call on a fresh context"""
    y, X, t_fit, has_c = _case("daily")
    start = np.datetime64("2019-01-01", "D")
    eng = mmf.ForecastEngine()
    eng.plan_calendars([start, start + 30], [t_fit, t_fit - 30], "D", 28)
    eng.plan_backtest(start, t_fit, "D", 28, 3)
    eng.plan(X, t_fit, has_c)
    yd = _dev(y, t_fit + 28)
    yf = yd[:, :t_fit]

    def calls():
        bt = eng.backtest(yf)
        return (eng.fit_forecast(yf, t_fit, 28).clone(), eng.fit_forecast(yf, 0, t_fit + 64).clone(),
                eng.fit_forecast_ar(yf, 2, t_fit, 28)["pred"].clone(), eng.fit_select_ar(yd, 28, (0, 1, 2))["pred"].clone(),
                eng.fit_forecast_ragged(yf, [0, 70, len(y)]).clone(), bt["pred"].clone(), bt["metrics"].clone(),
                bt["status"].clone())

    before = calls()
    eng.plan_arima(X, t_fit, 2)
    shared = [_np(eng.fit_forecast_arima(yf, p, d, ps, npred))
              for p, d, ps, npred in ((2, 1, t_fit, 28), (0, 2, 0, t_fit + 64), (8, 2, t_fit, 64))]
    after = calls()
    assert all(_same_bits(a, b) for a, b in zip(before, after))
    fresh_eng = mmf.ForecastEngine()
    fresh_eng.plan_arima(X, t_fit, 2)
    fresh = [_np(fresh_eng.fit_forecast_arima(yf, p, d, ps, npred))
             for p, d, ps, npred in ((2, 1, t_fit, 28), (0, 2, 0, t_fit + 64), (8, 2, t_fit, 64))]
    for a, b in zip(shared, fresh):
        for k in a:
            assert np.ascontiguousarray(a[k]).tobytes() == np.ascontiguousarray(b[k]).tobytes(), k
    eng.close()
    fresh_eng.close()


_NEGCTL = """
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np, torch
import test_gpu_arima as T
from arima_oracle import fit_forecast_arima_packed, arima_bound, z_tau
from conftest import forecast_leverage
import mmf
from oracle import mmf_oracle as O
n, t, h = 400, 400, 28
rng = np.random.default_rng(8)
X = O.design_matrix(O.calendar_grid("2019-01-01", t + h, "D"), t)
w = np.zeros((n, t))
eps = rng.normal(0, 5, (n, t))
for k in range(t):
    w[:, k] = eps[:, k] + (0.9 * w[:, k - 1] if k else 0)
y = (1000 + np.cumsum(w + 2.0, axis=1)).astype(np.float32)
rows = np.arange(0, n, 2)
for i in rows:
    y[i, t - 1 - (i // 2) % 4:t] = np.nan                     # gaps at t_fit - 1 .. t_fit - 4
eng = mmf.ForecastEngine()
eng.plan_arima(X, t, 1)
got = T._np(eng.fit_forecast_arima(T._dev(y), 1, 1, t, h))
want = fit_forecast_arima_packed(y, X, t, t, h, 1, 1)
lev = forecast_leverage(want["D"], t - 1, 0, t + h - 1)
b = arima_bound(want, z_tau(want), z_tau(want, lev), t, t, h)
r = (np.abs(got["pred"] - want["pred"]) / b)[rows].max(axis=1)
print(json.dumps({{"worst": float(r.max()), "rows_over": int((r > 1).sum()), "rows": len(rows), "lib": mmf.LIB_PATH}}))
"""


@pytest.mark.parametrize("lib", ["product", "nolevelfill"])
def test_negative_control_without_the_level_fill(lib):
    """random walks with drift whose differences are AR(1) with phi = 0.9, gaps at t_fit - 1 .. t_fit - 4: the build that
    takes a missing fit value's level as the last observed level (tests/_build/libmmf_arima_nolevelfill.so) must exceed
    the bound on at least half of those rows; the product library stays within it"""
    env = dict(os.environ)
    env.pop("MMF_LIB", None)
    if lib == "nolevelfill":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_arima_nolevelfill.so")
        assert os.path.exists(env["MMF_LIB"]), "negative-control library missing: run __graft_entry__.build()"
    r = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    record_err("test_negative_control_without_the_level_fill", got["worst"], 1.0, what=lib, rows_over=got["rows_over"],
               rows=got["rows"])
    if lib == "product":
        assert got["worst"] <= 1.0, got
    else:
        assert got["lib"].endswith("libmmf_arima_nolevelfill.so") and got["rows_over"] >= got["rows"] // 2, got


@pytest.mark.parametrize("frame", ["daily", "weekly"])
def test_forecast_groups_with_arima(frame):
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
        kw = dict(freq="D", horizon=28, mode="future")
        f = "D"
    out = mmf.forecast_groups(pdf, ar=2, diff=1, **kw)
    plain = mmf.forecast_groups(pdf, **kw)
    assert list(out.columns) == list(plain.columns) and len(out) == len(plain)
    worst = 0.0
    for key, g in out.groupby(["Product", "SKU"], sort=True):
        src = pdf[(pdf["Product"] == key[0]) & (pdf["SKU"] == key[1])].sort_values("Date")
        d0, d1 = np.datetime64(src["Date"].min(), "D"), np.datetime64(src["Date"].max(), "D")
        step = O.FREQ_DAYS[f]
        t_len = int((d1 - d0).astype(int) // step + 1)
        y = np.full((1, t_len), np.nan)
        pos = ((src["Date"].to_numpy().astype("datetime64[D]") - d0).astype(int) // step)
        y[0, pos] = src["Demand"].to_numpy()
        if kw["mode"] == "holdout":
            t_fit, ps, npred = t_len - kw["horizon"], 0, t_len
            X = O.design_matrix(O.calendar_grid(d0, t_len, f), t_fit)
        else:
            t_fit, ps, npred = t_len, t_len, kw["horizon"]
            X = O.design_matrix(O.calendar_grid(d0, t_len + npred, f), t_fit)
        want = fit_forecast_arima_packed(y, X, t_fit, ps, npred, 2, 1)
        D = want["D"]
        nz = ps + npred - 1
        lev = forecast_leverage(D, t_fit - 1, 0, nz)
        ones = np.ones(1)
        b = arima_bound(want, z_tau(want) * _mask_factor(want["z"], D, t_fit - 1, 0, t_fit - 1, ones),
                        z_tau(want, lev) * _mask_factor(want["z"], D, t_fit - 1, 0, nz, ones), t_fit, ps, npred)
        got = g["Demand_Fitted"].to_numpy().astype(np.float64)
        assert np.array_equal(np.isnan(got), np.isnan(want["pred"][0])), key
        fin = np.isfinite(got)
        worst = max(worst, float((np.abs(got[fin] - want["pred"][0][fin]) / b[0][fin]).max()))
    _le(worst, 1.0, f"forecast_groups(ar=2, diff=1) {frame}: error / bound")
