"""GPU (-m gpu): regression with AR(p) errors (mmf_fit_forecast_ar_f32, DESIGN.md section 2 item 9) against the float64
oracle of tests/ar_oracle.py.

Every batch carries the row mix of test_gpu_abi_contract.py (gap-free, isolated gaps, leading gaps, 45 gaps in one chunk
parity, mostly missing, a single value, empty, +Inf) plus rows with gaps exactly at t_fit - 1 .. t_fit - 8 and a run of
20 missing values.  Statuses must equal the plain call's bit for bit; orders must equal the oracle's except on rows whose
oracle |kappa| lies within KAPPA_MARGIN of the limit (counted and logged); predictions must lie within the first-order
bound of ar_oracle.ar_bound, whose coefficient term bounds the error in phi that reaches them."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mmf
from ar_oracle import AR_MAX, ar_bound, coef_bounds, fit_forecast_ar_packed, kappa_margin
from conftest import ROOT, forecast_leverage, record_err
from oracle import mmf_oracle as O
from test_gpu_abi_contract import KINDS, PATTERN, _kind_cols, _mask_factor
from test_gpu_edges import _le, _row_tol, _same_bits

pytestmark = pytest.mark.gpu

AR_KINDS = KINDS + ("origin8", "origin1", "run20")
KAPPA_MARGIN = 1e-3


def _ar_cols(kind, t_fit):
    if kind == "origin8":
        return np.arange(t_fit - 8, t_fit)
    if kind == "origin1":
        return np.array([t_fit - 1])
    if kind == "run20":
        return np.arange(t_fit // 2, t_fit // 2 + 20)
    return _kind_cols(kind, t_fit)


def _plant(y, t_fit):
    for i in range(y.shape[0]):
        kind = AR_KINDS[i % len(AR_KINDS)]
        y[i, _ar_cols(kind, t_fit)] = np.inf if kind == "inf" else np.nan
    return y


def _case(cal, n=150, seed=3):
    """(y [n, t_fit] float32 with the row mix, X, t_fit, has_constant)"""
    if cal == "daily":
        t = 400
        y, start = mmf.synth.daily_store_item_demand(n, t, seed=seed)
        X = O.design_matrix(O.calendar_grid(start, t + 64, "D"), t)
        return _plant(y, t), X, t, True
    if cal == "weekly":
        t = 130
        rng = np.random.default_rng(seed)
        X = O.design_matrix(O.calendar_grid("2018-01-01", t + 64, "W-MON"), t)
    elif cal == "exog_only":
        t = 300
        rng = np.random.default_rng(seed)
        X = O.design_matrix(O.calendar_grid("2019-06-03", t + 64, "D"), t, "exog_only")
    else:                                                            # a caller design with a constant, 5 columns
        t = 250
        rng = np.random.default_rng(seed)
        s = np.arange(t + 64, dtype=np.float64)
        X = np.column_stack([np.ones_like(s), (s - t / 2) / t, np.sqrt(s / t), np.sin(2 * np.pi * s / 30.5),
                             np.cos(2 * np.pi * s / 30.5)])
    has_c = cal != "exog_only"
    beta = rng.normal(0, 20, (n, X.shape[1]))
    base = 100.0 + beta @ X[:t].T if has_c else 100.0 * (1 + X[:t, :3].sum(1)) + beta @ X[:t].T
    noise = np.zeros((n, t))
    phi = rng.uniform(0.1, 0.9, n)
    eps = rng.normal(0, 5, (n, t))
    for k in range(t):
        noise[:, k] = eps[:, k] + (phi * noise[:, k - 1] if k else 0)
    return _plant((base + noise).astype(np.float32), t), X, t, has_c


def _windows(t_fit, n_rows):
    return {"future": (t_fit, min(64, n_rows - t_fit)), "holdout": (0, n_rows), "mid": (t_fit // 3, t_fit // 2 + 40)}


def _run(eng, yd, p, ps, npred):
    r = eng.fit_forecast_ar(yd, p, ps, npred)
    return {k: v.cpu().numpy() for k, v in r.items()}


def _ratio(err, bound):
    """err / bound, with 0 where both are 0 (a bound of 0 then still requires an exact result)"""
    err, bound = np.asarray(err, dtype=np.float64), np.asarray(bound, dtype=np.float64)
    out = np.full(err.shape, np.inf)
    np.divide(err, bound, out=out, where=bound > 0)
    return np.where(err == 0, 0.0, out)


def _compare(got, want, y, X, t_fit, ps, npred, what):
    """orders exact outside the kappa margin; predictions within ar_bound, phi and sigma within coef_bounds (phi of
    order-0 rows exactly 0); returns the worst ratio of the three"""
    st = want["status"]
    near = kappa_margin(want) < KAPPA_MARGIN
    live = (st != 1) & ~near
    record_err("ar_near_limit_rows", float(near.sum()), float(len(st)), what=what)
    bad = np.flatnonzero(live & (got["order"] != want["order"]))
    assert bad.size == 0, (what, bad[:8], got["order"][bad[:8]], want["order"][bad[:8]])
    assert np.isnan(got["pred"][st == 1]).all() and np.isnan(got["sigma"][st == 1]).all(), what
    assert (got["order"][st == 1] == 0).all() and not got["phi"][st == 1].any(), what
    lev = forecast_leverage(X, t_fit, ps, npred)
    tau_fit = _row_tol(y[:, :t_fit]) * _mask_factor(y, X, t_fit, 0, t_fit, np.ones(len(y)))
    tau_pred = _row_tol(y[:, :t_fit], lev) * _mask_factor(y, X, t_fit, ps, npred, np.ones(len(y)))
    tau_fit = np.where(np.isfinite(tau_fit), tau_fit, 0)
    tau_pred = np.where(np.isfinite(tau_pred), tau_pred, 0)
    bound = ar_bound(want, tau_fit, tau_pred, t_fit, ps, npred)
    err = _ratio(np.abs(got["pred"][live].astype(np.float64) - want["pred"][live]), bound[live])
    worst = float(err.max()) if err.size else 0.0
    _le(worst, 1.0, f"{what}: prediction error / ar_bound")
    assert not got["phi"][live & (want["order"] == 0)].any(), what
    assert not got["phi"][live][np.arange(AR_MAX)[None, :] >= got["order"][live][:, None]].any(), what
    dphi, dsig = coef_bounds(want, tau_fit)
    pos = live & (want["order"] > 0)
    e_phi = _ratio(np.abs(got["phi"][pos].astype(np.float64) - want["phi"][pos]).sum(axis=1), dphi[pos])
    w_phi = float(e_phi.max()) if e_phi.size else 0.0
    _le(w_phi, 1.0, f"{what}: |dphi|_1 / coef_bounds")
    e_sig = _ratio(np.abs(got["sigma"][live].astype(np.float64) - want["sigma"][live]), dsig[live])
    w_sig = float(e_sig.max()) if e_sig.size else 0.0
    _le(w_sig, 1.0, f"{what}: |dsigma| / coef_bounds")
    return max(worst, w_phi, w_sig)


@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
@pytest.mark.parametrize("p", [1, 2, 4, 8])
def test_ar_matches_the_oracle(cal, p):
    y, X, t_fit, has_c = _case(cal)
    engs = {k: mmf.ForecastEngine(kernel=k) for k in ("auto", "tc", "warp")}
    worst = 0.0
    for name, (ps, npred) in _windows(t_fit, X.shape[0]).items():
        for k, eng in engs.items():
            eng.plan(X, t_fit, has_c)
        want = fit_forecast_ar_packed(y, X, t_fit, ps, npred, p)
        full = torch.zeros((len(y), (t_fit + 3) & ~3), device="cuda")     # 16-B row pitch: the tensor-core kernel
        full[:, :t_fit] = torch.from_numpy(y).cuda()
        yd = full[:, :t_fit]
        for k, eng in engs.items():
            got = _run(eng, yd, p, ps, npred)
            plain = eng.fit_forecast(yd, ps, npred, want_status=True)
            assert np.array_equal(got["status"], plain["status"].cpu().numpy()), (cal, p, name, k)
            worst = max(worst, _compare(got, want, y, X, t_fit, ps, npred, f"{cal} p={p} {name} {k}"))
    for e in engs.values():
        e.close()
    record_err("test_ar_matches_the_oracle", worst, 1.0, what=f"{cal} p={p}")


def test_exact_power_of_two_scaling():
    y, X, t_fit, has_c = _case("daily")
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    yd = torch.from_numpy(y).cuda()
    a = _run(eng, yd, 3, t_fit, 28)
    b = _run(eng, yd * 8.0, 3, t_fit, 28)
    diff = {}
    for k, f in (("pred", 8.0), ("phi", 1.0), ("order", 1), ("sigma", 8.0)):
        w = a[k] * f
        bad = ~((b[k] == w) | (np.isnan(b[k]) & np.isnan(w)))
        rows = np.flatnonzero(bad.reshape(len(y), -1).any(axis=1))
        diff[k] = [(int(i), AR_KINDS[i % len(AR_KINDS)]) for i in rows[:6]] + [len(rows)]
    assert all(v[-1] == 0 for v in diff.values()), diff
    eng.close()


def test_slabs_are_bit_equal_to_per_slab_calls():
    n, t = (1 << 20) + 1001, 48
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=9, nan_frac=0.01)
    X = O.design_matrix(O.calendar_grid(start, t + 8, "D"), t)
    eng = mmf.ForecastEngine()
    eng.plan(X, t, True)
    yd = torch.from_numpy(y).cuda()
    whole = eng.fit_forecast_ar(yd, 2, t, 8)
    for lo, hi in ((0, 1 << 19), (1 << 19, n)):
        part = eng.fit_forecast_ar(yd[lo:hi], 2, t, 8)
        for k in ("pred", "phi", "order", "sigma", "status"):
            assert _same_bits(whole[k][lo:hi], part[k]), k
    eng.close()


def test_long_hourly_series():
    """70,001 fit rows (the hourly grid of the ABI contract tests): bound x sqrt(t_fit / 1095)"""
    t = 70001
    s = np.arange(t + 48, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), (s - t / 2) / t, np.sin(2 * np.pi * s / 24), np.cos(2 * np.pi * s / 24)])
    rng = np.random.default_rng(4)
    n = 24
    noise = np.zeros((n, t))
    eps = rng.normal(0, 3, (n, t))
    for k in range(1, t):
        noise[:, k] = 0.7 * noise[:, k - 1] + eps[:, k]
    y = (200 + 10 * X[:t, 2] + noise).astype(np.float32)
    y[1, t - 3:] = np.nan
    y[2, 1000:1400] = np.nan
    eng = mmf.ForecastEngine()
    eng.plan(X, t, True)
    got = _run(eng, torch.from_numpy(y).cuda(), 2, t, 48)
    want = fit_forecast_ar_packed(y, X, t, t, 48, 2)
    lev = forecast_leverage(X, t, t, 48)
    sc = np.sqrt(t / 1095)
    bound = ar_bound(want, _row_tol(y) * sc, _row_tol(y, lev) * sc, t, t, 48)
    assert np.array_equal(got["order"], want["order"])
    _le(float((np.abs(got["pred"] - want["pred"]) / bound).max()), 1.0, "hourly 70,001: error / scaled bound")
    eng.close()


def test_nullable_outputs_and_a_wide_table():
    y, X, t_fit, has_c = _case("daily")
    n = len(y)
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    lib, h = eng._lib, eng._h
    yd = torch.from_numpy(y).cuda()
    ref = eng.fit_forecast_ar(yd, 2, t_fit, 28)
    wide = torch.full((n, 41), float(np.float32(PATTERN)), device="cuda")
    view = wide[:, 5:33]                                           # any base pointer, ld_out = 41
    rc = lib.mmf_fit_forecast_ar_f32(h, yd.data_ptr(), n, t_fit, 2, t_fit, 28, view.data_ptr(), 41,
                                     None, None, None, None, None)
    assert rc == 0
    torch.cuda.synchronize()
    assert _same_bits(view, ref["pred"])
    assert (wide[:, :5] == float(np.float32(PATTERN))).all() and (wide[:, 33:] == float(np.float32(PATTERN))).all()
    eng.close()


def test_refused_arguments_write_nothing():
    y, X, t_fit, has_c = _case("daily", n=40)
    n = len(y)
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    lib, h = eng._lib, eng._h
    yd = torch.from_numpy(y).cuda()
    out = torch.full((n, 28), 7.0, device="cuda")
    phi = torch.full((n, AR_MAX), 7.0, device="cuda")
    order = torch.full((n,), 7, device="cuda", dtype=torch.int32)
    sig = torch.full((n,), 7.0, device="cuda")
    status = torch.full((n,), 7, device="cuda", dtype=torch.int32)
    host_out = np.zeros((n, 28), dtype=np.float32)
    calls = [(0, t_fit, 28, out.data_ptr(), 28), (9, t_fit, 28, out.data_ptr(), 28), (2, -1, 28, out.data_ptr(), 28),
             (2, t_fit, 65, out.data_ptr(), 65), (2, t_fit, 28, out.data_ptr(), 27), (2, t_fit, 28, None, 28),
             (2, t_fit, 28, host_out.ctypes.data, 28)]
    for p, ps, npred, optr, ld in calls:
        rc = lib.mmf_fit_forecast_ar_f32(h, yd.data_ptr(), n, t_fit, p, ps, npred, optr, ld, phi.data_ptr(),
                                         order.data_ptr(), sig.data_ptr(), status.data_ptr(), None)
        assert rc != 0, (p, ps, npred, ld)
    assert lib.mmf_fit_forecast_ar_f32(None, yd.data_ptr(), n, t_fit, 2, t_fit, 28, out.data_ptr(), 28, None, None,
                                       None, None, None) != 0
    torch.cuda.synchronize()
    assert (out == 7).all() and (phi == 7).all() and (order == 7).all() and (sig == 7).all() and (status == 7).all()
    assert not host_out.any()
    eng.close()


def test_other_calls_unchanged_by_an_ar_call():
    """plain (future and holdout), ragged and backtest calls on one context give the same bits before and after AR
    calls in both modes"""
    y, X, t_fit, has_c = _case("daily")
    start = np.datetime64(mmf.synth.daily_store_item_demand(1, t_fit, seed=3)[1], "D")
    eng = mmf.ForecastEngine()
    eng.plan_calendars([start, start + 30], [t_fit, t_fit - 30], "D", 28)
    eng.plan_backtest(start, t_fit, "D", 28, 3)
    eng.plan(X, t_fit, has_c)
    full = torch.zeros((len(y), (t_fit + 3) & ~3), device="cuda")
    full[:, :t_fit] = torch.from_numpy(y).cuda()
    yd = full[:, :t_fit]

    def calls():
        bt = eng.backtest(yd)
        return (eng.fit_forecast(yd, t_fit, 28).clone(), eng.fit_forecast(yd, 0, t_fit + 64).clone(),
                eng.fit_forecast_ragged(yd, [0, 70, len(y)]).clone(), bt["pred"].clone(), bt["metrics"].clone(),
                bt["status"].clone())

    before = calls()
    eng.fit_forecast_ar(yd, 4, 0, t_fit + 64)
    eng.fit_forecast_ar(yd, 2, t_fit, 28)
    after = calls()
    assert all(_same_bits(a, b) for a, b in zip(before, after))
    eng.close()


_NEGCTL = """
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np, torch
import test_gpu_ar as T
from ar_oracle import fit_forecast_ar_packed, ar_bound
from test_gpu_edges import _row_tol
import mmf
y, X, t_fit, has_c = T._case("daily", n=330)
rows = [i for i in range(len(y)) if T.AR_KINDS[i % len(T.AR_KINDS)] in ("origin8", "origin1")]
eng = mmf.ForecastEngine()
eng.plan(X, t_fit, has_c)
got = T._run(eng, torch.from_numpy(y).cuda(), 2, t_fit, 28)
want = fit_forecast_ar_packed(y, X, t_fit, t_fit, 28, 2)
b = ar_bound(want, _row_tol(y), _row_tol(y), t_fit, t_fit, 28)
r = (np.abs(got["pred"] - want["pred"]) / b)[rows].max(axis=1)
print(json.dumps({{"worst": float(r.max()), "rows_over": int((r > 1).sum()), "rows": len(rows), "lib": mmf.LIB_PATH}}))
"""


@pytest.mark.parametrize("lib", ["product", "nofill"])
def test_negative_control_without_the_fill(lib):
    """the build that counts a missing fit residual as 0 (tests/_build/libmmf_ar_nofill.so) must exceed the bound on
    rows with gaps at the origin; the product library stays within it"""
    env = dict(os.environ)
    env.pop("MMF_LIB", None)
    if lib == "nofill":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_ar_nofill.so")
        assert os.path.exists(env["MMF_LIB"]), "negative-control library missing: run __graft_entry__.build()"
    r = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    record_err("test_negative_control_without_the_fill", got["worst"], 1.0, what=lib, rows_over=got["rows_over"])
    if lib == "product":
        assert got["worst"] <= 1.0, got
    else:
        assert got["lib"].endswith("libmmf_ar_nofill.so") and got["rows_over"] >= got["rows"] // 2, got


@pytest.mark.parametrize("frame", ["daily", "weekly"])
def test_forecast_groups_with_ar(frame):
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
    out = mmf.forecast_groups(pdf, ar=2, **kw)
    plain = mmf.forecast_groups(pdf, **kw)
    assert list(out.columns) == list(plain.columns) and len(out) == len(plain)
    worst = 0.0
    for (key, g), (_, gp) in zip(out.groupby(["Product", "SKU"], sort=True), plain.groupby(["Product", "SKU"], sort=True)):
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
        want = fit_forecast_ar_packed(y, X, t_fit, ps, npred, 2)
        lev = forecast_leverage(X, t_fit, ps, npred)
        b = ar_bound(want, _row_tol(y[:, :t_fit]) * _mask_factor(y, X, t_fit, 0, t_fit, np.ones(1)),
                     _row_tol(y[:, :t_fit], lev) * _mask_factor(y, X, t_fit, ps, npred, np.ones(1)), t_fit, ps, npred)
        r = float((np.abs(g["Demand_Fitted"].to_numpy() - want["pred"][0]) / b[0]).max())
        worst = max(worst, r)
    _le(worst, 1.0, f"forecast_groups(ar=2) {frame}: error / bound")
