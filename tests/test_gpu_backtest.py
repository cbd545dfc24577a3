"""GPU: the rolling-origin backtest (mmf_plan_backtest / mmf_backtest_f32, DESIGN.md sections 2 item 8 and 4.12).

Every batch mixes the rows of test_gpu_abi_contract.py: gap-free, isolated gaps, 8 leading gaps, 45 gaps in one chunk
parity, mostly missing, a single value, empty and +Inf.  Origin k is held to the stated tolerance times
max(1, leverage_k) * max(1, ||T_k||_2) against the float64 oracle (tests/backtest_oracle.py); rows with gaps also take
the mask factor of their own normal equations."""
import os
import subprocess
import sys

import numpy as np
import pytest

import mmf
from conftest import ROOT, record_err, tolerance
from oracle import mmf_oracle as O
import backtest_oracle as B

pytestmark = pytest.mark.gpu

KINDS = ("clean", "isolated", "leading8", "parity45", "mostly_missing", "single", "empty", "inf")


def _kind_cols(kind, t_fit):
    c = np.arange(t_fit)
    par0 = c[(c // 32) % 2 == 0][:45]
    return {"clean": c[:0],
            "isolated": np.unique([t_fit // 5, t_fit // 2, t_fit - 1]),
            "leading8": c[:8],
            "parity45": par0,
            "mostly_missing": c[c % 3 != 0],
            "single": c[c != t_fit // 2],
            "empty": c,
            "inf": np.array([t_fit // 3])}[kind]


def _plant(y, t_fit, every=1):
    """row i (i % every == 0) gets kind KINDS[(i // every) % 8] over its first t_fit columns"""
    for i in range(0, y.shape[0], every):
        kind = KINDS[(i // every) % len(KINDS)]
        y[i, _kind_cols(kind, t_fit)] = np.inf if kind == "inf" else np.nan
    return y


def _straddling(origin):
    """gap patterns that differ from origin to origin: a gap exactly at each t_k and at t_k - 1; per chunk parity, 44
    gaps below the first origin and the 45th between the first two (and exactly at an origin where the parity allows),
    alone and with the other parity doing the same; more than half of [0, t_1) missing but not of [0, t_K)"""
    rows = []
    for t in origin:
        rows += [np.array([t]), np.array([t - 1]), np.array([t - 1, t]), np.array([t - 2, t, t + 1])]
    c = np.arange(8, origin[-1])
    over = []
    for par in (0, 1):
        pc = c[(c // 32) % 2 == par]
        below = pc[pc < origin[0]]
        if len(origin) > 1 and len(below) >= 44:
            between = pc[(pc >= origin[0]) & (pc < origin[1])]
            for b in between[:1].tolist() + [o for o in origin[:-1] if (o // 32) % 2 == par]:
                rows.append(np.r_[below[:44], b])
            if len(between):
                over.append(np.r_[below[:43], between[:2]])
    if len(over) == 2:
        rows.append(np.r_[over[0], over[1]])
    rows.append(np.arange(8, 8 + int(0.6 * origin[0])))
    return rows


def _with_straddling(y, origin):
    """y with one extra row per _straddling pattern (the rest of the row observed)"""
    pats = _straddling(origin)
    extra = np.repeat(y[:1], len(pats), axis=0).copy()
    for i, cols in enumerate(pats):
        cols = np.asarray(cols, dtype=np.int64)
        extra[i, cols[cols < y.shape[1]]] = np.nan
    return np.concatenate([y, extra]).astype(np.float32)


def _mask_factor(y, X, t, h, ratio):
    """1/min(1, ratio/0.25), or the forward-error amplification of the row's own normal equations where larger
    (the factor tests/test_gpu_abi_contract.py applies); gap-free rows get 1"""
    from test_gpu_abi_contract import _mask_factor as mf
    return mf(y, X[:t + h], t, t, h, ratio)


def _calendar(name, n):
    """(y [n, t_len] float32, X [t_len, P] of the whole window, has_constant)"""
    t_len, end, freq = {"daily": (1095, "2020-12-31", "D"),          # C2-like
                        "weekly": (156, "2020-12-28", "W-MON"),      # a weekly calendar
                        "covid": (365, "2020-05-30", "D")}[name]     # 2020-03-01 is grid row 273
    if freq == "D":
        y, start = mmf.synth.daily_store_item_demand(n, t_len, seed=7, end=np.datetime64(end))
    else:
        yd, start = mmf.synth.daily_store_item_demand(n, 7 * t_len - 6, seed=7, end=np.datetime64(end))
        y = np.ascontiguousarray(yd[:, ::7])
    days = mmf.design.calendar_grid(start, t_len, freq)
    return y.astype(np.float32), mmf.design.design_matrix(days, t_len - 28, "trend_season_exog"), True


def _run(eng, y, X, origin, h, has_constant=True):
    import torch
    o = np.asarray(origin, dtype=np.int32)
    Xc = np.ascontiguousarray(X, dtype=np.float64)
    lib = eng._lib
    mmf._native.check(lib.mmf_plan_backtest(eng._h, Xc.ctypes.data, Xc.shape[0], Xc.shape[1], int(has_constant),
                                            len(o), o.ctypes.data, int(h)))
    eng._backtest = (o, int(h), X.shape[0])
    res = eng.backtest(mmf.device_packed(y))
    torch.cuda.synchronize()
    return {k: (v.cpu().numpy() if v is not None else None) for k, v in res.items()}


def _plain(eng, y, X, origin, h):
    """the plain future-mode call per origin (design X[:t_k + h], t_fit = t_k): forecasts [K, n, h], status [K, n]"""
    yd = mmf.device_packed(y)
    pred, st = [], []
    for t in origin:
        eng.plan(X[:t + h], int(t), True)
        r = eng.fit_forecast(yd, int(t), h, want_status=True)
        pred.append(r["pred"].cpu().numpy()); st.append(r["status"].cpu().numpy())
    return np.stack(pred), np.stack(st)


def _check_oracle(name, y, X, origin, h, got, plain=None, plain_st=None):
    """every (row, origin) within the bound; with `plain` given, a forecast bit-equal to the plain per-origin call
    passes as well (rows the general pass finishes in both calls: the bound of those is the plain call's, whose mask
    factor does not cover long leading gaps), and the status must equal the plain call's (else the oracle's)"""
    want, wst, ratio = B.backtest_packed(y, X, origin, h, return_ratio=True)
    _, kappa, lev = B.change_of_basis(X, origin, h)
    worst = 0.0
    for k, t in enumerate(origin):
        mask = _mask_factor(y[:, :t], X, int(t), h, ratio[k])
        tol = tolerance(y[:, :t], max(1.0, lev[k]) * max(1.0, kappa[k])) * mask[:, None]
        ok = wst[k] != 1
        err = np.abs(got["pred"][k] - want[k])
        assert np.all(np.isnan(got["pred"][k][~ok])), (name, k)
        bad = ok[:, None] & ~(err <= tol)
        if plain is not None:
            bad &= got["pred"][k] != plain[k]
        assert not bad.any(), (name, k, int(t), np.argwhere(bad)[:5], float(np.nanmax(err / tol)))
        worst = max(worst, float(np.nanmax(np.where(ok[:, None], err / tol, 0.0))))
        ref = wst[k] if plain is None else plain_st[k]
        assert np.array_equal(got["status"][k], ref), (name, k, np.flatnonzero(got["status"][k] != ref)[:8])
    record_err(f"backtest[{name}]", worst, 1.0, origins=[int(t) for t in origin], horizon=h)
    # metrics: the GPU's own forecasts scored in float64
    m, cnt = B.metrics(got["pred"], B.actuals(y, origin, h))
    assert np.array_equal(got["count"], cnt)
    np.testing.assert_allclose(got["metrics"], m, rtol=1e-6, atol=0, equal_nan=True)


@pytest.mark.parametrize("cal,origin,h", [
    ("daily", [1095 - 28], 28),
    ("daily", [1095 - 28 - 3 * 28, 1095 - 28 - 2 * 28, 1095 - 28 - 28, 1095 - 28], 28),
    ("daily", [33, 64, 65, 95, 100, 120, 700, 1031], 64),         # t % 32 in {0, 1, 31}, two in one chunk, one apart
    ("daily", [640, 641, 1000, 1094], 1),
    ("daily", [500, 700, 900, 1055], 40),
    ("weekly", [100, 120, 140, 155], 1),
    ("weekly", [60, 80, 100, 128], 28),
    ("covid", [200, 250, 274, 290, 337], 28),                        # 2020-03-01 is grid row 274
])
def test_backtest_matches_oracle(cal, origin, h):
    y, X, _ = _calendar(cal, 301)
    _plant(y, origin[-1])                                  # the row mix over [0, t_K): gaps on both sides of origins
    y = _with_straddling(y, origin)
    eng = mmf.ForecastEngine(device=0)
    got = _run(eng, y, X, origin, h)
    plain, st = _plain(eng, y, X, origin, h)
    _check_oracle(f"{cal}-{len(origin)}-{h}", y, X, origin, h, got, plain, st)
    eng.close()


def test_single_origin_is_bit_equal_to_the_plain_future_call():
    y, X, _ = _calendar("daily", 301)
    _plant(y, 1095 - 28)
    t, h = 1095 - 28, 28
    eng = mmf.ForecastEngine(device=0)
    got = _run(eng, y, X, [t], h)
    eng.plan(X, t, True)
    ref = eng.fit_forecast(mmf.device_packed(y), t, h, want_status=True)
    assert np.array_equal(got["pred"][0], ref["pred"].cpu().numpy(), equal_nan=True)
    assert np.array_equal(got["status"][0], ref["status"].cpu().numpy())
    eng.close()


def test_exact_power_of_two_scaling():
    y, X, _ = _calendar("daily", 130)
    origin, h = [600, 800, 1000, 1067], 28
    _plant(y, 1067)
    y = _with_straddling(y, origin)
    eng = mmf.ForecastEngine(device=0)
    base = _run(eng, y, X, origin, h)
    for e in (-6, 5):
        s = _run(eng, (y * np.float32(2.0 ** e)).astype(np.float32), X, origin, h)
        assert np.array_equal(s["pred"], base["pred"] * np.float32(2.0 ** e), equal_nan=True)
        np.testing.assert_allclose(s["metrics"][..., 1:3], base["metrics"][..., 1:3] * 2.0 ** e, rtol=1e-6, equal_nan=True)
        np.testing.assert_allclose(s["metrics"][..., 0], base["metrics"][..., 0] * 4.0 ** e, rtol=1e-6, equal_nan=True)
        np.testing.assert_allclose(s["metrics"][..., 3], base["metrics"][..., 3], rtol=1e-6, equal_nan=True)
        assert np.array_equal(s["count"], base["count"])
    eng.close()


def test_metrics_edges():
    """NaN actual values, zero actual values (MAPE), an unobserved window (count 0: all four metrics NaN)"""
    y, X, _ = _calendar("daily", 64)
    origin, h = [900, 1067], 28
    y[1, 1067:1067 + 10] = np.nan
    y[2, 1067:] = 0.0
    y[3, 1067:] = np.nan
    y[4, 900:928] = np.nan
    eng = mmf.ForecastEngine(device=0)
    got = _run(eng, y, X, origin, h)
    m, cnt = B.metrics(got["pred"], B.actuals(y, origin, h))
    assert np.array_equal(got["count"], cnt)
    assert got["count"][1, 3] == 0 and np.isnan(got["metrics"][1, 3]).all()
    assert got["count"][1, 2] == h and np.isnan(got["metrics"][1, 2, 3])
    np.testing.assert_allclose(got["metrics"], m, rtol=1e-6, equal_nan=True)
    eng.close()


def test_slabs_and_long_hourly_series():
    import torch
    # 2^20 + 1,001 series x 100 days, K = 4: K * n output rows are split into slabs
    n, t_len, h = (1 << 20) + 1001, 100, 8
    rng = np.random.default_rng(3)
    y = (50 + 10 * rng.standard_normal((n, t_len))).astype(np.float32)
    gappy = np.arange(0, n, 65536)
    for j, i in enumerate(gappy):
        y[i, _kind_cols(KINDS[j % 8], 92)] = np.inf if KINDS[j % 8] == "inf" else np.nan
    days = mmf.design.calendar_grid("2020-01-01", t_len, "D")
    X = mmf.design.design_matrix(days, t_len - h, "trend_season_exog")
    origin = [60, 70, 84, 92]
    eng = mmf.ForecastEngine(device=0)
    got = _run(eng, y, X, origin, h)
    sample = np.unique(np.concatenate([gappy, rng.integers(0, n, 4000), [n - 1, (1 << 20) - 1, 1 << 20]]))
    plain, st = _plain(eng, y[sample], X, origin, h)
    _check_oracle("slabs", y[sample], X, origin, h, {k: v[:, sample] for k, v in got.items()}, plain, st)
    del got
    # a 70,001-row hourly series (tolerance x sqrt(t / 1095)): the restart fold across snapshots
    t_len = 70001
    yh = (100 + 20 * rng.standard_normal((5, t_len))).astype(np.float32)
    yh[1, 30000:30010] = np.nan
    hours = np.arange(t_len, dtype=np.float64)
    Xh = np.zeros((t_len, 16))
    Xh[:, 0] = 1.0
    Xh[:, 1] = (hours - t_len / 2) / t_len
    for j in range(1, 4):
        Xh[:, 2 * j] = np.sin(2 * np.pi * j * hours / 24)
        Xh[:, 2 * j + 1] = np.cos(2 * np.pi * j * hours / 24)
    origin = [20000, 40001, 65000, 65535 - 64]             # the last origin is at most 65,535 (gap positions are 16 bit)
    got = _run(eng, yh, Xh, origin, 64)
    want, wst = B.backtest_packed(yh, Xh, origin, 64)
    _, kappa, lev = B.change_of_basis(Xh, origin, 64)
    for k, t in enumerate(origin):
        tol = tolerance(yh[:, :t], max(1.0, lev[k]) * max(1.0, kappa[k])) * np.sqrt(t / 1095)
        err = float(np.abs(got["pred"][k] - want[k]).max())
        assert err <= tol, (k, t, err, tol)
        assert np.array_equal(got["status"][k], wst[k])
    eng.close()


def test_argument_errors_write_nothing_and_plans_stay_in_force():
    import torch
    y, X, _ = _calendar("daily", 40)
    yd = mmf.device_packed(y)
    eng = mmf.ForecastEngine(device=0)
    eng.plan(X, 1095 - 28, True)
    before = eng.fit_forecast(yd, 1095 - 28, 28).cpu().numpy()
    # a ragged plan beside it: two calendars (the second one 300 days shorter), rows 0-19 and 20-39
    start = mmf.design.calendar_grid("2018-01-01", 1, "D")[0]
    eng.plan_calendars([start, start + np.timedelta64(300, "D")], [1095 - 28, 1095 - 328], "D", 28)
    rows = [0, 20, 40]
    ragged_before = eng.fit_forecast_ragged(yd, rows).cpu().numpy()
    lib, h = eng._lib, eng._h
    Xc = np.ascontiguousarray(X, dtype=np.float64)

    def plan(origin, hz, n_rows=None):
        o = np.asarray(origin, dtype=np.int32)
        return lib.mmf_plan_backtest(h, Xc.ctypes.data, n_rows or Xc.shape[0], 16, 1, len(o), o.ctypes.data, hz)

    assert plan([32, 100], 28) != 0                       # first origin below 33
    assert plan([100, 100], 28) != 0                      # not increasing
    assert plan([100, 1080], 28) != 0                     # past the design
    assert plan([100], 65) != 0                           # horizon above 64
    assert plan(list(range(100, 100 + 9)), 28) != 0       # more than MMF_BT_MAX_ORIGINS
    assert lib.mmf_backtest_f32(h, yd.data_ptr(), 40, yd.stride(0), None, 0, None, None, None, None) == -4   # no plan
    assert plan([500, 1067], 28) == 0
    K, n = 2, 40
    pat = float(np.float32(1.2345))
    pred = torch.full((K, n, 28), pat, device="cuda")
    met = torch.full((K, n, 4), pat, device="cuda")
    cnt = torch.full((K, n), 7, dtype=torch.int32, device="cuda")
    st = torch.full((K, n), 7, dtype=torch.int32, device="cuda")
    args = lambda ldy, ldo: (h, yd.data_ptr(), n, ldy, pred.data_ptr(), ldo, met.data_ptr(), cnt.data_ptr(), st.data_ptr(), None)
    assert lib.mmf_backtest_f32(*args(yd.stride(0), 27)) != 0                  # ld_out < horizon
    assert lib.mmf_backtest_f32(*args(1094, 28)) != 0                          # ld_y below the last origin + horizon
    assert lib.mmf_backtest_f32(h, yd.data_ptr(), n, yd.stride(0), None, 28, None, None, None, None) != 0   # nothing out
    torch.cuda.synchronize()
    assert (pred == pat).all() and (met == pat).all() and (cnt == 7).all() and (st == 7).all()
    # the plain plan is still in force, bit for bit
    after = eng.fit_forecast(yd, 1095 - 28, 28).cpu().numpy()
    assert np.array_equal(before, after, equal_nan=True)
    # ... and so is the ragged plan
    assert np.array_equal(ragged_before, eng.fit_forecast_ragged(yd, rows).cpu().numpy(), equal_nan=True)
    # metrics only (no forecast table): the same numbers
    assert lib.mmf_backtest_f32(h, yd.data_ptr(), n, yd.stride(0), pred.data_ptr(), 28, met.data_ptr(), cnt.data_ptr(),
                                st.data_ptr(), None) == 0
    met2 = torch.empty_like(met)
    assert lib.mmf_backtest_f32(h, yd.data_ptr(), n, yd.stride(0), None, 0, met2.data_ptr(), None, None, None) == 0
    torch.cuda.synchronize()
    assert torch.equal(torch.nan_to_num(met, 9.0), torch.nan_to_num(met2, 9.0))
    eng.close()


_NEGCTL = r"""
import sys, numpy as np
sys.path[:0] = [{root!r}, {tests!r}]
import mmf, backtest_oracle as B
from conftest import tolerance
from test_gpu_backtest import _calendar, _run
y, X, _ = _calendar("daily", 4096)
origin, h = [952, 980, 1008, 1036], 28
eng = mmf.ForecastEngine(device=0)
got = _run(eng, y, X, origin, h)
want, _ = B.backtest_packed(y, X, origin, h)
_, kappa, lev = B.change_of_basis(X, origin, h)
bad = 0
for k in range(len(origin)):
    tol = tolerance(y[:, :origin[k]], max(1.0, lev[k]) * max(1.0, kappa[k]))
    bad += int((np.abs(got["pred"][k] - want[k]) > tol).any(axis=1).sum())
print("EXCEED", bad)
"""


@pytest.mark.parametrize("lib,expect_fail", [("product", False), ("negctl", True)])
def test_negative_control_exceeds_the_bound(lib, expect_fail):
    env = dict(os.environ)
    if lib == "negctl":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_negctl.so")
    code = _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    bad = int(out.stdout.split("EXCEED")[-1])
    assert (bad >= 100) if expect_fail else (bad == 0), bad


def test_engine_accepts_a_contiguous_unpitched_tensor():
    """a plain contiguous [n, 1095] tensor (row pitch not a multiple of 4 floats) is copied into a pitched buffer"""
    import torch
    y, X, _ = _calendar("daily", 50)
    _plant(y, 1067)
    eng = mmf.ForecastEngine(device=0)
    eng.plan_backtest(mmf.synth.daily_store_item_demand(1, 1095, seed=7, end=np.datetime64("2020-12-31"))[1], 1095,
                      "D", 28, 3)
    a = eng.backtest(torch.from_numpy(y).cuda())
    b = eng.backtest(mmf.device_packed(y))
    for key in ("pred", "metrics", "count", "status"):
        assert torch.equal(torch.nan_to_num(a[key].float(), 7.0), torch.nan_to_num(b[key].float(), 7.0)), key
    eng.close()


def test_backtest_groups_matches_the_oracle_stand_in():
    """the frame layer on the GPU (several calendar buckets, one call each) against the float64 stand-in engine of
    tests/test_backtest_frames.py: same rows, counts exact, metrics within what the forecast bound allows"""
    import pandas as pd
    import pyarrow as pa
    from test_backtest_frames import KW, _OracleBacktestEngine, weekly_frame
    df, spec = weekly_frame()
    eng = mmf.ForecastEngine(device=0)
    got = mmf.backtest_groups(df, engine=eng, **KW)
    ref = mmf.backtest_groups(df, engine=_OracleBacktestEngine(), **KW)
    assert got[["Product", "SKU", "Cutoff", "N"]].equals(ref[["Product", "SKU", "Cutoff", "N"]])
    h, K, step = KW["horizon"], KW["n_origins"], KW["step"]
    for p, sku, start, n in spec:
        g, r = got[got["SKU"] == sku], ref[ref["SKU"] == sku]
        if len(r) == 0:
            continue
        ys = df[df["SKU"] == sku].sort_values("Date")
        y = np.full((1, n), np.nan, dtype=np.float32)
        y[0, ((pd.to_datetime(ys["Date"]) - pd.Timestamp(start)).dt.days // 7).to_numpy()] = ys["Demand"].to_numpy(np.float32)
        origin = [t for t in (n - h - (K - 1 - k) * step for k in range(K)) if t >= 33]
        X = mmf.design.design_matrix(mmf.design.calendar_grid(np.datetime64(start), n, "W-MON"), n - h)
        _, kappa, lev = B.change_of_basis(X, origin, h)
        _, _, ratio = B.backtest_packed(y, X, origin, h, return_ratio=True)
        for k, t in enumerate(origin):
            tol = tolerance(y[:, :t], max(1.0, lev[k]) * max(1.0, kappa[k])) * float(_mask_factor(y[:, :t], X, t, h, ratio[k])[0])
            gm, rm = g.iloc[k], r.iloc[k]
            assert abs(gm["MAE"] - rm["MAE"]) <= tol and abs(gm["Bias"] - rm["Bias"]) <= tol, (sku, k)
            assert abs(gm["MSE"] - rm["MSE"]) <= 2 * tol * np.sqrt(rm["MSE"]) + tol * tol + 1e-6 * rm["MSE"], (sku, k)
            act = np.abs(y[0, t:t + h][np.isfinite(y[0, t:t + h]) & (y[0, t:t + h] != 0)])
            assert abs(gm["MAPE"] - rm["MAPE"]) <= tol / act.min() + 1e-6 * rm["MAPE"], (sku, k)
    # Arrow input: the same frame
    at = mmf.backtest_groups(pa.Table.from_pandas(df, preserve_index=False), engine=eng, **KW)
    assert at.equals(got)
    eng.close()
