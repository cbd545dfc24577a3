"""GPU (-m gpu): every model on intermittent, low-volume and degenerate demand series (tests/demand_shapes.py) against
the float64 oracles, row by row.

Every comparison is per row: the plain model's bound is tolerance(row, leverage) x the row's mask factor (never the
tolerance of a whole batch, which would let a level-0.3 row sitting beside a level-60,000 row be off by 100 %); the AR,
selection and ARIMA bounds are those of their oracle modules, evaluated with the same per-row tau.  Statuses equal the
oracle's everywhere.  The worst error / bound is logged (conftest.record_err) per entry point for the intermittent rows,
the mixed-scale rows and the degenerate rows (with their count).

Stated exceptions, measured on an H100 80GB HBM3 (700 W); the worst raw ratio of every kind is logged:
* statuses (and dof) are compared on the rows whose pivot ratios lie outside PIVOT_BAND of the threshold
  (test_gpu_ragged's rule): there fp32 and float64 may decide a column differently.  The rows inside the band are
  counted in the log; their empty / non-empty status is still compared;
* launched and discontinued rows (GAP_KINDS) are held to GAP_SLACK x their row bound (their tau in the AR and
  selection bounds carries the same factor): the mask factor of test_gpu_edges does not cover long leading or trailing
  gaps (as test_gpu_backtest notes).  Worst measured raw ratios: launch_late 18.1 (daily 365, future, a history of
  40-180 days), launch_early 3.3, discontinued 3.0, launch_after_xmas 0.85 (backtest: 3.9, 3.3, 1.9).  Their mask
  factors are already 1e2-1e6, so squaring it is no remedy; a bound for short histories is left open;
* rows whose values change sign (SIGN_KINDS: returns, mean-zero demand) are held to SIGN_SLACK x their row bound: the
  tolerance's 5e-6 max|y| is stated for data that varies little about its centring constant c (the first value), and
  on these rows |y - c| reaches 2 max|y|, so the fp32 moments carry up to twice the rounding (worst measured raw
  ratios: returns 1.86, signed 1.13).

Degenerate rows (ar_oracle.degenerate_rows: the oracle's RMS residual is within a few tau, so the first-order AR bounds
do not apply) are held to ar_oracle.degenerate_bound instead, and the rows the regression fits exactly (all zero,
constant) must come out with order 0, phi = 0, sigma = 0 and the plain call's predictions bit for bit.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mmf
import backtest_oracle as B
from ar_oracle import AR_MAX, FP32_EPS, degenerate_bound, degenerate_rows, fit_forecast_ar_packed
from ar_select_oracle import mse_bound, select_ar_packed
from arima_oracle import fit_forecast_arima_packed, z_tau
from interval_oracle import fit_forecast_se_packed
from conftest import ROOT, forecast_leverage, record_err, tolerance
from demand_shapes import DEGENERATE, EXACT_FIT, INTERMITTENT, SCALED, calendar, demand_batch, kind_rows
from oracle import mmf_oracle as O
from test_gpu_abi_contract import _check_beta, _mask_factor, _oracle
from test_gpu_edges import _le, _row_tol, _same_bits
from test_gpu_ragged import PIVOT_BAND, _pivot_distance

pytestmark = pytest.mark.gpu

N = 300                     # 2 full 128-row tiles and a partial one; 15 cycles of the 20 kinds
H = 28
EXACT = ("zeros", "const1", "const65534")          # residuals exactly 0 on every path
GAP_KINDS = ("launch_early", "launch_late", "discontinued", "launch_after_xmas")
GAP_SLACK = 32.0
SIGN_KINDS = ("returns", "signed")
SIGN_SLACK = 2.0


def _case(cal, h=H, mode="future", n=N, seed=0):
    """(y [n, t] float32, kinds, X, t_fit, ps, npred) of one calendar: future = fit all t rows and forecast h; holdout =
    fit t - h rows and evaluate every row"""
    start, t, freq, _ = calendar(cal)
    t_fit = t if mode == "future" else t - h
    y, kinds, _ = demand_batch(n, cal, seed=seed + sum(map(ord, cal)), t_fit=t_fit)
    n_rows = t + h if mode == "future" else t
    X = O.design_matrix(O.calendar_grid(start, n_rows, freq), t_fit)
    ps, npred = (t_fit, h) if mode == "future" else (0, t)
    return y, kinds, X, t_fit, ps, npred


def _dev(y, t_fit):
    """device copy with a 16-B row pitch (the tensor-core path's TMA needs it)"""
    full = torch.full((len(y), (y.shape[1] + 3) & ~3), float("nan"), device="cuda")
    full[:, :y.shape[1]] = torch.from_numpy(y).cuda()
    return full[:, :t_fit]


def _np(res):
    return {k: v.cpu().numpy() for k, v in res.items() if k != "stats"}


def _report(entry, ratio, kinds, what):
    """log the worst ratio of the intermittent, mixed-scale and degenerate rows; assert every ratio <= 1"""
    ratio = np.asarray(ratio, dtype=np.float64)
    for group, names in (("intermittent", INTERMITTENT), ("mixed_scale", SCALED), ("degenerate", DEGENERATE)):
        m = kind_rows(kinds, names) & np.isfinite(ratio)
        record_err(f"demand_shapes[{entry}]", float(ratio[m].max()) if m.any() else 0.0, 1.0, rows=group,
                   count=int(m.sum()), what=what)
    worst = float(np.nanmax(ratio)) if ratio.size else 0.0
    assert worst <= 1.0, (entry, what, worst, [kinds[i] for i in np.flatnonzero(ratio > 1.0)[:8]])
    return worst


def _slack(kinds):
    return np.where(kind_rows(kinds, GAP_KINDS), GAP_SLACK, np.where(kind_rows(kinds, SIGN_KINDS), SIGN_SLACK, 1.0))


def _per_kind(entry, raw, kinds, what):
    """log the worst raw ratio (before any slack) of every kind"""
    for kind in sorted(set(kinds)):
        m = kind_rows(kinds, (kind,)) & np.isfinite(raw)
        if m.any():
            record_err(f"demand_shapes[{entry} per kind]", float(raw[m].max()), 1.0, kind=kind, what=what)


def _plain_ratio(pred, status, y, X, t_fit, ps, npred, orc, what, kinds):
    """statuses equal the oracle's outside the pivot band, NaN rows exactly for status 1; per-row error /
    (tolerance(row, leverage) x mask factor x slack)"""
    want = orc["gamma"] @ orc["A"][ps:ps + npred].T
    sure = _pivot_distance(y, X, t_fit) > PIVOT_BAND
    record_err("demand_shapes[pivot band rows]", float((~sure).sum()), float(len(y)), what=what,
               differing=int((status != orc["status"]).sum()))
    assert np.array_equal(status[sure], orc["status"][sure]), (what, np.flatnonzero(sure & (status != orc["status"])))
    assert np.array_equal(status == 1, orc["status"] == 1), what
    empty = orc["status"] == 1
    assert np.isnan(pred[empty]).all() and np.isfinite(pred[~empty]).all(), what
    tol = (_row_tol(y[:, :t_fit], forecast_leverage(X, t_fit, ps, npred))
           * _mask_factor(y, X, t_fit, ps, npred, orc["ratio"]))
    r = np.zeros(len(y))
    r[~empty] = np.abs(pred[~empty] - want[~empty]).max(axis=1) / tol[~empty]
    _per_kind("plain", r, kinds, what)
    return r / _slack(kinds)


# =====================================================================================================================
# plain fit
# =====================================================================================================================
@pytest.mark.parametrize("cal,h,mode", [("daily1095", 28, "future"), ("daily1095", 64, "future"),
                                        ("daily1095", 28, "holdout"), ("daily365", 30, "future"),
                                        ("daily365", 28, "holdout"), ("weekly157", 28, "future"),
                                        ("weekly157", 28, "holdout")])
def test_plain_fit_per_row(cal, h, mode):
    y, kinds, X, t_fit, ps, npred = _case(cal, h, mode)
    orc = _oracle(y, X, t_fit)
    yd = _dev(y, t_fit)
    tight = ~kind_rows(kinds, GAP_KINDS)
    engs = {"auto": mmf.ForecastEngine(), "tc": mmf.ForecastEngine(kernel="tc"),
            "warp": mmf.ForecastEngine(kernel="warp"), "tc2": mmf.ForecastEngine(kernel="tc", tc_variant=2)}
    for k, eng in engs.items():
        eng.plan(X, t_fit, True)
        r = _np(eng.fit_forecast(yd, ps, npred, want_status=True, want_beta=True))
        _report(f"plain {k}", _plain_ratio(r["pred"], r["status"], y, X, t_fit, ps, npred, orc, f"{cal} {mode} {k}", kinds),
                kinds, f"{cal} h={h} {mode}")
        # X beta: test_gpu_abi_contract's bound, on the rows outside GAP_KINDS (its mask factor has the same limits)
        sub = dict(orc, gamma=orc["gamma"][tight], status=orc["status"][tight], ratio=orc["ratio"][tight])
        _check_beta(r["beta"][tight], y[tight], X, t_fit, sub, f"{cal} {mode} {k}")
        eng.close()
    # assume_finite on the gap-free rows: bit-equal to the default configuration
    free = np.flatnonzero(np.isfinite(y[:, :t_fit]).all(axis=1))
    assert free.size > 100
    yf = _dev(np.ascontiguousarray(y[free]), t_fit)
    a, b = mmf.ForecastEngine(), mmf.ForecastEngine(assume_finite=True)
    for e in (a, b):
        e.plan(X, t_fit, True)
    ra = a.fit_forecast(yf, ps, npred, want_status=True)
    rb = b.fit_forecast(yf, ps, npred, want_status=True)
    assert _same_bits(ra["pred"], rb["pred"]) and _same_bits(ra["status"], rb["status"]), (cal, mode)
    a.close()
    b.close()


def test_per_row_bound_catches_what_the_batch_bound_misses():
    """a level-0.3 row off by 0.1 passes conftest.tolerance of the whole batch (set by the level-60,000 rows) but fails
    its own row's bound"""
    y, kinds, X, t_fit, ps, npred = _case("daily365", 28)
    orc = _oracle(y, X, t_fit)
    want = orc["gamma"] @ orc["A"][ps:ps + npred].T
    i = next(j for j in range(len(y)) if kinds[j] == "regular" and 0.25 <= np.nanmax(np.abs(y[j])) <= 0.5)
    bad = want.copy()
    bad[i] += 0.1
    lev = forecast_leverage(X, t_fit, ps, npred)
    assert np.abs(bad - want).max() <= tolerance(y, lev)
    r = _plain_ratio(bad, orc["status"], y, X, t_fit, ps, npred, orc, "planted", kinds)
    assert r[i] > 10 and (np.delete(r, i) == 0).all()


# =====================================================================================================================
# prediction standard errors
# =====================================================================================================================
def test_standard_errors():
    from test_gpu_intervals import _check_se
    y, kinds, X, t_fit, ps, npred = _case("daily1095", 28)
    extra = np.full((4, y.shape[1]), np.nan, dtype=np.float32)
    for j, k in enumerate((20, 8, 3, 1)):                      # launched k days before t_fit
        extra[j, t_fit - k:] = np.arange(k) % 5 + 1
    y = np.concatenate([y, extra])
    kinds = kinds + ["launch_short"] * 4
    for kernel in ("auto", "tc", "warp"):
        eng = mmf.ForecastEngine(kernel=kernel)
        eng.plan(X, t_fit, True)
        yd = _dev(y, t_fit)
        plain = eng.fit_forecast(yd, ps, npred, want_status=True)
        got = eng.fit_forecast_se(yd, ps, npred)
        assert _same_bits(plain["pred"], got["pred"]) and torch.equal(plain["status"], got["status"]), kernel
        got = _np(got)
        # dof counts the kept columns; the exactly fit rows are checked exactly below (their oracle RSS is ~1e-16)
        sure = np.flatnonzero((_pivot_distance(y, X, t_fit) > PIVOT_BAND) & ~kind_rows(kinds, EXACT))
        ref = _check_se({k: v[sure] for k, v in got.items()}, y[sure], X, t_fit, ps, npred, f"demand shapes / {kernel}")
        assert (ref["dof"] <= 0).any() and np.isnan(got["se"][sure][ref["dof"] <= 0]).all(), kernel
        exact = kind_rows(kinds, EXACT)
        assert (got["sigma"][exact] == 0).all() and (got["se"][exact] == 0).all(), kernel
        ref_ex = fit_forecast_se_packed(y[exact], X, t_fit, ps, npred)
        assert np.array_equal(got["dof"][exact], ref_ex["dof"]), kernel
        eng.close()


# =====================================================================================================================
# AR(p)
# =====================================================================================================================
def _take(res, idx):
    """the rows idx of an oracle or GPU result dict"""
    n = len(res["status"])
    out = {}
    for k, v in res.items():
        if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == n:
            out[k] = v[idx]
        elif isinstance(v, list) and len(v) == n:
            out[k] = [v[i] for i in idx]
        else:
            out[k] = v
    return out


def _taus(y, X, t_fit, ps, npred, kinds):
    lev = forecast_leverage(X, t_fit, ps, npred)
    tf = _row_tol(y[:, :t_fit]) * _mask_factor(y, X, t_fit, 0, t_fit, np.ones(len(y))) * _slack(kinds)
    tp = _row_tol(y[:, :t_fit], lev) * _mask_factor(y, X, t_fit, ps, npred, np.ones(len(y))) * _slack(kinds)
    return np.where(np.isfinite(tf), tf, 0.0), np.where(np.isfinite(tp), tp, 0.0)


def _exact_rows_are_plain(got, plain, kinds, what):
    ex = kind_rows(kinds, EXACT)
    assert (got["order"][ex] == 0).all() and not got["phi"][ex].any() and (got["sigma"][ex] == 0).all(), what
    assert got["pred"][ex].tobytes() == plain[ex].tobytes(), what


@pytest.mark.parametrize("p", [1, 2, 8])
@pytest.mark.parametrize("cal,h,mode", [("daily1095", 28, "future"), ("daily1095", 64, "future"),
                                        ("weekly157", 28, "holdout")])
def test_ar_per_row(cal, h, mode, p):
    from test_gpu_ar import _compare
    y, kinds, X, t_fit, ps, npred = _case(cal, h, mode, n=160)
    want = fit_forecast_ar_packed(y, X, t_fit, ps, npred, p)
    tau_fit, tau_pred = _taus(y, X, t_fit, ps, npred, kinds)
    deg = degenerate_rows(want, tau_fit)
    nd = np.flatnonzero(~deg)
    yd = _dev(y, t_fit)
    for k in ("auto", "tc", "warp"):
        eng = mmf.ForecastEngine(kernel=k)
        eng.plan(X, t_fit, True)
        got = _np(eng.fit_forecast_ar(yd, p, ps, npred))
        plain = eng.fit_forecast(yd, ps, npred, want_status=True)
        assert np.array_equal(got["status"], plain["status"].cpu().numpy())
        what = f"{cal} {mode} h={h} p={p} {k}"
        _compare(_take(got, nd), _take(want, nd), y[nd], X, t_fit, ps, npred, what)
        _exact_rows_are_plain(got, plain["pred"].cpu().numpy(), kinds, what)
        _degenerate(got, want, deg, tau_fit, tau_pred, t_fit, ps, npred, kinds, what)
        eng.close()


def _degenerate(got, want, deg, tau_fit, tau_pred, t_fit, ps, npred, kinds, what):
    """degenerate rows: within degenerate_bound; logged with their count, the GPU's largest order and |phi|_1, and the
    error in units of the plain tolerance"""
    assert deg.any(), what
    idx = np.flatnonzero(deg)
    sub = _take(want, idx)
    b = degenerate_bound(sub, got["phi"][idx], tau_fit[idx], tau_pred[idx], t_fit, ps, npred)
    err = np.abs(got["pred"][idx].astype(np.float64) - sub["pred"])
    r = float((err / b).max())
    plain_units = float((err.max(axis=1) / tau_pred[idx]).max())
    record_err("demand_shapes[ar degenerate]", r, 1.0, count=int(deg.sum()), what=what,
               gpu_max_order=int(got["order"][idx].max()), oracle_max_order=int(sub["order"].max()),
               gpu_max_phi_l1=float(np.abs(got["phi"][idx]).sum(axis=1).max()), err_over_plain_tol=plain_units,
               kinds=sorted(set(kinds[i] for i in idx)))
    _le(r, 1.0, f"{what}: degenerate rows / degenerate_bound")


def test_residual_scale_of_exactly_fit_rows():
    """the GPU's fitted-value noise on the rows the regression fits exactly, in units of eps x RMS(y - c) (c the first
    value): the scale an AR fit on those rows sees"""
    for cal in ("daily1095", "weekly157"):
        y, kinds, X, t_fit, ps, npred = _case(cal, H, "holdout")
        yd = _dev(y, t_fit)
        rows = kind_rows(kinds, EXACT_FIT)
        for k in ("tc", "warp"):
            eng = mmf.ForecastEngine(kernel=k)
            eng.plan(X, t_fit, True)
            fit = eng.fit_forecast(yd, 0, y.shape[1]).cpu().numpy()[:, :t_fit].astype(np.float64)
            eng.close()
            yy = y[:, :t_fit].astype(np.float64)
            e = np.sqrt(((yy - fit) ** 2).mean(axis=1))
            s = np.sqrt(((yy - yy[:, :1]) ** 2).mean(axis=1))
            for kind in EXACT_FIT:
                m = kind_rows(kinds, (kind,))
                q = e[m] / np.maximum(FP32_EPS * s[m], 1e-300)
                record_err("demand_shapes[exact-fit residual / eps rms]", float(q.max()), 1.0, what=f"{cal} {k} {kind}",
                           rms_resid=float(e[m].max()), rms_centred=float(s[m].max()))
                assert (q <= 1000.0).all(), (cal, k, kind, float(q.max()))    # measured up to 153 (warp, daily)
            assert np.isfinite(e[rows]).all()


# =====================================================================================================================
# AR order selection
# =====================================================================================================================
def test_ar_selection_per_row():
    y, kinds, X, t_fit, ps, npred = _case("daily1095", H, "holdout", n=160)
    orders = tuple(range(AR_MAX + 1))
    n = len(y)
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, True)
    full = _dev(y, y.shape[1])
    got = _np(eng.fit_select_ar(full, H, orders, t_fit, H))
    eng.close()
    want = select_ar_packed(y, X, t_fit, H, orders, t_fit, H)
    tau_fit, tau_hold = _taus(y, X, t_fit, t_fit, H, kinds)
    deg = np.zeros(n, dtype=bool)
    for hres in want["hold"]:
        deg |= degenerate_rows(hres, tau_fit)
    # candidate m is by definition the fixed-order call: its phi sizes the degenerate rows' bound
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, True)
    phis = [np.zeros((n, AR_MAX)) if m == 0 else eng.fit_forecast_ar(full, m, t_fit, H)["phi"].cpu().numpy()
            for m in orders]
    eng.close()
    bound = np.where(deg[:, None], mse_bound(want, y, tau_fit, tau_hold, t_fit, H, orders, phi_gpu=phis),
                     mse_bound(want, y, tau_fit, tau_hold, t_fit, H, orders))
    live = want["status"] != 1
    cm = got["cand_mse"].astype(np.float64)
    assert np.array_equal(np.isnan(cm[live]), np.isnan(want["cand_mse"][live]))
    ok = live[:, None] & ~np.isnan(want["cand_mse"])
    ratio = np.where(ok, np.abs(cm - np.where(ok, want["cand_mse"], 0)) / np.where(bound > 0, bound, np.inf), 0)
    _report("select", ratio.max(axis=1), kinds, "daily1095 holdout 0..8")
    record_err("demand_shapes[select degenerate]", float(ratio[deg].max()), 1.0, count=int(deg.sum()),
               what="candidate MSEs of the degenerate rows / mse_bound with degenerate_bound")
    # the choice is optimal up to the bounds on every scored row
    rows = np.arange(n)
    gidx = np.array([orders.index(c) if c >= 0 else len(orders) - 1 for c in got["choice"]])
    oi = want["idx"]
    scored = live & ~np.isnan(want["cand_mse"]).all(axis=1)
    o_mse = want["cand_mse"]
    over = scored & (o_mse[rows, gidx] > o_mse[rows, oi] + bound[rows, gidx] + bound[rows, oi])
    assert not over.any(), np.flatnonzero(over)[:8]
    # every candidate is the same model on the exactly fit constant rows: bit-equal scores, the first order wins
    ex = kind_rows(kinds, EXACT)
    assert (got["cand_mse"][ex] == got["cand_mse"][ex][:, :1]).all() and (got["choice"][ex] == orders[0]).all()


# =====================================================================================================================
# ARIMA(p, d, 0)
# =====================================================================================================================
@pytest.mark.parametrize("p,d,h", [(0, 1, 28), (0, 2, 28), (1, 1, 28), (1, 2, 28), (2, 1, 28), (2, 2, 28),
                                   (2, 1, 64)])
def test_arima_per_row(p, d, h):
    from test_gpu_arima import _compare
    y, kinds, X, t_fit, ps, npred = _case("daily1095", h, "future", n=160)
    y[-1, 1::2] = np.nan                                   # z' (d >= 1) has no observed fit row: status 1
    want = fit_forecast_arima_packed(y, X, t_fit, ps, npred, p, d)
    zr = want["zres"]
    D = want["D"]
    tz = t_fit - d
    ones = np.ones(len(y))
    mf = _mask_factor(want["z"], D, tz, 0, tz, ones)
    deg = degenerate_rows(zr, np.where(np.isfinite(mf), z_tau(want) * mf, 0.0))
    nd = np.flatnonzero(~deg)
    eng = mmf.ForecastEngine()
    eng.plan_arima(X, t_fit, 2)
    got = _np(eng.fit_forecast_arima(_dev(y, t_fit), p, d, ps, npred))
    eng.close()
    assert got["status"][-1] == 1 and np.isnan(got["pred"][-1]).all()
    assert np.array_equal(got["status"], want["status"])
    sub = dict(want, zres=_take(zr, nd), **{k: want[k][nd] for k in ("pred", "status", "phi", "order", "sigma", "z",
                                                                       "zhat", "ytilde", "obs")})
    _compare(_take(got, nd), sub, t_fit, ps, npred, f"daily1095 p={p} d={d} h={h}")
    # the degenerate rows within the integrated degenerate_bound (future mode: the level error of step j sums the z' errors of
    # steps <= j once (d = 1) or twice (d = 2)); the constant-step walks continue exactly (y_{T-1} + h step)
    lev = forecast_leverage(D, tz, tz, npred)
    tau_fit = np.where(np.isfinite(mf), z_tau(want) * mf, 0.0)
    mp = _mask_factor(want["z"], D, tz, tz, npred, ones)
    tau_pred = np.where(np.isfinite(mp), z_tau(want, lev) * mp, 0.0)
    live = np.flatnonzero((want["status"] != 1) & (deg | kind_rows(kinds, ("walk", "line"))))
    zl = _take(zr, live)
    zl["pred"] = zl["pred"][:, tz:tz + npred]
    bz = degenerate_bound(zl, got["phi"][live], tau_fit[live], tau_pred[live], tz, tz, npred)
    bl = np.cumsum(bz, axis=1) if d == 1 else np.cumsum(np.cumsum(bz, axis=1), axis=1)
    bl += 4 * FP32_EPS * np.abs(want["pred"][live]) * np.arange(1, npred + 1)
    err = np.abs(got["pred"][live].astype(np.float64) - want["pred"][live])
    r_all = (err / bl).max(axis=1)
    dl = deg[live]
    if dl.any():
        record_err("demand_shapes[arima degenerate]", float(r_all[dl].max()), 1.0, count=int(dl.sum()),
                   what=f"p={p} d={d} h={h}", gpu_max_order=int(got["order"][deg].max()),
                   oracle_max_order=int(want["order"][deg].max()),
                   err_over_plain_tol=float((err[dl].max(axis=1) / tau_pred[live][dl]).max()))
    _le(float(r_all.max()), 1.0, f"p={p} d={d} h={h}: degenerate rows / integrated degenerate_bound")
    walk = kind_rows(kinds, ("walk", "line")) & (want["status"] != 1)
    step = y[walk, t_fit - 1].astype(np.float64) - y[walk, t_fit - 2]
    cont = y[walk, t_fit - 1][:, None] + step[:, None] * np.arange(1, npred + 1)[None, :]
    assert np.abs(want["pred"][walk] - cont).max() <= 1e-6 * np.abs(cont).max()
    wl = np.searchsorted(live, np.flatnonzero(walk))
    r = float((np.abs(got["pred"][walk] - cont) / (bl[wl] + 1e-6 * np.abs(cont))).max())
    record_err("demand_shapes[arima walk]", r, 1.0, count=int(walk.sum()), what=f"p={p} d={d} h={h}")
    _le(r, 1.0, f"p={p} d={d} h={h}: constant-step walk vs its exact continuation")


# =====================================================================================================================
# backtest
# =====================================================================================================================
def test_backtest_per_row():
    from test_gpu_backtest import _run
    start, t, freq, X = calendar("daily1095")
    y, kinds, _ = demand_batch(N, "daily1095", seed=5, t_fit=t - 4 * H)
    y[kind_rows(kinds, ("counts_sparse",)), t - H:] = 0.0          # an all-zero scored window
    origin = B.origins(t, H, 4)
    X = O.design_matrix(O.calendar_grid(start, t, freq), t - H)
    eng = mmf.ForecastEngine(device=0)
    got = _run(eng, y, X, origin, H)
    eng.close()
    want, wst, ratio = B.backtest_packed(y, X, origin, H, return_ratio=True)
    _, kappa, lev = B.change_of_basis(X, origin, H)
    worst = np.zeros(len(y))
    for k, tk in enumerate(origin):
        tk = int(tk)
        sure = _pivot_distance(y, X[:tk + H], tk) > PIVOT_BAND
        assert np.array_equal(got["status"][k][sure], wst[k][sure]) and np.array_equal(got["status"][k] == 1, wst[k] == 1)
        ok = wst[k] != 1
        mask = _mask_factor(y[:, :tk], X[:tk + H], tk, tk, H, ratio[k])
        tol = _row_tol(y[:, :tk], max(1.0, lev[k]) * max(1.0, kappa[k])) * mask
        err = np.abs(got["pred"][k] - want[k]).max(axis=1)
        assert np.isnan(got["pred"][k][~ok]).all()
        worst = np.maximum(worst, np.where(ok, err / tol, 0.0) / _slack(kinds))
    _per_kind("backtest", worst * _slack(kinds), kinds, "daily1095 K=4 H=28")
    _report("backtest", worst, kinds, "daily1095 K=4 H=28")
    m, cnt = B.metrics(got["pred"], B.actuals(y, origin, H))
    assert np.array_equal(got["count"], cnt)
    np.testing.assert_allclose(got["metrics"], m, rtol=1e-6, atol=0, equal_nan=True)
    zero = kind_rows(kinds, ("counts_sparse",))
    last = got["metrics"][-1][zero]
    assert np.isnan(last[:, 3]).all() and np.isfinite(last[:, :2]).all() and (got["count"][-1][zero] == H).all()


# =====================================================================================================================
# ragged: a daily and a weekly calendar in one launch
# =====================================================================================================================
def test_ragged_daily_and_weekly_in_one_launch():
    cals = []
    for name in ("daily1095", "weekly157"):
        start, t, freq, X = calendar(name, H)
        y, kinds, _ = demand_batch(150, name, seed=7)
        cals.append((y, kinds, X, t))
    eng = mmf.ForecastEngine()
    eng.plan_designs([c[2] for c in cals], [c[3] for c in cals], [c[3] for c in cals], [H, H], True)
    t_max = max(c[3] for c in cals)
    y = np.full((300, t_max), np.nan, dtype=np.float32)
    y[:150, :cals[0][3]] = cals[0][0]
    y[150:, :cals[1][3]] = cals[1][0]
    yd = _dev(y, t_max)
    res = eng.fit_forecast_ragged(yd, [0, 150, 300], want_status=True)
    single = mmf.ForecastEngine()
    for ci, (yc, kinds, X, t) in enumerate(cals):
        sl = slice(150 * ci, 150 * ci + 150)
        single.plan_designs([X], [t], [t], [H], True)
        r = single.fit_forecast_ragged(_dev(yc, t), [0, 150], want_status=True)
        assert _same_bits(r["pred"], res["pred"][sl]) and _same_bits(r["status"], res["status"][sl]), ci
        orc = _oracle(yc, X, t)
        _report("ragged", _plain_ratio(res["pred"][sl].cpu().numpy(), res["status"][sl].cpu().numpy(), yc, X, t, t, H,
                                       orc, f"cal {ci}", kinds), kinds, f"calendar {ci}")
    single.close()
    eng.close()


# =====================================================================================================================
# integer ingest and host narrowing
# =====================================================================================================================
def _integer_batch(n, t, seed, signed):
    rng = np.random.default_rng(seed)
    y, kinds, _ = demand_batch(n, "daily365", seed=seed)
    keep = kind_rows(kinds, ("counts", "counts_sparse", "zeros", "const1"))
    reg = np.round(np.abs(rng.normal(200, 100, (n, 1))) * (1 + 0.1 * rng.standard_normal((n, t))))
    y = np.where(keep[:, None], y, reg)
    so = rng.random(n) < 0.3                                  # stock-outs: true zeros, and missing on some rows
    for i in np.flatnonzero(so):
        a = int(rng.integers(0, t - 60))
        y[i, a:a + int(rng.integers(7, 61))] = 0.0 if i % 2 else np.nan
    if signed:
        ret = rng.random((n, t)) < 0.05
        y = np.where(ret & np.isfinite(y), -np.abs(y) - 1, y)
    return y.astype(np.float32)


@pytest.mark.parametrize("dtype", ["uint16", "int16", "int32"])
def test_integer_ingest_of_intermittent_demand(dtype):
    t = 365
    start, _, freq, _ = calendar("daily365")
    y = _integer_batch(N, t, seed=11, signed=dtype != "uint16")
    eng = mmf.ForecastEngine(chunk_series=128)
    _, ps, npred = eng.plan_calendar(start, t, "D", H, "future")
    want = eng.fit_forecast(mmf.device_packed(y), ps, npred, want_status=True)
    torch.cuda.synchronize()
    yi = mmf.alloc_packed(N, t, dtype=dtype)
    mmf.to_integer_demand(y, dtype, out=yi)
    res = eng.fit_forecast(yi, ps, npred, want_status=True, want_stats=True)
    assert res["stats"].h2d_bytes == N * t * np.dtype(dtype).itemsize
    assert np.array_equal(res["pred"], want["pred"].cpu().numpy(), equal_nan=True)
    assert np.array_equal(res["status"], want["status"].cpu().numpy())
    eng.close()


def test_host_narrowing_of_intermittent_demand_at_the_uint16_edge():
    """chunks of 128 rows; chunk 2 crosses as float32 by design.  65534 is narrowed; 65535 (the missing-value sentinel)
    sends its chunk as float32; the forecasts equal the device float32 call bit for bit either way"""
    t = 365
    start, _, freq, _ = calendar("daily365")
    n = 512
    y = _integer_batch(n, t, seed=12, signed=False)
    dev = mmf.ForecastEngine()
    _, ps, npred = dev.plan_calendar(start, t, "D", H, "future")
    eng = mmf.ForecastEngine(chunk_series=128, host_narrow="on", host_threads=4)
    eng.plan_calendar(start, t, "D", H, "future")
    for val, row, want_bytes in ((65534.0, 5, (384 * 2 + 128 * 4) * t), (65535.0, 400, (256 * 2 + 256 * 4) * t),
                                 (65535.0, 5, n * t * 4)):
        y2 = y.copy()
        y2[row, 100] = val
        yp = mmf.alloc_packed(n, t)
        yp[...] = y2
        res = eng.fit_forecast(yp, ps, npred, want_status=True, want_stats=True)
        ref = dev.fit_forecast(mmf.device_packed(y2), ps, npred, want_status=True)
        torch.cuda.synchronize()
        assert np.array_equal(res["pred"], ref["pred"].cpu().numpy(), equal_nan=True), (val, row)
        assert np.array_equal(res["status"], ref["status"].cpu().numpy()), (val, row)
        assert res["stats"].h2d_bytes == want_bytes, (val, row, res["stats"].h2d_bytes)
    eng.close()
    dev.close()


# =====================================================================================================================
# negative control: the build without the tensor-core lo term fails the per-row bound on high-level rows
# =====================================================================================================================
_NEGCTL = r"""
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np
import mmf
import test_gpu_demand_shapes as T
from demand_shapes import kind_rows, SCALED
y, kinds, X, t_fit, ps, npred = T._case("daily1095", 28)
orc = T._oracle(y, X, t_fit)
eng = mmf.ForecastEngine(kernel="tc")
eng.plan(X, t_fit, True)
r = T._np(eng.fit_forecast(T._dev(y, t_fit), ps, npred, want_status=True))
ratio = T._plain_ratio(r["pred"], r["status"], y, X, t_fit, ps, npred, orc, "negctl", kinds)
high = kind_rows(kinds, SCALED) & (np.nanmax(np.abs(y), axis=1) >= 1000)
print(json.dumps({{"worst": float(ratio.max()), "high_over": int((ratio[high] > 1).sum()), "high": int(high.sum()),
                  "lib": mmf.LIB_PATH}}))
"""


@pytest.mark.parametrize("lib", ["product", "negctl"])
def test_negative_control_fails_the_per_row_bound(lib):
    env = dict(os.environ)
    env.pop("MMF_LIB", None)
    if lib == "negctl":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_negctl.so")
        assert os.path.exists(env["MMF_LIB"]), "negative-control library missing: run __graft_entry__.build()"
    p = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    got = json.loads(p.stdout.strip().splitlines()[-1])
    record_err("demand_shapes[negative control]", got["worst"], 1.0, what=lib, high_over=got["high_over"])
    if lib == "product":
        assert got["worst"] <= 1.0, got
    else:
        assert got["lib"].endswith("libmmf_negctl.so") and got["high_over"] >= got["high"] // 4, got
