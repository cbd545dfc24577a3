"""GPU (-m gpu): the general contract of the C ABI (include/mmf.h) beyond the calendar defaults the other modules use.
Every case is checked against the float64 oracle O.fit_forecast_packed with the same design, or against a property
that must hold bit for bit.

A. Caller-planned designs (ForecastEngine.plan): p = 1 with and without a constant, p = 5, p = 16 without a constant
   (cond ~ 1e3, level 1e4), aliased columns; t_fit from 1 to 400.  Plan refusals keep the previous plan.
B. Prediction windows anywhere in the design, and bit-equality of a design row's value across windows of one store
   family (fit_tc epilogue, predict_tc_kernel, warp kernel).
C. Caller buffer layouts: y and out as views of wider tensors (the library picks the kernel the layout allows),
   integer views at odd offsets (widen's scalar path), selection on an unaligned y.
D. Mixed residence: every device / host combination of y, out, status and beta through the host pipeline.
E. Long series: fit_warp's shared-memory / global design split at 2,784 rows, and t_fit above 65,535 where the
   tensor-core kernel stops recording gap positions.
F. Argument errors leave the caller's buffers untouched and the context usable.

Every batch mixes rows of all kinds (KINDS), interleaved so that several kinds share a 128-row tile."""
import itertools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import mmf
from conftest import ROOT, forecast_leverage, record_err
from oracle import mmf_oracle as O
from test_gpu_edges import _ill_conditioning, _le, _row_tol, _same_bits

pytestmark = pytest.mark.gpu

H = 28
KINDS = ("clean", "isolated", "leading8", "parity45", "mostly_missing", "single", "empty", "inf")
BATCHES = (1, 127, 129, 301)                  # straddle one 128-row tile
PATTERN = 0x5EEDF00D                          # fill of caller memory the library must not write (a normal float)
FP32_EPS = 2.0 ** -24


def _round4(v):
    return (v + 3) & ~3


def _parity_cols(t_fit, k, parity):
    """the first k positions of [0, t_fit) that lie in 32-column chunks of the given parity (the tensor-core kernel
    counts gaps per chunk parity and records at most 44 per parity in the stream)"""
    c = np.arange(t_fit)
    return c[(c // 32) % 2 == parity][:k]


def _kind_cols(kind, t_fit):
    c = np.arange(t_fit)
    return {"clean": c[:0],
            "isolated": np.unique([t_fit // 5, t_fit // 2, t_fit - 1]),
            "leading8": c[:8],                                   # no centring constant: the general pass
            "parity45": _parity_cols(t_fit, 45, 0),              # one gap more than a parity's in-stream record
            "mostly_missing": c[c % 3 != 0],
            "single": c[c != t_fit // 2],
            "empty": c,
            "inf": np.array([t_fit // 3])}[kind]


def _plant(y, t_fit, shift=0, kinds=KINDS):
    """in place on a numpy [n, >= t_fit] float32 batch: row i gets kind kinds[(i + shift) % len(kinds)]"""
    for i in range(y.shape[0]):
        kind = kinds[(i + shift) % len(kinds)]
        y[i, _kind_cols(kind, t_fit)] = np.inf if kind == "inf" else np.nan
    return y


def _mask_factor(y, X, t_fit, ps, npred, ratio):
    """test_gpu_edges._mask_factor for a design of any width p: 1/min(1, ratio/0.25) or, where larger, the forward-error
    amplification of the row's own normal equations on the columns the oracle keeps.  Gap-free rows get 1."""
    X = np.asarray(X, dtype=np.float64)
    p = X.shape[1]
    W, _ = O.whiten(X[:t_fit])
    A = X @ W
    a_fit, a_pred = A[:t_fit], A[ps:ps + npred]
    lev = max(1.0, forecast_leverage(X, t_fit, ps, npred))
    out = _ill_conditioning(ratio)
    cache = {}
    for i, row in enumerate(np.asarray(y)[:, :t_fit]):
        obs = np.isfinite(row)
        if obs.all() or not obs.any():
            continue
        key = obs.tobytes()
        if key not in cache:
            G = a_fit[obs].T @ a_fit[obs]
            keep, L = [], np.zeros((p, p))
            for j in range(p):                               # the oracle's in-order pivot dropping (O.solve_series)
                d = G[j, j] - L[j, :j] @ L[j, :j] if G[j, j] > 0 else 0.0
                if G[j, j] <= 0 or d <= O.PIVOT_TOL * G[j, j]:
                    continue
                keep.append(j)
                L[j, j] = np.sqrt(d)
                L[j + 1:, j] = (G[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
            if not keep:
                cache[key] = 1.0
            else:
                Gk = G[np.ix_(keep, keep)]
                lam = max(float(np.linalg.eigvalsh(Gk)[0]), 1e-300)
                ak = a_pred[:, keep]
                lev_i = float(np.sqrt(np.einsum("ij,ij->i", ak @ np.linalg.inv(Gk), ak)).max())
                cache[key] = max(1.0, lev_i / lev) / np.sqrt(min(1.0, lam / 0.25))
        out[i] = max(out[i], cache[key])
    return out


def _oracle(y, X, t_fit):
    """(gamma [n, p], status, ratio, A = X W): the oracle's fit, from which any window's prediction is gamma A_w^T"""
    _, status, gamma, ratio = O.fit_forecast_packed(y, X, t_fit, 0, 1, return_gamma=True)
    W, _ = O.whiten(np.asarray(X, dtype=np.float64)[:t_fit])
    return dict(gamma=gamma, status=status, ratio=ratio, A=np.asarray(X, dtype=np.float64) @ W)


def _check(pred, status, y, X, t_fit, ps, npred, what, orc, scale=1.0):
    """statuses equal the oracle's, NaN rows exactly for status 1, every other row within
    tolerance(row, leverage) x mask factor x scale"""
    want = orc["gamma"] @ orc["A"][ps:ps + npred].T
    wst = orc["status"]
    assert np.array_equal(status, wst), (what, np.flatnonzero(status != wst)[:8], status[status != wst][:8])
    empty = wst == 1
    assert np.isnan(pred[empty]).all() and np.isfinite(pred[~empty]).all(), what
    if (~empty).any():
        tol = (_row_tol(y[:, :t_fit], forecast_leverage(X, t_fit, ps, npred))
               * _mask_factor(y, X, t_fit, ps, npred, orc["ratio"]) * scale)
        err = np.abs(pred[~empty] - want[~empty]).max(axis=1) / tol[~empty]
        _le(float(err.max()), 1.0, f"{what}: worst row error / row tolerance")


def _check_beta(beta, y, X, t_fit, orc, what):
    """X beta against the oracle's fitted values on the fit rows (test_beta_reproduces_fitted_values).  beta itself is
    not compared: with an ill-conditioned X it is large.  Forming beta = W gamma in fp32 (W rounded to fp32, 16-term
    sums) and evaluating X beta adds up to ~32 eps * sum_p |X_tp| (|beta_p| + sum_q |W_pq gamma_q|) per row; the bound
    allows twice that on top of 5x the row tolerance.  Columns beyond p are exactly zero, empty rows NaN."""
    X = np.asarray(X, dtype=np.float64)
    p = X.shape[1]
    live = orc["status"] != 1
    assert np.isnan(beta[~live]).all(), what
    assert not beta[live, p:].any(), what
    if not live.any():
        return
    W, _ = O.whiten(X[:t_fit])
    Xf = X[:t_fit]
    b = beta[live, :p].astype(np.float64)
    g = orc["gamma"][live]
    fitted = b @ Xf.T
    want = g @ orc["A"][:t_fit].T
    mag = np.abs(b) + np.abs(g[:, None, :] * W[None, :p, :p]).sum(axis=2)
    rounding = 64 * FP32_EPS * (mag @ np.abs(Xf).T).max(axis=1)
    tol = (5 * _row_tol(y[live][:, :t_fit]) * _mask_factor(y[live], X, t_fit, 0, t_fit, orc["ratio"][live])
           + rounding)
    _le(float((np.abs(fitted - want).max(axis=1) / tol).max()), 1.0, f"{what}: X beta vs fitted values / bound")


def _engines(**kw):
    return {k: mmf.ForecastEngine(kernel=k, **kw) for k in ("auto", "tc", "warp")}


def _close(engs):
    for e in engs.values():
        e.close()


def _np(res):
    return {k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in res.items() if k != "stats"}


# =====================================================================================================================
# A. caller-planned designs
# =====================================================================================================================
def _design(name, n_rows, t_fit, seed=0):
    """(X [n_rows, p], has_constant) of a caller-planned design"""
    t = np.arange(n_rows, dtype=np.float64)
    one = np.ones(n_rows)
    trend = (t - (t_fit - 1) / 2.0) / t_fit
    p5 = np.column_stack([one, trend, np.sqrt(t / t_fit), np.sin(2 * np.pi * t / 30.5), np.cos(2 * np.pi * t / 30.5)])
    if name == "mean":                                   # intercept only: the forecast is the mean of the fit values
        return one[:, None], True
    if name == "t1":                                     # one column x_t = t + 1, no constant
        return (t + 1.0)[:, None], False
    if name == "p5":
        return p5, True
    if name == "gauss16":                                # cond ~ 1e3, no constant
        rng = np.random.default_rng(seed)
        U, _ = np.linalg.qr(rng.normal(size=(16, 16)))
        V, _ = np.linalg.qr(rng.normal(size=(16, 16)))
        return rng.normal(size=(n_rows, 16)) @ (U * np.logspace(0, -3, 16)) @ V.T, False
    extra = {"dup": trend,                               # a duplicated column
             "zero": np.zeros(n_rows),                   # an all-zero column
             "fit_zero": (t >= t_fit).astype(np.float64),   # zero on the fit rows only: aliased, contributes nothing
             "twice_one": 2.0 * one}[name]               # 2 x the intercept
    return np.column_stack([p5, extra]), True


def _series(X, t_fit, n, seed, level):
    rng = np.random.default_rng(seed)
    coef = rng.normal(0.0, 1.0, (n, X.shape[1]))
    y = level + 0.05 * level * (coef @ X[:t_fit].T) + rng.normal(0.0, 0.02 * level, (n, t_fit))
    return y.astype(np.float32)


A_DESIGNS = ("mean", "t1", "p5", "gauss16", "dup", "zero", "fit_zero", "twice_one")
T_FITS = (1, 2, 7, 8, 9, 31, 32, 33, 64, 65, 400)


@pytest.mark.parametrize("name", A_DESIGNS)
def test_planned_design_matches_oracle(name):
    """every t_fit with the window [t_fit, t_fit + 28): tc and warp against the oracle (forecasts, statuses, X beta),
    auto bit-equal to tc, whitening() reports the oracle's kept set"""
    import torch
    engs = _engines()
    for i, t_fit in enumerate(T_FITS):
        X, has_c = _design(name, t_fit + H, t_fit, seed=i)
        p = X.shape[1]
        n = BATCHES[i % len(BATCHES)]
        y = _plant(_series(X, t_fit, n, 100 + i, 1e4 if name == "gauss16" else 500.0), t_fit, shift=i)
        yd = mmf.device_packed(y)
        what = f"{name} t_fit={t_fit} n={n}"
        kept_o = O.whiten(X[:t_fit])[1]
        got = {}
        for k, eng in engs.items():
            eng.plan(X, t_fit, has_c)
            kept = eng.whitening()[1]
            assert np.array_equal(kept[:p], kept_o) and not kept[p:].any(), (what, k, kept, kept_o)
            got[k] = eng.fit_forecast(yd, t_fit, H, want_status=True, want_beta=True, want_stats=True)
        torch.cuda.synchronize()
        assert got["auto"]["stats"].kernel_used == "tc", what
        for key in ("pred", "status", "beta"):
            assert _same_bits(got["auto"][key], got["tc"][key]), (what, key)
        orc = _oracle(y, X, t_fit)
        for k in ("tc", "warp"):
            r = _np(got[k])
            _check(r["pred"], r["status"], y, X, t_fit, t_fit, H, f"{what} {k}", orc)
            _check_beta(r["beta"], y, X, t_fit, orc, f"{what} {k}")
            if name == "mean":                           # closed form: the mean of the observed fit values
                live = orc["status"] != 1
                yf = np.where(np.isfinite(y[:, :t_fit]), y[:, :t_fit], np.nan).astype(np.float64)
                mean = np.nanmean(yf[live], axis=1)
                err = np.abs(r["pred"][live] - mean[:, None]).max(axis=1) / _row_tol(y[live][:, :t_fit])
                _le(float(err.max()), 1.0, f"{what} {k}: forecast vs mean of the observed fit values")
    _close(engs)


def test_plan_refusals_keep_the_previous_plan():
    """plan() refuses p = 0 and 17, t_fit > n_rows, a NaN in X and has_constant = 1 with X[k, 0] != 1 (MMF_E_INVALID);
    the plan before the refusal stays in force: the next call is bit-equal to the one before it"""
    import torch
    t_fit = 400
    X, _ = _design("p5", t_fit + H, t_fit)
    y = _plant(_series(X, t_fit, 301, 7, 500.0), t_fit)
    yd = mmf.device_packed(y)
    nan_x = X.copy()
    nan_x[17, 3] = np.nan
    not_one = X.copy()
    not_one[t_fit + 3, 0] = 1.5                          # a forecast row: the check covers every row
    bad = {"p=0": (np.zeros((t_fit + H, 0)), t_fit, False), "p=17": (np.ones((t_fit + H, 17)), t_fit, False),
           "t_fit > n_rows": (X, t_fit + H + 1, True), "NaN in X": (nan_x, t_fit, True),
           "X[k,0] != 1": (not_one, t_fit, True)}
    for kernel in ("auto", "warp"):
        eng = mmf.ForecastEngine(kernel=kernel)
        eng.plan(X, t_fit, True)
        before = eng.fit_forecast(yd, t_fit, H, want_status=True, want_beta=True)
        for what, (Xb, tf, hc) in bad.items():
            with pytest.raises(mmf.MmfError) as e:
                eng.plan(Xb, tf, hc)
            assert e.value.code == -1, (kernel, what, str(e.value))
            after = eng.fit_forecast(yd, t_fit, H, want_status=True, want_beta=True)
            torch.cuda.synchronize()
            for k in ("pred", "status", "beta"):
                assert _same_bits(before[k], after[k]), (kernel, what, k)
        eng.close()


# =====================================================================================================================
# B. prediction windows
# =====================================================================================================================
def _product_design(t_fit, n_rows, start="2019-01-01"):
    return O.design_matrix(O.calendar_grid(np.datetime64(start), n_rows, "D"), t_fit), True


def _windows(t_fit, n_rows):
    return [(0, 1), (5, 3), (17, 4), (t_fit - 1, 1), (t_fit - 3, 7), (t_fit, 28), (t_fit + 4, 24), (t_fit, 29),
            (0, 64), (0, 65), (100, 128), (100, 129), (0, n_rows), (n_rows - 1, 1)]


def _table_from_windows(eng, yd, n_rows, width):
    """[n, n_rows] table assembled from windows of at most `width` rows"""
    import torch
    parts = [eng.fit_forecast(yd, s, min(width, n_rows - s)) for s in range(0, n_rows, width)]
    return torch.cat(parts, dim=1)


@pytest.mark.parametrize("name", ["product", "p5"])
def test_prediction_windows(name):
    """Every window with auto, tc and warp against the oracle; auto bit-equal to tc.  Window independence: within one
    store family a design row's value is the same 16-term fma chain (fit_tc epilogue / solve_rows / fit_warp: dot16
    from c in column order; predict_tc_kernel: one wgmma accumulation per output column, whatever the column's place
    in the B tile), so every window is bit-equal to the slice of a reference table of its family:
      fit_tc epilogue (n_pred <= 64): a table assembled from 64-row windows;
      predict_tc_kernel (n_pred > 64): the tc window (0, n_rows);
      warp kernel: the warp window (0, n_rows).
    The product design has 401 rows (t_fit = 372) so that (t_fit, 29) is a valid window."""
    import torch
    t_fit, n_rows, n = 372, 401, 301
    X, has_c = _product_design(t_fit, n_rows) if name == "product" else _design("p5", n_rows, t_fit)
    if name == "product":
        y, _ = mmf.synth.daily_store_item_demand(n, t_fit, seed=71)
    else:
        y = _series(X, t_fit, n, 71, 500.0)
    _plant(y, t_fit, shift=3)
    yd = mmf.device_packed(y)
    engs = _engines()
    for eng in engs.values():
        eng.plan(X, t_fit, has_c)
    ref = {"fit_tc": _table_from_windows(engs["tc"], yd, n_rows, 64),
           "predict_tc": engs["tc"].fit_forecast(yd, 0, n_rows),
           "warp": engs["warp"].fit_forecast(yd, 0, n_rows)}
    torch.cuda.synchronize()
    orc = _oracle(y, X, t_fit)
    for ps, npred in _windows(t_fit, n_rows):
        got = {k: eng.fit_forecast(yd, ps, npred, want_status=True) for k, eng in engs.items()}
        torch.cuda.synchronize()
        w = f"{name} window ({ps}, {npred})"
        assert _same_bits(got["auto"]["pred"], got["tc"]["pred"]), w
        assert _same_bits(got["auto"]["status"], got["tc"]["status"]), w
        fam = "fit_tc" if npred <= 64 else "predict_tc"
        assert torch.equal(got["tc"]["pred"].contiguous().view(torch.int32),
                           ref[fam][:, ps:ps + npred].contiguous().view(torch.int32)), (w, fam)
        assert torch.equal(got["warp"]["pred"].contiguous().view(torch.int32),
                           ref["warp"][:, ps:ps + npred].contiguous().view(torch.int32)), (w, "warp")
        for k in ("tc", "warp"):
            r = _np(got[k])
            _check(r["pred"], r["status"], y, X, t_fit, ps, npred, f"{w} {k}", orc)
    _close(engs)


# =====================================================================================================================
# C. caller buffer layouts (device)
# =====================================================================================================================
def _layout_batch(n=301, t=373, seed=5):
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=seed)
    return _plant(y, t, shift=1), start


@pytest.mark.parametrize("s", [0, 1, 2, 3])
def test_y_view_of_a_wider_tensor(s):
    """y = big[1:n+1, s:s+t] of a NaN-filled tensor (guard rows above and below, NaN beside the view): auto is bit-equal
    to the tc engine on an aligned copy where the view is TMA-loadable (s % 4 == 0, pitch % 4 == 0) and to the warp
    engine otherwise, where kernel="tc" is refused on the host with the reason.  A read outside the view would show
    up as a changed status or a NaN forecast."""
    import torch
    t = 373
    y, start = _layout_batch(t=t)
    n = y.shape[0]
    X, has_c = _product_design(t, t + H, str(start))
    engs = _engines()
    for eng in engs.values():
        eng.plan(X, t, has_c)
    packed = mmf.device_packed(y)
    ref = {k: engs[k].fit_forecast(packed, t, H, want_status=True, want_beta=True) for k in ("tc", "warp")}
    torch.cuda.synchronize()
    orc = _oracle(y, X, t)
    for k in ("tc", "warp"):
        r = _np(ref[k])
        _check(r["pred"], r["status"], y, X, t, t, H, f"packed copy {k}", orc)
    for pitch in (s + t, _round4(s + t), _round4(s + t) + 4, s + t + 37):
        big = torch.full((n + 2, pitch), float("nan"), device="cuda")
        big[1:n + 1, s:s + t] = torch.from_numpy(y).cuda()
        view = big[1:n + 1, s:s + t]
        aligned = s % 4 == 0 and pitch % 4 == 0
        got = engs["auto"].fit_forecast(view, t, H, want_status=True, want_beta=True, want_stats=True)
        torch.cuda.synchronize()
        fam = "tc" if aligned else "warp"
        assert got["stats"].kernel_used == fam, (s, pitch)
        for k in ("pred", "status", "beta"):
            assert _same_bits(got[k], ref[fam][k]), (s, pitch, k)
        if aligned:
            tc = engs["tc"].fit_forecast(view, t, H, want_status=True)
            torch.cuda.synchronize()
            assert _same_bits(tc["pred"], ref["tc"]["pred"]), (s, pitch)
        else:
            with pytest.raises(mmf.MmfError) as e:
                engs["tc"].fit_forecast(view, t, H)
            assert e.value.code == -3, str(e.value)
            reason = "ld_y not a multiple of 4" if pitch % 4 else "y not 16-B aligned"
            assert reason in str(e.value), (s, pitch, str(e.value))
        del big, view
    _close(engs)


@pytest.mark.parametrize("n_pred", [1, 7, 28, 64, 65, 300])
def test_out_window_of_a_wider_table(n_pred):
    """out = table[1:n+1, o:o+n_pred] of a pattern-filled table, o in {0, 1, 3, 4}, pitch o + n_pred, the next multiple
    of 4, and that + 5.  Nothing outside the window changes, also on the rows the fix-up kernels rewrite and in the
    columns between n_pred and the next multiple of 4 (TMA stores of predict_tc_kernel clip at n_pred).  The window is
    bit-equal to a contiguous out of the same store family; n_pred > 64 with an out that predict_tc_kernel cannot
    store (base not 16-B aligned or pitch % 4 != 0) goes to the warp kernel, and kernel="tc" is refused."""
    import torch
    t_fit, n_rows = 372, 401
    y, start = _layout_batch(t=t_fit, seed=6)
    n = y.shape[0]
    X, has_c = _product_design(t_fit, n_rows, str(start))
    ps = t_fit if n_pred <= n_rows - t_fit else 0
    engs = _engines()
    for eng in engs.values():
        eng.plan(X, t_fit, has_c)
    yd = mmf.device_packed(y)
    ref = {k: engs[k].fit_forecast(yd, ps, n_pred, want_status=True) for k in ("auto", "warp")}
    torch.cuda.synchronize()
    orc = _oracle(y, X, t_fit)
    for k in ("auto", "warp"):
        r = _np(ref[k])
        _check(r["pred"], r["status"], y, X, t_fit, ps, n_pred, f"contiguous out {k} n_pred={n_pred}", orc)
    for o in (0, 1, 3, 4):
        for pitch in (o + n_pred, _round4(o + n_pred), _round4(o + n_pred) + 5):
            table = torch.full((n + 2, pitch), PATTERN, dtype=torch.int32, device="cuda")
            out = table.view(torch.float32)[1:n + 1, o:o + n_pred]
            aligned = o % 4 == 0 and pitch % 4 == 0
            fam = "warp" if (n_pred > 64 and not aligned) else "auto"
            status = torch.empty(n, dtype=torch.int32, device="cuda")
            engs["auto"].fit_forecast(yd, ps, n_pred, out=out, status=status)
            torch.cuda.synchronize()
            w = (n_pred, o, pitch)
            assert _same_bits(out, ref[fam]["pred"]) and _same_bits(status, ref[fam]["status"]), w
            outside = torch.ones_like(table, dtype=torch.bool)
            outside[1:n + 1, o:o + n_pred] = False
            assert bool((table[outside] == PATTERN).all()), (w, "caller memory outside the window changed")
            if n_pred > 64 and not aligned:
                with pytest.raises(mmf.MmfError) as e:
                    engs["tc"].fit_forecast(yd, ps, n_pred, out=out)
                assert e.value.code == -3 and "n_pred > 64" in str(e.value), (w, str(e.value))
            del table, out
    _close(engs)


@pytest.mark.parametrize("dtype", ["int16", "int32"])
def test_device_integer_views_at_an_odd_offset(dtype):
    """an integer series buffer on the device as a view at element offset 1 with an odd pitch (widen's scalar path):
    bit-equal to the float32 call on a packed copy.  Missing-value sentinels in the first and the last column and in
    the whole last row."""
    import torch
    t, n = 372, 301
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=12)
    miss = np.zeros(y.shape, dtype=bool)
    miss[:, 0] = miss[:, -1] = miss[-1, :] = True
    miss[5::9, 100:105] = True
    vals = np.clip(np.rint(np.where(np.isfinite(y), y, 0.0)), 0, 30000)
    sentinel = mmf._native.INT_MISSING[dtype]
    yi = np.where(miss, sentinel, vals).astype(dtype)
    yf = np.where(miss, np.nan, vals).astype(np.float32)
    tdt = {"int16": torch.int16, "int32": torch.int32}[dtype]
    pitch = t + 3                                          # odd
    big = torch.full((n, pitch), 4321, dtype=tdt, device="cuda")
    big[:, 1:1 + t] = torch.from_numpy(yi).cuda()
    view = big[:, 1:1 + t]
    for kernel in ("auto", "warp"):
        eng = mmf.ForecastEngine(kernel=kernel)
        eng.plan_calendar(start, t, "D", H, "future")
        got = eng.fit_forecast(view, t, H, want_status=True, want_beta=True)
        want = eng.fit_forecast(mmf.device_packed(yf), t, H, want_status=True, want_beta=True)
        torch.cuda.synchronize()
        for k in ("pred", "status", "beta"):
            assert _same_bits(got[k], want[k]), (dtype, kernel, k)
        eng.close()


def test_selection_on_an_unaligned_y_view():
    """fit_select_forecast on y = big[1:n+1, 1:t+1] (ld_y = t + 3, odd): bit-equal to the warp engine on a packed copy"""
    import torch
    n, t, h = 301, 400, 28
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=13)
    _plant(y, t - h, shift=2)
    big = torch.full((n + 2, t + 3), float("nan"), device="cuda")
    big[1:n + 1, 1:t + 1] = torch.from_numpy(y).cuda()
    view = big[1:n + 1, 1:t + 1]
    cands = (1, 3, 9, 13, 16)
    auto, warp = mmf.ForecastEngine(), mmf.ForecastEngine(kernel="warp")
    for eng in (auto, warp):
        eng.plan_calendar(start, t, "D", h, "holdout")
    got = auto.fit_select_forecast(view, h, cands, 0, t)
    want = warp.fit_select_forecast(mmf.device_packed(y), h, cands, 0, t)
    torch.cuda.synchronize()
    for k in ("pred", "choice", "mse", "status"):
        assert _same_bits(got[k], want[k]), k
    auto.close()
    warp.close()


# =====================================================================================================================
# D. mixed residence (host pipeline)
# =====================================================================================================================
def _host_view_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), np.ascontiguousarray(b).view(np.int32))


def test_mixed_residence_is_bit_equal_to_the_device_call():
    """chunk_series = 700, 2,501 rows (four chunks, a short last one): every device / host combination of y, out,
    status and beta (pageable host memory), pinned y and out, and a y pinned with mmf_host_register: pred, status and
    beta bit-equal to the all-device call, h2d / d2h bytes exactly what the combination moves, and a host out with
    ld_out > n_pred keeps its pad columns (the 2-D copy back)."""
    import torch
    n, t = 2501, 365
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=21)
    _plant(y, t, shift=5)
    eng = mmf.ForecastEngine(chunk_series=700, host_narrow="off")
    eng.plan_calendar(start, t, "D", H, "future")
    yd = mmf.device_packed(y)
    ref = _np(eng.fit_forecast(yd, t, H, want_status=True, want_beta=True))
    torch.cuda.synchronize()
    X, _ = _product_design(t, t + H, str(start))
    _check(ref["pred"], ref["status"], y, X, t, t, H, "all device", _oracle(y, X, t))

    def run(yb, o_dev, s_dev, b_dev, host_out=None):
        table = None
        if o_dev:
            out = torch.empty((n, H), device="cuda")
        elif host_out is not None:
            out = host_out
        else:
            table = np.full((n, H + 3), PATTERN, dtype=np.int32)
            out = table.view(np.float32)[:, :H]
        status = torch.empty(n, dtype=torch.int32, device="cuda") if s_dev else np.empty(n, dtype=np.int32)
        beta = torch.empty((n, 16), device="cuda") if b_dev else np.empty((n, 16), dtype=np.float32)
        res = eng.fit_forecast(yb, t, H, out=out, status=status, beta=beta, want_stats=True)
        torch.cuda.synchronize()
        got = _np(res)
        for k in ("pred", "status", "beta"):
            assert _host_view_equal(got[k], ref[k]), k
        if table is not None:
            assert (table[:, H:] == PATTERN).all(), "pad columns of the host table changed"
        return res["stats"]

    for y_dev, o_dev, s_dev, b_dev in itertools.product((True, False), repeat=4):
        what = dict(y=y_dev, out=o_dev, status=s_dev, beta=b_dev)
        st = run(yd if y_dev else np.ascontiguousarray(y), o_dev, s_dev, b_dev)
        want_h2d = 0 if y_dev else n * t * 4
        want_d2h = (0 if o_dev else n * H * 4) + (0 if s_dev else n * 4) + (0 if b_dev else n * 16 * 4)
        assert (st.h2d_bytes, st.d2h_bytes) == (want_h2d, want_d2h), what
    yp = mmf.alloc_packed(n, t)                         # pinned, 16-B pitch
    yp[...] = y
    op = mmf.alloc_packed(n, H)
    st = run(yp, False, True, False, host_out=op)
    assert (st.h2d_bytes, st.d2h_bytes) == (n * t * 4, n * H * 4 + n * 16 * 4)
    lib = mmf._native.load()
    buf = np.empty(n * t + 1024, dtype=np.float32)      # page-aligned, registered in place
    off = (-buf.ctypes.data % 4096) // 4
    yr = buf[off:off + n * t].reshape(n, t)
    yr[...] = y
    mmf._native.check(lib.mmf_host_register(yr.ctypes.data, yr.nbytes))
    try:
        st = run(yr, False, False, True)
        assert (st.h2d_bytes, st.d2h_bytes) == (n * t * 4, n * H * 4 + n * 4)
    finally:
        mmf._native.check(lib.mmf_host_unregister(yr.ctypes.data))
    eng.close()


# =====================================================================================================================
# E. long series
# =====================================================================================================================
# conftest.tolerance was derived for ~10^3 accumulated terms.  fp32 summation error grows about as sqrt(terms) as long
# as no single sum runs over the whole series, so the long series get tolerance x sqrt(max(1, t_fit / 1095)), for
# every kernel.  Before fit_tc restarted its wgmma accumulators every 18 chunks (and fit_warp its direct Gram sums every
# 2,048 positions) the error grew linearly instead: 36x the conftest tolerance on gap-free rows at 70,001 rows through
# the tensor-core kernel, 8.2x on mostly-missing rows through the warp kernel's general pass.  The negative-control
# build without the lo*A_hi term must still exceed the scaled bound at 70,001 rows
# (test_negative_control_exceeds_the_scaled_long_series_bound).
def _long_scale(t_fit):
    return float(np.sqrt(max(1.0, t_fit / 1095.0)))


SMEM_ROWS = 2784          # fit_warp_smem_bytes: (200 KB - 16 x 1,608 B of WarpScratch) / 64 B, a multiple of 32
LONG_KINDS = ("clean", "split", "last", "seg44", "seg45", "leading8", "inf", "mostly_missing", "empty")


def _hourly(n_rows, t_fit):
    """p = 6: intercept, trend, sin / cos with periods 24 and 168 (hourly data, daily and weekly cycle)"""
    t = np.arange(n_rows, dtype=np.float64)
    w = 2 * np.pi * t
    return np.column_stack([np.ones(n_rows), (t - (t_fit - 1) / 2.0) / t_fit, np.sin(w / 24), np.cos(w / 24),
                            np.sin(w / 168), np.cos(w / 168)])


def _long_cols(kind, t_fit):
    c = np.arange(t_fit)
    if kind == "split":       # both sides of fit_warp's shared-memory rows and of the uint16 position range
        return np.array([v for v in (100, 2700, 2783, 2784, 2790, 3500, 65535, 65536, 65600, t_fit - 2) if v < t_fit])
    if kind == "last":
        return np.array([t_fit - 1])
    if kind == "seg44":
        return _parity_cols(t_fit, 44, 0)
    if kind == "seg45":
        return _parity_cols(t_fit, 45, 1)
    return _kind_cols(kind, t_fit)


def _long_batch(n, t_fit, seed, kinds=LONG_KINDS):
    rng = np.random.default_rng(seed)
    X = _hourly(t_fit, t_fit)
    level = rng.uniform(200.0, 2000.0, (n, 1))
    coef = np.column_stack([np.zeros(n), rng.normal(0, 0.3, n), rng.normal(0, 0.3, n), rng.normal(0, 0.3, n),
                            rng.normal(0, 0.2, n), rng.normal(0, 0.2, n)])
    y = (level * (1.0 + coef @ X.T) + rng.normal(0, 1.0, (n, t_fit)) * np.sqrt(level)).astype(np.float32)
    for i in range(n):
        kind = kinds[i % len(kinds)]
        y[i, _long_cols(kind, t_fit)] = np.inf if kind == "inf" else np.nan
    return y


def _expected_pending(y, t_fit, has_constant=True):
    """rows the tensor-core kernel hands to the general pass (DESIGN.md 4.2): up to t_fit = 65,535 the rows without a
    centring constant (first 8 missing; only a design with a constant centres), with more than 44 gaps in one chunk
    parity or more than half the fit rows missing; above it gap positions are not recorded and every row with a
    missing fit value goes there"""
    bad = ~np.isfinite(y[:, :t_fit])
    if t_fit > 65535:
        return int(bad.any(axis=1).sum())
    seg = (np.arange(t_fit) // 32) % 2
    nm0, nm1 = bad[:, seg == 0].sum(axis=1), bad[:, seg == 1].sum(axis=1)
    no_centre = bad[:, :8].all(axis=1) & has_constant
    return int((no_centre | (nm0 > 44) | (nm1 > 44) | (2 * (nm0 + nm1) > t_fit)).sum())


@pytest.mark.parametrize("t_fit", [2783, 2784, 2785, 4000])
def test_long_series_across_the_shared_memory_design_rows(t_fit):
    """hourly design, 257 rows: holdout (every design row, n_pred > 64) and future (28 rows past t_fit) with the warp
    kernel, which stages 2,784 design rows in shared memory and reads the rest from global memory, with tc, and with
    auto (bit-equal to tc)"""
    import torch
    n = 257
    y = _long_batch(n, t_fit, seed=t_fit)
    yd = mmf.device_packed(y)
    for mode in ("holdout", "future"):
        n_rows = t_fit + H
        X = _hourly(n_rows, t_fit)
        ps, npred = (0, n_rows) if mode == "holdout" else (t_fit, H)
        orc = _oracle(y, X, t_fit)
        engs = _engines()
        got = {}
        for kernel, eng in engs.items():
            eng.plan(X, t_fit, True)
            got[kernel] = eng.fit_forecast(yd, ps, npred, want_status=True)
        torch.cuda.synchronize()
        for k in ("pred", "status"):
            assert _same_bits(got["auto"][k], got["tc"][k]), (t_fit, mode, k)
        for kernel in ("warp", "tc"):
            r = _np(got[kernel])
            _check(r["pred"], r["status"], y, X, t_fit, ps, npred, f"t_fit={t_fit} {mode} {kernel}", orc,
                   scale=_long_scale(t_fit))
        _close(engs)


def _long_case(t_fit, kernels, kinds=LONG_KINDS, holdout=False, n=257, seed=None):
    """fit a batch of 257 hourly rows with t_fit values each with every kernel in `kernels`
    -> (y, X, t_fit, ps, npred, {kernel: (result as numpy, stats)})"""
    import torch
    if holdout:                                    # every one of t_fit values of the calendar, 28 of them held out
        n_rows, tf, ps, npred = t_fit, t_fit - H, 0, t_fit
    else:
        n_rows, tf, ps, npred = t_fit + H, t_fit, t_fit, H
    y = _long_batch(n, tf, seed=seed if seed is not None else t_fit, kinds=kinds)
    X = _hourly(n_rows, tf)
    yd = mmf.device_packed(y)
    out = {}
    for kernel in kernels:
        eng = mmf.ForecastEngine(kernel=kernel)
        eng.plan(X, tf, True)
        res = eng.fit_forecast(yd, ps, npred, want_status=True, want_stats=True)
        torch.cuda.synchronize()
        out[kernel] = (_np(res), res["stats"])
        eng.close()
    return y, X, tf, ps, npred, out


def _assert_auto_is_tc(out, what):
    a, t = out["auto"][0], out["tc"][0]
    for k in ("pred", "status"):
        assert np.array_equal(a[k].view(np.int32), t[k].view(np.int32)), (what, k)


@pytest.mark.parametrize("t_fit", [65535, 65536, 70001])
def test_long_series_beyond_the_uint16_gap_positions(t_fit):
    """future h = 28 with tc (tensor-core kernel + fix-up), auto (bit-equal to tc) and warp: rows with a gap at
    t_fit - 1, gaps at positions >= 65,536, 44 and 45 gaps in one chunk parity, ...  stats.n_pending follows the rule
    of _expected_pending."""
    y, X, tf, ps, npred, out = _long_case(t_fit, ("auto", "tc", "warp"))
    _assert_auto_is_tc(out, t_fit)
    orc = _oracle(y, X, tf)
    for kernel in ("tc", "warp"):
        r, _ = out[kernel]
        _check(r["pred"], r["status"], y, X, tf, ps, npred, f"t_fit={t_fit} future {kernel}", orc,
               scale=_long_scale(tf))
    stats = out["auto"][1]
    assert stats.kernel_used == "tc"
    assert stats.n_pending == _expected_pending(y, tf), (stats.n_pending, _expected_pending(y, tf))


def test_long_series_holdout_through_the_predict_kernel():
    """70,001 values per row (t_fit = 69,973): predict_tc_kernel writes every date; auto bit-equal to tc"""
    y, X, tf, ps, npred, out = _long_case(70001, ("auto", "tc"), holdout=True)
    _assert_auto_is_tc(out, "holdout")
    r, stats = out["auto"]
    _check(r["pred"], r["status"], y, X, tf, ps, npred, "holdout 70,001", _oracle(y, X, tf), scale=_long_scale(tf))
    assert stats.kernel_used == "tc" and stats.n_pending == _expected_pending(y, tf)


def _long_error(t_fit, kernel):
    """worst error / scaled tolerance of the gap-free rows of a future call (the negative control runs this too)"""
    y, X, tf, ps, npred, out = _long_case(t_fit, (kernel,), kinds=("clean",), n=129, seed=3)
    orc = _oracle(y, X, tf)
    want = orc["gamma"] @ orc["A"][ps:ps + npred].T
    tol = _row_tol(y, forecast_leverage(X, tf, ps, npred)) * _long_scale(tf)
    return float((np.abs(out[kernel][0]["pred"] - want).max(axis=1) / tol).max())


_NEGCTL = r"""
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import test_gpu_abi_contract as T
print(json.dumps({{"ratio": T._long_error(70001, "tc")}}))
"""


def test_negative_control_exceeds_the_scaled_long_series_bound():
    """the build without the lo*A_hi tensor-core term (tests/_build/libmmf_negctl.so) must exceed the tolerance scaled
    by sqrt(t_fit / 1095) on the 70,001-row case, or the larger bound would no longer guard the tf32 split; the product
    must stay within it"""
    neg = os.path.join(ROOT, "tests", "_build", "libmmf_negctl.so")
    assert os.path.exists(neg), "negative-control library missing: run __graft_entry__.build()"
    _le(_long_error(70001, "tc"), 1.0, "product, gap-free rows at 70,001: error / scaled tolerance")
    env = dict(os.environ, MMF_LIB=neg)
    r = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    ratio = json.loads(r.stdout.strip().splitlines()[-1])["ratio"]
    record_err("test_negative_control_exceeds_the_scaled_long_series_bound", ratio, 1.0,
               what="negctl, gap-free rows at 70,001: error / scaled tolerance (must exceed 1)")
    assert ratio > 1.0, ("the scaled bound does not detect a missing lo*A_hi term", ratio)


# =====================================================================================================================
# F. argument errors
# =====================================================================================================================
def _raw_fit(eng, y_ptr, n, ld_y, ps, npred, out_ptr, ld_out, status_ptr):
    """mmf_fit_forecast_f32 straight through ctypes (the Python wrapper would catch some of these first)"""
    return eng._lib.mmf_fit_forecast_f32(eng._h, y_ptr, n, ld_y, ps, npred, out_ptr, ld_out, None, status_ptr, None)


def test_argument_errors_leave_buffers_untouched():
    """each refused call returns its code and writes neither out nor status; n = 0 returns OK and writes nothing;
    afterwards the next valid call is bit-equal to the same call on a fresh engine"""
    import torch
    t, n = 372, 301
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=31)
    _plant(y, t)
    yd = mmf.device_packed(y)
    big = torch.full((n, t + 3), float("nan"), device="cuda")
    big[:, 1:t + 1] = yd
    ymis = big[:, 1:t + 1]                                   # not TMA-loadable
    engs = {k: mmf.ForecastEngine(kernel=k) for k in ("auto", "tc")}
    for eng in engs.values():
        eng.plan_calendar(start, t, "D", H, "future")
        eng.set_stream(torch.cuda.current_stream().cuda_stream)
    table = torch.full((n, 32), PATTERN, dtype=torch.int32, device="cuda")
    status = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    keep_t, keep_s = table.clone(), status.clone()
    out_p, st_p, y_p, ld_y = table.data_ptr(), status.data_ptr(), yd.data_ptr(), yd.stride(0)
    cases = [("ld_y < t_fit", "auto", (y_p, n, t - 1, t, H, out_p, 32), -1),
             ("window past n_rows", "auto", (y_p, n, ld_y, t + 1, H, out_p, 32), -1),
             ("negative pred_start", "auto", (y_p, n, ld_y, -1, H, out_p, 32), -1),
             ("ld_out < n_pred", "auto", (y_p, n, ld_y, t, H, out_p, H - 1), -1),
             ("n_pred = 0", "auto", (y_p, n, ld_y, t, 0, out_p, 32), -1),
             ("tc, unaligned y", "tc", (ymis.data_ptr(), n, ymis.stride(0), t, H, out_p, 32), -3),
             ("n = 0", "auto", (y_p, 0, ld_y, t, H, out_p, 32), 0)]
    for what, k, args, code in cases:
        rc = _raw_fit(engs[k], *args, st_p)
        torch.cuda.synchronize()
        assert rc == code, (what, rc, mmf._native.load().mmf_last_error())
        assert torch.equal(table, keep_t) and torch.equal(status, keep_s), what
    fresh = mmf.ForecastEngine()
    fresh.plan_calendar(start, t, "D", H, "future")
    want = fresh.fit_forecast(yd, t, H, want_status=True, want_beta=True)
    for k in ("auto",):
        got = engs[k].fit_forecast(yd, t, H, want_status=True, want_beta=True)
        torch.cuda.synchronize()
        for key in ("pred", "status", "beta"):
            assert _same_bits(got[key], want[key]), (k, key)
    tc_fresh = mmf.ForecastEngine(kernel="tc")
    tc_fresh.plan_calendar(start, t, "D", H, "future")
    a = engs["tc"].fit_forecast(yd, t, H, want_status=True)
    b = tc_fresh.fit_forecast(yd, t, H, want_status=True)
    torch.cuda.synchronize()
    assert _same_bits(a["pred"], b["pred"]) and _same_bits(a["status"], b["status"])
    for eng in (*engs.values(), fresh, tc_fresh):
        eng.close()
