"""GPU (-m gpu): the general contract include/mmf.h gives every ARIMA-family call (mmf_fit_forecast_ar_f32, _arima_f32,
_arma_f32, _arma_css_f32, mmf_fit_select_ar_f32, _select_arima_f32, _select_arma_f32 and the post-pass mmf_arima_se_f32):
any prediction window of the planned design, any y layout the ABI accepts, mmf_config.kernel and assume_finite honoured.

  A  every window [pred_start, pred_start + n_pred), pred_start in [0, t_fit + 8], n_pred in {1, 31, 32, 33, to the end of
     the design}, is bit for bit the holdout call's slice, and every other output is the holdout call's: pass B of the AR
     and ARIMA kernels restarts at the latest row s0 <= min(pred_start, t_fit) (- d) whose state is made of observations,
     and the restart may not change bits.  The holdout call of each configuration is checked once against the float64
     oracles (or the selections' single calls) of the existing modules;
  B  three views of a NaN-padded buffer (unaligned bases, pitches that are not a multiple of 4, a sentinel in every
     column the call may not read): auto is bit-equal to the kernel the layout forces on each fit stage (fit_warp for the
     d = 0 fit of y, fit_tc for z' in the 16-B-pitch scratch); kernel = tc refuses a call with a d = 0 stage and writes
     nothing; a selection's n_pending counts the rows of its tensor-core stages only;
  C  assume_finite on gap-free rows: bit-equal, n_pending 0, two launches fewer per tensor-core fit stage;
  D  the build whose pass B may restart one row past S (tests/_build/libmmf_ar_laterestart.so) fails A.

The batch interleaves gap runs of every length 1 .. 11 and 33 ending on offsets 0, 1 and 31 of a 32-row block and at the
128-row staging-chunk edge, close runs, leading and trailing gaps, +Inf, rows empty in z' only and empty rows, so every
CTA (8 series) mixes kinds and its warps restart from different rows."""
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import mmf
from ar_oracle import AR_MAX, fit_forecast_ar_packed
from arima_oracle import fit_forecast_arima_packed
from arma_oracle import MA_MAX, fit_forecast_arma_packed
from conftest import ROOT, record_err
from test_gpu_abi_contract import PATTERN, _expected_pending
from test_gpu_ar import _compare as _ar_compare
from test_gpu_arima import _compare as _arima_compare
from test_gpu_arima import _z32
from test_gpu_arima_se import ULP, _ulp_err
from test_gpu_arima_se import _oracle as _se_oracle
from test_gpu_arima_select import N_HOLD, _single
from test_gpu_arima_select import _check_against_single_calls as _pd_check
from test_gpu_arima_select import _scores as _pd_scores
from test_gpu_arma import _check as _arma_check
from test_gpu_arma import _fallback
from test_gpu_arma_css import _check as _css_check
from test_gpu_arma_select import _Singles, _ms
from test_gpu_arma_select import _check_against_single_calls as _pdq_check

pytestmark = pytest.mark.gpu

T_FIT = 200
N_ROWS = T_FIT + 40
N = 304                                     # 38 CTAs of 8 series
ORDERS = (0, 1, 3, 8)
DIFFS = (0, 1, 2)
MAS = (0, 1, 2)
SENT_F = float(np.float32(PATTERN))        # fill of memory the library must not write or read
SENT_I = PATTERN
E_UNSUPPORTED = -3
ENTRIES = ("ar", "arima", "arma", "arma_css", "select_ar", "select_arima", "select_arma")
SELECTIONS = ("select_ar", "select_arima", "select_arma")
CONFIGS = {
    "ar": [dict(p=p) for p in ORDERS if p >= 1],
    "arima": [dict(p=p, d=d) for d in (1, 2) for p in ORDERS],
    "arma": [dict(p=p, d=d, q=q) for d in DIFFS for q in (1, 2) for p in ORDERS],
    "arma_css": [dict(p=p, d=d, q=q) for d in DIFFS for q in (1, 2) for p in ORDERS],
    "select_ar": [dict(orders=ORDERS, diffs=(0,))],
    "select_arima": [dict(orders=ORDERS, diffs=DIFFS)],
    "select_arma": [dict(orders=ORDERS, diffs=DIFFS, mas=MAS)],
}


# ---- the batch ---------------------------------------------------------------------------------------------------------
def _kinds():
    """{name: the columns planted missing (as +Inf for "inf")}"""
    k = {}
    for length in list(range(1, 12)) + [33]:            # 1 .. p + d + 1 for p = 8, d = 2, and longer than a block
        for last in (64, 65, 95, 127, 128):             # block offsets 0, 1, 31; the last row of the first staged chunk
            k[f"run{length}@{last}"] = np.arange(last - length + 1, last + 1)       # and the first row of the next
    for sep in (1, 2, 4, 7):                            # two runs closer than p rows: no restart row between them
        k[f"close{sep}"] = np.r_[100:102, 102 + sep:104 + sep]
    k["first1"], k["first2"], k["first9"] = np.arange(1), np.arange(2), np.arange(9)
    for m in (1, 2, 3, 8, 9):
        k[f"last{m}"] = np.arange(T_FIT - m, T_FIT)
    k["inf"] = np.array([40, 41, 130, 161])
    k["zprime_empty"] = np.arange(1, T_FIT, 2)          # every other value: z' has no observed row, y has half
    k["empty"] = np.arange(N_ROWS)
    return k


def _batch(seed=7):
    """(y [N, N_ROWS] float32, X [N_ROWS, 5], kind of every row, clean rows): a regression on a caller design with a
    constant plus an AR(1) error, integrated on even rows; the held-out columns are clean but for the empty rows"""
    rng = np.random.default_rng(seed)
    s = np.arange(N_ROWS, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), (s - T_FIT / 2) / T_FIT, np.sqrt(s / T_FIT), np.sin(2 * np.pi * s / 30.5),
                         np.cos(2 * np.pi * s / 30.5)])
    beta = rng.normal(0, 20, (N, X.shape[1]))
    phi = rng.uniform(0.1, 0.8, N)
    w = np.zeros((N, N_ROWS))
    eps = rng.normal(0, 4, (N, N_ROWS))
    for t in range(N_ROWS):
        w[:, t] = eps[:, t] + (phi * w[:, t - 1] if t else 0)
    w[::2] = np.cumsum(w[::2] + rng.normal(0, 0.5, (N // 2, 1)), axis=1)
    y = (500.0 + beta @ X.T + w).astype(np.float32)
    kinds = _kinds()
    names = list(kinds) + ["clean"] * 16
    order = rng.permutation(N) % len(names)
    row_kind = [names[j] for j in order]
    for i, name in enumerate(row_kind):
        if name != "clean":
            y[i, kinds[name]] = np.inf if name == "inf" else np.nan
    return y, X, row_kind, np.array([k == "clean" for k in row_kind])


@pytest.fixture(scope="module")
def batch():
    y, X, kinds, clean = _batch()
    return y, X, kinds, clean


def _engine(X, t_fit=T_FIT, **kw):
    eng = mmf.ForecastEngine(**kw)
    eng.plan(X, t_fit, True)
    eng.plan_arima(X, t_fit, 2)
    return eng


def _aligned(y, t):
    """y's first t columns on the device with a 16-B row pitch, NaN beyond"""
    full = torch.full((y.shape[0], (t + 3) & ~3), float("nan"), device="cuda")
    full[:, :t] = torch.from_numpy(np.ascontiguousarray(y[:, :t])).cuda()
    return full[:, :t]


def _views(y, t):
    """three views of y's first t columns in NaN-padded buffers, every column from t on the sentinel"""
    src = torch.from_numpy(np.ascontiguousarray(y[:, :t])).cuda()
    out = {}
    for name, off, ld in (("base+0 ld=t+1", 0, t + 1), ("base+4B ld=t_fit+n_hold", 1, T_FIT + N_HOLD),
                          ("base+8B ld=t+5", 2, t + 5)):
        flat = torch.full((off + len(y) * ld + 8,), float("nan"), device="cuda")
        v = flat.as_strided((len(y), ld), (ld, 1), off)
        v[:, t:] = SENT_F
        v[:, :t] = src
        out[name] = v[:, :t]
    return out


# ---- one raw call of any entry point, every output pre-filled with the sentinel -----------------------------------------
def _cols(entry):
    """the columns of y the call may read"""
    return T_FIT + N_HOLD if entry in SELECTIONS else T_FIT


def _call(eng, entry, cfg, y, ps, npred, stats=None, n_hold=N_HOLD):
    """(rc, {output: tensor}); y is any [n, >= _cols(entry)] float32 CUDA view"""
    n, ld = y.shape[0], y.stride(0)
    f = lambda *s: torch.full(s, SENT_F, device="cuda")                              # noqa: E731
    i = lambda *s: torch.full(s, SENT_I, device="cuda", dtype=torch.int32)          # noqa: E731
    arr = lambda v: (ctypes.c_int32 * len(v))(*v)                                    # noqa: E731
    o = {"pred": f(n, npred)}
    st = ctypes.byref(stats) if stats is not None else None
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    lib, head = eng._lib, (eng._h, y.data_ptr(), n, ld)
    P = lambda *ks: [o[k].data_ptr() for k in ks]                                    # noqa: E731
    if entry == "ar":
        o.update(phi=f(n, AR_MAX), order=i(n), sigma=f(n), status=i(n))
        rc = lib.mmf_fit_forecast_ar_f32(*head, cfg["p"], ps, npred, *P("pred"), npred,
                                         *P("phi", "order", "sigma", "status"), st)
    elif entry == "arima":
        o.update(phi=f(n, AR_MAX), order=i(n), sigma=f(n), status=i(n))
        rc = lib.mmf_fit_forecast_arima_f32(*head, cfg["p"], cfg["d"], ps, npred, *P("pred"), npred,
                                            *P("phi", "order", "sigma", "status"), st)
    elif entry == "arma":
        o.update(phi=f(n, AR_MAX), theta=f(n, MA_MAX), order=i(n), ma_order=i(n), sigma=f(n), status=i(n))
        rc = lib.mmf_fit_forecast_arma_f32(*head, cfg["p"], cfg["d"], cfg["q"], 0, ps, npred, *P("pred"), npred,
                                           *P("phi", "theta", "order", "ma_order", "sigma", "status"), st)
    elif entry == "arma_css":
        o.update(phi=f(n, AR_MAX), theta=f(n, MA_MAX), order=i(n), ma_order=i(n), sigma=f(n), status=i(n),
                 css_start=f(n), css=f(n), css_stop=i(n), iters=i(n))
        rc = lib.mmf_fit_forecast_arma_css_f32(*head, cfg["p"], cfg["d"], cfg["q"], 0, 0, ps, npred, *P("pred"),
                                               npred, *P("phi", "theta", "order", "ma_order", "sigma", "status",
                                                         "css_start", "css", "css_stop", "iters"), st)
    elif entry == "select_ar":
        no = len(cfg["orders"])
        o.update(choice=i(n), mse=f(n), cand_mse=f(n, no), phi=f(n, AR_MAX), order=i(n), sigma=f(n), status=i(n))
        rc = lib.mmf_fit_select_ar_f32(*head, n_hold, arr(cfg["orders"]), no, ps, npred, *P("pred"), npred,
                                       *P("choice", "mse", "cand_mse", "phi", "order", "sigma", "status"), st)
    elif entry == "select_arima":
        no, nd = len(cfg["orders"]), len(cfg["diffs"])
        o.update(choice_p=i(n), choice_d=i(n), mse=f(n), cand_mse=f(n, nd, no), phi=f(n, AR_MAX), order=i(n),
                 sigma=f(n), status=i(n))
        rc = lib.mmf_fit_select_arima_f32(*head, n_hold, arr(cfg["orders"]), no, arr(cfg["diffs"]), nd, ps, npred,
                                          *P("pred"), npred, *P("choice_p", "choice_d", "mse", "cand_mse", "phi",
                                                                "order", "sigma", "status"), st)
    else:
        no, nd, nq = len(cfg["orders"]), len(cfg["diffs"]), len(cfg["mas"])
        o.update(choice_p=i(n), choice_d=i(n), choice_q=i(n), mse=f(n), cand_mse=f(n, nd, nq, no), phi=f(n, AR_MAX),
                 theta=f(n, MA_MAX), order=i(n), ma_order=i(n), sigma=f(n), status=i(n))
        rc = lib.mmf_fit_select_arma_f32(*head, n_hold, arr(cfg["orders"]), no, arr(cfg["diffs"]), nd,
                                         arr(cfg["mas"]), nq, 0, ps, npred, *P("pred"), npred,
                                         *P("choice_p", "choice_d", "choice_q", "mse", "cand_mse", "phi", "theta",
                                            "order", "ma_order", "sigma", "status"), st)
    return rc, o


def _se(eng, entry, cfg, y, res, ps, npred):
    """mmf_arima_se_f32 on the call's own outputs (a selection's per-row d: its choice_d)"""
    n = y.shape[0]
    out = torch.full((n, npred), SENT_F, device="cuda")
    d = cfg.get("d", 0)
    diffs = res.get("choice_d")
    th, ma = res.get("theta"), res.get("ma_order")
    ptr = lambda x: None if x is None else x.data_ptr()                              # noqa: E731
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    rc = eng._lib.mmf_arima_se_f32(eng._h, y.data_ptr(), n, y.stride(0), T_FIT, d, ptr(diffs), ptr(res["phi"]),
                                   ptr(res["order"]), ptr(th), ptr(ma), ptr(res["sigma"]), ps, npred, out.data_ptr(),
                                   npred, None)
    assert rc == 0, eng._lib.mmf_last_error()
    return out


def _ndiff(a, b):
    """entries whose bits differ (NaN against NaN counts as equal), as a 0-d device tensor"""
    if a.dtype == torch.float32:
        return ((a.view(torch.int32) != b.view(torch.int32)) & ~(a.isnan() & b.isnan())).sum()
    return (a != b).sum()


def _same(a, b):
    return all(int(_ndiff(a[k], b[k])) == 0 for k in a) and a.keys() == b.keys()


def _np(res):
    return {k: v.cpu().numpy() for k, v in res.items()}


def _windows():
    """pred_start in [0, t_fit + 8], n_pred in {1, 31, 32, 33, to the end of the design} (those inside the design)"""
    return [(ps, npred) for ps in range(T_FIT + 9) for npred in sorted({1, 31, 32, 33, N_ROWS - ps})
            if ps + npred <= N_ROWS]


def _sweep(eng, entry, cfg, yd, with_se=True):
    """the holdout call and every window of _windows(): (holdout outputs, holdout se, [(ps, npred) of every window
    whose outputs are not the holdout call's slice], windows compared)"""
    rc, full = _call(eng, entry, cfg, yd, 0, N_ROWS)
    assert rc == 0, eng._lib.mmf_last_error()
    se_full = _se(eng, entry, cfg, yd, full, 0, N_ROWS) if with_se else None
    wins = _windows()
    counts = []
    for ps, npred in wins:
        rc, got = _call(eng, entry, cfg, yd, ps, npred)
        assert rc == 0, (entry, cfg, ps, npred, eng._lib.mmf_last_error())
        nd = sum(_ndiff(v, full[k][:, ps:ps + npred] if k == "pred" else full[k]) for k, v in got.items())
        if with_se:
            nd = nd + _ndiff(_se(eng, entry, cfg, yd, got, ps, npred), se_full[:, ps:ps + npred])
        counts.append(nd)
    counts = torch.stack(counts).cpu().numpy()
    return full, se_full, [w for w, c in zip(wins, counts) if c], len(wins)


# ---- A: every window is the holdout call's slice ------------------------------------------------------------------------
def _oracle_check(eng, entry, cfg, full, yd, y, X, what):
    """the holdout call against the existing modules' yardsticks; returns the worst ratio (0 for bit-equality checks)"""
    g = _np(full)
    yf = y[:, :T_FIT]
    if entry == "ar":
        want = fit_forecast_ar_packed(yf, X, T_FIT, 0, N_ROWS, cfg["p"])
        return _ar_compare(g, want, yf, X, T_FIT, 0, N_ROWS, what)
    if entry == "arima":
        want = fit_forecast_arima_packed(yf, X, T_FIT, 0, N_ROWS, cfg["p"], cfg["d"])
        return _arima_compare(g, want, T_FIT, 0, N_ROWS, what)
    if entry in ("arma", "arma_css"):
        p, d, q = cfg["p"], cfg["d"], cfg["q"]
        fb = _fallback(eng, yd, p, d, 0, N_ROWS, T_FIT)
        if entry == "arma":
            want = fit_forecast_arma_packed(yf, X, T_FIT, 0, N_ROWS, p, q, d, 0)
            return _arma_check(g, fb, want, yf, X, T_FIT, 0, N_ROWS, what)[0]
        hr = _np(eng.fit_forecast_arma(yd[:, :T_FIT], p, q, d, 0, N_ROWS))
        # the HR-row bit checks on every configuration; the float64 S and prediction bounds (a per-row CPU evaluation)
        # on the q = 1 ones, every p and d (tests/test_gpu_arma_css.py holds every (p, q, d) to them)
        return _css_check(g, hr, fb, yf, X, T_FIT, p, q, d, 0, what, oracle=q == 1, n_opt=1)[0]
    orders, diffs = cfg["orders"], cfg["diffs"]
    if entry == "select_arma":
        _pdq_check(g, _Singles(eng, yd, T_FIT), y, T_FIT, 0, N_ROWS, orders, diffs, cfg["mas"],
                   _ms(T_FIT, orders, diffs, cfg["mas"]), what)
        return 0.0
    fut = {(p, d): _single(eng, yd, p, d, T_FIT, N_HOLD) for p in orders for d in diffs}
    runs = {(p, d): _single(eng, yd, p, d, 0, N_ROWS) for p in orders for d in diffs}
    el = np.stack([fut[orders[0], d]["status"] != 1 for d in diffs], axis=1)
    if entry == "select_ar":
        g["choice_p"], g["choice_d"] = g["choice"], np.where(g["choice"] < 0, -1, 0)
        g["cand_mse"] = g["cand_mse"][:, None, :]
    _pd_check(g, runs, _pd_scores(fut, y, T_FIT, orders, diffs), el, orders, diffs, what)
    return 0.0


def _se_check(entry, cfg, full, se, y, what):
    g = _np(full)
    diffs = g.get("choice_d") if entry in ("select_arima", "select_arma") else None
    want = _se_oracle(g, y[:, :T_FIT], T_FIT, 0, N_ROWS, cfg.get("d", 0), diffs)
    e = _ulp_err(se.cpu().numpy(), want)
    assert e <= ULP, (what, e)
    return e


@pytest.mark.parametrize("entry", ENTRIES)
def test_every_window_is_the_holdout_slice(batch, entry):
    y, X, kinds, _ = batch
    eng = _engine(X)
    yd = _aligned(y, N_ROWS)[:, :_cols(entry)]
    t0 = time.perf_counter()
    n_cmp, worst, worst_se = 0, 0.0, 0.0
    for cfg in CONFIGS[entry]:
        what = f"{entry} {cfg}"
        full, se, bad, n_win = _sweep(eng, entry, cfg, yd)
        assert not bad, (what, len(bad), bad[:8])
        n_cmp += n_win
        worst = max(worst, _oracle_check(eng, entry, cfg, full, _aligned(y, N_ROWS), y, X, what))
        worst_se = max(worst_se, _se_check(entry, cfg, full, se, y, what))
    eng.close()
    record_err("arima_contract windows", 0.0, 0.0, what=entry, configurations=len(CONFIGS[entry]),
               window_comparisons=n_cmp, oracle_worst=worst, se_worst_ulp=worst_se,
               seconds=round(time.perf_counter() - t0, 1))


# ---- B: caller layouts of y ---------------------------------------------------------------------------------------------
def _layout_configs(entry):
    if entry == "ar":
        return [dict(p=3)]
    if entry == "arima":
        return [dict(p=3, d=d) for d in (1, 2)]
    if entry in ("arma", "arma_css"):
        return [dict(p=3, d=d, q=q) for d in DIFFS for q in (1, 2)]
    return CONFIGS[entry]


def _assert_refused(rc, out, eng, what):
    assert rc == E_UNSUPPORTED, (what, rc)
    assert b"tensor-core kernel not applicable" in eng._lib.mmf_last_error(), (what, eng._lib.mmf_last_error())
    torch.cuda.synchronize()
    for k, v in out.items():
        s = SENT_F if v.dtype == torch.float32 else SENT_I
        assert bool((v == s).all()), (what, k)


@pytest.mark.parametrize("entry", ("ar", "arima", "arma", "arma_css"))
def test_single_calls_on_caller_layouts(batch, entry):
    """auto on a view is the kernel the layout forces (fit_warp for a d = 0 fit of y, fit_tc for z'); tc refuses a
    d = 0 call and writes nothing, and runs a d >= 1 call bit-equal to auto on an aligned copy"""
    y, X, _, _ = batch
    engs = {k: _engine(X, kernel=k) for k in ("auto", "warp", "tc")}
    t = _cols(entry)
    copy = _aligned(y, t)
    n_cmp = n_refused = 0
    for cfg in _layout_configs(entry):
        d = cfg.get("d", 0)
        for ps, npred in ((0, N_ROWS), (T_FIT, 33)):
            rc, ref = _call(engs["warp" if d == 0 else "auto"], entry, cfg, copy, ps, npred)
            assert rc == 0
            for name, v in _views(y, t).items():
                what = f"{entry} {cfg} {name} ({ps}, {npred})"
                rc, got = _call(engs["auto"], entry, cfg, v, ps, npred)
                assert rc == 0, what
                assert _same(got, ref), what
                rc, got = _call(engs["tc"], entry, cfg, v, ps, npred)
                if d == 0:
                    _assert_refused(rc, got, engs["tc"], what)
                    n_refused += 1
                else:
                    assert rc == 0 and _same(got, ref), what
                n_cmp += 2
    for e in engs.values():
        e.close()
    record_err("arima_contract layouts", 0.0, 0.0, what=entry, comparisons=n_cmp, refusals=n_refused)


def _pending(y, diffs, tc_d0):
    """n_pending of a selection: the rows each tensor-core stage hands to the general pass (d = 0 on y with the
    constant of the level design, d >= 1 on z' of the differenced design, which has none); a fit_warp stage adds 0"""
    yf = y[:, :T_FIT]
    return sum((_expected_pending(yf, T_FIT, True) if tc_d0 else 0) if d == 0
               else _expected_pending(_z32(yf, d), T_FIT - d, False) for d in diffs)


def _singles_check(entry, cfg, eng, v, got, y, what):
    """the selection on view v against its winners' single calls on v"""
    g = _np(got)
    orders, diffs = cfg["orders"], cfg["diffs"]
    if entry == "select_arma":
        _pdq_check(g, _Singles(eng, v, T_FIT), y, T_FIT, 0, N_ROWS, orders, diffs, cfg["mas"],
                   _ms(T_FIT, orders, diffs, cfg["mas"]), what)
        return
    fut = {(p, d): _single(eng, v, p, d, T_FIT, N_HOLD) for p in orders for d in diffs}
    runs = {(p, d): _single(eng, v, p, d, 0, N_ROWS) for p in orders for d in diffs}
    el = np.stack([fut[orders[0], d]["status"] != 1 for d in diffs], axis=1)
    if entry == "select_ar":
        g["choice_p"], g["choice_d"] = g["choice"], np.where(g["choice"] < 0, -1, 0)
        g["cand_mse"] = g["cand_mse"][:, None, :]
    _pd_check(g, runs, _pd_scores(fut, y, T_FIT, orders, diffs), el, orders, diffs, what)


@pytest.mark.parametrize("entry", SELECTIONS)
def test_selections_on_caller_layouts(batch, entry):
    """a selection on a view mixes the kernels (fit_warp for d = 0, fit_tc for d >= 1): its outputs are its winners'
    single calls on the view, its cand_mse[:, d] the warp-engine (d = 0) or auto-engine (d >= 1) selection's on an
    aligned copy, its n_pending the tensor-core stages' only; tc refuses a list with d = 0 and writes nothing"""
    y, X, _, _ = batch
    engs = {k: _engine(X, kernel=k) for k in ("auto", "warp", "tc")}
    t = _cols(entry)
    copy = _aligned(y, t)
    cfg = CONFIGS[entry][0]
    diffs = cfg["diffs"]
    rc, by_warp = _call(engs["warp"], entry, cfg, copy, 0, N_ROWS)
    assert rc == 0
    st = mmf._native.MmfStats()
    rc, by_auto = _call(engs["auto"], entry, cfg, copy, 0, N_ROWS, stats=st)
    assert rc == 0
    pend = [("aligned copy", int(st.n_pending), _pending(y, diffs, True))]
    assert pend[0][1] == pend[0][2], pend
    n_refused = 0
    for name, v in _views(y, t).items():
        what = f"{entry} {name}"
        st = mmf._native.MmfStats()
        rc, got = _call(engs["auto"], entry, cfg, v, 0, N_ROWS, stats=st)
        assert rc == 0, what
        _singles_check(entry, cfg, engs["auto"], v, got, y, what)
        cm = got["cand_mse"] if entry != "select_ar" else got["cand_mse"][:, None]
        for k, d in enumerate(diffs):
            ref = (by_warp if d == 0 else by_auto)["cand_mse"]
            ref = ref[:, k] if entry != "select_ar" else ref
            assert int(_ndiff(cm[:, k], ref)) == 0, (what, d)
        pend.append((name, int(st.n_pending), _pending(y, diffs, False)))
        assert pend[-1][1] == pend[-1][2], pend
        rc, got = _call(engs["tc"], entry, cfg, v, 0, N_ROWS)
        _assert_refused(rc, got, engs["tc"], what)
        n_refused += 1
        if entry != "select_ar":                          # only d >= 1 stages: fit_tc on z', bit-equal to auto
            c1 = dict(cfg, diffs=(1, 2))
            rc, got = _call(engs["tc"], entry, c1, v, 0, N_ROWS)
            assert rc == 0, what
            rc, ref = _call(engs["auto"], entry, c1, copy, 0, N_ROWS)
            assert rc == 0 and _same(got, ref), what
    for e in engs.values():
        e.close()
    record_err("arima_contract selection layouts", 0.0, 0.0, what=entry, refusals=n_refused,
               n_pending=[f"{n}: reported {a}, predicted {b}" for n, a, b in pend])


# ---- C: assume_finite ---------------------------------------------------------------------------------------------------
def _tc_stages(entry, cfg):
    return len(cfg["diffs"]) if entry in ("select_arima", "select_arma") else 1


def _finite_pair(y, X, entry, cfg, t_fit, slabs, what, n_hold=N_HOLD):
    base, fin = _engine(X, t_fit), _engine(X, t_fit, assume_finite=True)
    yd = _aligned(y, y.shape[1])
    s0, s1 = mmf._native.MmfStats(), mmf._native.MmfStats()
    rc0, a = _call(base, entry, cfg, yd, t_fit, 8, stats=s0, n_hold=n_hold)
    rc1, b = _call(fin, entry, cfg, yd, t_fit, 8, stats=s1, n_hold=n_hold)
    assert rc0 == 0 and rc1 == 0, what
    assert _same(a, b), what
    assert s1.n_pending == 0 and s0.n_pending == 0, (what, s0.n_pending, s1.n_pending)
    assert s0.kernel_launches - s1.kernel_launches == 2 * slabs * _tc_stages(entry, cfg), \
        (what, s0.kernel_launches, s1.kernel_launches)
    base.close()
    fin.close()


@pytest.mark.parametrize("entry", ENTRIES)
def test_assume_finite_on_gap_free_rows(batch, entry):
    """no fit_warp(only_pending) and no solve_rows per tensor-core fit stage, the same bits"""
    y, X, _, clean = batch
    yc = y[clean]
    assert len(yc) >= 8
    t = _cols(entry)
    for cfg in CONFIGS[entry]:
        _finite_pair(yc[:, :t], X, entry, cfg, T_FIT, 1, f"{entry} {cfg}")


def test_assume_finite_on_a_multi_slab_batch():
    """2^20 + 1,001 gap-free rows (two slabs): one call of each kind"""
    n, t, hold = (1 << 20) + 1001, 48, 8
    rng = np.random.default_rng(3)
    s = np.arange(t + 16, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), s / t, np.sin(2 * np.pi * s / 7), np.cos(2 * np.pi * s / 7)])
    y = (100.0 + rng.normal(0, 10, (n, 4)).astype(np.float32) @ X[:t + hold].T.astype(np.float32)
         + rng.normal(0, 3, (n, t + hold)).astype(np.float32)).astype(np.float32)
    calls = (("ar", dict(p=2)), ("arima", dict(p=2, d=1)), ("arma", dict(p=1, d=1, q=1)),
             ("arma_css", dict(p=1, d=0, q=1)), ("select_ar", dict(orders=(0, 1, 2), diffs=(0,))),
             ("select_arima", dict(orders=(0, 2), diffs=(0, 1))), ("select_arma", dict(orders=(0, 1), diffs=(0, 1),
                                                                                         mas=(0, 1))))
    for entry, cfg in calls:
        _finite_pair(y if entry in SELECTIONS else y[:, :t], X, entry, cfg, t, 2, f"multi-slab {entry}", hold)


# ---- D: the late-restart control must fail A -----------------------------------------------------------------------------
CONTROL = (("ar", dict(p=3)), ("ar", dict(p=8)), ("arima", dict(p=3, d=1)), ("arima", dict(p=0, d=2)),
           ("select_ar", CONFIGS["select_ar"][0]), ("select_arima", CONFIGS["select_arima"][0]))

_NEGCTL = """
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import test_gpu_arima_contract as T
import mmf
y, X, kinds, clean = T._batch()
eng = T._engine(X)
yd = T._aligned(y, T.N_ROWS)
out = []
for entry, cfg in T.CONTROL:
    _, _, bad, n = T._sweep(eng, entry, cfg, yd[:, :T._cols(entry)], with_se=False)
    out.append([entry, str(cfg), len(bad), n])
print(json.dumps({{"lib": mmf.LIB_PATH, "sweeps": out}}))
"""


@pytest.mark.parametrize("lib", ["product", "laterestart"])
def test_negative_control_with_a_late_restart(lib):
    """the build whose pass B may restart one row past S must give windows that are not the holdout call's slice for
    AR, ARIMA and both selections; the product library gives none"""
    env = dict(os.environ)
    env.pop("MMF_LIB", None)
    if lib == "laterestart":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_ar_laterestart.so")
        assert os.path.exists(env["MMF_LIB"]), "negative-control library missing: run __graft_entry__.build()"
    r = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    record_err("arima_contract late-restart control", 0.0, 0.0, what=lib, sweeps=got["sweeps"])
    if lib == "product":
        assert all(b == 0 for _, _, b, _ in got["sweeps"]), got
    else:
        assert got["lib"].endswith("libmmf_ar_laterestart.so"), got
        for entry in ("ar", "arima", "select_ar", "select_arima"):
            assert any(b > 0 for e, _, b, _ in got["sweeps"] if e == entry), (entry, got)
