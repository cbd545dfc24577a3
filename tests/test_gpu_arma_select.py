"""GPU (-m gpu): (p, d, q) selection by hold-out MSE on levels (mmf_fit_select_arma_f32, DESIGN.md section 2 item 14).

Candidate (p, d, 0) is, by definition, mmf_fit_select_arima_f32's candidate (p, d) and candidate (p, d, q >= 1)
mmf_fit_forecast_arma_f32(p, d, q) with the call's long order m_d, so every series' outputs must be bit-equal to the
single call of its winner (theta, ma_order and choice_q exactly 0 for a q = 0 winner), and every candidate's score must
be the float64 MSE of that call's own future-mode predictions.  With mas = (0,) the call is mmf_fit_select_arima_f32,
bit for bit.  Against the float64 oracle of tests/arma_select_oracle.py the scores must lie within mse_bound.  Batches
carry test_gpu_arima_select.py's row mix (gaps, +Inf, fully missing held-out windows, z' empty for d >= 1 only, rows
empty for every d) with MA(1) errors on a third of the rows, so that q >= 1 wins somewhere."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mmf
from ar_oracle import AR_MAX, degenerate_rows, kappa_margin
from arima_oracle import z_tau
from arma_oracle import MA_MAX, near_threshold
from arma_select_oracle import choose, default_long_order, mse_bound, select_arma_packed
from conftest import ROOT, record_err
from oracle import mmf_oracle as O
from test_gpu_abi_contract import PATTERN
from test_gpu_ar import KAPPA_MARGIN
from test_gpu_arima_select import N_HOLD, _bits, _case, _device, _engine, _np, _single, _taus, _windows
from test_gpu_edges import _le, _same_bits

pytestmark = pytest.mark.gpu

REF = ((0, 1, 2, 3, 4), (0, 1, 2), (0, 1, 2, 3, 4))
# the last grid is the largest the ABI accepts: 32 (p, q >= 1) pairs, every lane a candidate, 26 row sets, 74,732 B
GRIDS = (REF, (tuple(range(9)), (0, 1, 2), (0, 1, 2, 3)), ((1,), (1,), (0, 1)), ((0,), (2,), (0, 4)),
         ((0, 1, 2, 3, 4), (0, 1, 2), (0,)), (tuple(range(1, 9)), (0, 1, 2), (0, 1, 2, 3, 4)))
SENT_F, SENT_I = float(np.float32(PATTERN)), -7


def _ma_case(cal, n=170, seed=5, n_hold=N_HOLD):
    """test_gpu_arima_select's rows, with every third row (not one of its special rows) an MA(1) theta = 0.6 error on
    its regression"""
    y, X, t_fit, has_c = _case(cal, n, seed, n_hold)
    rng = np.random.default_rng(seed + 200)
    tt = t_fit + n_hold
    eps = rng.normal(0, 4, (n, tt + 1))
    base = 400.0 + rng.normal(0, 20, (n, X.shape[1])) @ X[:tt].T
    for i in range(0, n - 2, 3):
        keep = np.isfinite(y[i]) | np.isposinf(y[i])
        v = (base[i] + eps[i, 1:] + 0.6 * eps[i, :-1]).astype(np.float32)
        y[i] = np.where(keep, np.where(np.isposinf(y[i]), np.inf, v), np.nan)
    return y, X, t_fit, has_c


def _call(eng, yd, orders, diffs, mas, ps, npred, long_order=0, n_hold=N_HOLD):
    """mmf_fit_select_arma_f32 with every output pre-filled with a sentinel (unwritten entries show)"""
    n = yd.shape[0]
    no, nd, nq = len(orders), len(diffs), len(mas)
    f = lambda *s: torch.full(s, SENT_F, device="cuda")
    i = lambda *s: torch.full(s, SENT_I, device="cuda", dtype=torch.int32)
    out = dict(pred=f(n, npred), choice_p=i(n), choice_d=i(n), choice_q=i(n), mse=f(n), cand_mse=f(n, nd, nq, no),
               phi=f(n, AR_MAX), theta=f(n, MA_MAX), order=i(n), ma_order=i(n), sigma=f(n), status=i(n))
    arr = lambda v: (ctypes.c_int32 * len(v))(*v)
    torch.cuda.synchronize()                                                   # the sentinels are in place
    rc = eng._lib.mmf_fit_select_arma_f32(
        eng._h, yd.data_ptr(), n, yd.stride(0), n_hold, arr(orders), no, arr(diffs), nd, arr(mas), nq, long_order, ps,
        npred, out["pred"].data_ptr(), npred,
        *[out[k].data_ptr() for k in ("choice_p", "choice_d", "choice_q", "mse", "cand_mse", "phi", "theta", "order",
                                      "ma_order", "sigma", "status")], None)
    assert rc == 0, eng._lib.mmf_last_error()
    torch.cuda.synchronize()
    return _np(out)


class _Singles:
    """single calls of every candidate, cached: (p, d, 0) as test_gpu_arima_select, (p, d, q) fit_forecast_arma"""

    def __init__(self, eng, yd, t_fit):
        self.eng, self.yd, self.t_fit, self.cache = eng, yd, t_fit, {}

    def __call__(self, p, d, q, m, ps, npred):
        key = (p, d, q, m if q else 0, ps, npred)
        if key not in self.cache:
            if q == 0:
                r = _single(self.eng, self.yd, p, d, ps, npred)
                n = len(r["status"])
                r["theta"], r["ma_order"] = np.zeros((n, MA_MAX), np.float32), np.zeros(n, np.int32)
            else:
                r = _np(self.eng.fit_forecast_arma(self.yd[:, :self.t_fit], p, q, d, ps, npred, long_order=m))
            self.cache[key] = r
        return self.cache[key]


def _scores(single, y, t_fit, orders, diffs, mas, ms):
    """[n, n_diffs, n_mas, n_orders] float64 MSE of every candidate's own future-mode predictions"""
    yh = y[:, t_fit:t_fit + N_HOLD].astype(np.float64)
    out = np.full((len(y), len(diffs), len(mas), len(orders)), np.nan)
    for k, d in enumerate(diffs):
        for l, q in enumerate(mas):
            for j, p in enumerate(orders):
                f = single(p, d, q, ms[k], t_fit, N_HOLD)["pred"][:, :N_HOLD].astype(np.float64)
                ok = np.isfinite(f) & np.isfinite(yh)
                cnt = ok.sum(axis=1)
                e = np.where(ok, yh - np.where(ok, f, 0), 0)
                with np.errstate(invalid="ignore"):
                    out[:, k, l, j] = np.where(cnt > 0, (e * e).sum(axis=1) / np.maximum(cnt, 1), np.nan)
    return out


def _ambiguous(scores, eligible):
    """rows whose two smallest eligible scores differ but lie within 1e-6 relative"""
    s = np.where(eligible[:, :, None, None], scores, np.nan).reshape(len(scores), -1)
    s = np.sort(np.where(np.isnan(s), np.inf, s), axis=1)
    if s.shape[1] < 2:
        return np.zeros(len(s), dtype=bool)
    a, b = s[:, 0], s[:, 1]
    with np.errstate(invalid="ignore"):
        return np.isfinite(b) & (b != a) & (b - a <= 1e-6 * np.abs(b))


def _check_against_single_calls(got, single, y, t_fit, ps, npred, orders, diffs, mas, ms, what):
    """scores against the single calls, the first-minimum choice, the winner's outputs bit for bit; returns the number
    of ambiguous rows and of q >= 1 winners"""
    n = len(y)
    sc = _scores(single, y, t_fit, orders, diffs, mas, ms)
    eligible = np.stack([single(orders[0], d, 0, 0, t_fit, N_HOLD)["status"] != 1 for d in diffs], axis=1)
    cm = got["cand_mse"].astype(np.float64)
    differ = (np.isnan(cm) != np.isnan(sc)).reshape(n, -1).any(axis=1)
    assert not differ.any(), (what, np.flatnonzero(differ)[:8])
    ok = ~np.isnan(sc)
    rel = np.abs(cm[ok] - sc[ok]) / np.maximum(np.abs(sc[ok]), 1e-30)
    _le(float(rel.max()) if rel.size else 0.0, 1e-6, f"{what}: cand_mse against the single calls")
    kk, ll, jj = choose(sc, eligible)
    amb = _ambiguous(sc, eligible)
    won = kk >= 0
    want_p = np.where(won, np.array(orders)[np.maximum(jj, 0)], -1)
    want_d = np.where(won, np.array(diffs)[np.maximum(kk, 0)], -1)
    want_q = np.where(won, np.array(mas)[np.maximum(ll, 0)], -1)
    cp, cd, cq = got["choice_p"], got["choice_d"], got["choice_q"]
    bad = np.flatnonzero(((cp != want_p) | (cd != want_d) | (cq != want_q)) & ~amb)
    assert bad.size == 0, (what, bad[:8], cp[bad[:8]], cd[bad[:8]], cq[bad[:8]], want_p[bad[:8]], want_d[bad[:8]],
                           want_q[bad[:8]])
    none = cp < 0
    assert (none == ~eligible.any(axis=1)).all() and ((cd < 0) == none).all() and ((cq < 0) == none).all(), what
    k_of = {d: k for k, d in enumerate(diffs)}
    for key in ("pred", "phi", "theta", "order", "ma_order", "sigma", "status"):
        want = np.empty_like(got[key])
        for p, d, q in set(zip(cp[~none].tolist(), cd[~none].tolist(), cq[~none].tolist())):
            s = (cp == p) & (cd == d) & (cq == q)
            want[s] = single(p, d, q, ms[k_of[d]], ps, npred)[key][s]
        if none.any():
            want[none] = {"pred": np.nan, "phi": 0.0, "theta": 0.0, "order": 0, "ma_order": 0, "sigma": np.nan,
                          "status": 1}[key]
        bad = np.flatnonzero((_bits(got[key]) != _bits(want)).reshape(n, -1).any(axis=1))
        assert bad.size == 0, (what, key, bad[:8], cp[bad[:8]], cd[bad[:8]], cq[bad[:8]])
    assert (got["ma_order"] == np.maximum(cq, 0)).all(), what                   # a winner with q >= 1 is gated
    l_of, j_of = {q: l for l, q in enumerate(mas)}, {p: j for j, p in enumerate(orders)}
    rows = np.flatnonzero(~none)
    win = got["cand_mse"][rows, [k_of[d] for d in cd[rows]], [l_of[q] for q in cq[rows]], [j_of[p] for p in cp[rows]]]
    assert np.array_equal(_bits(got["mse"][rows]), _bits(win)) and np.isnan(got["mse"][none]).all(), what
    return int(amb.sum()), int((cq > 0).sum())


def _ms(t_fit, orders, diffs, mas, long_order=0):
    return [long_order or default_long_order(t_fit, d, orders, mas) for d in diffs]


@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_mas_zero_is_bit_equal_to_pd_selection(cal):
    y, X, t_fit, has_c = _ma_case(cal)
    _, yd = _device(y)
    for kernel in ("auto", "tc", "warp"):
        eng = _engine(kernel, X, t_fit, has_c)
        for name, (ps, npred) in _windows(t_fit, X.shape[0]).items():
            for orders, diffs in (((0, 1, 2, 3, 4), (0, 1, 2)), (tuple(range(9)), (0, 1, 2)), ((1,), (1,)),
                                  ((0,), (2,)), ((8,), (0,))):
                got = _call(eng, yd, orders, diffs, (0,), ps, npred)
                ref = _np(eng.fit_select_arima(yd, N_HOLD, orders, diffs, ps, npred))
                what = f"{cal} {kernel} {name} {orders} x {diffs}"
                for k in ref:
                    g = got[k][:, :, 0, :] if k == "cand_mse" else got[k]
                    assert _bits(g).tobytes() == _bits(ref[k]).tobytes(), (what, k)
                assert np.array_equal(got["choice_q"], np.where(ref["choice_p"] < 0, -1, 0)), what
                assert not got["theta"].any() and not got["ma_order"].any(), what
        eng.close()


@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_bit_equal_to_the_winners_single_call(cal):
    y, X, t_fit, has_c = _ma_case(cal)
    _, yd = _device(y)
    amb_total = checked = q_wins = 0
    for kernel in ("auto", "tc", "warp"):
        eng = _engine(kernel, X, t_fit, has_c)
        single = _Singles(eng, yd, t_fit)
        for name, (ps, npred) in _windows(t_fit, X.shape[0]).items():
            for orders, diffs, mas in GRIDS:
                ms = _ms(t_fit, orders, diffs, mas)
                got = _call(eng, yd, orders, diffs, mas, ps, npred)
                a, w = _check_against_single_calls(got, single, y, t_fit, ps, npred, orders, diffs, mas, ms,
                                                   f"{cal} {kernel} {name} {orders} x {diffs} x {mas}")
                amb_total, q_wins, checked = amb_total + a, q_wins + w, checked + 1
        eng.close()
    assert q_wins > 0, cal
    record_err("arma_select_ambiguous_rows", float(amb_total), float(checked * len(y)), what=cal, q_wins=q_wins)


def test_caller_long_order():
    y, X, t_fit, has_c = _ma_case("daily", n=60)
    _, yd = _device(y)
    eng = _engine("auto", X, t_fit, has_c)
    single = _Singles(eng, yd, t_fit)
    for m in (4, 32):
        orders, diffs, mas = (0, 1, 2), (0, 1, 2), (0, 1, 2)
        got = _call(eng, yd, orders, diffs, mas, t_fit, 28, long_order=m)
        _check_against_single_calls(got, single, y, t_fit, t_fit, 28, orders, diffs, mas, [m] * 3, f"m={m}")
    eng.close()


def _near_rows(want, y, t_fit):
    """rows whose order, gate decision or long-AR order may go either way under a first-order perturbation in some
    candidate (test_gpu_arima_select's kappa margin, test_gpu_arma's near_threshold and degenerate rows)"""
    near = np.zeros(len(want["status"]), dtype=bool)
    for blk in want["hold"]:
        for l, row in enumerate(blk):
            for h in row:
                near |= kappa_margin(h.get("zres", h)) < KAPPA_MARGIN
                if l > 0:
                    zt = {"z": h["base"]["z"]} if h["d"] >= 1 else {"z": np.where(np.isfinite(y), y, np.nan)[:, :t_fit]}
                    near |= near_threshold(h) | degenerate_rows(h["zres"], z_tau(zt))
    return near


@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_scores_against_the_oracle(cal):
    y, X, t_fit, has_c = _ma_case(cal, n=60)
    orders, diffs, mas = REF
    _, yd = _device(y)
    eng = _engine("auto", X, t_fit, has_c)
    got = _call(eng, yd, orders, diffs, mas, t_fit, N_HOLD)
    eng.close()
    want = select_arma_packed(y, X, t_fit, N_HOLD, orders, diffs, mas, t_fit, N_HOLD)
    bound = mse_bound(want, y, _taus(y, X, t_fit, want_q0(want), diffs), t_fit, N_HOLD, orders, diffs, mas)
    near = _near_rows(want, y, t_fit)
    live = want["eligible"].any(axis=1) & ~near
    record_err("arma_select_near_limit_rows", float(near.sum()), float(len(y)), what=cal)
    assert np.array_equal(got["choice_p"] < 0, ~want["eligible"].any(axis=1)), cal
    cm = got["cand_mse"].astype(np.float64)
    assert np.array_equal(np.isnan(cm[live]), np.isnan(want["cand_mse"][live])), cal
    ok = live[:, None, None, None] & ~np.isnan(want["cand_mse"])
    err = np.abs(cm - np.where(ok, want["cand_mse"], 0))
    ratio = np.where(ok, err / np.where(bound > 0, bound, np.inf), 0)
    _le(float(ratio.max()), 1.0, f"{cal}: |cand_mse - oracle| / mse_bound")
    hist = {f"{q}": int((got["choice_q"] == q).sum()) for q in mas}
    record_err("arma_select_choice_q_histogram", 0.0, 1.0, what=cal, hist=hist)


def want_q0(want):
    """the q = 0 view of an arma_select_oracle result, for test_gpu_arima_select._taus"""
    return {"hold": [blk[0] for blk in want["hold"]]}


def test_y_beyond_the_held_out_window_is_never_read():
    y, X, t_fit, has_c = _ma_case("daily")
    eng = _engine("auto", X, t_fit, has_c)
    full, yd = _device(y, extra=40)
    ref = _call(eng, yd, (0, 1, 2), (0, 1, 2), (0, 1, 2), 0, t_fit + 64)
    full[:, t_fit + N_HOLD:] = 3.0e38
    other = _call(eng, yd, (0, 1, 2), (0, 1, 2), (0, 1, 2), 0, t_fit + 64)
    for k in ref:
        assert _bits(ref[k]).tobytes() == _bits(other[k]).tobytes(), k
    eng.close()


def test_exact_power_of_two_scaling():
    y, X, t_fit, has_c = _ma_case("daily")
    eng = _engine("auto", X, t_fit, has_c)
    _, yd = _device(y)
    a = _call(eng, yd, (0, 1, 3), (0, 1, 2), (0, 1, 2), t_fit, 28)
    b = _call(eng, yd * 8.0, (0, 1, 3), (0, 1, 2), (0, 1, 2), t_fit, 28)
    for k, f in (("pred", 8.0), ("phi", 1.0), ("theta", 1.0), ("order", 1), ("ma_order", 1), ("sigma", 8.0),
                 ("status", 1), ("mse", 64.0), ("cand_mse", 64.0), ("choice_p", 1), ("choice_d", 1), ("choice_q", 1)):
        w = a[k] * f
        same = (b[k] == w) | (np.isnan(b[k]) & np.isnan(w))
        assert same.all(), (k, np.flatnonzero(~same.reshape(len(y), -1).all(axis=1))[:6])
    assert (a["choice_q"] > 0).any()
    eng.close()


def test_slabs_are_bit_equal_to_per_slab_calls():
    n, t = (1 << 20) + 1001, 48
    y, start = mmf.synth.daily_store_item_demand(n, t + 8, seed=9, nan_frac=0.01)
    X = O.design_matrix(O.calendar_grid(start, t + 8, "D"), t)
    eng = _engine("auto", X, t, True)
    yd = torch.from_numpy(y).cuda()
    grid = ((0, 1, 2), (0, 1, 2), (0, 1, 2))
    whole = eng.fit_select_arma(yd, 8, *grid, t, 8)
    for lo, hi in ((0, 1 << 19), (1 << 19, n)):
        part = eng.fit_select_arma(yd[lo:hi], 8, *grid, t, 8)
        for k in whole:
            assert _same_bits(whole[k][lo:hi], part[k]), k
    assert (whole["choice_q"] > 0).any()
    eng.close()


def test_long_hourly_series():
    """70,001 fit rows: bounds x sqrt(t_fit / 1095)"""
    t, h = 70001, 48
    s = np.arange(t + h + 8, dtype=np.float64)
    X = np.column_stack([np.ones_like(s), (s - t / 2) / t, np.sin(2 * np.pi * s / 24), np.cos(2 * np.pi * s / 24)])
    rng = np.random.default_rng(4)
    n = 6
    eps = rng.normal(0, 3, (n, t + h + 1))
    w = eps[:, 1:] + 0.6 * eps[:, :-1]
    y = 2000 + 10 * X[:t + h, 2] + np.where(np.arange(n)[:, None] % 2 == 0, np.cumsum(w, axis=1) / 20, w)
    y = y.astype(np.float32)
    y[1, t - 3:t] = np.nan
    y[2, 1000:1400] = np.nan
    eng = _engine("auto", X, t, True)
    orders, diffs, mas = (0, 1), (0, 1), (0, 1)
    _, yd = _device(y)
    got = _call(eng, yd, orders, diffs, mas, t, h, n_hold=h)
    eng.close()
    want = select_arma_packed(y, X, t, h, orders, diffs, mas, t, h)
    bound = mse_bound(want, y, _taus(y, X, t, want_q0(want), diffs, h, np.sqrt(t / 1095)), t, h, orders, diffs, mas)
    ok = ~np.isnan(want["cand_mse"]) & ~_near_rows(want, y, t)[:, None, None, None]
    ratio = np.abs(got["cand_mse"].astype(np.float64)[ok] - want["cand_mse"][ok]) / bound[ok]
    _le(float(ratio.max()), 1.0, "hourly 70,001: |cand_mse - oracle| / mse_bound")
    assert np.array_equal(np.isnan(got["cand_mse"]), np.isnan(want["cand_mse"]))


def test_nullable_outputs_and_a_wide_table():
    y, X, t_fit, has_c = _ma_case("daily")
    n = len(y)
    eng = _engine("auto", X, t_fit, has_c)
    lib, h = eng._lib, eng._h
    _, yd = _device(y)
    orders, diffs, mas = (0, 2), (0, 1, 2), (0, 1)
    ref = eng.fit_select_arma(yd, N_HOLD, orders, diffs, mas, t_fit, 28)
    wide = torch.full((n, 41), SENT_F, device="cuda")
    view = wide[:, 5:33]
    torch.cuda.synchronize()
    arr = lambda v: (ctypes.c_int32 * len(v))(*v)
    rc = lib.mmf_fit_select_arma_f32(h, yd.data_ptr(), n, yd.stride(0), N_HOLD, arr(orders), 2, arr(diffs), 3,
                                     arr(mas), 2, 0, t_fit, 28, view.data_ptr(), 41, *([None] * 12))
    assert rc == 0
    torch.cuda.synchronize()
    assert _same_bits(view, ref["pred"])
    assert (wide[:, :5] == SENT_F).all() and (wide[:, 33:] == SENT_F).all()
    cq = torch.full((n,), 7, device="cuda", dtype=torch.int32)
    th = torch.full((n, MA_MAX), 7.0, device="cuda")
    torch.cuda.synchronize()
    rc = lib.mmf_fit_select_arma_f32(h, yd.data_ptr(), n, yd.stride(0), N_HOLD, arr(orders), 2, arr(diffs), 3,
                                     arr(mas), 2, 0, t_fit, 28, view.data_ptr(), 41, None, None, cq.data_ptr(), None,
                                     None, None, th.data_ptr(), None, None, None, None, None)
    assert rc == 0
    torch.cuda.synchronize()
    assert _same_bits(cq, ref["choice_q"]) and _same_bits(th, ref["theta"]) and _same_bits(view, ref["pred"])
    eng.close()


def test_refused_calls_write_nothing():
    y, X, t_fit, has_c = _ma_case("daily", n=40)
    n = len(y)
    eng = mmf.ForecastEngine()
    lib, h = eng._lib, eng._h
    _, yd = _device(y)
    ld = yd.stride(0)
    f = lambda *s: torch.full(s, 7.0, device="cuda")
    i = lambda *s: torch.full(s, 7, device="cuda", dtype=torch.int32)
    bufs = [f(n, 28), i(n), i(n), i(n), f(n), f(n, 9 * 3 * 5), f(n, AR_MAX), f(n, MA_MAX), i(n), i(n), f(n), i(n)]
    host_out = np.zeros((n, 28), dtype=np.float32)

    def call(orders=(1,), diffs=(0, 1), mas=(0, 1), long_order=0, n_hold=N_HOLD, ps=t_fit, npred=28, optr=None,
             ldo=28, ld_y=ld, ctx=h):
        arr = lambda v: (ctypes.c_int32 * max(len(v), 1))(*v) if v is not None else None
        return lib.mmf_fit_select_arma_f32(ctx, yd.data_ptr(), n, ld_y, n_hold, arr(orders), len(orders or ()),
                                           arr(diffs), len(diffs or ()), arr(mas), len(mas or ()), long_order, ps,
                                           npred, bufs[0].data_ptr() if optr is None else optr, ldo,
                                           *[b.data_ptr() for b in bufs[1:]], None)
    assert call(diffs=(0,)) == -4 and call(diffs=(1,)) == -4                   # MMF_E_NOPLAN: no plan at all
    eng.plan(X, t_fit, has_c)
    assert call(diffs=(0, 1)) == -4                                            # no ARIMA plan
    eng.plan_arima(X, t_fit, 1)
    refused = [dict(mas=(1,)), dict(mas=(1, 2)), dict(mas=()), dict(mas=None), dict(mas=(0, 0)), dict(mas=(0, 2, 1)),
               dict(mas=(0, 5)), dict(mas=(0, 1, 2, 3, 4, 4)), dict(orders=tuple(range(9)), mas=(0, 1, 2, 3, 4)),
               dict(orders=tuple(range(9)), mas=(0, 1, 2, 3, 4, 5)), dict(long_order=-1), dict(long_order=33),
               dict(orders=(1, 3), mas=(0, 2), long_order=2), dict(mas=(0, 4), long_order=3),
               dict(orders=()), dict(orders=None), dict(orders=(2, 1)), dict(orders=(0, 9)), dict(diffs=()),
               dict(diffs=None), dict(diffs=(1, 0)), dict(diffs=(0, 3)), dict(diffs=(0, 2)), dict(n_hold=0),
               dict(n_hold=X.shape[0] - t_fit + 1), dict(ld_y=t_fit + N_HOLD - 1), dict(ps=-1),
               dict(npred=X.shape[0] + 1), dict(ldo=27), dict(optr=host_out.ctypes.data), dict(ctx=None)]
    for kw in refused:
        assert call(**kw) != 0, kw
    torch.cuda.synchronize()
    assert all((b == 7).all() for b in bufs)
    assert call(orders=(0, 1, 2, 3, 4, 5, 6, 7), mas=(0, 1, 2, 3, 4)) == 0    # 32 pairs: accepted
    torch.cuda.synchronize()
    assert not all((b == 7).all() for b in bufs)
    for b in bufs:
        b.fill_(7)
    torch.cuda.synchronize()
    Xo = X.copy()
    Xo[5, 1] += 1e-9
    eng.plan_arima(Xo, t_fit, 2)
    assert call(diffs=(0, 1)) == -1                                            # MMF_E_INVALID: plans of different X
    torch.cuda.synchronize()
    assert all((b == 7).all() for b in bufs)
    assert not host_out.any()
    eng.close()


def test_other_calls_unchanged_and_a_shared_context_matches_a_fresh_one():
    y, X, t_fit, has_c = _ma_case("daily")
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
                eng.fit_forecast_arma(yf, 1, 1, 1, t_fit, 28)["pred"].clone(),
                eng.fit_select_arima(yd, N_HOLD, (0, 1, 2), (0, 1), t_fit, 28)["pred"].clone(),
                eng.fit_forecast_ragged(yf, [0, 70, len(y)]).clone(), bt["pred"].clone(), bt["metrics"].clone(),
                bt["status"].clone())

    args = ((REF, t_fit, 28), (((8,), (2,), (0, 4)), 0, t_fit + 64), (((1, 3), (0, 2), (0, 1, 3)), 50, 100))
    before = calls()
    shared = [_call(eng, yd, *g, ps, npred) for g, ps, npred in args]
    after = calls()
    assert all(_same_bits(a, b) for a, b in zip(before, after))
    fresh_eng = mmf.ForecastEngine()
    fresh_eng.plan(X, t_fit, has_c)
    fresh_eng.plan_arima(X, t_fit, 2)
    fresh = [_call(fresh_eng, yd, *g, ps, npred) for g, ps, npred in args]
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
import test_gpu_arma_select as T
from arma_select_oracle import mse_bound, select_arma_packed
from oracle import mmf_oracle as O
n, t, h = 120, 400, 28
rng = np.random.default_rng(8)
X = O.design_matrix(O.calendar_grid("2019-01-01", t + h, "D"), t)
w = np.zeros((n, t + h + 1))
eps = rng.normal(0, 5, (n, t + h + 1))
for k in range(1, t + h + 1):
    w[:, k] = 0.7 * w[:, k - 1] + eps[:, k] + 0.5 * eps[:, k - 1]
y = (1000 + w[:, 1:]).astype(np.float32)
orders, diffs, mas = (1,), (0, 1), (0, 1)
eng = T._engine("auto", X, t, True)
_, yd = T._device(y)
got = T._call(eng, yd, orders, diffs, mas, t, h)
want = select_arma_packed(y, X, t, h, orders, diffs, mas, t, h)
b = mse_bound(want, y, T._taus(y, X, t, T.want_q0(want), diffs), t, h, orders, diffs, mas)
ok = ~T._near_rows(want, y, t)[:, None, None]
r = np.abs(got["cand_mse"].astype(np.float64) - want["cand_mse"]) / b
gated = np.stack([want["hold"][k][1][0]["gated"] for k in range(len(diffs))], axis=1)
sel = (gated & ok[:, :, 0])
rq = r[:, :, 1, 0]
print(json.dumps({{"worst_q0": float(np.where(ok[:, :, 0], r[:, :, 0, 0], 0).max()),
                  "worst": float(np.where(sel, rq, 0).max()), "over": int((sel & (rq > 1)).sum()),
                  "cands": int(sel.sum()), "lib": mmf.LIB_PATH}}))
"""


@pytest.mark.parametrize("lib", ["product", "onestep"])
def test_negative_control_with_a_leaky_one_step_score(lib):
    """ARMA(1, 1) errors: the build that feeds each observed held-out value into the candidates' histories
    (tests/_build/libmmf_armasel_onestep.so) must exceed mse_bound on at least half of the gated q >= 1 candidates'
    rows; the product library stays within it"""
    env = dict(os.environ)
    env.pop("MMF_LIB", None)
    if lib == "onestep":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_armasel_onestep.so")
        assert os.path.exists(env["MMF_LIB"]), "negative-control library missing: run __graft_entry__.build()"
    r = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    record_err("test_gpu_arma_select negative control", got["worst"], 1.0, what=lib, over=got["over"],
               cands=got["cands"])
    assert got["cands"] > 0, got
    if lib == "product":
        assert got["worst"] <= 1.0 and got["worst_q0"] <= 1.0, got
    else:
        assert got["lib"].endswith("libmmf_armasel_onestep.so") and got["over"] >= got["cands"] // 2, got


@pytest.mark.parametrize("frame", ["daily", "weekly"])
def test_forecast_groups_with_pdq_selection(frame):
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
    orders, diffs, mas = REF
    out = mmf.forecast_groups(pdf, ar=orders, diff=diffs, ma=mas, **kw)
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
        want = select_arma_packed(y, X, t_fit, h, orders, diffs, mas, t_fit, h)
        b = mse_bound(want, y, _taus(y, X, t_fit, want_q0(want), diffs, h), t_fit, h, orders, diffs, mas)
        # the hold-out MSE of the group's forecast lies within two bounds of the oracle's minimum; groups whose score is
        # closest to another candidate's oracle score took another winner (two candidates within the bounds), counted
        got = g["Demand_Fitted"].to_numpy().astype(np.float64)
        fut = _score_of(got[t_fit:t_fit + h], y[0, t_fit:t_fit + h])
        best = want["cand_mse"][0, want["k"][0], want["l"][0], want["j"][0]]
        if not np.isnan(best) and not _near_rows(want, y, t_fit)[0]:
            worst = max(worst, float((fut - best) / max(2 * b[0].max(), 1e-30)))
            flat = want["cand_mse"][0].reshape(-1)
            near = int(np.nanargmin(np.abs(flat - fut)))
            amb += int(flat[near] != best)
    record_err("arma_select_frames_ambiguous_groups", float(amb), float(out.groupby(["Product", "SKU"]).ngroups),
               what=frame)
    _le(worst, 1.0, f"forecast_groups(ar=(0..4), diff=(0, 1, 2), ma=(0..4)) {frame}: hold-out MSE over the oracle's "
        "minimum / bound")


def _score_of(pred, yh):
    ok = np.isfinite(pred) & np.isfinite(yh)
    return float(np.mean((yh[ok].astype(np.float64) - pred[ok]) ** 2)) if ok.any() else np.nan
