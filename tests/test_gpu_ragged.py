"""GPU (-m gpu): ragged batches -- groups on many calendars in one launch (mmf_plan_calendars +
mmf_fit_forecast_ragged_f32, DESIGN.md 4.8) -- beyond the seven short daily calendars of test_gpu_configs.py.

A. Long and short calendars in one launch: t_fit from 33 to 65,535, ordered so that every CTA of the tensor-core
   kernel walks tiles that fold their accumulators (> 18 chunks) and tiles that do not, with both chunk parities;
   fit_warp's 2,784 shared-memory design rows through the per-calendar general pass.
B. Store paths: common horizons 1 to 64 into views of wider pattern-filled tables, and per-calendar windows anywhere
   in the design (a "many" plan, written by predict_tc_kernel<true> through per-calendar output maps).
C. Caller designs in a ragged plan (ForecastEngine.plan_designs): p = 1 with and without a constant, p = 16 without
   one, aliased columns that differ from calendar to calendar, exog_only calendars with every column aliased.
D. Many and degenerate calendars: 1,100 calendars of 0 to 3 series, empty calendars first, last and in between, one
   calendar owning every row, calendars of 128 and 129 series.
E. The host-side tables cached between calls (tiles, y maps, predict units, output maps) against a fresh engine.
F. Refused calls and plans write nothing and keep the plan in force.
G. Exact 2^k scaling, assume_finite, more than 2^20 rows, and a negative control for the section-A bound.
H. forecast_groups on multi-calendar frames against the per-group oracle UDF, each group within its own bound.

Every batch plants the row mix of test_gpu_abi_contract (KINDS) in every calendar, interleaved so that kinds share a
tile; columns past a row's own t_fit hold NaN.  Every forecast is checked against the float64 oracle (statuses equal,
values within tolerance(row, leverage of its calendar) x mask factor x max(1, sqrt(t_fit / 1095))) and, where the store
family is the same, bit for bit against single-calendar calls on the same rows: a plan whose calendars share one
window of <= 64 rows is written by the fit kernel's epilogue, as a single call of that window is; any other plan by
predict_tc_kernel, as a single call of a window of more than 64 rows is (a shorter window is compared with a longer
single-call window that contains it: within predict_tc_kernel a design row's value does not depend on the window)."""
import json
import os
import subprocess
import sys
from dataclasses import dataclass

import numpy as np
import pytest

import mmf
from conftest import ROOT, forecast_leverage, record_err
from oracle import mmf_oracle as O
from test_gpu_abi_contract import (KINDS, PATTERN, _check, _design, _expected_pending, _kind_cols, _long_scale,
                                   _mask_factor, _oracle, _plant, _round4, _series)
from test_gpu_edges import SCALES, _assert_equivariant, _le, _row_tol, _same_bits

pytestmark = pytest.mark.gpu

H = 28
LEVEL = 500.0
_X_CACHE = {}


@dataclass
class Cal:
    """one calendar of a ragged plan: `design(n_rows)` -> X [n_rows, p] (a row does not depend on n_rows, so a longer
    design for a single-calendar call has the same rows); fit rows [0, t_fit), evaluated rows [ps, ps + npred), n series.
    `key` names the design: calendars with one key share X."""
    design: object
    t_fit: int
    ps: int
    npred: int
    n: int
    key: tuple
    has_c: bool = True

    @property
    def n_rows(self):
        return max(self.t_fit, self.ps + self.npred)

    def X(self, n_rows=None):
        k = (self.key, n_rows or self.n_rows)
        if k not in _X_CACHE:
            _X_CACHE[k] = np.asarray(self.design(k[1]), dtype=np.float64)
        return _X_CACHE[k]


def _cal(design, t_fit, n, mode, key, has_c=True, h=H):
    """future: forecast h rows past t_fit; holdout: a calendar of t_fit + h dates, every one of them evaluated"""
    if mode == "future":
        return Cal(design, t_fit, t_fit, h, n, key, has_c)
    return Cal(design, t_fit, 0, t_fit + h, n, key, has_c)


def _daily(start, t_fit, design="trend_season_exog", freq="D"):
    return lambda n_rows: O.design_matrix(O.calendar_grid(np.datetime64(start, "D"), n_rows, freq), t_fit, design)


def _p5_16(t_fit):
    """the p5 caller design padded with 11 zero columns: p = 16 like the calendar design, 11 columns aliased"""
    return lambda n_rows: np.pad(_design("p5", n_rows, t_fit)[0], ((0, 0), (0, 11)))


def _caller(name, t_fit, seed=0):
    return lambda n_rows: _design(name, n_rows, t_fit, seed)[0]


def _batch(cals, seed, kinds=KINDS, width=None):
    """y [sum n, round4(max t_fit)] float32: every calendar's series on its own design, the row mix planted, NaN past
    each row's t_fit; rows = cal_row_start"""
    rows = np.concatenate([[0], np.cumsum([c.n for c in cals])]).astype(np.int64)
    y = np.full((int(rows[-1]), width or _round4(max(c.t_fit for c in cals))), np.nan, dtype=np.float32)
    for ci, c in enumerate(cals):
        if c.n:
            blk = y[rows[ci]:rows[ci + 1]]
            blk[:, :c.t_fit] = _series(c.X(), c.t_fit, c.n, seed + ci, LEVEL)
            _plant(blk, c.t_fit, shift=ci, kinds=kinds)
    return y, rows


def _plan(eng, cals):
    eng.plan_designs([c.X() for c in cals], [c.t_fit for c in cals], [c.ps for c in cals], [c.npred for c in cals],
                     cals[0].has_c)


def _ragged(eng, cals, y, rows, out=None, plan=True):
    import torch
    if plan:
        _plan(eng, cals)
    yd = y if hasattr(y, "cuda") else torch.from_numpy(y).cuda()
    res = eng.fit_forecast_ragged(yd, rows, out=out, want_status=True, want_stats=True)
    torch.cuda.synchronize()
    return res


def _family(cals):
    one = all(c.npred == cals[0].npred for c in cals) and cals[0].npred <= 64
    return "fit_tc" if one else "predict_tc"


def _groups(cals, rows):
    """[(calendar, row indices)]: calendars with the same design and window pooled (one oracle call each)"""
    g = {}
    for ci, c in enumerate(cals):
        if c.n:
            g.setdefault((c.key, c.t_fit, c.ps, c.npred), []).append(ci)
    return [(cals[v[0]], np.concatenate([np.arange(rows[i], rows[i + 1]) for i in v])) for v in g.values()]


def _assert_single_bits(engs, c, Y, pred_t, st_t, idx, fam, what):
    """the rows of one calendar through plan() + fit_forecast() of every engine: bit-equal to the ragged result"""
    import torch
    ps, npw, X = c.ps, c.npred, c.X()
    if fam == "predict_tc" and c.npred <= 64:         # a window of more than 64 rows around it: predict_tc_kernel too
        npw, X = 65, c.X(max(c.n_rows, c.ps + 65))
    yd = mmf.device_packed(np.ascontiguousarray(Y[:, :c.t_fit]))
    it = torch.from_numpy(idx).cuda()
    want_p, want_s = pred_t[it][:, :c.npred], st_t[it]
    for k, eng in engs.items():
        eng.plan(X, c.t_fit, c.has_c)
        r = eng.fit_forecast(yd, ps, npw, want_status=True)
        torch.cuda.synchronize()
        assert _same_bits(r["pred"][:, :c.npred], want_p), (what, k, "pred")
        assert _same_bits(r["status"], want_s), (what, k, "status")


# A row with a pivot d_j / G_jj of the oracle's in-order Cholesky (kept or dropped) within a factor PIVOT_BAND of
# PIVOT_TOL is held neither to the value bound nor to the oracle's status.  Within a factor of ~1.3 float32 may keep a
# column the oracle drops or the reverse; up to a factor of 3 the float32 Gram of the general pass is itself at the edge
# of the mask factor: a float32 emulation of the row with a 45-value gap (pivot 2.7e-3, 80 fit days) gives 0.85 of the
# bound through the Gram downdate and 0.99 through a Gram over the observed rows, and the GPU's own summation order
# 1.53.  The ragged launch must reproduce the single-calendar call bit for bit on these rows, so every group holding
# one is compared with that call, whatever the sampling; their count and their worst error / bound are logged.
PIVOT_BAND = 3.0


def _pivot_distance(Y, X, t_fit):
    """per row: min over the columns of max(r, PIVOT_TOL) / min(r, PIVOT_TOL), r = d_j / G_jj the pivot ratio of the
    oracle's in-order Cholesky of the row's own Gram (O.solve_series); inf for rows without an observed value"""
    W, _ = O.whiten(np.asarray(X, dtype=np.float64)[:t_fit])
    a = (np.asarray(X, dtype=np.float64) @ W)[:t_fit]
    out = np.full(len(Y), np.inf)
    for i, row in enumerate(np.asarray(Y)[:, :t_fit]):
        obs = np.isfinite(row)
        if not obs.any():
            continue
        G = a[obs].T @ a[obs]
        p = G.shape[0]
        L = np.zeros((p, p))
        for j in range(p):
            if G[j, j] <= 0:
                continue
            d = G[j, j] - L[j, :j] @ L[j, :j]
            r = max(d / G[j, j], 1e-300)
            out[i] = min(out[i], max(r, O.PIVOT_TOL) / min(r, O.PIVOT_TOL))
            if d <= O.PIVOT_TOL * G[j, j]:
                continue
            L[j, j] = np.sqrt(d)
            L[j + 1:, j] = (G[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return out


def _bound_ratio(pred, Y, c, orc):
    """per row: max error / (tolerance(row, leverage) x mask factor x sqrt scale), as _check computes it"""
    want = orc["gamma"] @ orc["A"][c.ps:c.ps + c.npred].T
    tol = (_row_tol(Y[:, :c.t_fit], forecast_leverage(c.X(), c.t_fit, c.ps, c.npred))
           * _mask_factor(Y, c.X(), c.t_fit, c.ps, c.npred, orc["ratio"]) * _long_scale(c.t_fit))
    return np.abs(pred[:, :c.npred] - want).max(axis=1) / tol


def _pending(y, t_fit, has_c):
    """_expected_pending; without a constant (has_constant = 0) there is nothing to centre on, so a missing first value
    sends no row to the general pass by itself"""
    if has_c:
        return _expected_pending(y, t_fit)
    bad = ~np.isfinite(y[:, :t_fit])
    seg = (np.arange(t_fit) // 32) % 2
    nm0, nm1 = bad[:, seg == 0].sum(axis=1), bad[:, seg == 1].sum(axis=1)
    return int(((nm0 > 44) | (nm1 > 44) | (2 * (nm0 + nm1) > t_fit)).sum())


def _verify(cals, y, rows, res, what, sample=1, kernels=("tc", "auto"), pending=True):
    """every calendar against the oracle (rows with an ambiguous kept set: bit for bit against the single-calendar
    call); every `sample`-th group bit for bit against single-calendar calls; stats.n_pending equal to the rows the
    masks send to the general pass"""
    pred_t, st_t = res["pred"], res["status"]
    pred, status = pred_t.cpu().numpy(), st_t.cpu().numpy()
    fam = _family(cals)
    engs = {k: mmf.ForecastEngine(kernel=k) for k in kernels}
    n_amb, worst_amb = 0, 0.0
    for gi, (c, idx) in enumerate(_groups(cals, rows)):
        Y = y[idx]
        w = f"{what}: t_fit={c.t_fit} window=({c.ps}, {c.npred}) {c.key[0]}"
        orc = _oracle(Y, c.X(), c.t_fit)
        ok = _pivot_distance(Y, c.X(), c.t_fit) > PIVOT_BAND          # (_check compares their statuses)
        sub = dict(orc, gamma=orc["gamma"][ok], status=orc["status"][ok], ratio=orc["ratio"][ok])
        if ok.any():
            _check(pred[idx][ok, :c.npred], status[idx][ok], Y[ok], c.X(), c.t_fit, c.ps, c.npred, w, sub,
                   scale=_long_scale(c.t_fit))
        amb = ~ok & (orc["status"] != 1) & (status[idx] != 1)
        if amb.any():
            n_amb += int(amb.sum())
            sub = dict(orc, gamma=orc["gamma"][amb], ratio=orc["ratio"][amb])
            worst_amb = max(worst_amb, float(_bound_ratio(pred[idx][amb], Y[amb], c, sub).max()))
        if gi % sample == 0 or not ok.all():
            _assert_single_bits(engs, c, Y, pred_t, st_t, idx, fam, w)
    for e in engs.values():
        e.close()
    record_err(os.environ.get("PYTEST_CURRENT_TEST", "?").split("::")[-1].split(" ")[0], 0.0, 1.0,
               what=f"{what}: rows with an ambiguous kept set, checked bit for bit against the single-calendar call",
               rows_ambiguous=n_amb, worst_ambiguous_err_over_bound=worst_amb)
    if pending:
        want = sum(_pending(y[rows[i]:rows[i + 1]], c.t_fit, c.has_c) for i, c in enumerate(cals) if c.n)
        assert res["stats"].n_pending == want, (what, res["stats"].n_pending, want)


def _pattern_out(n, width, pitch):
    """(buffer, out, mask of out's elements): out = an [n, width] view with row pitch `pitch` into a PATTERN-filled
    int32 buffer, a guard row and more above and below; out's first element is 16-B aligned"""
    import torch
    off = _round4(pitch + 1)
    buf = torch.full(((n + 2) * pitch + 8,), PATTERN, dtype=torch.int32, device="cuda")
    out = buf.view(torch.float32).as_strided((n, width), (pitch, 1), off)
    mine = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
    mine.as_strided((n, width), (pitch, 1), off).fill_(True)
    return buf, out, mine


# =====================================================================================================================
# A. long and short calendars in one launch
# =====================================================================================================================
# fit windows and chunks: 1152 (36: the longest that never folds), 1153 / 2784 / 2785 / 5000 (37 / 87 / 88 / 157: the
# accumulators fold every 18 chunks of a group), 33 / 64 / 65 / 400 / 576 (2 / 2 / 3 / 13 / 18).  Any three consecutive
# entries (cyclically) hold a folding and a non-folding window, an odd and an even chunk count.
A_ORDER = (2785, 65, 1152, 1153, 33, 2784, 64, 400, 5000, 576)
A_FOLDS = 1152


def _a_start(t):
    return np.datetime64("2011-01-03", "D") + np.timedelta64(int(t) % 97, "D")


@pytest.mark.parametrize("mode", ["future", "holdout"])
def test_long_and_short_calendars_share_every_cta(mode):
    """3 x SM-count one-tile calendars (8 to 16 series each) on the ten fit windows of A_ORDER: the grid has SM-count
    CTAs and CTA b walks tiles b, b + SMs, b + 2 SMs, whose windows are A_ORDER[(b, b + 1, b + 2) mod 10] -- a folding
    and a non-folding tile, an odd and an even chunk count for every CTA.  A second launch puts two 65,535-row calendars
    (the p5 design, zero-padded to 16 columns) between short daily ones."""
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    for b in range(len(A_ORDER)):
        win = [A_ORDER[(b + k) % len(A_ORDER)] for k in range(3)]
        assert {t > A_FOLDS for t in win} == {True, False} and {(t + 31) // 32 % 2 for t in win} == {0, 1}, win
    cals = []
    for i in range(3 * sm):
        t = A_ORDER[(i % sm + i // sm) % len(A_ORDER)]
        cals.append(_cal(_daily(_a_start(t), t), t, 8 + i % 9, mode, ("daily", str(_a_start(t)), t)))
    y, rows = _batch(cals, seed=11)
    eng = mmf.ForecastEngine()
    res = _ragged(eng, cals, y, rows)
    assert res["stats"].kernel_launches >= (1 if mode == "future" else 2)
    _verify(cals, y, rows, res, f"A {mode}")
    longest = [_cal(_p5_16(65535), 65535, 16, mode, ("p5", 65535)), _cal(_daily(_a_start(33), 33), 33, 11, mode,
               ("daily", str(_a_start(33)), 33)), _cal(_p5_16(65535), 65535, 9, mode, ("p5", 65535)),
               _cal(_daily(_a_start(400), 400), 400, 16, mode, ("daily", str(_a_start(400)), 400))]
    y2, rows2 = _batch(longest, seed=12)
    res2 = _ragged(eng, longest, y2, rows2)
    _verify(longest, y2, rows2, res2, f"A {mode} 65,535")
    eng.close()


# =====================================================================================================================
# B. store paths: common horizons into wider tables, per-calendar windows
# =====================================================================================================================
B_CALS = ((33, 1), (64, 127), (65, 129), (400, 40), (1153, 200))     # (t_fit, series)


@pytest.mark.parametrize("h", [1, 3, 4, 7, 28, 29, 32, 64])
def test_common_horizon_into_views_of_a_wider_table(h):
    """future mode, one horizon for every calendar (the fit kernel's epilogue: bulk stores for ld_out == h <= 28 and
    h % 4 == 0, 16-B or scalar stores otherwise): out with pitch h, the next multiple of 4 + 4 and h + 5 (rows not
    16-B aligned) -- bit-equal to each other, nothing outside [0, h) of any row written"""
    cals = [_cal(_daily(_a_start(t), t), t, n, "future", ("daily", str(_a_start(t)), t), h=h) for t, n in B_CALS]
    y, rows = _batch(cals, seed=20 + h)
    n = int(rows[-1])
    eng = mmf.ForecastEngine()
    _plan(eng, cals)
    first = None
    for pitch in (h, _round4(h) + 4, h + 5):
        buf, out, mine = _pattern_out(n, h, pitch)
        res = _ragged(eng, cals, y, rows, out=out, plan=False)
        assert bool((buf[~mine] == PATTERN).all()), (h, pitch, "caller memory outside [0, h) changed")
        if first is None:
            first = res
            _verify(cals, y, rows, res, f"B h={h}")
        else:
            assert _same_bits(res["pred"], first["pred"]) and _same_bits(res["status"], first["status"]), (h, pitch)
    eng.close()


def test_per_calendar_windows_in_a_many_plan():
    """(pred_start, n_pred) per calendar through mmf_plan_calendars: (t_fit, 5), (t_fit, 64), (t_fit, 65), (0, 200),
    a window inside the fit rows and one across t_fit; out with ld_out = round4(max n_pred) + 8.  Nothing from
    round4(n_pred_c) on is written in a row of calendar c, nor outside the view."""
    spec = ((372, 372, 5, 130), (100, 100, 64, 1), (250, 250, 65, 129), (400, 0, 200, 64), (300, 120, 40, 200),
            (65, 40, 60, 57))                                      # (t_fit, pred_start, n_pred, series)
    cals = [Cal(_daily(_a_start(t), t), t, ps, npd, n, ("daily", str(_a_start(t)), t)) for t, ps, npd, n in spec]
    y, rows = _batch(cals, seed=31)
    n = int(rows[-1])
    n_out = max(c.npred for c in cals)
    pitch = _round4(n_out) + 8
    buf, out, mine = _pattern_out(n, n_out, pitch)
    may = mine.clone()
    off = _round4(pitch + 1)
    for ci, c in enumerate(cals):                 # columns [round4(n_pred_c), n_out) of calendar c: not to be written
        for r in range(int(rows[ci]), int(rows[ci + 1])):
            may[off + r * pitch + _round4(c.npred):off + r * pitch + n_out] = False
    eng = mmf.ForecastEngine()
    res = _ragged(eng, cals, y, rows, out=out)
    assert bool((buf[~may] == PATTERN).all()), "caller memory outside round4(n_pred_c) changed"
    _verify(cals, y, rows, res, "B many")
    eng.close()


# =====================================================================================================================
# C. caller designs in a ragged plan
# =====================================================================================================================
C_FITS = (33, 47, 64, 65, 128, 400)
C_SERIES = (1, 127, 129, 40, 200, 16)
C_PLANS = {
    "mean": [("mean", t, 0) for t in C_FITS],
    "t1": [("t1", t, 0) for t in C_FITS],
    "gauss16": [("gauss16", t, 100 + i) for i, t in enumerate(C_FITS)],
    "p6_aliased": [("dup", 33, 0), ("zero", 97, 0), ("fit_zero", 200, 0), ("twice_one", 400, 0)],
}
# (start, t_fit, freq): none of covid / christmas / new_year in the first fit window (every column aliased), only covid
# in the second, all three in the others
C_EXOG = (("2019-06-03", 60, "D"), ("2020-04-01", 90, "D"), ("2019-11-20", 120, "D"), ("2019-12-01", 400, "D"),
          ("2019-01-07", 80, "W-MON"), ("2020-06-01", 40, "W-MON"), ("2017-03-06", 150, "W-MON"))


@pytest.mark.parametrize("mode", ["future", "holdout"])
@pytest.mark.parametrize("plan", list(C_PLANS) + ["exog_only"])
def test_caller_designs_in_a_ragged_plan(plan, mode):
    """p and has_constant are per plan: every calendar of a plan gets its own design of that kind (its own seed for
    gauss16, its own aliased column for p6), so the epilogue reloads a different kept mask per calendar"""
    if plan == "exog_only":
        cals = [_cal(_daily(s, t, "exog_only", f), t, C_SERIES[i % len(C_SERIES)], mode, ("exog", s, t, f), False)
                for i, (s, t, f) in enumerate(C_EXOG)]
        kept = [O.whiten(c.X()[:c.t_fit])[1][:3] for c in cals]
        assert not kept[0].any() and kept[1].tolist() == [True, False, False] and kept[3].all()
    else:
        cals = []
        for i, (name, t, seed) in enumerate(C_PLANS[plan]):
            has_c = _design(name, t + 1, t)[1]
            cals.append(_cal(_caller(name, t, seed), t, C_SERIES[i % len(C_SERIES)], mode, (name, t, seed), has_c))
    y, rows = _batch(cals, seed=40)
    eng = mmf.ForecastEngine()
    res = _ragged(eng, cals, y, rows)
    _verify(cals, y, rows, res, f"C {plan} {mode}")
    eng.close()


# =====================================================================================================================
# D. many and degenerate calendars
# =====================================================================================================================
def _d_cal(c, n, mode, t=None):
    t = t or 33 + (7 * c) % 90
    start = np.datetime64("2018-01-01", "D") + np.timedelta64(c, "D")
    return _cal(_daily(start, t), t, n, mode, ("daily", str(start), t))


def test_a_thousand_calendars_of_one_to_three_series():
    """1,100 calendars (every group on its own first date and length, as forecast_groups builds them), 1 to 3 series
    each, empty calendars first, in the middle and last: every calendar against the oracle, every 37th bit for bit
    against a single-calendar call"""
    n_cal = 1100
    cals = [_d_cal(c, 0 if c in (0, 550, n_cal - 1) else 1 + c % 3, "future") for c in range(n_cal)]
    y, rows = _batch(cals, seed=50)
    eng = mmf.ForecastEngine()
    res = _ragged(eng, cals, y, rows)
    _verify(cals, y, rows, res, "D 1,100 calendars", sample=37)
    eng.close()


@pytest.mark.parametrize("mode", ["future", "holdout"])
def test_empty_calendars_one_owner_and_tile_edges(mode):
    """[empty, every row, empty] and [empty, empty, 129, empty, 128, 1, empty] series per calendar"""
    eng = mmf.ForecastEngine()
    for li, counts in enumerate(((0, 300, 0), (0, 0, 129, 0, 128, 1, 0))):
        cals = [_d_cal(7 * li + c, n, mode, t=(64, 400, 47, 1153, 65, 200, 96)[c]) for c, n in enumerate(counts)]
        y, rows = _batch(cals, seed=60 + li)
        res = _ragged(eng, cals, y, rows)
        _verify(cals, y, rows, res, f"D {mode} {counts}")
    eng.close()


# =====================================================================================================================
# E. cached tables
# =====================================================================================================================
def _per_cal_equal(a, b, cals, rows, what):
    """pred [:, :n_pred_c] and status of every calendar bit-equal (columns past round4(n_pred_c) are the caller's)"""
    assert _same_bits(a["status"], b["status"]), (what, "status")
    for ci, c in enumerate(cals):
        r0, r1 = int(rows[ci]), int(rows[ci + 1])
        assert _same_bits(a["pred"][r0:r1, :c.npred], b["pred"][r0:r1, :c.npred]), (what, ci)


def _fresh(cals, yd, rows):
    eng = mmf.ForecastEngine()
    res = _ragged(eng, cals, yd, rows)
    res = {"pred": res["pred"].clone(), "status": res["status"].clone()}
    eng.close()
    return res


@pytest.mark.parametrize("mode", ["future", "holdout"])
def test_cached_tables_follow_their_keys(mode):
    """one engine, a sequence of calls that hit or miss the tile table / y maps (keyed on y, n, ld_y, the row split)
    and the predict units / output maps (also on out, ld_out); every call bit-equal to a fresh engine's"""
    import torch
    cals = [_d_cal(c, n, mode, t=t) for c, (t, n) in enumerate(((64, 130), (400, 1), (1153, 200), (33, 57)))]
    other = [_d_cal(10 + c, n, mode, t=t) for c, (t, n) in enumerate(((100, 130), (33, 1), (700, 200), (65, 57)))]
    width = _round4(1153)
    y1, rows = _batch(cals, seed=70, width=width)
    y1b, _ = _batch(cals, seed=71, width=width)
    y2, _ = _batch(other, seed=72, width=width)
    yd = torch.from_numpy(y1).cuda()
    eng = mmf.ForecastEngine()
    n_out = max(c.npred for c in cals)
    out0 = _pattern_out(int(rows[-1]), n_out, _round4(n_out))[1] if mode == "holdout" else None

    def call(cs, rs, out=out0, plan=False, what=""):
        got = _ragged(eng, cs, yd, rs, out=out, plan=plan)
        _per_cal_equal(got, _fresh(cs, yd, rs), cs, rs, f"{mode}: {what}")
        return got

    call(cals, rows, plan=True, what="first call")
    call(cals, rows, what="same buffers again")
    yd.copy_(torch.from_numpy(y1b))
    call(cals, rows, what="new contents at the same y")
    split = rows.copy()
    split[1:-1] = (64, 65, 300)
    call(cals, split, what="another row split, same y and n")
    if mode == "holdout":
        for pitch in (_round4(n_out) + 4, _round4(n_out) + 12):
            _, out, _ = _pattern_out(int(rows[-1]), n_out, pitch)
            call(cals, rows, out=out, what=f"another out, ld_out={pitch}")
    yd.copy_(torch.from_numpy(y2))
    _plan(eng, other)
    last = call(other, rows, what="re-plan with other calendars, same n_cal, y and row split")
    X = _daily("2019-01-01", 400)(428)                   # a plain plan and a backtest plan in between
    eng.plan(X, 400, True)
    eng.fit_forecast(mmf.device_packed(y2[:, :400]), 400, H)
    eng.plan_backtest("2019-01-01", 428, "D", H, 3)
    yb = mmf.device_packed(np.where(np.isfinite(y2[:, :428]), y2[:, :428], 1.0))
    eng.backtest(yb)
    torch.cuda.synchronize()
    again = _ragged(eng, other, yd, rows, plan=False)
    _per_cal_equal(again, last, other, rows, f"{mode}: after plan() and plan_backtest()")
    eng.close()


# =====================================================================================================================
# F. refusals write nothing
# =====================================================================================================================
def _raw(eng, y_ptr, n, ld_y, rows, out_ptr, ld_out, st_ptr):
    r = np.ascontiguousarray(rows, dtype=np.int64)
    return eng._lib.mmf_fit_forecast_ragged_f32(eng._h, y_ptr, n, ld_y, r.ctypes.data, out_ptr, ld_out, st_ptr, None)


def _raw_plan(eng, X, n_rows, t_fit, ps, npred, p, has_c):
    a = [np.ascontiguousarray(v, dtype=np.int32) for v in (n_rows, t_fit, ps, npred)]
    X = np.ascontiguousarray(X, dtype=np.float64)
    return eng._lib.mmf_plan_calendars(eng._h, X.ctypes.data, len(a[0]), a[0].ctypes.data, a[1].ctypes.data,
                                       a[2].ctypes.data, a[3].ctypes.data, p, has_c)


def test_refused_calls_and_plans_write_nothing():
    """each refused mmf_fit_forecast_ragged_f32 returns its code and leaves the pattern-filled out and status as they
    were; each refused mmf_plan_calendars keeps the previous plan (the next call is bit-equal to the one before)"""
    import torch
    cals = [_d_cal(c, n, "holdout", t=t) for c, (t, n) in enumerate(((64, 130), (400, 1), (200, 57)))]
    y, rows = _batch(cals, seed=80)
    n, ld = int(rows[-1]), y.shape[1]
    t_max, n_out = max(c.t_fit for c in cals), max(c.npred for c in cals)
    yd = torch.from_numpy(y).cuda()
    ybig = torch.full((n, ld + 8), float("nan"), device="cuda")
    ybig[:, :ld] = yd
    eng = mmf.ForecastEngine()
    _plan(eng, cals)
    before = _ragged(eng, cals, yd, rows, plan=False)
    ld_out = _round4(n_out) + 4
    table = torch.full((n, ld_out + 8), PATTERN, dtype=torch.int32, device="cuda")
    status = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    keep_t, keep_s = table.clone(), status.clone()
    hy, ho = np.zeros((n, ld), np.float32), np.zeros((n, ld_out), np.float32)
    y_p, o_p, s_p = yd.data_ptr(), table.data_ptr(), status.data_ptr()
    bad_rows = rows.copy()
    bad_rows[1], bad_rows[2] = bad_rows[2], bad_rows[1]
    # (a cal_row_start that does not end at n: test_gpu_configs.test_ragged_rejects_what_it_cannot_do)
    cases = [("ld_y < t_fit_max", (y_p, n, _round4(t_max) - 4, rows, o_p, ld_out, s_p), -1),
             ("ld_y % 4 != 0", (ybig.data_ptr(), n, ld + 1, rows, o_p, ld_out, s_p), -3),
             ("y off by one float", (y_p + 4, n, ld, rows, o_p, ld_out, s_p), -3),
             ("out off by one float", (y_p, n, ld, rows, o_p + 4, ld_out, s_p), -3),
             ("ld_out % 4 != 0", (y_p, n, ld, rows, o_p, ld_out + 1, s_p), -1),
             ("ld_out < n_pred_max", (y_p, n, ld, rows, o_p, _round4(n_out) - 4, s_p), -1),
             ("host y", (hy.ctypes.data, n, ld, rows, o_p, ld_out, s_p), -1),
             ("host out", (y_p, n, ld, rows, ho.ctypes.data, ld_out, s_p), -1),
             ("non-monotone cal_row_start", (y_p, n, ld, bad_rows, o_p, ld_out, s_p), -1)]
    for what, args, code in cases:
        rc = _raw(eng, *args)
        torch.cuda.synchronize()
        assert rc == code, (what, rc, mmf._native.load().mmf_last_error())
        assert torch.equal(table, keep_t) and torch.equal(status, keep_s), what
    fresh = mmf.ForecastEngine()
    assert _raw(fresh, y_p, n, ld, rows, o_p, ld_out, s_p) == -4, "no plan"
    fresh.close()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="relaxed"):
        eng.set_stream(s.cuda_stream)
        rc = _raw(eng, y_p, n, ld, rows, o_p, ld_out, s_p)
    del g
    assert rc == -3, ("capturing stream", rc)
    torch.cuda.synchronize()
    assert torch.equal(table, keep_t) and torch.equal(status, keep_s), "capturing stream"
    after = _ragged(eng, cals, yd, rows, plan=False)
    _per_cal_equal(after, before, cals, rows, "after the refused calls")
    Xs = [c.X() for c in cals]
    X = np.concatenate(Xs)
    nr, tf = [c.n_rows for c in cals], [c.t_fit for c in cals]
    ps, npd = [c.ps for c in cals], [c.npred for c in cals]
    nan_x = X.copy()
    nan_x[nr[0] + 5, 7] = np.inf
    not_one = X.copy()
    not_one[nr[0] + nr[1] + 3, 0] = 1.5                     # a row of the last calendar
    plans = [("t_fit < 33", (X, nr, [32, tf[1], tf[2]], ps, npd, 16, 1), -3),
             ("t_fit > 65,535", (np.zeros((65536 + nr[1] + nr[2], 16)), [65536] + nr[1:], [65536] + tf[1:], ps, npd, 16,
                                 0), -3),
             ("n_cal = 0", (X, [], [], [], [], 16, 1), -1),
             ("n_cal = 65,536", (X, nr, tf, ps, npd, 16, 1), -1),
             ("non-finite X", (nan_x, nr, tf, ps, npd, 16, 1), -1),
             ("has_constant with X[:,0] != 1", (not_one, nr, tf, ps, npd, 16, 1), -1)]
    one = np.zeros(1, np.int32)
    for what, (Xb, a, b, c_, d, p, hc), code in plans:
        if what == "n_cal = 65,536":       # refused before any per-calendar array is read
            rc = eng._lib.mmf_plan_calendars(eng._h, Xb.ctypes.data, 65536, *(one.ctypes.data,) * 4, p, hc)
        else:
            rc = _raw_plan(eng, Xb, a, b, c_, d, p, hc)
        assert rc == code, (what, rc, mmf._native.load().mmf_last_error())
        after = _ragged(eng, cals, yd, rows, plan=False)
        _per_cal_equal(after, before, cals, rows, f"after the refused plan: {what}")
    eng.close()


# =====================================================================================================================
# G. exactness and controls
# =====================================================================================================================
@pytest.mark.parametrize("mode", ["future", "holdout"])
def test_ragged_forecasts_scale_exactly(mode):
    """each calendar's rows in 6 interleaved copies (2^k for k in SCALES, then negated): the copies' forecasts are 2^k
    (or -1) times the k = 0 copy's, bit for bit, through one ragged launch"""
    base = [_d_cal(c, n, mode, t=t) for c, (t, n) in enumerate(((150, 16), (400, 9), (1153, 24), (33, 8)))]
    yb, rb = _batch(base, seed=90)
    nc = len(SCALES) + 1
    blocks = []
    for ci in range(len(base)):
        b = yb[rb[ci]:rb[ci + 1]]
        blocks.append(np.stack([b * np.float32(2.0 ** k) for k in SCALES] + [-b], axis=1).reshape(-1, yb.shape[1]))
    cals = [Cal(c.design, c.t_fit, c.ps, c.npred, c.n * nc, c.key) for c in base]
    y = np.concatenate(blocks)
    rows = np.concatenate([[0], np.cumsum([c.n for c in cals])]).astype(np.int64)
    eng = mmf.ForecastEngine()
    res = _ragged(eng, cals, y, rows)
    pred, status = res["pred"].cpu().numpy(), res["status"].cpu().numpy()
    for ci, c in enumerate(cals):
        r0, r1 = int(rows[ci]), int(rows[ci + 1])
        _assert_equivariant(pred[r0:r1, :c.npred], status[r0:r1], nc, (mode, ci))
    eng.close()


@pytest.mark.parametrize("mode", ["future", "holdout"])
def test_assume_finite_is_bit_equal_on_finite_data(mode):
    """gap-free rows (NaN only past each row's t_fit, which no tensor map reads): assume_finite=True skips the general
    passes -- 1 launch in future mode, 2 (fit + predict) in holdout -- and changes no bit"""
    cals = [_d_cal(c, n, mode, t=t) for c, (t, n) in enumerate(((150, 130), (1153, 1), (33, 200), (2785, 129)))]
    y, rows = _batch(cals, seed=95, kinds=("clean",))
    plain, finite = mmf.ForecastEngine(), mmf.ForecastEngine(assume_finite=True)
    a = _ragged(plain, cals, y, rows)
    b = _ragged(finite, cals, y, rows)
    assert _same_bits(a["pred"], b["pred"]) and _same_bits(a["status"], b["status"]), mode
    assert b["stats"].kernel_launches == (1 if mode == "future" else 2), b["stats"].kernel_launches
    assert a["stats"].n_pending == 0 and (a["status"] == 0).all()
    plain.close()
    finite.close()


def test_more_than_2_20_rows_bit_equal_to_per_calendar_calls():
    """2^20 + 1,001 series over 4 calendars (one of 2^20 + 1 series, whose single-calendar call runs in two slabs):
    one ragged launch allocates its scratch for every row; bit-equal to the per-calendar calls"""
    import torch
    counts, fits = (500, (1 << 20) + 1, 300, 200), (100, 64, 33, 150)
    cals = [_d_cal(c, n, "future", t=t) for c, (t, n) in enumerate(zip(fits, counts))]
    rows = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    y = np.full((int(rows[-1]), _round4(max(fits))), np.nan, dtype=np.float32)
    for ci, c in enumerate(cals):
        blk = y[rows[ci]:rows[ci + 1]]
        blk[:, :c.t_fit] = _series(c.X(), c.t_fit, c.n, 100 + ci, LEVEL)
        for k, kind in enumerate(KINDS):                  # _plant's mix, a kind per residue class of rows
            blk[(k - ci) % len(KINDS)::len(KINDS), _kind_cols(kind, c.t_fit)] = np.inf if kind == "inf" else np.nan
    eng = mmf.ForecastEngine()
    res = _ragged(eng, cals, y, rows)
    single = mmf.ForecastEngine(kernel="tc")
    for ci, c in enumerate(cals):
        r0, r1 = int(rows[ci]), int(rows[ci + 1])
        single.plan(c.X(), c.t_fit, True)
        r = single.fit_forecast(mmf.device_packed(y[r0:r1, :c.t_fit]), c.ps, c.npred, want_status=True)
        torch.cuda.synchronize()
        assert _same_bits(r["pred"], res["pred"][r0:r1]) and _same_bits(r["status"], res["status"][r0:r1]), ci
    assert res["stats"].n_pending == sum(_expected_pending(y[rows[i]:rows[i + 1]], c.t_fit) for i, c in enumerate(cals))
    single.close()
    eng.close()


def _negctl_case():
    """~10,000 series on 8 daily calendars of 1,000 to 1,095 days, future mode, half of the rows gap-free and the row mix
    in the other half -> per-row error / section-A bound of the rows the oracle does not leave empty"""
    fits = (1000, 1013, 1027, 1040, 1055, 1068, 1081, 1095)
    cals = [_d_cal(200 + c, 1250, "future", t=t) for c, t in enumerate(fits)]
    y, rows = _batch(cals, seed=300, kinds=KINDS + ("clean",) * len(KINDS))
    eng = mmf.ForecastEngine()
    res = _ragged(eng, cals, y, rows)
    pred, status = res["pred"].cpu().numpy(), res["status"].cpu().numpy()
    eng.close()
    ratios = []
    for c, idx in _groups(cals, rows):
        Y, X = y[idx], c.X()
        orc = _oracle(Y, X, c.t_fit)
        want = orc["gamma"] @ orc["A"][c.ps:c.ps + c.npred].T
        live = (orc["status"] != 1) & (_pivot_distance(Y, X, c.t_fit) > PIVOT_BAND)
        assert np.array_equal(status[idx], orc["status"])
        tol = (_row_tol(Y[:, :c.t_fit], forecast_leverage(X, c.t_fit, c.ps, c.npred))
               * _mask_factor(Y, X, c.t_fit, c.ps, c.npred, orc["ratio"]) * _long_scale(c.t_fit))
        ratios.append((np.abs(pred[idx][live, :c.npred] - want[live]).max(axis=1) / tol[live]))
    return np.concatenate(ratios)


_NEGCTL = r"""
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import test_gpu_ragged as T
r = T._negctl_case()
print(json.dumps({{"worst": float(r.max()), "rows_over": int((r > 1.0).sum()), "rows": int(r.size)}}))
"""


def test_negative_control_exceeds_the_ragged_bound():
    """the build without the lo*A_hi tensor-core term (tests/_build/libmmf_negctl.so) must exceed the section-A bound in
    at least 100 rows of a ragged batch on calendars of 1,000 to 1,095 days; the product library stays within it"""
    neg = os.path.join(ROOT, "tests", "_build", "libmmf_negctl.so")
    assert os.path.exists(neg), "negative-control library missing: run __graft_entry__.build()"
    r = _negctl_case()
    _le(float(r.max()), 1.0, "product, ragged batch on 1,000-1,095-day calendars: error / bound")
    env = dict(os.environ, MMF_LIB=neg)
    p = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    got = json.loads(p.stdout.strip().splitlines()[-1])
    record_err("test_negative_control_exceeds_the_ragged_bound", got["worst"], 1.0,
               what="negctl, ragged batch: error / bound (must exceed 1 in >= 100 rows)", rows_over=got["rows_over"])
    assert got["rows_over"] >= 100, ("the ragged bound does not detect a missing lo*A_hi term", got)


# =====================================================================================================================
# H. the DataFrame boundary, each group within its own bound
# =====================================================================================================================
def _frame(freq, n_groups, t_range, seed):
    """groups with different first dates and lengths on a daily or weekly grid, ~4 % of the dates dropped (not the
    first and the last)"""
    import pandas as pd
    rng = np.random.default_rng(seed)
    step = O.FREQ_DAYS[freq]
    frames = []
    for g in range(n_groups):
        t = int(rng.integers(*t_range))
        start = np.datetime64("2019-10-07") + np.timedelta64(step * int(rng.integers(0, 30)), "D")
        days = start + np.arange(t) * np.timedelta64(step, "D")
        vals = np.round(1000 + 3 * np.arange(t) + rng.normal(0, 20, t)).astype(np.float32)
        keep = rng.random(t) > 0.04
        keep[0] = keep[-1] = True
        frames.append(pd.DataFrame({"Product": f"p{g % 5}", "SKU": f"s{g:03d}",
                                    "Date": days[keep].astype("datetime64[ns]"), "Demand": vals[keep]}))
    df = pd.concat(frames, ignore_index=True).sample(frac=1.0, random_state=seed)
    df["Date"] = df["Date"].dt.date
    return df


def _frame_ratio(df, got, want, freq, horizon, mode, design, keys=("Product", "SKU")):
    """worst |got - want| of Demand_Fitted / (tolerance(group, max(1, leverage of its calendar)) x mask factor) over the
    groups, `want` = O.fanout_apply(build_tune_and_score_model) (both frames: groups in key order, dates ascending);
    NaN exactly where the UDF's is.  The group's grid (for its tolerance) is rebuilt as the UDF builds it."""
    gf, wf = got["Demand_Fitted"].to_numpy(), want["Demand_Fitted"].to_numpy()
    assert len(gf) == len(wf) and np.array_equal(np.isnan(gf), np.isnan(wf))
    step, pos, worst = O.FREQ_DAYS[freq], 0, 0.0
    for kv, g in df.groupby(list(keys), sort=True):
        dates = [O.to_date(d) for d in g["Date"]]
        d0 = min(dates)
        T = (max(dates) - d0).days // step + 1
        y = np.full((1, T), np.nan, dtype=np.float32)
        on = np.array([(d - d0).days % step == 0 for d in dates])      # off-grid dates vanish under asfreq
        y[0, [(d - d0).days // step for d, o in zip(dates, on) if o]] = g["Demand"].to_numpy(dtype=np.float32)[on]
        if mode == "holdout":
            t_fit, grid, ps, npred = T - horizon, O.calendar_grid(d0, T, freq), 0, T
        else:
            t_fit, grid, ps, npred = T, O.calendar_grid(d0, T + horizon, freq), T, horizon
        assert tuple(want.iloc[pos][list(keys)]) == tuple(kv), (kv, pos)
        X = O.design_matrix(grid, t_fit, design)
        ratio = O.fit_forecast_packed(y, X, t_fit, ps, 1, return_gamma=True)[3]
        part, ref = gf[pos:pos + npred], wf[pos:pos + npred].astype(np.float64)
        pos += npred
        if np.isnan(ref).all():
            continue
        tol = (_row_tol(y[:, :t_fit], forecast_leverage(X, t_fit, ps, npred))
               * _mask_factor(y, X, t_fit, ps, npred, ratio))[0]
        worst = max(worst, float(np.abs(part - ref).max() / tol))
    assert pos == len(gf)
    return worst


@pytest.mark.parametrize("mode", ["future", "holdout"])
@pytest.mark.parametrize("design", ["trend_season_exog", "exog_only"])
@pytest.mark.parametrize("freq", ["W-MON", "D"])
def test_forecast_groups_on_many_calendars_within_each_groups_bound(freq, design, mode):
    """forecast_groups (pack="host" and "device") on frames whose groups start and end on different dates: one ragged
    launch; every group within tolerance x max(1, leverage) x mask factor of the per-group oracle, and the frame
    equal to O.fanout_apply(build_tune_and_score_model) in keys, dates and Demand"""
    horizon = (8 if mode == "future" else 40) if freq == "W-MON" else 28
    df = _frame(freq, 48, (80, 140) if freq == "W-MON" else (90, 400), seed=sum(map(ord, freq + design + mode)))
    kw = dict(freq=freq, horizon=horizon, mode=mode, design=design)
    want = O.fanout_apply(df, lambda p: O.build_tune_and_score_model(p, **kw), ("Product", "SKU"))
    for pack in ("host", "device"):
        got = mmf.forecast_groups(df, pack=pack, **kw)
        assert len(got) == len(want)
        assert (got["SKU"].to_numpy() == want["SKU"].to_numpy()).all()
        assert (got["Date"].dt.date.to_numpy() == want["Date"].to_numpy()).all()
        assert np.array_equal(got["Demand"].to_numpy(), want["Demand"].to_numpy(), equal_nan=True)
        _le(_frame_ratio(df, got, want, freq, horizon, mode, design), 1.0, f"{freq} {design} {mode} pack={pack}")
