"""GPU (-m gpu): the state a context carries from one call to the next -- the ping-pong counter sets and the capture set
(with the tile-claim word of fit_tc), the gap-record scratch, the gamma / c hand-off, the status and backtest scratch,
the ARIMA family's z' scratch, running best, q = 0 score scratch and per-(slab, d) pending counts, and the plain,
ARIMA, ragged and backtest plans that stay in force together -- against a fresh context.

The reference of every call is the same call, with the same arguments and data, on a FRESH engine, compared bit for
bit: pred, status and every extra output (beta; se / sigma / dof; phi / theta / order / ma_order / sigma; choice /
choice_p / d / q, mse, cand_mse; backtest metrics / counts), and stats.n_pending where stats are asked for.  Every
output is pre-filled with a sentinel (the NaN payload 0x7fc0dead, status -7), so a row that no kernel wrote shows.  The
fresh references are anchored once: the plain and ragged kinds against the float64 oracle with the bounds of
test_gpu_ragged._verify, every selection against its winner's single call (with q >= 1 winners where q is searched),
every standard error within 4 ulp of arima_se_oracle on the GPU's own parameters; the other kinds are held to their
oracles by their own modules.

1. Call kinds (KINDS below): one engine, plain, ARIMA (same X) and backtest plans planned once.  A ragged plan is
   planned when a ragged kind of the other mode (future / holdout) than the one in force comes up.  Every batch plants
   the row mix of test_gpu_abi_contract (gaps, leading gaps, mostly missing, empty rows), so records and pending counts
   are never zero; the ARIMA batches carry MA(1) errors on every third row.  The CSS kinds (ARIMA(1, 1, 1), and
   ARIMA(8, 2, 4) with m = 32 and max_iter = 64 with phi / theta / ma_order NULL) keep the HR estimate in the
   context's per-slab scratch between the HR kernels and the LM kernel.
2. Sequences on one stream: every ordered pair, the ping-pong triples, (capture, eager call, replay) with the eager call
   plain or ARIMA, and a seeded sequence of ~100 calls with two multi-slab calls (2^20 + 1,001 rows, one of them
   ARIMA(2, 1, 0)).
3. Tile counts 1, grid - 1, grid, grid + 1, 4 grid + 1 and a 128 k +- 1 row tail (grid = the SM count) for every
   fit_tc instantiation (<8, 1>, tc_variant = 2, standard errors, backtest, ragged, the ARIMA hand-off), with 1, 7, 8,
   9 rows for the ARIMA warp kernels and 64 grid +- 1 for the standard-error pass: stats.n_pending equals the count the
   masks predict (a tile fit twice counts twice), and reversing the 128-row tiles of y reverses them in the outputs,
   bit for bit.
4. Streams: a plain or ARIMA call on stream B between two calls on a sleeping stream A (mmf_set_stream orders the
   switch), the seeded sequence spread over two streams without host syncs, and two engines driven from two threads."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

import mmf
from mmf import _native as N
from oracle import mmf_oracle as O
from test_gpu_abi_contract import KINDS as ROW_KINDS, _expected_pending, _kind_cols, _plant, _round4
from test_gpu_ar_select import _fixed_runs, _gather, _scores as _ar_scores
from test_gpu_arima_se import ULP as SE_ULP, _oracle as _se_oracle, _ulp_err
from test_gpu_arma_select import _Singles, _check_against_single_calls, _ms
from test_gpu_ragged import Cal, _batch, _cal, _daily, _plan, _verify

pytestmark = pytest.mark.gpu

SENT_F = 0x7FC0DEAD                 # NaN payload of every pre-filled float output
SENT_I = -7                         # pre-filled status / count / order / choice
START = "2019-01-01"
T_FIT, H = 400, 28
N_ROWS = T_FIT + H
T_BT, K_BT = 420, 4                 # backtest window and origins
N_HOLD = H
CHUNK = 256                         # host-buffer path: series per pipelined chunk
BIG = (1 << 20) + 1001              # more than one slab
RAGGED_CALS = (("2019-03-05", 333), ("2018-07-09", 365), ("2020-02-01", 150))


# ---- outputs ---------------------------------------------------------------------------------------------------------
def _f(rows, cols, pitch=None):
    """[rows, cols] float32 view (row pitch `pitch`, default cols rounded up to 4) of a sentinel-filled buffer"""
    pitch = pitch or _round4(cols)
    return torch.full((rows, pitch), SENT_F, dtype=torch.int32, device="cuda").view(torch.float32)[:, :cols]


def _f1(n):
    return torch.full((n,), SENT_F, dtype=torch.int32, device="cuda").view(torch.float32)


def _i(*shape):
    return torch.full(shape, SENT_I, dtype=torch.int32, device="cuda")


def _bits(t):
    if isinstance(t, np.ndarray):
        return t.view(np.int32) if t.dtype == np.float32 else t
    return (t.view(torch.int32) if t.dtype == torch.float32 else t).cpu().numpy()


def _stats(st):
    return C.byref(st) if st is not None else None


def _diff(got, want, what):
    """assert bit equality of every output; the message counts the rows that differ and the rows still holding the
    sentinel (never written)"""
    assert got.keys() == want.keys(), (what, sorted(got), sorted(want))
    for k in want:
        g, w = got[k], want[k]
        if isinstance(w, (int, np.integer)):
            assert g == w, (what, k, g, w)
            continue
        if np.array_equal(g, w):
            continue
        g2, w2 = g.reshape(g.shape[0], -1), w.reshape(w.shape[0], -1)
        if k in ("metrics", "count", "status_bt", "pred_bt"):         # [K, n, ...]: rows are the second axis
            g2 = np.moveaxis(g, 1, 0).reshape(g.shape[1], -1)
            w2 = np.moveaxis(w, 1, 0).reshape(w.shape[1], -1)
        bad = (g2 != w2).any(axis=1)
        is_sent = (g2 == SENT_F) | (g2 == SENT_I)
        sent = is_sent.any(axis=1) & bad
        raise AssertionError(f"{what}: {k}: {int(bad.sum())} of {len(bad)} rows differ from the fresh context, "
                             f"{int(sent.sum())} of them hold the sentinel (never written; {int(is_sent.sum())} "
                             f"sentinel elements in all), first rows {np.flatnonzero(bad)[:8].tolist()}")


# ---- inputs ----------------------------------------------------------------------------------------------------------
def _plain_cal(n, ps=T_FIT, npred=H):
    return Cal(_daily(START, T_FIT), T_FIT, ps, npred, n, ("plain", START))


def _plain_X():
    return _plain_cal(1).X(N_ROWS)


def _ragged_cals(ns, mode):
    return [_cal(_daily(s, t), t, n, mode, ("ragged", s)) for (s, t), n in zip(RAGGED_CALS, ns)]


def _synth(n, t, seed, plant_t):
    y, _ = mmf.synth.daily_store_item_demand(n, t, seed=seed)
    return _plant(y, plant_t, shift=seed)


def _plant_torch(yd, t_fit):
    for j, kind in enumerate(ROW_KINDS):
        cols = torch.from_numpy(_kind_cols(kind, t_fit)).cuda()
        if len(cols):
            yd[j::len(ROW_KINDS), cols] = float("inf") if kind == "inf" else float("nan")
    return yd


_INPUTS = {}


def _input(name):
    """the seeded input of a call kind (built once)"""
    if name in _INPUTS:
        return _INPUTS[name]
    n, seed = KIND_ROWS[name]
    if name in ("future", "future_b", "holdout", "replay", "aba_1", "aba_2", "aba_3"):
        y, _ = _batch([_plain_cal(n)], seed)
        inp = dict(y=y, yd=mmf.device_packed(y))
    elif name in ("big", "big_arima"):
        yd, _ = mmf.synth.daily_store_item_demand_torch(n, T_FIT, seed=seed, ld=_round4(T_FIT))
        inp = dict(yd=_plant_torch(yd, T_FIT))
    elif name == "arima_se":
        inp = _arima_se_input(n, seed)
    elif name in ARIMA_RAW:
        y = _arima_y(n, seed)
        inp = dict(y=y, yd=mmf.device_packed(y))
    elif name == "warp":                                   # ld_y % 4 != 0: the tensor maps cannot take it
        y, _ = _batch([_plain_cal(n)], seed)
        wide = torch.full((n, T_FIT + 1), float("nan"), device="cuda")
        wide[:, :T_FIT] = torch.from_numpy(y[:, :T_FIT]).cuda()
        inp = dict(y=y, yd=wide[:, :T_FIT])
    elif name in ("se_future", "se_holdout", "ar2", "bcast"):
        y, _ = _batch([_plain_cal(n)], seed)
        inp = dict(yd=mmf.device_packed(y))
    elif name in ("select", "refused"):                    # the held-out rows follow the fit rows
        inp = dict(yd=mmf.device_packed(_synth(n, N_ROWS, seed, T_FIT)))
    elif name == "backtest":
        inp = dict(yd=mmf.device_packed(_synth(n, T_BT, seed, T_BT)))
    elif name in ("ragged_future", "ragged_holdout"):
        cals = _ragged_cals(n, name.split("_")[1])
        y, rows = _batch(cals, seed)
        inp = dict(y=y, rows=rows, cals=cals, yd=torch.from_numpy(y).cuda())
    elif name == "host":                                   # integer-valued: narrowed to uint16 on the host
        y = np.rint(_synth(n, T_FIT, seed, T_FIT))
        y[~np.isfinite(y)] = np.nan
        inp = dict(y=np.ascontiguousarray(y, dtype=np.float32))
    elif name == "int16":
        y = _synth(n, T_FIT, seed, T_FIT)
        yi = np.where(np.isfinite(y), np.clip(np.rint(y), 0, 32000), -32768).astype(np.int16)
        inp = dict(yd=torch.from_numpy(yi).cuda())
    else:
        raise KeyError(name)
    _INPUTS[name] = inp
    return inp


# ---- engines ---------------------------------------------------------------------------------------------------------
class Ctx:
    """one engine with the plain and backtest plans in force; the ragged plan of the mode last used"""

    def __init__(self, **kw):
        self.eng = mmf.ForecastEngine(host_narrow="on", chunk_series=CHUNK, **kw)
        self.eng.plan(_plain_X(), T_FIT, True)
        self.eng.plan_arima(_plain_X(), T_FIT, 2)          # the same X: selections listing d = 0 and d >= 1 may run
        self.eng.plan_backtest(START, T_BT, "D", H, K_BT, step=H)
        self.ragged = None

    def close(self):
        self.eng.close()


def _stream(eng):
    eng.set_stream(torch.cuda.current_stream().cuda_stream)


# ---- call kinds: (ctx, input, stats) -> {output name: tensor / array / int} ------------------------------------------
def _k_plain(ps, npred, beta=False):
    def run(ctx, inp, stats):
        n = inp["yd"].shape[0]
        out, status = _f(n, npred), _i(n)
        b = _f(n, N.MMF_P) if beta else None
        res = ctx.eng.fit_forecast(inp["yd"], ps, npred, out=out, status=status, beta=b, want_stats=stats)
        r = {"pred": out, "status": status}
        if beta:
            r["beta"] = b
        if stats:
            r["n_pending"] = res["stats"].n_pending
        return r
    return run


def _se_raw(eng, yd, ps, npred, stats):
    n = yd.shape[0]
    out, se, sigma, dof, status = _f(n, npred), _f(n, npred), _f1(n), _i(n), _i(n)
    st = N.MmfStats() if stats else None
    _stream(eng)
    N.check(eng._lib.mmf_fit_forecast_se_f32(eng._h, yd.data_ptr(), n, yd.stride(0), ps, npred, out.data_ptr(),
                                             out.stride(0), se.data_ptr(), se.stride(0), sigma.data_ptr(),
                                             dof.data_ptr(), status.data_ptr(), _stats(st)))
    r = {"pred": out, "se": se, "sigma": sigma, "dof": dof, "status": status}
    if stats:
        r["n_pending"] = st.n_pending
    return r


def _k_se(ps, npred):
    return lambda ctx, inp, stats: _se_raw(ctx.eng, inp["yd"], ps, npred, stats)


def _k_ar(ctx, inp, stats):
    yd = inp["yd"]
    n = yd.shape[0]
    out, phi, order, sigma, status = _f(n, H), _f(n, N.AR_MAX), _i(n), _f1(n), _i(n)
    st = N.MmfStats() if stats else None
    _stream(ctx.eng)
    N.check(ctx.eng._lib.mmf_fit_forecast_ar_f32(ctx.eng._h, yd.data_ptr(), n, yd.stride(0), 2, T_FIT, H,
                                                 out.data_ptr(), out.stride(0), phi.data_ptr(), order.data_ptr(),
                                                 sigma.data_ptr(), status.data_ptr(), _stats(st)))
    r = {"pred": out, "phi": phi, "order": order, "sigma": sigma, "status": status}
    if stats:
        r["n_pending"] = st.n_pending
    return r


CANDS = (1, 3, 9, 13, 16)


def _select(ctx, yd, out):
    n = yd.shape[0]
    choice, mse, status = _i(n), _f1(n), _i(n)
    cand = (C.c_int32 * len(CANDS))(*CANDS)
    _stream(ctx.eng)
    rc = ctx.eng._lib.mmf_fit_select_forecast_f32(ctx.eng._h, yd.data_ptr(), n, yd.stride(0), N_HOLD, cand, len(CANDS),
                                                  0, N_ROWS, out.data_ptr(), out.stride(0), choice.data_ptr(),
                                                  mse.data_ptr(), status.data_ptr())
    return rc, {"pred": out, "choice": choice, "mse": mse, "status": status}


def _k_select(ctx, inp, stats):
    rc, r = _select(ctx, inp["yd"], _f(inp["yd"].shape[0], N_ROWS))
    N.check(rc)
    return r


def _k_refused(ctx, inp, stats):
    """selection into an out whose row pitch is not a multiple of 4: refused before anything is enqueued"""
    rc, r = _select(ctx, inp["yd"], _f(inp["yd"].shape[0], N_ROWS, pitch=N_ROWS + 1))
    r["rc"] = int(rc)
    return r


def _k_bcast(ctx, inp, stats):
    yd = inp["yd"]
    n = yd.shape[0]
    reps = [_f(n, H) for _ in range(3)]
    status = _i(n)
    ctx.eng.fit_forecast_bcast(yd, T_FIT, H, [r.data_ptr() for r in reps], reps[0].stride(0), status=status)
    return {"pred": reps[0], "replica1": reps[1], "replica2": reps[2], "status": status}


def _k_ragged(mode):
    def run(ctx, inp, stats):
        cals = inp["cals"]
        if ctx.ragged != mode:
            _plan(ctx.eng, cals)
            ctx.ragged = mode
        n, width = inp["yd"].shape[0], max(c.npred for c in cals)
        out, status = _f(n, width), _i(n)
        res = ctx.eng.fit_forecast_ragged(inp["yd"], inp["rows"], out=out, status=status, want_stats=stats)
        r = {"pred": out, "status": status}
        if stats:
            r["n_pending"] = res["stats"].n_pending
        return r
    return run


def _backtest_raw(eng, yd, stats, k=K_BT):
    n = yd.shape[0]
    pred = torch.full((k, n, _round4(H)), SENT_F, dtype=torch.int32, device="cuda").view(torch.float32)[:, :, :H]
    metrics = torch.full((k, n, N.BT_NMETRIC), SENT_F, dtype=torch.int32, device="cuda").view(torch.float32)
    count, status = _i(k, n), _i(k, n)
    st = N.MmfStats() if stats else None
    _stream(eng)
    N.check(eng._lib.mmf_backtest_f32(eng._h, yd.data_ptr(), n, yd.stride(0), pred.data_ptr(), pred.stride(1),
                                      metrics.data_ptr(), count.data_ptr(), status.data_ptr(), _stats(st)))
    r = {"pred_bt": pred, "metrics": metrics, "count": count, "status_bt": status}
    if stats:
        r["n_pending"] = st.n_pending
    return r


def _k_backtest(ctx, inp, stats):
    return _backtest_raw(ctx.eng, inp["yd"], stats)


def _k_host(ctx, inp, stats):
    y = inp["y"]
    out = np.full((len(y), H), SENT_F, dtype=np.int32).view(np.float32)
    status = np.full(len(y), SENT_I, dtype=np.int32)
    res = ctx.eng.fit_forecast(y, T_FIT, H, out=out, status=status, want_stats=stats)
    r = {"pred": out.copy(), "status": status.copy()}
    if stats:
        r["n_pending"] = res["stats"].n_pending
    return r


def _k_replay(ctx, inp, stats):
    """capture the plain future call, overwrite its outputs with the sentinel again, replay it"""
    g, out, status = _capture(ctx, inp)
    g.replay()
    g.close()
    return {"pred": out, "status": status}


def _capture(ctx, inp):
    n = inp["yd"].shape[0]
    out, status = _f(n, H), _i(n)
    g, _ = ctx.eng.capture(inp["yd"], T_FIT, H, out=out, status=status)
    out.view(torch.int32).fill_(SENT_F)
    status.fill_(SENT_I)
    return g, out, status


# ---- ARIMA-family call kinds: (eng, input, stats) -> (return code, {output name: tensor / int}) ----------------------
# Every output, the [n][n_diffs][n_mas][n_orders] score table included, is a sentinel-filled buffer of its own; the
# standard errors of want_se are mmf_arima_se_f32 on the call's outputs, enqueued behind it as ForecastEngine does.
AR_ORDERS = (0, 1, 2, 3, 4)
REF = ((0, 1, 2, 3, 4), (0, 1, 2), (0, 1, 2, 3, 4))        # 215 entries, 14,620 B: no attribute set
GRID_52K = (tuple(range(9)), (0, 1, 2), (0, 1, 2, 3))      # 769 entries, 52,292 B
GRID_MAX = (tuple(range(1, 9)), (0, 1, 2), (0, 1, 2, 3, 4))  # 32 pairs, 1,099 entries, 74,732 B: the largest accepted
MID = (T_FIT // 3, T_FIT // 2 + 20)                         # a window inside the design


def _fc(*shape):
    """contiguous sentinel-filled float32 buffer (the tables the ABI takes without a row pitch)"""
    return torch.full(shape, SENT_F, dtype=torch.int32, device="cuda").view(torch.float32)


def _p(t):
    return None if t is None else t.data_ptr()


def _arr(v):
    return (C.c_int32 * max(len(v), 1))(*v)


def _model_outs(n, npred, ma):
    r = {"pred": _f(n, npred), "phi": _f(n, N.AR_MAX), "order": _i(n), "sigma": _f1(n), "status": _i(n)}
    if ma:
        r["theta"], r["ma_order"] = _f(n, N.MA_MAX), _i(n)
    return r


def _done(rc, r, st):
    if rc == 0 and st is not None:
        r["n_pending"] = st.n_pending
    return rc, r


def _se_into(eng, yd, r, t_fit, d, diffs, ps, npred):
    n = yd.shape[0]
    r["se"] = _f(n, npred)
    return eng._lib.mmf_arima_se_f32(eng._h, yd.data_ptr(), n, yd.stride(0), t_fit, d, _p(diffs), _p(r["phi"]),
                                     _p(r["order"]), _p(r.get("theta")), _p(r.get("ma_order")), _p(r["sigma"]), ps,
                                     npred, _p(r["se"]), r["se"].stride(0), None)


def _r_ar_select(eng, yd, stats, orders=AR_ORDERS, ps=0, npred=N_ROWS):
    n = yd.shape[0]
    r = _model_outs(n, npred, False)
    r.update(choice=_i(n), mse=_f1(n), cand_mse=_fc(n, len(orders)))
    st = N.MmfStats() if stats else None
    _stream(eng)
    rc = eng._lib.mmf_fit_select_ar_f32(eng._h, yd.data_ptr(), n, yd.stride(0), N_HOLD, _arr(orders), len(orders), ps,
                                        npred, _p(r["pred"]), r["pred"].stride(0),
                                        *[_p(r[k]) for k in ("choice", "mse", "cand_mse", "phi", "order", "sigma",
                                                             "status")], _stats(st))
    return _done(rc, r, st)


def _r_arima(eng, yd, stats, p, d, ps, npred):
    n = yd.shape[0]
    r = _model_outs(n, npred, False)
    st = N.MmfStats() if stats else None
    _stream(eng)
    rc = eng._lib.mmf_fit_forecast_arima_f32(eng._h, yd.data_ptr(), n, yd.stride(0), p, d, ps, npred, _p(r["pred"]),
                                             r["pred"].stride(0), _p(r["phi"]), _p(r["order"]), _p(r["sigma"]),
                                             _p(r["status"]), _stats(st))
    return _done(rc, r, st)


def _r_arma(eng, yd, stats, p, q, d, ps, npred, long_order=0, se=False, t_fit=T_FIT):
    n = yd.shape[0]
    r = _model_outs(n, npred, True)
    st = N.MmfStats() if stats else None
    _stream(eng)
    rc = eng._lib.mmf_fit_forecast_arma_f32(eng._h, yd.data_ptr(), n, yd.stride(0), p, d, q, long_order, ps, npred,
                                            _p(r["pred"]), r["pred"].stride(0),
                                            *[_p(r[k]) for k in ("phi", "theta", "order", "ma_order", "sigma",
                                                                 "status")], _stats(st))
    if rc == 0 and se:
        rc = _se_into(eng, yd, r, t_fit, d, None, ps, npred)
    return _done(rc, r, st)


def _r_css(eng, yd, stats, p, q, d, ps, npred, long_order=0, max_iter=0):
    """mmf_fit_forecast_arma_css_f32: the HR call, then LM from its (phi, theta), which the context keeps in per-slab
    scratch for the outputs a caller passes as NULL (here none: every output is a sentinel-filled buffer)"""
    n = yd.shape[0]
    r = _model_outs(n, npred, True)
    r.update(css_start=_f1(n), css=_f1(n), css_stop=_i(n), iters=_i(n))
    st = N.MmfStats() if stats else None
    _stream(eng)
    rc = eng._lib.mmf_fit_forecast_arma_css_f32(
        eng._h, yd.data_ptr(), n, yd.stride(0), p, d, q, long_order, max_iter, ps, npred, _p(r["pred"]),
        r["pred"].stride(0), *[_p(r[k]) for k in ("phi", "theta", "order", "ma_order", "sigma", "status", "css_start",
                                                  "css", "css_stop", "iters")], _stats(st))
    return _done(rc, r, st)


def _r_css_scratch(eng, yd, stats, p, q, d, ps, npred, long_order=0, max_iter=0):
    """the same call with phi, theta and ma_order NULL: the HR estimate and the gate then live in the context's
    scratch (52 B per row per slab) between the HR kernels and arma_css_kernel"""
    n = yd.shape[0]
    r = {"pred": _f(n, npred), "order": _i(n), "sigma": _f1(n), "status": _i(n), "css_start": _f1(n), "css": _f1(n),
         "css_stop": _i(n), "iters": _i(n)}
    st = N.MmfStats() if stats else None
    _stream(eng)
    rc = eng._lib.mmf_fit_forecast_arma_css_f32(
        eng._h, yd.data_ptr(), n, yd.stride(0), p, d, q, long_order, max_iter, ps, npred, _p(r["pred"]),
        r["pred"].stride(0), None, None, _p(r["order"]), None, *[_p(r[k]) for k in ("sigma", "status", "css_start",
                                                                                    "css", "css_stop", "iters")],
        _stats(st))
    return _done(rc, r, st)


def _r_select(eng, yd, stats, grid, ps, npred, se=False, t_fit=T_FIT):
    """mmf_fit_select_arma_f32 on grid = (orders, diffs, mas); mas = None: mmf_fit_select_arima_f32"""
    orders, diffs, mas = grid
    n = yd.shape[0]
    r = _model_outs(n, npred, mas is not None)
    r.update(choice_p=_i(n), choice_d=_i(n), mse=_f1(n))
    st = N.MmfStats() if stats else None
    _stream(eng)
    if mas is None:
        r["cand_mse"] = _fc(n, len(diffs), len(orders))
        rc = eng._lib.mmf_fit_select_arima_f32(
            eng._h, yd.data_ptr(), n, yd.stride(0), N_HOLD, _arr(orders), len(orders), _arr(diffs), len(diffs), ps,
            npred, _p(r["pred"]), r["pred"].stride(0),
            *[_p(r[k]) for k in ("choice_p", "choice_d", "mse", "cand_mse", "phi", "order", "sigma", "status")],
            _stats(st))
    else:
        r["choice_q"], r["cand_mse"] = _i(n), _fc(n, len(diffs), len(mas), len(orders))
        rc = eng._lib.mmf_fit_select_arma_f32(
            eng._h, yd.data_ptr(), n, yd.stride(0), N_HOLD, _arr(orders), len(orders), _arr(diffs), len(diffs),
            _arr(mas), len(mas), 0, ps, npred, _p(r["pred"]), r["pred"].stride(0),
            *[_p(r[k]) for k in ("choice_p", "choice_d", "choice_q", "mse", "cand_mse", "phi", "theta", "order",
                                 "ma_order", "sigma", "status")], _stats(st))
    if rc == 0 and se:
        rc = _se_into(eng, yd, r, t_fit, 0, r["choice_d"], ps, npred)
    return _done(rc, r, st)


def _r_arima_se(eng, inp, ps=0, npred=N_ROWS):
    """mmf_arima_se_f32 on the outputs of an earlier selection (per-series d = its choice_d, -1 where none won)"""
    r = {k: inp[k] for k in ("phi", "order", "theta", "ma_order", "sigma")}
    _stream(eng)
    rc = _se_into(eng, inp["yd"], r, T_FIT, 0, inp["choice_d"], ps, npred)
    return rc, {"se": r["se"]}


# name: (model call, window, want_se) of every ARIMA-family kind; the window of a selection is (pred_start, n_pred)
ARIMA_RAW = {
    "ar_select": lambda e, inp, s: _r_ar_select(e, inp["yd"], s),
    "arima21": lambda e, inp, s: _r_arima(e, inp["yd"], s, 2, 1, T_FIT, H),
    "arima12_mid": lambda e, inp, s: _r_arima(e, inp["yd"], s, 1, 2, *MID),
    "select_arima": lambda e, inp, s: _r_select(e, inp["yd"], s, (REF[0], REF[1], None), T_FIT, H),
    "arma111_se": lambda e, inp, s: _r_arma(e, inp["yd"], s, 1, 1, 1, T_FIT, H, se=True),
    "arma824": lambda e, inp, s: _r_arma(e, inp["yd"], s, 8, 4, 2, T_FIT, H, long_order=32, se=True),
    "select_arma_ref": lambda e, inp, s: _r_select(e, inp["yd"], s, REF, 0, N_ROWS, se=True),
    "select_arma_52k": lambda e, inp, s: _r_select(e, inp["yd"], s, GRID_52K, *MID),
    "select_arma_max": lambda e, inp, s: _r_select(e, inp["yd"], s, GRID_MAX, T_FIT, H),
    "arima_se": lambda e, inp, s: _r_arima_se(e, inp),
    "refused_arima": lambda e, inp, s: _r_select(e, inp["yd"], s, ((1,), (0, 1), (1, 2)), T_FIT, H),
    "css111": lambda e, inp, s: _r_css(e, inp["yd"], s, 1, 1, 1, T_FIT, H),
    "css824": lambda e, inp, s: _r_css_scratch(e, inp["yd"], s, 8, 4, 2, T_FIT, H, long_order=32, max_iter=64),
    "big_arima": lambda e, inp, s: _r_arima(e, inp["yd"], s, 2, 1, T_FIT, H),
    "aba_arima": lambda e, inp, s: _r_arima(e, inp["yd"], s, 2, 1, T_FIT, H),
}


def _k_arima(name):
    def run(ctx, inp, stats):
        rc, r = ARIMA_RAW[name](ctx.eng, inp, stats)
        if name == "refused_arima":                        # mas[0] != 0: refused before anything is enqueued
            r["rc"] = int(rc)
        else:
            N.check(rc)
        return r
    return run


def _arima_y(n, seed):
    """levels on N_ROWS columns: the row mix over the fit rows, and every third row an MA(1) theta = 0.6 error on a
    regression on the planned design (test_gpu_arma_select._ma_case), so that q >= 1 wins somewhere"""
    y = _synth(n, N_ROWS, seed, T_FIT)
    X = _plain_X()
    rng = np.random.default_rng(seed + 200)
    eps = rng.normal(0, 4, (n, N_ROWS + 1))
    base = 400.0 + rng.normal(0, 20, (n, X.shape[1])) @ X[:N_ROWS].T
    for i in range(0, n, 3):
        v = (base[i] + eps[i, 1:] + 0.6 * eps[i, :-1]).astype(np.float32)
        y[i] = np.where(np.isfinite(y[i]), v, y[i])
    return np.ascontiguousarray(y, dtype=np.float32)


def _arima_se_input(n, seed):
    """y and the outputs of a fresh-engine (p, d, q) selection on the reference grid: the parameters mmf_arima_se_f32
    takes"""
    y = _arima_y(n, seed)
    yd = mmf.device_packed(y)
    ctx = Ctx()
    rc, r = _r_select(ctx.eng, yd, False, REF, T_FIT, H)
    N.check(rc)
    torch.cuda.synchronize()
    ctx.close()
    return dict(y=y, yd=yd, **{k: r[k] for k in ("phi", "order", "theta", "ma_order", "sigma", "choice_d")})


# name: (rows, seed); every kind has its own row count (the rows of the ragged kinds are per calendar)
KIND_ROWS = {
    "future": (1000, 11), "holdout": (777, 12), "warp": (515, 13), "se_future": (650, 14), "se_holdout": (611, 15),
    "ar2": (333, 16), "select": (430, 17), "bcast": (301, 18), "ragged_future": ((129, 200, 1), 19),
    "ragged_holdout": ((64, 300, 131), 20), "backtest": (700, 21), "host": (900, 22), "int16": (600, 23),
    "replay": (450, 24), "refused": (256, 25),
    "ar_select": (437, 41), "arima21": (1003, 42), "arima12_mid": (389, 43), "select_arima": (517, 44),
    "arma111_se": (629, 45), "arma824": (333, 46), "select_arma_ref": (301, 47), "select_arma_52k": (285, 48),
    "select_arma_max": (259, 49), "arima_se": (707, 50), "refused_arima": (131, 51), "css111": (587, 53),
    "css824": (313, 54),
    "future_b": (1000, 26), "big": (BIG, 27), "big_arima": (BIG, 52),
    "aba_1": (40000, 31), "aba_2": (40000, 32), "aba_3": (40000, 33), "aba_arima": (40003, 34),
}
RUN = {
    "future": _k_plain(T_FIT, H, beta=True), "holdout": _k_plain(0, N_ROWS), "warp": _k_plain(T_FIT, H),
    "se_future": _k_se(T_FIT, H), "se_holdout": _k_se(0, N_ROWS), "ar2": _k_ar, "select": _k_select,
    "bcast": _k_bcast, "ragged_future": _k_ragged("future"), "ragged_holdout": _k_ragged("holdout"),
    "backtest": _k_backtest, "host": _k_host, "int16": _k_plain(T_FIT, H), "replay": _k_replay,
    "refused": _k_refused,
    "future_b": _k_plain(T_FIT, H), "big": _k_plain(T_FIT, H),
    "aba_1": _k_plain(T_FIT, H), "aba_2": _k_plain(T_FIT, H), "aba_3": _k_plain(T_FIT, H),
    **{name: _k_arima(name) for name in ARIMA_RAW},
}
ARIMA_KINDS = tuple(KIND_ROWS)[15:28]
KINDS = tuple(KIND_ROWS)[:28]                             # the kinds every sequence draws from
HAS_STATS = ("future", "holdout", "warp", "se_future", "se_holdout", "ar2", "ragged_future", "ragged_holdout",
             "backtest", "host", "int16", "future_b", "big", "ar_select", "arima21", "arima12_mid", "select_arima",
             "arma111_se", "arma824", "select_arma_ref", "select_arma_52k", "select_arma_max", "css111", "css824",
             "big_arima", "aba_arima")
SEL_GRIDS = {"ar_select": (AR_ORDERS, (0,), (0,), (0, N_ROWS)), "select_arima": (*REF[:2], (0,), (T_FIT, H)),
             "select_arma_ref": (*REF, (0, N_ROWS)), "select_arma_52k": (*GRID_52K, MID),
             "select_arma_max": (*GRID_MAX, (T_FIT, H))}
FLOAT_KEYS = ("pred", "mse", "cand_mse", "phi", "theta", "sigma", "se", "css_start", "css")


def _call(ctx, name, stats=False):
    return RUN[name](ctx, _input(name), stats and name in HAS_STATS)


def _host(res):
    return {k: (v if isinstance(v, int) else _bits(v)) for k, v in res.items()}


_FRESH = {}


def _fresh(name, stats=False):
    """the call on a fresh engine, with the same arguments and data"""
    key = (name, stats and name in HAS_STATS)
    if key not in _FRESH:
        ctx = Ctx()
        res = _call(ctx, name, stats)
        torch.cuda.synchronize()
        _FRESH[key] = _host(res)
        ctx.close()
    return _FRESH[key]


def _check(name, stats, res, what):
    torch.cuda.synchronize()
    _diff(_host(res), _fresh(name, stats), f"{what}: {name}")


# =====================================================================================================================
# 1. the fresh references against the float64 oracle
# =====================================================================================================================
@pytest.mark.parametrize("name", ["future", "holdout", "warp", "ragged_future", "ragged_holdout"])
def test_fresh_references_match_the_oracle(name):
    res = _fresh(name, stats=True)
    inp = _input(name)
    if name.startswith("ragged"):
        cals, rows, y = inp["cals"], inp["rows"], inp["y"]
    else:
        n = inp["yd"].shape[0]
        ps, npred = (0, N_ROWS) if name == "holdout" else (T_FIT, H)
        cals, rows, y = [_plain_cal(n, ps, npred)], np.array([0, n]), inp["y"]
    out = {"pred": torch.from_numpy(res["pred"].view(np.float32)).cuda(), "status": torch.from_numpy(res["status"]).cuda(),
           "stats": mmf.Stats(0.0, 0.0, len(y), res["n_pending"], 0, 0, 0, "")}
    _verify(cals, y, rows, out, name, kernels=("warp",) if name == "warp" else ("tc", "auto"),
            pending=name != "warp")
    assert res["n_pending"] > 0 or name == "warp"


def test_fresh_refused_call_writes_nothing():
    res = _fresh("refused")
    assert res["rc"] == -3                                   # MMF_E_UNSUPPORTED
    for k in ("pred", "choice", "mse", "status"):
        assert ((res[k] == SENT_F) | (res[k] == SENT_I)).all(), k


def test_fresh_refused_arima_call_writes_nothing():
    res = _fresh("refused_arima")
    assert res["rc"] == -1                                   # MMF_E_INVALID: mas[0] != 0
    for k, v in res.items():
        if k != "rc":
            assert ((v == SENT_F) | (v == SENT_I)).all(), k


def _floats(res):
    """a fresh reference (int32 bit patterns) with its float outputs viewed as float32 again"""
    return {k: (v.view(np.float32) if k in FLOAT_KEYS else v) for k, v in res.items() if k not in ("n_pending", "rc")}


@pytest.mark.parametrize("name", list(SEL_GRIDS))
def test_fresh_selections_equal_their_winners_single_calls(name):
    """the fresh reference of every selection kind is bit-equal to its winner's single call
    (test_gpu_arma_select._check_against_single_calls; the AR-order selection by test_gpu_ar_select's identity), and
    the (p, d, q) selections have q >= 1 winners"""
    orders, diffs, mas, (ps, npred) = SEL_GRIDS[name]
    got = _floats(_fresh(name, stats=True))
    inp = _input(name)
    y, yd = inp["y"], inp["yd"]
    n = len(y)
    ctx = Ctx()
    if name == "ar_select":
        runs = _fixed_runs(ctx.eng, yd, ps, npred)
        ch, st = got["choice"], got["status"]
        assert np.array_equal(st, runs[1]["status"]) and ((ch == -1) == (st == 1)).all(), name
        for k in ("pred", "phi", "order", "sigma", "status"):
            bad = np.flatnonzero((_bits(got[k]) != _bits(_gather(runs, ch, orders, k))).reshape(n, -1).any(axis=1))
            assert bad.size == 0, (name, k, bad[:8], ch[bad[:8]])
        fut = _fixed_runs(ctx.eng, yd, T_FIT, N_HOLD)
        sc = _ar_scores(fut, y, T_FIT, orders)
        cm = got["cand_mse"].astype(np.float64)
        assert np.array_equal(np.isnan(cm), np.isnan(sc)), name
        ok = ~np.isnan(sc)
        assert (np.abs(cm[ok] - sc[ok]) <= 1e-6 * np.abs(sc[ok])).all(), name
    else:
        if name == "select_arima":                          # the (p, d, 0) view of a (p, d, q) selection
            none = got["choice_p"] < 0
            got["choice_q"] = np.where(none, -1, 0).astype(np.int32)
            got["theta"] = np.zeros((n, N.MA_MAX), np.float32)
            got["ma_order"] = np.zeros(n, np.int32)
            got["cand_mse"] = got["cand_mse"][:, :, None, :]
        single = _Singles(ctx.eng, yd, T_FIT)
        _, q_wins = _check_against_single_calls(got, single, y, T_FIT, ps, npred, orders, diffs, mas,
                                                _ms(T_FIT, orders, diffs, mas), name)
        assert q_wins > 0 or mas == (0,), name
    ctx.close()


@pytest.mark.parametrize("name", ["arma111_se", "arma824", "select_arma_ref", "arima_se"])
def test_fresh_standard_errors_match_the_oracle(name):
    """se of the fresh reference within 4 ulp of arima_se_oracle fed the GPU's own parameters"""
    res = _floats(_fresh(name))
    inp = _input(name)
    if name == "arima_se":
        params = {k: inp[k].cpu().numpy() for k in ("phi", "order", "theta", "ma_order", "sigma", "choice_d")}
        want = _se_oracle(params, inp["y"], T_FIT, 0, N_ROWS, 0, params["choice_d"])
    elif name == "select_arma_ref":
        want = _se_oracle(res, inp["y"], T_FIT, 0, N_ROWS, 0, res["choice_d"])
    else:
        want = _se_oracle(res, inp["y"], T_FIT, T_FIT, H, {"arma111_se": 1, "arma824": 2}[name])
    assert _ulp_err(res["se"], want) <= SE_ULP, name
    assert np.isfinite(res["se"]).any(), name


# =====================================================================================================================
# 2. sequences on one stream
# =====================================================================================================================
def test_every_ordered_pair_of_call_kinds():
    """X then Y on one engine, for every ordered pair: Y (and X) equal their fresh-engine calls"""
    for name in KINDS:
        _fresh(name)
    ctx = Ctx()
    for x in KINDS:
        for y in KINDS:
            rx = _call(ctx, x)
            ry = _call(ctx, y)
            _check(x, False, rx, f"pair ({x}, {y}), first")
            _check(y, False, ry, f"pair ({x}, {y}), second")
    ctx.close()


@pytest.mark.parametrize("middle", ["warp", "ragged_future", "backtest", "refused", "select_arma_max", "arima21",
                                    "arima_se", "css824"])
def test_ping_pong_triples(middle):
    """(TC, X, TC): a call that uses the counter sets differently -- the warp kernel (does not zero the next set), a
    ragged or backtest call (memsets its set, toggles nothing), a refused call (enqueues nothing), the fit_tc hand-off
    of an ARIMA call or a selection (one fit per listed d), a standard-error pass (no fit) -- between two tensor-core
    calls; with stats on the last one, so its pending count is checked too"""
    ctx = Ctx()
    for stats in (False, True):
        a = _call(ctx, "future")
        b = _call(ctx, middle, stats)
        c = _call(ctx, "future_b", stats)
        _check("future", False, a, f"triple {middle}")
        _check(middle, stats, b, f"triple {middle}")
        _check("future_b", stats, c, f"triple {middle}")
    ctx.close()


def test_capture_eager_replay():
    """a graph captured, an eager call on the same engine, then the replay: both equal their fresh-engine calls"""
    ctx = Ctx()
    _call(ctx, "future")                                  # scratch for the eager call below, before the graph pins it
    g, out, status = _capture(ctx, _input("replay"))
    e = _call(ctx, "future", stats=True)
    g.replay()
    g.close()
    _check("future", True, e, "eager between capture and replay")
    _check("replay", False, {"pred": out, "status": status}, "replay after an eager call")
    ctx.close()


@pytest.mark.parametrize("middle", ["arima21", "select_arma_max", "arma111_se"])
def test_capture_arima_call_replay(middle):
    """(capture, ARIMA-family eager call, replay) with the ARIMA scratch grown before the capture: the eager call and
    the replay equal their fresh-engine calls"""
    ctx = Ctx()
    _call(ctx, middle)                                    # z', gamma / c, running best: grown before the graph pins them
    g, out, status = _capture(ctx, _input("replay"))
    e = _call(ctx, middle, stats=True)
    g.replay()
    g.close()
    _check(middle, True, e, "ARIMA call between capture and replay")
    _check("replay", False, {"pred": out, "status": status}, "replay after an ARIMA call")
    ctx.close()


@pytest.mark.parametrize("middle", ["arima21", "select_arma_max"])
def test_pinned_context_refuses_an_arima_call_that_must_grow_scratch(middle):
    """a captured graph pins the context's scratch; an ARIMA-family call that needs scratch the context never grew is
    refused with MMF_E_UNSUPPORTED, writes nothing, and the replay is unaffected"""
    ctx = Ctx()
    g, out, status = _capture(ctx, _input("replay"))
    rc, r = ARIMA_RAW[middle](ctx.eng, _input(middle), True)
    with pytest.raises(N.MmfError) as err:
        N.check(rc)
    assert err.value.code == -3, err.value              # MMF_E_UNSUPPORTED
    g.replay()
    g.close()
    torch.cuda.synchronize()
    for k, v in _host(r).items():
        assert ((v == SENT_F) | (v == SENT_I)).all(), (middle, k)
    _check("replay", False, {"pred": out, "status": status}, "replay after a refused ARIMA call")
    _check(middle, True, _call(ctx, middle, stats=True), "the same call once the graph is released")
    ctx.close()


def _sequence(seed, n_calls=100, kinds=KINDS, big_at=(30, 70)):
    """seeded calls; the ones at big_at are multi-slab, the first the plain fit, the second ARIMA(2, 1, 0)"""
    rng = np.random.default_rng(seed)
    seq = [(str(rng.choice(kinds)), bool(rng.integers(2))) for _ in range(n_calls)]
    for i, big in zip(big_at, ("big", "big_arima")):
        seq[i] = (big, bool(rng.integers(2)))
    return seq


def test_seeded_sequence_on_one_stream():
    seq = _sequence(2024)
    for name, stats in seq:
        _fresh(name, stats)
    ctx = Ctx()
    for i, (name, stats) in enumerate(seq):
        _check(name, stats, _call(ctx, name, stats), f"call {i}")
    ctx.close()


# =====================================================================================================================
# 3. tile counts
# =====================================================================================================================
# every instantiation at t_fit 32, 33 and 1,095; ragged calendars and backtest origins need t_fit >= 33, so the ragged
# kind runs at 33, 65 and 1,095 and the backtest at 33 (one origin), 36 (origins 33 .. 36) and 1,095
# The fit_tc hand-off instantiation (gamma / c to the ARIMA-family warp kernels, no forecast store) through
# ARIMA(2, 1, 0) and the (p, d, q) selection on the reference grid, and the standard-error pass behind ARIMA(1, 1, 1)
TILE_CASES = ([(inst, t) for inst in ("tc", "variant2", "se") for t in (32, 33, 1095)]
              + [("ragged", t) for t in (33, 65, 1095)] + [("backtest", t) for t in (33, 36, 1095)]
              + [(inst, t) for inst in ("arima21", "select_arma", "css") for t in (65, 1095)] + [("arima_se", T_FIT)])
ARIMA_INSTS = ("arima21", "select_arma", "arima_se", "css")


def _sizes(grid, inst=None):
    sizes = [128, 128 * (grid - 1), 128 * grid, 128 * (grid + 1), 128 * (4 * grid + 1), 256 * grid - 1, 256 * grid + 1]
    if inst in ARIMA_INSTS:                                # the ARIMA warp kernels: one series per warp, 8 per CTA
        sizes = [1, 7, 8, 9] + sizes
    if inst == "arima_se":                                 # at most 16 SM blocks of 4 warps, then a grid stride
        sizes += [64 * grid - 1, 64 * grid + 1]
    return sizes


def _z_pending(y, t_fit, diffs):
    """the pending count of one fit per listed d: the mask of y for d = 0, of z' = Delta^d y on t_fit - d rows for
    d >= 1, whose plan of D_d has no constant (so no row lacks a centring constant)"""
    total = 0
    for d in diffs:
        z = y[:, :t_fit].astype(np.float32)
        for _ in range(d):
            with np.errstate(invalid="ignore", over="ignore"):
                z = z[:, 1:] - z[:, :-1]
        total += _expected_pending(z, t_fit - d, has_constant=d == 0)
    return total


def _tile_perm(bounds):
    """row permutation that reverses the whole 128-row tiles of every segment [a, b) and keeps its partial tail"""
    perm = []
    for a, b in bounds:
        whole = (b - a) // 128
        for t in reversed(range(whole)):
            perm.extend(range(a + 128 * t, a + 128 * t + 128))
        perm.extend(range(a + 128 * whole, b))
    return np.array(perm, dtype=np.int64)


_MASTER = {}


def _master(t_fit, rows):
    if t_fit not in _MASTER:
        yd, _ = mmf.synth.daily_store_item_demand_torch(rows, t_fit + H, seed=t_fit, ld=_round4(t_fit + H))
        _plant_torch(yd, t_fit)
        _MASTER.clear()
        _MASTER[t_fit] = yd
    return _MASTER[t_fit]


def _run_inst(inst, eng, yd, t_fit, bounds):
    """one call of a fit_tc instantiation: {outputs}, n_pending"""
    n = yd.shape[0]
    if inst in ("tc", "variant2"):
        out, status = _f(n, H), _i(n)
        res = eng.fit_forecast(yd, t_fit, H, out=out, status=status, want_stats=True)
        assert res["stats"].kernel_used == "tc"
        return {"pred": out, "status": status}, res["stats"].n_pending
    if inst == "se":
        r = _se_raw(eng, yd, t_fit, H, True)
        return r, r.pop("n_pending")
    if inst == "backtest":
        r = _backtest_raw(eng, yd, True, len(eng._backtest[0]))
        return r, r.pop("n_pending")
    if inst in ARIMA_INSTS:
        rc, r = {"arima21": lambda: _r_arima(eng, yd, True, 2, 1, t_fit, H),
                 "select_arma": lambda: _r_select(eng, yd, True, REF, t_fit, H),
                 "arima_se": lambda: _r_arma(eng, yd, True, 1, 1, 1, t_fit, H, se=True, t_fit=t_fit),
                 "css": lambda: _r_css(eng, yd, True, 1, 1, 1, t_fit, H)}[inst]()
        N.check(rc)
        return r, r.pop("n_pending")
    out, status = _f(n, H), _i(n)
    res = eng.fit_forecast_ragged(yd, np.array([b[0] for b in bounds] + [n]), out=out, status=status, want_stats=True)
    return {"pred": out, "status": status}, res["stats"].n_pending


@pytest.mark.parametrize("inst, t_fit", TILE_CASES)
def test_tile_counts_around_the_grid(inst, t_fit):
    grid = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = _sizes(grid, inst)
    master = _master(t_fit, max(sizes))
    eng = mmf.ForecastEngine(kernel="tc" if inst in ("tc", "variant2", "se") + ARIMA_INSTS else "auto",
                             tc_variant=2 if inst == "variant2" else 0)
    starts = ("2019-01-01", "2019-05-17")
    if inst == "backtest":
        eng.plan_backtest(START, t_fit + H, "D", H, 1 if t_fit < 36 else K_BT, step=1)    # last origin t_fit
    elif inst != "ragged":
        eng.plan(_design_x(START, t_fit), t_fit, True)
    if inst in ARIMA_INSTS:
        eng.plan_arima(_design_x(START, t_fit), t_fit, 2)
    for n in sizes:
        bounds = [(0, n)]
        if inst == "ragged":                               # two calendars, the first a whole number of tiles
            half = (n // 256) * 128
            bounds = [(0, half), (half, n)] if half else [(0, n)]
            eng.plan_designs([_design_x(s, t_fit) for s in starts[:len(bounds)]], [t_fit] * len(bounds),
                             [t_fit] * len(bounds), [H] * len(bounds), True)
        y = master[:n]
        got, pend = _run_inst(inst, eng, y, t_fit, bounds)
        perm = _tile_perm(bounds)
        y_rev = torch.empty((n, master.stride(0)), device="cuda")[:, :master.shape[1]]
        y_rev.copy_(y[torch.from_numpy(perm).cuda()])
        rev, pend_rev = _run_inst(inst, eng, y_rev, t_fit, bounds)
        torch.cuda.synchronize()
        what = f"{inst} t_fit={t_fit} n={n} ({n / 128:.2f} tiles, grid {grid})"
        if inst == "backtest":
            want = _backtest_pieces(eng, y, grid)
        elif inst in ARIMA_INSTS:
            want = _z_pending(y.cpu().numpy(), t_fit, REF[1] if inst == "select_arma" else (1,))
        else:
            mask = y[:, :t_fit].cpu().numpy()
            want = sum(_expected_pending(mask[a:b], t_fit) for a, b in bounds)
        assert pend == want and pend_rev == want, (what, pend, pend_rev, want)
        for k, v in got.items():
            a, b = _bits(v), _bits(rev[k])
            axis = 1 if k in ("pred_bt", "metrics", "count", "status_bt") else 0
            assert not (a == SENT_F).any() and not (a == SENT_I).any(), (what, k, "sentinel left")
            assert np.array_equal(np.take(a, perm, axis=axis), b), (what, k, "reversed tiles")
    eng.close()


def _design_x(start, t_fit):
    return O.design_matrix(O.calendar_grid(np.datetime64(start, "D"), t_fit + H, "D"), t_fit)


def _backtest_pieces(eng, y, grid):
    """the backtest's pending count as the sum over calls of fewer tiles than CTAs (no tile is claimed dynamically)"""
    piece = 128 * max(1, grid - 1)
    total = 0
    for a in range(0, y.shape[0], piece):
        total += _backtest_raw(eng, y[a:a + piece], True, len(eng._backtest[0]))["n_pending"]
    return total


# =====================================================================================================================
# 4. streams
# =====================================================================================================================
def test_a_call_on_another_stream_between_two_calls_on_a_sleeping_stream():
    """Call 1 on stream A behind a long sleep, call 2 on stream B, call 3 on stream A.  The host hands call 2 the counter
    set that call 1's kernel is to zero, and skips the memset.  Without ordering at the stream switch, call 2 reaches the
    device before call 1 has run and starts from the counts of the call before it (tile claims, pending count, work
    list), and call 3 from whatever call 1 left.  All three calls have the same row count and different data, so every
    stale index stays inside the call's own buffers and shows as wrong or unwritten rows."""
    for name in ("aba_1", "aba_2", "aba_3"):
        _fresh(name)
    ctx = Ctx()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    for name in ("aba_1", "aba_2", "aba_3"):               # scratch grown before the sequence: no allocation in it
        _call(ctx, name)
    torch.cuda.synchronize()
    n = KIND_ROWS["aba_1"][0]
    outs = {name: {"pred": _f(n, H), "status": _i(n)} for name in ("aba_1", "aba_2", "aba_3")}
    torch.cuda.synchronize()
    for name, stream in (("aba_1", a), ("aba_2", b), ("aba_3", a)):
        with torch.cuda.stream(stream):
            if name == "aba_1":
                torch.cuda._sleep(200_000_000)             # ~0.1 s: call 2 reaches the device first
            ctx.eng.fit_forecast(_input(name)["yd"], T_FIT, H, out=outs[name]["pred"], status=outs[name]["status"])
    torch.cuda.synchronize()
    for name, out in outs.items():
        _diff(_host(out), _fresh(name), f"A / B / A: {name}")
    ctx.close()


def test_an_arima_call_on_another_stream_between_two_calls_on_a_sleeping_stream():
    """the A / B / A case with ARIMA(2, 1, 0) on stream B: its diff, fit (gamma / c hand-off) and arima kernels take the
    counter set call 1 is to zero, and call 3 the set the ARIMA fit is to zero"""
    names = ("aba_1", "aba_arima", "aba_3")
    for name in names:
        _fresh(name)
    ctx = Ctx()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    for name in names:                                     # scratch grown before the sequence: no allocation in it
        _call(ctx, name)
    n = KIND_ROWS["aba_1"][0]
    outs = {name: {"pred": _f(n, H), "status": _i(n)} for name in ("aba_1", "aba_3")}
    torch.cuda.synchronize()
    with torch.cuda.stream(a):
        torch.cuda._sleep(200_000_000)                     # ~0.1 s: call 2 reaches the device first
        ctx.eng.fit_forecast(_input("aba_1")["yd"], T_FIT, H, out=outs["aba_1"]["pred"], status=outs["aba_1"]["status"])
    with torch.cuda.stream(b):
        outs["aba_arima"] = _call(ctx, "aba_arima")
    with torch.cuda.stream(a):
        ctx.eng.fit_forecast(_input("aba_3")["yd"], T_FIT, H, out=outs["aba_3"]["pred"], status=outs["aba_3"]["status"])
    torch.cuda.synchronize()
    for name, out in outs.items():
        _diff(_host(out), _fresh(name), f"A / B / A: {name}")
    ctx.close()


def test_seeded_sequence_on_two_streams():
    """the seeded sequence, each call on one of two streams chosen by the seed, no host synchronisation in between"""
    seq = _sequence(2025)
    rng = np.random.default_rng(7)
    for name, stats in seq:
        _fresh(name, stats)
    streams = (torch.cuda.Stream(), torch.cuda.Stream())
    ctx = Ctx()
    torch.cuda.synchronize()
    results = []
    for name, stats in seq:
        with torch.cuda.stream(streams[int(rng.integers(2))]):
            results.append(_call(ctx, name, stats))
    torch.cuda.synchronize()
    for i, ((name, stats), res) in enumerate(zip(seq, results)):
        _check(name, stats, res, f"call {i}")
    ctx.close()


def test_two_engines_from_two_threads():
    """two engines, each driven by its own thread on its own stream: they share no state.  Every fourth call of each
    sequence is a (p, d, q) selection, alternating between grids that need 52,292 B and 74,732 B of dynamic shared
    memory, the two threads out of phase: arma_select_kernel's shared-memory attribute is per function and
    process-wide, and a launch must not fail because the other thread set it for its own call in between."""
    kinds = tuple(k for k in KINDS if k != "replay")       # a capture would stop the other thread's work
    seqs = [_sequence(3000 + t, n_calls=40, kinds=kinds, big_at=()) for t in range(2)]
    for t, seq in enumerate(seqs):
        for j, i in enumerate(range(t, 40, 4)):
            seq[i] = (("select_arma_52k", "select_arma_max")[(j + t) % 2], seq[i][1])
    for seq in seqs:
        for name, stats in seq:
            _fresh(name, stats)
    ctxs = [Ctx(), Ctx()]
    results, errors = [[], []], []

    def work(t):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                for name, stats in seqs[t]:
                    results[t].append(_call(ctxs[t], name, stats))
        except BaseException as e:                          # re-raised on the main thread
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    if errors:
        raise errors[0]
    torch.cuda.synchronize()
    for t in range(2):
        for i, ((name, stats), res) in enumerate(zip(seqs[t], results[t])):
            _check(name, stats, res, f"thread {t} call {i}")
    for c in ctxs:
        c.close()
