"""Every argument check of the device-buffer fit entry points: return code and full mmf_last_error() text.

One table, one case per check: each case starts from arguments the call accepts (test_defaults_are_accepted runs them)
and changes exactly one.  The expected codes and messages are the library's refusals as callers see them; a change of
wording, of code or of which check fires first for a given argument list shows up here."""
import ctypes as C

import numpy as np
import pytest

import mmf
from mmf import _native as N

pytestmark = pytest.mark.gpu

T, H, NR = 120, 28, 148          # fit rows, horizon, planned design rows
LD_Y, LD_OUT, NS = 152, 32, 8    # row pitch of y (>= T + H, 16-B rows), of the output table; series per call
INV, CUDA, UNS, NOPLAN = -1, -2, -3, -4


def _design(n_rows, p=4):
    t = np.arange(n_rows, dtype=np.float64)
    X = np.empty((n_rows, p), dtype=np.float64)
    X[:, 0] = 1.0
    X[:, 1] = t / n_rows
    X[:, 2] = np.sin(2 * np.pi * t / 7)
    X[:, 3] = np.cos(2 * np.pi * t / 7)
    return X


def _i32(*v):
    return (C.c_int32 * len(v))(*v)


@pytest.fixture(scope="module")
def env():
    import torch
    X = _design(NR)
    engs = {k: mmf.ForecastEngine(device=0) for k in ("plain", "none", "d1", "mixed", "ragged", "bt")}
    engs["plain"].plan(X, T, True)
    engs["plain"].plan_arima(X, T, 2)
    engs["d1"].plan(X, T, True)
    engs["d1"].plan_arima(X, T, 1)
    X2 = X.copy()
    X2[:, 1] *= 2.0                                          # same rows, t_fit and columns; other bytes
    engs["mixed"].plan(X, T, True)
    engs["mixed"].plan_arima(X2, T, 2)
    engs["ragged"].plan_designs([X, _design(128)], [T, 100], [T, 100], [H, H], True)
    lib = engs["bt"]._lib
    N.check(lib.mmf_plan_backtest(engs["bt"]._h, X.ctypes.data, NR, 4, 1, 2, _i32(92, 120), H))
    g = torch.Generator(device="cuda").manual_seed(3)
    bufs = {"y": 10.0 + torch.rand((NS, LD_Y), generator=g, device="cuda"),
            "yi": torch.full((NS, LD_Y), 7, dtype=torch.int16, device="cuda"),
            "host": np.zeros((NS, 512), dtype=np.float32)}
    yield {"engs": engs, "lib": lib, "bufs": bufs}
    for e in engs.values():
        e.close()


def _defaults(b):
    """the accepted arguments of every entry point, by name; pointers as integers.  Every output (and every input of
    mmf_arima_se_f32) has a zeroed device buffer of its own."""
    import torch

    def dev(name, dtype=torch.float32):
        if name not in b:
            b[name] = torch.zeros((NS, 512), dtype=dtype, device="cuda")
        return b[name].data_ptr()

    f = dev
    i = lambda name: dev(name, torch.int32)                    # noqa: E731
    y, out = b["y"].data_ptr(), dev("out")
    fit = dict(y=y, n=NS, ld_y=LD_Y, pred_start=T, n_pred=H, out=out, ld_out=LD_OUT)
    return {
        "fit_f32": dict(fit, beta=None, status=i("status")),
        "fit_int": dict(fit, y=b["yi"].data_ptr(), dtype=N.DT_I16, beta=None, status=i("status")),
        "se": dict(fit, se=f("se"), ld_se=LD_OUT, sigma=f("sigma"), dof=i("dof"), status=i("status")),
        "ar": dict(fit, ar_order=2, phi=f("phi"), order=i("order"), sigma=f("sigma"), status=i("status")),
        "select_ar": dict(fit, n_hold=H, orders=(0, 1, 2), choice=i("choice"), mse=f("mse"), cand_mse=f("cand_mse"),
                          phi=f("phi"), order=i("order"), sigma=f("sigma"), status=i("status")),
        "arima": dict(fit, ar_order=1, diff_order=1, phi=f("phi"), order=i("order"), sigma=f("sigma"),
                      status=i("status")),
        "arma": dict(fit, ar_order=1, diff_order=1, ma_order=1, long_order=0, phi=f("phi"), theta=f("theta"),
                     order=i("order"), ma_ord=i("ma_ord"), sigma=f("sigma"), status=i("status")),
        "arma_css": dict(fit, ar_order=1, diff_order=1, ma_order=1, long_order=0, max_iter=0, phi=f("phi"),
                         theta=f("theta"), order=i("order"), ma_ord=i("ma_ord"), sigma=f("sigma"), status=i("status"),
                         css_start=f("css_start"), css=f("css"), css_stop=i("css_stop"), iters=i("iters")),
        # inputs nothing else writes: zero orders, zero coefficients
        "arima_se": dict(y=y, n=NS, ld_y=LD_Y, t_fit=T, diff_order=1, diffs=None, phi=f("in_phi"), order=i("in_order"),
                         theta=f("in_theta"), ma_ord=i("in_ma_ord"), sigma=f("in_sigma"), pred_start=T, n_pred=H,
                         se=f("se"), ld_se=LD_OUT),
        "select_arima": dict(fit, n_hold=H, orders=(0, 1, 2), diffs=(0, 1, 2), choice_p=i("choice_p"),
                             choice_d=i("choice_d"), mse=f("mse"), cand_mse=f("cand_mse"), phi=f("phi"),
                             order=i("order"), sigma=f("sigma"), status=i("status")),
        "select_arma": dict(fit, n_hold=H, orders=(0, 1, 2), diffs=(0, 1), mas=(0, 1, 2), long_order=0,
                            choice_p=i("choice_p"), choice_d=i("choice_d"), choice_q=i("choice_q"), mse=f("mse"),
                            cand_mse=f("cand_mse"), phi=f("phi"), theta=f("theta"), order=i("order"),
                            ma_ord=i("ma_ord"), sigma=f("sigma"), status=i("status")),
        "ragged": dict(y=y, n=NS, ld_y=LD_Y, rows=(0, 5, NS), out=out, ld_out=LD_OUT, status=i("status")),
        "backtest": dict(y=y, n=NS, ld_y=LD_Y, out=f("bt_out"), ld_out=LD_OUT, metrics=f("metrics"), count=i("count"),
                         status=i("status")),
        "bcast": dict(fit, ptrs=(out,), n_out=1, multimem=0, beta=None, status=i("status")),
        "select_forecast": dict(fit, n_hold=H, cands=(1, 4), choice=i("choice"), mse=f("mse"), status=i("status")),
    }


def _call(lib, h, entry, a):
    i32 = lambda v: None if v is None else _i32(*v)            # noqa: E731
    st = N.MmfStats()
    s = C.byref(st)
    if entry == "fit_f32":
        return lib.mmf_fit_forecast_f32(h, a["y"], a["n"], a["ld_y"], a["pred_start"], a["n_pred"], a["out"],
                                        a["ld_out"], a["beta"], a["status"], s)
    if entry == "fit_int":
        return lib.mmf_fit_forecast_int(h, a["y"], a["dtype"], a["n"], a["ld_y"], a["pred_start"], a["n_pred"],
                                        a["out"], a["ld_out"], a["beta"], a["status"], s)
    if entry == "se":
        return lib.mmf_fit_forecast_se_f32(h, a["y"], a["n"], a["ld_y"], a["pred_start"], a["n_pred"], a["out"],
                                           a["ld_out"], a["se"], a["ld_se"], a["sigma"], a["dof"], a["status"], s)
    if entry == "ar":
        return lib.mmf_fit_forecast_ar_f32(h, a["y"], a["n"], a["ld_y"], a["ar_order"], a["pred_start"], a["n_pred"],
                                           a["out"], a["ld_out"], a["phi"], a["order"], a["sigma"], a["status"], s)
    if entry == "select_ar":
        o = a["orders"]
        return lib.mmf_fit_select_ar_f32(h, a["y"], a["n"], a["ld_y"], a["n_hold"], i32(o),
                                         a.get("n_orders", len(o or ())), a["pred_start"], a["n_pred"], a["out"],
                                         a["ld_out"], a["choice"], a["mse"],
                                         a["cand_mse"], a["phi"], a["order"], a["sigma"], a["status"], s)
    if entry == "arima":
        return lib.mmf_fit_forecast_arima_f32(h, a["y"], a["n"], a["ld_y"], a["ar_order"], a["diff_order"],
                                              a["pred_start"], a["n_pred"], a["out"], a["ld_out"], a["phi"], a["order"],
                                              a["sigma"], a["status"], s)
    if entry == "arma":
        return lib.mmf_fit_forecast_arma_f32(h, a["y"], a["n"], a["ld_y"], a["ar_order"], a["diff_order"],
                                             a["ma_order"], a["long_order"], a["pred_start"], a["n_pred"], a["out"],
                                             a["ld_out"], a["phi"], a["theta"], a["order"], a["ma_ord"], a["sigma"],
                                             a["status"], s)
    if entry == "arma_css":
        return lib.mmf_fit_forecast_arma_css_f32(h, a["y"], a["n"], a["ld_y"], a["ar_order"], a["diff_order"],
                                                 a["ma_order"], a["long_order"], a["max_iter"], a["pred_start"],
                                                 a["n_pred"], a["out"], a["ld_out"], a["phi"], a["theta"], a["order"],
                                                 a["ma_ord"], a["sigma"], a["status"], a["css_start"], a["css"],
                                                 a["css_stop"], a["iters"], s)
    if entry == "arima_se":
        return lib.mmf_arima_se_f32(h, a["y"], a["n"], a["ld_y"], a["t_fit"], a["diff_order"], a["diffs"], a["phi"],
                                    a["order"], a["theta"], a["ma_ord"], a["sigma"], a["pred_start"], a["n_pred"],
                                    a["se"], a["ld_se"], s)
    if entry == "select_arima":
        o, d = a["orders"], a["diffs"]
        return lib.mmf_fit_select_arima_f32(h, a["y"], a["n"], a["ld_y"], a["n_hold"], i32(o),
                                            a.get("n_orders", len(o or ())), i32(d), a.get("n_diffs", len(d or ())),
                                            a["pred_start"], a["n_pred"], a["out"], a["ld_out"], a["choice_p"],
                                            a["choice_d"], a["mse"], a["cand_mse"], a["phi"], a["order"], a["sigma"],
                                            a["status"], s)
    if entry == "select_arma":
        o, d, q = a["orders"], a["diffs"], a["mas"]
        return lib.mmf_fit_select_arma_f32(h, a["y"], a["n"], a["ld_y"], a["n_hold"], i32(o),
                                           a.get("n_orders", len(o or ())), i32(d), a.get("n_diffs", len(d or ())),
                                           i32(q), a.get("n_mas", len(q or ())), a["long_order"], a["pred_start"],
                                           a["n_pred"], a["out"], a["ld_out"], a["choice_p"], a["choice_d"],
                                           a["choice_q"], a["mse"], a["cand_mse"], a["phi"], a["theta"], a["order"],
                                           a["ma_ord"], a["sigma"], a["status"], s)
    if entry == "ragged":
        rows = None if a["rows"] is None else np.array(a["rows"], dtype=np.int64)
        return lib.mmf_fit_forecast_ragged_f32(h, a["y"], a["n"], a["ld_y"], None if rows is None else rows.ctypes.data,
                                               a["out"], a["ld_out"], a["status"], s)
    if entry == "backtest":
        return lib.mmf_backtest_f32(h, a["y"], a["n"], a["ld_y"], a["out"], a["ld_out"], a["metrics"], a["count"],
                                    a["status"], s)
    if entry == "bcast":
        p = a["ptrs"]
        ptrs = None if p is None else (C.c_uint64 * len(p))(*p)
        return lib.mmf_fit_forecast_bcast_f32(h, a["y"], a["n"], a["ld_y"], a["pred_start"], a["n_pred"], ptrs,
                                              a["n_out"], a["multimem"], a["ld_out"], a["beta"], a["status"])
    if entry == "select_forecast":
        c = a["cands"]
        return lib.mmf_fit_select_forecast_f32(h, a["y"], a["n"], a["ld_y"], a["n_hold"], i32(c),
                                               a.get("n_cand", len(c or ())), a["pred_start"], a["n_pred"], a["out"],
                                               a["ld_out"], a["choice"], a["mse"], a["status"])
    raise KeyError(entry)


WINDOW = "prediction rows [120,149) outside the planned design (148 rows)"
HOST = "host"           # stands for a host (NumPy) buffer in a case's arguments

# (entry point, engine, the one changed argument, code, mmf_last_error())
CASES = [
    # ---- mmf_fit_forecast_f32 (host buffers are accepted: no device-pointer check)
    ("fit_f32", "none", {}, NOPLAN, "mmf_plan_design has not been called"),
    ("fit_f32", "plain", {"n": -1}, INV, "n < 0"),
    ("fit_f32", "plain", {"y": None}, INV, "y or out_pred is NULL"),
    ("fit_f32", "plain", {"out": None}, INV, "y or out_pred is NULL"),
    ("fit_f32", "plain", {"ld_y": T - 1}, INV, "ld_y=119 < t_fit=120"),
    ("fit_f32", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("fit_f32", "plain", {"pred_start": -1}, INV, "prediction rows [-1,27) outside the planned design (148 rows)"),
    ("fit_f32", "plain", {"n_pred": 0}, INV, "prediction rows [120,120) outside the planned design (148 rows)"),
    ("fit_f32", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    # ---- mmf_fit_forecast_int
    ("fit_int", "plain", {"dtype": N.DT_F32}, INV,
     "mmf_fit_forecast_int takes MMF_DT_I16 / U16 / I32; use mmf_fit_forecast_f32"),
    ("fit_int", "plain", {"dtype": 7}, INV, "dtype 7 is not one of MMF_DT_F32 / I16 / U16 / I32"),
    ("fit_int", "none", {}, NOPLAN, "mmf_plan_design has not been called"),
    ("fit_int", "plain", {"n": -1}, INV, "n < 0"),
    ("fit_int", "plain", {"y": None}, INV, "y or out_pred is NULL"),
    ("fit_int", "plain", {"ld_y": T - 1}, INV, "ld_y=119 < t_fit=120"),
    ("fit_int", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("fit_int", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    # ---- mmf_fit_forecast_se_f32
    ("se", "none", {}, NOPLAN, "mmf_plan_design has not been called"),
    ("se", "plain", {"n": -1}, INV, "n < 0"),
    ("se", "plain", {"out": None}, INV, "y or out_pred is NULL"),
    ("se", "plain", {"se": None, "sigma": None, "dof": None}, INV,
     "out_se, out_sigma and out_dof are all NULL: use mmf_fit_forecast_f32"),
    ("se", "plain", {"ld_y": T - 1}, INV, "ld_y=119 < t_fit=120"),
    ("se", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("se", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    ("se", "plain", {"ld_se": H - 1}, INV, "ld_se=27 < n_pred=28"),
    ("se", "plain", {"sigma": HOST}, UNS, "mmf_fit_forecast_se_f32 takes device buffers only"),
    ("se", "plain", {"y": HOST}, UNS, "mmf_fit_forecast_se_f32 takes device buffers only"),
    # ---- mmf_fit_forecast_ar_f32
    ("ar", "none", {}, NOPLAN, "mmf_plan_design has not been called"),
    ("ar", "plain", {"n": -1}, INV, "n < 0"),
    ("ar", "plain", {"y": None}, INV, "y or out_pred is NULL"),
    ("ar", "plain", {"ar_order": 0}, INV, "ar_order=0 outside [1,8]"),
    ("ar", "plain", {"ar_order": 9}, INV, "ar_order=9 outside [1,8]"),
    ("ar", "plain", {"ld_y": T - 1}, INV, "ld_y=119 < t_fit=120"),
    ("ar", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("ar", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    ("ar", "plain", {"phi": HOST}, UNS, "mmf_fit_forecast_ar_f32 takes device buffers only"),
    ("ar", "plain", {"status": HOST}, UNS, "mmf_fit_forecast_ar_f32 takes device buffers only"),
    # ---- mmf_fit_select_ar_f32
    ("select_ar", "none", {}, NOPLAN, "mmf_plan_design has not been called"),
    ("select_ar", "plain", {"n": -1}, INV, "n < 0"),
    ("select_ar", "plain", {"out": None}, INV, "y or out_pred is NULL"),
    ("select_ar", "plain", {"orders": None, "n_orders": 3}, INV, "n_orders=3 outside [1,9] (or orders is NULL)"),
    ("select_ar", "plain", {"orders": tuple(range(10))}, INV, "n_orders=10 outside [1,9] (or orders is NULL)"),
    ("select_ar", "plain", {"orders": (2, 1)}, INV, "orders must be ascending and distinct in [0,8] (orders[1]=1)"),
    ("select_ar", "plain", {"orders": (0, 9)}, INV, "orders must be ascending and distinct in [0,8] (orders[1]=9)"),
    ("select_ar", "plain", {"orders": (-1, 2)}, INV, "orders must be ascending and distinct in [0,8] (orders[0]=-1)"),
    ("select_ar", "plain", {"n_hold": 0}, INV, "held-out rows [120,120) outside the planned design (148 rows)"),
    ("select_ar", "plain", {"n_hold": H + 1}, INV, "held-out rows [120,149) outside the planned design (148 rows)"),
    ("select_ar", "plain", {"ld_y": T + H - 1}, INV, "ld_y=147 < t_fit + n_hold=148"),
    ("select_ar", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("select_ar", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    ("select_ar", "plain", {"cand_mse": HOST}, UNS, "mmf_fit_select_ar_f32 takes device buffers only"),
    # ---- mmf_fit_forecast_arima_f32
    ("arima", "none", {}, NOPLAN, "mmf_plan_arima has not been called"),
    ("arima", "plain", {"n": -1}, INV, "n < 0"),
    ("arima", "plain", {"y": None}, INV, "y or out_pred is NULL"),
    ("arima", "plain", {"ar_order": -1}, INV, "ar_order=-1 outside [0,8]"),
    ("arima", "plain", {"ar_order": 9}, INV, "ar_order=9 outside [0,8]"),
    ("arima", "plain", {"diff_order": 0}, INV, "diff_order=0 outside [1,2] (the planned max_diff)"),
    ("arima", "d1", {"diff_order": 2}, INV, "diff_order=2 outside [1,1] (the planned max_diff)"),
    ("arima", "plain", {"ld_y": T - 1}, INV, "ld_y=119 < t_fit=120"),
    ("arima", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("arima", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    ("arima", "plain", {"sigma": HOST}, UNS, "mmf_fit_forecast_arima_f32 takes device buffers only"),
    # ---- mmf_fit_forecast_arma_f32
    ("arma", "plain", {"n": -1}, INV, "n < 0"),
    ("arma", "plain", {"out": None}, INV, "y or out_pred is NULL"),
    ("arma", "plain", {"ar_order": 9}, INV, "ar_order=9 outside [0,8]"),
    ("arma", "plain", {"ma_order": 0}, INV, "ma_order=0 outside [1,4]"),
    ("arma", "plain", {"ma_order": 5}, INV, "ma_order=5 outside [1,4]"),
    ("arma", "plain", {"diff_order": 3}, INV, "diff_order=3 outside [0,2]"),
    ("arma", "none", {"diff_order": 0}, NOPLAN, "mmf_plan_design has not been called"),
    ("arma", "none", {}, NOPLAN, "mmf_plan_arima has not been called"),
    ("arma", "d1", {"diff_order": 2}, INV, "diff_order=2 above the planned max_diff=1"),
    ("arma", "plain", {"long_order": 33}, INV, "long_order=33 outside {0} and [1,32]"),
    ("arma", "plain", {"ar_order": 3, "long_order": 2}, INV, "long_order=2 outside {0} and [3,32]"),
    ("arma", "plain", {"ld_y": T - 1}, INV, "ld_y=119 < t_fit=120"),
    ("arma", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("arma", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    ("arma", "plain", {"theta": HOST}, UNS, "mmf_fit_forecast_arma_f32 takes device buffers only"),
    ("arma", "plain", {"diff_order": 0, "ma_ord": HOST}, UNS, "mmf_fit_forecast_arma_f32 takes device buffers only"),
    # ---- mmf_fit_forecast_arma_css_f32 (max_iter is checked first)
    ("arma_css", "none", {"max_iter": -1}, INV, "max_iter=-1 outside [0,64]"),
    ("arma_css", "plain", {"max_iter": 65}, INV, "max_iter=65 outside [0,64]"),
    ("arma_css", "plain", {"n": -1}, INV, "n < 0"),
    ("arma_css", "plain", {"y": None}, INV, "y or out_pred is NULL"),
    ("arma_css", "plain", {"ma_order": 0}, INV, "ma_order=0 outside [1,4]"),
    ("arma_css", "none", {}, NOPLAN, "mmf_plan_arima has not been called"),
    ("arma_css", "plain", {"long_order": 33}, INV, "long_order=33 outside {0} and [1,32]"),
    ("arma_css", "plain", {"ld_y": T - 1}, INV, "ld_y=119 < t_fit=120"),
    ("arma_css", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("arma_css", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    ("arma_css", "plain", {"css": HOST}, UNS, "mmf_fit_forecast_arma_css_f32 takes device buffers only"),
    ("arma_css", "plain", {"iters": HOST}, UNS, "mmf_fit_forecast_arma_css_f32 takes device buffers only"),
    ("arma_css", "plain", {"phi": HOST}, UNS, "mmf_fit_forecast_arma_css_f32 takes device buffers only"),
    # ---- mmf_arima_se_f32 (no plan needed)
    ("arima_se", "plain", {"n": -1}, INV, "n < 0"),
    ("arima_se", "plain", {"phi": None}, INV, "y, phi, order, sigma or out_se is NULL"),
    ("arima_se", "plain", {"se": None}, INV, "y, phi, order, sigma or out_se is NULL"),
    ("arima_se", "plain", {"ma_ord": None}, INV, "theta and ma_order must both be given or both be NULL"),
    ("arima_se", "plain", {"diff_order": 3}, INV, "diff_order=3 outside [0,2]"),
    ("arima_se", "plain", {"t_fit": 0}, INV, "t_fit=0 < 1"),
    ("arima_se", "plain", {"t_fit": LD_Y + 1}, INV, "ld_y=152 < t_fit=153"),
    ("arima_se", "plain", {"n_pred": 0}, INV, "prediction rows [120,120) outside [0,2147483647]"),
    ("arima_se", "plain", {"pred_start": -1}, INV, "prediction rows [-1,27) outside [0,2147483647]"),
    ("arima_se", "plain", {"ld_se": H - 1}, INV, "ld_se=27 < n_pred=28"),
    ("arima_se", "plain", {"phi": HOST}, UNS, "mmf_arima_se_f32 takes device buffers only"),
    ("arima_se", "plain", {"theta": HOST}, UNS, "mmf_arima_se_f32 takes device buffers only"),
    # ---- mmf_fit_select_arima_f32
    ("select_arima", "plain", {"n": -1}, INV, "n < 0"),
    ("select_arima", "plain", {"y": None}, INV, "y or out_pred is NULL"),
    ("select_arima", "plain", {"orders": None, "n_orders": 3}, INV, "n_orders=3 outside [1,9] (or orders is NULL)"),
    ("select_arima", "plain", {"orders": (1, 1)}, INV, "orders must be ascending and distinct in [0,8] (orders[1]=1)"),
    ("select_arima", "plain", {"diffs": None, "n_diffs": 2}, INV, "n_diffs=2 outside [1,3] (or diffs is NULL)"),
    ("select_arima", "plain", {"diffs": (0, 1, 2, 3)}, INV, "n_diffs=4 outside [1,3] (or diffs is NULL)"),
    ("select_arima", "plain", {"diffs": (1, 0)}, INV, "diffs must be ascending and distinct in [0,2] (diffs[1]=0)"),
    ("select_arima", "plain", {"diffs": (0, 3)}, INV, "diffs must be ascending and distinct in [0,2] (diffs[1]=3)"),
    ("select_arima", "none", {}, NOPLAN, "diffs lists 0 and mmf_plan_design has not been called"),
    ("select_arima", "none", {"diffs": (1, 2)}, NOPLAN, "diffs lists d >= 1 and mmf_plan_arima has not been called"),
    ("select_arima", "d1", {}, INV, "diffs lists d=2 above the planned max_diff=1"),
    ("select_arima", "mixed", {}, INV, "the mmf_plan_design and mmf_plan_arima plans were built from different designs "
     "(rows 148 / 148, t_fit 120 / 120, columns 4 / 4)"),
    ("select_arima", "plain", {"n_hold": 0}, INV, "held-out rows [120,120) outside the planned design (148 rows)"),
    ("select_arima", "plain", {"diffs": (1, 2), "n_hold": H + 1}, INV,
     "held-out rows [120,149) outside the planned design (148 rows)"),
    ("select_arima", "plain", {"ld_y": T + H - 1}, INV, "ld_y=147 < t_fit + n_hold=148"),
    ("select_arima", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("select_arima", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    ("select_arima", "plain", {"choice_d": HOST}, UNS, "mmf_fit_select_arima_f32 takes device buffers only"),
    ("select_arima", "plain", {"y": HOST}, UNS, "mmf_fit_select_arima_f32 takes device buffers only"),
    # ---- mmf_fit_select_arma_f32
    ("select_arma", "plain", {"n": -1}, INV, "n < 0"),
    ("select_arma", "plain", {"out": None}, INV, "y or out_pred is NULL"),
    ("select_arma", "plain", {"orders": (0, 9)}, INV, "orders must be ascending and distinct in [0,8] (orders[1]=9)"),
    ("select_arma", "plain", {"diffs": (2, 1)}, INV, "diffs must be ascending and distinct in [0,2] (diffs[1]=1)"),
    ("select_arma", "plain", {"mas": None, "n_mas": 3}, INV, "n_mas=3 outside [1,5] (or mas is NULL)"),
    ("select_arma", "plain", {"mas": (0, 1, 2, 3, 4, 5)}, INV, "n_mas=6 outside [1,5] (or mas is NULL)"),
    ("select_arma", "plain", {"mas": (1, 2)}, INV, "mas[0]=1: the MA orders must start with 0"),
    ("select_arma", "plain", {"mas": (0, 2, 2)}, INV, "mas must be ascending and distinct in [0,4] (mas[2]=2)"),
    ("select_arma", "plain", {"mas": (0, 5)}, INV, "mas must be ascending and distinct in [0,4] (mas[1]=5)"),
    ("select_arma", "plain", {"orders": tuple(range(9)), "mas": (0, 1, 2, 3, 4)}, INV,
     "9 x 4 (p, q >= 1) pairs above MMF_ARMASEL_MAX_PQ=32"),
    ("select_arma", "plain", {"long_order": 1}, INV, "long_order=1 outside {0} and [2,32]"),
    ("select_arma", "plain", {"long_order": 33}, INV, "long_order=33 outside {0} and [2,32]"),
    ("select_arma", "none", {}, NOPLAN, "diffs lists 0 and mmf_plan_design has not been called"),
    ("select_arma", "none", {"diffs": (1,)}, NOPLAN, "diffs lists d >= 1 and mmf_plan_arima has not been called"),
    ("select_arma", "d1", {"diffs": (0, 2)}, INV, "diffs lists d=2 above the planned max_diff=1"),
    ("select_arma", "mixed", {}, INV, "the mmf_plan_design and mmf_plan_arima plans were built from different designs "
     "(rows 148 / 148, t_fit 120 / 120, columns 4 / 4)"),
    ("select_arma", "plain", {"n_hold": H + 1}, INV, "held-out rows [120,149) outside the planned design (148 rows)"),
    ("select_arma", "plain", {"ld_y": T + H - 1}, INV, "ld_y=147 < t_fit + n_hold=148"),
    ("select_arma", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("select_arma", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    ("select_arma", "plain", {"choice_q": HOST}, UNS, "mmf_fit_select_arma_f32 takes device buffers only"),
    ("select_arma", "plain", {"theta": HOST}, UNS, "mmf_fit_select_arma_f32 takes device buffers only"),
    # ---- mmf_fit_forecast_ragged_f32
    ("ragged", "plain", {}, NOPLAN, "mmf_plan_calendars has not been called"),
    ("ragged", "ragged", {"n": -1}, INV, "bad y / out_pred / cal_row_start / n"),
    ("ragged", "ragged", {"rows": None}, INV, "bad y / out_pred / cal_row_start / n"),
    ("ragged", "ragged", {"out": None}, INV, "bad y / out_pred / cal_row_start / n"),
    ("ragged", "ragged", {"rows": (1, 5, NS)}, INV, "cal_row_start must run from 0 to n"),
    ("ragged", "ragged", {"rows": (0, 5, NS - 1)}, INV, "cal_row_start must run from 0 to n"),
    ("ragged", "ragged", {"rows": (0, NS + 1, NS)}, INV, "cal_row_start must be non-decreasing"),
    ("ragged", "ragged", {"ld_y": T - 1}, INV, "ld_y=119 < the longest calendar's t_fit=120"),
    ("ragged", "ragged", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    ("ragged", "ragged", {"y": HOST}, INV, "the ragged entry point takes device buffers only"),
    ("ragged", "ragged", {"status": HOST}, INV, "the ragged entry point takes device buffers only"),
    ("ragged", "ragged", {"ld_y": LD_Y - 2}, UNS,
     "ragged batches need 16-B aligned y / out_pred and ld_y % 4 == 0 (TMA)"),
    # ---- mmf_backtest_f32
    ("backtest", "plain", {}, NOPLAN, "mmf_plan_backtest has not been called"),
    ("backtest", "bt", {"n": -1}, INV, "bad y / n"),
    ("backtest", "bt", {"y": None}, INV, "bad y / n"),
    ("backtest", "bt", {"out": None, "metrics": None}, INV, "out_pred and out_metrics are both NULL"),
    ("backtest", "bt", {"ld_y": T + H - 1}, INV, "ld_y=147 < last origin + horizon = 148 (the actual values are read)"),
    ("backtest", "bt", {"ld_out": H - 1}, INV, "ld_out=27 < horizon=28"),
    ("backtest", "bt", {"ld_y": LD_Y - 2}, UNS, "backtests need a 16-B aligned y with ld_y % 4 == 0 (TMA)"),
    ("backtest", "bt", {"metrics": HOST}, UNS, "mmf_backtest_f32 takes device buffers only"),
    ("backtest", "bt", {"count": HOST}, UNS, "mmf_backtest_f32 takes device buffers only"),
    # ---- mmf_fit_forecast_bcast_f32
    ("bcast", "none", {}, NOPLAN, "mmf_plan_design has not been called"),
    ("bcast", "plain", {"n": -1}, INV, "bad y / out_ptrs / n"),
    ("bcast", "plain", {"ptrs": None}, INV, "bad y / out_ptrs / n"),
    ("bcast", "plain", {"n_out": 0}, INV, "n_out=0 outside [1,8]"),
    ("bcast", "plain", {"n_out": 9}, INV, "n_out=9 outside [1,8]"),
    ("bcast", "plain", {"multimem": 3}, INV,
     "multimem must be 0, 1 (multimem.st) or 2 (bulk stores to the multicast address)"),
    ("bcast", "plain", {"multimem": 1, "n_out": 2}, INV, "multimem=1 takes exactly one (multicast) pointer"),
    ("bcast", "plain", {"ld_y": T - 1}, INV, "ld_y=119 < t_fit=120"),
    ("bcast", "plain", {"n_pred": H + 1}, INV, WINDOW),
    ("bcast", "plain", {"ld_out": H - 1}, INV, "ld_out=27 < n_pred=28"),
    ("bcast", "plain", {"y": HOST}, INV, "the broadcast variant takes device buffers only"),
    # ---- mmf_fit_select_forecast_f32 (its own terse messages)
    ("select_forecast", "none", {}, NOPLAN, "mmf_plan_design has not been called"),
    ("select_forecast", "plain", {"n": -1}, INV, "bad y / out_pred / n"),
    ("select_forecast", "plain", {"out": None}, INV, "bad y / out_pred / n"),
    ("select_forecast", "plain", {"cands": None, "n_cand": 2}, INV, "need 1..8 candidates"),
    ("select_forecast", "plain", {"cands": tuple(range(1, 10))}, INV, "need 1..8 candidates"),
    ("select_forecast", "plain", {"cands": (4, 1)}, INV, "candidates must be ascending column counts in [1,16]"),
    ("select_forecast", "plain", {"cands": (1, 17)}, INV, "candidates must be ascending column counts in [1,16]"),
    ("select_forecast", "plain", {"n_hold": H + 1}, INV, "held-out rows exceed the planned design"),
    ("select_forecast", "plain", {"n_hold": 0}, INV, "held-out rows exceed the planned design"),
    ("select_forecast", "plain", {"ld_y": T + H - 1}, INV, "y must hold the fit rows and the held-out rows"),
    ("select_forecast", "plain", {"n_pred": H + 1}, INV, "prediction rows outside the planned design"),
    ("select_forecast", "plain", {"ld_out": H - 1}, INV, "ld_out < n_pred"),
    ("select_forecast", "plain", {"out": HOST}, INV, "device buffers only"),
]


def _case_id(c):
    entry, eng, over, _, _ = c
    return f"{entry}-{eng}-" + ("defaults" if not over else ",".join(f"{k}={v}" for k, v in over.items()))


def _args(env, entry, over):
    a = dict(_defaults(env["bufs"])[entry])
    host = env["bufs"]["host"].ctypes.data
    a.update({k: host if v == HOST else v for k, v in over.items()})
    return a


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_refusal(env, case):
    import torch
    entry, eng_key, over, code, msg = case
    eng = env["engs"][eng_key]
    rc = _call(env["lib"], eng._h, entry, _args(env, entry, over))
    torch.cuda.synchronize()
    assert (rc, env["lib"].mmf_last_error().decode()) == (code, msg)


@pytest.mark.parametrize("entry", sorted({c[0] for c in CASES}))
def test_defaults_are_accepted(env, entry):
    """the arguments every refusal case starts from are accepted on the engine most cases use"""
    import torch
    eng = env["engs"]["ragged" if entry == "ragged" else "bt" if entry == "backtest" else "plain"]
    rc = _call(env["lib"], eng._h, entry, _args(env, entry, {}))
    torch.cuda.synchronize()
    assert rc == 0, env["lib"].mmf_last_error().decode()
