"""GPU (-m gpu): the (p, d, q) selection's winners refit by exact likelihood (mmf_fit_select_arma_ml_f32) and predicted
with that likelihood's Kalman filter (mmf_fit_select_arma_ml_kf_f32), DESIGN.md section 2 item 21.

The contract is a composition, so it is checked as one, as tests/test_gpu_arma_select_css.py checks the CSS refit: a
winner with q >= 1 must get every output of the fixed-order ML (ML + Kalman) call at its own (p, d, q) with long_order =
m_d, bit for bit, se included; a winner with q = 0 and a row with no eligible candidate keep mmf_fit_select_arma_f32's
outputs bit for bit, with loglik_start, loglik NaN and ml_stop, iters 0, and their se is mmf_arima_se_f32 of the call's
outputs with the per-series d; choice_*, mse and cand_mse are the selection's.  The fixed-order calls run on the whole
batch and are compared on the rows of each class (a row's outputs depend on its own data only)."""
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
from ar_oracle import AR_MAX
from arma_oracle import MA_MAX
from conftest import ROOT, record_err
from test_gpu_arima_select import N_HOLD, _bits, _device, _engine, _np
from test_gpu_arma_select import REF, SENT_F, SENT_I, _call, _ma_case, _ms
from test_gpu_arma_select_css import _gapped
from test_gpu_edges import _same_bits

pytestmark = pytest.mark.gpu

SEL_OUT = ("choice_p", "choice_d", "choice_q", "mse", "cand_mse")
KEPT_OUT = ("pred", "phi", "theta", "order", "ma_order", "sigma", "status")
FIX_OUT = KEPT_OUT + ("loglik_start", "loglik", "ml_stop", "iters")
NULLABLE = ("choice_p", "choice_d", "choice_q", "mse", "cand_mse", "phi", "theta", "order", "ma_order", "sigma",
            "status", "loglik_start", "loglik", "ml_stop", "iters", "se")
SMALL = ((0, 1, 2), (0, 1, 2), (0, 1, 2))


def _refit(eng, yd, orders, diffs, mas, ps, npred, kf, max_iter=0, null=(), lib=None, ld_se=None):
    """the ML (kf: ML + Kalman, with out_se) refit through the C ABI, every output pre-filled with a sentinel; `null`:
    outputs passed as NULL"""
    lib = lib or eng._lib
    n = yd.shape[0]
    no, nd, nq = len(orders), len(diffs), len(mas)
    f = lambda *s: torch.full(s, SENT_F, device="cuda")
    i = lambda *s: torch.full(s, SENT_I, device="cuda", dtype=torch.int32)
    ld_se = ld_se or npred
    out = dict(pred=f(n, npred), choice_p=i(n), choice_d=i(n), choice_q=i(n), mse=f(n), cand_mse=f(n, nd, nq, no),
               phi=f(n, AR_MAX), theta=f(n, MA_MAX), order=i(n), ma_order=i(n), sigma=f(n), status=i(n),
               loglik_start=f(n), loglik=f(n), ml_stop=i(n), iters=i(n), se=f(n, ld_se))
    ptr = lambda k: None if k in null else out[k].data_ptr()
    arr = lambda v: (ctypes.c_int32 * len(v))(*v)
    head = (eng._h, yd.data_ptr(), n, yd.stride(0), N_HOLD, arr(orders), no, arr(diffs), nd, arr(mas), nq, 0,
            max_iter, ps, npred, out["pred"].data_ptr(), npred)
    tail = [ptr(k) for k in ("choice_p", "choice_d", "choice_q", "mse", "cand_mse", "phi", "theta", "order",
                             "ma_order", "sigma", "status", "loglik_start", "loglik", "ml_stop", "iters")]
    torch.cuda.synchronize()
    if kf:
        rc = lib.mmf_fit_select_arma_ml_kf_f32(*head, *tail, ptr("se"), ld_se, None)
    else:
        rc = lib.mmf_fit_select_arma_ml_f32(*head, *tail, None)
    assert rc == 0, lib.mmf_last_error()
    torch.cuda.synchronize()
    res = _np(out)
    if not kf:
        del res["se"]
    else:
        res["se"] = res["se"][:, :npred]
    return res


def _fixed(eng, yd, t_fit, p, d, q, m, ps, npred, kf, max_iter=0):
    kw = dict(predictor="kalman", want_se=True) if kf else {}
    return _np(eng.fit_forecast_arma(yd[:, :t_fit], p, q, d, ps, npred, long_order=m, estimator="ml",
                                     max_iter=max_iter, **kw))


def _se_of(eng, yd, t_fit, got, ps, npred):
    """mmf_arima_se_f32 of the call's outputs with the per-series d"""
    r = {k: torch.from_numpy(np.ascontiguousarray(got[k])).cuda() for k in ("phi", "order", "theta", "ma_order", "sigma")}
    eng._add_se(r, yd, t_fit, ps, npred, 0, diffs=torch.from_numpy(got["choice_d"]).cuda())
    return r["se"].cpu().numpy()


def _check(eng, yd, t_fit, orders, diffs, mas, ps, npred, kf, max_iter=0, what="", count_only=False):
    """the refit call against the selection and the fixed-order calls, class by class.  Returns (refit rows, rows that
    differ from their fixed-order call); with count_only the q >= 1 classes are counted instead of asserted"""
    got = _refit(eng, yd, orders, diffs, mas, ps, npred, kf, max_iter)
    sel = _call(eng, yd, orders, diffs, mas, ps, npred)
    m_of = dict(zip(diffs, _ms(t_fit, orders, diffs, mas)))
    n = yd.shape[0]
    for k in SEL_OUT:
        assert (_bits(got[k]) == _bits(sel[k])).all(), (what, k)
    cp, cd, cq = got["choice_p"], got["choice_d"], got["choice_q"]
    refit = cq >= 1
    kept = ~refit
    for k in KEPT_OUT:                                    # q = 0 winners, no eligible candidate
        same = (_bits(got[k]) == _bits(sel[k])).reshape(n, -1).all(axis=1)
        assert same[kept].all(), (what, k, np.flatnonzero(kept & ~same)[:8])
    assert np.isnan(got["loglik_start"][kept]).all() and np.isnan(got["loglik"][kept]).all(), what
    assert (got["ml_stop"][kept] == 0).all() and (got["iters"][kept] == 0).all(), what
    if kf:
        want_se = _se_of(eng, yd, t_fit, got, ps, npred)
        assert (_bits(got["se"][kept]) == _bits(want_se[kept])).all(), (what, "se of the kept rows")
    bad = 0
    for p, d, q in sorted(set(zip(cp[refit].tolist(), cd[refit].tolist(), cq[refit].tolist()))):
        s = (cp == p) & (cd == d) & (cq == q)
        want = _fixed(eng, yd, t_fit, p, d, q, m_of[d], ps, npred, kf, max_iter)
        differ = np.zeros(n, dtype=bool)
        for k in FIX_OUT + (("se",) if kf else ()):
            differ |= ~(_bits(got[k]) == _bits(want[k])).reshape(n, -1).all(axis=1)
        if not count_only:
            assert not differ[s].any(), (what, (p, d, q), np.flatnonzero(s & differ)[:8])
        bad += int((s & differ).sum())
    return int(refit.sum()), bad


@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_winners_bit_equal_to_the_fixed_order_calls(cal):
    """every (p, d, q >= 1) class equals the fixed-order ML and ML + Kalman calls at m_d, bit for bit (se included), in
    the holdout and a mid-design window: the case's own gaps under auto / tc / warp, 1e-3 extra gaps under auto and
    15 % under warp"""
    t0 = time.time()
    y, X, t_fit, has_c = _ma_case(cal)
    rows = refit_rows = 0
    for gaps, kernels in (("case", ("auto", "tc", "warp")), ("1e-3", ("auto",)), ("heavy", ("warp",))):
        yy = y if gaps == "case" else _gapped(y, t_fit, 1e-3 if gaps == "1e-3" else 0.15, seed={"1e-3": 1, "heavy": 2}[gaps])
        _, yd = _device(yy)
        for kernel in kernels:
            eng = _engine(kernel, X, t_fit, has_c)
            n_rows = X.shape[0]
            for name, (ps, npred) in {"holdout": (0, n_rows), "mid": (t_fit // 3, t_fit // 2 + 20)}.items():
                for kf in (False, True):
                    r, bad = _check(eng, yd, t_fit, *REF, ps, npred, kf, what=f"{cal} {gaps} {kernel} {name} {kf}")
                    assert bad == 0
                    rows += len(y)
                    refit_rows += r
            eng.close()
    assert refit_rows > 0, cal
    record_err("arma_select_ml refit rows", float(refit_rows), float(rows), what=cal, seconds=time.time() - t0)


def test_assume_finite_and_max_iter():
    """gap-free rows under assume_finite, and max_iter 1 / 20: still the fixed-order calls' bits"""
    y, X, t_fit, has_c = _ma_case("daily")
    ok = np.isfinite(y).all(axis=1)
    _, yd = _device(np.ascontiguousarray(y[ok]))
    eng = mmf.ForecastEngine(assume_finite=True)
    eng.plan(X, t_fit, has_c)
    eng.plan_arima(X, t_fit, 2)
    refit = 0
    for kf in (False, True):
        for max_iter in (0, 1, 20):
            r, _ = _check(eng, yd, t_fit, *REF, 0, X.shape[0], kf, max_iter, what=f"finite {kf} {max_iter}")
            refit += r
    assert refit > 0
    eng.close()


@pytest.mark.parametrize("kf", [False, True])
def test_null_outputs_leave_the_others_unchanged(kf):
    """each nullable output NULL alone, and all of them together: the other outputs bit-equal to the full call (the
    winner's phi, theta, orders, sigma and choices then come from scratch); a wide ld_se writes columns [0, n_pred)"""
    y, X, t_fit, has_c = _ma_case("daily")
    _, yd = _device(y)
    eng = _engine("auto", X, t_fit, has_c)
    args = (eng, yd, *REF, 0, X.shape[0], kf)
    full = _refit(*args)
    assert (full["choice_q"] > 0).any() and (full["ml_stop"] > 0).any()
    names = [k for k in NULLABLE if kf or k != "se"]
    for null in [(k,) for k in names] + [tuple(names), tuple(k for k in names if k != "se")]:
        got = _refit(*args, null=null)
        for k in full:
            if k not in null:
                assert (_bits(got[k]) == _bits(full[k])).all(), (null, k)
            else:
                assert (_bits(got[k]) == _bits(np.full_like(got[k], SENT_F if got[k].dtype == np.float32
                                                            else SENT_I))).all(), (null, k)
    if kf:
        wide = _refit(*args, ld_se=X.shape[0] + 5)
        for k in full:
            assert (_bits(wide[k]) == _bits(full[k])).all(), ("wide ld_se", k)
    eng.close()


def test_slabs_are_bit_equal_to_smaller_batches():
    """2^20 + 1,001 rows (two slabs) against the same rows in two smaller calls, ML and ML + Kalman with se"""
    n, t = (1 << 20) + 1001, 48
    from oracle import mmf_oracle as O
    y, start = mmf.synth.daily_store_item_demand(n, t + 8, seed=9, nan_frac=0.01)
    X = O.design_matrix(O.calendar_grid(start, t + 8, "D"), t)
    eng = _engine("auto", X, t, True)
    yd = torch.from_numpy(y).cuda()
    for kw in (dict(refit="ml"), dict(refit="ml", predictor="kalman", want_se=True)):
        whole = eng.fit_select_arma(yd, 8, *SMALL, t, 8, max_iter=5, **kw)
        assert (whole["choice_q"] > 0).any() and (whole["ml_stop"] > 0).any()
        for lo, hi in ((0, 1 << 19), (1 << 19, n)):
            part = eng.fit_select_arma(yd[lo:hi], 8, *SMALL, t, 8, max_iter=5, **kw)
            for k in whole:
                assert _same_bits(whole[k][lo:hi], part[k]), (kw, k)
        del whole
    eng.close()


def test_shared_context_matches_a_fresh_one_across_streams():
    y, X, t_fit, has_c = _ma_case("weekly")
    _, yd = _device(y)
    npred = X.shape[0]
    kws = (dict(refit="ml"), dict(refit="ml", predictor="kalman", want_se=True), dict(refit="ml", predictor="kalman"))

    def run(eng):
        return [_np(eng.fit_select_arma(yd, N_HOLD, *REF, 0, npred, **kw)) for kw in kws]

    fresh = _engine("auto", X, t_fit, has_c)
    want = run(fresh)
    fresh.close()
    eng = _engine("auto", X, t_fit, has_c)
    got = [run(eng)]
    eng.fit_forecast_arma(yd[:, :t_fit], 2, 1, 1, 0, npred, estimator="ml", predictor="kalman", want_se=True)
    eng.fit_select_arma(yd, N_HOLD, *REF, 0, npred, refit="css")
    eng.fit_forecast_arma(yd[:, :t_fit], 1, 2, 0, 0, npred, estimator="css", joint_beta=True)
    eng.fit_select_arima(yd, N_HOLD, (0, 1, 2), (0, 1, 2), 0, npred)
    got.append(run(eng))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got.append(run(eng))
    s.synchronize()
    for g in got:
        for j in range(len(kws)):
            for k in want[j]:
                assert (_bits(g[j][k]) == _bits(want[j][k])).all(), (j, k)
    eng.close()


def test_want_se_with_the_recursion_is_the_fixed_order_calls():
    """refit="ml" with the recursion and want_se: per (p, d, q >= 1) class the fixed-order ML call's se, q = 0 rows the
    selection's"""
    y, X, t_fit, has_c = _ma_case("daily")
    _, yd = _device(y)
    eng = _engine("auto", X, t_fit, has_c)
    npred = X.shape[0]
    ms = dict(zip(REF[1], _ms(t_fit, *REF)))
    got = _np(eng.fit_select_arma(yd, N_HOLD, *REF, 0, npred, want_se=True, refit="ml"))
    sel = _np(eng.fit_select_arma(yd, N_HOLD, *REF, 0, npred, want_se=True))
    cp, cd, cq = got["choice_p"], got["choice_d"], got["choice_q"]
    kept = cq < 1
    assert (_bits(got["se"][kept]) == _bits(sel["se"][kept])).all()
    for p, d, q in set(zip(cp[~kept].tolist(), cd[~kept].tolist(), cq[~kept].tolist())):
        s = (cp == p) & (cd == d) & (cq == q)
        want = _np(eng.fit_forecast_arma(yd[:, :t_fit], p, q, d, 0, npred, long_order=ms[d], want_se=True,
                                         estimator="ml"))
        assert (_bits(got["se"][s]) == _bits(want["se"][s])).all(), (p, d, q)
    eng.close()


def test_refused_calls_write_nothing():
    """max_iter outside [0, 64] is checked first; ld_se < n_pred with out_se is refused; every other refusal is the
    selection's, with its code and text"""
    y, X, t_fit, has_c = _ma_case("daily", n=40)
    _, yd = _device(y)
    eng = _engine("auto", X, t_fit, has_c)
    lib = eng._lib
    cases = [dict(max_iter=-1), dict(max_iter=65), dict(mas=(1, 2)), dict(orders=(2, 1)), dict(n_hold=0),
             dict(max_iter=65, mas=(1,)), dict(ld_se=15)]
    for kf in (False, True):
        for c in cases:
            if "ld_se" in c and not kf:
                continue
            orders, diffs, mas = c.get("orders", (0, 1)), (0, 1), c.get("mas", (0, 1))
            n_hold = c.get("n_hold", N_HOLD)
            out = torch.full((len(y), 16), SENT_F, device="cuda")
            ll = torch.full((len(y),), SENT_F, device="cuda")
            se = torch.full((len(y), 16), SENT_F, device="cuda")
            arr = lambda v: (ctypes.c_int32 * len(v))(*v)
            head = (eng._h, yd.data_ptr(), len(y), yd.stride(0), n_hold, arr(orders), len(orders), arr(diffs), 2,
                    arr(mas), len(mas), 0)
            nulls = [None] * 11
            if kf:
                rc = lib.mmf_fit_select_arma_ml_kf_f32(*head, c.get("max_iter", 0), t_fit, 16, out.data_ptr(), 16,
                                                       *nulls, ll.data_ptr(), None, None, None, se.data_ptr(),
                                                       c.get("ld_se", 16), None)
            else:
                rc = lib.mmf_fit_select_arma_ml_f32(*head, c.get("max_iter", 0), t_fit, 16, out.data_ptr(), 16,
                                                    *nulls, ll.data_ptr(), None, None, None, None)
            msg = lib.mmf_last_error().decode()
            if "max_iter" in c:
                assert rc == -1 and msg == f"max_iter={c['max_iter']} outside [0,64]", (c, msg)
            elif "ld_se" in c:
                assert rc == -1 and msg == "ld_se=15 < n_pred=16", (c, msg)
            else:
                rc_sel = lib.mmf_fit_select_arma_f32(*head, t_fit, 16, out.data_ptr(), 16, *nulls, None)
                assert rc == rc_sel and rc != 0 and msg == lib.mmf_last_error().decode(), (c, msg)
            torch.cuda.synchronize()
            assert (out == SENT_F).all() and (ll == SENT_F).all() and (se == SENT_F).all(), c
    eng.close()


_NEGCTL = r"""
import json, sys
sys.path[:0] = [{root!r}, {tests!r}]
import mmf
from test_gpu_arma_select import REF, _ma_case
from test_gpu_arima_select import _device, _engine
from test_gpu_arma_select_ml import _check
y, X, t_fit, has_c = _ma_case("daily")
_, yd = _device(y)
eng = _engine("auto", X, t_fit, has_c)
rows = bad = 0
for kf in (False, True):
    r, b = _check(eng, yd, t_fit, *REF, 0, X.shape[0], kf, count_only=True)
    rows, bad = rows + r, bad + b
print(json.dumps({{"rows": rows, "bad": bad, "lib": mmf.LIB_PATH}}))
"""


@pytest.mark.parametrize("lib", ["product", "callorders"])
def test_negative_control_refitting_at_the_call_orders(lib):
    """the build whose ML and Kalman list kernels take the call's largest listed (p, q) for every listed row
    (tests/_build/libmmf_armaselml_callorders.so) must differ from the fixed-order calls on most refit rows; the
    product on none"""
    env = dict(os.environ)
    env.pop("MMF_LIB", None)
    if lib == "callorders":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_armaselml_callorders.so")
        assert os.path.exists(env["MMF_LIB"]), "negative-control library missing: run __graft_entry__.build()"
    r = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tests=os.path.join(ROOT, "tests"))], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    record_err("test_gpu_arma_select_ml negative control", float(got["bad"]), float(got["rows"]), what=lib)
    assert got["rows"] > 0, got
    if lib == "product":
        assert got["bad"] == 0, got
    else:
        assert got["lib"].endswith("libmmf_armaselml_callorders.so") and got["bad"] >= got["rows"] // 2, got


def test_forecast_groups_with_the_ml_refit_and_the_kalman_predictor():
    """refit="ml" (and predictor="kalman") through the frame layer on the reference's weekly frame: the selection's
    schema, conf_int bands around the refit's values, and forecast_table's values"""
    import pyarrow as pa
    pdf = mmf.synth.reference_weekly_demand(4)
    kw = dict(freq="W-MON", horizon=40, mode="holdout", ar=REF[0], diff=REF[1], ma=REF[2])
    sel = mmf.forecast_groups(pdf, **kw)
    for extra in (dict(refit="ml"), dict(refit="ml", predictor="kalman")):
        out = mmf.forecast_groups(pdf, **extra, **kw)
        assert list(out.columns) == list(sel.columns) and len(out) == len(sel)
        a, b = out["Demand_Fitted"].to_numpy(), sel["Demand_Fitted"].to_numpy()
        assert (np.isnan(a) == np.isnan(b)).all() and (a[~np.isnan(a)] != b[~np.isnan(b)]).any(), extra
        band = mmf.forecast_groups(pdf, conf_int=0.9, **extra, **kw)
        assert np.array_equal(band["Demand_Fitted"].to_numpy(), a, equal_nan=True), extra
        ok = ~np.isnan(a)
        lo, hi = band["Demand_Lower"].to_numpy()[ok], band["Demand_Upper"].to_numpy()[ok]
        assert (lo <= a[ok]).all() and (a[ok] <= hi).all(), extra
        tab = mmf.forecast_table(pa.Table.from_pandas(pdf, preserve_index=False), **extra, **kw)
        t = np.sort(tab.column("Demand_Fitted").to_numpy(zero_copy_only=False).astype(np.float32))
        assert np.array_equal(t, np.sort(a), equal_nan=True), extra
