"""GPU: mmf_fit_forecast_arma_joint_f32 (DESIGN.md section 2 item 17) against the CSS call, the HR call, the plain fit and
the float64 joint oracle.

With J empty (the fit_zero design of tests/test_gpu_arma_css_replay.py) every output is the CSS call's bit for bit.  On
any design: css_start is the CSS call's bit for bit, rows that fail the gate, empty rows and max_iter = 1 rows are the
HR call's (sigma of the gated ones excepted), and d = 0 rows that kept the fit's gamma have mmf_fit_forecast_f32's
out_beta bit for bit.  Against the oracle, at the GPU's (beta, phi, theta): S within css_bound of the GPU's S, converged
rows within OPT_RTOL + 2 css_bound / S of SciPy's joint optimum, predictions within a relative fp32 bound."""
import numpy as np
import pytest
import torch

import mmf
import arma_css_oracle as S
import arma_joint_oracle as JO
from arima_oracle import z_tau
from arima_se_oracle import arima_se
from arma_oracle import _integrate, fit_forecast_arma_packed, recursion
from conftest import record_err
from oracle import mmf_oracle as O
from test_arma_css_oracle import OPT_RTOL
from test_arma_joint_oracle import BETA_TRUE, joint_rows
from test_gpu_abi_contract import PATTERN
from test_gpu_arima import _dev, _np, _windows
from test_gpu_arma import _arma_case, _engines
from test_gpu_arma_css_replay import NPRED, _design, _gaps, _levels
from test_gpu_edges import _le, _same_bits

pytestmark = pytest.mark.gpu

SHARED = ("pred", "phi", "theta", "order", "ma_order", "sigma", "status")
CSS_OUT = SHARED + ("css_start", "css", "css_stop", "iters")


def _joint(eng, yd, p, q, d, ps, npred, m=0, max_iter=0, **kw):
    return _np(eng.fit_forecast_arma(yd, p, q, d, ps, npred, long_order=m, estimator="css", max_iter=max_iter,
                                     joint_beta=True, **kw))


def _css(eng, yd, p, q, d, ps, npred, m=0, max_iter=0):
    return _np(eng.fit_forecast_arma(yd, p, q, d, ps, npred, long_order=m, estimator="css", max_iter=max_iter))


def _hr(eng, yd, p, q, d, ps, npred):
    return _np(eng.fit_forecast_arma(yd, p, q, d, ps, npred))


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


@pytest.fixture(scope="module")
def zero_engine():
    t_fit = 157
    eng = mmf.ForecastEngine()
    X = _design(t_fit)
    eng.plan(X, t_fit, False)
    eng.plan_arima(X, t_fit, 2)
    yield eng, t_fit
    eng.close()


@pytest.mark.parametrize("d", [0, 1, 2])
@pytest.mark.parametrize("p", [0, 1, 2, 8])
def test_identity_route_equals_the_css_call(zero_engine, p, d):
    """J empty: every output the CSS call's bit for bit, q = 1..4, the replay's gap patterns; beta 0 on every non-empty
    row (gamma = 0, no constant), NaN on empty rows"""
    eng, t_fit = zero_engine
    for q in (1, 2, 3, 4):
        y = _gaps(_levels(p, q, d, 20, t_fit, seed=8000 + 100 * p + 10 * q + d), "mix", seed=p * 7 + q, p=p)
        y[7] = np.nan                                   # one empty row
        yd = _dev(y.astype(np.float32))
        got = _joint(eng, yd, p, q, d, t_fit, NPRED)
        want = _css(eng, yd, p, q, d, t_fit, NPRED)
        for k in CSS_OUT:
            assert _bits(got[k]) == _bits(want[k]), (p, q, d, k)
        empty = got["status"] == 1
        assert empty[7] and np.isnan(got["beta"][empty]).all() and (got["beta"][~empty] == 0).all(), (p, q, d)
        assert (got["css_stop"] > 0).sum() >= 1, (p, q, d)


def _oracle_check(got, y, X, t_fit, p, q, d, what, n_opt=3):
    """S at the GPU's (beta, phi, theta) within css_bound of the GPU's S; SciPy's joint optimum on the first n_opt
    converged rows; predictions at the GPU's parameters -> worst ratio"""
    want = fit_forecast_arma_packed(y, X, t_fit, 0, X.shape[0], p, q, d)
    z, Dm, W, kept, Af, g0 = JO.plan_of(y, X, t_fit, d)
    T = t_fit - d
    zt = {"z": want["base"]["z"]} if d >= 1 else {"z": np.where(np.isfinite(y), y, np.nan)[:, :t_fit]}
    tau = z_tau(zt)
    refined = (got["css_stop"] > 0) & want["gated"] & (got["status"] == 0)
    worst, left = 0.0, n_opt
    endz = X.shape[0] - d
    for i in np.flatnonzero(refined):
        obs = np.isfinite(z[i, :T])
        b = got["beta"][i, :Dm.shape[1]].astype(np.float64)     # a caller design may have fewer than 16 columns
        x = np.r_[got["phi"][i, :p], got["theta"][i, :q]].astype(np.float64)
        none = np.zeros(0, dtype=np.int64)
        Sg, _, eps, C = JO.joint_eval(z[i], obs, Dm[:T], T, p, q, x, b, none)
        e = JO.residuals(z[i], obs, Dm[:T], b)
        bound = S.css_bound(e, obs, T, p, q, x, tau[i])
        w = abs(Sg - float(got["css"][i])) / bound
        _le(w, 1.0, f"{what} row {i}: |S_oracle(gpu x) - css| / css_bound")
        worst = max(worst, w)
        if got["css_stop"][i] == 1 and left > 0:
            left -= 1
            cols = JO.used_cols(Dm[:T], obs, kept)
            gap = JO.optimality_gap(z[i], obs, Dm[:T], T, p, q, np.r_[x, b[cols]], b, cols)
            _le(gap, OPT_RTOL + 2 * bound / Sg, f"{what} row {i}: joint optimality gap")
        # predictions: X beta + the recursion at the GPU's (phi, theta), integrated to levels
        pr, _, _ = recursion(e, obs, T, x[:p], x[p:], endz)
        zh = np.full(X.shape[0], np.nan)
        zh[d:] = Dm[:endz] @ b + pr
        if d == 0:
            yh = zh
        else:
            yl = np.asarray(y, np.float64)[i:i + 1, :t_fit]
            yh = _integrate(zh[None], yl, np.isfinite(yl), t_fit, d, X.shape[0])[0][0]
        scale = np.nanmax(np.abs(y[i, :t_fit])) + 1.0
        fin = np.isfinite(yh)
        err = np.abs(got["pred"][i][fin] - yh[fin]) / (1e-4 * (np.abs(yh[fin]) + scale) + 8 * np.sqrt(bound / C.sum()))
        _le(float(err.max()), 1.0, f"{what} row {i}: prediction at the GPU's parameters")
    return worst, int(refined.sum())


@pytest.mark.parametrize("d", [0, 1, 2])
@pytest.mark.parametrize("p,q", [(0, 1), (1, 1), (2, 2), (8, 4)])
@pytest.mark.parametrize("cal", ["daily", "weekly", "exog_only", "caller"])
def test_joint_on_any_design(cal, p, q, d):
    """css_start the CSS call's; fallback / empty rows the HR call's; d = 0 rows that kept the fit's gamma have the plain
    fit's out_beta; css <= css_start; the oracle at the GPU's parameters; every window a slice of the holdout rows"""
    y, X, t_fit, has_c = _arma_case(cal, n=48)
    engs = _engines(X, t_fit, has_c)
    yd = _dev(y, t_fit + 1)
    n_rows = X.shape[0]
    worst, refined = 0.0, 0
    for k, eng in engs.items():
        what = f"{cal} p={p} q={q} d={d} {k}"
        got = _joint(eng, yd[:, :t_fit], p, q, d, 0, n_rows)
        css = _css(eng, yd[:, :t_fit], p, q, d, 0, n_rows)
        hr = _hr(eng, yd[:, :t_fit], p, q, d, 0, n_rows)
        gated = hr["ma_order"] > 0
        assert np.array_equal(got["css_stop"] > 0, gated), what
        assert _bits(got["css_start"]) == _bits(css["css_start"]), what
        for key in SHARED:
            assert _bits(got[key][~gated]) == _bits(hr[key][~gated]), (what, key)
        assert (got["css"][gated] <= got["css_start"][gated]).all(), what
        empty = got["status"] == 1
        assert np.isnan(got["beta"][empty]).all() and np.isfinite(got["beta"][~empty]).all(), what
        if d == 0:
            plain = eng.fit_forecast(yd[:, :t_fit], 0, n_rows, want_beta=True)["beta"].cpu().numpy()
            kept_hr = (got["phi"] == hr["phi"]).all(1) & (got["theta"] == hr["theta"]).all(1)
            same_beta = (got["beta"] == plain).all(1) | empty
            assert same_beta[~gated].all(), what
            rows = kept_hr & same_beta          # no step accepted: every output the HR call's but sigma
            for key in SHARED:
                if key != "sigma":
                    assert _bits(got[key][rows]) == _bits(hr[key][rows]), (what, key)
        if k == "auto":
            w, r = _oracle_check(got, y, X, t_fit, p, q, d, what)
            worst, refined = max(worst, w), r
            for name, (ps, npred) in _windows(t_fit, n_rows).items():
                win = _joint(eng, yd[:, :t_fit], p, q, d, ps, npred)
                hw = _hr(eng, yd[:, :t_fit], p, q, d, ps, npred)
                for key in win:
                    ref = got[key][:, ps:ps + npred] if key == "pred" else got[key]
                    if key == "pred":
                        ref = np.where(gated[:, None], ref, hw["pred"])
                    assert _bits(win[key]) == _bits(ref), (what, name, key)
    for e in engs.values():
        e.close()
    record_err("test_joint_on_any_design", worst, 1.0, what=f"{cal} p={p} q={q} d={d}", refined=refined)


def test_dummy_beta_rmse_on_the_gpu():
    """2,400 rows of 157 weekly rows with ARMA(1, 1) errors (0.8, 0.4): the dummies' beta RMSE <= 0.6 x OLS's"""
    y, X = joint_rows(2400, 157, [0.8], [0.4], 21)
    eng = mmf.ForecastEngine()
    eng.plan(X, 157, True)
    yd = _dev(y)
    got = _joint(eng, yd, 1, 1, 0, 157, 8, max_iter=64)
    ols = eng.fit_forecast(yd, 157, 8, want_beta=True)["beta"].cpu().numpy()
    g = got["ma_order"] > 0
    assert g.sum() >= 2000
    ratios = [np.sqrt(np.mean((got["beta"][g, k] - BETA_TRUE[k]) ** 2)) /
              np.sqrt(np.mean((ols[g, k] - BETA_TRUE[k]) ** 2)) for k in (2, 3)]
    record_err("test_dummy_beta_rmse_on_the_gpu", max(ratios), 0.6, what=f"ratios {ratios[0]:.3f} {ratios[1]:.3f}",
               stops=np.bincount(got["css_stop"][g], minlength=4).tolist())
    assert max(ratios) <= 0.6, ratios
    eng.close()


def test_y_beyond_t_fit_never_read_and_power_of_two_scaling():
    y, X, t_fit, _ = _arma_case("daily")
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, True)
    eng.plan_arima(X, t_fit, 2)
    base = _dev(y, t_fit + 40)
    for d in (0, 1, 2):
        ref = _joint(eng, base[:, :t_fit], 1, 1, d, 0, X.shape[0])
        assert (ref["css_stop"] > 0).any()
        for fill in (float("nan"), 1e30, -7.0):
            yd = _dev(y, t_fit + 40)
            yd[:, t_fit:] = fill
            got = _joint(eng, yd, 1, 1, d, 0, X.shape[0])
            for k in ref:
                assert _bits(got[k]) == _bits(ref[k]), (fill, d, k)
        a = _joint(eng, base[:, :t_fit], 2, 1, d, t_fit, 28)
        b = _joint(eng, base[:, :t_fit] * 8.0, 2, 1, d, t_fit, 28)
        for k, f in (("pred", 8.0), ("phi", 1.0), ("theta", 1.0), ("order", 1), ("ma_order", 1), ("sigma", 8.0),
                     ("status", 1), ("css", 64.0), ("css_start", 64.0), ("css_stop", 1), ("iters", 1), ("beta", 8.0)):
            w = a[k] * f
            assert ((b[k] == w) | (np.isnan(b[k]) & np.isnan(w))).all(), (d, k)
    eng.close()


def test_slabs_are_bit_equal_to_per_slab_calls():
    n, t = (1 << 20) + 1001, 48
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=9, nan_frac=0.01)
    X = O.design_matrix(O.calendar_grid(start, t + 8, "D"), t)
    eng = mmf.ForecastEngine()
    eng.plan(X, t, True)
    eng.plan_arima(X, t, 2)
    yd = torch.from_numpy(y).cuda()
    for d in (0, 2):
        whole = eng.fit_forecast_arma(yd, 1, 1, d, t, 8, estimator="css", joint_beta=True)
        assert (whole["iters"] > 1).any()
        for lo, hi in ((0, 1 << 19), (1 << 19, n)):
            part = eng.fit_forecast_arma(yd[lo:hi], 1, 1, d, t, 8, estimator="css", joint_beta=True)
            for k in CSS_OUT + ("beta",):
                assert _same_bits(whole[k][lo:hi], part[k]), (d, k)
    eng.close()


def test_nullable_outputs_wide_table_max_iter_and_refusals():
    y, X, t_fit, _ = _arma_case("daily", n=40)
    n = len(y)
    eng = mmf.ForecastEngine()
    lib, h = eng._lib, eng._h
    eng.plan(X, t_fit, True)
    eng.plan_arima(X, t_fit, 1)
    yd = _dev(y)
    keys = ("beta", "phi", "theta", "order", "ma_order", "sigma", "status", "css_start", "css", "css_stop", "iters")
    for d in (0, 1):
        ref = eng.fit_forecast_arma(yd, 1, 1, d, t_fit, 28, estimator="css", joint_beta=True)
        wide = torch.full((n, 41), float(np.float32(PATTERN)), device="cuda")
        view = wide[:, 5:33]
        assert lib.mmf_fit_forecast_arma_joint_f32(h, yd.data_ptr(), n, yd.stride(0), 1, d, 1, 0, 0, t_fit, 28,
                                                   view.data_ptr(), 41, *(None,) * 12) == 0
        torch.cuda.synchronize()
        assert _same_bits(view, ref["pred"])
        assert (wide[:, :5] == float(np.float32(PATTERN))).all() and (wide[:, 33:] == float(np.float32(PATTERN))).all()
        for j, key in enumerate(keys):
            bufs = [None] * 11
            t_ = torch.empty_like(ref[key])
            bufs[j] = t_.data_ptr()
            out = torch.empty((n, 28), device="cuda")
            assert lib.mmf_fit_forecast_arma_joint_f32(h, yd.data_ptr(), n, yd.stride(0), 1, d, 1, 0, 0, t_fit, 28,
                                                       out.data_ptr(), 28, *bufs, None) == 0
            torch.cuda.synchronize()
            assert _same_bits(out, ref["pred"]) and _same_bits(t_, ref[key]), (d, key)
    # max_iter 1: one pass, no step: every shared output the HR call's but sigma, beta the plain fit's
    one = _joint(eng, yd, 1, 1, 0, t_fit, 28, max_iter=1)
    hr = _hr(eng, yd, 1, 1, 0, t_fit, 28)
    plain = eng.fit_forecast(yd, t_fit, 28, want_beta=True)["beta"].cpu().numpy()
    g = hr["ma_order"] > 0
    assert (one["iters"][g] == 1).all() and (one["css_stop"][g] == 3).all()
    assert (one["css"][g] == one["css_start"][g]).all()
    for k in SHARED:
        if k != "sigma":
            assert _bits(one[k]) == _bits(hr[k]), k
    assert _bits(one["beta"]) == _bits(plain)
    big = _joint(eng, yd, 1, 1, 0, t_fit, 28, max_iter=64)
    dflt = _joint(eng, yd, 1, 1, 0, t_fit, 28)
    assert (big["iters"] <= 64).all() and (dflt["iters"] <= 20).all()
    assert (big["css"][g] <= dflt["css"][g]).all()
    assert ((big["iters"] == dflt["iters"]) | (dflt["css_stop"] == 3)).all()
    # refusals: the code and the full message of each check; refused calls write nothing
    out = torch.full((n, 28), 7.0, device="cuda")
    cs = torch.full((n,), 7.0, device="cuda")
    bt = torch.full((n, 16), 7.0, device="cuda")
    host_out = np.zeros((n, 28), dtype=np.float32)
    host_beta = np.zeros((n, 16), dtype=np.float32)
    name = "mmf_fit_forecast_arma_joint_f32"
    table = [
        ((1, 0, 1, 0, -1), (t_fit, 28, out.data_ptr(), 28, bt.data_ptr()), -1, "max_iter=-1 outside [0,64]"),
        ((1, 0, 1, 0, 65), (t_fit, 28, out.data_ptr(), 28, bt.data_ptr()), -1, "max_iter=65 outside [0,64]"),
        ((1, 0, 0, 0, 0), (t_fit, 28, out.data_ptr(), 28, bt.data_ptr()), -1, "ma_order=0 outside [1,4]"),
        ((1, 3, 1, 0, 0), (t_fit, 28, out.data_ptr(), 28, bt.data_ptr()), -1, "diff_order=3 outside [0,2]"),
        ((9, 0, 1, 0, 0), (t_fit, 28, out.data_ptr(), 28, bt.data_ptr()), -1, "ar_order=9 outside [0,8]"),
        ((1, 0, 1, 33, 0), (t_fit, 28, out.data_ptr(), 28, bt.data_ptr()), -1, "long_order=33 outside {0} and [1,32]"),
        ((1, 2, 1, 0, 0), (t_fit, 28, out.data_ptr(), 28, bt.data_ptr()), -1,
         "diff_order=2 above the planned max_diff=1"),
        ((1, 0, 1, 0, 0), (t_fit, 28, host_out.ctypes.data, 28, bt.data_ptr()), -3, f"{name} takes device buffers only"),
        ((1, 0, 1, 0, 0), (t_fit, 28, out.data_ptr(), 28, host_beta.ctypes.data), -3,
         f"{name} takes device buffers only"),
    ]
    for (p, d, q, m, mi), (ps, npred, o, ld, b), code, msg in table:
        rc = lib.mmf_fit_forecast_arma_joint_f32(h, yd.data_ptr(), n, yd.stride(0), p, d, q, m, mi, ps, npred, o, ld,
                                                 b, *(None,) * 7, cs.data_ptr(), None, None, None)
        err = lib.mmf_last_error().decode()
        assert rc == code and err == msg, (p, d, q, m, mi, rc, err)
    rc = lib.mmf_fit_forecast_arma_joint_f32(h, yd.data_ptr(), n, yd.stride(0), 1, 0, 1, 0, 0, t_fit, 28,
                                             out.data_ptr(), 27, bt.data_ptr(), *(None,) * 7, cs.data_ptr(), None,
                                             None, None)
    assert rc != 0
    torch.cuda.synchronize()
    assert (out == 7.0).all() and (cs == 7.0).all() and (bt == 7.0).all() and not host_out.any()
    assert not host_beta.any()
    with pytest.raises(ValueError, match="joint_beta=True needs estimator='css'"):
        eng.fit_forecast_arma(yd, 1, 1, 0, t_fit, 28, joint_beta=True)
    eng.close()


def test_other_calls_unchanged_a_shared_context_matches_a_fresh_one_and_a_second_stream():
    y, X, t_fit, has_c = _arma_case("daily")
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    eng.plan_arima(X, t_fit, 2)
    yd = _dev(y, t_fit + 28)
    yf = yd[:, :t_fit]

    def calls():
        return (eng.fit_forecast(yf, t_fit, 28).clone(), eng.fit_forecast_ar(yf, 2, t_fit, 28)["pred"].clone(),
                eng.fit_forecast_arima(yf, 2, 1, t_fit, 28)["pred"].clone(),
                eng.fit_forecast_arma(yf, 1, 1, 1, t_fit, 28)["pred"].clone(),
                eng.fit_forecast_arma(yf, 1, 1, 1, t_fit, 28, estimator="css")["pred"].clone(),
                eng.fit_select_arma(yd, 28, (0, 1), (0, 1), (0, 1), t_fit, 28)["pred"].clone())

    args = ((1, 1, 0, t_fit, 28, 0), (8, 4, 2, 0, t_fit + 64, 32), (0, 2, 1, 50, 100, 2))
    before = calls()
    shared = [_joint(eng, yf, p, q, d, ps, npred, m) for p, q, d, ps, npred, m in args]
    after = calls()
    assert all(_same_bits(a, b) for a, b in zip(before, after))
    fresh = mmf.ForecastEngine()
    fresh.plan(X, t_fit, has_c)
    fresh.plan_arima(X, t_fit, 2)
    for (p, q, d, ps, npred, m), a in zip(args, shared):
        b = _joint(fresh, yf, p, q, d, ps, npred, m)
        for k in a:
            assert _bits(a[k]) == _bits(b[k]), (p, q, d, k)
    s2 = torch.cuda.Stream()
    with torch.cuda.stream(s2):
        c = _joint(eng, yf, 1, 1, 0, t_fit, 28)
    a = _joint(eng, yf, 1, 1, 0, t_fit, 28)
    for k in a:
        assert _bits(a[k]) == _bits(c[k]), k
    eng.close()
    fresh.close()


@pytest.mark.parametrize("d", [0, 1, 2])
def test_standard_errors_take_the_joint_estimate(d):
    y, X, t_fit, has_c = _arma_case("weekly")
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    eng.plan_arima(X, t_fit, 2)
    yd = _dev(y, t_fit)
    res = _joint(eng, yd, 1, 1, d, 0, X.shape[0], want_se=True)
    want = arima_se(y, t_fit, res["phi"], res["order"], res["sigma"], 0, X.shape[0], d, theta=res["theta"],
                    ma_order=res["ma_order"])
    fin = np.isfinite(want)
    assert np.array_equal(fin, np.isfinite(res["se"]))
    ulp = np.abs(res["se"][fin].astype(np.float64) - want[fin]) / np.spacing(np.abs(want[fin]).astype(np.float32))
    _le(float(ulp.max()), 4.0, f"d={d}: se ulp")
    eng.close()


@pytest.mark.parametrize("name", ["daily1095", "weekly157"])
def test_demand_shapes_are_hr_rows_or_lower_css(name):
    from demand_shapes import calendar, demand_batch
    start, t, freq, _ = calendar(name)
    t_fit = t - 28
    y, kinds, _ = demand_batch(150, name, seed=11, t_fit=t_fit)
    X = O.design_matrix(O.calendar_grid(start, t, freq), t_fit)
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, True)
    eng.plan_arima(X, t_fit, 2)
    yd = _dev(y)
    for d in (0, 1, 2):
        got = _joint(eng, yd[:, :t_fit], 1, 1, d, 0, X.shape[0])
        hr = _hr(eng, yd[:, :t_fit], 1, 1, d, 0, X.shape[0])
        g = hr["ma_order"] > 0
        assert (got["css"][g] <= got["css_start"][g]).all() and np.isfinite(got["css"][g]).all(), d
        for k in SHARED:
            assert _bits(got[k][~g]) == _bits(hr[k][~g]), (d, k)
    eng.close()


@pytest.mark.parametrize("diff", [1, 2])
def test_forecast_groups_with_joint_beta(diff):
    """forecast_groups(ar=1, diff=d, ma=1, estimator='css', joint_beta=True): every group the engine call on its rows"""
    pdf = mmf.synth.reference_weekly_demand(6)
    horizon = 40
    out = mmf.forecast_groups(pdf, freq="W-MON", horizon=horizon, mode="holdout", ar=1, diff=diff, ma=1,
                              estimator="css", joint_beta=True)
    css = mmf.forecast_groups(pdf, freq="W-MON", horizon=horizon, mode="holdout", ar=1, diff=diff, ma=1,
                              estimator="css")
    assert list(out.columns) == list(css.columns) and len(out) == len(css)
    eng = mmf.ForecastEngine()
    for (prod, sku), g in out.groupby(["Product", "SKU"], sort=True):
        src = pdf[(pdf["Product"] == prod) & (pdf["SKU"] == sku)].sort_values("Date")
        y = src["Demand"].to_numpy(dtype=np.float32)[None, :]
        t_len, t_fit = y.shape[1], y.shape[1] - horizon
        X = O.design_matrix(O.calendar_grid(np.datetime64(src["Date"].min(), "D"), t_len, "W-MON"), t_fit)
        eng.plan(X, t_fit, True)
        eng.plan_arima(X, t_fit, 2)
        want = _joint(eng, _dev(y)[:, :t_fit], 1, 1, diff, 0, t_len)["pred"][0]
        got = g["Demand_Fitted"].to_numpy(dtype=np.float32)
        ok = (got == want) | (np.isnan(got) & np.isnan(want))
        assert ok.all() or np.nanmax(np.abs(got - want) / (np.abs(want) + 1.0)) < 1e-3, (prod, sku)
    conf = mmf.forecast_groups(pdf, freq="W-MON", horizon=horizon, mode="holdout", ar=1, diff=diff, ma=1,
                               estimator="css", joint_beta=True, conf_int=0.9)
    assert np.array_equal(conf["Demand_Fitted"].to_numpy(), out["Demand_Fitted"].to_numpy(), equal_nan=True)
    assert "Demand_Lower" in conf.columns
    eng.close()


@pytest.mark.parametrize("lib", ["product", "whitebeta"])
def test_negative_control(lib):
    """the white-beta build fails the joint optimality check on at least half of its converged rows; the product's
    converged rows pass it"""
    import json
    import os
    import subprocess
    import sys
    from conftest import ROOT
    y, X = joint_rows(40, 157, [0.8], [0.4], 31)
    np.save("/tmp/_joint_y.npy", y)
    np.save("/tmp/_joint_X.npy", X)
    env = dict(os.environ)
    if lib == "whitebeta":
        env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", "libmmf_armajoint_whitebeta.so")
    code = f"""
import json, sys
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, "tests")!r}]
import numpy as np, torch, mmf
y = np.load("/tmp/_joint_y.npy"); X = np.load("/tmp/_joint_X.npy")
eng = mmf.ForecastEngine(); eng.plan(X, 157, True)
r = eng.fit_forecast_arma(torch.from_numpy(y).cuda(), 1, 1, 0, 157, 8, estimator="css", joint_beta=True, max_iter=64)
print(json.dumps({{k: r[k].cpu().numpy().tolist() for k in ("phi", "theta", "beta", "css_stop", "ma_order")}}))
"""
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, check=True)
    got = {k: np.array(v) for k, v in json.loads(out.stdout.strip().splitlines()[-1]).items()}
    z, Dm, W, kept, Af, g0 = JO.plan_of(y, X, 157, 0)
    rows = np.flatnonzero((got["ma_order"] > 0) & (got["css_stop"] == 1))
    assert len(rows) >= 10
    fails = 0
    for i in rows:
        obs = np.isfinite(z[i])
        cols = JO.used_cols(Dm[:157], obs, kept)
        b = got["beta"][i].astype(np.float64)
        x = np.r_[got["phi"][i][:1], got["theta"][i][:1], b[cols]]
        gap = JO.optimality_gap(z[i], obs, Dm[:157], 157, 1, 1, x, b, cols)
        if lib == "product":
            _le(gap, OPT_RTOL + 1e-6, f"row {i}: optimality gap")
        fails += gap > OPT_RTOL + 1e-6
    record_err("test_negative_control_joint", fails / len(rows), 0.5, what=lib)
    if lib == "whitebeta":
        assert fails >= 0.5 * len(rows), (fails, len(rows))
