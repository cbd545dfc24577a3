"""GPU (-m gpu): standard errors of the ARIMA-family forecasts (mmf_arima_se_f32, DESIGN.md section 2 item 15).

Yardstick: the float64 oracle of tests/arima_se_oracle.py fed the GPU's own fp32 parameters (phi, theta, orders, sigma,
d).  The GPU value is the float32 rounding of the same float64 quantity computed in another order, so it is held to
4 fp32 ulp of the oracle, with identical NaN / Inf patterns.  The no-gaps build (tests/_build/libmmf_arimase_nogaps.so)
must exceed that bound on at least 100 gappy rows."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mmf
from mmf import _native as N
from arima_se_oracle import arima_se
from conftest import ROOT, record_err
from test_gpu_abi_contract import PATTERN
from test_gpu_arima import _case, _dev, _np, _windows
from test_gpu_edges import _same_bits

pytestmark = pytest.mark.gpu

ULP = 4


def _ulp_err(got, want):
    """max |got - want| in fp32 ulp of want over the finite entries; asserts identical NaN / +-Inf patterns"""
    got = np.asarray(got, dtype=np.float32)
    w32 = np.asarray(want, dtype=np.float64).astype(np.float32)
    assert np.array_equal(np.isnan(got), np.isnan(w32)), np.argwhere(np.isnan(got) != np.isnan(w32))[:8]
    assert np.array_equal(np.isinf(got), np.isinf(w32))
    assert np.array_equal(got[np.isinf(got)], w32[np.isinf(w32)])
    fin = np.isfinite(w32)
    if not fin.any():
        return 0.0
    err = np.abs(got[fin].astype(np.float64) - np.asarray(want, dtype=np.float64)[fin])
    return float((err / np.spacing(np.abs(w32[fin]))).max())


def _oracle(res, y, t_fit, ps, npred, d=0, diffs=None):
    th = res.get("theta")
    return arima_se(y, t_fit, res["phi"], res["order"], res["sigma"], ps, npred, d, diffs=diffs, theta=th,
                    ma_order=res.get("ma_order"))


def _se_raw(eng, y, t_fit, d, diffs, phi, order, theta, ma, sigma, ps, npred, out, ld_se, stats=None):
    lib = N.load()
    eng.set_stream(torch.cuda.current_stream().cuda_stream)     # enqueue where torch reads the results
    p = lambda x: None if x is None else x.data_ptr()                                    # noqa: E731
    return lib.mmf_arima_se_f32(eng._h, y.data_ptr(), y.shape[0], y.stride(0), t_fit, d, p(diffs), p(phi), p(order),
                                p(theta), p(ma), p(sigma), ps, npred, out.data_ptr() if out is not None else None, ld_se,
                                C.byref(stats) if stats is not None else None)


@pytest.fixture(scope="module", params=["daily", "weekly", "exog_only", "caller"])
def cal(request):
    y, X, t_fit, has_c = _case(request.param, n=170, seed=11)
    # a few MA rows and long gaps on top of test_gpu_arima's row mix
    y[20, 30:60] = np.nan
    y[21, t_fit - 9:t_fit] = np.nan
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    eng.plan_arima(X, t_fit, 2)
    hold = 20
    sel = mmf.ForecastEngine()
    sel.plan(X, t_fit - hold, has_c)
    sel.plan_arima(X, t_fit - hold, 2)
    return request.param, y, X, t_fit, eng, sel, hold


def _calls(eng, sel, yd, t_fit, hold, ps, npred, want_se):
    """the six model calls (label, result dict as numpy, plan t_fit, d, diffs)"""
    out = []
    out.append(("ar2", _np(eng.fit_forecast_ar(yd, 2, ps, npred, want_se=want_se)), t_fit, 0, None))
    for d in (1, 2):
        out.append((f"arima1{d}", _np(eng.fit_forecast_arima(yd, 1, d, ps, npred, want_se=want_se)), t_fit, d, None))
    for p, q, d in ((1, 1, 0), (1, 1, 1), (1, 1, 2), (2, 2, 1), (0, 1, 2), (4, 4, 0)):
        out.append((f"arma{p}{d}{q}", _np(eng.fit_forecast_arma(yd, p, q, d, ps, npred, want_se=want_se)), t_fit, d,
                    None))
    tf = t_fit - hold
    r = _np(sel.fit_select_ar(yd, hold, (0, 1, 2, 4), ps, npred, want_se=want_se))
    out.append(("select_ar", r, tf, 0, None))
    r = _np(sel.fit_select_arima(yd, hold, (0, 1, 2), (0, 1, 2), ps, npred, want_se=want_se))
    out.append(("select_arima", r, tf, 0, r["choice_d"]))
    r = _np(sel.fit_select_arma(yd, hold, (0, 1, 2, 3, 4), (0, 1, 2), (0, 1, 2), ps, npred, want_se=want_se))
    out.append(("select_arma", r, tf, 0, r["choice_d"]))
    return out


@pytest.mark.parametrize("window", ["future", "holdout", "mid"])
def test_parity_of_every_model_call(cal, window):
    """all six calls on four calendars and three windows: se within 4 ulp of the oracle on the GPU's own parameters;
    NaN exactly where the prediction is NaN for rows with a finite sigma; every other output bit-equal to want_se=False"""
    name, y, X, t_fit, eng, sel, hold = cal
    ps, npred = _windows(t_fit, X.shape[0])[window]
    yd = _dev(y)
    worst = 0.0
    plain = _calls(eng, sel, yd, t_fit, hold, ps, npred, False)
    for (label, res, tf, d, diffs), (_, ref, _, _, _) in zip(_calls(eng, sel, yd, t_fit, hold, ps, npred, True), plain):
        for k, v in ref.items():
            assert np.ascontiguousarray(v).tobytes() == np.ascontiguousarray(res[k]).tobytes(), (label, k)
        want = _oracle(res, y, tf, ps, npred, d, diffs)
        e = _ulp_err(res["se"], want)
        worst = max(worst, e)
        assert e <= ULP, (name, window, label, e)
        fin = np.isfinite(res["sigma"])
        assert np.array_equal(np.isnan(res["se"][fin]), np.isnan(res["pred"][fin])), (name, window, label)
        assert np.isnan(res["se"][~fin]).all()
    record_err(f"arima_se parity {name} {window}", worst, ULP)


@pytest.mark.parametrize("shape", ["weekly157", "daily365"])
def test_parity_on_demand_shapes(shape):
    from demand_shapes import calendar, demand_batch
    _, t, _, X = calendar(shape, extra=28)
    y, kinds, _ = demand_batch(124, shape, seed=9)
    hold = 28 if shape == "daily365" else 12
    eng = mmf.ForecastEngine()
    eng.plan(X, t - hold, True)
    eng.plan_arima(X, t - hold, 2)
    yd = _dev(y)
    for ps, npred in ((0, t + 28), (t - hold, 28 + hold)):
        r = _np(eng.fit_select_arma(yd, hold, (0, 1, 2), (0, 1, 2), (0, 1, 2), ps, npred, want_se=True))
        e = _ulp_err(r["se"], _oracle(r, y, t - hold, ps, npred, 0, r["choice_d"]))
        assert e <= ULP, (shape, ps, e)
        r = _np(eng.fit_forecast_arma(yd, 1, 1, 2, ps, npred, want_se=True))
        assert _ulp_err(r["se"], _oracle(r, y, t - hold, ps, npred, 2)) <= ULP


def _params(n, p, q, rng, scale=0.3):
    phi = torch.zeros((n, 8), device="cuda")
    theta = torch.zeros((n, 4), device="cuda")
    phi[:, :p] = torch.from_numpy(rng.uniform(-scale, scale, (n, p)) / max(p, 1)).float()
    theta[:, :q] = torch.from_numpy(rng.uniform(-scale, scale, (n, q)) / max(q, 1)).float()
    return phi, theta


def test_hand_built_parameters_identities_and_edges():
    eng = mmf.ForecastEngine()
    rng = np.random.default_rng(1)
    n, t_fit, h = 64, 90, 40
    y = torch.randn((n, t_fit), device="cuda")
    sigma = torch.from_numpy(rng.uniform(0.5, 20, n)).float().cuda()
    out = torch.empty((n, h), device="cuda")
    zi = torch.zeros(n, dtype=torch.int32, device="cuda")
    phi, theta = _params(n, 0, 0, rng)
    # p = q = d = 0: sigma everywhere; d = 1, p = q = 0: sigma sqrt(h)
    assert _se_raw(eng, y, t_fit, 0, None, phi, zi, theta, zi, sigma, 0, h, out, h) == 0
    assert _same_bits(out, sigma[:, None].expand(n, h).contiguous())
    assert _se_raw(eng, y, t_fit, 1, None, phi, zi, None, None, sigma, t_fit, h, out, h) == 0
    want = sigma.double()[:, None] * torch.arange(1, h + 1, device="cuda").double().sqrt()[None, :]
    assert float(((out.double() - want).abs() / want).max()) < 1e-6
    # out-of-range per-row values give NaN rows
    order = torch.tensor([1, 9, -1, 1, 1, 1] * 11, dtype=torch.int32, device="cuda")[:n]
    ma = torch.tensor([1, 1, 1, 5, -2, 1] * 11, dtype=torch.int32, device="cuda")[:n]
    diffs = torch.tensor([1, 1, 1, 1, 1, -1, 3, 2] * 8, dtype=torch.int32, device="cuda")[:n]
    phi, theta = _params(n, 1, 1, rng)
    assert _se_raw(eng, y, t_fit, 0, diffs, phi, order, theta, ma, sigma, 0, t_fit + h, torch.empty((n, t_fit + h),
                   device="cuda"), t_fit + h) == 0
    got = torch.empty((n, t_fit + h), device="cuda")
    _se_raw(eng, y, t_fit, 0, diffs, phi, order, theta, ma, sigma, 0, t_fit + h, got, t_fit + h)
    g = got.cpu().numpy()
    o, m, dd = order.cpu().numpy(), ma.cpu().numpy(), diffs.cpu().numpy()
    bad = (o < 0) | (o > 8) | (m < 0) | (m > 4) | (dd < 0) | (dd > 2)
    assert bad.any() and np.isnan(g[bad]).all() and np.isfinite(g[~bad][:, 2:]).all()
    want = arima_se(y.cpu().numpy(), t_fit, phi.cpu().numpy(), o, sigma.cpu().numpy(), 0, t_fit + h, diffs=dd,
                    theta=theta.cpu().numpy(), ma_order=m)
    assert _ulp_err(g, want) <= ULP
    # explosive parameters: +Inf far out, no fault
    phi = torch.zeros((n, 8), device="cuda")
    phi[:, 0] = 3.0
    big = torch.empty((n, 2000), device="cuda")
    assert _se_raw(eng, y, t_fit, 2, None, phi, zi + 1, None, None, sigma, t_fit, 2000, big, 2000) == 0
    torch.cuda.synchronize()
    assert torch.isinf(big[:, -1]).all() and torch.isfinite(big[:, 0]).all()


def test_y_beyond_t_fit_is_never_read_and_only_finiteness_matters():
    y, X, t_fit, has_c = _case("daily", n=170, seed=3)
    eng = mmf.ForecastEngine()
    eng.plan_arima(X, t_fit, 2)
    yd = _dev(y)
    res = eng.fit_forecast_arma(yd, 1, 1, 1, 0, X.shape[0], want_se=True)
    wide = torch.full((y.shape[0], t_fit + 64), float("nan"), device="cuda")
    wide[:, :t_fit] = yd
    outs = []
    for fill, scale in ((float("nan"), 1.0), (1e30, 1.0), (-7.0, 0.5)):
        wide[:, t_fit:] = fill
        ys = wide.clone()
        ys[:, :t_fit] *= scale
        out = torch.empty((y.shape[0], X.shape[0]), device="cuda")
        assert _se_raw(eng, ys, t_fit, 1, None, res["phi"], res["order"], res["theta"], res["ma_order"], res["sigma"],
                       0, X.shape[0], out, X.shape[0]) == 0
        outs.append(out)
    assert _same_bits(outs[0], res["se"]) and _same_bits(outs[1], outs[0]) and _same_bits(outs[2], outs[0])


def test_layouts_nullables_and_many_rows():
    eng = mmf.ForecastEngine()
    rng = np.random.default_rng(4)
    n, t_fit, npred = 300, 120, 37
    yh = rng.normal(size=(n, t_fit)).astype(np.float32)
    yh[rng.random(yh.shape) < 0.05] = np.nan
    y = torch.from_numpy(yh).cuda()
    phi, theta = _params(n, 2, 2, rng)
    order = torch.full((n,), 2, dtype=torch.int32, device="cuda")
    ma = torch.full((n,), 2, dtype=torch.int32, device="cuda")
    d1 = torch.ones(n, dtype=torch.int32, device="cuda")
    sigma = torch.ones(n, device="cuda")
    ref = torch.empty((n, npred), device="cuda")
    assert _se_raw(eng, y, t_fit, 1, None, phi, order, theta, ma, sigma, 50, npred, ref, npred) == 0
    assert _ulp_err(ref.cpu().numpy(), arima_se(yh, t_fit, phi.cpu().numpy(), order.cpu().numpy(), np.ones(n), 50,
                                               npred, 1, theta=theta.cpu().numpy(), ma_order=ma.cpu().numpy())) <= ULP
    pat = torch.tensor([PATTERN], dtype=torch.int32).view(torch.float32).item()
    for ld, off in ((npred + 3, 0), (41, 1), (npred, 3)):
        buf = torch.full((n * ld + off + 8,), pat, device="cuda")
        view = buf[off:off + n * ld].view(n, ld)
        assert _se_raw(eng, y, t_fit, 0, d1, phi, order, theta, ma, sigma, 50, npred, view, ld) == 0
        assert _same_bits(view[:, :npred].contiguous(), ref)
        rest = torch.cat([buf[:off], view[:, npred:].reshape(-1), buf[off + n * ld:]])
        assert (rest.view(torch.int32) == PATTERN).all(), (ld, off)
    # theta / ma_order NULL equals zeros bit for bit
    a, b = torch.empty_like(ref), torch.empty_like(ref)
    _se_raw(eng, y, t_fit, 1, None, phi, order, None, None, sigma, 50, npred, a, npred)
    _se_raw(eng, y, t_fit, 1, None, phi, order, torch.zeros_like(theta), torch.zeros_like(ma), sigma, 50, npred, b, npred)
    assert _same_bits(a, b)
    # n = 0 and more than 2^20 rows (eight distinct rows tiled)
    assert _se_raw(eng, y[:0], t_fit, 1, None, phi, order, theta, ma, sigma, 0, 5, ref, 5) == 0
    big = (1 << 20) + 5
    idx = torch.arange(big, device="cuda") % 8
    out = torch.empty((big, 16), device="cuda")
    assert _se_raw(eng, y[idx], t_fit, 1, None, phi[idx], order[idx], theta[idx], ma[idx], sigma[idx], t_fit - 8, 16,
                   out, 16) == 0
    small = torch.empty((8, 16), device="cuda")
    _se_raw(eng, y[:8], t_fit, 1, None, phi[:8], order[:8], theta[:8], ma[:8], sigma[:8], t_fit - 8, 16, small, 16)
    assert _same_bits(out, small[idx])


def test_refusals_write_nothing():
    eng = mmf.ForecastEngine()
    n, t_fit = 8, 40
    y = torch.randn((n, t_fit), device="cuda")
    phi = torch.zeros((n, 8), device="cuda")
    th = torch.zeros((n, 4), device="cuda")
    o = torch.ones(n, dtype=torch.int32, device="cuda")
    s = torch.ones(n, device="cuda")
    pat = torch.tensor([PATTERN], dtype=torch.int32).view(torch.float32).item()
    out = torch.full((n, 10), pat, device="cuda")
    lib = N.load()
    base = dict(t_fit=t_fit, d=1, diffs=None, phi=phi, order=o, theta=th, ma=o, sigma=s, ps=t_fit, npred=10, ld=10)
    bad = [dict(d=3), dict(d=-1), dict(t_fit=0), dict(t_fit=t_fit + 1), dict(npred=0), dict(ps=-1), dict(ld=9),
           dict(theta=None), dict(ma=None), dict(phi=None), dict(sigma=None), dict(order=None)]
    for b in bad:
        a = {**base, **b}
        rc = _se_raw(eng, y, a["t_fit"], a["d"], a["diffs"], a["phi"], a["order"], a["theta"], a["ma"], a["sigma"],
                     a["ps"], a["npred"], out, a["ld"])
        assert rc == -1, b
    yh = np.zeros((n, t_fit), dtype=np.float32)
    torch.cuda.synchronize()
    rc = lib.mmf_arima_se_f32(eng._h, yh.ctypes.data, n, t_fit, t_fit, 1, None, phi.data_ptr(), o.data_ptr(), None,
                              None, s.data_ptr(), t_fit, 10, out.data_ptr(), 10, None)
    assert rc == -3
    assert rc == -3 and (out.view(torch.int32) == PATTERN).all()
    assert lib.mmf_arima_se_f32(None, y.data_ptr(), n, t_fit, t_fit, 1, None, phi.data_ptr(), o.data_ptr(), None, None,
                                s.data_ptr(), t_fit, 10, out.data_ptr(), 10, None) == -1


def test_context_stream_and_shared_state():
    from test_gpu_arima import _case as case
    y, X, t_fit, has_c = case("weekly", n=96, seed=2)
    yd = _dev(y)
    fresh = mmf.ForecastEngine()
    fresh.plan(X, t_fit, has_c)
    fresh.plan_arima(X, t_fit, 2)
    want = _np(fresh.fit_forecast_arma(yd, 1, 1, 1, 0, X.shape[0], want_se=True))
    shared = mmf.ForecastEngine()
    shared.plan(X, t_fit, has_c)
    shared.plan_arima(X, t_fit, 2)
    before = _np(shared.fit_forecast(yd, 0, X.shape[0], want_status=True))
    shared.fit_select_arma(_dev(np.concatenate([y, y[:, -12:]], axis=1)), 12, (0, 1), (0, 1), (0, 1))
    got = _np(shared.fit_forecast_arma(yd, 1, 1, 1, 0, X.shape[0], want_se=True))
    for k in want:
        assert want[k].tobytes() == got[k].tobytes(), k
    after = _np(shared.fit_forecast(yd, 0, X.shape[0], want_status=True))
    for k in before:
        assert before[k].tobytes() == after[k].tobytes(), k
    # a borrowed stream, and no host synchronisation without stats: the call returns while the stream still sleeps
    st = torch.cuda.Stream()
    res = shared.fit_forecast_arma(yd, 1, 1, 1, 0, X.shape[0])
    torch.cuda.synchronize()
    out = torch.empty((y.shape[0], X.shape[0]), device="cuda")
    with torch.cuda.stream(st):
        shared.set_stream(st.cuda_stream)
        torch.cuda._sleep(200_000_000)
        assert _se_raw(shared, yd, t_fit, 1, None, res["phi"], res["order"], res["theta"], res["ma_order"],
                       res["sigma"], 0, X.shape[0], out, X.shape[0]) == 0
        assert not st.query()
    st.synchronize()
    assert out.cpu().numpy().tobytes() == want["se"].tobytes()
    stats = N.MmfStats()
    assert _se_raw(shared, yd, t_fit, 1, None, res["phi"], res["order"], res["theta"], res["ma_order"], res["sigma"],
                   0, X.shape[0], out, X.shape[0], stats) == 0
    assert stats.kernel_launches == 1 and stats.n_series == y.shape[0] and stats.kernel_ms > 0


_NEG_SCRIPT = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import mmf
from mmf import _native as N
from test_gpu_arima import _case, _dev
import ctypes as C
y, X, t_fit, has_c = _case("daily", n=170, seed=11)
rng = np.random.default_rng(0)
for i in range(0, 170, 3):
    a = int(rng.integers(20, t_fit - 30)); y[i, a:a + int(rng.integers(1, 6))] = np.nan
eng = mmf.ForecastEngine(); eng.plan_arima(X, t_fit, 2)
yd = _dev(y)
res = eng.fit_forecast_arma(yd, 1, 1, 1, 0, X.shape[0])
out = torch.empty((170, X.shape[0]), device="cuda")
rc = N.load().mmf_arima_se_f32(eng._h, yd.data_ptr(), 170, yd.stride(0), t_fit, 1, None, res["phi"].data_ptr(),
    res["order"].data_ptr(), res["theta"].data_ptr(), res["ma_order"].data_ptr(), res["sigma"].data_ptr(), 0,
    X.shape[0], out.data_ptr(), X.shape[0], None)
assert rc == 0
np.savez(sys.argv[2], se=out.cpu().numpy(), y=y, **{k: v.cpu().numpy() for k, v in res.items()})
"""


@pytest.mark.parametrize("lib", ["product", "nogaps"])
def test_negative_control(lib, tmp_path):
    path = os.path.join(ROOT, "dss-ml-at-scale_b200", "libmmf.so") if lib == "product" else \
        os.path.join(ROOT, "tests", "_build", "libmmf_arimase_nogaps.so")
    assert os.path.exists(path)
    out = str(tmp_path / "r.npz")
    env = {**os.environ, "MMF_LIB": path}
    subprocess.run([sys.executable, "-c", _NEG_SCRIPT, ROOT, out], check=True, env=env)
    r = dict(np.load(out))
    want = arima_se(r["y"], r["y"].shape[1], r["phi"], r["order"], r["sigma"], 0, r["se"].shape[1], 1,
                    theta=r["theta"], ma_order=r["ma_order"])
    fin = np.isfinite(want) & np.isfinite(r["se"])
    w32 = want.astype(np.float32)
    ulps = np.abs(r["se"][fin] - want[fin]) / np.spacing(np.abs(w32[fin]))
    n_bad = int((ulps > ULP).sum())
    record_err(f"arima_se negative control {lib}", n_bad, 100, worst_ulp=float(ulps.max()))
    if lib == "product":
        assert n_bad == 0, float(ulps.max())
    else:
        assert n_bad >= 100, n_bad


def _coverage(T, freq, hold, n, seed):
    """simulate n series of ARIMA(1, 1, 1) errors (phi 0.5, theta 0.3, sigma 1) on a regression and measure the 90 %
    coverage at h = 1, 7, 28 of the forecast from t_fit: of the reference-grid fit_select_arma (want_se=True), and of
    the true order fixed (fit_forecast_arma(1, 1, 1)).  -> (selected, fixed)"""
    from statistics import NormalDist
    from oracle import mmf_oracle as O
    start = np.datetime64("2019-01-07")
    X = O.design_matrix(O.calendar_grid(start, T, freq), T - hold)
    g = torch.Generator(device="cuda").manual_seed(seed)
    eps = torch.randn((n, T), device="cuda", generator=g, dtype=torch.float64)
    u = torch.zeros_like(eps)
    for s in range(T):
        u[:, s] = eps[:, s] + (0.5 * u[:, s - 1] + 0.3 * eps[:, s - 1] if s else 0.0)
    beta = torch.randn((n, X.shape[1]), device="cuda", generator=g, dtype=torch.float64) * 5.0
    y = torch.empty((n, (T + 3) & ~3), device="cuda")[:, :T]          # 16-B row pitch: the tensor-core path
    y.copy_(200.0 + beta @ torch.from_numpy(X).cuda().T + torch.cumsum(u, dim=1))
    del eps, u
    eng = mmf.ForecastEngine()
    eng.plan(X, T - hold, True)
    eng.plan_arima(X, T - hold, 2)
    z = NormalDist().inv_cdf(0.95)
    out = []
    for r in (eng.fit_select_arma(y, hold, pred_start=T - hold, n_pred=hold, want_se=True),
              eng.fit_forecast_arma(y, 1, 1, 1, T - hold, hold, want_se=True)):
        cov = {}
        for h in (1, 7, 28):
            e = (y[:, T - hold + h - 1] - r["pred"][:, h - 1]).abs()
            ok = torch.isfinite(r["se"][:, h - 1])
            cov[h] = float(((e <= z * r["se"][:, h - 1]) & ok).sum() / ok.sum())
        out.append(cov)
    return out


def test_end_to_end_coverage_of_the_selected_model():
    """200,000 simulated ARIMA(1, 1, 1) + regression series, 1,095 daily rows.  The selected model's coverage is
    measured on the held-out rows that chose it, so it is biased upward (the winner of 75 candidates has the smallest
    errors there, DESIGN.md section 6): it must not fall below 0.88.  The true order fixed uses no held-out value: within
    0.02 of 0.90 at h = 1 and 7; at h = 28 the estimation error of beta and (phi, theta), which the band leaves out and
    which the integration accumulates, shows (0.869 measured), so only 0.85 is required there.  The 117-week shape is
    reported, not gated."""
    sel, fixed = _coverage(1095, "D", 28, 200_000, seed=1)
    wsel, wfixed = _coverage(157, "W-MON", 40, 200_000, seed=2)
    record_err("arima_se coverage daily1095", max(abs(v - 0.9) for v in fixed.values()), 0.02,
               selected=json.dumps(sel), fixed=json.dumps(fixed), weekly_selected=json.dumps(wsel),
               weekly_fixed=json.dumps(wfixed))
    print("coverage daily 1095: selected", sel, "fixed", fixed, "| weekly 157 (not gated): selected", wsel, "fixed",
          wfixed)
    for h in fixed:
        assert abs(fixed[h] - 0.9) <= 0.02 if h < 28 else fixed[h] >= 0.85, (h, fixed[h])
        assert sel[h] >= 0.88, (h, sel[h])


def test_frames_conf_int_equals_the_engine():
    from statistics import NormalDist
    import pandas as pd
    from test_intervals_oracle import _weekly_frame
    df = _weekly_frame()
    eng = mmf.ForecastEngine()
    kw = dict(ar=(0, 1, 2, 3, 4), diff=(0, 1, 2), ma=(0, 1, 2, 3, 4))
    got = mmf.forecast_groups(df, freq="W-MON", horizon=12, mode="holdout", engine=eng, conf_int=0.9, **kw)
    z = NormalDist().inv_cdf(0.95)
    for sku, g in df.groupby("SKU"):
        s = g.set_index(pd.to_datetime(g["Date"]))["Demand"].asfreq("W-MON")
        _, ps, npred = eng.plan_calendar(np.datetime64(s.index[0].date(), "D"), len(s), "W-MON", 12, "holdout", max_diff=2)
        yd = _dev(s.to_numpy(np.float32)[None, :])
        r = eng.fit_select_arma(yd, 12, kw["ar"], kw["diff"], kw["ma"], ps, npred, want_se=True)
        pred, se = r["pred"].cpu().numpy()[0].astype(np.float64), r["se"].cpu().numpy()[0].astype(np.float64)
        rows = got[got["SKU"] == sku]
        assert np.array_equal(rows["Demand_Fitted"].to_numpy(), pred.astype(np.float32), equal_nan=True)
        assert np.array_equal(rows["Demand_Lower"].to_numpy(), (pred - z * se).astype(np.float32), equal_nan=True)
        assert np.array_equal(rows["Demand_Upper"].to_numpy(), (pred + z * se).astype(np.float32), equal_nan=True)
