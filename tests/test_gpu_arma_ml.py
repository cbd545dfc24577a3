"""GPU: mmf_fit_forecast_arma_ml_f32 (DESIGN.md section 2 item 19) against the float64 oracle ``arma_ml_oracle`` and
against the CSS and HR calls it builds on.

The exact-input route of test_gpu_arma_css_replay: the plain plan takes a caller design that is zero on every fit row and
no constant, so the residual e the kernel filters is y (d = 0) or the fp32 Delta^d y (d >= 1), bit-identical to the
oracle's on integer levels.  On that route:
  - loglik_start is the float32 of the oracle's log-likelihood at the CSS call's fp32 point within 1 ulp;
  - loglik >= loglik_start, and loglik lies within LL_TOL (relative to n_obs) of the oracle's own LM run from the same
    point (measured on an H100 80GB HBM3 at 700 W, see the record_err lines);
  - sigma is the float32 of sqrt(S_w / n) at the shipped point within 4 ulps;
  - pred of a refined row is the oracle recursion at the shipped fp32 (phi, theta), integrated to levels;
  - a gated row that accepted no step keeps the CSS call's pred, phi, theta, order, ma_order and status bit for bit;
  - a row the HR gate refused, or an empty row, keeps the CSS call's outputs bit for bit with NaN, NaN, 0, 0.
The negative-control builds libmmf_armaml_nologdet.so and libmmf_armaml_gapzero.so must fail the loglik_start check."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mmf
import arma_ml_oracle as ML
from arma_oracle import _integrate, recursion
from conftest import ROOT, record_err
from test_gpu_arima import _np
from test_gpu_arma_css_replay import NPRED, _bits, _engine, _exact, _levels, _ulps

pytestmark = pytest.mark.gpu

SHARED = ("pred", "phi", "theta", "order", "ma_order", "status")
LL_TOL = 2e-5          # |loglik_gpu - loglik_oracle| / n_obs on refined rows that both runs stopped converged


def _gappy(y, frac, seed, d):
    """NaN at a fraction of the fit rows (at least one row when frac > 0), never in the first d + 1 rows"""
    y = y.copy()
    if frac <= 0:
        return y
    rng = np.random.default_rng(seed)
    t = y.shape[1]
    for i in range(len(y)):
        k = max(1, int(round(frac * t)))
        y[i, rng.choice(np.arange(d + 1, t), size=k, replace=False)] = np.nan
    return y


def _run(eng, y, p, q, d, max_iter=0):
    t_fit = y.shape[1]
    yd = torch.from_numpy(y.astype(np.float32)).cuda()
    ml = _np(eng.fit_forecast_arma(yd, p, q, d, t_fit, NPRED, estimator="ml", max_iter=max_iter))
    css = _np(eng.fit_forecast_arma(yd, p, q, d, t_fit, NPRED, estimator="css", max_iter=max_iter))
    return ml, css


def _check(ml, css, y, p, q, d, max_iter, what):
    """every row against the CSS call and the oracle -> counts"""
    gated = css["css_stop"] > 0
    ng = ~gated
    for k in SHARED + ("sigma",):
        assert _bits(ml[k][ng]) == _bits(css[k][ng]), (what, k)
    assert np.isnan(ml["loglik"][ng]).all() and np.isnan(ml["loglik_start"][ng]).all()
    assert not ml["iters"][ng].any() and not ml["ml_stop"][ng].any()
    rows = np.flatnonzero(gated)
    E, OBS = _exact(y, d)
    T = E.shape[1]
    t_fit = y.shape[1]
    worst = {"ll_start_ulps": 0, "ll_gap": 0.0, "pred": 0.0}
    n_ref = 0
    for i in rows:
        x0 = np.r_[css["phi"][i, :p], css["theta"][i, :q]].astype(np.float32)
        r = ML.lm(E[i], OBS[i], T, p, q, x0, max_iter)
        why = (what, int(i))
        if not r["ok"]:
            assert ml["ml_stop"][i] == 0 and np.isnan(ml["loglik"][i]), why
            for k in SHARED + ("sigma",):
                assert _bits(ml[k][i]) == _bits(css[k][i]), (why, k)
            continue
        u = int(_ulps(ml["loglik_start"][i:i + 1], np.array([r["loglik0"]]))[0]) if r["loglik0"] > 0 else int(
            _ulps(-ml["loglik_start"][i:i + 1], np.array([-r["loglik0"]]))[0])
        worst["ll_start_ulps"] = max(worst["ll_start_ulps"], u)
        assert u <= 1, (why, "loglik_start", ml["loglik_start"][i], r["loglik0"])
        assert ml["loglik"][i] >= ml["loglik_start"][i], why
        assert 1 <= ml["iters"][i] <= (max_iter or 20) and 1 <= ml["ml_stop"][i] <= 3, why
        n_obs = int(OBS[i].sum())
        if ml["ml_stop"][i] == 1 and r["stop"] == 1:
            gap = abs(float(ml["loglik"][i]) - r["loglik"]) / n_obs
            worst["ll_gap"] = max(worst["ll_gap"], gap)
            assert gap <= LL_TOL, (why, ml["loglik"][i], r["loglik"])
        xs = np.r_[ml["phi"][i, :p], ml["theta"][i, :q]].astype(np.float64)
        ev = ML.ml_eval(E[i], OBS[i], T, p, q, xs)
        assert ev["ok"], why
        assert _ulps(ml["sigma"][i:i + 1], np.array([ev["sigma"]]))[0] <= 4, (why, ml["sigma"][i], ev["sigma"])
        refined = _bits(np.r_[ml["phi"][i], ml["theta"][i]]) != _bits(np.r_[css["phi"][i], css["theta"][i]])
        if not refined:
            for k in SHARED:
                assert _bits(ml[k][i]) == _bits(css[k][i]), (why, k)
            continue
        n_ref += 1
        end = t_fit + NPRED
        pr, _, _ = recursion(E[i], OBS[i], T, xs[:p], xs[p:], end - d)
        zhat = np.full((1, end), np.nan)
        zhat[0, d:end] = pr
        if d == 0:
            want = zhat[0, t_fit:end]
        else:
            yh, _ = _integrate(zhat, y[i:i + 1].astype(np.float64), np.isfinite(y[i:i + 1]), t_fit, d, end)
            want = yh[0, t_fit:end]
        scale = max(np.nanmax(np.abs(y[i])), np.abs(want).max()) + 1.0   # an integrated forecast can leave y's range
        err = float(np.max(np.abs(ml["pred"][i] - want))) / scale
        worst["pred"] = max(worst["pred"], err)
        assert err <= 1e-4, (why, ml["pred"][i], want)
    record_err("arma_ml", worst["ll_gap"], LL_TOL, what=what, gated=len(rows), refined=n_ref, **worst)
    return len(rows), n_ref


@pytest.mark.parametrize("gaps", [0.0, 1e-3, 0.16])
@pytest.mark.parametrize("d", [0, 1, 2])
@pytest.mark.parametrize("p,q", [(0, 1), (1, 1), (2, 2), (4, 4), (8, 4)])
def test_weekly_exact_route(p, q, d, gaps):
    t_fit = 157
    n = 16 if p + q <= 2 else 8 if p + q <= 4 else 4
    eng = _engine(t_fit)
    y = _gappy(_levels(p, q, d, n, t_fit, seed=11000 + 100 * p + 10 * q + d), gaps, seed=p + q + d, d=d)
    ml, css = _run(eng, y, p, q, d)
    ng, nr = _check(ml, css, y, p, q, d, 0, f"weekly p={p} q={q} d={d} gaps={gaps}")
    if p + q <= 4:
        assert ng >= n // 2 and nr >= 1, (ng, nr)
    eng.close()


@pytest.mark.parametrize("t_fit", [117, 40])
def test_short_weekly_shapes_and_over_differencing(t_fit):
    """the weekly 117 / 40 shapes, and ARIMA(0, 2, 1) on a random walk, whose MA root sits near the unit circle"""
    eng = _engine(t_fit)
    for p, q, d, d_true in ((1, 1, 1, 1), (0, 1, 2, 1)):
        y = _levels(p, q, d, 16, t_fit, seed=12000 + t_fit + d, d_true=d_true)
        ml, css = _run(eng, y, p, q, d, max_iter=64)
        _check(ml, css, y, p, q, d, 64, f"short t_fit={t_fit} p={p} q={q} d={d}/{d_true}")
    eng.close()


def test_daily_calendar_null_outputs_assume_finite_and_windows():
    """the daily calendar with its real design: the CSS call's outputs on every row the ML stage leaves alone; NULL
    outputs write nothing else; assume_finite on gap-free rows gives the same bits; holdout and mid-design windows"""
    from test_gpu_arima import _case
    y, X, t_fit, has_c = _case("daily")[:4]
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    yd = torch.from_numpy(np.ascontiguousarray(y[:64], dtype=np.float32)).cuda()
    for ps, npred in ((t_fit, 28), (0, t_fit + 28), (t_fit // 2, 40)):
        ml = _np(eng.fit_forecast_arma(yd, 1, 1, 0, ps, npred, estimator="ml"))
        css = _np(eng.fit_forecast_arma(yd, 1, 1, 0, ps, npred, estimator="css"))
        gated = css["css_stop"] > 0
        assert gated.sum() >= 32
        same = (_bits(ml["phi"][i]) == _bits(css["phi"][i]) and _bits(ml["theta"][i]) == _bits(css["theta"][i])
                for i in range(len(gated)))
        for i, s in enumerate(same):
            if s:
                assert _bits(ml["pred"][i]) == _bits(css["pred"][i]), (ps, i)
        assert (ml["loglik"][gated] >= ml["loglik_start"][gated]).all()
        # NULL outputs: the C call with only pred, then every row's pred equals the full call's
        lib, h = eng._lib, eng._h
        out = torch.full((len(yd), npred), 7.0, device="cuda")
        rc = lib.mmf_fit_forecast_arma_ml_f32(h, yd.data_ptr(), len(yd), yd.stride(0), 1, 0, 1, 0, 0, ps, npred,
                                              out.data_ptr(), npred, *(None,) * 11)
        assert rc == 0
        torch.cuda.synchronize()
        assert _bits(out.cpu().numpy()) == _bits(ml["pred"]), ps
    eng.close()
    fin = mmf.ForecastEngine(assume_finite=True)
    fin.plan(X, t_fit, has_c)
    rows = np.flatnonzero(np.isfinite(y[:64, :t_fit]).all(axis=1))
    yf = torch.from_numpy(np.ascontiguousarray(y[rows], dtype=np.float32)).cuda()
    a = _np(fin.fit_forecast_arma(yf, 1, 1, 0, t_fit, 28, estimator="ml"))
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, has_c)
    b = _np(eng.fit_forecast_arma(yf, 1, 1, 0, t_fit, 28, estimator="ml"))
    for k in a:
        assert _bits(a[k]) == _bits(b[k]), k
    fin.close()
    eng.close()


def test_refusals_write_nothing_and_want_se():
    t_fit = 157
    eng = _engine(t_fit)
    y = _levels(1, 1, 1, 8, t_fit, seed=13000)
    yd = torch.from_numpy(y.astype(np.float32)).cuda()
    lib, h = eng._lib, eng._h
    out = torch.full((8, NPRED), 7.0, device="cuda")
    ll = torch.full((8,), 7.0, device="cuda")
    for (p, d, q, mi) in ((1, 1, 1, 65), (1, 1, 1, -1), (9, 1, 1, 0), (1, 1, 5, 0), (1, 3, 1, 0), (1, 1, 0, 65)):
        rc = lib.mmf_fit_forecast_arma_ml_f32(h, yd.data_ptr(), 8, yd.stride(0), p, d, q, 0, mi, t_fit, NPRED,
                                              out.data_ptr(), NPRED, *(None,) * 8, ll.data_ptr(), None, None, None)
        assert rc != 0, (p, d, q, mi)
    torch.cuda.synchronize()
    assert (out == 7.0).all() and (ll == 7.0).all()
    with pytest.raises(ValueError, match="estimator must be 'hr' or 'css'"):
        eng.fit_forecast_arma(yd, 1, 1, 1, t_fit, NPRED, estimator="mle")
    with pytest.raises(ValueError, match="joint_beta=True needs estimator='css'"):
        eng.fit_forecast_arma(yd, 1, 1, 1, t_fit, NPRED, estimator="ml", joint_beta=True)
    res = _np(eng.fit_forecast_arma(yd, 1, 1, 1, t_fit, NPRED, estimator="ml", want_se=True))
    assert np.isfinite(res["se"]).all() and (res["se"] > 0).all()
    eng.close()


def test_forecast_groups_with_ml_and_conf_int():
    pdf = mmf.synth.reference_weekly_demand(6)
    out = mmf.forecast_groups(pdf, freq="W-MON", horizon=40, mode="holdout", ar=1, diff=1, ma=1, estimator="ml",
                              conf_int=0.9)
    css = mmf.forecast_groups(pdf, freq="W-MON", horizon=40, mode="holdout", ar=1, diff=1, ma=1, estimator="css",
                              conf_int=0.9)
    assert list(out.columns) == list(css.columns) and (out.dtypes == css.dtypes).all()
    v = out["Demand_Fitted"].to_numpy(dtype=np.float64)
    assert np.isfinite(v).any()
    lo = [c for c in out.columns if c.endswith("_Lower")]
    assert lo and np.isfinite(out[lo[0]].to_numpy(dtype=np.float64)).any()


def test_shared_context_across_streams_matches_fresh():
    t_fit = 157
    y = _gappy(_levels(2, 2, 1, 24, t_fit, seed=14000), 0.05, seed=3, d=1)
    eng = _engine(t_fit)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    yd = torch.from_numpy(y.astype(np.float32)).cuda()
    with torch.cuda.stream(s1):
        a = eng.fit_forecast_arma(yd, 2, 2, 1, t_fit, NPRED, estimator="ml")
    s1.synchronize()
    with torch.cuda.stream(s2):
        b = eng.fit_forecast_arma(yd, 2, 2, 1, t_fit, NPRED, estimator="ml")
    s2.synchronize()
    fresh = _engine(t_fit)
    c = fresh.fit_forecast_arma(yd, 2, 2, 1, t_fit, NPRED, estimator="ml")
    for k in a:
        assert _bits(_np({k: a[k]})[k]) == _bits(_np({k: c[k]})[k]) == _bits(_np({k: b[k]})[k]), k
    eng.close()
    fresh.close()


@pytest.mark.parametrize("lib_name,gaps", [("libmmf_armaml_nologdet.so", 0.0), ("libmmf_armaml_gapzero.so", 0.16)])
def test_negative_controls_fail_the_loglik_check(tmp_path, lib_name, gaps):
    t_fit = 157
    p, q, d = 1, 1, 1
    y = _gappy(_levels(p, q, d, 32, t_fit, seed=15000), gaps, seed=15, d=d)
    src = str(tmp_path / "y.npy")
    np.save(src, y.astype(np.float32))
    env = dict(os.environ, MMF_LIB=os.path.join(ROOT, "tests", "_build", lib_name))
    code = f"""
import json, sys
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, "tests")!r}]
import numpy as np, torch, mmf
from test_gpu_arma_ml import _engine, _run
y = np.load({src!r})
eng = _engine({t_fit})
ml, css = _run(eng, y, {p}, {q}, {d})
print(json.dumps({{"ll0": ml["loglik_start"].tolist(), "phi": css["phi"].tolist(), "theta": css["theta"].tolist(),
                   "stop": css["css_stop"].tolist()}}))
"""
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, check=True)
    got = json.loads(out.stdout.strip().splitlines()[-1])
    E, OBS = _exact(y.astype(np.float32), d)
    bad = n = 0
    for i in range(len(y)):
        if got["stop"][i] == 0:
            continue
        x0 = np.r_[got["phi"][i][:p], got["theta"][i][:q]].astype(np.float32)
        ev = ML.ml_eval(E[i], OBS[i], E.shape[1], p, q, x0)
        if not ev["ok"]:
            continue
        n += 1
        bad += abs(got["ll0"][i] - ev["loglik"]) > 1e-4 * abs(ev["loglik"])
    bad = int(bad)
    record_err("arma_ml_control_" + lib_name, bad / max(n, 1), 0.5, rows=n, failing=bad)
    assert n >= 16 and bad >= 0.5 * n, (bad, n)
