"""Prediction standard errors on the GPU (mmf_fit_forecast_se_f32, DESIGN.md section 2 item 7 and section 4.11).

Every batch mixes the rows of test_gpu_abi_contract (gap-free, isolated gaps, 8 leading gaps, 45 gaps in one chunk
parity, mostly missing, a single value, empty, +Inf), interleaved so that several kinds share a 128-row tile.

* pred / status bit-equal to mmf_fit_forecast_f32 for auto, tc and warp, in future mode (h = 1, 28, 64), holdout mode
  and a window in the middle of the design; dof equal to the oracle's; sigma and se within the bounds below.
* An oracle-free check: sigma^2 dof against the squared residuals of the GPU's own holdout fitted values.
* Edges: 33 fit rows with horizon 28 (leverage in the hundreds), a near-perfect fit, dof <= 0, 70,001-row hourly
  series, 2^21 + 1,001 rows (bit-equal to calls of at most 2^20 rows), every output nullable on its own, out_se as a
  view of a wider table, argument errors, exact scaling by 2^k.
* Coverage of the nominal 90 % interval on 100,000 Gaussian series with per-series noise levels.

Bounds.  The library forms RSS = S - b'gamma, S = sum_obs (y - c)^2, so its rounding is relative to S, not to RSS:
    |sigma^2 dof - RSS_ref| <= TAU * max(1, sqrt(t_fit / 1095)) * S_ref * m_i
with m_i the mask factor of test_gpu_edges.  Then |sigma - sigma_ref| <= sqrt(that / dof), and se = sigma sqrt(1 + h)
adds the error of h (fp32 forward substitution on the row's own factor, or the float64 |a_t|^2 of the fp32 design):
    |se - se_ref| <= sqrt(1 + h_ref) * (sqrt(bound / dof) + H_REL * m_i * sigma_ref).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import mmf
from interval_oracle import fit_forecast_se_packed
from oracle import mmf_oracle as O
from test_gpu_abi_contract import KINDS, PATTERN, _hourly, _mask_factor, _plant, _round4
from test_gpu_edges import _bits, _le, _row_tol, _same_bits

pytestmark = pytest.mark.gpu

TAU = 2e-5        # S-relative bound on sigma^2 dof (fp32 moments and squares, f64 sums)
H_REL = 1e-4      # relative bound on sqrt(1 + h), times the mask factor
START = "2019-01-01"


def _tau(t_fit):
    return TAU * max(1.0, float(np.sqrt(t_fit / 1095.0)))


def _batch(n, t_fit, seed, X, shift=0):
    rng = np.random.default_rng(seed)
    level = rng.uniform(20.0, 500.0, (n, 1))
    sd = rng.uniform(0.02, 0.3, (n, 1)) * level
    beta = rng.normal(0, 1, (n, X.shape[1])) * 0.1
    beta[:, 0] = 0.0
    y = level + level * (beta @ X[:t_fit].T) + sd * rng.normal(0, 1, (n, t_fit))
    return _plant(y.astype(np.float32), t_fit, shift)


def _daily(t_fit, n_rows):
    return O.design_matrix(O.calendar_grid(START, n_rows, "D"), t_fit)


def _engines():
    return {k: mmf.ForecastEngine(kernel=k) for k in ("auto", "tc", "warp")}


def _np(res):
    return {k: v.cpu().numpy() for k, v in res.items() if k != "stats"}


def _check_se(got, y, X, t_fit, ps, npred, what):
    """dof exact, sigma and se within the bounds of the module docstring, NaN exactly where dof <= 0"""
    ref = fit_forecast_se_packed(y, X, t_fit, ps, npred)
    assert np.array_equal(got["dof"], ref["dof"]), (what, np.flatnonzero(got["dof"] != ref["dof"])[:8])
    bad = ref["dof"] <= 0
    assert np.isnan(got["sigma"][bad]).all() and np.isnan(got["se"][bad]).all(), what
    ok = ~bad
    assert np.isfinite(got["sigma"][ok]).all() and (got["sigma"][ok] >= 0).all(), what
    assert np.isfinite(got["se"][ok]).all(), what
    m = _mask_factor(y, X, t_fit, ps, npred, ref["ratio"])[ok]
    dof = ref["dof"][ok].astype(np.float64)
    bound = _tau(t_fit) * ref["S"][ok] * m
    s2 = got["sigma"][ok].astype(np.float64) ** 2 * dof
    _le(float((np.abs(s2 - ref["rss"][ok]) / np.maximum(bound, 1e-300)).max()), 1.0, f"{what}: sigma^2 dof vs RSS / bound")
    sq = np.sqrt(1.0 + ref["h"][ok])
    tol = sq * (np.sqrt(bound / dof) + H_REL * m * ref["sigma"][ok])[:, None]
    _le(float((np.abs(got["se"][ok] - ref["se"][ok]) / tol).max()), 1.0, f"{what}: se vs oracle / bound")
    return ref


WINDOWS = {                      # name: (t_fit, n_rows, pred_start, n_pred)
    "h1": (365, 366, 365, 1),
    "h28": (365, 393, 365, 28),
    "h64": (365, 429, 365, 64),
    "holdout": (337, 365, 0, 365),
    "middle": (365, 393, 100, 50),
    "short33": (33, 61, 33, 28),        # leverage in the hundreds
}


@pytest.mark.parametrize("window", sorted(WINDOWS))
def test_se_matches_plain_call_and_oracle(window):
    t_fit, n_rows, ps, npred = WINDOWS[window]
    X = _daily(t_fit, n_rows)
    y = _batch(301, t_fit, seed=sorted(WINDOWS).index(window), X=X)
    yd = mmf.device_packed(y)
    for kernel, eng in _engines().items():
        eng.plan(X, t_fit, True)
        plain = eng.fit_forecast(yd, ps, npred, want_status=True)
        got = eng.fit_forecast_se(yd, ps, npred)
        assert _same_bits(plain["pred"], got["pred"]), (window, kernel)
        assert torch.equal(plain["status"], got["status"]), (window, kernel)
        _check_se(_np(got), y, X, t_fit, ps, npred, f"{window}/{kernel}")
        eng.close()


def test_sigma_against_the_gpus_own_residuals():
    """oracle-free: sigma^2 dof against sum_obs (y - yhat_gpu)^2 with the GPU's holdout fitted values"""
    t_fit, n_rows = 337, 365
    X = _daily(t_fit, n_rows)
    y = _batch(301, t_fit, seed=11, X=X)
    yd = mmf.device_packed(y)
    for kernel, eng in _engines().items():
        eng.plan(X, t_fit, True)
        got = _np(eng.fit_forecast_se(yd, 0, n_rows))
        obs = np.isfinite(y)
        ok = got["dof"] > 0
        r = np.where(obs, y.astype(np.float64) - got["pred"][:, :t_fit], 0.0)
        rss = (r ** 2).sum(axis=1)
        n_obs = obs.sum(axis=1)
        ref = fit_forecast_se_packed(y, X, t_fit, 0, n_rows)
        m = np.where(ok, _mask_factor(y, X, t_fit, 0, n_rows, ref["ratio"]), 1.0)
        d = _row_tol(np.where(obs, y, 0.0)) * m
        bound = 2 * np.sqrt(rss * n_obs) * d + n_obs * d ** 2 + _tau(t_fit) * ref["S"] * m
        s2 = got["sigma"].astype(np.float64) ** 2 * got["dof"]
        _le(float((np.abs(s2 - rss)[ok] / bound[ok]).max()), 1.0, f"{kernel}: sigma^2 dof vs own residuals / bound")
        eng.close()


def test_near_perfect_fit_and_nonpositive_dof():
    """R^2 ~ 1 - 1e-8: S - b'gamma cancels; sigma stays finite, >= 0 and within the S-relative bound.  A p = 5 design
    fit on 5 rows has dof = 0: NaN."""
    t_fit, n_rows = 365, 393
    X = _daily(t_fit, n_rows)
    rng = np.random.default_rng(3)
    n = 257
    W, _ = O.whiten(X[:t_fit])
    A = X @ W
    g = rng.normal(0, 1, (n, 16)) * 1e2 * (np.abs(W).sum(axis=0) > 0)
    y = (1000.0 + g @ A[:t_fit].T + 1e-2 * rng.normal(0, 1, (n, t_fit))).astype(np.float32)
    y = _plant(y, t_fit)
    for kernel, eng in _engines().items():
        eng.plan(X, t_fit, True)
        got = _np(eng.fit_forecast_se(mmf.device_packed(y), t_fit, 28))
        _check_se(got, y, X, t_fit, t_fit, 28, f"near-perfect/{kernel}")
        Xs = np.random.default_rng(4).normal(0, 1, (9, 5))
        Xs[:, 0] = 1.0
        eng.plan(Xs, 5, True)
        ys = np.random.default_rng(5).normal(10, 1, (7, 5)).astype(np.float32)
        got = _np(eng.fit_forecast_se(mmf.device_packed(ys), 5, 4))
        assert (got["dof"] == 0).all() and np.isnan(got["sigma"]).all() and np.isnan(got["se"]).all(), kernel
        eng.close()


def test_long_hourly_series():
    t_fit = 70001
    X = _hourly(t_fit + 24, t_fit)
    y = _batch(18, t_fit, seed=7, X=X)
    yd = mmf.device_packed(y)
    for kernel, eng in _engines().items():
        eng.plan(X, t_fit, True)
        plain = eng.fit_forecast(yd, t_fit, 24, want_status=True)
        got = eng.fit_forecast_se(yd, t_fit, 24)
        assert _same_bits(plain["pred"], got["pred"]) and torch.equal(plain["status"], got["status"]), kernel
        _check_se(_np(got), y, X, t_fit, t_fit, 24, f"hourly/{kernel}")
        eng.close()


def test_multi_slab_batch_is_bit_equal_to_single_slab_calls():
    t_fit, h = 100, 28
    X = _daily(t_fit, t_fit + h)
    n = (1 << 21) + 1001
    rng = np.random.default_rng(9)
    y = (100.0 + 10.0 * rng.normal(0, 1, (n, t_fit))).astype(np.float32)
    for s in range(0, n, 1 << 19):
        _plant(y[s:s + 64], t_fit, shift=s)
    yd = mmf.device_packed(y)
    del y
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, True)
    for ps, npred in ((t_fit, h), (0, t_fit + h)):
        whole = eng.fit_forecast_se(yd, ps, npred)
        for a in range(0, n, 1 << 20):
            part = eng.fit_forecast_se(yd[a:a + (1 << 20)], ps, npred)
            for k in ("pred", "se", "sigma", "dof", "status"):
                assert _same_bits(whole[k][a:a + (1 << 20)], part[k]), (ps, a, k)
    eng.close()


def _raw(eng, yd, ps, npred, out, se, ld_se, sigma, dof, status):
    ptr = lambda t: t.data_ptr() if t is not None else None
    return eng._lib.mmf_fit_forecast_se_f32(eng._h, yd.data_ptr(), yd.shape[0], yd.stride(0), ps, npred, ptr(out),
                                            out.stride(0), ptr(se), ld_se, ptr(sigma), ptr(dof), ptr(status), None)


def _filled(shape, dtype=torch.float32):
    """caller memory the library must not write: every word is PATTERN"""
    return torch.full(shape, PATTERN, dtype=torch.int32, device="cuda").view(dtype)


def _same_values(a, b):
    """bit equality with NaN where the other has NaN (the library's NaN and torch's may differ in payload)"""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(_bits(torch.where(na, 0.0, a)), _bits(torch.where(nb, 0.0, b)))


def test_outputs_nullable_wide_se_view_and_argument_errors():
    t_fit, h = 365, 28
    X = _daily(t_fit, t_fit + 64)
    y = _batch(301, t_fit, seed=13, X=X)
    yd = mmf.device_packed(y)
    n = yd.shape[0]
    for kernel, eng in _engines().items():
        eng.plan(X, t_fit, True)
        ref = eng.fit_forecast_se(yd, t_fit, h)
        torch.cuda.synchronize()
        for want in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1)):
            out = torch.empty((n, _round4(h)), device="cuda")[:, :h]
            se = torch.empty((n, _round4(h)), device="cuda")[:, :h] if want[0] else None
            sg = torch.empty(n, device="cuda") if want[1] else None
            dof = torch.empty(n, device="cuda", dtype=torch.int32) if want[2] else None
            st = torch.empty(n, device="cuda", dtype=torch.int32)
            mmf._native.check(_raw(eng, yd, t_fit, h, out, se, se.stride(0) if se is not None else 0, sg, dof, st))
            torch.cuda.synchronize()
            assert _same_bits(out, ref["pred"]) and torch.equal(st, ref["status"]), (kernel, want)
            for got, k in ((se, "se"), (sg, "sigma"), (dof, "dof")):
                if got is not None:
                    assert _same_bits(got, ref[k]), (kernel, want, k)
        # out_se as a window of a wider table: nothing outside it is written
        for npred in (h, 27, 1):
            wide = _filled((n, 40))
            out = torch.empty((n, _round4(npred)), device="cuda")[:, :npred]
            mmf._native.check(_raw(eng, yd, t_fit, npred, out, wide[:, 3:], 40, None, None, None))
            torch.cuda.synchronize()
            w = wide.view(torch.int32).cpu().numpy()
            assert (w[:, :3] == PATTERN).all() and (w[:, 3 + npred:] == PATTERN).all(), (kernel, npred)
            full = eng.fit_forecast_se(yd, t_fit, npred)["se"]
            assert _same_bits(wide[:, 3:3 + npred].contiguous(), full.contiguous()), (kernel, npred)
        # argument errors: return code, every output untouched
        bufs = dict(out=_filled((n, 32)), se=_filled((n, 32)), sigma=_filled((n,)), dof=_filled((n,), torch.int32),
                    status=_filled((n,), torch.int32))
        before = {k: v.clone() for k, v in bufs.items()}
        b = bufs
        cases = [                                    # MMF_E_INVALID
            (-1, dict(ps=t_fit, npred=h, se=None, ld_se=0, sigma=None, dof=None)),
            (-1, dict(ps=t_fit, npred=h, se=b["se"], ld_se=h - 1, sigma=b["sigma"], dof=b["dof"])),
            (-1, dict(ps=t_fit, npred=65, se=b["se"], ld_se=32, sigma=b["sigma"], dof=b["dof"])),
            (-1, dict(ps=-1, npred=h, se=b["se"], ld_se=32, sigma=b["sigma"], dof=b["dof"])),
        ]
        for code, kw in cases:
            rc = _raw(eng, yd, kw["ps"], kw["npred"], b["out"], kw["se"], kw["ld_se"], kw["sigma"], kw["dof"], b["status"])
            assert rc == code, (kernel, kw, rc)
        host_se = np.zeros((n, 32), dtype=np.float32)
        rc = eng._lib.mmf_fit_forecast_se_f32(eng._h, yd.data_ptr(), n, yd.stride(0), t_fit, h, b["out"].data_ptr(), 32,
                                              host_se.ctypes.data, 32, None, None, None, None)
        assert rc == -3 and not host_se.any(), (kernel, rc)           # MMF_E_UNSUPPORTED
        torch.cuda.synchronize()
        for k in bufs:
            assert torch.equal(bufs[k].view(torch.int32), before[k].view(torch.int32)), (kernel, k)
        eng.close()


@pytest.mark.parametrize("kernel", ["auto", "warp"])
def test_scaling_by_powers_of_two_is_exact(kernel):
    t_fit, h = 365, 28
    X = _daily(t_fit, t_fit + h)
    y = _batch(301, t_fit, seed=17, X=X)
    eng = mmf.ForecastEngine(kernel=kernel)
    eng.plan(X, t_fit, True)
    base = eng.fit_forecast_se(mmf.device_packed(y), t_fit, h)
    for k in range(-12, 15, 2):
        got = eng.fit_forecast_se(mmf.device_packed(y * np.float32(2.0 ** k)), t_fit, h)
        for key in ("sigma", "se"):
            assert _same_values(got[key], base[key] * (2.0 ** k)), (kernel, k, key)
        assert torch.equal(got["dof"], base["dof"])
    eng.close()


def test_coverage_of_the_nominal_90_percent_interval():
    """100,000 Gaussian series x 365 days with a per-series noise level (the generator's Variance_RN idea), horizon 28:
    pred -+ t_{dof, 0.95} se covers 90 % +- 0.5 % of the future values."""
    from scipy import stats
    t_fit, h, n = 365, 28, 100_000
    X = _daily(t_fit, t_fit + h)
    rng = np.random.default_rng(21)
    level = rng.uniform(20.0, 500.0, (n, 1))
    sd = level * rng.uniform(0.05, 0.5, (n, 1))
    beta = rng.normal(0, 0.05, (n, X.shape[1]))
    beta[:, 0] = 0.0
    mean = level + level * (beta @ X.T)
    ally = (mean + sd * rng.normal(0, 1, mean.shape)).astype(np.float32)
    eng = mmf.ForecastEngine()
    eng.plan(X, t_fit, True)
    got = _np(eng.fit_forecast_se(mmf.device_packed(ally[:, :t_fit]), t_fit, h))
    q = stats.t.ppf(0.95, got["dof"])[:, None]
    fut = ally[:, t_fit:]
    cover = (np.abs(fut - got["pred"]) <= q * got["se"]).mean()
    _le(abs(float(cover) - 0.9), 0.005, f"coverage {cover:.4f}")
    eng.close()
