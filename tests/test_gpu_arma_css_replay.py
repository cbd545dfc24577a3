"""GPU: mmf_fit_forecast_arma_css_f32 (DESIGN.md section 2 item 16) replayed pass by pass by the float64 oracle.

The exact-input route: the plain plan takes a caller design whose one column is zero on every fit row (test_gpu_abi_contract's
``fit_zero``) and no constant, so gamma = 0, c = 0 and the kernel's fitted value is exactly 0 on every fit row.  Its
residual e is then y for d = 0 and the fp32 Delta^d y for d >= 1, which is exact for integer levels below 2^20.  The
kernel and ``arma_css_oracle.lm_replay`` therefore see bit-identical residuals, and the replay starts from the HR
call's fp32 (phi, theta), which is exactly the kernel's start.  On every gated row whose path the replay does not mark
ambiguous (a decision within the float64 noise of its threshold, ``lm_replay``'s docstring), the GPU must have taken the
same path: iters, css_stop and "refined" equal, phi and theta bit-equal, css_start, css and sigma = sqrt(S / |C|) the
float32 of the replay's float64 values within 1 ulp.  Rows that fail the HR gate keep the HR call's outputs bit for
bit.  Every case decides a stated minimum of rows.  Ambiguous rows are counted; over the cases that ran they must stay
under AMBIGUOUS_MAX of the gated rows (measured on an H100 80GB HBM3 at 700 W: 467 of 4,754 gated rows, 9.8 %, nearly
all high-order fits with a nearly singular step system; 465 of those 467 took the replay's path all the same)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

import mmf
import arma_css_oracle as S
from conftest import ROOT, record_err
from test_arma_css_oracle import _random_poly
from test_gpu_arima import _dev, _np

pytestmark = pytest.mark.gpu

SHARED = ("pred", "phi", "theta", "order", "ma_order", "sigma", "status")
NPRED = 4
AMBIGUOUS_MAX = 0.12
TOTALS = {"gated": 0, "ambiguous": 0, "stops": [0, 0, 0, 0], "refined": 0}


@pytest.fixture(scope="module", autouse=True)
def _ambiguous_share():
    """after the module's cases, whichever of them ran: the ambiguous rows stay under AMBIGUOUS_MAX of the gated rows"""
    yield
    if TOTALS["gated"]:
        record_err("css_replay_totals", TOTALS["ambiguous"] / TOTALS["gated"], AMBIGUOUS_MAX, **TOTALS)
        assert TOTALS["ambiguous"] <= AMBIGUOUS_MAX * TOTALS["gated"], TOTALS


def _design(t_fit):
    """the fit_zero design: one column, 0 on the fit rows and 1 on the NPRED rows after them; no constant"""
    return (np.arange(t_fit + NPRED) >= t_fit).astype(np.float64)[:, None]


def _engine(t_fit):
    eng = mmf.ForecastEngine()
    X = _design(t_fit)
    eng.plan(X, t_fit, False)
    eng.plan_arima(X, t_fit, 2)
    return eng


def _levels(p, q, d, n, t_fit, seed, d_true=None, sd=1.0):
    """n rows of integer levels whose Delta^d_true is a simulated ARMA(p, q) error with random stationary and invertible
    parameters (d_true = d by default), scaled so that |y| < 2^19"""
    rng = np.random.default_rng(seed)
    d_true = d if d_true is None else d_true
    y = np.zeros((n, t_fit))
    for i in range(n):
        ph, th = _random_poly(rng, p), -_random_poly(rng, q)
        eps = rng.normal(0, sd, t_fit + 300)
        z = lfilter(np.r_[1.0, th], np.r_[1.0, -ph], eps)[300 + d_true:]
        for _ in range(d_true):
            z = np.concatenate([[0.0], np.cumsum(z)])
        y[i] = z[:t_fit]
    scale = np.minimum(50.0, 2.0 ** 19 / np.maximum(np.abs(y).max(axis=1, keepdims=True), 1e-9))
    return np.round(y * scale)


def _gaps(y, kind, seed, p=0):
    """NaN patterns on the levels: first missing row at s, a run of 40, the last fit row, 12 % isolated"""
    y = y.copy()
    rng = np.random.default_rng(seed)
    t = y.shape[1]
    for i in range(len(y)):
        k = kind if kind != "mix" else ("none", "first", "run", "last", "iso")[i % 5]
        if k == "first":
            s = [max(p - 1, 0), 31, 32, 127, 128][(i // 5) % 5]
            if s < t - 2:
                y[i, s] = np.nan
                y[i, rng.integers(s + 1, t, size=max(t // 40, 1))] = np.nan
        elif k == "run" and t > 110:
            y[i, 64:104] = np.nan
        elif k == "last":
            y[i, t - 1] = np.nan
        elif k == "iso":
            y[i, rng.choice(np.arange(t), size=int(0.12 * t), replace=False)] = np.nan
    return y


def _exact(y, d):
    """(e, obs) the kernel sees: Delta^d y in float64 (exact on integer levels), 0 where missing"""
    z = np.asarray(y, dtype=np.float64)
    for _ in range(d):
        z = z[:, 1:] - z[:, :-1]
    obs = np.isfinite(z)
    return np.where(obs, z, 0.0), obs


def _run(eng, y, p, q, d, max_iter=0, m=0):
    t_fit = y.shape[1]
    yd = _dev(y.astype(np.float32))
    css = _np(eng.fit_forecast_arma(yd, p, q, d, t_fit, NPRED, long_order=m, estimator="css", max_iter=max_iter))
    hr = _np(eng.fit_forecast_arma(yd, p, q, d, t_fit, NPRED, long_order=m))
    return css, hr


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def _ulps(got, want64):
    """|got - fp32(want)| in fp32 ulps (positive finite values)"""
    w = np.asarray(want64, dtype=np.float64).astype(np.float32)
    return np.abs(got.astype(np.float32).view(np.int32).astype(np.int64) - w.view(np.int32).astype(np.int64))


def _check(css, hr, y, p, q, d, max_iter, what, min_decided):
    """HR rows bit for bit, gated rows against lm_replay; at least ``min_decided`` gated rows whose path the replay
    decides -> (replay, gated row indices)"""
    gated = hr["ma_order"] == q
    assert np.array_equal(css["css_stop"] > 0, gated), what
    ng = ~gated
    for k in SHARED:
        assert _bits(css[k][ng]) == _bits(hr[k][ng]), (what, k)
    assert np.isnan(css["css"][ng]).all() and np.isnan(css["css_start"][ng]).all() and not css["iters"][ng].any()
    rows = np.flatnonzero(gated)
    if len(rows) == 0:
        assert min_decided == 0, (what, "nothing gated")
        return None, rows
    E, OBS = _exact(y, d)
    T = E.shape[1]
    X0 = np.concatenate([hr["phi"][rows, :p], hr["theta"][rows, :q]], axis=1).astype(np.float32)
    r = S.lm_replay(E[rows], OBS[rows], T, p, q, X0, max_iter=max_iter)
    # css_start on every gated row: S at x0 is one float64 evaluation of the same residuals
    u = _ulps(css["css_start"][rows], r["S0"])
    assert (u <= 1).all(), (what, "css_start ulps", rows[u > 1][:8], u.max())
    amb = r["ambiguous"]
    refined = r["n_acc"] > 0
    for j, i in enumerate(rows):
        if amb[j]:
            continue
        why = (what, int(i), {k: float(v[j]) for k, v in r["margin"].items()}, int(css["iters"][i]), int(r["iters"][j]),
               int(css["css_stop"][i]), int(r["stop"][j]))
        assert css["iters"][i] == r["iters"][j] and css["css_stop"][i] == r["stop"][j], why
        xg = np.r_[css["phi"][i, :p], css["theta"][i, :q]].astype(np.float32)
        assert _bits(xg) == _bits(r["x"][j]), (why, xg, r["x"][j])
        assert (_bits(np.r_[css["phi"][i], css["theta"][i]]) != _bits(np.r_[hr["phi"][i], hr["theta"][i]])) == \
            refined[j], why
        assert _ulps(css["css"][i:i + 1], r["S"][j:j + 1])[0] <= 1, (why, css["css"][i], r["S"][j])
        sig = np.sqrt(r["S"][j] / r["n_C"][j])
        assert _ulps(css["sigma"][i:i + 1], np.array([sig]))[0] <= 1, (why, css["sigma"][i], sig)
        if not refined[j]:
            for k in SHARED:
                if k != "sigma":
                    assert _bits(css[k][i]) == _bits(hr[k][i]), (why, k)
    # ambiguous rows that took the replay's path all the same (how conservative the margins are)
    same = [bool(css["iters"][i] == r["iters"][j] and css["css_stop"][i] == r["stop"][j] and
                 _bits(np.r_[css["phi"][i, :p], css["theta"][i, :q]].astype(np.float32)) == _bits(r["x"][j]))
            for j, i in enumerate(rows) if amb[j]]
    n_amb = int(amb.sum())
    assert len(rows) - n_amb >= min_decided, (what, len(rows), n_amb, min_decided)
    stops = np.bincount(r["stop"][~amb], minlength=4).tolist()
    TOTALS["gated"] += len(rows)
    TOTALS["ambiguous"] += n_amb
    TOTALS["ambiguous_same_path"] = TOTALS.get("ambiguous_same_path", 0) + int(sum(same))
    TOTALS["refined"] += int(refined[~amb].sum())
    TOTALS["stops"] = [a + b for a, b in zip(TOTALS["stops"], stops)]
    record_err("css_replay", n_amb / len(rows), AMBIGUOUS_MAX, what=what, gated=len(rows), ambiguous=n_amb, stops=stops,
               ambiguous_same_path=int(sum(same)),
               ambiguous_margins=[{k: float(v[j]) for k, v in r["margin"].items() if k != "lam"}
                                  for j in np.flatnonzero(amb)][:4])
    return r, rows


# ---- the route itself ------------------------------------------------------------------------------------------------
def test_exact_route_css_start_is_the_oracle_s0():
    """the plain plan accepts the fit_zero design, keeps no column, every row with observations has status 0, and
    css_start is fp32 of the oracle's S0 from the same residuals within 1 ulp (d = 0, 1, 2)"""
    t_fit = 157
    eng = _engine(t_fit)
    for d in (0, 1, 2):
        y = _gaps(_levels(1, 1, d, 48, t_fit, seed=100 + d), "mix", seed=d)
        css, hr = _run(eng, y, 1, 1, d)
        assert (css["status"] == 0).all(), (d, np.unique(css["status"]))
        r, rows = _check(css, hr, y, 1, 1, d, 0, f"route d={d}", min_decided=30)
    eng.close()


# ---- every (p, q), d in {0, 1, 2} -----------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [0, 1, 2])
@pytest.mark.parametrize("q", [1, 2, 3, 4])
@pytest.mark.parametrize("p", list(range(9)))
def test_every_order_on_the_weekly_shape(p, q, d):
    """every packed-entry layout of the per-lane system (p + q + 1)(p + q + 2) / 2 = 3 .. 91 entries, on 157 weekly rows
    with a mix of gap patterns"""
    t_fit = 157
    eng = _engine(t_fit)
    y = _gaps(_levels(p, q, d, 20, t_fit, seed=1000 + 100 * p + 10 * q + d), "mix", seed=p * 7 + q, p=p)
    css, hr = _run(eng, y, p, q, d)
    _check(css, hr, y, p, q, d, 0, f"weekly p={p} q={q} d={d}", min_decided=10 if p + q <= 3 else 1)
    eng.close()


@pytest.mark.parametrize("d", [0, 1, 2])
@pytest.mark.parametrize("p,q", [(0, 1), (1, 1), (2, 2), (3, 4), (5, 3), (7, 1), (8, 4)])
def test_orders_on_the_daily_shape(p, q, d):
    t_fit = 1095
    eng = _engine(t_fit)
    y = _gaps(_levels(p, q, d, 10, t_fit, seed=2000 + 100 * p + 10 * q + d), "mix", seed=p + q, p=p)
    css, hr = _run(eng, y, p, q, d)
    _check(css, hr, y, p, q, d, 0, f"daily p={p} q={q} d={d}", min_decided=5 if p + q <= 3 else 1)
    eng.close()


# ---- block and chunk edges -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [0, 1])
@pytest.mark.parametrize("p,q", [(1, 1), (2, 3), (8, 4)])
@pytest.mark.parametrize("T", ["pq2", 31, 32, 33, 127, 128, 129, 255, 257])
def test_block_and_chunk_edges(T, p, q, d):
    """T (rows of z) at the 32-row blocks and 128-row chunks; the first missing row before p, at 31, 32, 127, 128; a
    40-row run that empties a whole 32-row block of C; a missing last fit row; 12 % isolated gaps.  Shapes too short
    for the HR gate (T = p + q + 2, and (8, 4) below 64 rows) gate nothing and keep the HR call's bits; every other case
    decides at least one row, (1, 1) and (2, 3) at least 3 (T <= 33) or 5 rows"""
    Tz = p + q + 2 if T == "pq2" else T
    t_fit = Tz + d
    eng = _engine(t_fit)
    y = _gaps(_levels(p, q, d, 40, t_fit, seed=3000 + Tz * 10 + p + d), "mix", seed=Tz + p, p=p)
    css, hr = _run(eng, y, p, q, d)
    if T == "pq2" or (p + q >= 12 and Tz < 64):
        need = 0
    else:
        need = 1 if p + q >= 12 else 3 if Tz <= 33 else 5
    _check(css, hr, y, p, q, d, 0, f"edges T={Tz} p={p} q={q} d={d}", min_decided=need)
    eng.close()


# ---- every stop code ------------------------------------------------------------------------------------------------
def test_every_stop_code_on_decided_rows():
    """max_iter in {1, 2, 3, 20, 64} on ARMA rows, and over-differenced rows (d = 2 on a random walk, d = 1 on white
    noise), whose optimum lies on the invertibility boundary: step-down retries and stalls"""
    t_fit = 157
    eng = _engine(t_fit)
    seen = np.zeros(4, dtype=np.int64)
    for mi in (1, 2, 3, 20, 64):
        for p, q, d, d_true in ((1, 1, 0, 0), (2, 2, 0, 0), (0, 1, 2, 1), (1, 2, 2, 1), (0, 2, 1, 0)):
            y = _levels(p, q, d, 32, t_fit, seed=4000 + mi * 10 + p + q + d, d_true=d_true)
            css, hr = _run(eng, y, p, q, d, max_iter=mi)
            r, rows = _check(css, hr, y, p, q, d, mi, f"stops max_iter={mi} p={p} q={q} d={d}/{d_true}",
                             min_decided=8)
            if mi == 1:
                assert (css["iters"][rows] == 1).all() and (css["css_stop"][rows] == 3).all()
            seen += np.bincount(r["stop"][~r["ambiguous"]], minlength=4)
    record_err("css_replay_stop_codes", 0.0, 0.0, stops=seen.tolist())
    assert (seen[1:] > 0).all(), seen.tolist()
    eng.close()


# ---- mixed pass counts in one CTA ------------------------------------------------------------------------------------
def _mixed_pool(n, t_fit, seed):
    """rows that converge in a few passes (clean MA(1)) interleaved with over-differenced rows that run long"""
    fast = _levels(0, 1, 1, n, t_fit, seed=seed)
    slow = _levels(0, 0, 1, n, t_fit, seed=seed + 1, d_true=0)
    y = fast.copy()
    y[1::2] = slow[1::2]
    return y


def test_mixed_pass_counts_in_one_cta_are_bit_equal_alone_and_permuted():
    """batches of 1, 7, 8, 9 and 8 SM +- 1 rows: every row bit-equal in every output to the same row called alone and to
    the same row at another position of a permuted batch; the whole pool against the replay with max_iter = 64"""
    t_fit = 157
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    pool = _mixed_pool(8 * n_sm + 1, t_fit, seed=5000)
    eng = _engine(t_fit)
    full, hr = _run(eng, pool, 0, 1, 1, max_iter=64)
    _check(full, hr, pool, 0, 1, 1, 64, "mixed pool", min_decided=len(pool) // 2)
    it = full["iters"][: (len(pool) // 8) * 8].reshape(-1, 8)
    assert ((it.min(1) <= 4) & (it.max(1) >= 12)).any(), "no CTA mixes short and long rows"
    rng = np.random.default_rng(5)
    singles = {}
    for n in (1, 7, 8, 9, 8 * n_sm - 1, 8 * n_sm + 1):
        y = pool[:n]
        got, _ = _run(eng, y, 0, 1, 1, max_iter=64)
        perm = rng.permutation(n)
        gp, _ = _run(eng, y[perm], 0, 1, 1, max_iter=64)
        for k in got:
            assert _bits(got[k]) == _bits(full[k][:n]), (n, k)
            assert _bits(gp[k]) == _bits(got[k][perm]), (n, k, "permuted")
        for i in rng.choice(n, size=min(n, 6), replace=False):
            if i not in singles:
                singles[i], _ = _run(eng, pool[i:i + 1], 0, 1, 1, max_iter=64)
            for k in got:
                assert _bits(singles[i][k][0]) == _bits(got[k][i]), (n, int(i), k, "alone")
    eng.close()


# ---- a long series ---------------------------------------------------------------------------------------------------
def test_long_hourly_series():
    """three rows of a 70,001-row hourly series with gaps, ARMA(1, 1) and ARIMA(1, 1, 1), five passes"""
    t_fit = 70001
    eng = _engine(t_fit)
    for d in (0, 1):
        y = _gaps(_levels(1, 1, d, 3, t_fit, seed=6000 + d), "iso", seed=6 + d)
        css, hr = _run(eng, y, 1, 1, d, max_iter=5)
        _check(css, hr, y, 1, 1, d, 5, f"hourly d={d}", min_decided=2)
    eng.close()


# ---- the negative control --------------------------------------------------------------------------------------------
def test_diagonal_step_control_fails_the_replay(tmp_path):
    """libmmf_armacss_diagstep.so solves each step with diag(H) only; S still falls at every accepted step, but its path
    departs from the replay (iters, css_stop or x) on at least half of the refined, decided rows"""
    t_fit = 157
    p, q, d = 2, 2, 0
    y = _gaps(_levels(p, q, d, 64, t_fit, seed=7000), "mix", seed=7)
    src = str(tmp_path / "y.npy")
    np.save(src, y.astype(np.float32))
    env = dict(os.environ, MMF_LIB=os.path.join(ROOT, "tests", "_build", "libmmf_armacss_diagstep.so"))
    code = f"""
import json, sys
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, "tests")!r}]
import numpy as np, torch, mmf
from test_gpu_arma_css_replay import _engine, _run
y = np.load({src!r})
eng = _engine({t_fit})
css, hr = _run(eng, y, {p}, {q}, {d})
print(json.dumps({{"css": {{k: v.tolist() for k, v in css.items()}}, "hr": {{k: v.tolist() for k, v in hr.items()}}}}))
"""
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, check=True)
    got = json.loads(out.stdout.strip().splitlines()[-1])
    css = {k: np.array(v, dtype=np.float32 if isinstance(v[0], list) or isinstance(v[0], float) else np.int32)
           for k, v in got["css"].items()}
    hr = {k: np.array(v, dtype=np.float32 if isinstance(v[0], list) or isinstance(v[0], float) else np.int32)
          for k, v in got["hr"].items()}
    rows = np.flatnonzero(hr["ma_order"] == q)
    assert len(rows) >= 30
    E, OBS = _exact(y.astype(np.float32), d)
    X0 = np.concatenate([hr["phi"][rows, :p], hr["theta"][rows, :q]], axis=1).astype(np.float32)
    r = S.lm_replay(E[rows], OBS[rows], E.shape[1], p, q, X0)
    dec = ~r["ambiguous"] & (r["n_acc"] > 0)
    fails = 0
    for j in np.flatnonzero(dec):
        i = rows[j]
        xg = np.r_[css["phi"][i, :p], css["theta"][i, :q]].astype(np.float32)
        fails += bool(css["iters"][i] != r["iters"][j] or css["css_stop"][i] != r["stop"][j] or
                      _bits(xg) != _bits(r["x"][j]))
        assert css["css"][i] <= css["css_start"][i]
    record_err("css_replay_diagstep_control", fails / max(dec.sum(), 1), 0.5, refined=int(dec.sum()), fails=fails)
    assert dec.sum() >= 20 and fails >= 0.5 * dec.sum(), (fails, int(dec.sum()))
