"""GPU (-m gpu): the CUDA path, called through the C ABI (ctypes -> libmmf.so), against the float64
oracle on identical seeded inputs, the frozen golden vectors, and size-independent properties at
BASELINE.json's sizes.  Tolerance (stated, SURVEY.md 8c): |yhat_gpu - yhat_ref| <= 1e-4*max|y| + 1e-3."""
import datetime as dt

import numpy as np
import pytest

import mmf
from conftest import forecast_leverage, record_err, tolerance
from oracle import mmf_oracle as O

pytestmark = pytest.mark.gpu


def _le(err, tol, what=""):
    """assert err <= tol, leaving the measured error in the scratch log of conftest.record_err"""
    import os
    name = os.environ.get("PYTEST_CURRENT_TEST", "?").split("::")[-1].split(" ")[0]
    record_err(name, err, tol, what=str(what))
    assert err <= tol, (what, float(err), float(tol))


@pytest.fixture(scope="module")
def engines():
    e = {k: mmf.ForecastEngine(kernel=k) for k in ("auto", "warp", "tc")}
    yield e
    for x in e.values():
        x.close()


def _oracle(y, start, freq, horizon, mode):
    T = y.shape[1]
    if mode == "holdout":
        grid = O.calendar_grid(start, T, freq)
        return O.fit_forecast_packed(y, O.design_matrix(grid, T - horizon), T - horizon, 0, T)
    grid = O.calendar_grid(start, T + horizon, freq)
    return O.fit_forecast_packed(y, O.design_matrix(grid, T), T, T, horizon)


def _run(eng, y, start, freq, horizon, mode, **kw):
    import torch
    yd = mmf.device_packed(y)                       # row pitch multiple of 4 floats (TMA-eligible)
    res = mmf.forecast_packed(yd, start, freq, horizon, mode, engine=eng, want_status=True, **kw)
    torch.cuda.synchronize()
    return res["pred"].cpu().numpy(), res["status"].cpu().numpy(), res


# ---- frozen golden vectors -------------------------------------------------------------------------
def test_golden_reference_weekly_holdout(engines, oracle_golden):
    g = oracle_golden
    y = g["ref_weekly_y"]
    start = g["ref_weekly_start"][0].astype("datetime64[D]")
    for k in ("auto", "warp"):
        pred, status, _ = _run(engines[k], y, start, "W-MON", 40, "holdout")
        _le(np.abs(pred - g["ref_weekly_fitted"]).max(), tolerance(y))
        assert np.array_equal(status, g["ref_weekly_status"])


def test_golden_daily365_future_with_gaps(engines, oracle_golden):
    g = oracle_golden
    y = g["daily365_y"]
    start = g["daily365_start"][0].astype("datetime64[D]")
    for k in ("auto", "warp", "tc"):
        pred, status, _ = _run(engines[k], y, start, "D", 28, "future")
        _le(np.abs(pred - g["daily365_pred"]).max(), tolerance(y), k)
        assert np.array_equal(status, g["daily365_status"]), k


def test_golden_daily1095(engines, oracle_golden):
    g = oracle_golden
    y = g["daily1095_y"]
    start = g["daily1095_start"][0].astype("datetime64[D]")
    for k in ("auto", "warp", "tc"):
        pred, _, _ = _run(engines[k], y, start, "D", 28, "future")
        _le(np.abs(pred - g["daily1095_future"]).max(), tolerance(y), k)
    pred, _, _ = _run(engines["auto"], y, start, "D", 28, "holdout")
    _le(np.abs(pred - g["daily1095_holdout"]).max(), tolerance(y))


# ---- seeded parity, every kernel, BASELINE config 2 shape (10k x 1095 is covered below at reduced N) --
@pytest.mark.parametrize("kernel", ["warp", "tc", "auto"])
@pytest.mark.parametrize("n,t", [(1, 1095), (127, 1095), (128, 1095), (129, 1095), (1000, 1095), (300, 365), (64, 33),
                                 (40, 32), (9, 5)])
def test_parity_full_series(engines, kernel, n, t):
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=100 + n + t)
    want, wst = _oracle(y, start, "D", 28, "future")
    pred, status, _ = _run(engines[kernel], y, start, "D", 28, "future")
    lev = forecast_leverage(O.design_matrix(O.calendar_grid(start, t + 28, "D"), t), t, t, 28)   # < 1 from t = 365 up
    _le(np.abs(pred - want).max(), tolerance(y, lev), f"leverage {lev:.3g}")
    assert np.array_equal(status, wst)


def test_parity_config2_10k_by_1095(engines):
    """BASELINE.json configs[1]: 10k groups x 1,095 days fp32, single H100, parity on ALL series."""
    y, start = mmf.synth.daily_store_item_demand(10_000, 1095, seed=1234)
    want, _ = _oracle(y, start, "D", 28, "future")
    for k in ("tc", "warp"):
        pred, status, res = _run(engines[k], y, start, "D", 28, "future", want_stats=True)
        err = np.abs(pred - want)
        _le(err.max(), tolerance(y), k)
        assert (status == 0).all()
        assert res["stats"].kernel_used == k


@pytest.mark.parametrize("kernel", ["warp", "auto", "tc"])
def test_parity_masked_series(engines, kernel):
    y, start = mmf.synth.daily_store_item_demand(300, 1095, seed=7, nan_frac=0.02)
    y[5, :400] = np.nan          # long leading gap
    y[6, 700:] = np.nan          # long trailing gap
    y[7, ::2] = np.nan           # every other day
    y[8, 100] = np.inf           # Inf == missing
    want, wst, _, ratio = O.fit_forecast_packed(y, *_design(start, 1095, 28), return_gamma=True)
    pred, status, res = _run(engines[kernel], y, start, "D", 28, "future", want_stats=True)
    # ill-conditioned masks amplify fp32 rounding by ~1/min_pivot_ratio; scale the stated tolerance by it
    tol = tolerance(y) / np.minimum(1.0, ratio / 0.25)
    rel = np.abs(pred - want).max(axis=1) / tol
    _le(rel.max(), 1.0, f"{kernel}: worst row error / row tolerance")
    assert np.array_equal(status, wst)
    if kernel != "warp":
        # rows whose first value is missing (or with > 44 gaps per transform group) take the general pass;
        # every other gappy row is solved from the record the tensor-core kernel queued
        assert 0 < res["stats"].n_pending < 300


def test_gap_counts_around_record_capacity(engines):
    """The tensor-core kernel notes gap positions per transform group (alternate 32-step chunks) in two 44-entry
    segments that the solve kernel reads four at a time: every count 0..48 in one group (all tails of the 4-wide
    groups, the capacity edge and the overflow to the general pass), both groups, must match the oracle."""
    t, h = 1095, 28
    y0, start = mmf.synth.daily_store_item_demand(1, t, seed=21)
    rows = []
    for parity in (0, 1):
        slots = np.array([p for p in range(1, t) if (p // 32) % 2 == parity])
        rng = np.random.default_rng(parity)
        for k in range(0, 49):
            r = y0[0].copy()
            r[rng.choice(slots, size=k, replace=False)] = np.nan
            rows.append(r)
    both = y0[0].copy()                                              # 44 in each group: the largest record
    for parity in (0, 1):
        slots = np.array([p for p in range(1, t) if (p // 32) % 2 == parity])
        both[np.random.default_rng(7 + parity).choice(slots, size=44, replace=False)] = np.nan
    rows.append(both)
    y = np.stack(rows).astype(np.float32)
    want, wst = O.fit_forecast_packed(y, *_design(start, t, h))
    for k in ("auto", "tc"):
        pred, status, res = _run(engines[k], y, start, "D", h, "future", want_stats=True)
        assert np.array_equal(status, wst), k
        _le(np.abs(pred - want).max(), tolerance(y), k)
        assert res["stats"].n_pending == 2 * 4, k                    # counts 45..48 of either group overflow


def test_cuda_graph_replay_matches_direct_calls(engines):
    """capture(): the three launches of a small batch replayed as one CUDA graph -- same forecasts and statuses as
    direct calls, also after y changes in place, with gap rows (the queued solve) and on repeated replays (the
    graph zeroes its own work counters)."""
    import torch
    n, t, h = 3000, 400, 28
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=5, nan_frac=0.0)
    y[::7, 50:60] = np.nan
    y[11, :20] = np.nan                                              # first values missing: general pass
    eng = engines["auto"]
    _, ps, npred = eng.plan_calendar(start, t, "D", h, "future")
    yd = mmf.device_packed(y)
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    graph, out = eng.capture(yd, ps, npred, status=status)
    for rep in range(3):
        if rep:
            yd[:, 100:120] += float(rep)                             # new data, same buffers
            yd[rep, 5] = float("nan")
        graph.replay()
        torch.cuda.synchronize()
        want = eng.fit_forecast(yd, ps, npred, want_status=True)
        assert torch.equal(out, want["pred"]) or np.array_equal(out.cpu().numpy(), want["pred"].cpu().numpy(), equal_nan=True)
        assert torch.equal(status, want["status"])
    ref, wst = O.fit_forecast_packed(yd.cpu().numpy(), *_design(start, t, h))
    _le(np.abs(out.cpu().numpy() - ref).max(), tolerance(y))
    assert np.array_equal(status.cpu().numpy(), wst)


def _design(start, t, h):
    grid = O.calendar_grid(start, t + h, "D")
    return O.design_matrix(grid, t), t, t, h


def test_empty_single_and_rank_deficient_rows(engines):
    t, h = 200, 28
    start = dt.date(2019, 1, 1)
    y = np.full((6, t), np.nan, dtype=np.float32)
    y[1, 17] = 7.5                                   # one observation
    y[2] = 100 + 2 * np.arange(t)                    # a clean line
    y[3] = y[2]; y[3, 5:60] = np.nan                 # line with a hole
    y[4, 150:] = 50 + np.arange(50)                  # short tail only
    y[5] = 42.0
    want, wst = O.fit_forecast_packed(y, *_design(start, t, h))
    for k in ("warp", "auto", "tc"):
        pred, status, _ = _run(engines[k], y, start, "D", h, "future")
        assert np.array_equal(status, wst), k
        assert np.isnan(pred[0]).all()
        assert np.abs(pred[1] - 7.5).max() < 1e-3
        assert np.abs(pred[2] - (100 + 2 * np.arange(t, t + h))).max() < 0.05
        assert np.abs(pred[3] - (100 + 2 * np.arange(t, t + h))).max() < 0.05
        assert np.abs(pred[5] - 42.0).max() < 1e-3
        assert np.isfinite(pred[4]).all()
        # row 4 (50 observations for 16 columns) is ill-conditioned: its forecast is not comparable at fp32,
        # but its fitted values on the observed rows are (projection onto the span is stable)
    eng = engines["warp"]
    import torch
    days, ps, npred = eng.plan_calendar(start, t, "D", h, "future")
    fit = eng.fit_forecast(mmf.device_packed(y), 0, t).cpu().numpy()
    wfit, _ = O.fit_forecast_packed(y, _design(start, t, h)[0], t, 0, t)
    assert np.abs(fit[4, 150:] - wfit[4, 150:]).max() <= 0.05
    assert np.abs(fit[4, 150:] - y[4, 150:]).max() <= 0.05          # a line segment is fitted exactly


def test_beta_reproduces_fitted_values(engines):
    y, start = mmf.synth.daily_store_item_demand(50, 400, seed=3)
    eng = engines["warp"]
    days, ps, npred = eng.plan_calendar(start, 400, "D", 28, "holdout")
    import torch
    res = eng.fit_forecast(mmf.device_packed(y), ps, npred, want_beta=True)
    eng.synchronize()
    X = mmf.design.design_matrix(mmf.design.calendar_grid(start, 400, "D"), 372)
    fitted = res["beta"].cpu().numpy().astype(np.float64) @ X.T
    assert np.abs(fitted - res["pred"].cpu().numpy()).max() <= 5 * tolerance(y)
    res_tc = mmf.forecast_packed(mmf.device_packed(y), start, "D", 28, "future", engine=engines["tc"], want_beta=True)
    res_w = mmf.forecast_packed(mmf.device_packed(y), start, "D", 28, "future", engine=engines["warp"], want_beta=True)
    engines["tc"].synchronize(); engines["warp"].synchronize()
    assert np.abs(res_tc["beta"].cpu().numpy() - res_w["beta"].cpu().numpy()).max() <= 1e-2 * np.abs(res_w["beta"].cpu().numpy()).max()


# ---- host-buffer (C ABI with HOST pointers) path: pipelined chunks == device path --------------------
def test_host_buffer_path_matches_device_path():
    y, start = mmf.synth.daily_store_item_demand(5000, 365, seed=9, nan_frac=0.001)
    eng = mmf.ForecastEngine(chunk_series=700)        # forces 8 chunks through 3 staging buffers
    _, ps, npred = eng.plan_calendar(start, 365, "D", 28, "future")
    yp = mmf.alloc_packed(5000, 365)                  # pinned, pitched
    yp[...] = y
    res = eng.fit_forecast(yp, ps, npred, want_status=True, want_beta=True, want_stats=True)
    assert isinstance(res["pred"], np.ndarray) and res["stats"].h2d_bytes == 5000 * 365 * 4
    dev = eng.fit_forecast(mmf.device_packed(y), ps, npred, want_status=True, want_beta=True)
    eng.synchronize()
    assert np.array_equal(res["pred"], dev["pred"].cpu().numpy(), equal_nan=True)
    assert np.array_equal(res["status"], dev["status"].cpu().numpy())
    assert np.array_equal(res["beta"], dev["beta"].cpu().numpy(), equal_nan=True)
    # pageable, unpadded host array (T=365 is not a multiple of 4): the library re-pitches while staging
    res2 = eng.fit_forecast(np.ascontiguousarray(y), ps, npred)
    assert np.array_equal(res2, res["pred"], equal_nan=True)
    eng.close()


# ---- size-independent properties at BASELINE sizes -----------------------------------------------------
@pytest.mark.parametrize("kernel", ["tc", "warp"])
def test_properties_at_100k_by_1095(engines, kernel):
    """configs[2] shape: linearity, shift equivariance, row-permutation equivariance, exact lines."""
    import torch
    n, t, h = 100_000, 1095, 28
    yd, start = mmf.synth.daily_store_item_demand_torch(n, t, seed=42)
    eng = engines[kernel]
    _, ps, npred = eng.plan_calendar(start, t, "D", h, "future")
    f = lambda z: eng.fit_forecast(mmf.device_packed(z), ps, npred)
    base = f(yd)
    scale = float(yd.abs().max())
    tol = 5e-6 * scale + 1e-3
    # shift equivariance (intercept in the span): f(y + c) = f(y) + c
    _le(float((f(yd + 1000.0) - (base + 1000.0)).abs().max()), 2 * tol, "shift")
    # linearity: f(2y - 3z) = 2 f(y) - 3 f(z) with z a row-rolled copy
    lin = f(2.0 * yd - 3.0 * torch.roll(yd, 1, 0))
    _le(float((lin - (2.0 * base - 3.0 * torch.roll(base, 1, 0))).abs().max()), 8 * tol, "linearity")
    # exact answer: rows that are pure lines forecast the line
    tt = torch.arange(t + h, device="cuda", dtype=torch.float32)
    a = torch.linspace(100, 20000, 4096, device="cuda")[:, None]
    b = torch.linspace(-5, 5, 4096, device="cuda")[:, None]
    out = f(a + b * tt[None, :t])
    _le(float((out - (a + b * tt[None, t:])).abs().max()), tol, "exact lines")
    eng.synchronize()


def test_tc_and_warp_agree_on_1m_rows(engines):
    """configs[3] size on one GPU: the two independent CUDA implementations agree row by row."""
    import torch
    n, t, h = 1_000_000, 1095, 28
    yd, start = mmf.synth.daily_store_item_demand_torch(n, t, seed=43)
    outs = {}
    for k in ("tc", "warp"):
        eng = engines[k]
        _, ps, npred = eng.plan_calendar(start, t, "D", h, "future")
        outs[k] = eng.fit_forecast(yd, ps, npred)
        eng.synchronize()
    tol = 5e-6 * float(yd.abs().max()) + 1e-3
    _le(float((outs["tc"] - outs["warp"]).abs().max()), tol, "tc vs warp, 1M rows")
    # and a sampled slice against the oracle
    idx = torch.randint(0, n, (512,), device="cuda")
    ys = yd[idx].cpu().numpy()
    want, _ = _oracle(ys, start, "D", h, "future")
    _le(np.abs(outs["tc"][idx].cpu().numpy() - want).max(), tol, "512 sampled rows vs oracle")


# ---- the DataFrame / Arrow boundary ---------------------------------------------------------------------
def test_forecast_groups_matches_reference_shaped_udf():
    df = mmf.synth.reference_weekly_demand(n_skus=3)
    df = df[~((df["SKU"] == df["SKU"].iloc[0]) & (df["Date"] == dt.date(2019, 5, 6)))]   # one gap
    got = mmf.forecast_groups(df.sample(frac=1.0, random_state=0))                       # defaults = 02:341,526
    want = O.fanout_apply(df, O.build_tune_and_score_model, ("Product", "SKU"))
    assert list(got.columns) == ["Product", "SKU", "Date", "Demand", "Demand_Fitted"]
    assert len(got) == len(want) == 15 * 157
    assert (got["Product"].to_numpy() == want["Product"].to_numpy()).all()
    assert (got["SKU"].to_numpy() == want["SKU"].to_numpy()).all()
    assert (got["Date"].dt.date.to_numpy() == want["Date"].to_numpy()).all()
    assert np.array_equal(got["Demand"].to_numpy(), want["Demand"].to_numpy(), equal_nan=True)
    assert got["Demand_Fitted"].dtype == np.float32
    tol = tolerance(df["Demand"].to_numpy())
    _le(np.abs(got["Demand_Fitted"].to_numpy() - want["Demand_Fitted"].to_numpy()).max(), tol)
    # single group == literal applyInPandas drop-in (02:527)
    one = df[df["SKU"] == df["SKU"].iloc[-1]]
    g1 = mmf.forecast_groups(one)
    w1 = O.build_tune_and_score_model(one)
    _le(np.abs(g1["Demand_Fitted"].to_numpy() - w1["Demand_Fitted"].to_numpy()).max(), tol, "one group")


def test_forecast_groups_config1_daily_100x365_and_arrow():
    """BASELINE.json configs[0]: 100 (store,item) groups x 365 days through the DataFrame boundary."""
    import pandas as pd
    import pyarrow as pa
    y, start = mmf.synth.daily_store_item_demand(100, 365, seed=5)
    days = mmf.design.calendar_grid(start, 365, "D")
    df = pd.DataFrame({"store": np.repeat([f"s{i // 10}" for i in range(100)], 365),
                       "item": np.repeat([f"i{i:03d}" for i in range(100)], 365),
                       "date": np.tile(days, 100), "sales": y.reshape(-1)})
    kw = dict(keys=("store", "item"), date_col="date", value_col="sales", freq="D", horizon=28, mode="future")
    got = mmf.forecast_groups(df, **kw)
    assert len(got) == 100 * 28 and got["sales"].isna().all()
    want, _ = _oracle(y, start, "D", 28, "future")
    _le(np.abs(got["sales_Fitted"].to_numpy().reshape(100, 28) - want).max(), tolerance(y))
    tbl = mmf.forecast_table(pa.Table.from_pandas(df), **kw)
    assert tbl.schema.names == ["store", "item", "date", "sales", "sales_Fitted"]
    assert tbl.schema.field("date").type == pa.date32() and tbl.schema.field("sales_Fitted").type == pa.float32()
    assert tbl.num_rows == 2800


def test_exog_only_design_on_gpu(engines):
    df = mmf.synth.reference_weekly_demand(n_skus=1)
    got = mmf.forecast_groups(df, design="exog_only")
    want = O.fanout_apply(df, lambda g: O.build_tune_and_score_model(g, design="exog_only"), ("Product", "SKU"))
    _le(np.abs(got["Demand_Fitted"].to_numpy() - want["Demand_Fitted"].to_numpy()).max(), tolerance(df["Demand"].to_numpy()))


def test_broadcast_stores_write_every_replica(engines):
    """mmf_fit_forecast_bcast_f32 with plain device pointers: every forecast row lands in all replicas
    (the NVLink P2P / multicast variants use the same store path with peer or multicast addresses)."""
    import torch
    y, start = mmf.synth.daily_store_item_demand(1000, 400, seed=21, nan_frac=0.0)
    y[7, 10:20] = np.nan                                  # one row goes through the masked fix-up pass
    yd = mmf.device_packed(y)
    for k in ("auto", "warp"):
        eng = engines[k]
        _, ps, npred = eng.plan_calendar(start, 400, "D", 28, "future")
        want = eng.fit_forecast(yd, ps, npred)
        reps = [torch.zeros((1000, 28), device="cuda") for _ in range(3)]
        eng.fit_forecast_bcast(yd, ps, npred, [r.data_ptr() for r in reps], 28)
        torch.cuda.synchronize()
        for r in reps:
            assert torch.equal(r, want), k


@pytest.mark.parametrize("n,t", [(300, 1095), (1000, 400), (129, 157), (5, 130)])
def test_holdout_on_tensor_cores_matches_oracle_and_warp(engines, n, t):
    """Reference contract (02:484-494): a value for EVERY grid date.  auto/tc = fit kernels + predict_tc_kernel
    (wgmma GEMM + TMA stores), warp = CUDA-core path; both against the float64 oracle, incl. rows with gaps."""
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=300 + n)
    y[1, 10:40] = np.nan
    y[2, :] = np.nan                                  # empty row -> NaN everywhere, status 1
    y[3, 0] = np.nan
    want, wst = _oracle(y, start, "D", 28, "holdout")
    outs = {}
    for k in ("auto", "tc", "warp"):
        pred, status, res = _run(engines[k], y, start, "D", 28, "holdout", want_stats=True)
        assert np.array_equal(status, wst), k
        ok = wst != 1
        assert np.isnan(pred[~ok]).all()
        _le(np.abs(pred[ok] - want[ok]).max(), tolerance(y), k)
        outs[k] = pred
        assert res["stats"].kernel_used == ("warp" if k == "warp" else "tc")
    _le(np.nanmax(np.abs(outs["auto"] - outs["warp"])), tolerance(y), "auto vs warp")


# ---- device-side packer (SURVEY 8f rank 1): Arrow buffers -> padded series on the GPU ---------------------
def _long_frame(seed=0):
    import pandas as pd
    rng = np.random.default_rng(seed)
    rows = []
    for g in range(40):
        start = dt.date(2021, 1, 4) + dt.timedelta(weeks=int(rng.integers(0, 3)))     # three different calendars
        n = int(rng.integers(30, 60))
        for i in range(n):
            if rng.random() < 0.05:
                continue                                                               # gaps
            rows.append((f"prod{g % 7}", f"sku_{g:03d}", start + dt.timedelta(weeks=i), float(rng.normal(1000, 50))))
    rows.append(("prod1", "sku_001", dt.date(2021, 2, 3), 123.0))                      # off-grid (a Wednesday)
    df = pd.DataFrame(rows, columns=["Product", "SKU", "Date", "Demand"]).astype({"Demand": np.float32})
    return df.sample(frac=1.0, random_state=seed).reset_index(drop=True)               # arbitrary row order


def test_device_packer_equals_host_packer():
    import pyarrow as pa
    from mmf.packer import pack_table_device
    df = _long_frame(3)
    host = mmf.pack_groups(df, freq="W-MON", pinned=False)
    for table in (pa.Table.from_pandas(df, preserve_index=False),                                    # utf8 keys
                  pa.Table.from_pandas(df, preserve_index=False).set_column(
                      0, "Product", pa.array(df["Product"]).dictionary_encode())):                    # dictionary key
        dev = pack_table_device(table, freq="W-MON")
        assert len(dev) == len(host)
        for bd, bh in zip(dev, host):
            assert (str(bd.start), bd.t_len) == (str(bh.start), bh.t_len)
            assert bd.key_frame.values.tolist() == bh.key_frame.values.tolist()
            assert bd.y.stride(0) % 4 == 0
            assert np.array_equal(bd.y.cpu().numpy(), bh.y, equal_nan=True)


def test_forecast_groups_with_device_packer_matches_host_path():
    import pyarrow as pa
    df = _long_frame(5)
    kw = dict(freq="W-MON", horizon=8, mode="holdout")
    a = mmf.forecast_groups(df, **kw)
    b = mmf.forecast_groups(df, pack="device", **kw)
    assert list(a.columns) == list(b.columns) and len(a) == len(b)
    assert (a["SKU"].to_numpy() == b["SKU"].to_numpy()).all() and (a["Date"].to_numpy() == b["Date"].to_numpy()).all()
    assert np.array_equal(a["Demand"].to_numpy(), b["Demand"].to_numpy(), equal_nan=True)
    assert np.array_equal(a["Demand_Fitted"].to_numpy(), b["Demand_Fitted"].to_numpy(), equal_nan=True)
    t = mmf.forecast_table(pa.Table.from_pandas(df, preserve_index=False), pack="device", **kw)
    assert t.num_rows == len(a)


def test_device_packer_large_daily():
    """100k groups x 120 days = 12M long-format rows, shuffled: device packer == direct packed array."""
    import pyarrow as pa
    import torch
    from mmf.packer import pack_table_device
    n, t = 100_000, 120
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=77)
    days = mmf.design.calendar_grid(start, t, "D").astype("datetime64[D]").astype(np.int32)
    rng = np.random.default_rng(1)
    perm = rng.permutation(n * t)
    item = np.repeat(np.arange(n, dtype=np.int32), t)[perm]
    table = pa.table({"store": pa.array((item % 50).astype(np.int32)), "item": pa.array(item),
                      "date": pa.array(np.tile(days, n)[perm], type=pa.int32()).cast(pa.date32()),
                      "sales": pa.array(y.reshape(-1)[perm])})
    (b,) = pack_table_device(table, keys=("store", "item"), date_col="date", value_col="sales", freq="D", sort_keys=True)
    assert b.t_len == t and b.y.shape == (n, t)
    # sort_keys orders groups by (store, item); map back to item order
    order = b.key_frame["item"].to_numpy().astype(np.int64)
    got = torch.empty_like(b.y)
    got[torch.as_tensor(order, device="cuda", dtype=torch.long)] = b.y
    assert np.array_equal(got.cpu().numpy(), y)


def test_packer_detects_hash_collisions_and_rehashes():
    """Grouping is by 64-bit hash; verify_* compares every row's key with its group head's key.  A merged pair of
    groups (what a collision would produce) is counted; a different hash basis regroups the same keys identically."""
    import ctypes as C
    import pyarrow as pa
    import torch
    from mmf import _native as N
    from mmf import packer as PK
    df = _long_frame(7)
    table = pa.Table.from_pandas(df, preserve_index=False)
    eng = mmf.default_engine()
    lib, h = eng._lib, eng._h
    dev = torch.device("cuda", torch.cuda.current_device())
    eng.set_stream(torch.cuda.current_stream(dev).cuda_stream)
    n = table.num_rows
    for keys in (["Product", "SKU"], ["SKU"]):
        staged = PK._stage_keys(table, keys, n, dev)
        gid, first_row, G = PK.group_rows_device(lib, h, staged, n, dev)
        assert G == df.groupby(keys).ngroups
        assert PK._count_collisions(lib, h, staged, n, gid, first_row, dev) == 0
        # same partition of the rows under another hash basis (codes are numbered in hash order, so compare via heads)
        h2 = PK._hash_keys(lib, h, staged, n, dev, seed=2)
        gid2 = torch.empty_like(gid); fr2 = torch.empty_like(first_row); g2 = C.c_int32(0)
        N.check(lib.mmf_pack_group_codes(h, h2.data_ptr(), n, gid2.data_ptr(), fr2.data_ptr(), C.byref(g2)))
        assert g2.value == G and not torch.equal(h2, PK._hash_keys(lib, h, staged, n, dev, seed=1))
        pair = torch.stack([gid.long(), gid2.long()], 1).unique(dim=0)
        assert pair.shape[0] == G                                     # a bijection between the two codings
        # fake a collision: fold group 1 into group 0
        merged = torch.where(gid == 1, torch.zeros_like(gid), gid)
        bad = PK._count_collisions(lib, h, staged, n, merged, first_row, dev)
        assert bad in (int((gid == 1).sum()) * k for k in range(1, len(keys) + 1))
    # integer / dictionary keys go through verify_i32
    t2 = table.set_column(1, "SKU", pa.array(df["SKU"]).dictionary_encode())
    staged = PK._stage_keys(t2, ["Product", "SKU"], n, dev)
    gid, first_row, G = PK.group_rows_device(lib, h, staged, n, dev)
    merged = torch.where(gid == 2, torch.ones_like(gid), gid)
    c = int((gid == 2).sum())                                         # counted once per differing key column
    assert PK._count_collisions(lib, h, staged, n, merged, first_row, dev) in (c, 2 * c)


# ---- on-device model selection (SURVEY 8f rank 2): the hyperopt-loop analogue ---------------------------------
def test_model_selection_on_device_matches_oracle(engines):
    n, t, h = 600, 400, 28
    rng = np.random.default_rng(9)
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=61)
    y[:100] = np.round(5000 + rng.normal(0, 30, (100, t)))          # pure level + noise: small models should win
    tt = np.arange(t)
    y[100:200] = np.round(3000 + 4.0 * tt[None, :] + rng.normal(0, 20, (100, t)))   # level + trend
    y[5, 50:80] = np.nan                                             # gaps in the fit window
    y[6, t - 10:t - 3] = np.nan                                      # gaps in the held-out window
    y[7, t - h:] = np.nan                                            # nothing held out is observed -> full model
    y[8, :] = np.nan                                                 # empty
    cands = (1, 3, 9, 13, 16)
    grid = O.calendar_grid(start, t, "D")
    X = O.design_matrix(grid, t - h)
    want, wchoice, wmse, wst = O.select_forecast_packed(y, X, t - h, h, cands, 0, t)
    eng = engines["auto"]
    eng.plan_calendar(start, t, "D", h, "holdout")
    res = eng.fit_select_forecast(mmf.device_packed(y), h, cands, 0, t)
    import torch
    torch.cuda.synchronize()
    pred, choice, mse, st = (res[k].cpu().numpy() for k in ("pred", "choice", "mse", "status"))
    assert np.array_equal(st, wst)
    assert choice[8] == 0 and np.isnan(pred[8]).all() and choice[7] == 16
    # every row: the choice is optimal up to fp32 noise (it may differ from the oracle's only where two candidates score
    # within that noise), the MSE and the prediction of the GPU's own choice match the float64 oracle
    from test_gpu_edges import check_selection
    check_selection({"pred": pred, "choice": choice, "mse": mse, "status": st}, y, X, t - h, h, cands, 0, t)
    assert (choice[:100] <= 3).mean() > 0.5 and (choice[100:200] <= 9).mean() > 0.5      # simple series -> small models


def test_forecast_groups_with_selection():
    df = mmf.synth.reference_weekly_demand(n_skus=2)
    full = mmf.forecast_groups(df)
    sel = mmf.forecast_groups(df, select=(1, 3, 13, 16))
    sel_dev = mmf.forecast_groups(df, select=(1, 3, 13, 16), pack="device")
    assert list(sel.columns) == list(full.columns) and len(sel) == len(full)
    assert np.array_equal(sel["Demand_Fitted"].to_numpy(), sel_dev["Demand_Fitted"].to_numpy())
    want = O.fanout_apply(df, O.build_tune_and_score_model, ("Product", "SKU"))          # full model, for scale only
    assert np.isfinite(sel["Demand_Fitted"].to_numpy()).all()
    # the selected model can only do better (or equal) on the held-out 40 weeks than ... itself being a candidate:
    def hold_mse(frame):
        e = (frame["Demand"] - frame["Demand_Fitted"]).to_numpy().reshape(-1, 157)[:, -40:]
        return (e * e).mean(axis=1)
    assert (hold_mse(sel) <= hold_mse(full) * (1 + 1e-4)).all()
    assert len(want) == len(sel)


def test_long_horizon_future_mode_uses_predict_kernel(engines):
    """horizon > 64 in future mode: fit kernels + predict_tc_kernel, against the oracle and the warp kernel."""
    y, start = mmf.synth.daily_store_item_demand(700, 500, seed=88)
    want, _ = _oracle(y, start, "D", 120, "future")
    for k in ("auto", "warp"):
        pred, status, _ = _run(engines[k], y, start, "D", 120, "future")
        assert pred.shape == (700, 120) and (status == 0).all()
        _le(np.abs(pred - want).max(), tolerance(y), k)


@pytest.mark.parametrize("horizon", [1, 7, 30, 40, 64])
def test_epilogue_store_paths_for_various_horizons(engines, horizon):
    """bulk-store epilogue (n_pred % 4 == 0, <= 28), vectorised stores (<= 64), scalar stores (odd n_pred)."""
    y, start = mmf.synth.daily_store_item_demand(517, 300, seed=500 + horizon)
    y[11, 100:130] = np.nan
    want, wst = _oracle(y, start, "D", horizon, "future")
    for k in ("auto", "warp"):
        pred, status, _ = _run(engines[k], y, start, "D", horizon, "future")
        assert pred.shape == (517, horizon) and np.array_equal(status, wst)
        _le(np.abs(pred - want).max(), tolerance(y), (k, horizon))


def test_device_packer_null_keys_null_dates_and_duplicates():
    """ADVICE round 1: a null key is its own group (distinct from ""), like the host packer; a null date is rejected;
    duplicate (key, date) rows raise like the reference's asfreq (02:423) instead of racing in the scatter."""
    import pandas as pd
    import pyarrow as pa
    from mmf.packer import pack_table_device
    rows = []
    for sku in ("", None, "a"):
        for i in range(12):
            rows.append(("p", sku, dt.date(2021, 1, 4) + dt.timedelta(weeks=i), float(10 * i + (0 if sku is None else 1))))
    df = pd.DataFrame(rows, columns=["Product", "SKU", "Date", "Demand"]).astype({"Demand": np.float32})
    table = pa.Table.from_pandas(df, preserve_index=False)
    assert table.column("SKU").null_count == 12
    host = mmf.frames.pack_table_host(table, freq="W-MON", pinned=False)
    dev = pack_table_device(table, freq="W-MON")
    assert len(host) == len(dev) == 1 and dev[0].y.shape[0] == host[0].y.shape[0] == 3
    hk = [None if pd.isna(v) else v for v in host[0].key_frame["SKU"].tolist()]
    dk = [None if pd.isna(v) else v for v in dev[0].key_frame["SKU"].tolist()]
    got = {k: dev[0].y[i].cpu().numpy() for i, k in enumerate(dk)}
    want = {k: host[0].y[i] for i, k in enumerate(hk)}
    assert set(got) == set(want) == {"", None, "a"}
    for k in want:
        assert np.array_equal(got[k], want[k], equal_nan=True), k
    bad = pa.Table.from_pandas(df.assign(Date=[None] + df["Date"].tolist()[1:]), preserve_index=False)
    with pytest.raises(ValueError, match="null"):
        pack_table_device(bad, freq="W-MON")
    dup = pa.Table.from_pandas(pd.concat([df, df.iloc[[5, 20]]], ignore_index=True), preserve_index=False)
    with pytest.raises(ValueError, match="duplicate"):
        pack_table_device(dup, freq="W-MON")


def test_device_packer_equals_pandas_asfreq_on_random_frames():
    """The device packer against pandas itself (what the reference runs per group, 02:422-423: sort_values + set_index +
    asfreq): random groups, start dates, missing and off-grid dates, NaN demand, shuffled rows, daily and weekly grids."""
    hyp = pytest.importorskip("hypothesis")
    import pandas as pd
    import pyarrow as pa
    from mmf.packer import pack_table_device
    st = hyp.strategies

    @st.composite
    def frames(draw):
        freq = draw(st.sampled_from(["D", "W-MON"]))
        step = 1 if freq == "D" else 7
        rows = []
        for gi in range(draw(st.integers(1, 6))):
            start = dt.date(2021, 1, 4) + dt.timedelta(days=step * draw(st.integers(0, 30)))
            n = draw(st.integers(1, 60))
            keep = draw(st.lists(st.booleans(), min_size=n, max_size=n))
            if not any(keep):
                keep[0] = True
            first, last = keep.index(True), n - 1 - keep[::-1].index(True)
            for i in range(n):
                if keep[i]:
                    v = draw(st.one_of(st.integers(0, 60000).map(float), st.just(float("nan"))))
                    rows.append(("P%d" % (gi % 2), "S%d" % gi, start + dt.timedelta(days=step * i), v))
                    if step == 7 and first < i < last and draw(st.integers(0, 9)) == 0:
                        rows.append(("P%d" % (gi % 2), "S%d" % gi, start + dt.timedelta(days=step * i + 2), 777.0))
        order = draw(st.permutations(list(range(len(rows)))))
        df = pd.DataFrame([rows[i] for i in order], columns=["Product", "SKU", "Date", "Demand"])
        df["Date"] = pd.to_datetime(df["Date"]).dt.date
        return freq, df.astype({"Demand": np.float32})

    @hyp.settings(max_examples=40, deadline=None, derandomize=True, database=None,
                  suppress_health_check=list(hyp.HealthCheck))
    @hyp.given(frames())
    def check(case):
        freq, df = case
        ref = df.assign(Date=pd.to_datetime(df["Date"]))
        want = {}
        for key, g in ref.groupby(["Product", "SKU"], sort=True):
            s = g.sort_values("Date").set_index("Date")["Demand"].asfreq(freq)
            want[key] = (str(s.index[0].date()), len(s), s.to_numpy(dtype=np.float32))
        got = {}
        for b in pack_table_device(pa.Table.from_pandas(df, preserve_index=False), freq=freq):
            yb = b.y.cpu().numpy()
            for r, key in enumerate(b.key_frame.itertuples(index=False)):
                got[(key.Product, key.SKU)] = (str(b.start), b.t_len, yb[r, :b.t_len])
        assert got.keys() == want.keys()
        for key, (start, t_len, vals) in want.items():
            gs, gt, gv = got[key]
            assert (gs[:10], gt) == (start, t_len), key
            assert np.array_equal(gv, vals, equal_nan=True), key

    check()
