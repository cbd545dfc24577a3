"""GPU (-m gpu): BASELINE.json's configurations at their full sizes against the oracle, the negative control that
proves the stated tolerance guards the tensor-core path's 3-term tf32 split, the fused multi-GPU path against the
oracle (needs >= 2 GPUs, skipped otherwise), and the CUDA-graph / scratch lifetime rules of the C ABI.

Every CUDA call goes ctypes -> libmmf.so (include/mmf.h); the oracle (oracle/, float64) is only the checker."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import mmf
from conftest import ROOT, record_err, tolerance
from oracle import mmf_oracle as O
from test_gpu_ragged import _frame_ratio

pytestmark = pytest.mark.gpu


def _design(start, t, h, mode="future"):
    if mode == "holdout":
        grid = O.calendar_grid(start, t, "D")
        return O.design_matrix(grid, t - h), t - h, 0, t
    grid = O.calendar_grid(start, t + h, "D")
    return O.design_matrix(grid, t), t, t, h


def _le(err, tol, what=""):
    name = os.environ.get("PYTEST_CURRENT_TEST", "?").split("::")[-1].split(" ")[0]
    record_err(name, err, tol, what=str(what))
    assert err <= tol, (what, float(err), float(tol))


# ---- BASELINE configs[2]: 100k x 1,095, ALL rows against the oracle ------------------------------------
@pytest.mark.parametrize("kernel", ["tc", "warp"])
def test_parity_config3_100k_by_1095_all_rows(kernel):
    """Every one of the 100,000 series against the float64 oracle (its C restatement, pinned to the NumPy oracle
    by tests/test_oracle.py, runs them in a fraction of a second on the host cores)."""
    import torch
    n, t, h = 100_000, 1095, 28
    yd, start = mmf.synth.daily_store_item_demand_torch(n, t, seed=4242)
    y = yd.cpu().numpy()
    want, wst = O.fit_forecast_packed_c(y, *_design(start, t, h))
    eng = mmf.ForecastEngine(kernel=kernel)
    res = mmf.forecast_packed(yd, start, "D", h, "future", engine=eng, want_status=True, want_stats=True)
    torch.cuda.synchronize()
    pred = res["pred"].cpu().numpy()
    assert res["stats"].kernel_used == kernel
    assert np.array_equal(res["status"].cpu().numpy(), wst) and (wst == 0).all()
    _le(np.abs(pred - want).max(), tolerance(y), kernel)
    eng.close()


def test_parity_config3_holdout_and_gaps_all_rows():
    """The reference contract (a value for every date, 02:484-494) and the gap path at configs[2] size, all rows."""
    import torch
    n, t, h = 100_000, 1095, 28
    yd, start = mmf.synth.daily_store_item_demand_torch(n, t, seed=4243, nan_frac=0.01)
    y = yd.cpu().numpy()
    eng = mmf.ForecastEngine()
    for mode in ("future", "holdout"):
        X, t_fit, ps, npred = _design(start, t, h, mode)
        want, wst = O.fit_forecast_packed_c(y, X, t_fit, ps, npred)
        res = mmf.forecast_packed(yd, start, "D", h, mode, engine=eng, want_status=True)
        torch.cuda.synchronize()
        assert np.array_equal(res["status"].cpu().numpy(), wst)
        # ~11 gaps out of 1,095 rows: the per-series Gram stays well conditioned (pivot ratios ~ 0.99)
        _le(np.abs(res["pred"].cpu().numpy() - want).max(), 2 * tolerance(y), mode)
    eng.close()


# ---- BASELINE configs[4]: 10M x 365 --------------------------------------------------------------------
def test_config5_10m_by_365_device_and_host_spill():
    """10 M series x 365 days (14.6 GB): (a) device-resident, (b) streamed from pinned host memory in chunks through
    the 3-slot H2D / kernel / D2H pipeline (the "host-DRAM spill" of configs[4]).  (a) == (b) bit for bit on all
    10 M rows, every status is OK, and an 8,192-row sample agrees with the oracle."""
    import torch
    n, t, h = 10_000_000, 365, 28
    free, _ = torch.cuda.mem_get_info()
    if free < 40e9:
        pytest.skip("needs 40 GB of free device memory")
    yd, start = mmf.synth.daily_store_item_demand_torch(n, t, seed=55)       # [n, 365] view of a pitch-368 buffer
    eng = mmf.ForecastEngine()
    _, ps, npred = eng.plan_calendar(start, t, "D", h, "future")
    dev = eng.fit_forecast(yd, ps, npred, want_status=True)
    torch.cuda.synchronize()
    assert int((dev["status"] != 0).sum()) == 0
    idx = torch.randint(0, n, (8192,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    ys = yd[idx].cpu().numpy()
    want, _ = O.fit_forecast_packed_c(ys, *_design(start, t, h))
    _le(np.abs(dev["pred"][idx].cpu().numpy() - want).max(), tolerance(ys), "device-resident, 8192 sampled rows")
    # host spill: the same rows from page-locked host memory, chunked
    try:
        yh = mmf.alloc_packed(n, t)                       # 14.7 GB pinned
        oh = mmf.pinned_empty((n, h))
    except mmf.MmfError:
        pytest.skip("cannot pin 15 GB of host memory on this box")
    torch.from_numpy(yh).copy_(yd)
    eng2 = mmf.ForecastEngine(chunk_series=262_144)
    eng2.plan_calendar(start, t, "D", h, "future")
    res = eng2.fit_forecast(yh, ps, npred, out=oh, want_status=True, want_stats=True)
    # integer-valued demand: on a single-GPU host the path narrows each chunk to uint16 on the way (exactly), half the
    # bytes cross PCIe; with several GPUs visible automatic mode leaves the float32 copies alone
    assert n * t * 2 <= res["stats"].h2d_bytes <= n * t * 4 and res["stats"].d2h_bytes >= n * h * 4
    assert int((res["status"] != 0).sum()) == 0
    got = torch.from_numpy(oh)
    ref = dev["pred"].cpu()
    assert torch.equal(got, ref), "host-spill path differs from the device-resident path"
    record_err("test_config5_10m_by_365_device_and_host_spill", 0.0, 0.0, what="host spill == device bit for bit",
               e2e_series_per_s=n / (res["stats"].total_ms * 1e-3))
    eng.close()
    eng2.close()
    mmf.release_pinned_pool()


# ---- negative control: the tolerance must catch a tf32-grade tensor-core path ------------------------------
_NEGCTL = r"""
import json, sys
import numpy as np, torch
sys.path.insert(0, {root!r})
import mmf
from oracle import mmf_oracle as O
y, start = mmf.synth.daily_store_item_demand(10_000, 1095, seed=1234)
grid = O.calendar_grid(start, 1095 + 28, "D")
want, _ = O.fit_forecast_packed_c(y, O.design_matrix(grid, 1095), 1095, 1095, 28)
eng = mmf.ForecastEngine(kernel="tc")
pred = mmf.forecast_packed(mmf.device_packed(y), start, "D", 28, "future", engine=eng)
torch.cuda.synchronize()
err = np.abs(pred.cpu().numpy() - want)
print(json.dumps({{"lib": mmf.LIB_PATH, "max_err": float(err.max()), "p99_row_err": float(np.percentile(err.max(axis=1), 99)),
                  "rows_over": int((err.max(axis=1) > {tol}).sum()), "max_abs_y": float(np.abs(y).max())}}))
"""


def test_negative_control_without_lo_term_fails_config2():
    """BASELINE configs[1] (10k x 1,095, all rows) through two builds of the same ABI: the product library must pass
    the stated tolerance, and tests/_build/libmmf_negctl.so -- the tensor-core kernel compiled WITHOUT the lo*A_hi MMA of
    the 3-term tf32 split (-DMMF_TC_NO_LO_TERM) -- must FAIL it.  If the second half ever passes, the tolerance no
    longer guards the property that makes the tensor-core path legitimate."""
    neg = os.path.join(ROOT, "tests", "_build", "libmmf_negctl.so")
    assert os.path.exists(neg), "negative-control library missing: run __graft_entry__.build()"
    y, _ = mmf.synth.daily_store_item_demand(10_000, 1095, seed=1234)
    tol = tolerance(y)
    out = {}
    for name, lib in (("product", ""), ("negctl", neg)):
        env = dict(os.environ)
        env.pop("MMF_LIB", None)
        if lib:
            env["MMF_LIB"] = lib
        r = subprocess.run([sys.executable, "-c", _NEGCTL.format(root=ROOT, tol=tol)], env=env, capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        out[name] = json.loads(r.stdout.strip().splitlines()[-1])
        record_err("test_negative_control_without_lo_term_fails_config2", out[name]["max_err"], tol, what=name,
                   **{k: v for k, v in out[name].items() if k != "max_err"})
    assert out["negctl"]["lib"].endswith("libmmf_negctl.so") and out["product"]["lib"].endswith("libmmf.so")
    assert out["product"]["max_err"] <= tol, out
    assert out["negctl"]["max_err"] > tol, ("the tolerance does not detect a missing lo*A_hi term", out)
    assert out["negctl"]["rows_over"] >= 100, out            # not one unlucky row: the whole batch degrades


# ---- the fused multi-GPU path against the oracle -------------------------------------------------------------
@pytest.mark.parametrize("mode", ["p2p", "multicast-bulk"])
def test_symmetric_table_fused_gather_matches_oracle(mode, tmp_path):
    """world_size >= 2 (one process per GPU, torchrun): every rank fits its shard and the fit kernel's epilogue
    stores each forecast tile into every rank's copy of the table (NVLink P2P bulk stores / NVLS multicast); every
    rank's whole table must equal the ORACLE's forecasts of all shards (not just NCCL's gather of the same numbers),
    including rows with gaps (fix-up kernels write through the same destinations)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    world = min(torch.cuda.device_count(), 8)
    out = str(tmp_path / f"symm_{mode}.json")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", "29617", os.path.join(ROOT, "tests", "_symm_worker.py"),
           "--mode", mode, "--out", out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
    with open(out) as f:
        res = json.load(f)
    if res.get("skipped"):
        pytest.skip(res["skipped"])
    assert res["world"] == world
    for rk in res["ranks"]:
        _le(rk["max_err_vs_oracle"], res["tol"], f"rank {rk['rank']} {mode}")
        assert rk["status_equal"] and rk["equals_nccl_gather"], rk


# ---- CUDA-graph capture: counters and scratch lifetime (ADVICE round 1) ------------------------------------
def test_capture_does_not_leave_stale_counters_for_eager_calls():
    """The work counters are ping-ponged between eager calls and zeroed by the previous call's kernel; a capture only
    RECORDS its kernels.  After capturing on gappy data (every row queues a record), eager calls and further
    captures must still start from zero counters: no out-of-bounds record slots, no stale DEFERRED statuses."""
    import torch
    n, t, h = 4000, 400, 28
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=77, nan_frac=0.02)       # every row has gaps
    want, wst = O.fit_forecast_packed(y, *_design(start, t, h))
    eng = mmf.ForecastEngine()
    _, ps, npred = eng.plan_calendar(start, t, "D", h, "future")
    yd = mmf.device_packed(y)
    graphs = []
    for rep in range(3):                                  # several captures in a row, eager calls in between
        st = torch.full((n,), -7, dtype=torch.int32, device="cuda")
        g, out = eng.capture(yd, ps, npred, status=st)
        graphs.append((g, out, st))
        res = eng.fit_forecast(yd, ps, npred, want_status=True, want_stats=True)      # eager, no replay before it
        torch.cuda.synchronize()
        assert np.array_equal(res["status"].cpu().numpy(), wst), rep
        assert res["stats"].n_pending < n
        _le(np.abs(res["pred"].cpu().numpy() - want).max(), 2 * tolerance(y), f"eager after capture {rep}")
    for g, out, st in graphs:                             # replays interleaved with eager calls
        g.replay()
        res = eng.fit_forecast(yd, ps, npred, want_status=True)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(st.cpu().numpy(), wst) and np.array_equal(res["status"].cpu().numpy(), wst)
        assert torch.equal(out, res["pred"])
    for g, _, _ in graphs:
        g.close()
    eng.close()


def test_captured_graph_pins_scratch_and_plan():
    """A captured graph holds raw pointers into the context: re-planning or a larger batch must be refused while it
    is alive (MMF_E_UNSUPPORTED), and work again once it is closed."""
    import torch
    n, t, h = 2000, 300, 28
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=3, nan_frac=0.01)
    eng = mmf.ForecastEngine()
    _, ps, npred = eng.plan_calendar(start, t, "D", h, "future")
    yd = mmf.device_packed(y)
    g, out = eng.capture(yd, ps, npred)
    big = mmf.device_packed(np.tile(y, (3, 1)))
    with pytest.raises(mmf.MmfError) as e1:
        eng.fit_forecast(big, ps, npred)                  # needs 3x the record scratch
    assert e1.value.code == -3 and "graph" in str(e1.value)
    with pytest.raises(mmf.MmfError) as e2:
        eng.plan_calendar(start, t, "D", 14, "future")    # another design would free the planned one
    assert e2.value.code == -3
    g.replay()                                            # still valid
    torch.cuda.synchronize()
    small = eng.fit_forecast(yd[:500], ps, npred)         # fits the existing scratch (the status scratch, which no
                                                          # graph references, may still grow): allowed
    torch.cuda.synchronize()
    assert torch.equal(small, out[:500])
    g.close()
    eng.fit_forecast(big, ps, npred)                      # unpinned: scratch may grow again
    eng.plan_calendar(start, t, "D", 14, "future")
    torch.cuda.synchronize()
    eng.close()


def test_select_rejects_too_many_held_out_rows():
    import torch
    t, hold = 5000, 3600                                  # > MMF_SELECT_MAX_HOLD
    y, start = mmf.synth.daily_store_item_demand(8, t, seed=1)
    eng = mmf.ForecastEngine()
    eng.plan_calendar(start, t, "D", hold, "holdout")
    with pytest.raises(mmf.MmfError) as e:
        eng.fit_select_forecast(mmf.device_packed(y), hold, (1, 16), 0, t)
    assert e.value.code == -3 and "n_hold" in str(e.value)
    eng.close()


def test_mostly_missing_weekly_rows_take_the_direct_gram():
    """Reference workload shape (weekly, 117 fit rows): rows with 59..88 missing weeks.  The in-stream gap path would
    form G_i = I - sum a a^T with more than half the rows missing (catastrophic cancellation); they are routed to
    the general pass, which builds the Gram over the observed rows -- so kernel=auto and kernel=warp agree."""
    rng = np.random.default_rng(5)
    df = mmf.synth.reference_weekly_demand(n_skus=2)
    b = mmf.pack_groups(df, freq="W-MON", pinned=False)[0]
    y0 = b.y[:1]
    rows = []
    for miss in (30, 58, 59, 60, 70, 80, 88):
        r = y0[0].copy()
        r[rng.choice(np.arange(1, 117), size=miss, replace=False)] = np.nan
        rows.append(r)
    y = np.stack(rows).astype(np.float32)
    t, h = y.shape[1], 40
    grid = O.calendar_grid(b.start, t, "W-MON")
    want, wst, _, ratio = O.fit_forecast_packed(y, O.design_matrix(grid, t - h), t - h, 0, t, return_gamma=True)
    outs = {}
    for k in ("auto", "warp"):
        eng = mmf.ForecastEngine(kernel=k)
        res = mmf.forecast_packed(mmf.device_packed(y), b.start, "W-MON", h, "holdout", engine=eng, want_status=True)
        outs[k] = res["pred"].cpu().numpy()
        assert np.array_equal(res["status"].cpu().numpy(), wst), k
        tol = tolerance(y) / np.minimum(1.0, ratio / 0.25)
        rel = np.abs(outs[k] - want).max(axis=1) / tol
        _le(rel.max(), 1.0, f"{k}: worst row error / row tolerance")
        eng.close()
    heavy = np.array([np.isnan(r[:t - h]).sum() * 2 > (t - h) for r in y])
    assert heavy.any()
    # same kernel and Gram route on both paths (row grouping inside a warp differs, so not the same bits)
    _le(np.abs(outs["auto"][heavy] - outs["warp"][heavy]).max(), tolerance(y), "auto vs warp, mostly-missing rows")


# ---- integer demand columns (int16 / uint16 / int32): half the PCIe bytes, bit-equal forecasts --------------------
@pytest.mark.parametrize("dtype", ["uint16", "int16", "int32"])
def test_integer_ingest_is_bit_equal_to_float32_ingest(dtype):
    """mmf_fit_forecast_int: the reference's demand is integer valued (01-data-generator.py:304 round()); an integer
    series buffer with the type's sentinel for missing values must produce exactly the float32 path's forecasts and
    statuses -- host buffers (chunked, ragged last chunk, pitched and unpitched rows) and device buffers."""
    import torch
    n, t, h = 3001, 365, 28
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=31, nan_frac=0.003)
    y = np.where(np.isfinite(y), np.clip(y, 0, 32000), np.nan).astype(np.float32)
    y[17, :] = np.nan                                            # empty row
    eng = mmf.ForecastEngine(chunk_series=700)
    _, ps, npred = eng.plan_calendar(start, t, "D", h, "future")
    want = eng.fit_forecast(mmf.device_packed(y), ps, npred, want_status=True)
    torch.cuda.synchronize()
    wp, ws = want["pred"].cpu().numpy(), want["status"].cpu().numpy()
    yi = mmf.alloc_packed(n, t, dtype=dtype)                     # pinned, 16-B row pitch
    mmf.to_integer_demand(y, dtype, out=yi)
    res = eng.fit_forecast(yi, ps, npred, want_status=True, want_stats=True)
    assert res["stats"].h2d_bytes == n * t * np.dtype(dtype).itemsize
    assert np.array_equal(res["pred"], wp, equal_nan=True) and np.array_equal(res["status"], ws)
    res2 = eng.fit_forecast(np.ascontiguousarray(yi), ps, npred)  # pageable, unpitched rows (ld = 365)
    assert np.array_equal(res2, wp, equal_nan=True)
    if dtype != "uint16":                                         # torch has no general uint16 support
        yd = torch.from_numpy(np.ascontiguousarray(yi)).cuda()
        res3 = eng.fit_forecast(yd, ps, npred, want_status=True)
        torch.cuda.synchronize()
        assert np.array_equal(res3["pred"].cpu().numpy(), wp, equal_nan=True)
        assert np.array_equal(res3["status"].cpu().numpy(), ws)
    with pytest.raises(ValueError):
        mmf.to_integer_demand(y + 0.5, dtype)
    eng.close()


# ---- ragged batches: groups on many calendars, ONE launch ---------------------------------------------------------
def _ragged_case(seed=0, short=64):
    """Calendars with different first dates AND lengths, group counts around the 128-row tile edge, rows with gaps,
    rows the streaming pass must hand to the general pass, an empty row; columns beyond a row's own length hold NaN
    on purpose (the per-calendar tensor maps must clip them away)."""
    import datetime as dt
    rng = np.random.default_rng(seed)
    cals = [(dt.date(2019, 1, 1), 400, 300), (dt.date(2019, 3, 5), 333, 127), (dt.date(2018, 7, 9), 365, 128),
            (dt.date(2020, 2, 1), 97, 129), (dt.date(2019, 1, 2), 400, 1), (dt.date(2017, 12, 25), short, 5),
            (dt.date(2019, 6, 30), 250, 700)]
    t_max = max(t for _, t, _ in cals)
    ld = (t_max + 3) & ~3
    blocks, rows = [], [0]
    for ci, (start, t, n) in enumerate(cals):
        yb, _ = mmf.synth.daily_store_item_demand(n, t, seed=1000 + ci, end=np.datetime64(start) + np.timedelta64(t - 1, "D"))
        full = np.full((n, ld), np.nan, dtype=np.float32)
        full[:, :t] = yb
        if n >= 5:
            full[1, 10:25] = np.nan                           # in-stream gap path
            full[2, :9] = np.nan                              # first values missing: general pass (per-calendar launch)
            full[3, :t] = np.nan                              # empty
            full[4, rng.choice(np.arange(1, t), size=min(60, t // 3), replace=False)] = np.nan
        blocks.append(full)
        rows.append(rows[-1] + n)
    return cals, np.concatenate(blocks), np.array(rows, dtype=np.int64), ld


def test_ragged_calendars_one_launch_matches_oracle_and_per_bucket_calls():
    import torch
    h = 28
    cals, y, rows, ld = _ragged_case()
    eng = mmf.ForecastEngine()
    dates = eng.plan_calendars([c[0] for c in cals], [c[1] for c in cals], "D", h)
    assert dates.shape == (len(cals), h)
    yd = torch.from_numpy(y).cuda()
    res = eng.fit_forecast_ragged(yd, rows, want_status=True, want_stats=True)
    torch.cuda.synchronize()
    pred, status = res["pred"].cpu().numpy(), res["status"].cpu().numpy()
    assert res["stats"].n_pending >= sum(1 for c in cals if c[2] >= 5)          # the leading-gap rows
    eng1 = mmf.ForecastEngine()
    for ci, (start, t, n) in enumerate(cals):
        r0, r1 = int(rows[ci]), int(rows[ci + 1])
        yb = y[r0:r1, :t]
        grid = O.calendar_grid(start, t + h, "D")
        want, wst, _, ratio = O.fit_forecast_packed(yb, O.design_matrix(grid, t), t, t, h, return_gamma=True)
        assert np.array_equal(status[r0:r1], wst), ci
        assert str(dates[ci][0]) == str(np.datetime64(start) + np.timedelta64(t, "D"))
        ok = wst != 1
        assert np.isnan(pred[r0:r1][~ok]).all()
        from conftest import forecast_leverage
        lev = forecast_leverage(O.design_matrix(grid, t), t, t, h)
        tol = tolerance(yb, lev) / np.minimum(1.0, ratio[ok] / 0.25)
        rel = np.abs(pred[r0:r1][ok] - want[ok]).max(axis=1) / tol
        _le(rel.max(), 1.0, f"calendar {ci}: t={t} n={n} leverage {lev:.3g}")
        # the same rows through the single-calendar entry point: same kernel, same arithmetic per row
        single = mmf.forecast_packed(mmf.device_packed(yb), start, "D", h, "future", engine=eng1).cpu().numpy()
        assert np.array_equal(single, pred[r0:r1], equal_nan=True), ci
    eng.close()
    eng1.close()


def test_ragged_rejects_what_it_cannot_do():
    import torch
    eng = mmf.ForecastEngine()
    with pytest.raises(mmf.MmfError):
        eng.plan_calendars(["2020-01-01"], [20], "D", 28)                        # < 33 fit rows
    eng.plan_calendars(["2020-01-01"], [100], "D", 80)                           # > 64 forecast rows: predict kernel
    with pytest.raises(ValueError):
        eng.plan_calendars(["2020-01-01"], [100], "D", 120, mode="holdout")      # nothing left to fit
    eng.plan_calendars(["2020-01-01", "2020-02-01"], [100, 90], "D", 28)
    y = torch.zeros((10, 100), device="cuda")
    with pytest.raises(mmf.MmfError):
        eng.fit_forecast_ragged(y, [0, 4, 9])                                    # does not end at n
    eng.close()


def test_forecast_groups_many_calendars_future_mode_uses_one_ragged_launch():
    """DataFrame boundary: groups with different first dates / lengths (the reference re-grids each group on its own
    calendar, 02:422-423) in future mode go through the ragged launch and match the per-group oracle UDF."""
    import pandas as pd
    rng = np.random.default_rng(3)
    frames = []
    for g in range(60):
        t = int(rng.integers(40, 90))
        start = np.datetime64("2021-01-04") + np.timedelta64(7 * int(rng.integers(0, 6)), "D")
        days = start + np.arange(t) * np.timedelta64(7, "D")
        vals = np.round(1000 + 5 * np.arange(t) + rng.normal(0, 20, t)).astype(np.float32)
        keep = rng.random(t) > 0.04
        keep[0] = keep[-1] = True
        frames.append(pd.DataFrame({"Product": f"p{g % 5}", "SKU": f"s{g:03d}", "Date": days[keep].astype("datetime64[ns]"),
                                    "Demand": vals[keep]}))
    df = pd.concat(frames, ignore_index=True).sample(frac=1.0, random_state=1)
    df["Date"] = df["Date"].dt.date
    kw = dict(freq="W-MON", horizon=8, mode="future")
    got = mmf.forecast_groups(df, **kw)
    want = O.fanout_apply(df, lambda p: O.build_tune_and_score_model(p, **kw), ("Product", "SKU"))
    assert len(got) == len(want) == 60 * 8
    assert (got["SKU"].to_numpy() == want["SKU"].to_numpy()).all()
    assert (got["Date"].dt.date.to_numpy() == want["Date"].to_numpy()).all()
    # weekly histories of 40-90 points extrapolated 8 weeks: every group within tolerance x max(1, the leverage of its
    # own calendar) x its mask factor
    _le(_frame_ratio(df, got, want, **kw, design="trend_season_exog"), 1.0, "ragged DataFrame batch vs per-group oracle UDF")


# ---- host-side narrowing of float32 chunks (half the PCIe bytes), exact or not used ------------------------------------
def test_host_narrowing_is_exact_or_not_used():
    """mmf_fit_forecast_f32 with HOST float32 buffers: chunks whose finite values are all integers in [0, 65534] cross
    PCIe as uint16 (narrowed on host threads, widened on the device); any other chunk goes as float32.  Either way the
    forecasts equal the device-resident float32 path bit for bit."""
    import torch
    n, t, h = 6000, 365, 28
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=12, nan_frac=0.002)
    y[100, :] = np.nan
    y[101, 5] = np.inf
    dev = mmf.ForecastEngine()
    _, ps, npred = dev.plan_calendar(start, t, "D", h, "future")

    def device_result(arr):
        r = dev.fit_forecast(mmf.device_packed(arr), ps, npred, want_status=True)
        torch.cuda.synchronize()
        return r["pred"].cpu().numpy(), r["status"].cpu().numpy()

    for mode, chunk in (("on", 700), ("on", 6000), ("off", 700)):
        eng = mmf.ForecastEngine(chunk_series=chunk, host_narrow=mode, host_threads=4)
        eng.plan_calendar(start, t, "D", h, "future")
        yp = mmf.alloc_packed(n, t)
        yp[...] = y
        res = eng.fit_forecast(yp, ps, npred, want_status=True, want_stats=True)
        wp, ws = device_result(y)
        assert np.array_equal(res["pred"], wp, equal_nan=True) and np.array_equal(res["status"], ws), (mode, chunk)
        # (every 3rd chunk crosses as float32 on purpose: the link is the faster of the two resources, see mmf_api.cu)
        direct_rows = sum(min(chunk, n - off) for it, off in enumerate(range(0, n, chunk)) if it % 3 == 2)
        want_bytes = (n - direct_rows) * t * 2 + direct_rows * t * 4 if mode == "on" else n * t * 4
        assert res["stats"].h2d_bytes == want_bytes, (mode, chunk)
        # pageable, unpitched rows narrow too
        res2 = eng.fit_forecast(np.ascontiguousarray(y), ps, npred)
        assert np.array_equal(res2, wp, equal_nan=True)
        # a chunk with a value uint16 cannot carry exactly falls back to float32 from that chunk on
        for badval in (0.5, -3.0, 70000.0):
            y2 = y.copy()
            y2[2200, 17] = badval                              # chunk 3 of the 700-row chunks: a narrowed one
            yp[...] = y2
            r3 = eng.fit_forecast(yp, ps, npred, want_stats=True)
            wp3, _ = device_result(y2)
            assert np.array_equal(r3["pred"], wp3, equal_nan=True), (mode, chunk, badval)
            if mode == "on" and chunk == 700:
                # chunks 0-1 narrowed, chunk 2 direct by design, chunk 3 cannot be narrowed: float32 from there on
                assert r3["stats"].h2d_bytes == 1400 * t * 2 + (n - 1400) * t * 4
        eng.close()
    dev.close()


def test_retired_tuning_options_have_no_effect():
    """mmf_config.tc_variant = 3 (a balanced launch) and stream_solve = 1 (a solve of the series with gaps beside the
    tensor-core kernel) are accepted and ignored: forecasts, statuses and coefficients are bit-equal to the default and
    the call launches the same kernels -- on a batch large enough, and with enough gaps, for either to have applied."""
    import torch
    n, t, h = 70_000, 400, 28
    y, start = mmf.synth.daily_store_item_demand(n, t, seed=91, nan_frac=0.01)
    y[5, :9] = np.nan                                         # general pass (fit_warp) queues a record of its own
    y[6, :] = np.nan
    yd = mmf.device_packed(y)
    base = mmf.ForecastEngine(kernel="tc")
    base.plan_calendar(start, t, "D", h, "future")
    want = base.fit_forecast(yd, t, h, want_status=True, want_beta=True, want_stats=True)
    torch.cuda.synchronize()
    assert want["stats"].n_pending > 0 and int((want["status"] == 0).sum()) < n
    for variant, stream_solve in ((3, False), (0, True), (3, True)):
        eng = mmf.ForecastEngine(kernel="tc", tc_variant=variant, stream_solve=stream_solve)
        eng.plan_calendar(start, t, "D", h, "future")
        got = eng.fit_forecast(yd, t, h, want_status=True, want_beta=True, want_stats=True)
        torch.cuda.synchronize()
        for k in ("pred", "status", "beta"):
            assert torch.equal(got[k].view(torch.int32), want[k].view(torch.int32)), (variant, stream_solve, k)
        assert got["stats"].kernel_launches == want["stats"].kernel_launches, (variant, stream_solve)
        eng.close()
    base.close()


def test_ragged_holdout_matches_oracle_and_per_bucket_calls():
    """The reference's contract (hold out the last `horizon` rows, a value for EVERY date, 02:372-380 + 484-494) for a
    batch whose groups sit on different calendars: one pass of the fit kernel + one of the predict kernel, each
    calendar's block of the table written through its own tensor map (tiles that straddle two calendars, chunks that
    run past a calendar's last date)."""
    import torch
    h = 28
    cals, y, rows, ld = _ragged_case(seed=4, short=150)       # (36 fit rows for 16 columns would be a coin toss in any precision)
    eng = mmf.ForecastEngine()
    dates = eng.plan_calendars([c[0] for c in cals], [c[1] for c in cals], "D", h, mode="holdout")
    assert [len(d) for d in dates] == [c[1] for c in cals]
    yd = torch.from_numpy(y).cuda()
    res = eng.fit_forecast_ragged(yd, rows, want_status=True)
    torch.cuda.synchronize()
    pred, status = res["pred"].cpu().numpy(), res["status"].cpu().numpy()
    assert pred.shape == (y.shape[0], max(c[1] for c in cals))
    eng1 = mmf.ForecastEngine()
    for ci, (start, t, n) in enumerate(cals):
        r0, r1 = int(rows[ci]), int(rows[ci + 1])
        yb = y[r0:r1, :t]
        if t - h < 33:
            continue                                            # (not in this case set)
        grid = O.calendar_grid(start, t, "D")
        want, wst, _, ratio = O.fit_forecast_packed(yb, O.design_matrix(grid, t - h), t - h, 0, t, return_gamma=True)
        assert np.array_equal(status[r0:r1], wst), ci
        # columns beyond the calendar's own length stay NaN -- from the next multiple of 4 on: the TMA store clips at the
        # calendar's n_pred with 16-byte granularity, so up to 3 columns behind a row's last date are unspecified
        t4 = (t + 3) & ~3
        tail = pred[r0:r1, t4:]
        assert np.isnan(tail).all(), (ci, t, int(np.argmax(np.isnan(pred[r0, t:]))), int((~np.isnan(tail)).sum()))
        ok = wst != 1
        assert np.isnan(pred[r0:r1, :t][~ok]).all()
        from conftest import forecast_leverage
        lev = forecast_leverage(O.design_matrix(grid, t - h), t - h, 0, t)
        tol = tolerance(yb, lev) / np.minimum(1.0, ratio[ok] / 0.25)
        rel = np.abs(pred[r0:r1, :t][ok] - want[ok]).max(axis=1) / tol
        _le(rel.max(), 1.0, f"calendar {ci}: t={t} n={n} leverage {lev:.3g}")
        single = mmf.forecast_packed(mmf.device_packed(yb), start, "D", h, "holdout", engine=eng1).cpu().numpy()
        assert np.array_equal(single, pred[r0:r1, :t], equal_nan=True), ci
    eng.close()
    eng1.close()


def test_forecast_groups_many_calendars_holdout_mode_one_ragged_launch():
    """DataFrame boundary, reference defaults (holdout): groups on different calendars == the per-group oracle UDF."""
    import pandas as pd
    rng = np.random.default_rng(8)
    frames = []
    for g in range(40):
        t = int(rng.integers(80, 140))
        start = np.datetime64("2020-01-06") + np.timedelta64(7 * int(rng.integers(0, 5)), "D")
        days = start + np.arange(t) * np.timedelta64(7, "D")
        vals = np.round(2000 + 3 * np.arange(t) + rng.normal(0, 25, t)).astype(np.float32)
        keep = rng.random(t) > 0.03
        keep[0] = keep[-1] = True
        frames.append(pd.DataFrame({"Product": f"p{g % 4}", "SKU": f"s{g:03d}", "Date": days[keep].astype("datetime64[ns]"),
                                    "Demand": vals[keep]}))
    df = pd.concat(frames, ignore_index=True).sample(frac=1.0, random_state=2)
    df["Date"] = df["Date"].dt.date
    got = mmf.forecast_groups(df)                               # freq W-MON, horizon 40, holdout: 02:341, 526
    want = O.fanout_apply(df, O.build_tune_and_score_model, ("Product", "SKU"))
    assert len(got) == len(want)
    assert (got["SKU"].to_numpy() == want["SKU"].to_numpy()).all()
    assert (got["Date"].dt.date.to_numpy() == want["Date"].to_numpy()).all()
    assert np.array_equal(got["Demand"].to_numpy(), want["Demand"].to_numpy(), equal_nan=True)
    _le(_frame_ratio(df, got, want, "W-MON", 40, "holdout", "trend_season_exog"), 1.0,
        "ragged holdout DataFrame batch vs per-group oracle UDF")


# ---- batches of less than one wave of 128-row tiles on the tensor-core kernel ---------------------------------------
@pytest.mark.parametrize("n", [1, 7, 8, 9, 127, 129, 1000, 10_000, 20_011])
@pytest.mark.parametrize("mode", ["future", "holdout"])
def test_small_tc_batches_match_the_oracle(n, mode):
    """Batches of 1 to 20,011 rows (one short tile, a tile and a row, under and about one wave of tiles) with gaps,
    leading gaps and mostly-missing rows: statuses equal to the oracle's, forecasts within the tolerance."""
    import torch
    t, h = 365, 28
    yd, start = mmf.synth.daily_store_item_demand_torch(n, t, seed=77 + n, nan_frac=0.02)
    yd[::5, :3] = float("nan")                   # leading gaps: general pass
    if n > 3:
        yd[3, 10:] = float("nan")                # (almost) empty row
    y = yd.cpu().numpy()
    eng = mmf.ForecastEngine(kernel="tc")
    res = mmf.forecast_packed(yd, start, "D", h, mode, engine=eng, want_status=True)
    torch.cuda.synchronize()
    pred, status = res["pred"].cpu().numpy(), res["status"].cpu().numpy()
    eng.close()
    want, wst = O.fit_forecast_packed_c(y, *_design(start, t, h, mode))
    assert np.array_equal(status, wst)
    ok = (wst == 0) & (np.arange(n) % 5 != 0) & (np.arange(n) != 3)      # ~7 scattered gaps: well conditioned
    if ok.any():
        _le(np.abs(pred[ok] - want[ok]).max(), 4 * tolerance(y[ok]), (n, mode))


def test_gappy_rows_do_not_depend_on_their_position_in_the_launch():
    """A series' forecast must not depend on which tile of which SM it lands in.  With an odd number of 32-step chunks
    (t_fit = 400 -> 13) the two transform groups of the tensor-core kernel swap roles from one tile of a CTA to the next;
    the gap positions are therefore filed by the chunk's parity inside the tile, not by the group that saw them, so the
    solve applies them in one canonical order.  Rows of a CTA's SECOND tile, fit again as a batch of their own (first
    tile of another CTA), must come out bit-identical -- with gaps."""
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    t, h = 400, 28
    n = sm * 128 + 3000
    yd, start = mmf.synth.daily_store_item_demand_torch(n, t, seed=5, nan_frac=0.02)
    eng = mmf.ForecastEngine(kernel="tc")
    eng.plan_calendar(start, t, "D", h, "future")
    whole = eng.fit_forecast(yd, t, h, want_status=True)
    part = eng.fit_forecast(yd[sm * 128:], t, h, want_status=True)
    torch.cuda.synchronize()
    assert int((whole["status"] == 0).sum()) == n
    assert torch.equal(whole["status"][sm * 128:], part["status"])
    assert np.array_equal(whole["pred"][sm * 128:].cpu().numpy(), part["pred"].cpu().numpy())
    eng.close()
