"""DataFrame-in / DataFrame-out boundary: the drop-in for the reference's grouped-map UDF.

``forecast_groups`` has the contract of ``build_tune_and_score_model``
(group_apply/02_Fine_Grained_Demand_Forecasting.py:417-494) -- rows of
``enriched_schema`` (02:360-370) in, rows of ``tuning_schema`` (02:498-506) out,
one output row per date of each group's regular grid, sorted by date -- but it
accepts ANY number of groups in one frame and fits them in one GPU pass.  It
can therefore be passed to ``applyInPandas`` unchanged (one group per call, the
literal drop-in at 02:527) or, the intended fast use, once per shard:

    df.groupBy(shard_id).applyInPandas(forecast_groups, schema=tuning_schema)

The packer replaces the per-group ``sort_values("Date")`` +
``set_index("Date").asfreq(freq)`` (02:422-423) with one vectorised scatter into
padded ``y[N, T]`` float32 rows (NaN = missing).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import pandas as pd

from . import design as D
from .engine import ForecastEngine, alloc_packed, default_engine
from ._native import AR_MAX, ARMASEL_MAX_PQ, DIFF_MAX, MA_MAX

FORECAST_HORIZON = 40                      # 02:341
DEFAULT_KEYS = ("Product", "SKU")          # 02:526
EXO_FIELDS = ("covid", "christmas", "new_year")   # 02:431


# ---- schemas (02:360-370, 02:498-506) as pyarrow; pyspark StructTypes on demand ---------
def tuning_schema(keys=DEFAULT_KEYS, date_col="Date", value_col="Demand", interval: bool = False):
    """``interval=True``: the schema of ``forecast_groups(..., interval=level)``, with ``{value}_Lower`` /
    ``{value}_Upper`` float32 columns behind ``{value}_Fitted``."""
    import pyarrow as pa

    extra = [(value_col + "_Lower", pa.float32()), (value_col + "_Upper", pa.float32())] if interval else []
    return pa.schema([(k, pa.string()) for k in keys]
                     + [(date_col, pa.date32()), (value_col, pa.float32()), (value_col + "_Fitted", pa.float32())]
                     + extra)


BACKTEST_METRICS = ("MSE", "MAE", "Bias", "MAPE")


def backtest_schema(keys=DEFAULT_KEYS):
    """The rows of ``backtest_groups``: keys..., ``Cutoff`` (the first forecast date of the origin), ``N`` (scored
    points) and the four metrics."""
    import pyarrow as pa

    return pa.schema([(k, pa.string()) for k in keys] + [("Cutoff", pa.date32()), ("N", pa.int32())]
                     + [(m, pa.float32()) for m in BACKTEST_METRICS])


def enriched_schema(keys=DEFAULT_KEYS, date_col="Date", value_col="Demand"):
    import pyarrow as pa

    return pa.schema([(date_col, pa.date32())] + [(k, pa.string()) for k in keys]
                     + [(value_col, pa.float32())] + [(c, pa.float32()) for c in EXO_FIELDS])


def spark_schemas(keys=DEFAULT_KEYS, date_col="Date", value_col="Demand"):
    """(enriched_schema, tuning_schema) as pyspark StructTypes -- needs pyspark."""
    from pyspark.sql.types import DateType, FloatType, StringType, StructField, StructType

    enriched = StructType([StructField(date_col, DateType())] + [StructField(k, StringType()) for k in keys]
                          + [StructField(value_col, FloatType())] + [StructField(c, FloatType()) for c in EXO_FIELDS])
    tuning = StructType([StructField(k, StringType()) for k in keys]
                        + [StructField(date_col, DateType()), StructField(value_col, FloatType()),
                           StructField(value_col + "_Fitted", FloatType())])
    return enriched, tuning


# ---- mirrors of the small reference helpers ------------------------------------------------
def add_exo_variables(pdf: pd.DataFrame, keys=DEFAULT_KEYS, date_col="Date", value_col="Demand") -> pd.DataFrame:
    """Vectorised ``add_exo_variables`` (02:343-358): same columns, same order, same 0/1 floats."""
    exo = D.exo_variables(D.as_days(pdf[date_col].to_numpy()))
    out = pdf.assign(covid=exo[:, 0], christmas=exo[:, 1], new_year=exo[:, 2])
    return out[[date_col, *keys, value_col, *EXO_FIELDS]]


def split_train_score_data(data, forecast_horizon: int = FORECAST_HORIZON):
    """02:372-380: first ``len - horizon`` rows train, last ``horizon`` rows score."""
    n = len(data)
    is_history = np.arange(n) < (n - forecast_horizon)
    if hasattr(data, "iloc"):
        return data.iloc[is_history], data.iloc[~is_history]
    return data[is_history], data[~is_history]


# ---- packing ---------------------------------------------------------------------------------
import os as _os

PARALLEL_MIN_ROWS = int(_os.environ.get("MMF_PARALLEL_MIN_ROWS", 8_000_000))   # below: Arrow string kernels stay on the calling thread


def _n_threads() -> int:
    import os

    return max(1, min(16, len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)))


def _parallel(fn, items):
    """Arrow compute kernels release the GIL: string hashing / expansion of a big column runs on a few threads."""
    if len(items) <= 1 or _n_threads() == 1:
        return [fn(it) for it in items]
    from concurrent.futures import ThreadPoolExecutor

    with ThreadPoolExecutor(_n_threads()) as ex:
        return list(ex.map(fn, items))


def _slices(n, k):
    cuts = np.linspace(0, n, k + 1).astype(np.int64)
    return [(int(cuts[i]), int(cuts[i + 1])) for i in range(k) if cuts[i + 1] > cuts[i]]


def _dictionary_encode(col):
    """Arrow column (Array or ChunkedArray) -> one DictionaryArray (nulls encoded as a value); big columns are
    hashed piecewise on several threads and the dictionaries unified."""
    import pyarrow as pa
    import pyarrow.compute as pc

    n = len(col)
    chunks = col.chunks if isinstance(col, pa.ChunkedArray) else [col]
    if chunks and pa.types.is_dictionary(chunks[0].type):
        return col.unify_dictionaries().combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    if n >= PARALLEL_MIN_ROWS and _n_threads() > 1:
        if len(chunks) < 2:
            arr = chunks[0]
            chunks = [arr.slice(a, b - a) for a, b in _slices(n, _n_threads())]
        parts = _parallel(lambda c: pc.dictionary_encode(c, null_encoding="encode"), chunks)
        return pa.chunked_array(parts).unify_dictionaries().combine_chunks()
    arr = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    return pc.dictionary_encode(arr, null_encoding="encode")


def _expand_strings(values, row_of: np.ndarray):
    """``values[row_of]`` as an Arrow string column, built from a dictionary (never one Python string per row)."""
    import pyarrow as pa

    values = values.cast(pa.string())

    def piece(ab):
        return pa.DictionaryArray.from_arrays(pa.array(row_of[ab[0]:ab[1]]), values).cast(pa.string())

    if row_of.size >= PARALLEL_MIN_ROWS and _n_threads() > 1:
        return pa.chunked_array(_parallel(piece, _slices(row_of.size, _n_threads())), type=pa.string())
    return piece((0, row_of.size))


@dataclass
class Bucket:
    """Groups that share one calendar (same first date, same grid length)."""
    start: np.datetime64
    t_len: int
    key_frame: pd.DataFrame      # one row per series, key columns only
    y: np.ndarray                # [n, t_len] float32 view of a pitched (pinned) buffer, NaN = missing
    rank: np.ndarray | None = None       # position of each series in the key order of ALL groups of the call
    key_arrow: dict | None = None        # Arrow front end: {key: pyarrow array of this bucket's n key values}


def _combine_codes(codes, sizes):
    """Per-column codes (each numbering its column's values in sort order) -> (group id per row, per-column code
    of every group), groups numbered in lexicographic key order.  One hash pass over a mixed-radix code when the
    product of the cardinalities fits 62 bits, else re-factorised column by column."""
    sizes = [max(int(z), 1) for z in sizes]
    total = 1
    for z in sizes:
        total *= z
    if total < (1 << 62):
        comb = np.asarray(codes[0], dtype=np.int64)
        for j in range(1, len(codes)):
            comb = comb * np.int64(sizes[j]) + np.asarray(codes[j], dtype=np.int64)
        gid, uniq = pd.factorize(comb, sort=True)
        uniq = np.asarray(uniq, dtype=np.int64)
        cols = []
        for j in range(len(codes) - 1, -1, -1):
            cols.append(uniq % np.int64(sizes[j]))
            uniq = uniq // np.int64(sizes[j])
        return gid.astype(np.int64, copy=False), np.stack(cols[::-1], axis=1)
    gid = np.asarray(codes[0], dtype=np.int64)
    per_key = None                                     # [n_groups_so_far, columns_so_far]
    for j in range(len(codes)):
        comb = gid if j == 0 else gid * np.int64(sizes[j]) + np.asarray(codes[j], dtype=np.int64)
        gid, uniq = pd.factorize(comb, sort=True)
        uniq = np.asarray(uniq, dtype=np.int64)
        if j == 0:
            per_key = uniq[:, None]
        else:
            per_key = np.concatenate([per_key[uniq // np.int64(sizes[j])], (uniq % np.int64(sizes[j]))[:, None]], axis=1)
    return gid.astype(np.int64, copy=False), per_key


def _pack_from_codes(gid, n_groups, days, vals, freq, pinned):
    """Shared tail of the pandas and the Arrow packer: rows (group id, day, value) -> calendar buckets.
    Returns [(start_day, t_len, members, y)] with ``members`` = the group ids of the bucket in key order."""
    step = D.FREQ_DAYS[freq]
    if n_groups == 1:                                                        # the one-group-per-call drop-in
        gmin, gmax = np.array([days.min()], dtype=np.int64), np.array([days.max()], dtype=np.int64)
    elif days.size < 50_000:
        gmin = np.full(n_groups, np.iinfo(np.int64).max)
        gmax = np.full(n_groups, np.iinfo(np.int64).min)
        np.minimum.at(gmin, gid, days)
        np.maximum.at(gmax, gid, days)
    else:
        span = pd.Series(days).groupby(gid, sort=True).agg(["min", "max"])   # gid is dense: row g = group g
        gmin, gmax = span["min"].to_numpy(dtype=np.int64), span["max"].to_numpy(dtype=np.int64)
    if freq == "W-MON" and np.any((gmin + 3) % 7 != 0):
        raise ValueError("W-MON series must start on a Monday")
    t_len = (gmax - gmin) // step + 1
    off = days - gmin[gid]
    pos = off // step
    on_grid = None if step == 1 else (off % step == 0)                       # off-grid rows vanish under asfreq
    if on_grid is not None and on_grid.all():
        on_grid = None
    out = []
    # buckets in (first day, length) order: one sortable integer per group
    uniq, bucket_id = np.unique(gmin * np.int64(1 << 32) + t_len, return_inverse=True)
    bucket_keys = [(int(u >> 32), int(u & 0xFFFFFFFF)) for u in uniq.tolist()]
    single = len(bucket_keys) == 1
    for b, (start_day, tl) in enumerate(bucket_keys):
        members = np.arange(n_groups) if single else np.flatnonzero(bucket_id == b)
        pin = (members.size * int(tl) * 4 >= (1 << 20)) if pinned is None else pinned
        y = alloc_packed(members.size, int(tl), pinned=pin)
        y[...] = np.nan
        ld = y.strides[0] // 4
        flat = np.lib.stride_tricks.as_strided(y, shape=(members.size * ld,), strides=(4,))   # the pitched rows, 1-D
        if single:
            row, sel = gid, on_grid
        else:
            local = np.full(n_groups, -1, dtype=np.int64)
            local[members] = np.arange(members.size)
            row = local[gid]
            sel = (row >= 0) if on_grid is None else (on_grid & (row >= 0))
        idx = row * ld + pos
        if sel is not None:
            idx, v = idx[sel], vals[sel]
        else:
            v = vals
        seen = np.zeros(flat.size, dtype=bool)
        seen[idx] = True
        if int(seen.sum()) != idx.size:        # the reference's set_index("Date").asfreq() raises here too (02:423)
            raise ValueError(f"cannot reindex on an axis with duplicate labels: {idx.size - int(seen.sum())} rows repeat "
                             f"a (group, date) combination")
        flat[idx] = v
        out.append((int(start_day), int(tl), members, y))
    return out


def pack_groups(pdf: pd.DataFrame, keys=DEFAULT_KEYS, date_col="Date", value_col="Demand", freq="W-MON",
                pinned: bool | None = None) -> list:
    """Long frame -> calendar buckets of packed series (02:422-423 for all groups at once).
    ``pinned=None`` page-locks buckets of >= 1 MiB (worth the cudaHostAlloc), False never."""
    keys = list(keys)
    if len(pdf) == 0:
        return []
    days = D.as_days(pdf[date_col].to_numpy()).astype(np.int64)
    codes, uniques = [], []
    for k in keys:                                    # one hash pass per key column, never a tuple per row
        c, u = pd.factorize(pdf[k], sort=True, use_na_sentinel=False)
        codes.append(c)
        uniques.append(u)
    gid, per_key = _combine_codes(codes, [len(u) for u in uniques])
    vals = pdf[value_col].to_numpy(dtype=np.float32, na_value=np.nan)
    buckets = []
    for start_day, tl, members, y in _pack_from_codes(gid, per_key.shape[0], days, vals, freq, pinned):
        key_frame = pd.DataFrame({k: pd.Series(uniques[j].take(per_key[members, j]), dtype=pdf[k].dtype)
                                  for j, k in enumerate(keys)})
        buckets.append(Bucket(np.datetime64(start_day, "D"), tl, key_frame, y, rank=members))
    return buckets


def pack_table_host(table, keys=DEFAULT_KEYS, date_col="Date", value_col="Demand", freq="W-MON",
                    pinned: bool | None = None) -> list:
    """Arrow ``Table`` -> the same buckets as ``pack_groups`` without a pandas frame of the rows: key columns
    are dictionary-encoded by Arrow, dates and values are read as NumPy views of the column buffers."""
    import pyarrow as pa
    import pyarrow.compute as pc

    keys = list(keys)
    if table.num_rows == 0:
        return []
    codes, uniques = [], []
    for k in keys:
        col = _dictionary_encode(table.column(k))
        dic = col.dictionary
        order = pc.sort_indices(dic).to_numpy()                      # dictionary is in first-seen order: rank it
        rank = np.empty(len(dic), dtype=np.int64)
        rank[order] = np.arange(len(dic))
        idx = col.indices.to_numpy(zero_copy_only=False)
        codes.append(rank[idx.astype(np.int64, copy=False)])
        uniques.append(dic.take(pa.array(order)))
    gid, per_key = _combine_codes(codes, [len(u) for u in uniques])
    dcol = table.column(date_col).combine_chunks()
    if not pa.types.is_date32(dcol.type):
        dcol = pc.cast(dcol, pa.date32())
    days = dcol.cast(pa.int32()).to_numpy(zero_copy_only=False).astype(np.int64)
    vcol = pc.cast(table.column(value_col).combine_chunks(), pa.float32())
    vals = vcol.fill_null(float("nan")).to_numpy(zero_copy_only=False) if vcol.null_count else vcol.to_numpy(zero_copy_only=False)
    buckets = []
    for start_day, tl, members, y in _pack_from_codes(gid, per_key.shape[0], days, vals, freq, pinned):
        key_arrow = {k: uniques[j].take(pa.array(per_key[members, j])) for j, k in enumerate(keys)}
        key_frame = pa.table(key_arrow).to_pandas()
        buckets.append(Bucket(np.datetime64(start_day, "D"), tl, key_frame, y, rank=members, key_arrow=key_arrow))
    return buckets


# ---- the drop-in UDF ---------------------------------------------------------------------------
RAGGED_MIN_BUCKETS = 2        # from this many calendars on, a batch goes through ONE ragged launch


def _fit_buckets_ragged(buckets, eng, freq, horizon, mode, design, on_device):
    """All calendars of the batch in one launch (``mmf_plan_calendars`` + ``mmf_fit_forecast_ragged_f32``): the groups'
    rows are laid out calendar after calendar in one device buffer, each calendar's design is whitened in the same
    host call, and one pass of the tensor-core kernel fits every group against its own calendar (02:422-423 per group);
    in holdout mode one pass of the predict kernel then writes a value for every date of every group (02:484-494)."""
    import torch

    dev = torch.device("cuda", torch.cuda.current_device())
    t_max = max(b.t_len for b in buckets)
    rows = np.cumsum([0] + [b.y.shape[0] for b in buckets]).astype(np.int64)
    y = torch.zeros((int(rows[-1]), (t_max + 3) & ~3), dtype=torch.float32, device=dev)
    for i, b in enumerate(buckets):
        src = b.y if on_device else torch.from_numpy(b.y)
        y[int(rows[i]):int(rows[i + 1]), :b.t_len].copy_(src, non_blocking=True)
    dates = eng.plan_calendars([b.start for b in buckets], [b.t_len for b in buckets], freq, horizon, design, mode)
    pred = eng.fit_forecast_ragged(y, rows).cpu().numpy()
    for i, b in enumerate(buckets):
        y_host = b.y.cpu().numpy() if on_device else b.y
        n_pred = horizon if mode == "future" else b.t_len
        yield b, dates[i], n_pred, y_host, np.ascontiguousarray(pred[int(rows[i]):int(rows[i + 1]), :n_pred]), None


def _host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _fit_buckets(buckets, eng, freq, horizon, mode, design, select, on_device, interval=False, ar=None, diff=None,
                 ma=None, want_se=False, estimator=None, joint_beta=False, refit=None, predictor=None):
    """Run the engine over every bucket: yields (bucket, out_days, n_pred, y_host, pred_host, se_host or None).
    ``interval``: prediction standard errors too (``fit_forecast_se``), one call per calendar bucket.
    ``ar``: regression with AR(ar) errors (``fit_forecast_ar``), one call per calendar bucket; a tuple of orders
    chooses the order per series by hold-out MSE over the last ``horizon`` rows (``fit_select_ar``).
    ``diff``: regression with ARIMA(ar, diff, 0) errors (``fit_forecast_arima``), one call per calendar bucket; a tuple
    of differencing orders (with ``ar`` a tuple of orders) chooses (p, d) per series by hold-out MSE over the last
    ``horizon`` rows (``fit_select_arima``).
    ``ma``: regression with ARIMA(ar, diff or 0, ma) errors (``fit_forecast_arma``), one call per calendar bucket; a
    tuple of MA orders (with ``ar`` and ``diff`` tuples) chooses (p, d, q) per series by hold-out MSE over the last
    ``horizon`` rows (``fit_select_arma``).
    ``want_se``: the ARIMA-family call's forecast standard errors too (``want_se=True``, DESIGN.md section 2 item 15).
    ``estimator``: the fixed-order ARIMA(p, d, q) call's estimator (None: the engine's default, Hannan-Rissanen);
    ``joint_beta``: with ``estimator="css"``, beta estimated jointly with (phi, theta).
    ``refit``: with candidate MA orders, the winner refit by conditional least squares (``joint_beta`` with it: beta
    jointly), or "ml" by exact likelihood.
    ``predictor``: with ``estimator="ml"`` or ``refit="ml"``, "kalman" predicts with the filter of the exact likelihood
    (None: the recursion)."""
    se_kw = {"want_se": True} if want_se else {}
    if interval and select is not None:
        raise ValueError("interval= is not offered with select= (model selection returns point forecasts)")
    t_fit_min = min((b.t_len - (horizon if mode == "holdout" else 0)) for b in buckets) if buckets else 0
    if (select is None and not interval and ar is None and len(buckets) >= RAGGED_MIN_BUCKETS and (mode == "holdout" or 1 <= horizon <= 64)
            and hasattr(eng, "fit_forecast_ragged") and t_fit_min >= 33 and all(b.t_len <= 65535 for b in buckets)):
        yield from _fit_buckets_ragged(buckets, eng, freq, horizon, mode, design, on_device)
        return
    for b in buckets:
        if diff is None or (isinstance(diff, tuple) and max(diff) == 0):
            out_days, pred_start, n_pred = eng.plan_calendar(b.start, b.t_len, freq, horizon, mode, design)
        else:
            out_days, pred_start, n_pred = eng.plan_calendar(b.start, b.t_len, freq, horizon, mode, design,
                                                             max_diff=max(diff) if isinstance(diff, tuple) else diff)
        se = None
        if isinstance(ma, tuple):
            from .engine import device_packed
            yd = b.y if (on_device or not isinstance(eng, ForecastEngine)) else device_packed(b.y)
            ref_kw = {"refit": refit, "joint_beta": joint_beta} if refit is not None else {}
            if predictor is not None:                # only when given: engines without predictor= keep working
                ref_kw["predictor"] = predictor
            res = eng.fit_select_arma(yd, horizon, ar, diff, ma, pred_start, n_pred, **se_kw, **ref_kw)
            pred, se = _host(res["pred"]), (_host(res["se"]) if want_se else None)
        elif ma is not None:
            from .engine import device_packed
            yd = b.y if (on_device or not isinstance(eng, ForecastEngine)) else device_packed(b.y)
            est_kw = {"estimator": estimator} if estimator is not None else {}
            if joint_beta:
                est_kw["joint_beta"] = True
            if predictor is not None:
                est_kw["predictor"] = predictor
            res = eng.fit_forecast_arma(yd, ar, ma, diff or 0, pred_start, n_pred, **se_kw, **est_kw)
            pred, se = _host(res["pred"]), (_host(res["se"]) if want_se else None)
        elif isinstance(diff, tuple):
            from .engine import device_packed
            yd = b.y if (on_device or not isinstance(eng, ForecastEngine)) else device_packed(b.y)
            res = eng.fit_select_arima(yd, horizon, ar, diff, pred_start, n_pred, **se_kw)
            pred, se = _host(res["pred"]), (_host(res["se"]) if want_se else None)
        elif diff is not None:
            from .engine import device_packed
            yd = b.y if (on_device or not isinstance(eng, ForecastEngine)) else device_packed(b.y)
            res = eng.fit_forecast_arima(yd, ar, diff, pred_start, n_pred, **se_kw)
            pred, se = _host(res["pred"]), (_host(res["se"]) if want_se else None)
        elif isinstance(ar, tuple):
            from .engine import device_packed
            yd = b.y if (on_device or not isinstance(eng, ForecastEngine)) else device_packed(b.y)
            res = eng.fit_select_ar(yd, horizon, ar, pred_start, n_pred, **se_kw)
            pred, se = _host(res["pred"]), (_host(res["se"]) if want_se else None)
        elif ar is not None:
            from .engine import device_packed
            yd = b.y if (on_device or not isinstance(eng, ForecastEngine)) else device_packed(b.y)
            res = eng.fit_forecast_ar(yd, ar, pred_start, n_pred, **se_kw)
            pred, se = _host(res["pred"]), (_host(res["se"]) if want_se else None)
        elif interval:
            from .engine import device_packed
            yd = b.y if (on_device or not isinstance(eng, ForecastEngine)) else device_packed(b.y)
            res = eng.fit_forecast_se(yd, pred_start, n_pred)
            pred, se = _host(res["pred"]), _host(res["se"])
        elif select is not None:
            if mode != "holdout":
                raise ValueError("select= needs mode='holdout' (the held-out rows score the candidates)")
            from .engine import device_packed
            yd = b.y if on_device else device_packed(b.y)
            pred = eng.fit_select_forecast(yd, horizon, tuple(select), pred_start, n_pred)["pred"].cpu().numpy()
        else:
            pred = eng.fit_forecast(b.y, pred_start, n_pred)
            if on_device:
                pred = pred.cpu().numpy()
        y_host = b.y.cpu().numpy() if on_device else b.y
        yield b, out_days, n_pred, y_host, pred, se


def _z_of(interval):
    """normal quantile of a two-sided interval at level ``interval`` (what SARIMAX's conf_int uses); None: no interval"""
    if interval is None:
        return None
    from statistics import NormalDist
    level = float(interval)
    if not 0.0 < level < 1.0:
        raise ValueError(f"interval must be a level in (0, 1), got {interval!r}")
    return NormalDist().inv_cdf(0.5 + level / 2.0)


def _conf_z(conf_int, ar, select, interval):
    """normal quantile of ``conf_int=`` (None: no band).  It is the band of the ARIMA-family forecasts (DESIGN.md
    section 2 item 15), so it needs ``ar=``; ``interval=`` is the plain regression's band, a different quantity"""
    if conf_int is None:
        return None
    if ar is None:
        raise ValueError("conf_int= needs ar= (it is the band of the AR / ARIMA forecasts; the plain regression's band "
                         "is interval=)")
    if interval is not None:
        raise ValueError("conf_int= and interval= are different bands: pass one of them")
    if select is not None:
        raise ValueError("conf_int= is not offered with select=")
    level = float(conf_int)
    if not 0.0 < level < 1.0:
        raise ValueError(f"conf_int must be a level in (0, 1), got {conf_int!r}")
    return _z_of(level)


def _ar_order(ar, select, interval, mode="holdout"):
    """validated AR order of ``ar=`` (None: the plain model), or the tuple of candidate orders of a sequence"""
    if ar is None:
        return None
    if select is not None or interval is not None:
        raise ValueError("ar= is not offered with select= or interval= (AR forecasts come without either)")
    if isinstance(ar, (list, tuple, np.ndarray)):
        orders = list(ar)
        if not orders:
            raise ValueError("ar= needs at least one candidate order")
        if any(isinstance(m, bool) or not isinstance(m, (int, np.integer)) or not 0 <= int(m) <= AR_MAX for m in orders):
            raise ValueError(f"ar= candidate orders must be integers in [0, {AR_MAX}], got {ar!r}")
        orders = [int(m) for m in orders]
        if any(b <= a for a, b in zip(orders, orders[1:])):
            raise ValueError(f"ar= candidate orders must be ascending and distinct, got {ar!r}")
        if mode != "holdout":
            raise ValueError("ar= with candidate orders needs mode='holdout' (the last horizon rows score the candidates)")
        return tuple(orders)
    if isinstance(ar, bool) or not isinstance(ar, (int, np.integer)) or not 1 <= int(ar) <= AR_MAX:
        raise ValueError(f"ar must be an AR order in [1, {AR_MAX}], got {ar!r}")
    return int(ar)


def _diff_order(diff, ar, select, interval, mode="holdout"):
    """validated differencing order of ``diff=`` (None: no differencing); ``ar`` must then be one order in 0..8.  A
    sequence of differencing orders gives the tuple of candidate d's; ``ar`` is then one order or a sequence of them"""
    if diff is None:
        return None
    if select is not None or interval is not None:
        raise ValueError("diff= is not offered with select= or interval= (ARIMA forecasts come without either)")
    if isinstance(diff, (list, tuple, np.ndarray)):
        diffs = list(diff)
        if not diffs:
            raise ValueError("diff= needs at least one candidate differencing order")
        if any(isinstance(d, bool) or not isinstance(d, (int, np.integer)) or not 0 <= int(d) <= DIFF_MAX for d in diffs):
            raise ValueError(f"diff= candidate differencing orders must be integers in [0, {DIFF_MAX}], got {diff!r}")
        diffs = [int(d) for d in diffs]
        if any(b <= a for a, b in zip(diffs, diffs[1:])):
            raise ValueError(f"diff= candidate differencing orders must be ascending and distinct, got {diff!r}")
        if mode != "holdout":
            raise ValueError("diff= with candidate differencing orders needs mode='holdout' (the last horizon rows score "
                             "the candidates)")
        return tuple(diffs)
    if isinstance(diff, bool) or not isinstance(diff, (int, np.integer)) or not 1 <= int(diff) <= DIFF_MAX:
        raise ValueError(f"diff must be a differencing order in [1, {DIFF_MAX}], got {diff!r}")
    if isinstance(ar, bool) or not isinstance(ar, (int, np.integer)) or not 0 <= int(ar) <= AR_MAX:
        raise ValueError(f"diff= needs one integer AR order ar in [0, {AR_MAX}], got ar={ar!r}")
    return int(diff)


def _arma_orders(ma, ar, diff, select, interval, mode="holdout"):
    """validated (ar, diff, ma) of ``ma=``: one MA order in 1..4 with one AR order in 0..8 and ``diff`` None (d = 0) or
    one differencing order in 1..2.  A sequence of MA orders (ascending, distinct, in 0..4, starting with 0) chooses
    (p, d, q) per series: it needs a sequence of AR orders, ``diff`` None (d = 0) or a sequence of differencing orders,
    and ``mode='holdout'``; the result is then three tuples."""
    if select is not None or interval is not None:
        raise ValueError("ma= is not offered with select= or interval= (ARMA forecasts come without either)")
    if isinstance(ma, (list, tuple, np.ndarray)):
        mas = list(ma)
        if (not mas or any(isinstance(q, bool) or not isinstance(q, (int, np.integer)) or not 0 <= int(q) <= MA_MAX
                           for q in mas)):
            raise ValueError(f"ma= candidate MA orders must be integers in [0, {MA_MAX}], got ma={ma!r}")
        mas = [int(q) for q in mas]
        if mas[0] != 0 or any(b <= a for a, b in zip(mas, mas[1:])):
            raise ValueError(f"ma= candidate MA orders must be ascending and distinct and start with 0, got ma={ma!r}")
        if not isinstance(ar, (list, tuple, np.ndarray)):
            raise ValueError(f"ma= with candidate MA orders needs candidate AR orders ar=(...) in [0, {AR_MAX}], "
                             f"got ar={ar!r}")
        if diff is not None and not isinstance(diff, (list, tuple, np.ndarray)):
            raise ValueError(f"ma= with candidate MA orders needs diff=None or candidate differencing orders, "
                             f"got diff={diff!r}")
        diffs = _diff_order((0,) if diff is None else diff, ar, select, interval, mode)
        orders = _ar_orders_for(diffs, ar, select, interval, mode)
        if len(orders) * (len(mas) - 1) > ARMASEL_MAX_PQ:
            raise ValueError(f"ar= and ma= give {len(orders) * (len(mas) - 1)} (p, q >= 1) pairs, more than "
                             f"{ARMASEL_MAX_PQ}")
        return tuple(orders), diffs, tuple(mas)
    if isinstance(ma, bool) or not isinstance(ma, (int, np.integer)) or not 1 <= int(ma) <= MA_MAX:
        raise ValueError(f"ma must be an MA order in [1, {MA_MAX}], got {ma!r}")
    if isinstance(ar, bool) or not isinstance(ar, (int, np.integer)) or not 0 <= int(ar) <= AR_MAX:
        raise ValueError(f"ma= needs one integer AR order ar in [0, {AR_MAX}], got ar={ar!r}")
    if diff is not None and (isinstance(diff, bool) or not isinstance(diff, (int, np.integer))
                             or not 0 <= int(diff) <= DIFF_MAX):
        raise ValueError(f"ma= takes one differencing order diff in [0, {DIFF_MAX}] (or None), got diff={diff!r}")
    return int(ar), (int(diff) if diff else None), int(ma)


def _estimator(estimator, ma, select, interval):
    """validated ``estimator=`` of the fixed-order ARIMA(p, d, q) forecasts: None (Hannan-Rissanen, as before), "hr",
    "css" (DESIGN.md section 2 item 16) or "ml" (item 19).  It needs one MA order ``ma=q``."""
    if estimator is None:
        return None
    if estimator not in ("hr", "css", "ml"):
        raise ValueError(f"estimator must be 'hr' or 'css' (or 'ml' for the exact likelihood), got {estimator!r}")
    if select is not None or interval is not None:
        raise ValueError("estimator= is not offered with select= or interval= (ARMA forecasts come without either)")
    if ma is None:
        raise ValueError("estimator= needs one MA order ma=q in [1, 4] (it chooses how ARIMA(p, d, q) is estimated)")
    if isinstance(ma, (list, tuple, np.ndarray)):
        raise ValueError(f"estimator= is not offered with candidate MA orders (order selection scores Hannan-Rissanen "
                         f"fits), got ma={ma!r}")
    return estimator


def _refit(refit, ma, estimator, select, interval):
    """validated ``refit=``: None (the selection's Hannan-Rissanen winners, as before), "css", the winner of the
    (p, d, q) selection refit by conditional least squares (DESIGN.md section 2 item 18), or "ml", that refit refined by
    exact likelihood (item 21).  It needs candidate MA orders."""
    if refit is None:
        return None
    if refit not in ("css", "ml"):
        raise ValueError(f"refit must be None or 'css' (or 'ml' for the exact likelihood), got {refit!r}")
    if select is not None or interval is not None:
        raise ValueError("refit= is not offered with select= or interval= (ARMA forecasts come without either)")
    if estimator is not None:
        raise ValueError(f"refit= is not offered with estimator= (estimator= chooses how a fixed ma=q is estimated, "
                         f"refit= refits a selection's winner), got estimator={estimator!r}")
    if not isinstance(ma, (list, tuple, np.ndarray)):
        raise ValueError(f"refit= needs candidate MA orders ma=(0, ...) (it refits the winner of the (p, d, q) "
                         f"selection), got ma={ma!r}")
    return refit


def _predictor(predictor, estimator, refit=None):
    """validated ``predictor=``: None (the recursion, as before), "recursion", or "kalman" with ``estimator="ml"``
    (DESIGN.md section 2 item 20) or ``refit="ml"`` (item 21)"""
    if predictor is None:
        return None
    if predictor not in ("recursion", "kalman"):
        raise ValueError(f"predictor must be 'recursion' or 'kalman', got {predictor!r}")
    if predictor == "kalman" and estimator != "ml" and refit != "ml":
        raise ValueError(f"predictor='kalman' needs estimator='ml' (or refit='ml' for a selection: the filter of the "
                         f"exact-likelihood fit), got estimator={estimator!r}, refit={refit!r}")
    return predictor


def _joint_beta(joint_beta, estimator, refit=None):
    """validated ``joint_beta=``: True needs ``estimator="css"`` (DESIGN.md section 2 item 17) or ``refit="css"`` (item
    18)"""
    if not joint_beta:
        return False
    if refit == "css":
        return True
    if refit == "ml":
        raise ValueError("joint_beta=True needs estimator='css' or refit='css' (joint beta by the exact likelihood is "
                         "not offered), got refit='ml'")
    if estimator != "css":
        raise ValueError(f"joint_beta=True needs estimator='css' (beta joins the conditional least-squares fit), "
                         f"got estimator={estimator!r}")
    return True


def _ar_orders_for(diff, ar, select, interval, mode):
    """``ar=`` validated against ``diff=``: one order in 0..8 for a single d, the tuple of candidate orders for a tuple
    of d's, and _ar_order's result without differencing"""
    if diff is None:
        return _ar_order(ar, select, interval, mode)
    if not isinstance(diff, tuple):
        return int(ar)
    if not isinstance(ar, (list, tuple, np.ndarray)):
        raise ValueError(f"diff= with candidate differencing orders needs candidate AR orders ar=(...) in [0, {AR_MAX}], "
                         f"got ar={ar!r}")
    return _ar_order(ar, select, interval, mode)


def _bounds(pred, se, z):
    """(lower, upper) float32 rows of pred -+ z * se"""
    p = np.asarray(pred, dtype=np.float64).reshape(-1)
    s = np.asarray(se, dtype=np.float64).reshape(-1)
    return (p - z * s).astype(np.float32), (p + z * s).astype(np.float32)


def _global_order(buckets, keys, lengths):
    """Row permutation that puts the concatenated per-bucket blocks into (key, date) order: a sort of one integer
    per output row (the series' rank), never of the key strings."""
    if all(b.rank is not None for b in buckets):
        ranks = [np.asarray(b.rank, dtype=np.int64) for b in buckets]
    else:                                               # e.g. device packer: rank the (few) key rows here
        kf = pd.concat([b.key_frame for b in buckets], ignore_index=True)
        order = kf.sort_values(list(keys), kind="stable").index.to_numpy()
        r = np.empty(len(kf), dtype=np.int64)
        r[order] = np.arange(len(kf))
        cuts = np.cumsum([0] + [len(b.key_frame) for b in buckets])
        ranks = [r[cuts[i]:cuts[i + 1]] for i in range(len(buckets))]
    per_row = np.concatenate([np.repeat(rk, n) for rk, n in zip(ranks, lengths)])
    return np.argsort(per_row, kind="stable")


def _buckets_for(pdf, keys, date_col, value_col, freq, pack, eng):
    import pyarrow as pa

    if pack == "device":
        from .packer import pack_table_device
        return pack_table_device(pdf, keys, date_col, value_col, freq, engine=eng)
    if pack != "host":
        raise ValueError("pack must be 'host' or 'device'")
    if isinstance(pdf, (pa.Table, pa.RecordBatch)):
        return pack_table_host(pa.Table.from_batches([pdf]) if isinstance(pdf, pa.RecordBatch) else pdf,
                               keys, date_col, value_col, freq)
    return pack_groups(pdf, keys, date_col, value_col, freq)


SINGLE_GROUP_MAX_ROWS = 4096


def _single_group_fast(pdf, keys, date_col, value_col, freq, horizon, mode, design, eng, null_keys_on_gaps):
    """The literal drop-in -- ``applyInPandas`` hands over ONE group per call (02:523-528) -- without the machinery
    that many groups need (key factorisation, bucket bookkeeping, a key frame): returns the output frame, or None
    when the frame holds more than one group (or null keys) and the general path must run.  Same rows, dtypes and
    values as the general path (tests compare them)."""
    n = len(pdf)
    if n == 0 or n > SINGLE_GROUP_MAX_ROWS:
        return None
    key_cols = []
    for k in keys:
        col = pdf[k]
        vals = col.to_numpy()
        first = vals[0]
        if pd.isna(first):
            return None                                   # null keys: the general path (a null key is its own group)
        same = vals == first
        if not (isinstance(same, np.ndarray) and same.dtype == bool and same.all()):
            return None
        key_cols.append(col)
    dvals = pdf[date_col].to_numpy()
    if dvals.dtype.kind == "M":
        days = dvals.astype("datetime64[D]").astype(np.int64)
    elif dvals.dtype == object and n and hasattr(dvals[0], "toordinal"):
        days = np.fromiter((d.toordinal() for d in dvals), dtype=np.int64, count=n) - 719163    # 1970-01-01
    else:
        days = D.as_days(dvals).astype(np.int64)
    vals = pdf[value_col].to_numpy(dtype=np.float32, na_value=np.nan)
    step = D.FREQ_DAYS[freq]
    d0, d1 = int(days.min()), int(days.max())
    if freq == "W-MON" and (d0 + 3) % 7 != 0:
        raise ValueError("W-MON series must start on a Monday")
    t_len = (d1 - d0) // step + 1
    off = days - d0
    pos = off // step
    if step > 1:
        on = off % step == 0
        if not on.all():
            pos, vals = pos[on], vals[on]
    y = np.full((1, (t_len + 3) & ~3), np.nan, dtype=np.float32)[:, :t_len]
    seen = np.zeros(t_len, dtype=bool)
    seen[pos] = True
    if int(seen.sum()) != pos.size:            # the reference's set_index("Date").asfreq() raises here too (02:423)
        raise ValueError(f"cannot reindex on an axis with duplicate labels: {pos.size - int(seen.sum())} rows repeat "
                         f"a (group, date) combination")
    y[0, pos] = vals
    out_days, pred_start, n_pred = eng.plan_calendar(np.datetime64(d0, "D"), int(t_len), freq, horizon, mode, design)
    pred = eng.fit_forecast(y, pred_start, n_pred)
    take0 = np.zeros(n_pred, dtype=np.intp)
    frame = {k: pd.Series(c.array.take(take0), dtype=c.dtype, copy=False) for k, c in zip(keys, key_cols)}
    frame[date_col] = np.asarray(out_days).astype("datetime64[ns]")
    frame[value_col] = np.ascontiguousarray(y[0]) if mode == "holdout" else np.full(n_pred, np.nan, dtype=np.float32)
    frame[value_col + "_Fitted"] = np.asarray(pred).reshape(-1)
    if null_keys_on_gaps and mode == "holdout":
        gap = np.isnan(frame[value_col])
        if gap.any():
            for k in keys:
                frame[k] = frame[k].astype(object).where(~gap, None)
    return pd.DataFrame(frame)


def forecast_groups(pdf, *, keys=DEFAULT_KEYS, date_col="Date", value_col="Demand",
                    freq="W-MON", horizon=FORECAST_HORIZON, mode="holdout", design="trend_season_exog",
                    engine: ForecastEngine | None = None, pack: str = "host", select=None,
                    null_keys_on_gaps: bool = False, interval=None, ar=None, diff=None, ma=None,
                    conf_int=None, estimator=None, joint_beta=False, refit=None, predictor=None) -> pd.DataFrame:
    """Fit + forecast every group in ``pdf``; returns ``tuning_schema`` rows
    (keys..., Date, Demand, Demand_Fitted), groups in key order, dates ascending.

    ``mode="holdout"`` reproduces the reference's contract (fit on all but the last
    ``horizon`` grid rows, emit fitted + forecast values for every grid date, 02:484-494);
    ``mode="future"`` fits on everything and emits the ``horizon`` dates after the end
    (``Demand`` is NaN there).

    ``select=(1, 3, 9, 13, 16)`` (holdout mode only) turns on the per-series model selection that stands in for the
    reference's hyperopt loop (02:435-481): nested designs on the first ``m`` whitened columns are scored by their
    MSE over the held-out rows and the winner produces ``Demand_Fitted`` (``ForecastEngine.fit_select_forecast``).

    ``pack="device"`` groups, sorts and re-grids the rows on the GPU (``packer.pack_table_device``: Arrow
    buffers in, padded series out) instead of with pandas on the host; ``pdf`` may then be an Arrow table.

    ``null_keys_on_gaps=True`` (holdout mode) reproduces a detail of the reference's output assembly: it reads the
    key columns from the re-indexed frame (02:490), so rows that ``asfreq`` inserted for missing dates carry NaN in
    ``Product`` / ``SKU``.  By default the keys are filled on every row (a grid row without a ``Demand`` is still
    that group's row); with the option, rows whose ``Demand`` is missing get null keys.

    ``interval=0.9`` appends float32 ``Demand_Lower`` / ``Demand_Upper`` = ``Demand_Fitted -+ z * se`` with the normal
    quantile ``z = NormalDist().inv_cdf(0.5 + level / 2)`` and ``se`` the prediction standard error of each row
    (``ForecastEngine.fit_forecast_se``; NaN where a series has no residual degrees of freedom).  Every calendar bucket
    then takes its own call.  ``interval=None`` leaves the frame as it was.

    ``ar=p`` (1 <= p <= 8) fits regression with AR(p) errors (``ForecastEngine.fit_forecast_ar``, DESIGN.md section 2
    item 9): ``Demand_Fitted`` holds one-step-ahead predictions on the fit dates and the dynamic forecast after them.
    The schema is unchanged; every calendar bucket takes its own call.  Not offered with ``select=`` or ``interval=``.
    ``ar=(0, 1, 2, 3, 4)`` (ascending distinct orders in 0..8; the reference's ``p`` range by default) chooses each
    series' order by the MSE of its dynamic forecast over the last ``horizon`` dates, the held-out rows of
    ``mode='holdout'`` (``ForecastEngine.fit_select_ar``, DESIGN.md section 2 item 10); ``Demand_Fitted`` comes from each
    series' winner.  Holdout mode only.

    ``diff=d`` (1 or 2) with ``ar=p`` (0 <= p <= 8) fits regression with ARIMA(p, d, 0) errors
    (``ForecastEngine.fit_forecast_arima``, DESIGN.md section 2 item 11): the AR(p) model of the d-times differenced
    series on the differenced design, integrated back to levels.  ``Demand_Fitted`` holds one-step-ahead level
    predictions on the fit dates (NaN / null on the first d dates of a group) and the integrated dynamic forecast after
    them.  The schema is unchanged; every calendar bucket takes its own call.  ``diff=None`` leaves everything as it
    was; an integer ``diff`` is not offered with ``select=``, ``interval=`` or a tuple of AR orders.
    ``diff=(0, 1, 2)`` (ascending distinct orders in 0..2) with ``ar=(0, 1, 2, 3, 4)`` (a tuple of orders) chooses each
    series' (p, d) by the MSE of its dynamic level forecast over the last ``horizon`` dates, the held-out rows of
    ``mode='holdout'`` (``ForecastEngine.fit_select_arima``, DESIGN.md section 2 item 12); ``Demand_Fitted`` comes from
    each series' winner.  Holdout mode only, one call per calendar bucket, schema unchanged.

    ``ma=q`` (1 <= q <= 4) with ``ar=p`` (0 <= p <= 8) and ``diff=d`` (None for d = 0, or 1, 2) fits regression with
    ARIMA(p, d, q) errors by Hannan-Rissanen (``ForecastEngine.fit_forecast_arma``, DESIGN.md section 2 item 13);
    ``ar=1, diff=2, ma=1`` is the reference notebook's order.  A series whose estimate fails the gate gets the
    ARIMA(p, d, 0) forecast.  One call per calendar bucket, schema unchanged; ``ma=None`` leaves everything as it was.
    Not offered with ``select=`` or ``interval=``.
    ``ma=(0, 1, 2, 3, 4)`` (ascending distinct orders in 0..4 starting with 0) with ``ar=(0, 1, 2, 3, 4)`` and
    ``diff=(0, 1, 2)`` (or None for d = 0) chooses each series' (p, d, q) by the MSE of its dynamic level forecast over
    the last ``horizon`` dates (``ForecastEngine.fit_select_arma``, DESIGN.md section 2 item 14): the reference's search
    space, searched exhaustively.  At most 32 pairs (p, q >= 1).  Holdout mode only, one call per calendar bucket,
    schema unchanged.

    ``conf_int=0.9`` with any accepted ``ar=`` / ``diff=`` / ``ma=`` (fixed or tuples) appends float32 ``Demand_Lower``
    / ``Demand_Upper`` = ``Demand_Fitted -+ z * se``, ``z`` as for ``interval=`` and ``se`` the standard error of the
    ARIMA-family forecast (``want_se=True``, DESIGN.md section 2 item 15: the fitted model taken as true, no estimation
    uncertainty; NaN where ``Demand_Fitted`` is NaN).  Schema ``tuning_schema(interval=True)``.  Refused without
    ``ar=``, with ``interval=`` (the plain regression's band, a different quantity) or ``select=``, and for a level
    outside (0, 1).

    ``estimator="css"`` with a fixed ``ma=q`` refines every gated series' Hannan-Rissanen (phi, theta) by conditional
    least squares (``ForecastEngine.fit_forecast_arma(..., estimator="css")``, DESIGN.md section 2 item 16); schema
    unchanged, ``conf_int=`` works as above.  ``estimator=None`` (or ``"hr"``) leaves everything as it was.  Refused
    without ``ma=``, with candidate MA orders, ``select=`` or ``interval=``.  ``estimator="ml"`` refines that CSS
    estimate by the exact Gaussian likelihood (``ForecastEngine.fit_forecast_arma(..., estimator="ml")``, DESIGN.md
    section 2 item 19), with the same arguments, refusals, schema and ``conf_int=``.  ``predictor="kalman"`` with
    ``estimator="ml"`` predicts with that likelihood's Kalman filter (``ForecastEngine.fit_forecast_arma(...,
    predictor="kalman")``, DESIGN.md section 2 item 20: SARIMAX's ``predict()`` / ``get_forecast()``), ``conf_int=``
    bands from its own standard errors; refused with any other estimator.
    ``joint_beta=True`` with ``estimator="css"`` estimates the design's coefficients jointly with (phi, theta)
    (``ForecastEngine.fit_forecast_arma(..., joint_beta=True)``, DESIGN.md section 2 item 17: regression with ARIMA errors
    as SARIMAX fits it, by the conditional likelihood); schema unchanged, ``conf_int=`` works as above.  Refused without
    ``estimator="css"``.
    ``refit="css"`` with candidate MA orders refits every series' winning (p, d, q) by conditional least squares, as the
    reference fits its final model on the tuned order (``ForecastEngine.fit_select_arma(..., refit="css")``, DESIGN.md
    section 2 item 18); ``joint_beta=True`` with it estimates beta jointly in that refit.  Schema unchanged, ``conf_int=``
    works as above.  Refused with a fixed ``ma=``, with ``estimator=``, ``select=`` or ``interval=``, and for any value
    other than ``"css"`` or ``"ml"``.  ``refit="ml"`` refines that refit by exact likelihood
    (``ForecastEngine.fit_select_arma(..., refit="ml")``, DESIGN.md section 2 item 21), and ``predictor="kalman"`` with
    it predicts with the likelihood's Kalman filter, ``conf_int=`` bands from its own standard errors: the reference's
    final model and its ``predict()``.  ``joint_beta=True`` is refused with ``refit="ml"``.
    """
    eng = engine or default_engine()
    keys = list(keys)
    fitted_col = value_col + "_Fitted"
    z = _z_of(interval)
    cz = _conf_z(conf_int, ar, select, interval)
    est = _estimator(estimator, ma, select, interval)
    pr = _predictor(predictor, est, refit)
    ref = _refit(refit, ma, est, select, interval)
    jb = _joint_beta(joint_beta, est, ref)
    if ma is None:
        diff = _diff_order(diff, ar, select, interval, mode)
        ar = _ar_orders_for(diff, ar, select, interval, mode)
    else:
        ar, diff, ma = _arma_orders(ma, ar, diff, select, interval, mode)
    zb = z if z is not None else cz               # the band's quantile, whichever of the two asked for it
    if pack == "host" and select is None and z is None and ar is None and isinstance(pdf, pd.DataFrame):
        one = _single_group_fast(pdf, keys, date_col, value_col, freq, horizon, mode, design, eng, null_keys_on_gaps)
        if one is not None:
            return one
    buckets = _buckets_for(pdf, keys, date_col, value_col, freq, pack, eng)
    parts, lengths = [], []
    for b, out_days, n_pred, y_host, pred, se in _fit_buckets(buckets, eng, freq, horizon, mode, design, select,
                                                              pack == "device", z is not None, ar, diff, ma,
                                                              cz is not None, est, jb, ref, pr):
        n = y_host.shape[0]
        row_of = np.repeat(np.arange(n), n_pred)
        # key columns keep the dtype they came in with (no per-row string inference on N x T values)
        frame = {k: pd.Series(b.key_frame[k].array.take(row_of), dtype=b.key_frame[k].dtype, copy=False) for k in keys}
        frame[date_col] = np.tile(out_days.astype("datetime64[ns]"), n)
        if mode == "holdout":
            frame[value_col] = np.ascontiguousarray(y_host).reshape(-1)
        else:
            frame[value_col] = np.full(n * n_pred, np.nan, dtype=np.float32)
        frame[fitted_col] = pred.reshape(-1)
        if zb is not None:
            frame[value_col + "_Lower"], frame[value_col + "_Upper"] = _bounds(pred, se, zb)
        if null_keys_on_gaps and mode == "holdout":
            gap = np.isnan(frame[value_col])
            if gap.any():
                for k in keys:
                    frame[k] = frame[k].astype(object).where(~gap, None)
        parts.append(pd.DataFrame(frame))
        lengths.append(n_pred)
    if not parts:
        bounds = ({value_col + "_Lower": pd.Series(dtype=np.float32), value_col + "_Upper": pd.Series(dtype=np.float32)}
                  if zb is not None else {})
        return pd.DataFrame({**{k: pd.Series(dtype=object) for k in keys},
                             date_col: pd.Series(dtype="datetime64[ns]"),
                             value_col: pd.Series(dtype=np.float32), fitted_col: pd.Series(dtype=np.float32), **bounds})
    if len(parts) == 1:
        return parts[0]
    out = pd.concat(parts, ignore_index=True)
    return out.take(_global_order(buckets, keys, lengths)).reset_index(drop=True)


def backtest_groups(pdf, *, keys=DEFAULT_KEYS, date_col="Date", value_col="Demand", freq="W-MON",
                    horizon=FORECAST_HORIZON, n_origins=3, step=None, design="trend_season_exog",
                    pack: str = "host", engine: ForecastEngine | None = None) -> pd.DataFrame:
    """Rolling-origin backtest of every group in ``pdf`` (pandas, or Arrow with ``pack="device"`` / an Arrow table):
    each group is cut at ``n_origins`` origins placed relative to its OWN last date, ``t_k = t_len - horizon -
    (n_origins-1-k) * step`` grid rows (``step`` defaults to ``horizon``), so the last origin is the reference's train /
    score split (02:372-380).  Origin k fits the group's rows before t_k and its ``horizon`` forecasts are scored
    against the actual values (``ForecastEngine.backtest``: one pass over the data and one call per calendar bucket).

    Returns ``backtest_schema(keys)`` rows in (key, Cutoff) order: keys..., ``Cutoff`` (first forecast date of the
    origin), ``N`` (scored points: forecast and actual value both present), ``MSE``, ``MAE``, ``Bias`` (mean of
    forecast - actual) and ``MAPE`` (over the scored points with a non-zero actual value), float32, NaN where nothing is
    averaged.  A (group, origin) with fewer than 33 fit rows is left out (the engine's minimum fit window), so a short
    group contributes fewer origins or no row at all."""
    eng = engine or default_engine()
    keys = list(keys)
    K, horizon = int(n_origins), int(horizon)
    step = horizon if step is None else int(step)
    if K < 1 or step < 1:
        raise ValueError("need n_origins >= 1 and step >= 1")
    buckets = _buckets_for(pdf, keys, date_col, value_col, freq, pack, eng)
    parts, used, lengths = [], [], []
    for b in buckets:
        first = b.t_len - horizon - (K - 1) * step
        k0 = 0 if first >= 33 else -(-(33 - first) // step)      # origins below 33 fit rows are left out
        if k0 >= K:
            continue
        origins = np.asarray(eng.plan_backtest(b.start, b.t_len, freq, horizon, K - k0, step, design))
        yd = b.y
        if pack != "device" and isinstance(eng, ForecastEngine):
            from .engine import device_packed
            yd = device_packed(b.y)
        res = eng.backtest(yd, want_pred=False)
        met = np.asarray(_host(res["metrics"]), dtype=np.float32)          # [k, n, 4]
        cnt = np.asarray(_host(res["count"]), dtype=np.int32)              # [k, n]
        k, n = cnt.shape
        row_of = np.repeat(np.arange(n), k)
        cut = D.calendar_grid(b.start, b.t_len, freq)[origins].astype("datetime64[ns]")
        frame = {c: pd.Series(b.key_frame[c].array.take(row_of), dtype=b.key_frame[c].dtype, copy=False) for c in keys}
        frame["Cutoff"] = np.tile(cut, n)
        frame["N"] = np.ascontiguousarray(cnt.T).reshape(-1)
        mt = np.ascontiguousarray(met.transpose(1, 0, 2)).reshape(-1, len(BACKTEST_METRICS))
        for j, m in enumerate(BACKTEST_METRICS):
            frame[m] = mt[:, j]
        parts.append(pd.DataFrame(frame))
        used.append(b)
        lengths.append(k)
    if not parts:
        return pd.DataFrame({**{c: pd.Series(dtype=object) for c in keys}, "Cutoff": pd.Series(dtype="datetime64[ns]"),
                             "N": pd.Series(dtype=np.int32), **{m: pd.Series(dtype=np.float32) for m in BACKTEST_METRICS}})
    if len(parts) == 1:
        return parts[0]
    out = pd.concat(parts, ignore_index=True)
    return out.take(_global_order(used, keys, lengths)).reset_index(drop=True)


def forecast_table(table, *, keys=DEFAULT_KEYS, date_col="Date", value_col="Demand",
                   freq="W-MON", horizon=FORECAST_HORIZON, mode="holdout", design="trend_season_exog",
                   engine: ForecastEngine | None = None, pack: str = "host", select=None,
                   null_keys_on_gaps: bool = False, interval=None, ar=None, diff=None, ma=None,
                   conf_int=None, estimator=None, joint_beta=False, refit=None, predictor=None):
    """Arrow ``Table``/``RecordBatch`` in -> Arrow ``Table`` with ``tuning_schema`` out (the ``mapInArrow``
    flavour of the boundary).  No pandas frame of the rows on either side: keys are dictionary-encoded on the way
    in and expanded from a dictionary on the way out, dates and values are NumPy views of Arrow buffers.
    ``interval=level`` adds the ``{value}_Lower`` / ``{value}_Upper`` columns of ``forecast_groups`` (schema:
    ``tuning_schema(..., interval=True)``).  ``ar=p`` fits regression with AR(p) errors and ``ar=(0, 1, 2, 3, 4)`` chooses the order per series, as in
    ``forecast_groups``; ``diff=d`` with ``ar=p`` fits ARIMA(p, d, 0) errors as there, and ``ma=q`` ARIMA(p, d, q); tuples of ``ar``, ``diff`` and
    ``ma`` choose (p, d, q) per series.  ``conf_int=level`` adds the same two columns for those forecasts, and
    ``estimator="css"`` (or ``"ml"``) refines a fixed ``ma=q``'s estimate and ``joint_beta=True`` adds beta to it, and ``refit="css"``
    (or ``"ml"``) refits the selection's winners (with ``joint_beta=True``: beta jointly), and ``predictor="kalman"`` with
    ``estimator="ml"`` or ``refit="ml"`` predicts with the Kalman filter, as in ``forecast_groups``."""
    import pyarrow as pa

    if isinstance(table, pa.RecordBatch):
        table = pa.Table.from_batches([table])
    eng = engine or default_engine()
    keys = list(keys)
    z = _z_of(interval)
    cz = _conf_z(conf_int, ar, select, interval)
    est = _estimator(estimator, ma, select, interval)
    pr = _predictor(predictor, est, refit)
    ref = _refit(refit, ma, est, select, interval)
    jb = _joint_beta(joint_beta, est, ref)
    if ma is None:
        diff = _diff_order(diff, ar, select, interval, mode)
        ar = _ar_orders_for(diff, ar, select, interval, mode)
    else:
        ar, diff, ma = _arma_orders(ma, ar, diff, select, interval, mode)
    zb = z if z is not None else cz
    schema = tuning_schema(keys, date_col, value_col, interval=zb is not None)
    buckets = _buckets_for(table, keys, date_col, value_col, freq, pack, eng)
    parts, lengths = [], []
    for b, out_days, n_pred, y_host, pred, se in _fit_buckets(buckets, eng, freq, horizon, mode, design, select,
                                                              pack == "device", z is not None, ar, diff, ma,
                                                              cz is not None, est, jb, ref, pr):
        n = y_host.shape[0]
        row_of = np.repeat(np.arange(n, dtype=np.int32), n_pred)
        cols = []
        demand = (np.ascontiguousarray(y_host).reshape(-1) if mode == "holdout"
                  else np.full(n * n_pred, np.nan, dtype=np.float32))
        gap = np.isnan(demand) if (null_keys_on_gaps and mode == "holdout") else None
        for k in keys:
            kv = b.key_arrow[k] if b.key_arrow is not None else pa.array(b.key_frame[k].astype(str).to_numpy(dtype=object))
            col = _expand_strings(kv, row_of)
            if gap is not None and gap.any():                  # reference 02:490: asfreq rows have no key values
                import pyarrow.compute as pc
                col = pc.if_else(pa.array(gap), pa.scalar(None, pa.string()), col)
            cols.append(col)
        day32 = out_days.astype("datetime64[D]").astype(np.int32)
        cols.append(pa.array(np.tile(day32, n)).cast(pa.date32()))
        cols.append(pa.array(demand, from_pandas=True))               # NaN -> null, like the pandas route
        cols.append(pa.array(np.ascontiguousarray(pred).reshape(-1), from_pandas=True))
        if zb is not None:
            cols.extend(pa.array(v, from_pandas=True) for v in _bounds(pred, se, zb))
        parts.append(pa.Table.from_arrays(cols, schema=schema))
        lengths.append(n_pred)
    if not parts:
        return schema.empty_table()
    if len(parts) == 1:
        return parts[0]
    return pa.concat_tables(parts).combine_chunks().take(pa.array(_global_order(buckets, keys, lengths)))


def forecast_arrow_batches(batches, **kw):
    """``mapInArrow`` adapter: an iterator of RecordBatches (one Spark partition) -> batches."""
    import pyarrow as pa

    batches = list(batches)
    if not batches:
        return
    yield from forecast_table(pa.Table.from_batches(batches), **kw).to_batches()
