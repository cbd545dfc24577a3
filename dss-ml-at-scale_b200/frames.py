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

FORECAST_HORIZON = 40                      # 02:341
DEFAULT_KEYS = ("Product", "SKU")          # 02:526
EXO_FIELDS = ("covid", "christmas", "new_year")   # 02:431


# ---- schemas (02:360-370, 02:498-506) as pyarrow; pyspark StructTypes on demand ---------
def tuning_schema(keys=DEFAULT_KEYS, date_col="Date", value_col="Demand"):
    import pyarrow as pa

    return pa.schema([(k, pa.string()) for k in keys]
                     + [(date_col, pa.date32()), (value_col, pa.float32()), (value_col + "_Fitted", pa.float32())])


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
        yield b, dates[i], n_pred, y_host, np.ascontiguousarray(pred[int(rows[i]):int(rows[i + 1]), :n_pred])


def _fit_buckets(buckets, eng, freq, horizon, mode, design, select, on_device):
    """Run the engine over every bucket: yields (bucket, out_days, n_pred, y_host, pred_host)."""
    t_fit_min = min((b.t_len - (horizon if mode == "holdout" else 0)) for b in buckets) if buckets else 0
    if (select is None and len(buckets) >= RAGGED_MIN_BUCKETS and (mode == "holdout" or 1 <= horizon <= 64)
            and hasattr(eng, "fit_forecast_ragged") and t_fit_min >= 33 and all(b.t_len <= 65535 for b in buckets)):
        yield from _fit_buckets_ragged(buckets, eng, freq, horizon, mode, design, on_device)
        return
    for b in buckets:
        out_days, pred_start, n_pred = eng.plan_calendar(b.start, b.t_len, freq, horizon, mode, design)
        if select is not None:
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
        yield b, out_days, n_pred, y_host, pred


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
                    null_keys_on_gaps: bool = False) -> pd.DataFrame:
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
    """
    eng = engine or default_engine()
    keys = list(keys)
    fitted_col = value_col + "_Fitted"
    if pack == "host" and select is None and isinstance(pdf, pd.DataFrame):
        one = _single_group_fast(pdf, keys, date_col, value_col, freq, horizon, mode, design, eng, null_keys_on_gaps)
        if one is not None:
            return one
    buckets = _buckets_for(pdf, keys, date_col, value_col, freq, pack, eng)
    parts, lengths = [], []
    for b, out_days, n_pred, y_host, pred in _fit_buckets(buckets, eng, freq, horizon, mode, design, select, pack == "device"):
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
        if null_keys_on_gaps and mode == "holdout":
            gap = np.isnan(frame[value_col])
            if gap.any():
                for k in keys:
                    frame[k] = frame[k].astype(object).where(~gap, None)
        parts.append(pd.DataFrame(frame))
        lengths.append(n_pred)
    if not parts:
        return pd.DataFrame({**{k: pd.Series(dtype=object) for k in keys},
                             date_col: pd.Series(dtype="datetime64[ns]"),
                             value_col: pd.Series(dtype=np.float32), fitted_col: pd.Series(dtype=np.float32)})
    if len(parts) == 1:
        return parts[0]
    out = pd.concat(parts, ignore_index=True)
    return out.take(_global_order(buckets, keys, lengths)).reset_index(drop=True)


def forecast_table(table, *, keys=DEFAULT_KEYS, date_col="Date", value_col="Demand",
                   freq="W-MON", horizon=FORECAST_HORIZON, mode="holdout", design="trend_season_exog",
                   engine: ForecastEngine | None = None, pack: str = "host", select=None,
                   null_keys_on_gaps: bool = False):
    """Arrow ``Table``/``RecordBatch`` in -> Arrow ``Table`` with ``tuning_schema`` out (the ``mapInArrow``
    flavour of the boundary).  No pandas frame of the rows on either side: keys are dictionary-encoded on the way
    in and expanded from a dictionary on the way out, dates and values are NumPy views of Arrow buffers."""
    import pyarrow as pa

    if isinstance(table, pa.RecordBatch):
        table = pa.Table.from_batches([table])
    eng = engine or default_engine()
    keys = list(keys)
    schema = tuning_schema(keys, date_col, value_col)
    buckets = _buckets_for(table, keys, date_col, value_col, freq, pack, eng)
    parts, lengths = [], []
    for b, out_days, n_pred, y_host, pred in _fit_buckets(buckets, eng, freq, horizon, mode, design, select, pack == "device"):
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
