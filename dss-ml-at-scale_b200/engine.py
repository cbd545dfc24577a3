"""``ForecastEngine`` -- the Python face of one ``mmf_ctx`` (one per process / per GPU).

Replaces, for every group at once, what one Spark Python worker does per group in
``build_tune_and_score_model`` (group_apply/02_Fine_Grained_Demand_Forecasting.py:
435-494): fit on the train rows, predict the requested rows.  Inputs are packed
series ``y[N, ld]`` float32 (NaN = missing) that share one calendar.

Buffers may be NumPy arrays (host; pinned ones from :func:`pinned_empty` copy at
PCIe speed) or CUDA ``torch`` tensors (device; zero copies).  PyTorch is only
plumbing here (device memory / streams); all arithmetic is in ``libmmf.so``.
"""
from __future__ import annotations

import ctypes as C
import threading
import weakref
from dataclasses import dataclass

import numpy as np

from . import _native as N
from . import design as D


def _is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


def _describe(x, name: str):
    """-> (ptr, rows, cols, ld) of a 1-D/2-D float32/int32 buffer with unit inner stride."""
    if _is_torch(x):
        if x.dim() == 1:
            return x.data_ptr(), x.shape[0], 1, 1
        if x.dim() != 2 or (x.shape[1] > 1 and x.stride(1) != 1):
            raise ValueError(f"{name}: need a 2-D tensor with unit inner stride")
        return x.data_ptr(), x.shape[0], x.shape[1], x.stride(0)
    a = x
    if not isinstance(a, np.ndarray):
        raise TypeError(f"{name}: expected numpy.ndarray or torch.Tensor, got {type(x)}")
    if a.ndim == 1:
        return a.ctypes.data, a.shape[0], 1, 1
    if a.ndim != 2 or (a.shape[1] > 1 and a.strides[1] != a.itemsize):
        raise ValueError(f"{name}: need a 2-D array with unit inner stride")
    if a.strides[0] % a.itemsize:
        raise ValueError(f"{name}: row stride is not a multiple of the item size")
    return a.ctypes.data, a.shape[0], a.shape[1], a.strides[0] // a.itemsize


class _PinnedPool:
    """Page-locked blocks are expensive on both ends (cudaHostAlloc ~ 0.5 ms/MB, cudaFreeHost more): blocks a
    NumPy view no longer references go back to a small free list (capped) instead of to the driver, so a worker
    that packs one batch after another pins its staging memory once."""
    MAX_BYTES = 4 << 30
    MAX_BLOCKS = 8

    def __init__(self):
        self.free = []                       # [(size, address)]
        self.lock = threading.Lock()

    def take(self, lib, nbytes):
        gran = max(4096, 1 << max(0, nbytes.bit_length() - 4))          # <= 6 % over-allocation
        size = -(-nbytes // gran) * gran
        with self.lock:
            fits = [blk for blk in self.free if size <= blk[0] <= size + size // 4]
            if fits:
                blk = min(fits)
                self.free.remove(blk)
                return blk[1], blk[0]
        p = C.c_void_p()
        N.check(lib.mmf_alloc_pinned(size, C.byref(p)))
        return p.value, size

    def give(self, lib, addr, size):
        with self.lock:
            if len(self.free) < self.MAX_BLOCKS and sum(b[0] for b in self.free) + size <= self.MAX_BYTES:
                self.free.append((size, addr))
                return
        lib.mmf_free_pinned(addr)

    def clear(self, lib):
        with self.lock:
            blocks, self.free = self.free, []
        for _, addr in blocks:
            lib.mmf_free_pinned(addr)


_pinned_pool = _PinnedPool()


def pinned_empty(shape, dtype=np.float32) -> np.ndarray:
    """NumPy array over page-locked host memory (``mmf_alloc_pinned``): the Arrow/NumPy ->
    device hop becomes one ``cudaMemcpyAsync`` per chunk.  Blocks are recycled through a small pool."""
    lib = N.load()
    dtype = np.dtype(dtype)
    count = int(np.prod(shape))
    addr, size = _pinned_pool.take(lib, max(count * dtype.itemsize, 1))
    buf = (C.c_byte * size).from_address(addr)
    arr = np.frombuffer(buf, dtype=dtype, count=count).reshape(shape)
    weakref.finalize(buf, _pinned_pool.give, lib, addr, size)
    return arr


def release_pinned_pool() -> None:
    """Hand the recycled page-locked blocks back to the driver."""
    _pinned_pool.clear(N.load())


def device_packed(y, device="cuda"):
    """Copy packed series (NumPy [n,t] or torch) into a CUDA tensor whose row pitch is a multiple of
    4 floats -- the layout the TMA/wgmma fast path needs.  Returns the [n, t] view."""
    import torch

    src = torch.from_numpy(np.ascontiguousarray(y)) if isinstance(y, np.ndarray) else y
    n, t = src.shape
    full = torch.empty((n, (t + 3) & ~3), dtype=torch.float32, device=device)
    view = full[:, :t]
    view.copy_(src)
    return view


def alloc_packed(n: int, t: int, pinned: bool = True, dtype=np.float32):
    """Host buffer for ``n`` packed series of length ``t`` with a TMA-friendly row pitch
    (multiple of 16 bytes).  Returns the [n, t] view; ``view.base`` keeps the padded rows.
    ``dtype`` int16 / uint16 / int32: an integer demand buffer for ``fit_forecast`` (half the PCIe bytes for 16 bit)."""
    dtype = np.dtype(dtype)
    per16 = 16 // dtype.itemsize
    ld = -(-t // per16) * per16
    full = pinned_empty((n, ld), dtype) if pinned else np.empty((n, ld), dtype=dtype)
    return full[:, :t]


def to_integer_demand(y: np.ndarray, dtype=np.uint16, out=None) -> np.ndarray:
    """float32 series (NaN = missing) -> an integer demand buffer with the type's sentinel for missing values.
    Raises if a value is not an integer or does not fit (the integer ingest must stay bit-exact)."""
    dtype = np.dtype(dtype)
    info = np.iinfo(dtype)
    miss = N.INT_MISSING[dtype.name]
    lo, hi = (info.min + 1, info.max) if miss == info.min else (info.min, info.max - 1)
    if out is None:
        out = np.empty(y.shape, dtype=dtype)
    y2, o2 = (y.reshape(1, -1), out.reshape(1, -1)) if y.ndim == 1 else (y, out)
    block = max(1, (32 << 20) // max(y2.shape[1], 1))                   # ~128 MB of float32 per pass
    for i0 in range(0, y2.shape[0], block):
        yb = y2[i0:i0 + block]
        fin = np.isfinite(yb)
        yv = np.where(fin, yb, 0)
        if not (np.array_equal(yv, np.rint(yv)) and yv.min(initial=0) >= lo and yv.max(initial=0) <= hi):
            raise ValueError(f"values are not integers within [{lo}, {hi}]: cannot be carried as {dtype.name}")
        o2[i0:i0 + block] = np.where(fin, yv, miss).astype(dtype)
    return out


@dataclass
class Stats:
    kernel_ms: float
    total_ms: float
    n_series: int
    n_pending: int
    h2d_bytes: int
    d2h_bytes: int
    kernel_launches: int
    kernel_used: str


class ForecastEngine:
    """One library context: streams, staging buffers, the planned calendar design.

    ``stream_solve`` is accepted for compatibility and has no effect."""

    def __init__(self, device: int | None = None, kernel: str = "auto", assume_finite: bool = False,
                 chunk_series: int = 0, stream: int | None = None, tc_variant: int = 0,
                 host_narrow: str = "auto", host_threads: int = 0, stream_solve: bool = False):
        self._lib = N.load()
        cfg = N.MmfConfig()
        cfg.device = -1 if device is None else int(device)
        cfg.kernel = N.KERNELS[kernel]
        cfg.assume_finite = 1 if assume_finite else 0
        cfg.chunk_series = int(chunk_series)
        cfg.tc_variant = int(tc_variant)
        cfg.stream = stream
        # host (NumPy) float32 input: narrow integer-valued chunks to uint16 on host threads so that half the bytes
        # cross PCIe ("auto" / "on" / "off"); exact or not used -- the forecasts are bit-equal either way
        cfg.host_narrow = {"auto": 0, "on": 1, "off": 2}[host_narrow]
        cfg.host_threads = int(host_threads)
        # no effect: the library accepts and ignores the field (series with gaps are always solved in a pass of their
        # own after the tensor-core kernel)
        cfg.stream_solve = 1 if stream_solve else 0
        h = C.c_void_p()
        N.check(self._lib.mmf_create(C.byref(cfg), C.byref(h)))
        self._h = h
        self._finalizer = weakref.finalize(self, self._lib.mmf_destroy, h)
        self.t_fit = None
        self.n_rows = None
        self.launches = 0            # kernels launched through this engine (bench reports it)

    # ---- lifecycle -----------------------------------------------------------
    def close(self) -> None:
        if self._finalizer.alive:
            self._finalizer()

    def set_stream(self, cuda_stream_ptr: int | None) -> None:
        """Enqueue on a caller-owned stream (e.g. ``torch.cuda.current_stream().cuda_stream``)."""
        N.check(self._lib.mmf_set_stream(self._h, C.c_void_p(cuda_stream_ptr or 0)))

    def synchronize(self) -> None:
        N.check(self._lib.mmf_synchronize(self._h))

    # ---- design --------------------------------------------------------------
    def plan(self, X: np.ndarray, t_fit: int, has_constant: bool) -> None:
        """Plan a raw design ``X[n_rows, p<=16]`` (float64): rows [0,t_fit) fit, the rest forecast."""
        X = np.ascontiguousarray(X, dtype=np.float64)
        if X.ndim != 2:
            raise ValueError("X must be 2-D")
        N.check(self._lib.mmf_plan_design(self._h, X.ctypes.data, X.shape[0], X.shape[1], int(t_fit),
                                          1 if has_constant else 0))
        self.t_fit = int(t_fit)
        self.n_rows = int(X.shape[0])
        self._calendar_key = None

    def plan_calendar(self, start, t_len: int, freq: str = "D", horizon: int = 28, mode: str = "future",
                      design: str = "trend_season_exog", max_diff: int | None = None):
        """Build and plan the design for a bucket of series that start at ``start`` and have
        ``t_len`` grid rows.  Returns ``(dates_of_prediction_rows, pred_start, n_pred)``.
        The calendar planned last is remembered: the literal drop-in (one group per call, every group on the same
        calendar, 02:523-528) whitens and uploads its design once per worker, not once per group.
        ``max_diff`` (1 .. MMF_DIFF_MAX) also plans the differenced designs of ``fit_forecast_arima`` on the same
        calendar (``plan_arima``); None leaves the ARIMA plan as it is."""
        key = (str(np.datetime64(start, "D")), int(t_len), freq, int(horizon), mode, design,
               None if max_diff is None else int(max_diff))
        if getattr(self, "_calendar_key", None) == key:
            return self._calendar_plan
        if mode == "holdout":                       # reference semantics, 02:372-380 + 484-488
            t_fit = t_len - horizon
            if t_fit < 1:
                raise ValueError("series shorter than the forecast horizon")
            days = D.calendar_grid(start, t_len, freq)
            pred_start, n_pred = 0, t_len
        elif mode == "future":
            t_fit = t_len
            days = D.calendar_grid(start, t_len + horizon, freq)
            pred_start, n_pred = t_len, horizon
        else:
            raise ValueError(f"mode must be 'holdout' or 'future', got {mode!r}")
        X = D.design_matrix(days, t_fit, design)
        self.plan(X, t_fit, D.design_has_constant(design))
        if max_diff is not None:
            self.plan_arima(X, t_fit, max_diff)
        self._calendar_key = key
        self._calendar_plan = (days[pred_start:pred_start + n_pred], pred_start, n_pred)
        return self._calendar_plan

    # ---- ragged batches: many calendars, one launch ----------------------------------------------
    def plan_calendars(self, starts, t_lens, freq: str = "D", horizon: int = 28, design: str = "trend_season_exog",
                       mode: str = "future"):
        """Plan ALL calendars of a ragged batch: calendar ``c`` starts at ``starts[c]`` and has ``t_lens[c]`` grid rows.
        ``mode="future"``: every series is fit on its whole history and forecast ``horizon`` rows past its end;
        ``mode="holdout"`` (the reference's contract, 02:372-380 + 484-494): the last ``horizon`` rows are held out and a
        value is produced for EVERY date of the calendar.  One host call whitens every calendar (``mmf_plan_calendars``);
        ``fit_forecast_ragged`` then fits all groups in one pass of the tensor-core kernel (+ one of the predict kernel in
        holdout mode).  Returns the prediction dates per calendar: ``[n_cal, horizon]`` datetime64[D] (future) or a list
        of ``t_lens[c]``-long arrays (holdout)."""
        starts = [np.datetime64(s, "D") for s in starts]
        t_lens = [int(t) for t in t_lens]
        if len(starts) != len(t_lens) or not starts:
            raise ValueError("starts and t_lens must have the same non-zero length")
        if mode not in ("future", "holdout"):
            raise ValueError(f"mode must be 'holdout' or 'future', got {mode!r}")
        blocks, dates, t_fit, p_start, n_pred = [], [], [], [], []
        for st, tl in zip(starts, t_lens):
            if mode == "future":
                days = D.calendar_grid(st, tl + horizon, freq)
                tf, ps, npd = tl, tl, horizon
            else:
                if tl - horizon < 1:
                    raise ValueError("series shorter than the forecast horizon")
                days = D.calendar_grid(st, tl, freq)
                tf, ps, npd = tl - horizon, 0, tl
            blocks.append(D.design_matrix(days, tf, design))
            dates.append(np.asarray(days[ps:ps + npd], dtype="datetime64[D]"))
            t_fit.append(tf); p_start.append(ps); n_pred.append(npd)
        self.plan_designs(blocks, t_fit, p_start, n_pred, D.design_has_constant(design))
        self._ragged = self._ragged[:3] + (mode,)        # holdout tables are NaN-filled even when one window fits all
        return np.stack(dates) if mode == "future" else dates

    def plan_designs(self, Xs, t_fit, pred_start, n_pred, has_constant: bool) -> None:
        """Plan a ragged batch on caller designs (``mmf_plan_calendars``): calendar ``c`` has the raw design ``Xs[c]``
        ``[n_rows_c, p]`` (float64, one ``p <= 16`` for all), fits rows ``[0, t_fit[c])`` and evaluates rows
        ``[pred_start[c], pred_start[c] + n_pred[c])``.  One common ``n_pred <= 64`` is written by the fit kernel's
        epilogue; anything else by the predict kernel, and ``fit_forecast_ragged`` then returns a NaN-filled table as
        wide as the largest ``n_pred[c]``."""
        blocks = [np.asarray(X, dtype=np.float64) for X in Xs]
        if not blocks or any(b.ndim != 2 or b.shape[1] != blocks[0].shape[1] for b in blocks):
            raise ValueError("Xs must be a non-empty list of 2-D designs with the same number of columns")
        arr = [np.array(v, dtype=np.int32) for v in ([b.shape[0] for b in blocks], t_fit, pred_start, n_pred)]
        if any(a.shape != (len(blocks),) for a in arr[1:]):
            raise ValueError("t_fit, pred_start and n_pred need one entry per design")
        X = np.ascontiguousarray(np.concatenate(blocks, axis=0))
        N.check(self._lib.mmf_plan_calendars(self._h, X.ctypes.data, len(blocks), arr[0].ctypes.data, arr[1].ctypes.data,
                                             arr[2].ctypes.data, arr[3].ctypes.data, X.shape[1],
                                             1 if has_constant else 0))
        npd = arr[3]
        # (n_cal, columns of the output table, columns y must have, who writes the table: the fit kernel's epilogue
        # ("future") or the predict kernel ("holdout"), as mmf_plan_calendars decides)
        one_window = bool((npd == npd[0]).all() and npd[0] <= 64)
        self._ragged = (len(blocks), int(npd.max()), int(arr[1].max()), "future" if one_window else "holdout")

    def fit_forecast_ragged(self, y, cal_row_start, out=None, status=None, want_status: bool = False,
                            want_stats: bool = False):
        """Fit a ragged batch: ``y`` [n, ld] float32 CUDA tensor whose rows are grouped by calendar -- calendar ``c``
        owns rows ``[cal_row_start[c], cal_row_start[c+1])`` and reads columns ``[0, t_fit_c)`` of them.  Returns the
        ``[n, horizon]`` forecast table (future mode) or ``[n, longest calendar]`` with a value for every date of each
        row's own calendar and NaN beyond it (holdout mode) -- or a dict with ``status`` / ``stats``."""
        import torch
        if getattr(self, "_ragged", None) is None:
            raise RuntimeError("plan_calendars() must be called first")
        n_cal, n_out, t_max, mode = self._ragged
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32) or t_have < t_max:
            raise ValueError(f"y must be a float32 CUDA tensor with at least {t_max} columns")
        rows = np.ascontiguousarray(cal_row_start, dtype=np.int64)
        if rows.shape != (n_cal + 1,):
            raise ValueError("cal_row_start needs n_cal + 1 entries")
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        if out is None:
            if mode == "future":
                out = torch.empty((n, n_out), device=y.device, dtype=torch.float32)
            else:       # holdout: [n, longest calendar]; columns beyond a row's own calendar stay NaN
                out = torch.full((n, (n_out + 3) & ~3), float("nan"), device=y.device, dtype=torch.float32)[:, :n_out]
        if want_status and status is None:
            status = torch.empty(n, device=y.device, dtype=torch.int32)
        st = N.MmfStats() if want_stats else None
        N.check(self._lib.mmf_fit_forecast_ragged_f32(self._h, yp, n, ld_y, rows.ctypes.data, out.data_ptr(), out.stride(0),
                                                      status.data_ptr() if status is not None else None,
                                                      C.byref(st) if st is not None else None))
        if not (want_status or want_stats):
            return out
        res = {"pred": out}
        if status is not None:
            res["status"] = status
        if st is not None:
            self.launches += st.kernel_launches
            res["stats"] = Stats(st.kernel_ms, st.total_ms, st.n_series, st.n_pending, st.h2d_bytes, st.d2h_bytes,
                                 st.kernel_launches, "tc")
        return res

    # ---- rolling-origin backtest: K origins, one pass over the data -----------------------------------------------
    def plan_backtest(self, start, t_len: int, freq: str = "D", horizon: int = 28, n_origins: int = 3,
                      step: int | None = None, design: str = "trend_season_exog"):
        """Plan a backtest of series that start at ``start`` and have ``t_len`` grid rows: origin ``k`` of ``n_origins``
        fits rows ``[0, t_k)`` and forecasts ``[t_k, t_k + horizon)``, ``t_k = t_len - horizon - (n_origins-1-k) * step``
        (``step`` defaults to ``horizon``), so the last origin is the reference's train / score split (02:372-380).
        Every origin's model is the plain model planned with ``t_fit = t_k`` on the design of the whole window
        (``mmf_plan_backtest``).  Returns the origins (int32 array); the first forecast date of origin k is
        ``calendar_grid(start, t_len)[t_k]``."""
        step = int(horizon if step is None else step)
        n_origins, horizon, t_len = int(n_origins), int(horizon), int(t_len)
        if step < 1:
            raise ValueError("step must be >= 1")
        origins = np.array([t_len - horizon - (n_origins - 1 - k) * step for k in range(n_origins)], dtype=np.int32)
        days = D.calendar_grid(start, t_len, freq)
        X = np.ascontiguousarray(D.design_matrix(days, t_len - horizon, design), dtype=np.float64)
        N.check(self._lib.mmf_plan_backtest(self._h, X.ctypes.data, X.shape[0], X.shape[1],
                                            1 if D.design_has_constant(design) else 0, len(origins),
                                            origins.ctypes.data, horizon))
        self._backtest = (origins, horizon, t_len)
        return origins

    def backtest(self, y, want_pred: bool = True, want_stats: bool = False):
        """Run the planned backtest on ``y`` [n, >= t_len] (float32 CUDA tensor, NaN = missing).  Returns
        ``{"pred": [K, n, horizon] or None, "metrics": [K, n, 4] (MSE, MAE, bias, MAPE), "count": [K, n],
        "status": [K, n]}`` as CUDA tensors; forecasts are scored on the device (``mmf_backtest_f32``).  The kernel reads
        ``y`` with TMA: a tensor whose row pitch is not a multiple of 4 floats or that is not 16-B aligned is first copied
        into a pitched buffer (``device_packed``)."""
        import torch
        if getattr(self, "_backtest", None) is None:
            raise RuntimeError("plan_backtest() must be called first")
        origins, h, t_len = self._backtest
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32) or t_have < t_len:
            raise ValueError(f"y must be a float32 CUDA tensor with at least {t_len} columns")
        if ld_y % 4 or yp % 16:
            y = device_packed(y, device=y.device)
            yp, n, t_have, ld_y = _describe(y, "y")
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        k = len(origins)
        pred = torch.empty((k, n, (h + 3) & ~3), device=y.device, dtype=torch.float32)[:, :, :h] if want_pred else None
        metrics = torch.empty((k, n, N.BT_NMETRIC), device=y.device, dtype=torch.float32)
        count = torch.empty((k, n), device=y.device, dtype=torch.int32)
        status = torch.empty((k, n), device=y.device, dtype=torch.int32)
        st = N.MmfStats() if want_stats else None
        N.check(self._lib.mmf_backtest_f32(self._h, yp, n, ld_y, pred.data_ptr() if pred is not None else None,
                                           pred.stride(1) if pred is not None else 0, metrics.data_ptr(),
                                           count.data_ptr(), status.data_ptr(), C.byref(st) if st is not None else None))
        res = {"pred": pred, "metrics": metrics, "count": count, "status": status}
        if st is not None:
            self.launches += st.kernel_launches
            res["stats"] = Stats(st.kernel_ms, st.total_ms, st.n_series, st.n_pending, st.h2d_bytes, st.d2h_bytes,
                                 st.kernel_launches, "tc")
        return res

    def whitening(self):
        W = np.zeros((N.MMF_P, N.MMF_P), dtype=np.float64)
        kept = np.zeros(N.MMF_P, dtype=np.int32)
        N.check(self._lib.mmf_get_whitening(self._h, W.ctypes.data, kept.ctypes.data))
        return W, kept.astype(bool)

    # ---- the hot path --------------------------------------------------------
    def fit_forecast(self, y, pred_start: int, n_pred: int, out=None, beta=None, status=None,
                     want_beta: bool = False, want_status: bool = False, want_stats: bool = False):
        """Fit every row of ``y`` on the planned design and evaluate rows
        [pred_start, pred_start+n_pred).  Returns ``out`` or a dict when extras are requested."""
        if self.t_fit is None:
            raise RuntimeError("plan()/plan_calendar() must be called first")
        yp, n, t_have, ld_y = _describe(y, "y")
        if t_have < self.t_fit:
            raise ValueError(f"y has {t_have} columns, the plan needs t_fit={self.t_fit}")
        on_dev = _is_torch(y) and y.is_cuda
        dt_name = str(y.dtype).replace("torch.", "")
        if dt_name != "float32" and dt_name not in N.INT_DTYPES:
            raise TypeError("y must be float32, or int16 / uint16 / int32 with the type's missing-value sentinel "
                            f"({N.INT_MISSING}); got {y.dtype}")
        if on_dev:
            import torch
            # stream-ordered with the caller's torch work: enqueue on torch's current stream
            self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)

        def make(shape, np_dtype):
            if on_dev:
                import torch
                dt = torch.float32 if np_dtype == np.float32 else torch.int32
                if len(shape) == 2 and shape[1] % 4:          # 16-B row pitch: TMA-storable by predict_tc_kernel
                    return torch.empty((shape[0], (shape[1] + 3) & ~3), device=y.device, dtype=dt)[:, :shape[1]]
                return torch.empty(shape, device=y.device, dtype=dt)
            return np.empty(shape, dtype=np_dtype)

        if out is None:
            out = make((n, n_pred), np.float32)
        if want_beta and beta is None:
            beta = make((n, N.MMF_P), np.float32)
        if want_status and status is None:
            status = make((n,), np.int32)
        op, on, ocols, ld_out = _describe(out, "out")
        if on != n or ocols < n_pred:
            raise ValueError("out has the wrong shape")
        bp = _describe(beta, "beta")[0] if beta is not None else None
        sp = _describe(status, "status")[0] if status is not None else None
        st = N.MmfStats() if want_stats else None
        if dt_name == "float32":
            N.check(self._lib.mmf_fit_forecast_f32(self._h, yp, n, ld_y, int(pred_start), int(n_pred), op, ld_out,
                                                   bp, sp, C.byref(st) if st is not None else None))
        else:       # integer demand column (int16 / uint16 halve the PCIe bytes): widened on the device, same kernels
            N.check(self._lib.mmf_fit_forecast_int(self._h, yp, N.INT_DTYPES[dt_name], n, ld_y, int(pred_start),
                                                   int(n_pred), op, ld_out, bp, sp,
                                                   C.byref(st) if st is not None else None))
        if not (want_beta or want_status or want_stats):
            return out
        res = {"pred": out}
        if beta is not None:
            res["beta"] = beta
        if status is not None:
            res["status"] = status
        if st is not None:
            self.launches += st.kernel_launches
            res["stats"] = Stats(st.kernel_ms, st.total_ms, st.n_series, st.n_pending, st.h2d_bytes,
                                 st.d2h_bytes, st.kernel_launches,
                                 {N.KERNEL_WARP: "warp", N.KERNEL_TC: "tc"}.get(st.kernel_used, "?"))
        return res

    def fit_forecast_se(self, y, pred_start: int, n_pred: int, want_stats: bool = False):
        """``fit_forecast`` with prediction standard errors (``mmf_fit_forecast_se_f32``): ``y`` is a float32 CUDA
        tensor.  Returns ``{"pred", "se", "sigma", "dof", "status"}`` (torch tensors on y's device): ``sigma[i]`` the
        residual scale sqrt(RSS / dof), ``se[i, j] = sigma[i] * sqrt(1 + h)`` the standard error of a new observation
        at design row ``pred_start + j`` (NaN where dof <= 0).  ``pred`` / ``status`` are bit-equal to ``fit_forecast``."""
        import torch
        if self.t_fit is None:
            raise RuntimeError("plan()/plan_calendar() must be called first")
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32) or t_have < self.t_fit:
            raise ValueError(f"y must be a float32 CUDA tensor with at least t_fit={self.t_fit} columns")
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)

        def table():            # 16-B row pitch: the tensor-core store paths
            return torch.empty((n, (n_pred + 3) & ~3), device=y.device, dtype=torch.float32)[:, :n_pred]

        out, se = table(), table()
        sigma = torch.empty(n, device=y.device, dtype=torch.float32)
        dof = torch.empty(n, device=y.device, dtype=torch.int32)
        status = torch.empty(n, device=y.device, dtype=torch.int32)
        st = N.MmfStats() if want_stats else None
        N.check(self._lib.mmf_fit_forecast_se_f32(self._h, yp, n, ld_y, int(pred_start), int(n_pred), out.data_ptr(),
                                                  out.stride(0), se.data_ptr(), se.stride(0), sigma.data_ptr(),
                                                  dof.data_ptr(), status.data_ptr(),
                                                  C.byref(st) if st is not None else None))
        res = {"pred": out, "se": se, "sigma": sigma, "dof": dof, "status": status}
        if st is not None:
            self.launches += st.kernel_launches
            res["stats"] = Stats(st.kernel_ms, st.total_ms, st.n_series, st.n_pending, st.h2d_bytes, st.d2h_bytes,
                                 st.kernel_launches, {N.KERNEL_WARP: "warp", N.KERNEL_TC: "tc"}.get(st.kernel_used, "?"))
        return res

    def fit_forecast_ar(self, y, ar_order: int, pred_start: int, n_pred: int, want_stats: bool = False,
                        want_se: bool = False):
        """Regression with AR(``ar_order``) errors (``mmf_fit_forecast_ar_f32``, DESIGN.md section 2 item 9): the plain
        fit, then Yule-Walker AR coefficients of each series' residuals.  ``y`` is a float32 CUDA tensor.  Returns
        ``{"pred", "phi", "order", "sigma", "status"}`` (torch tensors on y's device): ``pred[i, j]`` the one-step-ahead
        prediction (in sample) or dynamic forecast from t_fit (beyond it) of design row ``pred_start + j``,
        ``phi[i, :MMF_AR_MAX]`` the coefficients (zero beyond ``order[i]``, the order the series supports), ``sigma[i]``
        the innovation standard deviation.  ``status`` is bit-equal to ``fit_forecast``'s."""
        import torch
        if self.t_fit is None:
            raise RuntimeError("plan()/plan_calendar() must be called first")
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32) or t_have < self.t_fit:
            raise ValueError(f"y must be a float32 CUDA tensor with at least t_fit={self.t_fit} columns")
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        out = torch.empty((n, n_pred), device=y.device, dtype=torch.float32)
        phi = torch.empty((n, N.AR_MAX), device=y.device, dtype=torch.float32)
        order = torch.empty(n, device=y.device, dtype=torch.int32)
        sigma = torch.empty(n, device=y.device, dtype=torch.float32)
        status = torch.empty(n, device=y.device, dtype=torch.int32)
        st = N.MmfStats() if want_stats else None
        N.check(self._lib.mmf_fit_forecast_ar_f32(self._h, yp, n, ld_y, int(ar_order), int(pred_start), int(n_pred),
                                                  out.data_ptr(), out.stride(0), phi.data_ptr(), order.data_ptr(),
                                                  sigma.data_ptr(), status.data_ptr(),
                                                  C.byref(st) if st is not None else None))
        res = {"pred": out, "phi": phi, "order": order, "sigma": sigma, "status": status}
        if want_se:
            self._add_se(res, y, self.t_fit, pred_start, n_pred, 0)
        if st is not None:
            self.launches += st.kernel_launches
            res["stats"] = Stats(st.kernel_ms, st.total_ms, st.n_series, st.n_pending, st.h2d_bytes, st.d2h_bytes,
                                 st.kernel_launches, {N.KERNEL_WARP: "warp", N.KERNEL_TC: "tc"}.get(st.kernel_used, "?"))
        return res

    def plan_arima(self, X: np.ndarray, t_fit: int, max_diff: int = 2) -> None:
        """Plan the differenced designs ``D_d = Delta^d X``, d = 1 .. ``max_diff``, of ``fit_forecast_arima``
        (``mmf_plan_arima``, DESIGN.md section 2 item 11): a plan of its own beside the one ``plan`` makes."""
        X = np.ascontiguousarray(X, dtype=np.float64)
        if X.ndim != 2:
            raise ValueError("X must be 2-D")
        N.check(self._lib.mmf_plan_arima(self._h, X.ctypes.data, X.shape[0], X.shape[1], int(t_fit), int(max_diff)))
        self._arima = (int(t_fit), int(X.shape[0]), int(max_diff))

    def fit_forecast_arima(self, y, ar_order: int, diff_order: int, pred_start: int, n_pred: int,
                           want_stats: bool = False, want_se: bool = False):
        """Regression with ARIMA(``ar_order``, ``diff_order``, 0) errors (``mmf_fit_forecast_arima_f32``, DESIGN.md
        section 2 item 11): ``fit_forecast_ar`` on the differenced series and design, integrated back to levels.
        ``y`` is a float32 CUDA tensor of levels.  Returns ``{"pred", "phi", "order", "sigma", "status"}`` (torch tensors
        on y's device): ``pred[i, j]`` the level prediction of design row ``pred_start + j`` (one step ahead in sample,
        the integrated dynamic forecast from t_fit beyond it, NaN for the first ``diff_order`` rows), ``phi`` / ``order``
        / ``sigma`` / ``status`` those of the AR part on the differenced series."""
        import torch
        if getattr(self, "_arima", None) is None:
            raise RuntimeError("plan_arima() (or plan_calendar(..., max_diff=d)) must be called first")
        t_fit = self._arima[0]
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32) or t_have < t_fit:
            raise ValueError(f"y must be a float32 CUDA tensor with at least t_fit={t_fit} columns")
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        out = torch.empty((n, n_pred), device=y.device, dtype=torch.float32)
        phi = torch.empty((n, N.AR_MAX), device=y.device, dtype=torch.float32)
        order = torch.empty(n, device=y.device, dtype=torch.int32)
        sigma = torch.empty(n, device=y.device, dtype=torch.float32)
        status = torch.empty(n, device=y.device, dtype=torch.int32)
        st = N.MmfStats() if want_stats else None
        N.check(self._lib.mmf_fit_forecast_arima_f32(self._h, yp, n, ld_y, int(ar_order), int(diff_order),
                                                     int(pred_start), int(n_pred), out.data_ptr(), out.stride(0),
                                                     phi.data_ptr(), order.data_ptr(), sigma.data_ptr(),
                                                     status.data_ptr(), C.byref(st) if st is not None else None))
        res = {"pred": out, "phi": phi, "order": order, "sigma": sigma, "status": status}
        if want_se:
            self._add_se(res, y, t_fit, pred_start, n_pred, int(diff_order))
        if st is not None:
            self.launches += st.kernel_launches
            res["stats"] = Stats(st.kernel_ms, st.total_ms, st.n_series, st.n_pending, st.h2d_bytes, st.d2h_bytes,
                                 st.kernel_launches, {N.KERNEL_WARP: "warp", N.KERNEL_TC: "tc"}.get(st.kernel_used, "?"))
        return res

    def fit_forecast_arma(self, y, ar_order: int, ma_order: int, diff_order: int = 0, pred_start: int = 0,
                          n_pred: int | None = None, long_order: int = 0, want_stats: bool = False,
                          want_se: bool = False, estimator: str = "hr", max_iter: int = 0, joint_beta: bool = False,
                          predictor: str = "recursion"):
        """Regression with ARIMA(``ar_order``, ``diff_order``, ``ma_order``) errors (``mmf_fit_forecast_arma_f32``,
        DESIGN.md section 2 item 13): the plain fit (on the differenced series and design for ``diff_order`` >= 1),
        then Hannan-Rissanen on its residuals -- a long AR of order ``long_order`` (0: the default) gives innovation
        estimates, one least-squares solve gives (phi, theta).  Not SARIMAX's Kalman-filter MLE, and beta is not
        re-estimated.  A series whose estimate fails the gate (too short, collinear, non-stationary AR or non-invertible
        MA part) gets ``fit_forecast_arima`` / ``fit_forecast_ar`` with ``ar_order`` bit for bit, ``ma_order`` 0 and
        theta 0.  ``diff_order`` 0 needs ``plan``'s design, >= 1 ``plan_arima``'s.  ``y`` is a float32 CUDA tensor of
        levels; ``n_pred`` defaults to every design row from ``pred_start`` on.  Returns ``{"pred", "phi", "theta",
        "order", "ma_order", "sigma", "status"}`` (torch tensors on y's device): ``pred[i, j]`` the level prediction of
        design row ``pred_start + j`` (one step ahead in sample, the dynamic forecast from t_fit beyond it).

        ``estimator="css"`` (``mmf_fit_forecast_arma_css_f32``, DESIGN.md section 2 item 16) refines every gated
        series' (phi, theta) by Levenberg-Marquardt on the conditional sum of squares S of the recursion above, started
        from the Hannan-Rissanen estimate, for at most ``max_iter`` passes (0: 20, at most 64).  A series that accepts no
        step keeps the HR outputs bit for bit; ``sigma`` is sqrt(S / |C|) for every gated series.  The result adds
        ``css_start`` (S at the HR estimate), ``css`` (S shipped), ``css_stop`` (1 converged, 2 stalled, 3 budget, 0 not
        refined) and ``iters`` (passes run).

        ``joint_beta=True`` with ``estimator="css"`` (``mmf_fit_forecast_arma_joint_f32``, DESIGN.md section 2 item 17)
        estimates the regression coefficients jointly with (phi, theta): the whitened coefficients of every gated series'
        used design columns join the Levenberg-Marquardt parameter vector, started from the plain fit's (regression with
        ARIMA errors, R's ``arima(xreg=, method="CSS")``).  The result adds ``beta`` [n, 16], the coefficients of the raw
        design columns the series ships (of the differenced design for ``diff_order`` >= 1; NaN for empty series).  With
        ``want_se=True`` the standard errors take the joint (phi, theta, sigma); beta's estimation uncertainty is not
        included.

        ``estimator="ml"`` (``mmf_fit_forecast_arma_ml_f32``, DESIGN.md section 2 item 19) runs ``estimator="css"``
        and then refines every gated series' (phi, theta) on the exact Gaussian likelihood of its residuals: a Kalman
        filter from the stationary start (missing rows predicted, not filled), the same Levenberg-Marquardt and
        ``max_iter`` (R's ``arima(method="CSS-ML")`` on the differenced series).  A series that accepts no step keeps the
        CSS outputs bit for bit; ``sigma`` is the ML estimate for every gated series.  The result adds ``loglik_start``
        (the exact log-likelihood at the CSS estimate), ``loglik`` (at the shipped one), ``ml_stop`` (the CSS codes) and
        ``iters`` (ML passes run).  ``want_se=True`` takes the ML (phi, theta, sigma).  Not with ``joint_beta=True``.

        ``predictor="kalman"`` with ``estimator="ml"`` (``mmf_fit_forecast_arma_ml_kf_f32``, DESIGN.md section 2 item
        20) predicts every gated series whose stationary start solves at the shipped (phi, theta) with the Kalman filter
        of the exact likelihood, as SARIMAX's ``predict()`` / ``get_forecast()`` do: one step ahead in sample from the
        observed rows before each row, the dynamic forecast beyond t_fit.  Every other output, and every row the filter
        does not cover, is ``estimator="ml"``'s bit for bit.  ``want_se=True`` takes the call's own standard errors
        (the variance of this predictor's error, gaps included).  The default ``predictor="recursion"`` is the
        library's recursion."""
        import torch
        if estimator not in ("hr", "css", "ml"):
            raise ValueError(f"estimator must be 'hr' or 'css' (or 'ml' for the exact likelihood), got {estimator!r}")
        if predictor not in ("recursion", "kalman"):
            raise ValueError(f"predictor must be 'recursion' or 'kalman', got {predictor!r}")
        kalman = predictor == "kalman"
        if kalman and estimator != "ml":
            raise ValueError(f"predictor='kalman' needs estimator='ml' (the filter of the exact-likelihood fit), "
                             f"got estimator={estimator!r}")
        ml = estimator == "ml"
        css = estimator == "css" or ml
        if not css and int(max_iter) != 0:
            raise ValueError("max_iter= is the pass budget of estimator='css'")
        if joint_beta and estimator != "css":
            raise ValueError(f"joint_beta=True needs estimator='css' (beta joins the conditional least-squares fit), "
                             f"got estimator={estimator!r}")
        if int(diff_order) >= 1:
            if getattr(self, "_arima", None) is None:
                raise RuntimeError("plan_arima() (or plan_calendar(..., max_diff=d)) must be called first")
            t_fit, n_rows = self._arima[0], self._arima[1]
        else:
            if self.t_fit is None:
                raise RuntimeError("plan()/plan_calendar() must be called first")
            t_fit, n_rows = self.t_fit, self.n_rows
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32) or t_have < t_fit:
            raise ValueError(f"y must be a float32 CUDA tensor with at least t_fit={t_fit} columns")
        if n_pred is None:
            n_pred = n_rows - int(pred_start)
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        dev = y.device
        out = torch.empty((n, n_pred), device=dev, dtype=torch.float32)
        phi = torch.empty((n, N.AR_MAX), device=dev, dtype=torch.float32)
        theta = torch.empty((n, N.MA_MAX), device=dev, dtype=torch.float32)
        order = torch.empty(n, device=dev, dtype=torch.int32)
        ma = torch.empty(n, device=dev, dtype=torch.int32)
        sigma = torch.empty(n, device=dev, dtype=torch.float32)
        status = torch.empty(n, device=dev, dtype=torch.int32)
        st = N.MmfStats() if want_stats else None
        if css:
            css_start = torch.empty(n, device=dev, dtype=torch.float32)
            css_end = torch.empty(n, device=dev, dtype=torch.float32)
            css_stop = torch.empty(n, device=dev, dtype=torch.int32)
            iters = torch.empty(n, device=dev, dtype=torch.int32)
            if kalman:
                se = torch.empty((n, n_pred), device=dev, dtype=torch.float32) if want_se else None
                N.check(self._lib.mmf_fit_forecast_arma_ml_kf_f32(
                    self._h, yp, n, ld_y, int(ar_order), int(diff_order), int(ma_order), int(long_order),
                    int(max_iter), int(pred_start), int(n_pred), out.data_ptr(), out.stride(0), phi.data_ptr(),
                    theta.data_ptr(), order.data_ptr(), ma.data_ptr(), sigma.data_ptr(), status.data_ptr(),
                    css_start.data_ptr(), css_end.data_ptr(), css_stop.data_ptr(), iters.data_ptr(),
                    se.data_ptr() if se is not None else None, se.stride(0) if se is not None else 0,
                    C.byref(st) if st is not None else None))
            elif ml:
                N.check(self._lib.mmf_fit_forecast_arma_ml_f32(
                    self._h, yp, n, ld_y, int(ar_order), int(diff_order), int(ma_order), int(long_order),
                    int(max_iter), int(pred_start), int(n_pred), out.data_ptr(), out.stride(0), phi.data_ptr(),
                    theta.data_ptr(), order.data_ptr(), ma.data_ptr(), sigma.data_ptr(), status.data_ptr(),
                    css_start.data_ptr(), css_end.data_ptr(), css_stop.data_ptr(), iters.data_ptr(),
                    C.byref(st) if st is not None else None))
            elif joint_beta:
                beta = torch.empty((n, N.MMF_P), device=dev, dtype=torch.float32)
                N.check(self._lib.mmf_fit_forecast_arma_joint_f32(
                    self._h, yp, n, ld_y, int(ar_order), int(diff_order), int(ma_order), int(long_order),
                    int(max_iter), int(pred_start), int(n_pred), out.data_ptr(), out.stride(0), beta.data_ptr(),
                    phi.data_ptr(), theta.data_ptr(), order.data_ptr(), ma.data_ptr(), sigma.data_ptr(),
                    status.data_ptr(), css_start.data_ptr(), css_end.data_ptr(), css_stop.data_ptr(), iters.data_ptr(),
                    C.byref(st) if st is not None else None))
            else:
                N.check(self._lib.mmf_fit_forecast_arma_css_f32(
                    self._h, yp, n, ld_y, int(ar_order), int(diff_order), int(ma_order), int(long_order),
                    int(max_iter), int(pred_start), int(n_pred), out.data_ptr(), out.stride(0), phi.data_ptr(),
                    theta.data_ptr(), order.data_ptr(), ma.data_ptr(), sigma.data_ptr(), status.data_ptr(),
                    css_start.data_ptr(), css_end.data_ptr(), css_stop.data_ptr(), iters.data_ptr(),
                    C.byref(st) if st is not None else None))
        else:
            N.check(self._lib.mmf_fit_forecast_arma_f32(self._h, yp, n, ld_y, int(ar_order), int(diff_order),
                                                        int(ma_order), int(long_order), int(pred_start), int(n_pred),
                                                        out.data_ptr(), out.stride(0), phi.data_ptr(), theta.data_ptr(),
                                                        order.data_ptr(), ma.data_ptr(), sigma.data_ptr(),
                                                        status.data_ptr(), C.byref(st) if st is not None else None))
        res = {"pred": out, "phi": phi, "theta": theta, "order": order, "ma_order": ma, "sigma": sigma,
               "status": status}
        if ml:
            res.update(loglik_start=css_start, loglik=css_end, ml_stop=css_stop, iters=iters)
        elif css:
            res.update(css_start=css_start, css=css_end, css_stop=css_stop, iters=iters)
            if joint_beta:
                res["beta"] = beta
        if want_se and kalman:
            res["se"] = se
        elif want_se:
            self._add_se(res, y, t_fit, pred_start, n_pred, int(diff_order))
        if st is not None:
            self.launches += st.kernel_launches
            res["stats"] = Stats(st.kernel_ms, st.total_ms, st.n_series, st.n_pending, st.h2d_bytes, st.d2h_bytes,
                                 st.kernel_launches, {N.KERNEL_WARP: "warp", N.KERNEL_TC: "tc"}.get(st.kernel_used, "?"))
        return res

    def fit_select_ar(self, y, n_hold: int, orders=(0, 1, 2, 3, 4), pred_start: int = 0, n_pred: int | None = None,
                      want_stats: bool = False, want_se: bool = False):
        """Regression with AR(p) errors, p chosen per series by hold-out MSE (``mmf_fit_select_ar_f32``, DESIGN.md
        section 2 item 10).  Candidate m of ``orders`` (ascending, distinct, 0 .. MMF_AR_MAX) is ``fit_forecast_ar``
        with ``ar_order = m`` (m = 0: the plain regression); it is scored by the MSE of its dynamic forecast from t_fit
        over the held-out design rows [t_fit, t_fit + n_hold) against y's columns there, and the first minimum wins.
        ``y`` is a float32 CUDA tensor with at least t_fit + n_hold columns.  ``n_pred`` defaults to every design row
        from ``pred_start`` on.  Returns ``{"pred", "choice", "mse", "cand_mse", "phi", "order", "sigma", "status"}``
        (torch tensors on y's device): ``pred`` the chosen candidate's predictions, ``choice[i]`` its order (-1 for empty
        series), ``mse[i]`` its hold-out MSE, ``cand_mse[i, j]`` that of ``orders[j]``, ``phi`` / ``order`` / ``sigma``
        as in ``fit_forecast_ar`` for the chosen order."""
        import torch
        if self.t_fit is None:
            raise RuntimeError("plan()/plan_calendar() must be called first")
        orders = [int(m) for m in orders]
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32) or t_have < self.t_fit + int(n_hold):
            raise ValueError(f"y must be a float32 CUDA tensor with at least t_fit + n_hold={self.t_fit + int(n_hold)} "
                             "columns")
        if n_pred is None:
            n_pred = self.n_rows - int(pred_start)
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        dev = y.device
        out = torch.empty((n, n_pred), device=dev, dtype=torch.float32)
        choice = torch.empty(n, device=dev, dtype=torch.int32)
        mse = torch.empty(n, device=dev, dtype=torch.float32)
        cand_mse = torch.empty((n, len(orders)), device=dev, dtype=torch.float32)
        phi = torch.empty((n, N.AR_MAX), device=dev, dtype=torch.float32)
        order = torch.empty(n, device=dev, dtype=torch.int32)
        sigma = torch.empty(n, device=dev, dtype=torch.float32)
        status = torch.empty(n, device=dev, dtype=torch.int32)
        cand = (C.c_int32 * max(len(orders), 1))(*orders)
        st = N.MmfStats() if want_stats else None
        N.check(self._lib.mmf_fit_select_ar_f32(self._h, yp, n, ld_y, int(n_hold), cand, len(orders), int(pred_start),
                                                int(n_pred), out.data_ptr(), out.stride(0), choice.data_ptr(),
                                                mse.data_ptr(), cand_mse.data_ptr(), phi.data_ptr(), order.data_ptr(),
                                                sigma.data_ptr(), status.data_ptr(),
                                                C.byref(st) if st is not None else None))
        res = {"pred": out, "choice": choice, "mse": mse, "cand_mse": cand_mse, "phi": phi, "order": order,
               "sigma": sigma, "status": status}
        if want_se:
            self._add_se(res, y, self.t_fit, pred_start, n_pred, 0)
        if st is not None:
            self.launches += st.kernel_launches
            res["stats"] = Stats(st.kernel_ms, st.total_ms, st.n_series, st.n_pending, st.h2d_bytes, st.d2h_bytes,
                                 st.kernel_launches, {N.KERNEL_WARP: "warp", N.KERNEL_TC: "tc"}.get(st.kernel_used, "?"))
        return res

    def fit_select_arima(self, y, n_hold: int, orders=(0, 1, 2, 3, 4), diffs=(0, 1, 2), pred_start: int = 0,
                         n_pred: int | None = None, want_stats: bool = False, want_se: bool = False):
        """Regression with ARIMA(p, d, 0) errors, (p, d) chosen per series by hold-out MSE on levels
        (``mmf_fit_select_arima_f32``, DESIGN.md section 2 item 12).  The candidates are every pair of ``orders``
        (ascending, distinct, 0 .. MMF_AR_MAX) and ``diffs`` (ascending, distinct, 0 .. MMF_DIFF_MAX), d-major: (p, 0)
        is ``fit_select_ar``'s candidate p, (p, d >= 1) is ``fit_forecast_arima(p, d)``.  Each is scored by the MSE of
        its dynamic level forecast from t_fit over the held-out rows [t_fit, t_fit + n_hold); the first minimum wins.
        A listed d = 0 needs ``plan``'s design, a listed d >= 1 ``plan_arima``'s of the same X (``plan_calendar(...,
        max_diff=)`` plans both).  ``y`` is a float32 CUDA tensor with at least t_fit + n_hold columns; ``n_pred``
        defaults to every design row from ``pred_start`` on.  Returns ``{"pred", "choice_p", "choice_d", "mse",
        "cand_mse", "phi", "order", "sigma", "status"}`` (torch tensors on y's device): ``pred`` the winner's
        predictions, ``choice_p[i]`` / ``choice_d[i]`` the winner (-1 / -1 when no candidate is eligible), ``mse[i]``
        its hold-out MSE, ``cand_mse[i, k, j]`` that of ``(orders[j], diffs[k])``, ``phi`` / ``order`` / ``sigma`` /
        ``status`` the winner's."""
        import torch
        orders = [int(m) for m in orders]
        diffs = [int(d) for d in diffs]
        if any(d >= 1 for d in diffs):
            if getattr(self, "_arima", None) is None:
                raise RuntimeError("plan_arima() (or plan_calendar(..., max_diff=d)) must be called first")
            t_fit, n_rows = self._arima[0], self._arima[1]
        else:
            if self.t_fit is None:
                raise RuntimeError("plan()/plan_calendar() must be called first")
            t_fit, n_rows = self.t_fit, self.n_rows
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32) or t_have < t_fit + int(n_hold):
            raise ValueError(f"y must be a float32 CUDA tensor with at least t_fit + n_hold={t_fit + int(n_hold)} "
                             "columns")
        if n_pred is None:
            n_pred = n_rows - int(pred_start)
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        dev = y.device
        out = torch.empty((n, n_pred), device=dev, dtype=torch.float32)
        choice_p = torch.empty(n, device=dev, dtype=torch.int32)
        choice_d = torch.empty(n, device=dev, dtype=torch.int32)
        mse = torch.empty(n, device=dev, dtype=torch.float32)
        cand_mse = torch.empty((n, len(diffs), len(orders)), device=dev, dtype=torch.float32)
        phi = torch.empty((n, N.AR_MAX), device=dev, dtype=torch.float32)
        order = torch.empty(n, device=dev, dtype=torch.int32)
        sigma = torch.empty(n, device=dev, dtype=torch.float32)
        status = torch.empty(n, device=dev, dtype=torch.int32)
        cand = (C.c_int32 * max(len(orders), 1))(*orders)
        dl = (C.c_int32 * max(len(diffs), 1))(*diffs)
        st = N.MmfStats() if want_stats else None
        N.check(self._lib.mmf_fit_select_arima_f32(self._h, yp, n, ld_y, int(n_hold), cand, len(orders), dl, len(diffs),
                                                   int(pred_start), int(n_pred), out.data_ptr(), out.stride(0),
                                                   choice_p.data_ptr(), choice_d.data_ptr(), mse.data_ptr(),
                                                   cand_mse.data_ptr(), phi.data_ptr(), order.data_ptr(),
                                                   sigma.data_ptr(), status.data_ptr(),
                                                   C.byref(st) if st is not None else None))
        res = {"pred": out, "choice_p": choice_p, "choice_d": choice_d, "mse": mse, "cand_mse": cand_mse, "phi": phi,
               "order": order, "sigma": sigma, "status": status}
        if want_se:
            self._add_se(res, y, t_fit, pred_start, n_pred, 0, diffs=choice_d)
        if st is not None:
            self.launches += st.kernel_launches
            res["stats"] = Stats(st.kernel_ms, st.total_ms, st.n_series, st.n_pending, st.h2d_bytes, st.d2h_bytes,
                                 st.kernel_launches, {N.KERNEL_WARP: "warp", N.KERNEL_TC: "tc"}.get(st.kernel_used, "?"))
        return res

    def fit_select_arma(self, y, n_hold: int, orders=(0, 1, 2, 3, 4), diffs=(0, 1, 2), mas=(0, 1, 2, 3, 4),
                        pred_start: int = 0, n_pred: int | None = None, long_order: int = 0, want_stats: bool = False,
                        want_se: bool = False, refit: str | None = None, joint_beta: bool = False, max_iter: int = 0,
                        predictor: str = "recursion"):
        """Regression with ARIMA(p, d, q) errors, (p, d, q) chosen per series by hold-out MSE on levels
        (``mmf_fit_select_arma_f32``, DESIGN.md section 2 item 14).  The candidates are every triple of ``orders``,
        ``diffs`` and ``mas`` (ascending, distinct, 0 .. MMF_MA_MAX, ``mas[0] == 0``), d, then q, then p ascending:
        (p, d, 0) is ``fit_select_arima``'s candidate (p, d), (p, d, q >= 1) is ``fit_forecast_arma(p, q, d,
        long_order=m_d)`` with one long order per d (``long_order``, or 0 for min(32, max(2 max(orders, mas),
        floor(ln(t_fit - d)^2)))).  At most 32 pairs (p, q >= 1).  Scores, eligibility and the first-minimum choice are
        ``fit_select_arima``'s; a q >= 1 candidate that fails the Hannan-Rissanen gate scores as (p, d, 0) and never
        wins.  Returns ``fit_select_arima``'s dict plus ``choice_q``, ``theta`` and ``ma_order``; ``cand_mse[i, k, l,
        j]`` is the score of ``(orders[j], diffs[k], mas[l])``.  With ``mas=(0,)`` the call is ``fit_select_arima``.

        ``refit="css"`` (``mmf_fit_select_arma_css_f32``, DESIGN.md section 2 item 18) refits every series' winner at its
        own (p, d, q), as the reference fits its final model on the tuned order: a winner with q >= 1 gets every output of
        ``fit_forecast_arma(p, q, d, long_order=m_d, estimator="css", max_iter=max_iter)`` bit for bit, a winner with
        q = 0 keeps the selection's.  The choice, ``mse`` and ``cand_mse`` stay the selection's (the refit does not choose
        again).  The result adds ``css_start``, ``css``, ``css_stop`` and ``iters`` (NaN, NaN, 0, 0 where nothing was
        refit).  ``joint_beta=True`` (``mmf_fit_select_arma_joint_f32``) refits the q >= 1 winners with beta estimated
        jointly (``fit_forecast_arma(..., joint_beta=True)``) and adds ``beta`` [n, 16]: the joint call's for those, W
        gamma of the winner's plain fit for q = 0 winners, NaN where no candidate is eligible.  With ``want_se=True`` the
        standard errors take the refit's (phi, theta, sigma).

        ``refit="ml"`` (``mmf_fit_select_arma_ml_f32``, DESIGN.md section 2 item 21) refines that CSS refit by exact
        likelihood: a winner with q >= 1 gets every output of ``fit_forecast_arma(p, q, d, long_order=m_d,
        estimator="ml", max_iter=max_iter)`` bit for bit, and the result adds ``loglik_start``, ``loglik``, ``ml_stop``
        and ``iters`` (NaN, NaN, 0, 0 where nothing was refit) in place of the CSS columns.  ``predictor="kalman"``
        with it (``mmf_fit_select_arma_ml_kf_f32``) predicts those winners with the likelihood's Kalman filter, as
        ``fit_forecast_arma(..., estimator="ml", predictor="kalman")`` does, and ``want_se=True`` then returns the
        call's own standard errors.  ``joint_beta=True`` is not offered with ``refit="ml"``."""
        import torch
        if refit not in (None, "css", "ml"):
            raise ValueError(f"refit must be None or 'css' (or 'ml' for the exact likelihood), got {refit!r}")
        if refit is None and int(max_iter) != 0:
            raise ValueError("max_iter= is the pass budget of refit='css' (or 'ml')")
        if joint_beta and refit is None:
            raise ValueError("joint_beta=True needs refit='css' (beta joins the conditional least-squares refit)")
        if joint_beta and refit == "ml":
            raise ValueError("joint_beta=True needs refit='css' (beta joins the conditional least-squares refit; joint "
                             "beta by the exact likelihood is not offered), got refit='ml'")
        if predictor not in ("recursion", "kalman"):
            raise ValueError(f"predictor must be 'recursion' or 'kalman', got {predictor!r}")
        kalman = predictor == "kalman"
        if kalman and refit != "ml":
            raise ValueError(f"predictor='kalman' needs estimator='ml' (or refit='ml' for a selection: the filter of "
                             f"the exact-likelihood fit), got refit={refit!r}")
        orders = [int(m) for m in orders]
        diffs = [int(d) for d in diffs]
        mas = [int(q) for q in mas]
        if any(d >= 1 for d in diffs):
            if getattr(self, "_arima", None) is None:
                raise RuntimeError("plan_arima() (or plan_calendar(..., max_diff=d)) must be called first")
            t_fit, n_rows = self._arima[0], self._arima[1]
        else:
            if self.t_fit is None:
                raise RuntimeError("plan()/plan_calendar() must be called first")
            t_fit, n_rows = self.t_fit, self.n_rows
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32) or t_have < t_fit + int(n_hold):
            raise ValueError(f"y must be a float32 CUDA tensor with at least t_fit + n_hold={t_fit + int(n_hold)} "
                             "columns")
        if n_pred is None:
            n_pred = n_rows - int(pred_start)
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        dev = y.device
        out = torch.empty((n, n_pred), device=dev, dtype=torch.float32)
        choice_p = torch.empty(n, device=dev, dtype=torch.int32)
        choice_d = torch.empty(n, device=dev, dtype=torch.int32)
        choice_q = torch.empty(n, device=dev, dtype=torch.int32)
        mse = torch.empty(n, device=dev, dtype=torch.float32)
        cand_mse = torch.empty((n, len(diffs), len(mas), len(orders)), device=dev, dtype=torch.float32)
        phi = torch.empty((n, N.AR_MAX), device=dev, dtype=torch.float32)
        theta = torch.empty((n, N.MA_MAX), device=dev, dtype=torch.float32)
        order = torch.empty(n, device=dev, dtype=torch.int32)
        ma_order = torch.empty(n, device=dev, dtype=torch.int32)
        sigma = torch.empty(n, device=dev, dtype=torch.float32)
        status = torch.empty(n, device=dev, dtype=torch.int32)
        cand = (C.c_int32 * max(len(orders), 1))(*orders)
        dl = (C.c_int32 * max(len(diffs), 1))(*diffs)
        ql = (C.c_int32 * max(len(mas), 1))(*mas)
        st = N.MmfStats() if want_stats else None
        res = {"pred": out, "choice_p": choice_p, "choice_d": choice_d, "choice_q": choice_q, "mse": mse,
               "cand_mse": cand_mse, "phi": phi, "theta": theta, "order": order, "ma_order": ma_order, "sigma": sigma,
               "status": status}
        head = (self._h, yp, n, ld_y, int(n_hold), cand, len(orders), dl, len(diffs), ql, len(mas), int(long_order))
        tail = (choice_p.data_ptr(), choice_d.data_ptr(), choice_q.data_ptr(), mse.data_ptr(), cand_mse.data_ptr(),
                phi.data_ptr(), theta.data_ptr(), order.data_ptr(), ma_order.data_ptr(), sigma.data_ptr(),
                status.data_ptr())
        if refit is None:
            N.check(self._lib.mmf_fit_select_arma_f32(*head, int(pred_start), int(n_pred), out.data_ptr(), out.stride(0),
                                                      *tail, C.byref(st) if st is not None else None))
        elif refit == "ml":
            res.update(loglik_start=torch.empty(n, device=dev, dtype=torch.float32),
                       loglik=torch.empty(n, device=dev, dtype=torch.float32),
                       ml_stop=torch.empty(n, device=dev, dtype=torch.int32),
                       iters=torch.empty(n, device=dev, dtype=torch.int32))
            ml_out = (res["loglik_start"].data_ptr(), res["loglik"].data_ptr(), res["ml_stop"].data_ptr(),
                      res["iters"].data_ptr())
            sp = C.byref(st) if st is not None else None
            if kalman:
                se = torch.empty((n, n_pred), device=dev, dtype=torch.float32) if want_se else None
                N.check(self._lib.mmf_fit_select_arma_ml_kf_f32(*head, int(max_iter), int(pred_start), int(n_pred),
                                                                out.data_ptr(), out.stride(0), *tail, *ml_out,
                                                                se.data_ptr() if se is not None else None,
                                                                se.stride(0) if se is not None else 0, sp))
                if se is not None:
                    res["se"] = se
            else:
                N.check(self._lib.mmf_fit_select_arma_ml_f32(*head, int(max_iter), int(pred_start), int(n_pred),
                                                             out.data_ptr(), out.stride(0), *tail, *ml_out, sp))
        else:
            res.update(css_start=torch.empty(n, device=dev, dtype=torch.float32),
                       css=torch.empty(n, device=dev, dtype=torch.float32),
                       css_stop=torch.empty(n, device=dev, dtype=torch.int32),
                       iters=torch.empty(n, device=dev, dtype=torch.int32))
            css_out = (res["css_start"].data_ptr(), res["css"].data_ptr(), res["css_stop"].data_ptr(),
                       res["iters"].data_ptr(), C.byref(st) if st is not None else None)
            if joint_beta:
                res["beta"] = torch.empty((n, N.MMF_P), device=dev, dtype=torch.float32)
                N.check(self._lib.mmf_fit_select_arma_joint_f32(*head, int(max_iter), int(pred_start), int(n_pred),
                                                                out.data_ptr(), out.stride(0), res["beta"].data_ptr(),
                                                                *tail, *css_out))
            else:
                N.check(self._lib.mmf_fit_select_arma_css_f32(*head, int(max_iter), int(pred_start), int(n_pred),
                                                              out.data_ptr(), out.stride(0), *tail, *css_out))
        if want_se and "se" not in res:
            self._add_se(res, y, t_fit, pred_start, n_pred, 0, diffs=choice_d)
        if st is not None:
            self.launches += st.kernel_launches
            res["stats"] = Stats(st.kernel_ms, st.total_ms, st.n_series, st.n_pending, st.h2d_bytes, st.d2h_bytes,
                                 st.kernel_launches, {N.KERNEL_WARP: "warp", N.KERNEL_TC: "tc"}.get(st.kernel_used, "?"))
        return res

    def _add_se(self, res, y, t_fit: int, pred_start: int, n_pred: int, diff_order: int, diffs=None) -> None:
        """``want_se=True`` of the ARIMA-family calls: ``res["se"]`` [n, n_pred] float32, the standard error of every
        prediction in ``res["pred"]`` (``mmf_arima_se_f32``, DESIGN.md section 2 item 15), from the call's own phi,
        theta, orders, sigma and d (``diffs``: the per-series d of a selection), enqueued on the same stream."""
        import torch
        yp, n, _, ld_y = _describe(y, "y")
        se = torch.empty((n, n_pred), device=y.device, dtype=torch.float32)
        theta, ma = res.get("theta"), res.get("ma_order")
        N.check(self._lib.mmf_arima_se_f32(self._h, yp, n, ld_y, int(t_fit), int(diff_order),
                                           diffs.data_ptr() if diffs is not None else None, res["phi"].data_ptr(),
                                           res["order"].data_ptr(), theta.data_ptr() if theta is not None else None,
                                           ma.data_ptr() if ma is not None else None, res["sigma"].data_ptr(),
                                           int(pred_start), int(n_pred), se.data_ptr(), se.stride(0), None))
        res["se"] = se

    def capture(self, y, pred_start: int, n_pred: int, out=None, status=None):
        """Record one device-resident ``fit_forecast`` call as a CUDA graph.  Small batches are launch-bound (three
        kernel launches plus the Python/ctypes hop cost more than the kernels themselves): ``graph.replay()``
        re-runs the whole fit on whatever ``y`` holds at that time and overwrites ``out`` / ``status``.
        Returns ``(graph, out)``; ``graph`` is a :class:`CapturedFit`.  torch provides the graph object; every node
        in it is a libmmf kernel (plus one 8-B memset of the graph's own work counters).

        Lifetime: the graph holds raw pointers to this engine's scratch and planned design.  While the returned
        object is alive the engine is *pinned*: planning another calendar or a call that needs more scratch (a
        larger batch) raises ``MmfError`` (MMF_E_UNSUPPORTED) instead of freeing memory under the graph.
        ``graph.close()`` (or dropping it) unpins."""
        import torch
        if not (_is_torch(y) and y.is_cuda):
            raise ValueError("capture() needs a CUDA tensor")
        n = y.shape[0]
        if out is None:
            out = torch.empty((n, (n_pred + 3) & ~3), device=y.device, dtype=torch.float32)[:, :n_pred]
        if status is None:
            status = torch.empty(n, device=y.device, dtype=torch.int32)
        self.fit_forecast(y, pred_start, n_pred, out=out, status=status)    # sizes the library's scratch outside capture
        torch.cuda.synchronize(y.device)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self.fit_forecast(y, pred_start, n_pred, out=out, status=status)
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        return CapturedFit(self, graph, (y, out, status)), out

    def fit_select_forecast(self, y, n_hold: int, candidates=(1, 3, 9, 13, 16), pred_start: int = 0,
                            n_pred: int | None = None):
        """Per-series model selection on the device (reference: the hyperopt loop + refit, 02:435-488).
        ``y`` [n, >= t_fit + n_hold] CUDA tensor: rows [0,t_fit) are fit, the next ``n_hold`` score the nested
        candidate designs (first ``m`` whitened columns); the winner predicts rows [pred_start, +n_pred).
        Returns ``{"pred", "choice", "mse", "status"}`` (torch tensors)."""
        import torch
        if self.t_fit is None:
            raise RuntimeError("plan()/plan_calendar() must be called first")
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32):
            raise ValueError("y must be a float32 CUDA tensor")
        n_pred = self.n_rows - pred_start if n_pred is None else n_pred
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        out = torch.empty((n, (n_pred + 3) & ~3), dtype=torch.float32, device=y.device)[:, :n_pred]
        choice = torch.empty(n, dtype=torch.int32, device=y.device)
        mse = torch.empty(n, dtype=torch.float32, device=y.device)
        status = torch.empty(n, dtype=torch.int32, device=y.device)
        cand = (C.c_int32 * len(candidates))(*[int(c) for c in candidates])
        N.check(self._lib.mmf_fit_select_forecast_f32(self._h, yp, n, ld_y, int(n_hold), cand, len(candidates),
                                                      int(pred_start), int(n_pred), out.data_ptr(), out.stride(0),
                                                      choice.data_ptr(), mse.data_ptr(), status.data_ptr()))
        return {"pred": out, "choice": choice, "mse": mse, "status": status}

    def fit_forecast_bcast(self, y, pred_start: int, n_pred: int, out_ptrs, ld_out: int, multimem: int = 0,
                           status=None):
        """Fit the rows of the CUDA tensor ``y`` and store every forecast row to all ``out_ptrs``
        (this GPU's slice first, then the peers' slices; or one NVLS multicast pointer with
        ``multimem=True``) from inside the kernel.  Enqueue-only; see ``sharding.SymmetricTable``."""
        import torch
        if self.t_fit is None:
            raise RuntimeError("plan()/plan_calendar() must be called first")
        yp, n, t_have, ld_y = _describe(y, "y")
        if not (_is_torch(y) and y.is_cuda and y.dtype == torch.float32) or t_have < self.t_fit:
            raise ValueError("y must be a float32 CUDA tensor with at least t_fit columns")
        self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        ptrs = (C.c_uint64 * len(out_ptrs))(*[int(p) for p in out_ptrs])
        sp = _describe(status, "status")[0] if status is not None else None
        N.check(self._lib.mmf_fit_forecast_bcast_f32(self._h, yp, n, ld_y, int(pred_start), int(n_pred), ptrs,
                                                     len(out_ptrs), int(multimem), int(ld_out), None, sp))


class CapturedFit:
    """A captured fit (``ForecastEngine.capture``): ``replay()`` re-runs it; the engine's scratch and plan stay
    pinned (``mmf_pin_scratch``) until ``close()`` / garbage collection."""

    def __init__(self, engine: ForecastEngine, graph, keep):
        self._graph, self._keep = graph, keep        # the graph's buffers must outlive it
        lib, h = engine._lib, engine._h
        N.check(lib.mmf_pin_scratch(h, 1))
        self._unpin = weakref.finalize(self, CapturedFit._release, lib, h, engine._finalizer)

    @staticmethod
    def _release(lib, h, engine_finalizer):
        if engine_finalizer.alive:                   # the context may already be gone at interpreter shutdown
            lib.mmf_pin_scratch(h, -1)

    def replay(self) -> None:
        if self._graph is None:
            raise RuntimeError("this captured fit has been closed")
        self._graph.replay()

    def close(self) -> None:
        self._graph = None
        if self._unpin.alive:
            self._unpin()


def bind_to_gpu_numa(device: int = 0):
    """Pin the calling process to the CPU cores local to CUDA device ``device`` (NVML's ideal affinity), so that the
    page-locked staging buffers it allocates next live on the GPU's NUMA node: with one process per GPU on a
    two-socket host, half of the ranks otherwise stream their 55 GB/s of host reads across the socket link.
    Returns the new CPU set, or None when NVML is unavailable (nothing changed)."""
    import os
    try:
        import pynvml
        import torch
        pynvml.nvmlInit()
        pr = torch.cuda.get_device_properties(device)
        try:
            bus = f"{pr.pci_domain_id:08X}:{pr.pci_bus_id:02X}:{pr.pci_device_id:02X}.0"
            h = pynvml.nvmlDeviceGetHandleByPciBusId(bus.encode() if hasattr(bus, "encode") else bus)
        except Exception:
            h = pynvml.nvmlDeviceGetHandleByIndex(device)
        pynvml.nvmlDeviceSetCpuAffinity(h)
        return sorted(os.sched_getaffinity(0))
    except Exception:
        return None


_default_engine: ForecastEngine | None = None


def default_engine() -> ForecastEngine:
    global _default_engine
    if _default_engine is None:
        _default_engine = ForecastEngine()
    return _default_engine


def forecast_packed(y, start, freq: str = "D", horizon: int = 28, mode: str = "future",
                    design: str = "trend_season_exog", engine: ForecastEngine | None = None, **kw):
    """``y[N,T]`` on one shared calendar -> predictions ``[N, horizon]`` (future) or ``[N, T]``
    (holdout: fitted values for the train dates + forecast for the held-out dates)."""
    eng = engine or default_engine()
    t_len = y.shape[1]
    _, pred_start, n_pred = eng.plan_calendar(start, t_len, freq, horizon, mode, design)
    return eng.fit_forecast(y, pred_start, n_pred, **kw)
