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
    """One library context: streams, staging buffers, the planned calendar design."""

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
        # series with gaps: True = solve them beside the streaming kernel (solve_stream_kernel; experimental), False = in
        # a pass of their own after it
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
                      design: str = "trend_season_exog"):
        """Build and plan the design for a bucket of series that start at ``start`` and have
        ``t_len`` grid rows.  Returns ``(dates_of_prediction_rows, pred_start, n_pred)``.
        The calendar planned last is remembered: the literal drop-in (one group per call, every group on the same
        calendar, 02:523-528) whitens and uploads its design once per worker, not once per group."""
        key = (str(np.datetime64(start, "D")), int(t_len), freq, int(horizon), mode, design)
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
        blocks, dates, n_rows, t_fit, p_start, n_pred = [], [], [], [], [], []
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
            n_rows.append(len(days)); t_fit.append(tf); p_start.append(ps); n_pred.append(npd)
        X = np.ascontiguousarray(np.concatenate(blocks, axis=0), dtype=np.float64)
        arr = [np.array(v, dtype=np.int32) for v in (n_rows, t_fit, p_start, n_pred)]
        N.check(self._lib.mmf_plan_calendars(self._h, X.ctypes.data, len(starts), arr[0].ctypes.data, arr[1].ctypes.data,
                                             arr[2].ctypes.data, arr[3].ctypes.data, X.shape[1],
                                             1 if D.design_has_constant(design) else 0))
        # (n_cal, columns of the output table, columns y must have)
        self._ragged = (len(starts), int(max(n_pred)), int(max(t_fit)), mode)
        return np.stack(dates) if mode == "future" else dates

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
