"""ctypes binding of ``libmmf.so`` (C ABI declared in ``include/mmf.h``).

There is deliberately no CPU implementation behind this module: if the shared
library is missing, or no H100 is visible, the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# MMF_LIB: load another build of the same ABI (tests use it for the negative-control build without the lo*A_hi
# tensor-core term); the default is the in-tree product library
LIB_PATH = os.environ.get("MMF_LIB") or os.path.join(_HERE, "libmmf.so")

MMF_P = 16
KERNEL_AUTO, KERNEL_WARP, KERNEL_TC = 0, 1, 2
STATUS_OK, STATUS_EMPTY, STATUS_RANKDEF, STATUS_PENDING = 0, 1, 2, -1
KERNELS = {"auto": KERNEL_AUTO, "warp": KERNEL_WARP, "tc": KERNEL_TC}
BT_MAX_ORIGINS, BT_NMETRIC = 8, 4                                          # MMF_BT_MAX_ORIGINS, MMF_BT_NMETRIC
AR_MAX, AR_KAPPA_MAX = 8, 0.999                                            # MMF_AR_MAX, MMF_AR_KAPPA_MAX
ARSEL_MAX_CAND = 9                                                         # MMF_ARSEL_MAX_CAND
DIFF_MAX = 2                                                               # MMF_DIFF_MAX
MA_MAX, HR_LONG_MAX, HR_PIVOT_TOL = 4, 32, 1e-5                            # MMF_MA_MAX, MMF_HR_LONG_MAX, MMF_HR_PIVOT_TOL
ARMASEL_MAX_PQ = 32                                                        # MMF_ARMASEL_MAX_PQ
CSS_LAMBDA0, CSS_LAMBDA_MAX, CSS_RTOL = 1e-3, 1e10, 1e-6                   # MMF_CSS_LAMBDA0, _LAMBDA_MAX, _RTOL
CSS_ITER_DEFAULT, CSS_ITER_MAX = 20, 64                                    # MMF_CSS_ITER_DEFAULT, MMF_CSS_ITER_MAX
DT_F32, DT_I16, DT_U16, DT_I32 = 0, 1, 2, 3
INT_DTYPES = {"int16": DT_I16, "uint16": DT_U16, "int32": DT_I32}          # series element types besides float32
INT_MISSING = {"int16": -32768, "uint16": 65535, "int32": -2147483648}     # the value that means "missing" in each

# every symbol include/mmf.h declares (tests/test_abi.py checks the library exports them all)
EXPORTS = (
    "mmf_version", "mmf_last_error", "mmf_device_count", "mmf_create", "mmf_destroy",
    "mmf_set_stream", "mmf_synchronize", "mmf_plan_design", "mmf_pin_scratch", "mmf_get_whitening",
    "mmf_fit_forecast_f32", "mmf_fit_forecast_int", "mmf_fit_forecast_se_f32", "mmf_fit_forecast_ar_f32",
    "mmf_fit_select_ar_f32", "mmf_plan_arima", "mmf_fit_forecast_arima_f32", "mmf_fit_select_arima_f32",
    "mmf_fit_forecast_arma_f32", "mmf_fit_forecast_arma_css_f32", "mmf_fit_forecast_arma_joint_f32",
    "mmf_fit_forecast_arma_ml_f32", "mmf_fit_forecast_arma_ml_kf_f32", "mmf_fit_select_arma_f32", "mmf_fit_select_arma_css_f32", "mmf_fit_select_arma_joint_f32",
    "mmf_fit_select_arma_ml_f32", "mmf_fit_select_arma_ml_kf_f32", "mmf_arima_se_f32",
    "mmf_plan_calendars", "mmf_fit_forecast_ragged_f32",
    "mmf_plan_backtest", "mmf_backtest_f32",
    "mmf_fit_forecast_bcast_f32", "mmf_fit_select_forecast_f32", "mmf_pack_hash_utf8", "mmf_pack_hash_i32",
    "mmf_pack_group_codes", "mmf_pack_verify_utf8", "mmf_pack_verify_i32", "mmf_pack_minmax", "mmf_pack_scatter_f32", "mmf_alloc_pinned", "mmf_free_pinned",
    "mmf_host_register", "mmf_host_unregister",
)


class MmfConfig(C.Structure):
    _fields_ = [
        ("device", C.c_int32),
        ("kernel", C.c_int32),
        ("assume_finite", C.c_int32),
        ("tc_variant", C.c_int32),
        ("chunk_series", C.c_int64),
        ("stream", C.c_void_p),
        ("host_narrow", C.c_int32),
        ("host_threads", C.c_int32),
        ("stream_solve", C.c_int32),
        ("reserved1", C.c_int32),
    ]


class MmfStats(C.Structure):
    _fields_ = [
        ("kernel_ms", C.c_float),
        ("total_ms", C.c_float),
        ("n_series", C.c_int64),
        ("n_pending", C.c_int64),
        ("h2d_bytes", C.c_int64),
        ("d2h_bytes", C.c_int64),
        ("kernel_launches", C.c_int32),
        ("kernel_used", C.c_int32),
    ]


class MmfError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"libmmf error {code}: {message}")
        self.code = code


_lib = None


def load() -> C.CDLL:
    """Load libmmf.so (built in-tree by ``__graft_entry__.build()`` / ``csrc/Makefile``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  This package has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    lib.mmf_version.restype = C.c_int
    lib.mmf_last_error.restype = C.c_char_p
    lib.mmf_device_count.argtypes = [C.POINTER(C.c_int32)]
    lib.mmf_create.argtypes = [C.POINTER(MmfConfig), C.POINTER(C.c_void_p)]
    lib.mmf_destroy.argtypes = [C.c_void_p]
    lib.mmf_set_stream.argtypes = [C.c_void_p, C.c_void_p]
    lib.mmf_synchronize.argtypes = [C.c_void_p]
    lib.mmf_plan_design.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.mmf_pin_scratch.argtypes = [C.c_void_p, C.c_int32]
    lib.mmf_get_whitening.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.mmf_fit_forecast_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32,
        C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(MmfStats),
    ]
    lib.mmf_fit_forecast_int.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_int32,
        C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(MmfStats),
    ]
    lib.mmf_fit_forecast_se_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32,
        C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(MmfStats),
    ]
    lib.mmf_fit_forecast_ar_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
        C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(MmfStats),
    ]
    lib.mmf_fit_select_ar_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32,
        C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
        C.POINTER(MmfStats),
    ]
    lib.mmf_plan_arima.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.mmf_fit_forecast_arima_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
        C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(MmfStats),
    ]
    lib.mmf_fit_forecast_arma_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
        C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
        C.POINTER(MmfStats),
    ]
    lib.mmf_fit_forecast_arma_css_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
        C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(MmfStats),
    ]
    lib.mmf_fit_forecast_arma_ml_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
        C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(MmfStats),
    ]
    lib.mmf_fit_forecast_arma_ml_kf_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
        C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(MmfStats),
    ]
    lib.mmf_fit_forecast_arma_joint_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
        C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(MmfStats),
    ]
    lib.mmf_fit_select_arima_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.POINTER(C.c_int32), C.c_int32,
        C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int64,
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
        C.POINTER(MmfStats),
    ]
    lib.mmf_fit_select_arma_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.POINTER(C.c_int32), C.c_int32,
        C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
        C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(MmfStats),
    ]
    # mmf_fit_select_arma_f32's arguments with max_iter after long_order and the four CSS outputs before stats; the
    # joint call adds out_beta after ld_out
    sel_head = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.POINTER(C.c_int32), C.c_int32,
                C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                C.c_int32, C.c_void_p, C.c_int64]
    sel_tail = [C.c_void_p] * 15 + [C.POINTER(MmfStats)]
    lib.mmf_fit_select_arma_css_f32.argtypes = sel_head + sel_tail
    lib.mmf_fit_select_arma_joint_f32.argtypes = sel_head + [C.c_void_p] + sel_tail
    # the ML refit: the four ML outputs in the CSS outputs' place; with the predictor out_se and ld_se before stats
    lib.mmf_fit_select_arma_ml_f32.argtypes = sel_head + sel_tail
    lib.mmf_fit_select_arma_ml_kf_f32.argtypes = sel_head + [C.c_void_p] * 15 + [C.c_void_p, C.c_int64, C.POINTER(MmfStats)]
    lib.mmf_arima_se_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
        C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.POINTER(MmfStats),
    ]
    lib.mmf_plan_calendars.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_int32, C.c_int32]
    lib.mmf_fit_forecast_ragged_f32.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                                C.c_int64, C.c_void_p, C.POINTER(MmfStats)]
    lib.mmf_plan_backtest.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_int32]
    lib.mmf_backtest_f32.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.POINTER(MmfStats)]
    lib.mmf_fit_forecast_bcast_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32,
        C.POINTER(C.c_uint64), C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p,
    ]
    lib.mmf_fit_select_forecast_f32.argtypes = [
        C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32,
        C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
    ]
    lib.mmf_pack_hash_utf8.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32]
    lib.mmf_pack_hash_i32.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32]
    lib.mmf_pack_group_codes.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
    lib.mmf_pack_verify_utf8.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.mmf_pack_verify_i32.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.mmf_pack_minmax.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]
    lib.mmf_pack_scatter_f32.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                         C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p]
    lib.mmf_alloc_pinned.argtypes = [C.c_size_t, C.POINTER(C.c_void_p)]
    lib.mmf_free_pinned.argtypes = [C.c_void_p]
    lib.mmf_host_register.argtypes = [C.c_void_p, C.c_size_t]
    lib.mmf_host_unregister.argtypes = [C.c_void_p]
    for name in EXPORTS:
        if name not in ("mmf_version", "mmf_last_error"):
            getattr(lib, name).restype = C.c_int
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load().mmf_last_error()
        raise MmfError(rc, msg.decode("utf-8", "replace") if msg else "")


def device_count() -> int:
    n = C.c_int32(0)
    check(load().mmf_device_count(C.byref(n)))
    return int(n.value)
