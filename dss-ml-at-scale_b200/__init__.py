"""dss-ml-at-scale_b200 -- H100-native many-models fit + forecast engine.

A drop-in for ONE hot path of sebrahimi1988/dss-ml-at-scale: the
``groupBy("Product","SKU").applyInPandas(build_tune_and_score_model, ...)`` fan-out of
group_apply/02_Fine_Grained_Demand_Forecasting.py:417-528.  All groups' series are packed
into padded device buffers and fitted by hand-written sm_90a kernels in ``libmmf.so``
(C ABI: ``include/mmf.h``).  There is no CPU implementation in this package.

The directory name is not a Python identifier; import it as ``import mmf`` (alias
package at the repo root) or ``importlib.import_module("dss-ml-at-scale_b200")``.
"""
from . import design, synth, sharding, packer, sink         # noqa: F401
from ._native import LIB_PATH, MmfError, device_count, load as load_library   # noqa: F401
from .engine import (ForecastEngine, Stats, alloc_packed, bind_to_gpu_numa, default_engine, device_packed, forecast_packed,
                     pinned_empty, release_pinned_pool, to_integer_demand)  # noqa: F401
from .frames import (DEFAULT_KEYS, EXO_FIELDS, FORECAST_HORIZON, add_exo_variables, backtest_groups,  # noqa: F401
                     backtest_schema, enriched_schema, forecast_arrow_batches, forecast_groups, forecast_table,
                     pack_groups, spark_schemas, split_train_score_data, tuning_schema)

__version__ = "0.1.0"
