import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def reference_fixtures():
    import numpy as np
    return dict(np.load(os.path.join(GOLDEN, "reference_fixtures.npz")))


@pytest.fixture(scope="session")
def oracle_golden():
    import numpy as np
    return dict(np.load(os.path.join(GOLDEN, "oracle_golden.npz")))


def tolerance(y, leverage=1.0):
    """Stated fp32 tolerance of the CUDA path against the float64 oracle, well-conditioned rows:
        |yhat_gpu - yhat_ref| <= (5e-6 * max|y| + 1e-3) * max(1, leverage)   per element.
    ``leverage`` = the largest 2-norm of a requested prediction row in the whitened basis (fit rows have norm <= 1;
    for every BASELINE calendar it is < 1 and the factor is 1).  A prediction is c + a_pred . gamma, so a rounding
    error in gamma is amplified by |a_pred|: forecasting 28 days from a 32-day history with 13 live columns has
    leverage ~750 in float64 already (test_parity_full_series's 32/33-day cases).
    fp32 epsilon at the data's scale is 6e-8 * max|y| per rounding; the 3-term tf32 split of the tensor-core path
    (hi*A_hi + hi*A_lo + lo*A_hi) keeps the products at fp32 grade, and ~10^3 accumulated terms leave a few 1e-6
    relative.  A build with the lo-term MMAs compiled out FAILS it (tests/test_gpu_configs.py negative control).  Rows with an
    ill-conditioned mask scale it by 1/min(1, min_pivot_ratio/0.25) (see test_parity_masked_series)."""
    import numpy as np
    return (5e-6 * float(np.nanmax(np.abs(np.where(np.isfinite(y), y, 0.0)))) + 1e-3) * max(1.0, float(leverage))


def forecast_leverage(X, t_fit, pred_start, n_pred):
    """max_k |a_k|_2 over the requested prediction rows of the whitened design A = X W (oracle whitening)."""
    import numpy as np
    from oracle import mmf_oracle as O
    W, _ = O.whiten(np.asarray(X, dtype=np.float64)[:t_fit])
    A = np.asarray(X, dtype=np.float64) @ W
    return float(np.linalg.norm(A[pred_start:pred_start + n_pred], axis=1).max())


def record_err(name, err, tol, **extra):
    """Append one measured parity error to the scratch log mmf_test_out/parity_errors.jsonl in the system temporary
    directory (best effort)."""
    import json
    import tempfile
    d = os.path.join(tempfile.gettempdir(), "mmf_test_out")
    try:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "parity_errors.jsonl"), "a") as f:
            f.write(json.dumps({"test": name, "err": float(err), "tol": float(tol), **extra}) + "\n")
    except OSError:
        pass
