"""CPU: the float64 backtest oracle (tests/backtest_oracle.py) against independent routes -- lstsq on the raw design per
origin, hand-computed metrics -- and the change of basis the library takes (one moment in the longest window's basis,
T_k^T b_k = gamma_k) on the daily, weekly, exog-only and covid-straddling calendars."""
import numpy as np
import pytest

import mmf
from oracle import mmf_oracle as O
import backtest_oracle as B


def _calendar(name, n, seed=5):
    t_len, end, freq, design = {"daily": (1095, "2020-12-31", "D", "trend_season_exog"),
                                "weekly": (156, "2020-12-28", "W-MON", "trend_season_exog"),
                                "exog_only": (400, "2020-12-31", "D", "exog_only"),
                                "covid": (365, "2020-05-30", "D", "trend_season_exog")}[name]
    if freq == "D":
        y, start = mmf.synth.daily_store_item_demand(n, t_len, seed=seed, end=np.datetime64(end))
    else:
        yd, start = mmf.synth.daily_store_item_demand(n, 7 * t_len - 6, seed=seed, end=np.datetime64(end))
        y = np.ascontiguousarray(yd[:, ::7])
    days = mmf.design.calendar_grid(start, t_len, freq)
    return y.astype(np.float64), mmf.design.design_matrix(days, t_len - 28, design)


ORIGINS = {"daily": [983, 1011, 1039, 1067], "weekly": [60, 80, 100, 128], "exog_only": [100, 200, 300, 372],
           "covid": [200, 250, 273, 274, 290, 337]}


@pytest.mark.parametrize("cal", sorted(ORIGINS))
def test_oracle_matches_lstsq_on_the_raw_design(cal):
    y, X = _calendar(cal, 6)
    y[1, 10:40] = np.nan
    y[2, ::5] = np.nan
    h = 28
    pred, status = B.backtest_packed(y, X, ORIGINS[cal], h)
    for k, t in enumerate(ORIGINS[cal]):
        for i in range(y.shape[0]):
            obs = np.isfinite(y[i, :t])
            ref = O.lstsq_reference(y[i, :t][obs], X[:t][obs], X[t:t + h])
            np.testing.assert_allclose(pred[k, i], ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max())


@pytest.mark.parametrize("cal", sorted(ORIGINS))
def test_change_of_basis_identity(cal):
    """b_k (moment over [0, t_k) in the longest window's basis) mapped by T_k^T is origin k's gamma, in float64"""
    y, X = _calendar(cal, 4)
    origin, h = ORIGINS[cal], 28
    T, kappa, lev = B.change_of_basis(X, origin, h)
    W, kept = O.whiten(X[:origin[-1]])
    A = X @ W
    for k, t in enumerate(origin):
        Wk, kept_k = O.whiten(X[:t])
        Ak = X @ Wk
        b = y[:, :t] @ A[:t]                         # gap-free rows: gamma = b in each basis
        gamma = y[:, :t] @ Ak[:t]
        np.testing.assert_allclose(b @ T[k], gamma, rtol=1e-9, atol=1e-9 * np.abs(gamma).max())
        np.testing.assert_allclose(Ak[t:t + h] @ T[k].T @ b.T, (Ak[t:t + h] @ gamma.T), rtol=1e-9,
                                   atol=1e-9 * np.abs(gamma).max())
        assert kappa[k] >= 1.0 - 1e-12 and lev[k] > 0
    if cal == "covid":                               # covid (column 13) dropped before 2020-03-01, kept after
        kept_at = [bool(O.whiten(X[:t])[1][13]) for t in origin]
        assert not kept_at[0] and kept_at[-1]


def test_metrics_by_hand():
    nan = np.nan
    pred = np.array([[1.0, 2.0, 3.0, 4.0],
                     [1.0, 2.0, nan, 4.0],          # a non-finite forecast is not scored
                     [1.0, 1.0, 1.0, 1.0],
                     [1.0, 2.0, 3.0, 4.0]])
    act = np.array([[2.0, 2.0, 1.0, 4.0],
                    [0.0, nan, 1.0, 2.0],           # y = 0 counts for MSE / MAE / bias, not for MAPE
                    [nan, nan, nan, nan],           # nothing scored: all four NaN, count 0
                    [0.0, 0.0, 0.0, 0.0]])          # MAPE has nothing to average
    m, cnt = B.metrics(pred, act)
    assert cnt.tolist() == [4, 2, 0, 4]
    np.testing.assert_allclose(m[0], [(1 + 0 + 4 + 0) / 4, (1 + 0 + 2 + 0) / 4, (-1 + 0 + 2 + 0) / 4,
                                      (0.5 + 0 + 2 + 0) / 4])
    np.testing.assert_allclose(m[1], [(1 + 4) / 2, (1 + 2) / 2, (1 + 2) / 2, 1.0])
    assert np.isnan(m[2]).all()
    np.testing.assert_allclose(m[3, :3], [30 / 4, 10 / 4, 10 / 4])
    assert np.isnan(m[3, 3])


def test_origins_end_at_the_reference_split():
    """the last origin fits exactly the rows split_train_score_data keeps for training (02:372-380)"""
    import pandas as pd
    o = B.origins(1095, 28, 4)
    assert o.tolist() == [983, 1011, 1039, 1067]
    df = pd.DataFrame({"Date": pd.date_range("2018-01-01", periods=1095, freq="D"), "Demand": np.arange(1095.0)})
    train, score = O.split_train_score_data(df, 28)
    assert len(train) == o[-1] and len(score) == 28
    assert B.origins(100, 7, 3, step=10).tolist() == [73, 83, 93]
