"""Seeded generator of retail demand shapes that the synthetic workloads of ``mmf.synth`` never produce: intermittent
(zero-inflated) counts, stock-outs as runs of true zeros (and the same rows with the run missing), products launched or
discontinued inside the window, returns (negative net demand), promotion spikes, degenerate rows the regression fits
exactly, and row levels from 0.1 to 60,000 interleaved row by row so that every 128-row tile mixes them.

``demand_batch(n, calendar, seed)`` returns float32 ``[n, t]`` (NaN = missing) and the kind of every row; the kind of
row i is ``KINDS[i % len(KINDS)]`` and its level ``LEVELS[i % len(LEVELS)]`` (the two cycle lengths are coprime, so
every kind meets every level).  Calendars: ``daily1095`` and ``daily365`` (daily, last date 2021-07-19, the synthetic
workloads' end) and ``weekly157`` (Mondays, same last date).
"""
from __future__ import annotations

import numpy as np

from oracle import mmf_oracle as O

END = np.datetime64("2021-07-19", "D")
CALENDARS = {"daily1095": (1095, "D"), "daily365": (365, "D"), "weekly157": (157, "W-MON")}

# level of row i: LEVELS[i % len(LEVELS)] (19 entries: coprime with len(KINDS))
LEVELS = (0.1, 60000.0, 3.0, 20000.0, 0.3, 5000.0, 12.0, 45000.0, 1.0, 800.0, 30000.0, 0.5, 150.0, 60000.0, 7.0,
          2500.0, 0.2, 40.0, 10000.0)

INTERMITTENT = ("counts", "counts_sparse", "stockout", "stockout_nan")
SCALED = ("regular", "launch_early", "launch_late", "discontinued", "launch_after_xmas", "returns", "signed", "promo",
          "promo_origin")
DEGENERATE = ("zeros", "const1", "const65534", "const_spike", "line", "level_weekly", "walk")
KINDS = INTERMITTENT + SCALED + DEGENERATE
# rows the regression fits to rounding level on every calendar (their residuals are float noise)
EXACT_FIT = ("zeros", "const1", "const65534", "line", "level_weekly", "walk")


def calendar(name: str, extra: int = 0):
    """(start date, t, freq, X [t + extra, P]) of one calendar, with the design fit on its t rows"""
    t, freq = CALENDARS[name]
    start = END - (t - 1) * np.timedelta64(O.FREQ_DAYS[freq], "D")
    X = O.design_matrix(O.calendar_grid(start, t + extra, freq), t)
    return start, t, freq, X


def _row_of(start, freq, date) -> int:
    """first grid row on or after ``date``"""
    step = O.FREQ_DAYS[freq]
    return int(-(-(np.datetime64(date, "D") - start).astype(np.int64) // step))


def landmarks(name: str, t_fit: int):
    """grid rows of the covid break (0 when it precedes the window) and of the first row after the last Christmas
    column of the fit window"""
    start, t, freq, X = calendar(name)
    covid = max(_row_of(start, freq, "2020-03-01"), 0)
    xmas = np.flatnonzero(X[:t_fit, O.COLUMN_NAMES.index("christmas")] > 0)
    return covid, int(xmas[-1]) + 1 if xmas.size else 0


def _regular(rng, t, level, weekday):
    """level x (weekly pattern) x (1 + 1 % noise), rounded to integers above level 50"""
    pat = rng.uniform(0.8, 1.2, 7)[weekday]
    y = level * pat * (1.0 + 0.01 * rng.standard_normal(t)) + 0.05 * level * np.sin(np.arange(t) / 40.0)
    return np.round(y) if level >= 50 else y


def _counts(rng, t, sparse):
    """zero-inflated integer counts: exactly round(q t) non-zero days, q 2.1-39 % (2.1-10 % when sparse), so 61-98 %
    zeros; each non-zero day 1 + Poisson, for a mean of 0.02-5"""
    q = rng.uniform(0.021, 0.1) if sparse else rng.uniform(0.021, 0.39)
    mean = rng.uniform(max(q, 0.02), min(5.0, 12.0 * q))
    k = min(max(int(np.ceil(0.02 * t)), int(round(q * t))), int(0.4 * t))           # 60-98 % zeros on any t
    row = np.zeros(t)
    row[rng.choice(t, k, replace=False)] = 1.0 + rng.poisson(mean / q - 1.0, k)
    return row


def demand_batch(n: int, name: str, seed: int, t_fit: int | None = None):
    """-> (y [n, t] float32, kinds [n] list of str, level [n]).  ``t_fit`` (default t) is the fit window the shapes
    are placed against (launch dates, spikes at t_fit - 1)."""
    start, t, freq, _ = calendar(name)
    t_fit = t if t_fit is None else t_fit
    rng = np.random.default_rng(seed)
    weekday = ((start - np.datetime64("1970-01-05", "D")).astype(np.int64) + O.FREQ_DAYS[freq] * np.arange(t)) % 7
    covid, after_xmas = landmarks(name, t_fit)
    y = np.empty((n, t))
    kinds = [KINDS[i % len(KINDS)] for i in range(n)]
    level = np.array([LEVELS[i % len(LEVELS)] for i in range(n)])
    s = np.arange(t, dtype=np.float64)
    runs = []
    for i, kind in enumerate(kinds):
        L = level[i]
        row = _regular(rng, t, L, weekday)
        if kind in ("counts", "counts_sparse"):
            row = _counts(rng, t, kind == "counts_sparse")
        elif kind == "stockout":
            runs = []
            for _ in range(rng.integers(1, 4)):
                run = int(rng.integers(7, 61)) if freq == "D" else int(rng.integers(2, 9))
                a = int(rng.integers(0, t_fit - run))
                row[a:a + run] = 0.0
                runs.append((a, run))
        elif kind == "stockout_nan":                              # the previous (stock-out) row, its runs missing
            row = y[i - 1].copy() if i > 0 and kinds[i - 1] == "stockout" else row
            level[i] = level[i - 1] if i > 0 and kinds[i - 1] == "stockout" else L
            for a, run in runs:
                row[a:a + run] = np.nan
        elif kind == "launch_early":                              # leading gap under half of the window
            row[:int(rng.integers(9, max(10, t_fit // 2)))] = np.nan
        elif kind == "launch_late":                               # leading gap over half of the window
            row[:int(rng.integers(t_fit // 2 + 1, t_fit - 39))] = np.nan
        elif kind == "discontinued":                              # last observation before the covid break
            stop = covid if covid > 40 else t_fit * 3 // 5
            row[int(rng.integers(stop // 2, stop)):] = np.nan
        elif kind == "launch_after_xmas":
            row[:min(after_xmas + int(rng.integers(0, 5)), t_fit - 40)] = np.nan
        elif kind == "returns":                                   # net demand with returns: some values negative
            ret = rng.random(t) < 0.15
            row = np.where(ret, -np.abs(row) * rng.uniform(0.05, 1.2, t), row)
        elif kind == "signed":                                    # mean ~ 0, changes sign
            row = L * rng.standard_normal(t)
            row = np.round(row) if L >= 50 else row
        elif kind in ("promo", "promo_origin"):
            days = rng.choice(np.arange(1, t_fit - 2), int(rng.integers(1, 4)), replace=False)
            if kind == "promo_origin":
                days = np.append(days, t_fit - 1)
            row[days] = np.round(L * rng.uniform(20, 100, len(days)))
        elif kind == "zeros":
            row = np.zeros(t)
        elif kind == "const1":
            row = np.ones(t)
        elif kind == "const65534":
            row = np.full(t, 65534.0)
        elif kind == "const_spike":
            row = np.full(t, np.round(max(L, 1.0)))
            row[int(rng.integers(0, t_fit))] *= 40.0
        elif kind == "line":                                      # exact integer line a + b s
            row = float(rng.integers(100, 2000)) + float(rng.integers(1, 5)) * s
        elif kind == "level_weekly":                              # exact level + weekly pattern (intercept + dow)
            row = float(rng.integers(100, 5000)) + rng.integers(-50, 50, 7).astype(np.float64)[weekday]
        elif kind == "walk":                                      # random walk with one constant integer step
            row = float(rng.integers(1000, 9000)) + float(rng.choice([-3, -2, -1, 1, 2, 3])) * s
        y[i] = row
    return y.astype(np.float32), kinds, level


def kind_rows(kinds, names):
    """boolean mask of the rows whose kind is in ``names``"""
    return np.array([k in names for k in kinds])
