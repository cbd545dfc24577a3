"""Cost and accuracy of regression with ARIMA(p, d, 0) errors (mmf_fit_forecast_arima_f32) against the plain call and the
AR(p) call with the same p, on three shapes: C4 (1 M series x 1,095 days of synth.daily_store_item_demand_torch) in
future mode (horizon 28) and in holdout mode, and the reference's weekly shape (1 M seeded series on its 157-week
calendar, synth.reference_calendar, 117 fit weeks, horizon 40) in holdout mode.  The arms alternate in one process,
several rounds of `--steps` calls each after a warm-up, timed with CUDA events; prints ms/step per arm (median), the
algorithmic bytes and GB/s of each arm, the card's name and power limit, and in holdout mode the hold-out MSE of each
arm over the last `horizon` dates.  `--profile` adds a torch.profiler split by kernel of one call per arm (a separate
run after the timed rounds).

    python scripts/bench_arima.py [--series 1000000] [--p 1] [--steps 10] [--rounds 5] [--profile] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmf  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def shape_of(name, n):
    """(y [n, t] CUDA view, first date, t, freq, horizon, mode)"""
    if name.startswith("C4"):
        y, start = mmf.synth.daily_store_item_demand_torch(n, 1095, seed=0)
        return y, start, 1095, "D", 28, "future" if name == "C4_future" else "holdout"
    days = mmf.synth.reference_calendar()[0]
    t = len(days)
    y, _ = mmf.synth.daily_store_item_demand_torch(n, t, seed=1)
    return y, days[0], t, "W-MON", 40, "holdout"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--p", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="torch.profiler table of one call per arm and shape")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    n, p = args.series, args.p
    eng = mmf.ForecastEngine()
    lib, hnd = eng._lib, eng._h
    check = mmf._native.check
    res = {"card": card(), "series": n, "p": p, "steps": args.steps, "rounds": args.rounds, "shapes": {}}
    for shape in ("C4_future", "C4_holdout", "weekly157"):
        y, start, t, freq, h, mode = shape_of(shape, n)
        _, ps, npred = eng.plan_calendar(start, t, freq, h, mode, max_diff=2)
        t_fit = t - h if mode == "holdout" else t
        out = torch.empty((n, (npred + 3) & ~3), device="cuda")[:, :npred]
        status = torch.empty(n, device="cuda", dtype=torch.int32)
        eng.set_stream(torch.cuda.current_stream().cuda_stream)

        def plain():
            check(lib.mmf_fit_forecast_f32(hnd, y.data_ptr(), n, y.stride(0), ps, npred, out.data_ptr(), out.stride(0),
                                           None, status.data_ptr(), None))

        def ar():
            check(lib.mmf_fit_forecast_ar_f32(hnd, y.data_ptr(), n, y.stride(0), p, ps, npred, out.data_ptr(),
                                              out.stride(0), None, None, None, status.data_ptr(), None))

        def arima(d):
            def call():
                check(lib.mmf_fit_forecast_arima_f32(hnd, y.data_ptr(), n, y.stride(0), p, d, ps, npred, out.data_ptr(),
                                                     out.stride(0), None, None, None, status.data_ptr(), None))
            return call

        arms = {"plain": plain, f"ar{p}": ar, f"arima{p}1": arima(1), f"arima{p}2": arima(2)}
        times = {k: [] for k in arms}
        for fn in arms.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for name, fn in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / args.steps)
        med = {k: float(np.median(v)) for k, v in times.items()}
        # algorithmic bytes per series.  plain: the fit window read, the table written.  AR(p): + pass A's read of the
        # fit window, + pass B's read of it in holdout mode (from the first date).  ARIMA(p, d): the differencing reads
        # y and writes z' (t_fit - d), the fit reads z', arima_kernel's pass A reads z' and in holdout mode pass B reads
        # z' and the levels y once more; the table written.
        win = 4 * npred
        b = {"plain": 4 * t_fit + win, f"ar{p}": 8 * t_fit + win + (4 * t_fit if mode == "holdout" else 0)}
        for d in (1, 2):
            tz = t_fit - d
            b[f"arima{p}{d}"] = 4 * t_fit + 3 * 4 * tz + win + ((4 * tz + 4 * t_fit) if mode == "holdout" else 0)
        gbs = {k: n * b[k] / (med[k] * 1e-3) / 1e9 for k in med}
        entry = {"t": t, "t_fit": t_fit, "horizon": h, "mode": mode, "ms_per_step": times, "median_ms": med,
                 "bytes_per_series": b, "GB_per_s": gbs}
        if mode == "holdout":
            act = y[:, t_fit:t]
            mse = {}
            for name, fn in arms.items():
                fn()
                err = (out[:, t_fit:t] - act) ** 2
                mse[name] = float(torch.nanmean(err).item())
            entry["holdout_mse"] = mse
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            entry["profile"] = {}
            for name, fn in arms.items():
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    fn()
                    torch.cuda.synchronize()
                split = {}
                for ev in prof.key_averages():
                    tm = getattr(ev, "device_time_total", None)
                    if tm is None:
                        tm = ev.cuda_time_total
                    if tm > 0:
                        split[ev.key[:60]] = tm / 1e3
                entry["profile"][name] = split
        res["shapes"][shape] = entry
        print(shape, json.dumps({k: entry[k] for k in entry if k not in ("ms_per_step",)}), flush=True)
        del y, out, status
        torch.cuda.empty_cache()
    print(json.dumps({k: v for k, v in res.items() if k != "shapes"}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
