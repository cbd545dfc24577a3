"""Cost and accuracy of regression with ARIMA(p, d, q) errors (mmf_fit_forecast_arma_f32, Hannan-Rissanen) against the
plain call, AR(1) and ARIMA(1, 1, 0), on three shapes: C4 (1 M series x 1,095 days of synth.daily_store_item_demand_torch) in
future mode (horizon 28) and in holdout mode, and the reference's weekly shape (1 M seeded series on its 157-week
calendar, synth.reference_calendar, 117 fit weeks, horizon 40) in holdout mode.  The arms alternate in one process,
several rounds of `--steps` calls each after a warm-up, timed with CUDA events; prints ms/step per arm (median), the
algorithmic bytes and GB/s of each arm, the card's name and power limit, the share of rows of each ARMA arm that fell
back to ARIMA(p, d, 0), and in holdout mode the hold-out MSE of each arm over the last `horizon` dates.  Arms: plain,
AR(1), ARIMA(1, 1, 0), ARMA(1, 0, 1), ARIMA(1, 1, 1), ARIMA(1, 2, 1).  `--profile` adds a torch.profiler split by kernel of one call per arm (a separate
run after the timed rounds).  `--split` attributes arma_kernel's time to its passes: it times the ARMA arms again with
the timing builds tests/_build/libmmf_arma_stop1.so (the kernel ends after pass A and step 1) and libmmf_arma_stop2.so
(after pass A2 and the solve), each in a process of its own, and reports the differences.  Those builds allocate
registers on their own, so the split is approximate.

    python scripts/bench_arma.py [--series 1000000] [--steps 10] [--rounds 5] [--profile] [--split] [--out FILE]
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


def split_passes(args):
    """median ms of the ARMA arms with the product library and the two timing builds; pass time = difference"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libs = {"full": None, "stop1": "libmmf_arma_stop1.so", "stop2": "libmmf_arma_stop2.so"}
    got = {}
    for name, lib in libs.items():
        env = dict(os.environ)
        env.pop("MMF_LIB", None)
        if lib:
            env["MMF_LIB"] = os.path.join(root, "tests", "_build", lib)
        cmd = [sys.executable, os.path.abspath(__file__), "--series", str(args.series), "--steps", str(args.steps),
               "--rounds", str(args.rounds), "--shapes", args.shapes, "--arms", "ar1,arima110,arma101,arima111"]
        out = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True).stdout
        got[name] = {ln.split(" ", 1)[0]: json.loads(ln.split(" ", 1)[1])["median_ms"] for ln in out.splitlines()
                     if ln.split(" ", 1)[0] in args.shapes.split(",")}
    res = {"card": card(), "series": args.series, "split": {}}
    for shape in args.shapes.split(","):
        f, a, b = got["full"][shape], got["stop1"][shape], got["stop2"][shape]
        fall = {"arma101": "ar1", "arima111": "arima110"}             # the call each ARMA arm runs before arma_kernel
        res["split"][shape] = {arm: {"call_ms": f[arm], "fallback_call_ms": f[fall[arm]],
                                     "passA_step1_ms": a[arm] - f[fall[arm]], "passA2_solve_ms": b[arm] - a[arm],
                                     "passB_ms": f[arm] - b[arm]}
                               for arm in ("arma101", "arima111")}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="torch.profiler table of one call per arm and shape")
    ap.add_argument("--split", action="store_true", help="time of arma_kernel per pass, from the timing builds")
    ap.add_argument("--shapes", default="C4_future,C4_holdout,weekly157")
    ap.add_argument("--arms", default=None, help="comma list of arms to time (default: all)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.split:
        split_passes(args)
        return
    n, p = args.series, 1
    eng = mmf.ForecastEngine()
    lib, hnd = eng._lib, eng._h
    check = mmf._native.check
    res = {"card": card(), "series": n, "p": p, "steps": args.steps, "rounds": args.rounds, "shapes": {}}
    for shape in args.shapes.split(","):
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

        ma_order = torch.empty(n, device="cuda", dtype=torch.int32)

        def arma(d):
            def call():
                check(lib.mmf_fit_forecast_arma_f32(hnd, y.data_ptr(), n, y.stride(0), p, d, 1, 0, ps, npred,
                                                    out.data_ptr(), out.stride(0), None, None, None,
                                                    ma_order.data_ptr(), None, status.data_ptr(), None))
            return call

        arms = {"plain": plain, "ar1": ar, "arima110": arima(1), "arma101": arma(0), "arima111": arma(1),
                "arima121": arma(2)}
        if args.arms:
            arms = {k: v for k, v in arms.items() if k in args.arms.split(",")}
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
        # algorithmic bytes per series.  plain: the fit window read, the table written.  AR(1): + pass A's read of the
        # fit window, + pass B's read of it in holdout mode.  ARIMA(1, 1, 0): the differencing reads y and writes z', the
        # fit and arima_kernel's pass A read z', in holdout mode pass B reads z' and y once more.  ARMA: the ARIMA(p, d, 0)
        # call it falls back to, then arma_kernel reads the modelled series three times (passes A, A2, B) and, for
        # d >= 1, the levels once, and writes the table again.
        win = 4 * npred
        b = {"plain": 4 * t_fit + win, "ar1": 8 * t_fit + win + (4 * t_fit if mode == "holdout" else 0)}
        tz = t_fit - 1
        b["arima110"] = 4 * t_fit + 3 * 4 * tz + win + ((4 * tz + 4 * t_fit) if mode == "holdout" else 0)
        b["arma101"] = b["ar1"] + 3 * 4 * t_fit + win
        b = {k: v for k, v in b.items() if k in arms} if args.arms else b
        for d in (1, 2):
            tz = t_fit - d
            b[f"arima1{d}1"] = (4 * t_fit + 3 * 4 * tz + win + ((4 * tz + 4 * t_fit) if mode == "holdout" else 0)
                                + 3 * 4 * tz + 4 * t_fit + win)
        gbs = {k: n * b[k] / (med[k] * 1e-3) / 1e9 for k in med}
        fell_back = {}
        for name in [a for a in ("arma101", "arima111", "arima121") if a in arms]:
            arms[name]()
            fell_back[name] = float((ma_order == 0).float().mean().item())
        entry = {"t": t, "t_fit": t_fit, "horizon": h, "mode": mode, "ms_per_step": times, "median_ms": med,
                 "bytes_per_series": b, "GB_per_s": gbs, "fell_back": fell_back}
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
        del y, out, status, ma_order
        torch.cuda.empty_cache()
    print(json.dumps({k: v for k, v in res.items() if k != "shapes"}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
