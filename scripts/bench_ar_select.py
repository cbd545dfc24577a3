"""Cost and accuracy of AR order selection by hold-out MSE (mmf_fit_select_ar_f32) against the plain holdout call and the
fixed AR(4) holdout call, on two shapes: C4 (1 M series x 1,095 days of synth.daily_store_item_demand_torch, horizon 28)
and the reference's weekly shape (1 M seeded series on its 157-week calendar, synth.reference_calendar, horizon 40).
Holdout mode: every date is predicted, the last `horizon` dates are held out.  The arms alternate in one process,
several rounds of `--steps` calls each after a warm-up, timed with CUDA events; prints ms/step per arm (median), the
selection-to-AR(4) ratio next to the algorithmic bytes, the card's name and power limit, the histogram of chosen orders
and the hold-out MSE by arm.  The winner's hold-out MSE is biased low: it was chosen on that same window.

    python scripts/bench_ar_select.py [--series 1000000] [--steps 10] [--rounds 5] [--profile] [--out FILE]
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

HBM_BYTES_PER_S = 3.35e12                 # H100 SXM data sheet
ORDERS = (0, 1, 2, 3, 4)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def shape_of(name, n):
    """(y [n, t] CUDA view, first date, t, freq, horizon)"""
    if name == "C4":
        y, start = mmf.synth.daily_store_item_demand_torch(n, 1095, seed=0)
        return y, start, 1095, "D", 28
    days = mmf.synth.reference_calendar()[0]
    t = len(days)
    y, _ = mmf.synth.daily_store_item_demand_torch(n, t, seed=1)
    return y, days[0], t, "W-MON", 40


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="torch.profiler table of one selection call per shape")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    n = args.series
    eng = mmf.ForecastEngine()
    lib, hnd = eng._lib, eng._h
    res = {"card": card(), "series": n, "steps": args.steps, "rounds": args.rounds, "shapes": {}}
    for shape in ("C4", "weekly157"):
        y, start, t, freq, h = shape_of(shape, n)
        _, ps, npred = eng.plan_calendar(start, t, freq, h, "holdout")
        t_fit = t - h
        out = torch.empty((n, (npred + 3) & ~3), device="cuda")[:, :npred]
        status = torch.empty(n, device="cuda", dtype=torch.int32)
        choice = torch.empty(n, device="cuda", dtype=torch.int32)
        cand_mse = torch.empty((n, len(ORDERS)), device="cuda")
        eng.set_stream(torch.cuda.current_stream().cuda_stream)
        import ctypes
        cand = (ctypes.c_int32 * len(ORDERS))(*ORDERS)

        def plain():
            mmf._native.check(lib.mmf_fit_forecast_f32(hnd, y.data_ptr(), n, y.stride(0), ps, npred, out.data_ptr(),
                                                       out.stride(0), None, status.data_ptr(), None))

        def ar4():
            mmf._native.check(lib.mmf_fit_forecast_ar_f32(hnd, y.data_ptr(), n, y.stride(0), 4, ps, npred,
                                                          out.data_ptr(), out.stride(0), None, None, None,
                                                          status.data_ptr(), None))

        def select():
            mmf._native.check(lib.mmf_fit_select_ar_f32(hnd, y.data_ptr(), n, y.stride(0), h, cand, len(ORDERS), ps,
                                                        npred, out.data_ptr(), out.stride(0), choice.data_ptr(), None,
                                                        cand_mse.data_ptr(), None, None, None, status.data_ptr(),
                                                        None))

        arms = {"plain": plain, "ar4": ar4, "select": select}
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
        # algorithmic bytes per series: every arm reads the fit window and writes the table; AR(4) in holdout mode
        # reads the fit window once more (pass B from the first date); selection adds the held-out rows and its
        # choice / candidate-MSE outputs
        b_plain = 4 * t_fit + 4 * npred
        b_ar = b_plain + 4 * t_fit
        b_sel = b_ar + 4 * h + 4 + 4 * len(ORDERS)
        nbytes = {"plain": b_plain, "ar4": b_ar, "select": b_sel}
        share = {k: (n * nbytes[k] / (med[k] * 1e-3)) / HBM_BYTES_PER_S for k in med}
        entry = {"t": t, "horizon": h, "ms_per_step": times, "median_ms": med, "bytes_per_series": nbytes,
                 "hbm_share": share, "select_over_ar4": med["select"] / med["ar4"],
                 "bytes_select_over_ar4": b_sel / b_ar}
        act = y[:, t_fit:t]
        mse = {}
        for name, fn in arms.items():
            fn()
            err = (out[:, t_fit:t] - act) ** 2
            mse[name] = float(torch.nanmean(err).item())
        entry["holdout_mse"] = mse
        select()
        hist = torch.bincount(choice[choice >= 0].long(), minlength=max(ORDERS) + 1).cpu().tolist()
        entry["chosen_orders"] = {str(m): hist[m] for m in ORDERS}
        entry["holdout_mse_by_candidate"] = {str(m): float(torch.nanmean(cand_mse[:, j]).item())
                                             for j, m in enumerate(ORDERS)}
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                select()
                torch.cuda.synchronize()
            entry["profile"] = prof.key_averages().table(sort_by="cuda_time_total", row_limit=8)
            print(entry["profile"], flush=True)
        res["shapes"][shape] = entry
        print(shape, json.dumps({k: entry[k] for k in ("median_ms", "select_over_ar4", "bytes_select_over_ar4",
                                                        "hbm_share", "holdout_mse", "chosen_orders",
                                                        "holdout_mse_by_candidate")}), flush=True)
        del y, out, status, choice, cand_mse
        torch.cuda.empty_cache()
    print(json.dumps({k: v for k, v in res.items() if k != "shapes"}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
