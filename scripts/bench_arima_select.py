"""Cost and accuracy of (p, d) selection by hold-out MSE on levels (mmf_fit_select_arima_f32) against the calls it
composes, on two holdout shapes: C4 (1 M series x 1,095 days of synth.daily_store_item_demand_torch, horizon 28) and the
reference's weekly shape (1 M seeded series on its 157-week calendar, synth.reference_calendar, 117 fit weeks, horizon
40).  The arms alternate in one process, several rounds of `--steps` calls each after a warm-up, timed with CUDA events:
  plain         the plain fit (holdout window);
  arsel         AR order selection over (0..4) (mmf_fit_select_ar_f32);
  arima41/42    ARIMA(4, 1) and ARIMA(4, 2) in holdout mode;
  compose       what a caller runs without the new call: the AR selection over (0..4) with the holdout window, one
                future-mode ARIMA call per (p, d >= 1) candidate, the scores and the first minimum on the GPU (torch),
                and one holdout ARIMA call per winning (p, d >= 1), scattered into the table;
  select        the new call over (0..4) x (0, 1, 2).
It checks that compose's choices and predictions equal the new call's, except on rows whose two best scores lie within
1e-6 relative, and prints ms/step per arm (median), the chosen (p, d) histogram, the mean hold-out MSE of the arms, and
the card's name and power limit.  `--profile` adds a torch.profiler split by kernel of one call of `select` (a separate
run after the timed rounds).

    python scripts/bench_arima_select.py [--series 1000000] [--steps 3] [--rounds 3] [--profile] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmf  # noqa: E402

ORDERS, DIFFS = (0, 1, 2, 3, 4), (0, 1, 2)


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
    if name == "C4_holdout":
        y, start = mmf.synth.daily_store_item_demand_torch(n, 1095, seed=0)
        return y, start, 1095, "D", 28
    days = mmf.synth.reference_calendar()[0]
    t = len(days)
    y, _ = mmf.synth.daily_store_item_demand_torch(n, t, seed=1)
    return y, days[0], t, "W-MON", 40


def mse_rows(pred, act):
    """float64 MSE per row over the points where both are finite (NaN where none is)"""
    ok = torch.isfinite(pred) & torch.isfinite(act)
    e = torch.where(ok, act.double() - pred.double(), torch.zeros((), dtype=torch.float64, device=pred.device))
    cnt = ok.sum(dim=1)
    nan = torch.tensor(float("nan"), dtype=torch.float64, device=pred.device)
    return torch.where(cnt > 0, (e * e).sum(dim=1) / cnt.clamp(min=1), nan)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="torch.profiler table of one call of the new arm per shape")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    n = args.series
    eng = mmf.ForecastEngine()
    lib, hnd = eng._lib, eng._h
    check = mmf._native.check
    res = {"card": card(), "series": n, "steps": args.steps, "rounds": args.rounds, "shapes": {}}
    cand = (C.c_int32 * len(ORDERS))(*ORDERS)
    dl = (C.c_int32 * len(DIFFS))(*DIFFS)
    for shape in ("C4_holdout", "weekly157"):
        y, start, t, freq, h = shape_of(shape, n)
        _, ps, npred = eng.plan_calendar(start, t, freq, h, "holdout", max_diff=2)
        t_fit = t - h
        dev = "cuda"
        out = torch.empty((n, (npred + 3) & ~3), device=dev)[:, :npred]
        tmp = torch.empty((n, (npred + 3) & ~3), device=dev)[:, :npred]
        fut = {(p, d): torch.empty((n, (h + 3) & ~3), device=dev)[:, :h] for p in ORDERS for d in DIFFS if d}
        status = torch.empty(n, device=dev, dtype=torch.int32)
        arsel_cm = torch.empty((n, len(ORDERS)), device=dev)
        cp = torch.empty(n, device=dev, dtype=torch.int32)
        cd = torch.empty(n, device=dev, dtype=torch.int32)
        cm = torch.empty((n, len(DIFFS), len(ORDERS)), device=dev)
        mse = torch.empty(n, device=dev)
        eng.set_stream(torch.cuda.current_stream().cuda_stream)
        act = y[:, t_fit:t]
        comp = {}

        def plain():
            check(lib.mmf_fit_forecast_f32(hnd, y.data_ptr(), n, y.stride(0), ps, npred, out.data_ptr(), out.stride(0),
                                           None, status.data_ptr(), None))

        def arsel():
            check(lib.mmf_fit_select_ar_f32(hnd, y.data_ptr(), n, y.stride(0), h, cand, len(ORDERS), ps, npred,
                                            out.data_ptr(), out.stride(0), None, None, arsel_cm.data_ptr(), None, None,
                                            None, status.data_ptr(), None))

        def arima(p, d, o, pst, npr):
            check(lib.mmf_fit_forecast_arima_f32(hnd, y.data_ptr(), n, y.stride(0), p, d, pst, npr, o.data_ptr(),
                                                 o.stride(0), None, None, None, status.data_ptr(), None))

        def compose():
            arsel()
            for (p, d), o in fut.items():
                arima(p, d, o, t_fit, h)
            scores = torch.stack([arsel_cm.double()] + [torch.stack([mse_rows(fut[p, d], act) for p in ORDERS], dim=1)
                                                         for d in DIFFS if d], dim=1)          # [n, 3, 5], d-major
            flat = scores.reshape(n, -1)
            win = torch.where(torch.isnan(flat), torch.full_like(flat, float("inf")), flat).argmin(dim=1)
            win = torch.where(torch.isnan(flat).all(dim=1), torch.full_like(win, flat.shape[1] - 1), win)
            wd, wp = win // len(ORDERS), win % len(ORDERS)
            for k in range(1, len(DIFFS)):
                for j in range(len(ORDERS)):
                    rows = (wd == k) & (wp == j)
                    if bool(rows.any()):
                        arima(ORDERS[j], DIFFS[k], tmp, ps, npred)
                        out[rows] = tmp[rows]
            comp.update(scores=flat, wd=wd, wp=wp)

        def select():
            check(lib.mmf_fit_select_arima_f32(hnd, y.data_ptr(), n, y.stride(0), h, cand, len(ORDERS), dl, len(DIFFS),
                                               ps, npred, out.data_ptr(), out.stride(0), cp.data_ptr(), cd.data_ptr(),
                                               mse.data_ptr(), cm.data_ptr(), None, None, None, status.data_ptr(),
                                               None))

        arms = {"plain": plain, "arsel": arsel, "arima41": lambda: arima(4, 1, out, ps, npred),
                "arima42": lambda: arima(4, 2, out, ps, npred), "compose": compose, "select": select}
        times = {k: [] for k in arms}
        for fn in arms.values():
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
        entry = {"t": t, "t_fit": t_fit, "horizon": h, "ms_per_step": times, "median_ms": med,
                 "gate_select_faster_than_compose": med["select"] < med["compose"],
                 "target_ms_arsel_plus_arima41_arima42": med["arsel"] + med["arima41"] + med["arima42"]}
        # agreement of compose and select: choices and predictions, except on rows whose two best scores are within 1e-6
        compose()
        pred_c = out.clone()
        select()
        torch.cuda.synchronize()
        s = torch.where(torch.isnan(comp["scores"]), torch.full_like(comp["scores"], float("inf")), comp["scores"])
        two = s.sort(dim=1).values[:, :2]
        amb = torch.isfinite(two[:, 1]) & (two[:, 1] - two[:, 0] <= 1e-6 * two[:, 1].abs())
        same_choice = (cd.long() == torch.tensor(DIFFS, device=dev)[comp["wd"]]) & \
                      (cp.long() == torch.tensor(ORDERS, device=dev)[comp["wp"]])
        same_pred = ((pred_c == out) | (torch.isnan(pred_c) & torch.isnan(out))).all(dim=1)
        entry["agreement"] = {"rows": n, "ambiguous": int(amb.sum()),
                              "choice_differs_outside_ambiguous": int((~same_choice & ~amb).sum()),
                              "pred_differs_outside_ambiguous": int((~same_pred & ~amb).sum())}
        hist = {}
        for d in DIFFS:
            for p in ORDERS:
                hist[f"{p},{d}"] = int(((cp == p) & (cd == d)).sum())
        entry["choice_histogram"] = hist
        means = {"select_chosen": float(torch.nanmean(mse.double()).item())}
        for name in ("plain", "arsel", "arima41", "arima42"):
            arms[name]()
            means[name] = float(torch.nanmean(mse_rows(out[:, t_fit:t], act)).item())
        arima(1, 1, out, ps, npred)
        means["arima11"] = float(torch.nanmean(mse_rows(out[:, t_fit:t], act)).item())
        entry["mean_holdout_mse"] = means
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                select()
                torch.cuda.synchronize()
            split = {}
            for ev in prof.key_averages():
                tm = getattr(ev, "device_time_total", None)
                if tm is None:
                    tm = ev.cuda_time_total
                if tm > 0:
                    split[ev.key[:60]] = tm / 1e3
            entry["profile_select_ms"] = split
        res["shapes"][shape] = entry
        print(shape, json.dumps({k: entry[k] for k in entry if k != "ms_per_step"}), flush=True)
        del y, out, tmp, fut, status, arsel_cm, cp, cd, cm, mse, comp
        torch.cuda.empty_cache()
    print(json.dumps({k: v for k, v in res.items() if k != "shapes"}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
