"""Cost and accuracy of regression with AR(p) errors: mmf_fit_forecast_f32 against mmf_fit_forecast_ar_f32 (p = 1, 3) on
C4 (1 M series x 1,095 days of synth.daily_store_item_demand_torch, AR(1) noise), future mode (h = 28) and holdout mode
(every date).  The calls alternate in one process, several rounds of `--steps` calls each, timed with CUDA events; prints
ms/step per call and mode (median), the algorithmic bytes as a share of 3.35 TB/s, the card's name and power limit, and
the hold-out MSE of both models at horizons 1, 7 and 28 (the holdout-mode fit, scored on its last 28 dates).

    python scripts/bench_ar.py [--series 1000000] [--days 1095] [--steps 10] [--rounds 5] [--out FILE]
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--days", type=int, default=1095)
    ap.add_argument("--horizon", type=int, default=28)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    n, t, h = args.series, args.days, args.horizon
    y, start = mmf.synth.daily_store_item_demand_torch(n, t, seed=0)
    eng = mmf.ForecastEngine()
    lib, hnd = eng._lib, eng._h
    res = {"card": card(), "series": n, "days": t, "horizon": h, "steps": args.steps, "rounds": args.rounds, "modes": {}}
    for mode in ("future", "holdout"):
        _, ps, npred = eng.plan_calendar(start, t, "D", h, mode)
        t_fit = t if mode == "future" else t - h
        out = torch.empty((n, (npred + 3) & ~3), device="cuda")[:, :npred]
        status = torch.empty(n, device="cuda", dtype=torch.int32)
        eng.set_stream(torch.cuda.current_stream().cuda_stream)

        def plain():
            mmf._native.check(lib.mmf_fit_forecast_f32(hnd, y.data_ptr(), n, y.stride(0), ps, npred, out.data_ptr(),
                                                       out.stride(0), None, status.data_ptr(), None))

        def ar(p):
            def call():
                mmf._native.check(lib.mmf_fit_forecast_ar_f32(hnd, y.data_ptr(), n, y.stride(0), p, ps, npred,
                                                              out.data_ptr(), out.stride(0), None, None, None,
                                                              status.data_ptr(), None))
            return call

        arms = {"plain": plain, "ar1": ar(1), "ar3": ar(3)}
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
        # algorithmic bytes per series: plain reads y once and writes the table; AR reads the fit window once more in
        # holdout mode (pass B from the first date) and only its last p values in future mode
        b_plain = 4 * t_fit + 4 * npred
        b_ar = b_plain + (4 * t_fit if mode == "holdout" else 0)
        share = {k: (n * (b_plain if k == "plain" else b_ar) / (med[k] * 1e-3)) / HBM_BYTES_PER_S for k in med}
        entry = {"ms_per_step": times, "median_ms": med, "hbm_share": share}
        if mode == "holdout":            # hold-out MSE of both models on the last h dates
            act = y[:, t_fit:t]
            mse = {}
            for name, fn in (("plain", plain), ("ar1", arms["ar1"]), ("ar3", arms["ar3"])):
                fn()
                err = (out[:, t_fit:t] - act) ** 2
                mse[name] = {f"h{k}": float(torch.nanmean(err[:, :k]).item()) for k in (1, 7, 28)}
            entry["holdout_mse"] = mse
        res["modes"][mode] = entry
        print(mode, json.dumps({"median_ms": med, "hbm_share": share, **({"holdout_mse": entry["holdout_mse"]}
                                                                           if "holdout_mse" in entry else {})}), flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
