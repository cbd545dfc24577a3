"""Cost of the prediction standard errors: mmf_fit_forecast_f32 against mmf_fit_forecast_se_f32 on C4 (1 M series x
1,095 days, daily calendar, fully observed unless --gap-frac), future mode (h = 28) and holdout mode (every date).
The two calls alternate in one process, several rounds of `--steps` calls each, timed with CUDA events; prints
ms/step per call and mode, the SE/plain ratio, the algorithmic-byte ratio and the card's name and power limit.

    python scripts/bench_intervals.py [--series 1000000] [--days 1095] [--steps 10] [--rounds 5] [--gap-frac 0]
                                      [--out FILE]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--days", type=int, default=1095)
    ap.add_argument("--horizon", type=int, default=28)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--gap-frac", type=float, default=0.0, help="probability that a value (after the first 8) is missing")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    n, t, h = args.series, args.days, args.horizon
    g = torch.Generator(device="cuda").manual_seed(0)
    full = torch.empty((n, (t + 3) & ~3), device="cuda")
    y = full[:, :t]
    level = 20.0 + 480.0 * torch.rand((n, 1), device="cuda", generator=g)
    y.copy_(level + 0.2 * level * torch.randn((n, t), device="cuda", generator=g))
    if args.gap_frac > 0:          # 1e-3: about two thirds of the series have a gap or two
        gaps = torch.rand((n, t), device="cuda", generator=g) < args.gap_frac
        gaps[:, :8] = False
        y[gaps] = float("nan")
        del gaps
    eng = mmf.ForecastEngine()
    res = {"card": card(), "series": n, "days": t, "horizon": h, "steps": args.steps, "rounds": args.rounds,
           "gap_frac": args.gap_frac, "modes": {}}
    for mode in ("future", "holdout"):
        if mode == "future":
            _, ps, npred = eng.plan_calendar("2019-01-01", t, "D", h, "future")
            t_fit = t
        else:
            _, ps, npred = eng.plan_calendar("2019-01-01", t, "D", h, "holdout")
            t_fit = t - h
        pitch = (npred + 3) & ~3
        out = torch.empty((n, pitch), device="cuda")[:, :npred]
        se = torch.empty((n, pitch), device="cuda")[:, :npred]
        sigma = torch.empty(n, device="cuda")
        dof = torch.empty(n, device="cuda", dtype=torch.int32)
        status = torch.empty(n, device="cuda", dtype=torch.int32)
        lib, hnd = eng._lib, eng._h
        eng.set_stream(torch.cuda.current_stream().cuda_stream)

        def plain():
            mmf._native.check(lib.mmf_fit_forecast_f32(hnd, y.data_ptr(), n, y.stride(0), ps, npred, out.data_ptr(),
                                                       out.stride(0), None, status.data_ptr(), None))

        def with_se():
            mmf._native.check(lib.mmf_fit_forecast_se_f32(hnd, y.data_ptr(), n, y.stride(0), ps, npred, out.data_ptr(),
                                                          out.stride(0), se.data_ptr(), se.stride(0), sigma.data_ptr(),
                                                          dof.data_ptr(), status.data_ptr(), None))

        times = {"plain": [], "se": []}
        for fn in (plain, with_se):
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for name, fn in (("plain", plain), ("se", with_se)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / args.steps)
        # algorithmic bytes per series: y read once, forecasts written (+ se rows, sigma, dof)
        b_plain = 4 * t_fit + 4 * npred
        b_se = b_plain + 4 * npred + 8
        med = {k: float(np.median(v)) for k, v in times.items()}
        res["modes"][mode] = {"ms_per_step": times, "median_ms": med, "se_over_plain": med["se"] / med["plain"],
                              "byte_ratio": b_se / b_plain}
        print(f"{mode:8s} plain {med['plain']:.3f} ms  se {med['se']:.3f} ms  ratio {med['se'] / med['plain']:.3f}"
              f"  (algorithmic bytes x{b_se / b_plain:.3f})", flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
