"""Cost of the ARIMA-family forecast standard errors (mmf_arima_se_f32, DESIGN.md section 2 item 15) against the model
calls that feed it and against a torch copy that moves the same bytes.

Shapes: C4 (1 M series x 1,095 days of synth.daily_store_item_demand_torch, device-resident) in future mode (horizon 28)
and holdout mode, gap-free and with `--gap-frac` of the values missing; and the reference's weekly shape (157 weeks,
117 fit, horizon 40) in holdout mode.  Parameters come from ARIMA(1, 1, 0), ARIMA(1, 1, 1) and (holdout mode) the
reference-grid fit_select_arma.  Per round the model call, the se call and the yardstick run once each after one
another (the se call and the yardstick `--steps` times, CUDA events); the medians over `--rounds` rounds are printed
with the algorithmic bytes (y rows read, se written, parameters) and the card's name and power limit.

    python scripts/bench_arima_se.py [--series 1000000] [--steps 5] [--rounds 5] [--gap-frac 1e-3] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmf  # noqa: E402
from mmf import _native as N  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def se_call(eng, y, t_fit, res, d, ps, npred, out):
    th, ma, dd = res.get("theta"), res.get("ma_order"), res.get("choice_d")
    p = lambda x: None if x is None else x.data_ptr()                                    # noqa: E731
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    N.check(N.load().mmf_arima_se_f32(eng._h, y.data_ptr(), y.shape[0], y.stride(0), t_fit, d, p(dd),
                                      res["phi"].data_ptr(), res["order"].data_ptr(), p(th), p(ma),
                                      res["sigma"].data_ptr(), ps, npred, out.data_ptr(), out.stride(0), None))


def run_shape(name, y, start, t, freq, horizon, mode, args, results):
    eng = mmf.ForecastEngine()
    _, ps, npred = eng.plan_calendar(start, t, freq, horizon, mode, max_diff=2)
    t_fit = t - horizon if mode == "holdout" else t
    n = y.shape[0]
    arms = {"arima110": (lambda: eng.fit_forecast_arima(y[:, :t_fit], 1, 1, ps, npred), 1, 0),
            "arima111": (lambda: eng.fit_forecast_arma(y[:, :t_fit], 1, 1, 1, ps, npred), 1, 1)}
    if mode == "holdout":
        arms["select_arma"] = (lambda: eng.fit_select_arma(y, horizon, pred_start=ps, n_pred=npred), 0, 4)
    out = torch.empty((n, npred), device="cuda")
    for arm, (model, d, q) in arms.items():
        res = model()
        torch.cuda.synchronize()
        # algorithmic bytes: y rows read (future mode, q = 0: only the p + d levels before t_fit), se written, parameters
        read = n * 4 * (t_fit if (mode == "holdout" or q > 0) else 2)
        nbytes = read + n * 4 * npred + n * 64
        src = torch.empty(nbytes // 8, dtype=torch.float32, device="cuda")
        dst = torch.empty_like(src)
        fn = lambda: se_call(eng, y, t_fit, res, d, ps, npred, out)                      # noqa: E731
        fn()
        dst.copy_(src)
        ms_model, ms_se, ms_yard = [], [], []
        for _ in range(args.rounds):
            ms_model.append(timed(model, 1))
            ms_se.append(timed(fn, args.steps))
            ms_yard.append(timed(lambda: dst.copy_(src), args.steps))
        r = {"shape": name, "mode": mode, "arm": arm, "model_ms": statistics.median(ms_model),
             "se_ms": statistics.median(ms_se), "yardstick_ms": statistics.median(ms_yard), "bytes": nbytes}
        r["se_over_yardstick"] = r["se_ms"] / r["yardstick_ms"]
        r["se_over_model"] = r["se_ms"] / r["model_ms"]
        r["se_GBps"] = nbytes / r["se_ms"] / 1e6
        print(json.dumps(r), flush=True)
        results.append(r)
        del src, dst, res
    eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--gap-frac", type=float, default=1e-3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    results = []
    y, start = mmf.synth.daily_store_item_demand_torch(args.series, 1095, seed=0)
    g = torch.Generator(device="cuda").manual_seed(1)
    for gaps in (False, True):
        if gaps:
            y[torch.rand(y.shape, device="cuda", generator=g) < args.gap_frac] = float("nan")
        for mode in ("future", "holdout"):
            run_shape("C4" + ("_gaps" if gaps else ""), y, start, 1095, "D", 28, mode, args, results)
    del y
    days = mmf.synth.reference_calendar()[0]
    yw, _ = mmf.synth.daily_store_item_demand_torch(args.series, len(days), seed=1)
    run_shape("weekly157", yw, days[0], len(days), "W-MON", 40, "holdout", args, results)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit": limit, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
