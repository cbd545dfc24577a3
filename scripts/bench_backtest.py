"""Rolling-origin backtest: one mmf_backtest_f32 call (K origins in one pass over the data) against two per-origin arms:
K single-origin mmf_backtest_f32 calls (each reads its own prefix [0, t_k) and scores with the same kernel; the library
has no entry point for the scoring kernel alone, so this is the per-origin arm that includes scoring), and K plain
future-mode mmf_fit_forecast_f32 calls without any scoring (a lower bound of what K plain calls plus scoring cost).
Device-resident, fully observed series, daily calendar; all plans are made before the timed region.  Times with CUDA events (warm-up, then the median over --steps steps of each
arm, the arms alternating), and reports the algorithmic bytes per second of the one-pass call as a share of the H100
SXM's 3.35 TB/s, the card's name and power limit read in the same run, and the largest difference between the two
arms' forecasts.

    python scripts/bench_backtest.py [--shape C4|C5] [--origins 4] [--horizon 28] [--step 28] [--steps 10] [--out FILE]

C4: 1 M series x 1,095 days; C5: 10 M series x 365 days.
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

HBM_GBS = 3350.0


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
    ap.add_argument("--shape", default="C4", choices=["C4", "C5"])
    ap.add_argument("--origins", type=int, default=4)
    ap.add_argument("--horizon", type=int, default=28)
    ap.add_argument("--step", type=int, default=None)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    n, t = {"C4": (1_000_000, 1095), "C5": (10_000_000, 365)}[args.shape]
    K, h = args.origins, args.horizon
    g = torch.Generator(device="cuda").manual_seed(0)
    full = torch.empty((n, (t + 3) & ~3), device="cuda")
    y = full[:, :t]
    for i0 in range(0, n, 1 << 20):                         # in blocks: the temporaries of 10 M x 365 at once do not fit
        i1 = min(n, i0 + (1 << 20))
        level = 20.0 + 480.0 * torch.rand((i1 - i0, 1), device="cuda", generator=g)
        y[i0:i1].copy_(level + 0.2 * level * torch.randn((i1 - i0, t), device="cuda", generator=g))
    start = "2019-01-01"
    one = mmf.ForecastEngine()
    origins = one.plan_backtest(start, t, "D", h, K, args.step)
    per, plain = [], []                                     # one context per origin: single-origin / plain plans
    X = mmf.design.design_matrix(mmf.design.calendar_grid(start, t, "D"), t - h)
    for k in range(K):
        e = mmf.ForecastEngine()
        e.plan_backtest(start, int(origins[k]) + h, "D", h, 1)
        per.append(e)
        e = mmf.ForecastEngine()
        e.plan(X[:int(origins[k]) + h], int(origins[k]), True)
        plain.append(e)
    pitch = (h + 3) & ~3
    pred = torch.empty((K, n, pitch), device="cuda")[:, :, :h]
    met = torch.empty((K, n, 4), device="cuda")
    cnt = torch.empty((K, n), device="cuda", dtype=torch.int32)
    st = torch.empty((K, n), device="cuda", dtype=torch.int32)
    pred1 = torch.empty((K, n, pitch), device="cuda")[:, :, :h]
    met1 = torch.empty((K, n, 4), device="cuda")
    cnt1 = torch.empty((K, n), device="cuda", dtype=torch.int32)
    st1 = torch.empty((K, n), device="cuda", dtype=torch.int32)
    stream = torch.cuda.current_stream().cuda_stream
    pred2 = torch.empty((K, n, pitch), device="cuda")[:, :, :h]
    st2 = torch.empty((K, n), device="cuda", dtype=torch.int32)
    for e in [one] + per + plain:
        e.set_stream(stream)

    def one_pass():
        mmf._native.check(one._lib.mmf_backtest_f32(one._h, y.data_ptr(), n, y.stride(0), pred.data_ptr(), pred.stride(1),
                                                    met.data_ptr(), cnt.data_ptr(), st.data_ptr(), None))

    def per_origin():
        for k, e in enumerate(per):
            mmf._native.check(e._lib.mmf_backtest_f32(e._h, y.data_ptr(), n, y.stride(0), pred1[k].data_ptr(),
                                                      pred1.stride(1), met1[k].data_ptr(), cnt1[k].data_ptr(),
                                                      st1[k].data_ptr(), None))

    def plain_calls():
        for k, e in enumerate(plain):
            mmf._native.check(e._lib.mmf_fit_forecast_f32(e._h, y.data_ptr(), n, y.stride(0), int(origins[k]), h,
                                                          pred2[k].data_ptr(), pred2.stride(1), None, st2[k].data_ptr(),
                                                          None))

    for _ in range(args.warmup):
        one_pass()
        per_origin()
        plain_calls()
    torch.cuda.synchronize()
    times = {"one_pass": [], "per_origin": [], "plain_no_scoring": []}
    for _ in range(args.steps):
        for name, fn in (("one_pass", one_pass), ("per_origin", per_origin), ("plain_no_scoring", plain_calls)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    med = {k: float(np.median(v)) for k, v in times.items()}
    # algorithmic bytes of the one-pass call: y over [0, t_K) once, the K*h actual values, forecasts, metrics and counts
    t_last = int(origins[-1])
    algo = n * (4.0 * t_last + 4.0 * K * h + 4.0 * K * h + 16.0 * K + 4.0 * K)
    diff = float(torch.nan_to_num((pred - pred1).abs(), 0.0).max())
    diff_plain = float(torch.nan_to_num((pred - pred2).abs(), 0.0).max())
    res = {"card": card(), "shape": args.shape, "series": n, "days": t, "origins": [int(o) for o in origins],
           "horizon": h, "steps": args.steps, "ms": times, "median_ms": med,
           "speedup_per_origin_over_one_pass": med["per_origin"] / med["one_pass"],
           "algorithmic_bytes": algo, "algorithmic_gbs": algo / (med["one_pass"] * 1e-3) / 1e9,
           "share_of_3350_gbs": algo / (med["one_pass"] * 1e-3) / 1e9 / HBM_GBS,
           "sum_tk_over_tK": float(origins.sum()) / t_last,
           "max_abs_forecast_diff": diff, "max_abs_forecast_diff_plain": diff_plain,
           "plain_no_scoring_over_one_pass": med["plain_no_scoring"] / med["one_pass"],
           "status_equal": bool(torch.equal(st, st1)) and bool(torch.equal(st, st2)), "count_equal": bool(torch.equal(cnt, cnt1))}
    print(f"{args.shape}: one pass {med['one_pass']:.3f} ms, {K} single-origin calls {med['per_origin']:.3f} ms "
          f"(x{res['speedup_per_origin_over_one_pass']:.2f}; sum t_k / t_K = {res['sum_tk_over_tK']:.2f}), "
          f"{K} plain calls without scoring {med['plain_no_scoring']:.3f} ms, "
          f"{res['algorithmic_gbs']:.0f} GB/s = {res['share_of_3350_gbs']:.3f} of 3.35 TB/s, max |diff| {diff:.3g}",
          flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
