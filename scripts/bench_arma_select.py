"""Cost and accuracy of (p, d, q) selection by hold-out MSE on levels (mmf_fit_select_arma_f32) against the calls it
composes, on two holdout shapes: C4 (1 M series x 1,095 days of synth.daily_store_item_demand_torch, horizon 28) and the
reference's weekly shape (1 M seeded series on its 157-week calendar, synth.reference_calendar, 117 fit weeks, horizon
40), over the reference grid (0..4) x (0, 1, 2) x (0..4).  The arms alternate in one process, several rounds of
`--steps` calls each after a warm-up, timed with CUDA events:
  plain         the plain fit (holdout window);
  pdsel         the (p, d) selection over (0..4) x (0, 1, 2) (mmf_fit_select_arima_f32);
  arma1d1       ARIMA(1, d, 1) in holdout mode, d = 0, 1, 2;
  compose       what a caller runs without the new call: the (p, d) selection with the holdout window (the q = 0 block,
                its cand_mse the scores), one future-mode ARMA call per (p, d, q >= 1) candidate with the call's long
                order m_d, the scores and the first minimum on the GPU (torch), and one holdout ARMA call per winning
                (p, d, q >= 1), scattered into the table;
  select        the new call.
It checks that compose's choices and predictions equal the new call's, except on rows whose two best scores lie within
1e-6 relative, and prints ms/step per arm (median), the chosen q histogram, the mean hold-out MSE of the arms, and the
card's name and power limit.  `--profile` adds a torch.profiler split by kernel of one call of `select`.  `--split`
times `select` again with the timing builds tests/_build/libmmf_armasel_stop{1,2,3}.so (arma_select_kernel ending after
pass A, after pass A2 and the solve, before pass B) and attributes the kernel's time to its passes by difference.

    python scripts/bench_arma_select.py [--series 1000000] [--steps 1] [--rounds 3] [--profile] [--split] [--out FILE]
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mmf  # noqa: E402

ORDERS, DIFFS, MAS = (0, 1, 2, 3, 4), (0, 1, 2), (0, 1, 2, 3, 4)


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


def long_order(t_fit, d):
    lt = math.log(t_fit - d)
    return min(32, max(2 * max(max(ORDERS), max(MAS)), int(math.floor(lt * lt))))


def split_passes(args):
    """median ms of `select` with the product library and each timing build (one subprocess each)"""
    libs = {"full": None, "stop1": "libmmf_armasel_stop1.so", "stop2": "libmmf_armasel_stop2.so",
            "stop3": "libmmf_armasel_stop3.so"}
    got = {}
    for name, lib in libs.items():
        env = dict(os.environ)
        env.pop("MMF_LIB", None)
        if lib:
            env["MMF_LIB"] = os.path.join(ROOT, "tests", "_build", lib)
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--series", str(args.series), "--steps",
                              str(args.steps), "--rounds", str(args.rounds), "--arms", "pdsel,select"], env=env,
                             capture_output=True, text=True, check=True).stdout
        got[name] = {ln.split(" ", 1)[0]: json.loads(ln.split(" ", 1)[1])["median_ms"] for ln in out.splitlines()
                     if ln.split(" ", 1)[0] in ("C4_holdout", "weekly157")}
    res = {"card": card(), "series": args.series, "split": {}}
    for shape in got["full"]:
        f, a, b, c = (got[k][shape]["select"] for k in ("full", "stop1", "stop2", "stop3"))
        pd = got["full"][shape]["pdsel"]
        res["split"][shape] = {"select_ms": f, "pdsel_ms": pd, "stop1_ms": a, "stop2_ms": b, "stop3_ms": c,
                               "pass_A_and_step1_ms": a - pd, "pass_A2_and_solve_ms": b - a,
                               "walk_and_choice_ms": c - b, "pass_B_ms": f - c}
        print(shape, json.dumps(res["split"][shape]), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--arms", default="plain,pdsel,arma1d1,compose,select")
    ap.add_argument("--profile", action="store_true", help="torch.profiler table of one call of the new arm per shape")
    ap.add_argument("--split", action="store_true", help="time of arma_select_kernel per pass, from the timing builds")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.split:
        split_passes(args)
        return
    n = args.series
    eng = mmf.ForecastEngine()
    lib, hnd = eng._lib, eng._h
    check = mmf._native.check
    res = {"card": card(), "series": n, "steps": args.steps, "rounds": args.rounds, "lib": mmf.LIB_PATH, "shapes": {}}
    arr = lambda v: (C.c_int32 * len(v))(*v)
    cand, dl, ql = arr(ORDERS), arr(DIFFS), arr(MAS)
    pairs = [(p, d, q) for d in DIFFS for q in MAS[1:] for p in ORDERS]
    for shape in ("C4_holdout", "weekly157"):
        y, start, t, freq, h = shape_of(shape, n)
        _, ps, npred = eng.plan_calendar(start, t, freq, h, "holdout", max_diff=2)
        t_fit = t - h
        dev = "cuda"
        wide = lambda m: torch.empty((n, (m + 3) & ~3), device=dev)[:, :m]
        out, tmp = wide(npred), wide(npred)
        fut = {c: wide(h) for c in pairs} if "compose" in args.arms else {}
        status = torch.empty(n, device=dev, dtype=torch.int32)
        cp, cd, cq = (torch.empty(n, device=dev, dtype=torch.int32) for _ in range(3))
        cm0 = torch.empty((n, len(DIFFS), len(ORDERS)), device=dev)
        cm = torch.empty((n, len(DIFFS), len(MAS), len(ORDERS)), device=dev)
        mse = torch.empty(n, device=dev)
        eng.set_stream(torch.cuda.current_stream().cuda_stream)
        act = y[:, t_fit:t]
        comp = {}

        def plain():
            check(lib.mmf_fit_forecast_f32(hnd, y.data_ptr(), n, y.stride(0), ps, npred, out.data_ptr(), out.stride(0),
                                           None, status.data_ptr(), None))

        def pdsel():
            check(lib.mmf_fit_select_arima_f32(hnd, y.data_ptr(), n, y.stride(0), h, cand, len(ORDERS), dl, len(DIFFS),
                                               ps, npred, out.data_ptr(), out.stride(0), None, None, None,
                                               cm0.data_ptr(), None, None, None, status.data_ptr(), None))

        def arma(p, d, q, o, pst, npr):
            check(lib.mmf_fit_forecast_arma_f32(hnd, y.data_ptr(), n, y.stride(0), p, d, q, long_order(t_fit, d), pst,
                                                npr, o.data_ptr(), o.stride(0), None, None, None, None, None,
                                                status.data_ptr(), None))

        def arma1d1():
            for d in DIFFS:
                arma(1, d, 1, out, ps, npred)

        def compose():
            pdsel()
            for (p, d, q), o in fut.items():
                arma(p, d, q, o, t_fit, h)
            blocks = []
            for k, d in enumerate(DIFFS):
                blocks.append(cm0[:, k, :].double())
                for q in MAS[1:]:
                    blocks.append(torch.stack([mse_rows(fut[p, d, q], act) for p in ORDERS], dim=1))
            flat = torch.cat(blocks, dim=1)                                   # list order: d, then q, then p
            win = torch.where(torch.isnan(flat), torch.full_like(flat, float("inf")), flat).argmin(dim=1)
            nq, no = len(MAS), len(ORDERS)
            wd, wq, wp = win // (nq * no), (win // no) % nq, win % no
            wq = torch.where(torch.isnan(flat).all(dim=1), torch.zeros_like(wq), wq)   # nothing scored: pdsel's
            for k, d in enumerate(DIFFS):
                for l in range(1, nq):
                    for j in range(no):
                        rows = (wd == k) & (wq == l) & (wp == j)
                        if bool(rows.any()):
                            arma(ORDERS[j], d, MAS[l], tmp, ps, npred)
                            out[rows] = tmp[rows]
            comp.update(scores=flat, wd=wd, wq=wq, wp=wp)

        def select():
            check(lib.mmf_fit_select_arma_f32(hnd, y.data_ptr(), n, y.stride(0), h, cand, len(ORDERS), dl, len(DIFFS),
                                              ql, len(MAS), 0, ps, npred, out.data_ptr(), out.stride(0), cp.data_ptr(),
                                              cd.data_ptr(), cq.data_ptr(), mse.data_ptr(), cm.data_ptr(), None, None,
                                              None, None, None, status.data_ptr(), None))

        arms = {"plain": plain, "pdsel": pdsel, "arma1d1": arma1d1, "compose": compose, "select": select}
        arms = {k: v for k, v in arms.items() if k in args.arms.split(",")}
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
        entry = {"t": t, "t_fit": t_fit, "horizon": h, "ms_per_step": times, "median_ms": med}
        if "compose" in arms and "select" in arms:
            entry["speedup_over_compose"] = med["compose"] / med["select"]
            entry["gate_5x_faster_than_compose"] = med["select"] * 5 <= med["compose"]
            # agreement of compose and select: choices and predictions, except on rows whose two best scores are within
            # 1e-6 relative
            compose()
            pred_c = out.clone()
            select()
            torch.cuda.synchronize()
            s = torch.where(torch.isnan(comp["scores"]), torch.full_like(comp["scores"], float("inf")), comp["scores"])
            two = s.sort(dim=1).values[:, :2]
            amb = torch.isfinite(two[:, 1]) & (two[:, 1] - two[:, 0] <= 1e-6 * two[:, 1].abs())
            tv = lambda v, i: torch.tensor(v, device=dev)[i]
            same_choice = ((cd.long() == tv(DIFFS, comp["wd"])) & (cq.long() == tv(MAS, comp["wq"])) &
                           (cp.long() == tv(ORDERS, comp["wp"])))
            same_pred = ((pred_c == out) | (torch.isnan(pred_c) & torch.isnan(out))).all(dim=1)
            entry["agreement"] = {"rows": n, "ambiguous": int(amb.sum()),
                                  "choice_differs_outside_ambiguous": int((~same_choice & ~amb).sum()),
                                  "pred_differs_outside_ambiguous": int((~same_pred & ~amb).sum())}
        if "select" in arms:
            select()
            torch.cuda.synchronize()
            entry["choice_q_histogram"] = {str(q): int((cq == q).sum()) for q in (-1,) + MAS}
            entry["choice_d_histogram"] = {str(d): int((cd == d).sum()) for d in (-1,) + DIFFS}
            means = {"select_chosen": float(torch.nanmean(mse.double()).item())}
            if "pdsel" in arms:
                pdsel()
                means["pdsel_chosen"] = float(torch.nanmean(mse_rows(out[:, t_fit:t], act)).item())
            for d in DIFFS:
                arma(1, d, 1, out, ps, npred)
                means[f"arima1{d}1"] = float(torch.nanmean(mse_rows(out[:, t_fit:t], act)).item())
            entry["mean_holdout_mse"] = means
        if args.profile and "select" in arms:
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
        del y, out, tmp, fut, status, cp, cd, cq, cm0, cm, mse, comp
        torch.cuda.empty_cache()
    print(json.dumps({k: v for k, v in res.items() if k != "shapes"}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
