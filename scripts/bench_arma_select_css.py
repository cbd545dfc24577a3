"""Cost and accuracy of the (p, d, q) selection's winner refit (mmf_fit_select_arma_css_f32 / _joint_f32) on two holdout
shapes: C4 (1 M series x 1,095 days, horizon 28) and the reference's weekly shape (157 weeks, 117 fit weeks, horizon 40),
gap-free and with 1e-3 of the values missing, over the reference grid p 0..4 x d 0..2 x q 0..4.  Four arms alternate over
several rounds after a warm-up, timed with CUDA events around work that ends in a synchronise:
  select   ForecastEngine.fit_select_arma (the selection alone);
  css      fit_select_arma(refit="css");
  joint    fit_select_arma(refit="css", joint_beta=True);
  compose  what the refit call replaces on the caller's side: the selection, then per winning (p, d, q >= 1) class a
           gather of its rows (16-B row pitch), the fixed-order CSS call with long_order = m_d, and a scatter of its
           outputs back.
Prints ms per call (median and spread), the refit rows' passes (mean, p50, p90) and stop shares, the share of rows
refit and refined, the hold-out MSE of the selection against each refit (NaN-aware), and the card's name and power limit.

--refit ml (mmf_fit_select_arma_ml_f32, DESIGN.md section 2 item 21) times select, css, ml (fit_select_arma(refit="ml"))
and, with --kalman, mlkf (refit="ml", predictor="kalman"); compose is then the composition of the last of them (the
fixed-order call with estimator="ml", and predictor="kalman" with --kalman).  The ML arms' pass statistics are those of
the ML refinement (iters, ml_stop).

    python scripts/bench_arma_select_css.py [--series 1000000] [--steps 1] [--rounds 3] [--shapes ...] [--out FILE]
                                            [--refit css|ml] [--kalman]
"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmf  # noqa: E402
from bench_arma import card, shape_of  # noqa: E402

GRID = ((0, 1, 2, 3, 4), (0, 1, 2), (0, 1, 2, 3, 4))


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps, r


def long_order(t_fit, d):
    """the selection's m_d for long_order = 0 (include/mmf.h)"""
    lt = math.log(t_fit - d)
    return min(32, max(2 * max(max(GRID[0]), max(GRID[2])), int(math.floor(lt * lt))))


def compose(eng, y, t_fit, h, ps, npred, **fixed):
    """the selection, then the fixed-order call (CSS, or `fixed`) per winning class on its gathered rows, scattered
    back"""
    res = eng.fit_select_arma(y, h, *GRID, ps, npred)
    cp, cd, cq = res["choice_p"], res["choice_d"], res["choice_q"]
    key = (cp * 100 + cd * 10 + cq)[cq >= 1]
    ld = (t_fit + 3) & ~3
    for k in torch.unique(key).tolist():
        p, d, q = k // 100, (k // 10) % 10, k % 10
        idx = torch.nonzero((cp == p) & (cd == d) & (cq == q)).squeeze(1)
        sub = torch.empty((len(idx), ld), device=y.device)
        sub[:, :t_fit] = y[idx, :t_fit]
        r = eng.fit_forecast_arma(sub[:, :t_fit], p, q, d, ps, npred, long_order=long_order(t_fit, d),
                                  **(fixed or {"estimator": "css"}))
        for name, v in r.items():
            if name in res:
                res[name][idx] = v
            else:
                res.setdefault(name, torch.full((len(y),) + tuple(v.shape[1:]), float("nan") if v.is_floating_point()
                                                else 0, device=y.device, dtype=v.dtype))[idx] = v
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="C4_holdout,weekly157")
    ap.add_argument("--gaps", default="0,0.001")
    ap.add_argument("--out", default=None)
    ap.add_argument("--refit", choices=("css", "ml"), default="css")
    ap.add_argument("--kalman", action="store_true", help="with --refit ml: also the Kalman predictor's arm")
    args = ap.parse_args()
    ml = args.refit == "ml"
    name, limit = card()
    rows = []
    for shape in args.shapes.split(","):
        y, start, t, freq, h, mode = shape_of(shape, args.series)
        t_fit = t - h
        eng = mmf.ForecastEngine()
        _, ps, npred = eng.plan_calendar(start, t, freq, h, mode, max_diff=2)
        for gap in (float(g) for g in args.gaps.split(",")):
            yg = y
            if gap:
                gen = torch.Generator(device=y.device).manual_seed(3)
                yg = y.clone()
                yg[torch.rand(yg.shape, device=y.device, generator=gen) < gap] = float("nan")
            arms = {
                "select": lambda: eng.fit_select_arma(yg, h, *GRID, ps, npred),
                "css": lambda: eng.fit_select_arma(yg, h, *GRID, ps, npred, refit="css"),
                "joint": lambda: eng.fit_select_arma(yg, h, *GRID, ps, npred, refit="css", joint_beta=True),
                "compose": lambda: compose(eng, yg, t_fit, h, ps, npred),
            }
            if ml:
                kf = dict(predictor="kalman") if args.kalman else {}
                del arms["joint"]
                arms = {"select": arms["select"], "css": arms["css"],
                        "ml": lambda: eng.fit_select_arma(yg, h, *GRID, ps, npred, refit="ml"),
                        **({"mlkf": lambda: eng.fit_select_arma(yg, h, *GRID, ps, npred, refit="ml", **kf)}
                           if args.kalman else {}),
                        "compose": lambda: compose(eng, yg, t_fit, h, ps, npred, estimator="ml", **kf)}
            for fn in arms.values():                          # warm-up: every shape the timed window uses
                fn()
                torch.cuda.synchronize()
            times, last = {k: [] for k in arms}, {}
            for _ in range(args.rounds):
                for k, fn in arms.items():
                    last.pop(k, None)
                    torch.cuda.empty_cache()
                    ms, last[k] = timed(fn, args.steps)
                    times[k].append(ms)
            sel, cs, cm = last["select"], last["css"], last["compose"]
            refit = (cs["choice_q"] >= 1).cpu().numpy()
            rec = dict(shape=shape, gaps=gap, series=args.series, refit_share=float(refit.mean()))
            for k in arms:
                rec[f"{k}_ms"] = float(np.median(times[k]))
                rec[f"{k}_ms_range"] = [float(min(times[k])), float(max(times[k]))]
            top = "css" if not ml else ("mlkf" if args.kalman else "ml")   # the arm compose stands in for
            cols = (("css", "css_start", "css_stop") if not ml else ("loglik", "loglik_start", "ml_stop"))
            same_bits = all(torch.equal(last[top][k].view(torch.int32) if cm[k].is_floating_point() else last[top][k],
                                        cm[k].view(torch.int32) if cm[k].is_floating_point() else cm[k])
                            for k in ("pred", "phi", "theta", "sigma", "iters") + cols)
            rec[f"{top}_equals_compose"] = bool(same_bits)
            yh = yg[:, t_fit:t].float()
            for k in [k for k in arms if k != "compose"]:
                r = last[k]
                if k != "select":
                    it = r["iters"].cpu().numpy()[refit]
                    stop = r["ml_stop" if k in ("ml", "mlkf") else "css_stop"].cpu().numpy()[refit]
                    refined = ((r["phi"] != sel["phi"]).any(1) | (r["theta"] != sel["theta"]).any(1)).cpu().numpy()
                    rec[f"{k}_passes"] = ([float(it.mean()), float(np.percentile(it, 50)), float(np.percentile(it, 90))]
                                          if it.size else [])
                    rec[f"{k}_stop_shares"] = (np.bincount(stop, minlength=4)[1:] / max(stop.size, 1)).tolist()
                    rec[f"{k}_refined_share"] = float(refined[refit].mean()) if refit.any() else 0.0
                e = r["pred"][:, t_fit:t] - yh
                ok = torch.isfinite(e)
                rec[f"mse_{k}"] = float((torch.where(ok, e, 0.0) ** 2).sum() / ok.sum())
            rows.append(rec)
            print(json.dumps(rec), flush=True)
            del last, sel, cs, cm
            torch.cuda.empty_cache()
        eng.close()
        del y
        torch.cuda.empty_cache()
    res = {"card": name, "power_limit": limit, "series": args.series, "rows": rows}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps({"card": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
