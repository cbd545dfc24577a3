"""Cost and accuracy of ARIMA(p, d, q) errors by conditional least squares (mmf_fit_forecast_arma_css_f32) against the
Hannan-Rissanen call it refines, on scripts/bench_arma.py's shapes (C4 future and holdout, the reference's weekly
holdout), gap-free and with 1e-3 of the values missing, for ARMA(1, 0, 1), ARIMA(1, 1, 1) and ARIMA(1, 2, 1).  Each arm
alternates the HR call with the CSS call over several rounds after a warm-up, timed with CUDA events; prints ms per call
(median), ms per pass (the CSS call's extra time over the mean pass count), the distribution of passes and stop codes,
the share of rows refined, in holdout mode the hold-out MSE of both, and the card's name and power limit.  ``--joint`` adds
the joint call (mmf_fit_forecast_arma_joint_f32, beta estimated with (phi, theta)) to the alternation, with its ms per
call and per pass, passes, stops, share refined and hold-out MSE.  ``--ml`` adds the exact-likelihood call
(mmf_fit_forecast_arma_ml_f32, which runs the CSS call and refines it) the same way, its ms per pass being its extra time
over the CSS call divided by its mean ML pass count.  ``--kalman`` (with ``--ml``) adds the ML call with the Kalman
predictor (mmf_fit_forecast_arma_ml_kf_f32): its ms, the predictor stage's cost (its extra time over the ML call) in
total and per series, and its hold-out MSE.

    python scripts/bench_arma_css.py [--series 1000000] [--steps 3] [--rounds 3] [--shapes ...] [--joint] [--ml] [--kalman]
                                     [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmf  # noqa: E402
from bench_arma import card, shape_of  # noqa: E402

ORDERS = {"arma101": (1, 0, 1), "arima111": (1, 1, 1), "arima121": (1, 2, 1)}     # (p, d, q)


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="C4_future,C4_holdout,weekly157")
    ap.add_argument("--gaps", default="0,0.001")
    ap.add_argument("--orders", default=",".join(ORDERS))
    ap.add_argument("--joint", action="store_true")
    ap.add_argument("--ml", action="store_true")
    ap.add_argument("--kalman", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    name, limit = card()
    rows = []
    for shape in args.shapes.split(","):
        y, start, t, freq, h, mode = shape_of(shape, args.series)
        t_fit = t if mode == "future" else t - h
        eng = mmf.ForecastEngine()
        _, ps, npred = eng.plan_calendar(start, t, freq, h, mode, max_diff=2)
        for gap in (float(g) for g in args.gaps.split(",")):
            yg = y
            if gap:
                gen = torch.Generator(device=y.device).manual_seed(3)
                yg = y.clone()
                yg[torch.rand(yg.shape, device=y.device, generator=gen) < gap] = float("nan")
            yf = yg[:, :t_fit]
            for oname in args.orders.split(","):
                p, d, q = ORDERS[oname]
                hr_call = lambda: eng.fit_forecast_arma(yf, p, q, d, ps, npred)          # noqa: E731
                css_call = lambda: eng.fit_forecast_arma(yf, p, q, d, ps, npred, estimator="css")  # noqa: E731
                joint_call = lambda: eng.fit_forecast_arma(yf, p, q, d, ps, npred, estimator="css",  # noqa: E731
                                                           joint_beta=True)
                ml_call = lambda: eng.fit_forecast_arma(yf, p, q, d, ps, npred, estimator="ml")  # noqa: E731
                kf_call = lambda: eng.fit_forecast_arma(yf, p, q, d, ps, npred, estimator="ml",  # noqa: E731
                                                        predictor="kalman")
                hr_call(), css_call()
                if args.joint:
                    joint_call()
                if args.ml:
                    ml_call()
                if args.kalman:
                    kf_call()
                t_hr, t_css, t_joint, t_ml, t_kf = [], [], [], [], []
                for _ in range(args.rounds):
                    ms, hr = timed(hr_call, args.steps)
                    t_hr.append(ms)
                    ms, cs = timed(css_call, args.steps)
                    t_css.append(ms)
                    if args.joint:
                        ms, jt = timed(joint_call, args.steps)
                        t_joint.append(ms)
                    if args.ml:
                        ms, ml = timed(ml_call, args.steps)
                        t_ml.append(ms)
                    if args.kalman:
                        ms, kf = timed(kf_call, args.steps)
                        t_kf.append(ms)
                g = (cs["css_stop"] > 0).cpu().numpy()
                it = cs["iters"].cpu().numpy()[g]
                stop = cs["css_stop"].cpu().numpy()[g]
                refined = ((cs["phi"] != hr["phi"]).any(1) | (cs["theta"] != hr["theta"]).any(1)).cpu().numpy()
                rec = dict(shape=shape, gaps=gap, order=oname, hr_ms=float(np.median(t_hr)),
                           css_ms=float(np.median(t_css)), gated=float(g.mean()), refined=float(refined.mean()),
                           iters_mean=float(it.mean()) if it.size else 0.0,
                           iters_pct=[float(v) for v in np.percentile(it, [50, 90, 100])] if it.size else [],
                           stops=np.bincount(stop, minlength=4)[1:].tolist())
                rec["ms_per_pass"] = (rec["css_ms"] - rec["hr_ms"]) / max(rec["iters_mean"], 1.0)
                arms = (("hr", hr), ("css", cs))
                if args.joint:
                    itj = jt["iters"].cpu().numpy()[g]
                    rec.update(joint_ms=float(np.median(t_joint)),
                               joint_refined=float(((jt["phi"] != hr["phi"]).any(1) | (jt["theta"] != hr["theta"]).any(1)
                                                    | ((jt["pred"] != hr["pred"]) & ~(jt["pred"].isnan() & hr["pred"].isnan()))
                                                    .any(1)).float().mean()),
                               joint_iters_mean=float(itj.mean()) if itj.size else 0.0,
                               joint_stops=np.bincount(jt["css_stop"].cpu().numpy()[g], minlength=4)[1:].tolist())
                    rec["joint_ms_per_pass"] = (rec["joint_ms"] - rec["hr_ms"]) / max(rec["joint_iters_mean"], 1.0)
                    arms += (("joint", jt),)
                if args.ml:
                    itm = ml["iters"].cpu().numpy()[g]
                    rec.update(ml_ms=float(np.median(t_ml)),
                               ml_refined=float(((ml["phi"] != cs["phi"]).any(1) | (ml["theta"] != cs["theta"]).any(1))
                                                .float().mean()),
                               ml_iters_mean=float(itm.mean()) if itm.size else 0.0,
                               ml_iters_pct=[float(v) for v in np.percentile(itm, [50, 90, 100])] if itm.size else [],
                               ml_stops=np.bincount(ml["ml_stop"].cpu().numpy()[g], minlength=4).tolist())
                    rec["ml_ms_per_pass"] = (rec["ml_ms"] - rec["css_ms"]) / max(rec["ml_iters_mean"], 1.0)
                    arms += (("ml", ml),)
                if args.kalman:
                    rec.update(kf_ms=float(np.median(t_kf)))
                    rec["kf_stage_ms"] = rec["kf_ms"] - rec["ml_ms"]
                    rec["kf_stage_ns_per_series"] = rec["kf_stage_ms"] * 1e6 / args.series
                    arms += (("kf", kf),)
                if mode == "holdout":
                    yh = yg[:, t_fit:t].float()
                    for k, r in arms:
                        e = (r["pred"][:, t_fit:t] - yh)
                        ok = torch.isfinite(e)
                        rec[f"mse_{k}"] = float((torch.where(ok, e, 0.0) ** 2).sum() / ok.sum())
                rows.append(rec)
                print(json.dumps(rec), flush=True)
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
