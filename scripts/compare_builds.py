"""Runs the same seeded workloads through two builds of libmmf.so and checks that every output is bit-identical.

Each build runs in its own process (the library is chosen with MMF_LIB when the package loads) and saves its outputs
to an .npz; the parent process then compares them array by array, NaN payloads included.  Exit code 1 on any
difference.  Needs one GPU.

    python scripts/compare_builds.py --lib-a before.so --lib-b dss-ml-at-scale_b200/libmmf.so [--n 262144] [--out DIR]

Workloads (synthetic daily demand, 1,095 days, 28-day horizon):
  future           future mode, the flagship call
  holdout          holdout mode (the reference's contract: a value for every date)
  missing2         2 % of the values missing in every series
  gaps10           a 10-day gap in 2 % of the series, plus rows whose first 8 values are all missing
  ragged64         64 calendars of 400 to 1,095 days in one ragged launch
  se               the standard-error call
  backtest4        a backtest at K = 4 origins
and the ARIMA-family calls, each on the gap-free series (.clean), missing2 (.missing2) and gaps10 (.gaps10):
  ar3, ar3h        AR(3) errors in future mode, and in holdout mode (every date) on the first n / 8 series
  arsel            AR order selection over (0 .. 4), 28 held-out days
  arima210, arima120  ARIMA(2, 1, 0) and ARIMA(1, 2, 0) errors
  arimasel         (p, d) selection over (0 .. 4) x (0, 1, 2)
  arma111, arma102    ARIMA(1, 1, 1) and ARMA(1, 0, 2) errors
  armasel          (p, d, q) selection over (0, 1, 2) x (0, 1) x (0, 1, 2)
  arimase          the standard errors of ARIMA(2, 1, 0)
  armacss111       ARIMA(1, 1, 1) errors refined by conditional least squares
and besides:
  select           fit_select_forecast over (1, 3, 4, 9, 16) leading columns, 28 held-out days
  u16dev, u16host  fit_forecast on a uint16 series buffer, on the device and in host memory
  seh              the standard-error call in holdout mode (a value for every date)
  bcast1           fit_forecast_bcast with one local output table
  slabs.*          2^20 + 4,096 series x 120 days, two slabs: the plain fit, AR(3), (p, d) selection and the CSS call
Every call that reports stats also saves its kernel launches, kernel used, pending rows and series count, so that the
sequence of launches is compared as well as the outputs (times are not saved).
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, H = 1095, 28


def produce(path, n):
    import torch
    sys.path.insert(0, ROOT)
    import mmf
    dev = torch.device("cuda", 0)
    y, start = mmf.synth.daily_store_item_demand_torch(n, T, seed=4321, device=dev)
    out = {}

    def keep(name, **arrays):
        for k, v in arrays.items():
            if isinstance(v, mmf.Stats):
                for f in ("kernel_launches", "kernel_used", "n_pending", "n_series"):
                    out[f"{name}.stats.{f}"] = np.asarray(getattr(v, f))
            else:
                out[f"{name}.{k}"] = v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)

    eng = mmf.ForecastEngine(device=0)
    _, ps, npred = eng.plan_calendar(start, T, "D", H, "future")
    r = eng.fit_forecast(y, ps, npred, want_status=True, want_stats=True)
    keep("future", **r)

    g = torch.Generator(device=dev).manual_seed(7)
    ym = mmf.device_packed(y, device=dev)         # keeps the 16-B row pitch the tensor-core path reads
    ym[torch.rand(ym.shape, generator=g, device=dev) < 0.02] = float("nan")
    r = eng.fit_forecast(ym, ps, npred, want_status=True, want_stats=True)
    keep("missing2", **r)

    yg = mmf.device_packed(y, device=dev)
    rows = torch.randperm(n, generator=g, device=dev)[: n // 50]
    first = torch.randint(30, T - 30, (rows.numel(),), generator=g, device=dev)
    for k in range(10):
        yg[rows, first + k] = float("nan")
    yg[rows[:64], :8] = float("nan")            # no finite value among the first 8: the centring rule's corner
    yg[rows[64:128], :5] = float("nan")
    r = eng.fit_forecast(yg, ps, npred, want_status=True, want_stats=True)
    keep("gaps10", **r)

    r = eng.fit_forecast_se(ym, ps, npred, want_stats=True)
    keep("se", **r)

    # uint16 series (65535 = missing), widened on the device: a device buffer, and host memory through the staged chunks
    yq = ym.cpu().numpy()
    yi = mmf.to_integer_demand(np.where(np.isfinite(yq), np.clip(np.rint(yq), 0, 65534), np.nan), np.uint16)
    yid = torch.from_numpy(yi.view(np.int16)).to(dev).view(torch.uint16)    # torch has few uint16 ops: bit copy
    keep("u16dev", **eng.fit_forecast(yid, ps, npred, want_status=True, want_stats=True))
    keep("u16host", **eng.fit_forecast(yi, ps, npred, want_status=True, want_stats=True))

    outb = torch.full((n, 32), float("nan"), device=dev)
    stb = torch.empty(n, dtype=torch.int32, device=dev)
    eng.fit_forecast_bcast(ym, ps, npred, [outb.data_ptr()], outb.stride(0), status=stb)
    keep("bcast1", pred=outb, status=stb)
    eng.close()

    engh = mmf.ForecastEngine(device=0)
    _, psh, nph = engh.plan_calendar(start, T, "D", H, "holdout")
    r = engh.fit_forecast(yg, psh, nph, want_status=True, want_stats=True)
    keep("holdout", **r)
    keep("seh", **engh.fit_forecast_se(yg[: n // 8], psh, nph, want_stats=True))
    keep("select", **engh.fit_select_forecast(ym, H, (1, 3, 4, 9, 16), psh, nph))
    engh.close()

    engr = mmf.ForecastEngine(device=0)
    C = 64
    t_lens = np.linspace(400, T, C).astype(int)
    starts = [np.datetime64(start, "D") + np.timedelta64(int(T - tl), "D") for tl in t_lens]
    engr.plan_calendars(starts, t_lens, "D", H)
    cal_rows = np.linspace(0, n, C + 1).astype(np.int64)
    r = engr.fit_forecast_ragged(ym, cal_rows, want_status=True, want_stats=True)
    keep("ragged64", **r)
    engr.close()

    engb = mmf.ForecastEngine(device=0)
    engb.plan_backtest(start, T, "D", H, n_origins=4)
    r = engb.backtest(yg, want_stats=True)
    keep("backtest4", **r)
    engb.close()

    # ARIMA family: future mode on the whole history; selection and holdout mode with the last H days held out
    engf = mmf.ForecastEngine(device=0)
    _, ps, npred = engf.plan_calendar(start, T, "D", H, "future", max_diff=2)
    engh = mmf.ForecastEngine(device=0)
    _, psh, nph = engh.plan_calendar(start, T, "D", H, "holdout", max_diff=2)
    tf = T - H
    st = {"want_stats": True}
    for tag, ys in (("clean", y), ("missing2", ym), ("gaps10", yg)):
        keep(f"ar3.{tag}", **engf.fit_forecast_ar(ys, 3, ps, npred, **st))
        keep(f"ar3h.{tag}", **engh.fit_forecast_ar(ys[: n // 8], 3, psh, nph, **st))
        keep(f"arsel.{tag}", **engh.fit_select_ar(ys, H, (0, 1, 2, 3, 4), tf, H, **st))
        keep(f"arima210.{tag}", **engf.fit_forecast_arima(ys, 2, 1, ps, npred, **st))
        keep(f"arima120.{tag}", **engf.fit_forecast_arima(ys, 1, 2, ps, npred, **st))
        keep(f"arimasel.{tag}", **engh.fit_select_arima(ys, H, (0, 1, 2, 3, 4), (0, 1, 2), tf, H, **st))
        keep(f"arma111.{tag}", **engf.fit_forecast_arma(ys, 1, 1, 1, ps, npred, **st))
        keep(f"arma102.{tag}", **engf.fit_forecast_arma(ys, 1, 2, 0, ps, npred, **st))
        keep(f"armacss111.{tag}", **engf.fit_forecast_arma(ys, 1, 1, 1, ps, npred, estimator="css", **st))
        keep(f"armasel.{tag}", **engh.fit_select_arma(ys, H, (0, 1, 2), (0, 1), (0, 1, 2), tf, H, **st))
        keep(f"arimase.{tag}", **engf.fit_forecast_arima(ys, 2, 1, ps, npred, want_se=True, **st))
    engf.close()
    engh.close()

    # more than 2^20 series on a short calendar: two slabs, each slab's pending count copied aside for the stats
    ns, ts = (1 << 20) + 4096, 120
    ysl = mmf.device_packed(y[:, :ts].repeat((ns + n - 1) // n, 1)[:ns], device=dev)
    ysl[torch.rand(ysl.shape, generator=g, device=dev) < 0.02] = float("nan")
    ysl[rows[:64], :8] = float("nan")
    engs = mmf.ForecastEngine(device=0)
    _, pss, nps = engs.plan_calendar(start, ts, "D", H, "future", max_diff=2)
    keep("slabs.plain", **engs.fit_forecast(ysl, pss, nps, want_status=True, **st))
    keep("slabs.ar3", **engs.fit_forecast_ar(ysl, 3, pss, nps, **st))
    keep("slabs.arma111css", **engs.fit_forecast_arma(ysl, 1, 1, 1, pss, nps, estimator="css", **st))
    del ysl
    engsh = mmf.ForecastEngine(device=0)
    _, pssh, npsh = engsh.plan_calendar(start, ts, "D", H, "holdout", max_diff=2)
    ysh = mmf.device_packed(y[:, :ts].repeat((ns + n - 1) // n, 1)[:ns], device=dev)
    keep("slabs.arimasel", **engsh.fit_select_arima(ysh, H, (0, 1, 2), (0, 1, 2), ts - H, H, **st))
    engs.close()
    engsh.close()
    torch.cuda.synchronize()
    np.savez(path, **out)


def same_bits(a, b):
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", required=True)
    ap.add_argument("--lib-b", required=True)
    ap.add_argument("--n", type=int, default=262144, help="series per workload")
    ap.add_argument("--out", default=None, help="keep the two .npz files here")
    ap.add_argument("--produce", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.produce:
        produce(args.produce, args.n)
        return
    out_dir = args.out or tempfile.mkdtemp(prefix="mmf_cmp_")
    os.makedirs(out_dir, exist_ok=True)
    files = []
    for tag, lib in (("a", args.lib_a), ("b", args.lib_b)):
        path = os.path.join(out_dir, f"outputs_{tag}.npz")
        env = dict(os.environ, MMF_LIB=os.path.abspath(lib))
        subprocess.run([sys.executable, os.path.abspath(__file__), "--lib-a", lib, "--lib-b", lib, "--n", str(args.n),
                        "--produce", path], env=env, check=True)
        files.append(path)
    a, b = np.load(files[0]), np.load(files[1])
    bad = []
    for k in sorted(set(a.files) | set(b.files)):
        if k not in a.files or k not in b.files or not same_bits(a[k], b[k]):
            bad.append(k)
        print(f"{k:32s} {'DIFFERS' if k in bad else 'bit-identical'}", flush=True)
    if bad:
        sys.exit(f"{len(bad)} outputs differ between {args.lib_a} and {args.lib_b}: {', '.join(bad)}")
    print(f"all {len(a.files)} outputs bit-identical")


if __name__ == "__main__":
    main()
