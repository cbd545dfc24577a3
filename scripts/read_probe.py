"""Runs the HBM read-pattern probe (csrc/tools/read_probe.cu, built by the package Makefile) and prints one JSON line:
per variant the median and min-max of the kernel time and of the read rate over the flagship's 4 * n * t_fit series
bytes, next to the card's name, power limit and SM clock (sampled while the probe runs).

    python scripts/read_probe.py [--rounds 7] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, "dss-ml-at-scale_b200", "read_probe")


def smi(fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, check=True).stdout
    return [s.strip() for s in out.strip().splitlines()[0].split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7, help="passes over all variants (each launch timed 5x)")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not os.path.exists(PROBE):
        sys.exit(f"{PROBE} is missing: build the package first (make -C dss-ml-at-scale_b200/csrc all)")
    name, power_limit, max_sm = smi("name,power.limit,clocks.max.sm")
    proc = subprocess.Popen([PROBE, str(args.rounds)], stdout=subprocess.PIPE, text=True)
    clocks = []
    while proc.poll() is None:          # SM clock under load, sampled through the run
        time.sleep(0.5)
        try:
            clocks.append(int(float(smi("clocks.sm")[0])))
        except (subprocess.CalledProcessError, ValueError):
            pass
    out = proc.stdout.read()
    if proc.returncode != 0:
        sys.exit(f"read_probe failed with exit code {proc.returncode}")
    runs, header = {}, ""
    for line in out.splitlines():
        if line.startswith("#"):
            header = line[1:].strip()
            continue
        v, ms, gbs = line.split()
        runs.setdefault(v, []).append((float(ms), float(gbs)))
    variants = {}
    for v, rs in runs.items():
        ms = [r[0] for r in rs]
        gbs = [r[1] for r in rs]
        variants[v] = {"ms_median": statistics.median(ms), "ms_min": min(ms), "ms_max": max(ms),
                       "GBps_median": statistics.median(gbs), "GBps_min": min(gbs), "GBps_max": max(gbs), "runs": len(rs)}
    p0 = variants["P0"]["ms_median"]
    for v in variants.values():
        v["speedup_vs_P0"] = p0 / v["ms_median"]
    line = {"probe": "read_probe", "gpu": name, "power_limit_W": float(power_limit), "sm_clock_max_MHz": int(float(max_sm)),
            "sm_clock_under_load_MHz": {"min": min(clocks), "median": statistics.median(clocks), "max": max(clocks)}
            if clocks else None,
            "setup": header, "variants": variants}
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
