#!/usr/bin/env python
"""Time the average-of-points temporal tile (option block_steps=2, the reference's -bt 2) against one step per sweep, on one GPU:
every entry that has a tile -- 3axis at radius 1 and 2, fp32 and fp64 -- at n^3 points, the same inputs on both paths.  (The
tiles of 3axis_with_diags at radius 1 and 2 and of 3plane and cube at radius 1 were measured with this file and were slower than
one step per sweep; they are not built, and block_steps=2 has no effect there.)

Per entry both solutions are prepared side by side and timed in alternating rounds (one step per sweep, then pairs), each round an
even number of steps after an even number of warm-up steps; the median and the spread (max - min) of the rounds are shown.  After
the rounds both paths have run the same steps, and the checksums of both valid steps must be equal.

Bytes per point-step: one step per sweep reads A(t) and writes A(t+1), 8 B in fp32 (16 in fp64); a pair reads A(t) and writes
A(t+2), 4 B per point-step (8 in fp64).  Each path's share of 3.35 TB/s (the H100 SXM data-sheet HBM figure) is at its own bytes.
Output: one line per entry and a JSON summary line, headed by the card, its power limit and its maximum SM clock.

usage: python bench_avepts_temporal.py [--n 1024] [--steps 10] [--warmup 2] [--rounds 3] [--prec fp32,fp64]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_avepts import HBM_BYTES_PER_S, device_info  # noqa: E402
from yask_b200 import capi  # noqa: E402
from yask_b200.synth import var_salt  # noqa: E402

TILED = [("3axis", 1), ("3axis", 2)]


def prepared(shape, R, eb, n, block_steps):
    s = capi.Solution(shape, radius=R, elem_bytes=eb)
    s.set_overall_domain_size_vec((n, n, n))
    s.set_option("block_steps", block_steps)
    s.prepare_solution(0)
    a = s.get_var("A")
    for t in (0, 1):
        a.fill_hash(t, 7, var_salt("A", t), -1.0, 1.0)
    return s


def timed(s, t0, steps):
    """ms per step of steps t0 .. t0 + steps - 1 (device synchronised around the window)."""
    s.sync()
    c0 = time.perf_counter()
    s.run_solution(t0, t0 + steps - 1)
    s.sync()
    return (time.perf_counter() - c0) * 1e3 / steps


def bench_entry(shape, R, eb, n, steps, warmup, rounds):
    solns = {"one": prepared(shape, R, eb, n, 1), "pairs": prepared(shape, R, eb, n, 2)}
    try:
        for s in solns.values():
            s.run_solution(0, warmup - 1)
        times = {k: [] for k in solns}
        t = warmup
        for _ in range(rounds):
            for k, s in solns.items():
                times[k].append(timed(s, t, steps))
            t += steps
        sums, tt = {}, {}
        for k, s in solns.items():
            a = s.get_var("A")
            tl = a.get_last_valid_step_index()
            sums[k] = [str(a.checksum(tl - 1)), str(a.checksum(tl))]
            tt[k] = int(s.get_option("tt_launches"))
    finally:
        for s in solns.values():
            s.close()
    return times, sums, tt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--prec", default="fp32,fp64")
    args = ap.parse_args()
    if args.steps % 2 or args.warmup % 2:
        raise SystemExit("bench_avepts_temporal.py: --steps and --warmup must be even (whole pairs)")
    if capi.device_count() < 1:
        raise SystemExit("bench_avepts_temporal.py: no CUDA device")
    dev = device_info()
    print(f"# {dev['name']}, power limit {dev['power_limit_w']:.0f} W, max SM clock {dev['max_sm_clock_mhz']:.0f} MHz, {dev['sms']} SMs; "
          f"{args.n}^3, {args.warmup} warm-up + {args.rounds} alternating rounds of {args.steps} steps; median (spread) of the rounds",
          flush=True)
    pts = args.n ** 3
    rows = []
    for prec in args.prec.split(","):
        eb = 4 if prec == "fp32" else 8
        for shape, R in TILED:
            times, sums, tt = bench_entry(shape, R, eb, args.n, args.steps, args.warmup, args.rounds)
            row = dict(shape=shape, radius=R, prec=prec, checksums_equal=sums["one"] == sums["pairs"],
                       fused_launches=tt["pairs"], checksums=sums["pairs"])
            for k, bpp in (("one", 2 * eb), ("pairs", eb)):
                ms = statistics.median(times[k])
                row[k] = dict(ms_per_step=round(ms, 4), spread_ms=round(max(times[k]) - min(times[k]), 4),
                              rounds=[round(x, 4) for x in times[k]], bytes_per_point_step=bpp,
                              of_hbm=round(pts * bpp / (ms * 1e-3) / HBM_BYTES_PER_S, 3))
            row["speedup"] = round(row["one"]["ms_per_step"] / row["pairs"]["ms_per_step"], 3)
            rows.append(row)
            o, p = row["one"], row["pairs"]
            print(f"{shape:17s} r{R} {prec}  one step per sweep {o['ms_per_step']:8.3f} ({o['spread_ms']:.3f}) ms/step "
                  f"{o['of_hbm'] * 100:5.1f} % HBM at {o['bytes_per_point_step']} B  |  pairs {p['ms_per_step']:8.3f} ({p['spread_ms']:.3f}) "
                  f"ms/step {p['of_hbm'] * 100:5.1f} % HBM at {p['bytes_per_point_step']} B  |  {row['speedup']:.2f}x  "
                  f"checksums {'equal' if row['checksums_equal'] else 'DIFFER'}", flush=True)
    print(json.dumps(dict(device=dev, n=args.n, steps=args.steps, warmup=args.warmup, rounds=args.rounds, results=rows)))
    if not all(r["checksums_equal"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
