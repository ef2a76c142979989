#!/usr/bin/env python
"""Time the average-of-points stencils (3axis, 3axis_with_diags, 3plane, cube) on one GPU: every shape at radius 1, 2, 4 and 8 in
fp32 and fp64 on the hand-written sweep, and the emitter-generated fp32 forms at their default radii (3axis and 3axis_with_diags
4, 3plane 3, cube 2).  Rounds alternate over the configurations; the median of the rounds is shown.

Each line states the roof it is measured against: the larger of
  * HBM: one read and one write per point-step (8 B in fp32, 16 B in fp64) over 3.35 TB/s, the H100 SXM data-sheet figure;
  * adds: pts - 1 additions and one multiply per point over the device's FP32 (128 per SM per clock) or FP64 (64 per SM per clock)
    issue rate at its maximum SM clock, as read from the device.
The fraction is roof time over measured time.  Output: one line per configuration and a JSON summary line.

usage: python bench_avepts.py [--n 1024] [--steps 3] [--rounds 3] [--shapes 3axis,cube] [--radii 1,8] [--prec fp32,fp64]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from tests.avepts_oracle import DEFAULT_RADIUS, SHAPES, npoints  # noqa: E402
from yask_b200 import capi  # noqa: E402
from yask_b200.synth import var_salt  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clk = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return dict(name=name, power_limit_w=float(power), max_sm_clock_mhz=float(clk), sms=sms)


def time_config(shape, R, eb, n, steps):
    """ms per step over `steps` steps after one warm-up step (device synchronised around the timed window)."""
    s = capi.Solution(shape, radius=R, elem_bytes=eb)
    s.set_overall_domain_size_vec((n, n, n))
    s.prepare_solution(0)
    a = s.get_var("A")
    for t in (0, 1):
        a.fill_hash(t, 7, var_salt("A", t), -1.0, 1.0)
    s.run_solution(0, 0)
    s.sync()
    t0 = time.perf_counter()
    s.run_solution(1, steps)
    s.sync()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    s.close()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--radii", default="1,2,4,8")
    ap.add_argument("--prec", default="fp32,fp64")
    args = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_avepts.py: no CUDA device")
    dev = device_info()
    shapes = args.shapes.split(",")
    cfgs = []
    for shape in shapes:
        cfgs.append((shape, DEFAULT_RADIUS[shape], 4, "generated"))
        for prec in args.prec.split(","):
            eb = 4 if prec == "fp32" else 8
            for R in map(int, args.radii.split(",")):
                if eb == 4 and R == DEFAULT_RADIUS[shape]:
                    continue        # served by the generated form (timed above)
                cfgs.append((shape, R, eb, "hand-written"))
    times = {c: [] for c in cfgs}
    for _ in range(args.rounds):
        for c in cfgs:
            times[c].append(time_config(c[0], c[1], c[2], args.n, args.steps))
    print(f"# {dev['name']}, power limit {dev['power_limit_w']:.0f} W, max SM clock {dev['max_sm_clock_mhz']:.0f} MHz, {dev['sms']} SMs; "
          f"{args.n}^3, {args.steps} steps per round, median of {args.rounds} rounds")
    rows = []
    pts = args.n ** 3
    for c in cfgs:
        shape, R, eb, form = c
        ms = statistics.median(times[c])
        npt = npoints(shape, R)
        hbm_ms = pts * 2 * eb / HBM_BYTES_PER_S * 1e3
        add_rate = dev["sms"] * dev["max_sm_clock_mhz"] * 1e6 * (128 if eb == 4 else 64)
        add_ms = pts * npt / add_rate * 1e3
        roof, roof_ms = ("HBM", hbm_ms) if hbm_ms >= add_ms else (("FP32" if eb == 4 else "FP64") + " add", add_ms)
        row = dict(shape=shape, radius=R, prec="fp32" if eb == 4 else "fp64", form=form, points=npt, ms_per_step=round(ms, 3),
                   gpts_per_s=round(pts / ms / 1e6, 2), roof=roof, roof_ms=round(roof_ms, 3), of_roof=round(roof_ms / ms, 3),
                   rounds=[round(x, 3) for x in times[c]])
        rows.append(row)
        print(f"{shape:17s} r{R} {row['prec']} {form:12s} {npt:5d} pts  {ms:10.3f} ms/step  {row['gpts_per_s']:8.2f} Gpts/s  "
              f"roof {roof:8s} {roof_ms:9.3f} ms  {row['of_roof'] * 100:5.1f} % of roof")
    print(json.dumps(dict(device=dev, n=args.n, steps=args.steps, rounds=args.rounds, results=rows)))


if __name__ == "__main__":
    main()
