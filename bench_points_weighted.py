#!/usr/bin/env python
"""Cost of weighted (between-grid-point) receivers: iso3dfd radius 8 (fp32) at 1024^3, 20 steps, one run_solution(0, 19) call:

  none         no points
  trilinear M  1 trilinear source at the centre plus M = 1, 1024, 1 048 576 trilinear receivers on the plane z = 511.5
               (set_sources_weighted / set_receivers_weighted, 8 support entries each)
  on-grid M    1 on-grid source plus the same counts of on-grid receivers on the plane z = 511 (set_sources / set_receivers)

Rounds alternate the forms (each round starts one form later); each form reports the median wall time of its rounds (host clock
around the call and a stream sync) and the spread (max - min).  Power limit and clocks are read (never set) with nvidia-smi.
Prints one JSON line per row; --out also writes them to a file.
"""
import argparse
import json
import statistics
import subprocess
import time

import numpy as np

from yask_b200 import capi
from yask_b200.synth import var_salt

SEED = 7


def gpu_state():
    try:
        q = "name,power.limit,power.draw,clocks.sm,clocks.mem,temperature.gpu"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=20).stdout.strip()
    except Exception as e:        # nvidia-smi missing: the numbers stand without it
        return f"unavailable ({e})"


def fill(s):
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.fill_hash(t, SEED, var_salt("p", t), -1.0, 1.0)
    v.fill_hash(0, SEED, var_salt("v", 0), 0.05, 0.3)


def plane(m, n, z, frac):
    """m receivers on a sqrt(m) x sqrt(m) lattice of the plane z, fractional (frac) or on grid points."""
    k = max(1, int(round(m ** 0.5)))
    assert k * k == m
    if frac:
        xs = np.linspace(0.25, n - 1.5, k) if k > 1 else np.array([n / 2 + 0.25])
    else:
        xs = np.linspace(0, n - 1, k).astype(np.int64) if k > 1 else np.array([n // 2])
    x, y = np.meshgrid(xs, xs, indexing="ij")
    return np.stack([x.ravel(), y.ravel(), np.full(m, z)], axis=1)


def timed(s, steps, setup):
    fill(s)
    s.clear_points()
    setup()
    s.sync()
    t0 = time.perf_counter()
    s.run_solution(0, steps - 1)
    s.sync()
    return time.perf_counter() - t0


def summary(times):
    ms = [x * 1e3 for x in times]
    return {"median_ms": round(statistics.median(ms), 3), "spread_ms": round(max(ms) - min(ms), 3), "n": len(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--receivers", default="1,1024,1048576")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n, steps = a.n, a.steps
    amp = np.random.default_rng(1).uniform(-1, 1, size=(steps, 1))
    sidx, sw = capi.trilinear([[n / 2 + 0.25, n / 2 + 0.5, n / 2 + 0.75]])
    src = [[n // 2, n // 2, n // 2]]
    state_before = gpu_state()
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec((n,) * 3)
    s.prepare_solution(0)
    timed(s, 4, lambda: None)              # warm-up: module load, first sweep
    rows = []
    for m in [int(x) for x in a.receivers.split(",")]:
        ridx, rw = capi.trilinear(plane(m, n, n / 2 - 0.5, True))
        gpts = plane(m, n, n // 2 - 1, False).astype(np.int64)

        def weighted():
            s.set_sources_weighted("p", sidx, sw, 1, amp)
            s.set_receivers_weighted("p", ridx, rw, 1, steps)

        def on_grid():
            s.set_sources("p", src, 1, amp)
            s.set_receivers("p", gpts, 1, steps)

        forms = {"none": lambda: None, "trilinear": weighted, "on_grid": on_grid}
        order = list(forms)
        times = {k: [] for k in forms}
        timed(s, 2, weighted)               # warm-up of this size's tables and kernels
        timed(s, 2, on_grid)
        for r in range(a.rounds):
            for k in order[r % 3:] + order[:r % 3]:
                times[k].append(timed(s, steps, forms[k]))
        launches = int(s.get_option("point_launches"))
        row = {"stencil": "iso3dfd", "radius": 8, "n": [n] * 3, "steps": steps, "sources": 1, "receivers": m,
               **{k: summary(v) for k, v in times.items()},
               "trilinear_minus_none_per_step_ms": round((statistics.median(times["trilinear"]) - statistics.median(times["none"])) * 1e3 / steps, 4),
               "on_grid_minus_none_per_step_ms": round((statistics.median(times["on_grid"]) - statistics.median(times["none"])) * 1e3 / steps, 4),
               "point_launches": launches}
        rows.append(row)
        print(json.dumps(row), flush=True)
    s.close()
    env = {"gpu_before": state_before, "gpu_after": gpu_state()}
    print(json.dumps(env), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"rows": rows, **env}, f, indent=1)


if __name__ == "__main__":
    main()
