#!/usr/bin/env python
"""Cost of injecting slices: iso3dfd radius 8 (fp32) at 1024^3, 20 steps, wall time of the whole call and a stream sync:

  none       run_solution(0, 19) without injecting
  x_plane    the same call with an `add` injector of the plane x = n/2 on every step (add_slice_injector)
  z_plane    the same with the plane z = n/2 (the unit-stride dim: one element per 32-byte sector)
  faces      `set` of the outer R = 8 planes of all six faces on every step (boundary replay)
  loop       the reference API loop injecting the z-plane: run_solution(t, t), get_elements_in_slice, add, set_elements_in_slice
  sources    the z-plane as n^2 on-grid sources of set_sources (the point kernel)

Rounds rotate the order of the forms; each form reports the median of its rounds and the spread (max - min).  z_plane, loop and
sources must leave the same checksum of p.  The card's name, power limit and max SM clock are read (never set) with nvidia-smi
in the same run.  Prints one JSON line per form and one summary line; --out also writes them to a file.
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
        q = "name,power.limit,clocks.max.sm,clocks.sm,temperature.gpu"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=20).stdout.strip()
    except Exception as e:        # nvidia-smi missing: the numbers stand without it
        return f"unavailable ({e})"


def fill(s):
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.fill_hash(t, SEED, var_salt("p", t), -1.0, 1.0)
    v.fill_hash(0, SEED, var_salt("v", 0), 0.05, 0.3)


def timed(s, fn):
    s.sync()
    t0 = time.perf_counter()
    fn()
    s.sync()
    return time.perf_counter() - t0


def frames_for(shape, rows, seed, scale=1e-3):
    return ((np.random.default_rng(seed).random((rows,) + tuple(shape), dtype=np.float32) - 0.5) * np.float32(scale))


def run_injectors(s, steps, injs):
    """injs: (first, last, frames, mode) each, added in order (frames uploaded here, not in the run)."""
    fill(s)
    s.clear_slice_injectors()
    for first, last, fr, mode in injs:
        s.add_slice_injector("p", first, last, 1, fr, mode=mode)
    dt = timed(s, lambda: s.run_solution(0, steps - 1))
    s.clear_slice_injectors()
    return dt, s.get_var("p").checksum(steps)


def run_loop(s, steps, n, zc, fr):
    fill(s)
    s.clear_slice_injectors()
    p = s.get_var("p")

    def loop():
        for t in range(steps):
            s.run_solution(t, t)
            f, l = [t + 1, 0, 0, zc], [t + 1, n[0] - 1, n[1] - 1, zc]
            box = p.get_elements_in_slice(f, l)
            p.set_elements_in_slice(np.ascontiguousarray(box + fr[t][:, :, None]), f, l)
    return timed(s, loop), p.checksum(steps)


def run_sources(s, steps, pts, amp):
    fill(s)
    s.clear_slice_injectors()
    s.set_sources("p", pts, 1, amp)                      # planned and uploaded here, not in the run
    dt = timed(s, lambda: s.run_solution(0, steps - 1))
    s.clear_points()
    return dt, s.get_var("p").checksum(steps)


def summary(times):
    ms = [x * 1e3 for x in times]
    return {"median_ms": round(statistics.median(ms), 3), "spread_ms": round(max(ms) - min(ms), 3), "rounds": len(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n, steps, R = (a.n,) * 3, a.steps, 8
    xc, zc = n[0] // 2, n[2] // 2
    hi = [m - 1 for m in n]
    state_before = gpu_state()
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec(n)
    s.prepare_solution(0)
    x_fr = frames_for((1, n[1], n[2]), steps, 1)
    z_fr = frames_for((n[0], n[1], 1), steps, 2)
    faces = []
    for d in range(3):
        for lo in (True, False):
            f, l = [0, 0, 0], list(hi)
            if lo:
                l[d] = R - 1
            else:
                f[d] = n[d] - R
            faces.append((f, l, frames_for([b - a + 1 for a, b in zip(f, l)], steps, 10 + len(faces), 1.0), "set"))
    pts = np.stack(np.meshgrid(np.arange(n[0]), np.arange(n[1]), [zc], indexing="ij"), -1).reshape(-1, 3)
    amp = z_fr.reshape(steps, -1).astype(np.float64)    # the same values as z_fr: float32 is exact in double
    run_injectors(s, 2, [([xc, 0, 0], [xc, hi[1], hi[2]], x_fr[:2], "add")])   # warm-up: module load, first sweeps and launches
    forms = {
        "none": lambda: run_injectors(s, steps, []),
        "x_plane": lambda: run_injectors(s, steps, [([xc, 0, 0], [xc, hi[1], hi[2]], x_fr, "add")]),
        "z_plane": lambda: run_injectors(s, steps, [([0, 0, zc], [hi[0], hi[1], zc], z_fr, "add")]),
        "faces": lambda: run_injectors(s, steps, faces),
        "loop": lambda: run_loop(s, steps, n, zc, z_fr[:, :, :, 0]),
        "sources": lambda: run_sources(s, steps, pts, amp),
    }
    order = list(forms)
    times = {k: [] for k in forms}
    cks = {}
    for r in range(a.rounds):
        for k in order[r % len(order):] + order[:r % len(order)]:
            dt, ck = forms[k]()
            times[k].append(dt)
            cks.setdefault(k, set()).add(ck)
    s.close()
    checks = {
        "checksums_repeat": all(len(v) == 1 for v in cks.values()),
        "z_plane_loop_sources_agree": len(cks["z_plane"] | cks["loop"] | cks["sources"]) == 1,
        "injection_changes_p": cks["z_plane"] != cks["none"],
    }
    rows = []
    for k in order:
        row = {"form": k, "stencil": "iso3dfd", "radius": 8, "domain": n, "steps": steps, **summary(times[k])}
        rows.append(row)
        print(json.dumps(row), flush=True)
    med = {k: statistics.median(v) * 1e3 for k, v in times.items()}
    derived = {"step_ms": round(med["none"] / steps, 4),
               **{f"{k}_ms_per_step": round((med[k] - med["none"]) / steps, 4) for k in order if k != "none"}}
    env = {"checks": checks, "derived": derived, "gpu_before": state_before, "gpu_after": gpu_state()}
    print(json.dumps(env), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"rows": rows, **env}, f, indent=1)
    if not all(checks.values()):
        raise SystemExit("bench_slice_injectors: the forms disagree: " + json.dumps(checks))


if __name__ == "__main__":
    main()
