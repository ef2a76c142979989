#!/usr/bin/env python
"""Cost of recording slices: iso3dfd radius 8 (fp32) at 1024^3, 20 steps, wall time of the whole call and a stream sync:

  none       run_solution(0, 19) without recording
  x_plane    the same call with a recorder of the plane x = n/2 on every step (add_slice)
  z_plane    the same with the plane z = n/2 (the unit-stride dim: one element per 32-byte sector)
  snapshot   the same with a (2,2,2)-decimated copy of the whole field every 5 steps
  loop       the reference API loop recording the z-plane: run_solution(t, t), then get_elements_in_slice of the plane
  receivers  the z-plane as n^2 receivers of set_receivers (the point kernel)

Rounds rotate the order of the forms; each form reports the median of its rounds and the spread (max - min).  The frames of
x_plane, z_plane, snapshot, loop and receivers must agree where they overlap, and every form must leave the same p checksum.
The card's name, power limit and max SM clock are read (never set) with nvidia-smi in the same run.  Prints one JSON line per
form and one summary line; --out also writes them to a file.
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


def run_recorder(s, steps, first, last, stride, t0, every, nrows):
    fill(s)
    s.clear_slices()
    rid = s.add_slice("p", first, last, t0, nrows, stride=stride, every=every)      # frames allocated here, not in the run
    dt = timed(s, lambda: s.run_solution(0, steps - 1))
    frames = s.get_slice_frames(rid)[0]
    s.clear_slices()
    return dt, frames, s.get_var("p").checksum(steps)


def run_none(s, steps):
    fill(s)
    s.clear_slices()
    return timed(s, lambda: s.run_solution(0, steps - 1)), None, s.get_var("p").checksum(steps)


def run_loop(s, steps, n, zc):
    fill(s)
    s.clear_slices()
    p = s.get_var("p")
    frames = np.zeros((steps, n[0], n[1]), np.float32)

    def loop():
        for t in range(steps):
            s.run_solution(t, t)
            frames[t] = p.get_elements_in_slice([t + 1, 0, 0, zc], [t + 1, n[0] - 1, n[1] - 1, zc])[:, :, 0]
    return timed(s, loop), frames, p.checksum(steps)


def run_receivers(s, steps, n, rcv):
    fill(s)
    s.clear_slices()
    s.set_receivers("p", rcv, 1, steps)                  # planned and uploaded here, not in the run
    dt = timed(s, lambda: s.run_solution(0, steps - 1))
    tr = s.get_traces()[0].reshape(steps, n[0], n[1])
    s.clear_points()
    return dt, tr, s.get_var("p").checksum(steps)


def summary(times):
    ms = [x * 1e3 for x in times]
    return {"median_ms": round(statistics.median(ms), 3), "spread_ms": round(max(ms) - min(ms), 3), "rounds": len(ms)}


def bits(a):
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n, steps = (a.n,) * 3, a.steps
    xc, zc = (n[0] // 2) & ~1, (n[2] // 2) & ~1          # even: on the (2,2,2) snapshot's lattice
    hi = [m - 1 for m in n]
    state_before = gpu_state()
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec(n)
    s.prepare_solution(0)
    run_none(s, 4)                                       # warm-up: module load, first sweeps, first recording launch
    run_recorder(s, 2, [xc, 0, 0], [xc, hi[1], hi[2]], None, 1, 1, 2)
    rcv = np.stack(np.meshgrid(np.arange(n[0]), np.arange(n[1]), [zc], indexing="ij"), -1).reshape(-1, 3)
    forms = {
        "none": lambda: run_none(s, steps),
        "x_plane": lambda: run_recorder(s, steps, [xc, 0, 0], [xc, hi[1], hi[2]], None, 1, 1, steps),
        "z_plane": lambda: run_recorder(s, steps, [0, 0, zc], [hi[0], hi[1], zc], None, 1, 1, steps),
        "snapshot": lambda: run_recorder(s, steps, [0, 0, 0], hi, [2, 2, 2], 5, 5, steps // 5),
        "loop": lambda: run_loop(s, steps, n, zc),
        "receivers": lambda: run_receivers(s, steps, n, rcv),
    }
    order = list(forms)
    times = {k: [] for k in forms}
    res = {}
    for r in range(a.rounds):
        for k in order[r % len(order):] + order[:r % len(order)]:
            dt, frames, ck = forms[k]()
            times[k].append(dt)
            res[k] = (frames, ck)
    s.close()
    z = res["z_plane"][0][:, :, :, 0]                    # (steps, nx, ny)
    snap = res["snapshot"][0]                            # rows at u = 5, 10, ...
    checks = {
        "checksums_equal": len({ck for _, ck in res.values()}) == 1,
        "loop_equals_z_plane": bool(np.array_equal(bits(res["loop"][0]), bits(z))),
        "receivers_equal_z_plane": bool(np.array_equal(bits(res["receivers"][0]), bits(z))),
        "x_plane_meets_z_plane": bool(np.array_equal(bits(np.ascontiguousarray(res["x_plane"][0][:, 0, :, zc])), bits(np.ascontiguousarray(z[:, xc, :])))),
        "snapshot_meets_z_plane": bool(all(np.array_equal(bits(np.ascontiguousarray(snap[r, :, :, zc // 2])),
                                                          bits(np.ascontiguousarray(z[5 * (r + 1) - 1, ::2, ::2])))
                                           for r in range(snap.shape[0]))),
    }
    rows = []
    for k in order:
        row = {"form": k, "stencil": "iso3dfd", "radius": 8, "domain": n, "steps": steps, **summary(times[k])}
        rows.append(row)
        print(json.dumps(row), flush=True)
    med = {k: statistics.median(v) * 1e3 for k, v in times.items()}
    derived = {"step_ms": round(med["none"] / steps, 4),
               **{f"{k}_ms_per_recorded_frame": round((med[k] - med["none"]) / (steps if k != "snapshot" else steps // 5), 4)
                  for k in ("x_plane", "z_plane", "snapshot", "loop", "receivers")},
               "receivers_over_z_plane": round(med["receivers"] / med["z_plane"], 3)}
    env = {"checks": checks, "derived": derived, "gpu_before": state_before, "gpu_after": gpu_state()}
    print(json.dumps(env), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"rows": rows, **env}, f, indent=1)
    if not all(checks.values()):
        raise SystemExit("bench_slices: the forms disagree: " + json.dumps(checks))


if __name__ == "__main__":
    main()
