#!/usr/bin/env python
"""Cost of point sources and receivers: iso3dfd radius 8 (fp32) at 1024^3, 20 steps, 1 source and M = 1, 64, 1024 receivers:

  (a) device   one run_solution(0, 19) call with the point sets on the device (set_sources / set_receivers)
  (b) loop     the reference API loop: run_solution(t, t), add_to_element through a one-element slice, one one-element
               slice read per receiver
  (c) none     one run_solution(0, 19) call without points
  plus iso3dfd radius 2 with block_steps=2: (c) with two steps per sweep, and (a) with 1 source + 1 receiver, which runs one
  step per launch -- the cost of that fallback.

Rounds alternate the forms (a, b, c, then b, c, a, ...); each form reports the median wall time of its rounds (host clock
around the call and a stream sync) and the spread (max - min).  (a) and (b) must give the same traces and the same p checksum.
Power limit and clocks are read (never set) with nvidia-smi.  Prints one JSON line per row; --out also writes them to a file.
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


def run_device(s, steps, src, amp, rcv):
    fill(s)
    s.clear_points()
    s.set_sources("p", src, 1, amp)
    s.set_receivers("p", rcv, 1, steps)
    s.sync()
    t0 = time.perf_counter()
    s.run_solution(0, steps - 1)
    s.sync()
    dt = time.perf_counter() - t0
    return dt, s.get_traces()[0], s.get_var("p").checksum(steps)


def run_none(s, steps):
    fill(s)
    s.clear_points()
    s.sync()
    t0 = time.perf_counter()
    s.run_solution(0, steps - 1)
    s.sync()
    return time.perf_counter() - t0, None, s.get_var("p").checksum(steps)


def run_loop(s, steps, src, amp, rcv):
    fill(s)
    s.clear_points()
    s.sync()
    p = s.get_var("p")
    tr = np.zeros((steps, len(rcv)), np.float32)
    t0 = time.perf_counter()
    for t in range(steps):
        s.run_solution(t, t)
        u = t + 1
        for i, q in enumerate(src):
            idx = [u] + list(q)
            cur = p.get_elements_in_slice(idx, idx).reshape(-1)[0]
            p.set_elements_in_slice(np.array([np.float32(cur) + np.float32(amp[u - 1][i])], np.float32), idx, idx)
        for j, q in enumerate(rcv):
            idx = [u] + list(q)
            tr[t, j] = p.get_elements_in_slice(idx, idx).reshape(-1)[0]
    s.sync()
    return time.perf_counter() - t0, tr, p.checksum(steps)


def summary(times):
    ms = [x * 1e3 for x in times]
    return {"median_ms": round(statistics.median(ms), 3), "spread_ms": round(max(ms) - min(ms), 3), "n": len(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--receivers", default="1,64,1024")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n, steps = (a.n,) * 3, a.steps
    rng = np.random.default_rng(1)
    src = [[n[0] // 2, n[1] // 2, n[2] // 2]]
    amp = rng.uniform(-1, 1, size=(steps, 1))
    rows = []
    state_before = gpu_state()
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec(n)
    s.prepare_solution(0)
    run_none(s, 4)                         # warm-up: module load, first sweep
    for m in [int(x) for x in a.receivers.split(",")]:
        rcv = rng.integers(0, n, size=(m, 3)).tolist()
        forms = {"device": lambda: run_device(s, steps, src, amp, rcv), "loop": lambda: run_loop(s, steps, src, amp, rcv),
                 "none": lambda: run_none(s, steps)}
        order = list(forms)
        times = {k: [] for k in forms}
        res = {}
        for r in range(a.rounds):
            for k in order[r % 3:] + order[:r % 3]:
                dt, tr, ck = forms[k]()
                times[k].append(dt)
                res[k] = (tr, ck)
        same = (np.array_equal(res["device"][0].view(np.uint32), res["loop"][0].view(np.uint32)) and res["device"][1] == res["loop"][1])
        row = {"stencil": "iso3dfd", "radius": 8, "n": n, "steps": steps, "sources": 1, "receivers": m,
               **{k: summary(v) for k, v in times.items()}, "device_equals_loop": bool(same)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    s.close()
    # radius 2, two steps per sweep: the one-step fallback while points are set
    s = capi.Solution("iso3dfd", radius=2)
    s.set_overall_domain_size_vec(n)
    s.set_option("block_steps", 2)
    s.prepare_solution(0)
    run_none(s, 4)
    rcv = [[n[0] // 3, n[1] // 3, n[2] // 3]]
    times = {"pairs_none": [], "device_one_step": []}
    for r in range(a.rounds):
        for k in (("pairs_none", "device_one_step") if r % 2 == 0 else ("device_one_step", "pairs_none")):
            times[k].append((run_none(s, steps) if k == "pairs_none" else run_device(s, steps, src, amp, rcv))[0])
    row = {"stencil": "iso3dfd", "radius": 2, "block_steps": 2, "n": n, "steps": steps, "sources": 1, "receivers": 1,
           **{k: summary(v) for k, v in times.items()}, "tt_launches": int(s.get_option("tt_launches"))}
    s.close()
    rows.append(row)
    print(json.dumps(row), flush=True)
    env = {"gpu_before": state_before, "gpu_after": gpu_state()}
    print(json.dumps(env), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"rows": rows, **env}, f, indent=1)


if __name__ == "__main__":
    main()
