#!/usr/bin/env python
"""Benchmark of large domains: ms/step and GPoints/s of four solutions at 1024^3 and at the largest cube that fits the device.

`python bench_large_domain.py` records the card's name and power limit, then for each case and size prepares the solution,
fills every var with fill_hash, runs the warm-up steps and times `--steps` steps `--rounds` times (device time, CUDA events on
the launching stream).  It prints one JSON line per case and size (median ms/step and GPoints/s, with the spread over the rounds)
and a closing line with the card.  "max" is the largest cube whose vars, as plan_geometry() lays them out, fit the free device
memory less a margin; the same search over the device's total memory gives the largest cube the card can hold.

  iso3dfd_sponge  radius 8 fp32 (emitter-generated)
  3axis           fp32 (emitter-generated)
  iso3dfd_fp64    iso3dfd radius 8 fp64 (emitter-generated)
  iso3dfd         radius 8 fp32 (hand-written resident sweep)

`python bench_large_domain.py --plan-only [--budget-mib M]` needs no device: it prints, for the solutions of README's "Large
domains" table, the largest cube (square for 2-D) whose vars fit M MiB (default: an H100 80GB's 81,559 MiB) less the margin,
with plan_geometry() laying out the vars.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# name -> (solution, radius, elem_bytes)
CASES = {"iso3dfd_sponge": ("iso3dfd_sponge", 8, 4), "3axis": ("3axis", 0, 0), "iso3dfd_fp64": ("iso3dfd", 8, 8),
         "iso3dfd": ("iso3dfd", 8, 4)}
# fill_hash value ranges (tests/golden/ranges.py), by var-name prefix
RANGES = {"p": (-1.0, 1.0), "v": (0.05, 0.3), "cr": (0.92, 1.0), "A": (-1.0, 1.0)}
MARGIN = 2 << 30
# --plan-only: label -> (solution, radius, elem_bytes, domain dims)
PLAN = {"iso3dfd_sponge radius 8 fp32 (generated)": ("iso3dfd_sponge", 8, 4, 3), "iso3dfd radius 8 fp32 (hand-written)": ("iso3dfd", 8, 4, 3),
        "iso3dfd radius 3 fp64 (generated)": ("iso3dfd", 3, 8, 3), "iso3dfd radius 8 fp64 (generated)": ("iso3dfd", 8, 8, 3),
        "iso3dfd_sponge radius 6 fp64 (generated)": ("iso3dfd_sponge", 6, 8, 3), "3axis": ("3axis", 0, 0, 3),
        "3axis_with_diags": ("3axis_with_diags", 0, 0, 3), "3plane": ("3plane", 0, 0, 3), "cube": ("cube", 0, 0, 3),
        "test_2d": ("test_2d", 0, 0, 2), "wave2d": ("wave2d", 0, 0, 2), "swe2d": ("swe2d", 0, 0, 2),
        "box_filter": ("box_filter", 0, 0, 2), "gaussian_filter": ("gaussian_filter", 0, 0, 2)}


def card():
    """Name, power limit and maximum SM clock of device 0, read with the measurement."""
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm,memory.total",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout.strip()
        name, power, clk, mem = [f.strip() for f in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk, "memory_total": mem}
    except Exception as e:      # the timing below still runs; the record says why the card is unknown
        return {"name": None, "error": f"nvidia-smi: {e}"}


def solution(capi, case, n, table=CASES):
    stencil, radius, eb = table[case][:3]
    s = capi.Solution(stencil, radius=radius, elem_bytes=eb)
    s.set_overall_domain_size_vec((n,) * (table[case][3] if len(table[case]) > 3 else 3))
    return s


def plan(capi, case, n, table=CASES):
    """(bytes of all vars, largest slot in elements) of an n^d domain, as plan_geometry() lays it out."""
    s = solution(capi, case, n, table)
    s.plan_geometry()
    b = sum(v.info.storage_bytes for v in s.get_vars())
    m = max(v.info.slot_elems for v in s.get_vars())
    s.close()
    return b, m


def largest_cube(capi, case, budget, table=CASES):
    lo, hi = 64, 64
    while plan(capi, case, hi, table)[0] <= budget:
        lo, hi = hi, hi * 2
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if plan(capi, case, mid, table)[0] <= budget:
            lo = mid
        else:
            hi = mid
    return lo


def plan_only(capi, budget_mib):
    budget = budget_mib * 2 ** 20 - MARGIN
    print(f"largest domain within {budget_mib} MiB less a 2 GiB margin (plan_geometry)")
    print("| solution | largest domain | storage, GB | largest slot, x 2^31 elements |")
    print("|---|---|---|---|")
    for label, (_, _, _, nd) in PLAN.items():
        n = largest_cube(capi, label, budget, PLAN)
        b, m = plan(capi, label, n, PLAN)
        print(f"| {label} | {n}^{nd} | {b / 1e9:.1f} | {m / 2 ** 31:.2f} |")


def fill(s, seed=5):
    from yask_b200.synth import var_salt
    for var in s.get_vars():
        vi = var.info
        name = vi.name.decode()
        lo, hi = max(((k, r) for k, r in RANGES.items() if name.startswith(k)), key=lambda kr: len(kr[0]))[1]
        for t in (range(vi.step_alloc) if vi.has_step else [0]):
            var.fill_hash(t, seed, var_salt(name, t), lo, hi)


def time_case(capi, case, n, steps, warmup, rounds):
    s = solution(capi, case, n)
    s.prepare_solution(0)
    fill(s)
    s.run_solution(0, warmup - 1)
    t, ms = warmup, []
    for _ in range(rounds):
        s.clear_stats()
        s.run_solution(t, t + steps - 1)
        s.sync()
        ms.append(s.get_stats().elapsed_secs / steps * 1e3)
        t += steps
    vi = max((v.info for v in s.get_vars()), key=lambda i: i.slot_elems)
    need = sum(v.info.storage_bytes for v in s.get_vars())
    s.close()
    gpts = [n ** 3 / (m * 1e-3) / 1e9 for m in ms]
    return {"case": case, "n": n, "slot_elems": vi.slot_elems, "past_2_31": vi.slot_elems >= 1 << 31, "storage_gb": round(need / 1e9, 2),
            "ms_per_step": round(statistics.median(ms), 4), "ms_min": round(min(ms), 4), "ms_max": round(max(ms), 4),
            "gpoints_s": round(statistics.median(gpts), 3), "gpoints_s_min": round(min(gpts), 3), "gpoints_s_max": round(max(gpts), 3),
            "rounds": rounds, "steps": steps, "warmup": warmup}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=",".join(CASES), help="comma-separated subset of " + ", ".join(CASES))
    ap.add_argument("--sizes", default="1024,max", help="comma-separated cube edges; 'max' = largest cube that fits the free memory")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--plan-only", action="store_true", help="print the largest domains that fit --budget-mib (no device)")
    ap.add_argument("--budget-mib", type=int, default=81559)
    a = ap.parse_args()
    from yask_b200 import capi
    if a.plan_only:
        plan_only(capi, a.budget_mib)
        return
    import torch
    if capi.device_count() < 1:
        raise SystemExit("bench_large_domain.py: no CUDA device (the engine has no CPU fallback)")
    info = card()
    print(json.dumps({"card": info}), flush=True)
    for case in a.cases.split(","):
        _, total = torch.cuda.mem_get_info()
        print(json.dumps({"case": case, "largest_cube_of_card": largest_cube(capi, case, total - MARGIN),
                          "card_memory_gb": round(total / 1e9, 1)}), flush=True)
        for sz in a.sizes.split(","):
            if sz == "max":
                free, _ = torch.cuda.mem_get_info()
                n = largest_cube(capi, case, free - MARGIN)
            else:
                n = int(sz)
            r = time_case(capi, case, n, a.steps, a.warmup, a.rounds)
            r["card"] = info.get("name")
            r["power_limit"] = info.get("power_limit")
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
