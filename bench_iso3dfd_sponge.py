"""iso3dfd_sponge on one GPU at 1024^3 against plain iso3dfd at the same radius, timed with CUDA events (through the engine's own
stats) in alternating rounds; the median of the rounds is reported.

  fp32: the hand-written sponge sweep at radius 1-7 and plain iso3dfd at the same radii, plus the generated sponge at radius 8;
  fp64: the hand-written sponge sweep at radius 1, 2, 3, 4, 5, 7 and 8 and plain fp64 iso3dfd at the same radii (generated at 3
        and 8), plus the generated sponge at radius 6.

Reports ms/step, GPoints/s and the sponge's time relative to plain iso3dfd.  The sponge adds three 1-D vars and three multiplies
per point and no full-size stream, so both move 4 elements per point-step.  Records the card's name and power limit in the same
run (read-only).  Prints one JSON line.

    python bench_iso3dfd_sponge.py [--size 1024] [--steps 10] [--warmup 3] [--rounds 3] [--prec fp32,fp64]
"""
import argparse
import json
import subprocess

import numpy as np

from yask_b200 import capi
from yask_b200.synth import var_salt

RADII = {4: (1, 2, 3, 4, 5, 6, 7), 8: (1, 2, 3, 4, 5, 7, 8)}
GENERATED_SPONGE = {4: 8, 8: 6}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def make(name, n, R, eb):
    s = capi.Solution(name, radius=R, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    s.prepare_solution(0)
    assert s.get_element_bytes() == eb
    p = s.get_var("p")
    for t in (0, 1):
        p.fill_hash(t, 7, var_salt("p", t), -1.0, 1.0)
    s.get_var("v").fill_hash(0, 7, var_salt("v", 0), 0.05, 0.3)
    if name == "iso3dfd_sponge":
        for c in ("cr_x", "cr_y", "cr_z"):
            s.get_var(c).fill_hash(0, 7, var_salt(c, 0), 0.92, 1.0)
    return s


def timed(s, steps, warmup):
    s.run_solution(0, warmup - 1)
    s.sync()
    s.clear_stats()
    s.run_solution(warmup, warmup + steps - 1)
    s.sync()
    st = s.get_stats()
    return st.elapsed_secs * 1e3 / st.num_steps_done


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--prec", default="fp32,fp64")
    args = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_iso3dfd_sponge.py: no CUDA device")
    n = (args.size,) * 3
    pts = float(args.size) ** 3
    info = card()
    ebs = [4 if p == "fp32" else 8 for p in args.prec.split(",")]
    runs = []      # (solution name, radius, element bytes)
    for eb in ebs:
        for R in RADII[eb]:
            runs += [("iso3dfd_sponge", R, eb), ("iso3dfd", R, eb)]
        runs.append(("iso3dfd_sponge", GENERATED_SPONGE[eb], eb))
    times = {r: [] for r in runs}
    for rnd in range(args.rounds):          # alternate: every case once per round, the order reversed every other round
        for r in (runs if rnd % 2 == 0 else runs[::-1]):
            s = make(r[0], n, r[1], r[2])
            times[r].append(timed(s, args.steps, args.warmup))
            s.close()
    med = {r: float(np.median(t)) for r, t in times.items()}
    rows = []
    for (name, R, eb) in runs:
        ms = med[(name, R, eb)]
        hand = not (name == "iso3dfd_sponge" and R == GENERATED_SPONGE[eb]) and not (name == "iso3dfd" and eb == 8 and R in (3, 8))
        row = dict(solution=name, radius=R, precision="fp32" if eb == 4 else "fp64", kernel="hand-written sweep" if hand else "generated",
                   ms_per_step=round(ms, 4), ms_all=[round(x, 4) for x in times[(name, R, eb)]],
                   gpoints_per_s=round(pts / (ms * 1e-3) / 1e9, 3))
        if name == "iso3dfd_sponge" and ("iso3dfd", R, eb) in med:
            row["vs_plain"] = round(ms / med[("iso3dfd", R, eb)], 4)
        rows.append(row)
    print(json.dumps(dict(bench="iso3dfd_sponge", size=list(n), steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                          card=info, results=rows)))


if __name__ == "__main__":
    main()
