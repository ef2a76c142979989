"""Double-precision iso3dfd on one GPU at 1024^3: the hand-written fp64 sweep at radius 1, 2, 4 and 7 and the emitter-generated
fp64 kernels at radius 3 and 8, timed with CUDA events (through the engine's own stats) in alternating rounds.

Reports ms/step, GPoints/s and the share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s) at 32 bytes per point-step
(read p(t), p(t-1), v; write p(t+1): four doubles).  Records the card's name and power limit in the same run, and checks that
the sweep and the direct kernel give the same bits at the timed size for every hand-kernel radius.  Prints one JSON line.

    python bench_iso3dfd_fp64.py [--size 1024] [--steps 20] [--warmup 3] [--rounds 3]
"""
import argparse
import json
import subprocess

import numpy as np

from yask_b200 import capi
from yask_b200.synth import var_salt

HAND = (1, 2, 4, 7)
GENERATED = (3, 8)
PEAK_BPS = 3.35e12
BYTES_PER_POINT = 32


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def make(n, R, opts=None):
    s = capi.Solution("iso3dfd", radius=R, elem_bytes=8)
    s.set_overall_domain_size_vec(n)
    for k, v in (opts or {}).items():
        s.set_option(k, v)
    s.prepare_solution(0)
    assert s.get_element_bytes() == 8
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.fill_hash(t, 7, var_salt("p", t), -1.0, 1.0)
    v.fill_hash(0, 7, var_salt("v", 0), 0.05, 0.3)
    return s


def timed(s, steps, warmup, t0):
    s.run_solution(t0, t0 + warmup - 1)
    s.sync()
    s.clear_stats()
    s.run_solution(t0 + warmup, t0 + warmup + steps - 1)
    s.sync()
    st = s.get_stats()
    return st.elapsed_secs * 1e3 / st.num_steps_done


def tma_equals_direct(n, R):
    outs = []
    for kernel in ("tma", "direct"):
        s = make(n, R, {"kernel": kernel})
        s.run_solution(0, 1)
        p = s.get_var("p")
        outs.append(p.get_elements_in_slice(*p.domain_box(p.get_last_valid_step_index())))
        s.close()
    return bool(np.array_equal(outs[0].view(np.uint64), outs[1].view(np.uint64)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_iso3dfd_fp64.py: no CUDA device")
    n = (args.size,) * 3
    pts = float(args.size) ** 3
    info = card()
    radii = sorted(HAND + GENERATED)
    times = {R: [] for R in radii}
    for rnd in range(args.rounds):          # alternate: every radius once per round
        for R in (radii if rnd % 2 == 0 else radii[::-1]):
            s = make(n, R)
            times[R].append(timed(s, args.steps, args.warmup, 0))
            s.close()
    rows = []
    for R in radii:
        ms = float(np.median(times[R]))
        rows.append(dict(radius=R, kernel="hand-written fp64 sweep" if R in HAND else "generated",
                         ms_per_step=round(ms, 4), ms_all=[round(x, 4) for x in times[R]],
                         gpoints_per_s=round(pts / (ms * 1e-3) / 1e9, 3),
                         hbm_share=round(pts * BYTES_PER_POINT / (ms * 1e-3) / PEAK_BPS, 4)))
    same = {R: tma_equals_direct(n, R) for R in HAND}
    print(json.dumps(dict(bench="iso3dfd_fp64", size=list(n), steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                          card=info, bytes_per_point_step=BYTES_PER_POINT, peak_bytes_per_s=PEAK_BPS, results=rows,
                          tma_equals_direct=same)))
    if not all(same.values()):
        raise SystemExit("tma and direct kernels differ")


if __name__ == "__main__":
    main()
