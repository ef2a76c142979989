"""Single-precision iso3dfd sweep on one GPU at 1024^3: every radius 1-8 on its default sweep kernel, the radius-8 memory probe
(`mem_probe=1`: the same TMA loads and stores as the sweep, no stencil arithmetic) and the radius-8 tile shapes (7: 16x128,
6: 32x64) in both forms (`resident=1`: each p(t) plane loaded once; `resident=0`: twice), set against a
plain 16 B/point stream (torch.addcmul over four 1024^3 fp32 tensors: three reads, one write) timed on the same card in the same
run.  The stream is the ceiling the card and its power limit allow at that moment; a sweep whose memory probe is as slow as the
sweep itself is limited by its access pattern, one whose probe is much faster by the SMs.

Times are CUDA events (the engine's own stats for the sweeps), one step per launch, in alternating rounds; the median is
reported with the spread.  Shares are over the H100 SXM data sheet's 3.35 TB/s at 16 bytes per point-step (read p(t), p(t-1),
v; write p(t+1)).  Records the card's name and power limit in the same run.  Prints one JSON line.

    python bench_iso3dfd_sweep.py [--size 1024] [--steps 20] [--warmup 3] [--rounds 3]
"""
import argparse
import json
import subprocess

import numpy as np

from yask_b200 import capi
from yask_b200.synth import var_salt

PEAK_BPS = 3.35e12
BYTES_PER_POINT = 16

# (label, radius, engine options)
CONFIGS = [(f"r{r} default", r, {}) for r in range(1, 9)] + [
    (f"r8 tile={tile} resident={res}{' mem_probe' if probe else ''}", 8, {"tile": tile, "resident": res, "mem_probe": probe})
    for tile in (7, 6) for res in (1, 0) for probe in (0, 1)
]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def sweep_ms(n, R, opts, steps, warmup):
    s = capi.Solution("iso3dfd", radius=R)
    s.set_overall_domain_size_vec(n)
    for k, v in opts.items():
        s.set_option(k, v)
    s.prepare_solution(0)
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.fill_hash(t, 7, var_salt("p", t), -1.0, 1.0)
    v.fill_hash(0, 7, var_salt("v", 0), 0.05, 0.3)
    s.run_solution(0, warmup - 1)
    s.sync()
    s.clear_stats()
    s.run_solution(warmup, warmup + steps - 1)
    s.sync()
    st = s.get_stats()
    s.close()
    return st.elapsed_secs * 1e3 / st.num_steps_done


def stream_ms(n, steps, warmup):
    import torch
    a, b, c, d = (torch.rand(n, device="cuda") for _ in range(4))
    for _ in range(warmup):
        torch.addcmul(a, b, c, out=d)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        torch.addcmul(a, b, c, out=d)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del a, b, c, d
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_iso3dfd_sweep.py: no CUDA device")
    n = (args.size,) * 3
    pts = float(args.size) ** 3
    info = card()
    times = {lab: [] for lab, _, _ in CONFIGS}
    times["stream"] = []
    for rnd in range(args.rounds):          # alternate: every configuration once per round, the order reversed every other round
        order = CONFIGS if rnd % 2 == 0 else CONFIGS[::-1]
        times["stream"].append(stream_ms(n, args.steps, args.warmup))
        for lab, R, opts in order:
            times[lab].append(sweep_ms(n, R, opts, args.steps, args.warmup))
    rows = []
    for lab, ms_all in times.items():
        ms = float(np.median(ms_all))
        rows.append(dict(config=lab, ms_per_step=round(ms, 4), ms_all=[round(x, 4) for x in ms_all],
                         spread_ms=round(max(ms_all) - min(ms_all), 4),
                         gpoints_per_s=round(pts / (ms * 1e-3) / 1e9, 2),
                         hbm_share=round(pts * BYTES_PER_POINT / (ms * 1e-3) / PEAK_BPS, 4)))
    print(json.dumps(dict(bench="iso3dfd_sweep_fp32", size=list(n), steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                          card=info, bytes_per_point_step=BYTES_PER_POINT, peak_bytes_per_s=PEAK_BPS, results=rows)))


if __name__ == "__main__":
    main()
