#!/usr/bin/env python
"""Temporal tile on rank grids: iso3dfd fp32 at radius 1 and 2, n^3 global points, four runs on ONE device, same inputs:

  1x1x1 one step per sweep | 1x1x1 fused pairs (block_steps=2) | 2x1x1 one step per launch | 2x1x1 fused pairs (block_steps=2,
  mega_block_steps=2: halos 2R deep, exchanged once per pair)

The two ranks of a 2x1x1 grid live in this process on the same device (peers wired with raw pointers), so the exchange moves
data within one HBM; what the grid adds over one rank is the exchange and the split of the domain.  After a warm-up run, at least
three rounds alternate the four runs; each is timed with a host clock around run_solution() on every rank and a synchronise of
every rank.  With at least --gpus devices visible the fused 2x1x1 ... Nx1x1 grid also runs with one process per device.
Prints ONE JSON line: per radius and run the median ms/step, its spread (max - min over the rounds), GPts/s, tt_launches of rank 0,
and whether the checksums of the last two steps agree across all four runs; the card's name and power limit come with it."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from yask_b200 import capi, multi
from yask_b200.synth import var_salt

SEED = 7
RUNS = {"1x1x1_one_step": ((1, 1, 1), {}),
        "1x1x1_fused_pairs": ((1, 1, 1), {"block_steps": 2}),
        "2x1x1_one_step": ((2, 1, 1), {}),
        "2x1x1_fused_pairs": ((2, 1, 1), {"block_steps": 2, "mega_block_steps": 2})}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:
        return {"gpu": "unknown", "power_limit": "unknown", "error": repr(e)[:120]}


def fill(s):
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.fill_hash(t, SEED, var_salt("p", t), -1.0, 1.0)
    v.fill_hash(0, SEED, var_salt("v", 0), 0.05, 0.3)


def make(R, n, grid, opts, rank=0, device=0):
    s = capi.Solution("iso3dfd", radius=R)
    s.set_overall_domain_size_vec((n, n, n))
    s.set_num_ranks_vec(grid)
    s.set_rank_index_vec(multi.grid_coords(rank, grid))
    for k, v in opts.items():
        s.set_option(k, v)
    s.prepare_solution(device)
    return s


def timed(solns, first, last):
    t0 = time.perf_counter()
    for s in solns:
        s.run_solution(first, last)
    for s in solns:
        s.sync()
    return time.perf_counter() - t0


def checksums(solns):
    """Checksums of the last two steps over the global domain (per-point hashes of global indices: ranks add up)."""
    out = []
    for back in (0, 1):
        tot = 0
        for s in solns:
            p = s.get_var("p")
            tot = (tot + p.checksum(p.get_last_valid_step_index() - back)) % (1 << 64)
        out.append(str(tot))
    return out


def run(R, n, grid, opts, warm, steps):
    solns = [make(R, n, grid, opts, r) for r in range(grid[0] * grid[1] * grid[2])]
    try:
        if len(solns) > 1:
            multi.connect_local(solns)
        for s in solns:
            fill(s)
        timed(solns, 0, warm - 1)
        secs = timed(solns, warm, warm + steps - 1)
        return {"ms_per_step": secs * 1e3 / steps, "tt_launches": int(solns[0].get_option("tt_launches")), "checksums": checksums(solns)}
    finally:
        for s in solns:
            s.close()


def _proc_worker(rank, world, R, n, warm, steps, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    s = make(R, n, (world, 1, 1), RUNS["2x1x1_fused_pairs"][1], rank, rank)
    multi.connect(s, dist, rank, world)
    fill(s)
    s.run_solution(0, warm - 1)
    s.sync()
    dist.barrier()
    t0 = time.perf_counter()
    s.run_solution(warm, warm + steps - 1)
    s.sync()
    dist.barrier()
    secs = time.perf_counter() - t0
    q.put((rank, secs, s.get_option("tt_launches")))
    dist.barrier()
    s.close()
    dist.destroy_process_group()


def run_processes(R, n, world, warm, steps, port):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_proc_worker, args=(r, world, R, n, warm, steps, port, q)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for pr in procs:
        pr.join(timeout=120)
    secs = max(r[1] for r in res)
    ms = secs * 1e3 / steps
    return {"ms_per_step": round(ms, 4), "gpoints_per_s": round(n ** 3 / ms / 1e6, 2),
            "tt_launches": int([r[2] for r in res if r[0] == 0][0])}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--radii", default="1,2")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warm", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--gpus", type=int, default=2, help="also run Nx1x1 fused pairs with one process per device when N are visible")
    a = ap.parse_args()
    out = {"bench": "temporal_ranks", "n": a.n, "steps": a.steps, "rounds": max(3, a.rounds), **card(), "radii": {}}
    for R in [int(r) for r in a.radii.split(",")]:
        times = {k: [] for k in RUNS}
        last = {}
        for _ in range(max(3, a.rounds)):        # alternating rounds: drifts of clock or temperature hit every run alike
            for name, (grid, opts) in RUNS.items():
                r = run(R, a.n, grid, opts, a.warm, a.steps)
                times[name].append(r["ms_per_step"])
                last[name] = r
        res = {}
        for name in RUNS:
            med = statistics.median(times[name])
            res[name] = {"ms_per_step": round(med, 4), "spread_ms": round(max(times[name]) - min(times[name]), 4),
                         "gpoints_per_s": round(a.n ** 3 / med / 1e6, 2), "tt_launches": last[name]["tt_launches"]}
        res["checksums_equal"] = len({tuple(r["checksums"]) for r in last.values()}) == 1
        try:
            import torch
            ndev = torch.cuda.device_count()
        except Exception:
            ndev = 0
        if ndev >= a.gpus >= 2:
            try:
                res[f"{a.gpus}x1x1_fused_pairs_one_process_per_gpu"] = run_processes(R, a.n, a.gpus, a.warm, a.steps, 29600 + R)
            except Exception as e:
                res[f"{a.gpus}x1x1_fused_pairs_one_process_per_gpu"] = {"error": repr(e)[:200]}
        else:
            res[f"{a.gpus}x1x1_fused_pairs_one_process_per_gpu"] = "not measured"
        out["radii"][str(R)] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
