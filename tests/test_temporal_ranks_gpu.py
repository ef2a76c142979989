"""GPU: the iso3dfd temporal tile on rank grids (block_steps=2 with mega_block_steps=2, the reference's -bt 2 -Mbt 2): two steps per
launch on every rank, halos 2R deep exchanged once per pair.  Bit for bit against the CPU oracle over the GLOBAL domain:

  * grids split in x, y, z, two and three dims, unevenly; radius 1 and 2; every compiled form (tt_variant); every FP mode; even
    and odd step counts (the odd step takes the one-step path behind the last deep exchange); runs split over several calls;
    v rewritten between runs (v reaches the neighbours only through the deep exchange at the start of a run);
  * ranks that disagree on the mode are refused when they are connected; where there is no temporal tile (fp64, iso3dfd_sponge,
    radius 3) mega_block_steps changes nothing;
  * two processes over CUDA IPC, the command-line harness, one physical device per rank (with at least two devices).

Ranks live in this process (peers wired with raw pointers, multi.connect_local) unless stated; inputs are hash fields of global
indices on every rank, so each rank's halo cells hold what the oracle sees there."""
import functools
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from yask_b200 import capi, multi
from yask_b200.synth import hash_field, var_salt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 43
FUSED = {"block_steps": 2, "mega_block_steps": 2}
N = (22, 34, 70)         # 3 tiles in y (ragged), one ragged tile in z; every split below leaves ranks of at least 2R points


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def inputs(n, R, dtype=np.float32, seed=SEED):
    return ({("p", t): hash_field(seed, var_salt("p", t), (-R,) * 3, [i + 2 * R for i in n], -1, 1, dtype) for t in (0, 1)} |
            {("v", 0): hash_field(seed, var_salt("v", 0), (0, 0, 0), n, 0.05, 0.3, dtype)})


@functools.lru_cache(maxsize=None)
def _oracle(n, R, steps, mode):
    ins = inputs(n, R)
    return O.iso3dfd_run(ins[("p", 0)], ins[("p", 1)], ins[("v", 0)], R, steps, mode)


def oracle(n, R, steps, mode):
    return _oracle(tuple(n), R, steps, mode)[R:-R, R:-R, R:-R]


def grid_solutions(n, grid, R, fp_mode=2, opts=None, per_rank_opts=None, stencil="iso3dfd", eb=4):
    solns = []
    for r in range(grid[0] * grid[1] * grid[2]):
        s = capi.Solution(stencil, radius=R, elem_bytes=eb)
        s.set_overall_domain_size_vec(n)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        s.set_option("fp_mode", fp_mode)
        for k, v in ((per_rank_opts[r] if per_rank_opts else opts) or {}).items():
            s.set_option(k, v)
        s.prepare_solution(0)
        solns.append(s)
    return solns


def fill(solns, seed=SEED):
    for s in solns:
        for var in s.get_vars():
            nm = var.get_name()
            if nm == "p":
                for t in (0, 1):
                    var.fill_hash(t, seed, var_salt("p", t), -1.0, 1.0)
            elif nm == "v":
                var.fill_hash(0, seed, var_salt("v", 0), 0.05, 0.3)
            else:                                   # iso3dfd_sponge's damping factors
                var.fill_hash(0, seed, var_salt(nm, 0), 0.9, 1.0)


def run_all(solns, runs):
    for first, last in runs:
        for s in solns:      # enqueue every rank before any waits: ranks wait for each other on the device
            s.run_solution(first, last)
    for s in solns:
        s.sync()


def gather(solns, n, dtype=np.float32):
    out = np.full(n, np.nan, dtype)
    for s in solns:
        p = s.get_var("p")
        f, l = p.domain_box(p.get_last_valid_step_index())
        out[f[1]:l[1] + 1, f[2]:l[2] + 1, f[3]:l[3] + 1] = p.get_elements_in_slice(f, l)
    return out


def run_grid(n, grid, R, steps, fp_mode=2, opts=FUSED, runs=None, **kw):
    """Global p after the run, and per rank (kernel launches, tt_launches)."""
    solns = grid_solutions(n, grid, R, fp_mode, opts, **kw)
    multi.connect_local(solns)
    fill(solns)
    run_all(solns, runs or [(0, steps - 1)])
    out = gather(solns, n, np.float32 if kw.get("eb", 4) == 4 else np.float64)
    counts = [(s.get_stats().kernel_launches, int(s.get_option("tt_launches"))) for s in solns]
    for s in solns:
        s.close()
    return out, counts


GRIDS = [(2, 1, 1), (1, 2, 1), (1, 1, 2), (2, 2, 1), (2, 2, 2), (3, 1, 1)]


@pytest.mark.parametrize("variant", [0, 1, 2, 3])
@pytest.mark.parametrize("R", [1, 2])
@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: "x".join(map(str, g)))
def test_fused_pairs_bit_exact(grid, R, variant):
    steps = 4
    got, counts = run_grid(N, grid, R, steps, opts=dict(FUSED, tt_variant=variant))
    assert np.array_equal(_bits(got), _bits(oracle(N, R, steps, 2)))
    assert [c[1] for c in counts] == [steps // 2] * len(counts)


@pytest.mark.parametrize("fp_mode", [0, 1])
@pytest.mark.parametrize("R", [1, 2])
@pytest.mark.parametrize("gi", range(len(GRIDS)), ids=["x".join(map(str, g)) for g in GRIDS])
def test_fused_pairs_fp_modes_odd_steps(gi, R, fp_mode):
    steps = 5         # two pairs and one one-step launch
    got, counts = run_grid(N, GRIDS[gi], R, steps, fp_mode, opts=dict(FUSED, tt_variant=gi % 4))
    assert np.array_equal(_bits(got), _bits(oracle(N, R, steps, fp_mode)))
    assert [c[1] for c in counts] == [2] * len(counts)


@pytest.mark.parametrize("R", [1, 2])
@pytest.mark.parametrize("grid", [(2, 1, 1), (2, 2, 1)], ids=lambda g: "x".join(map(str, g)))
def test_runs_split_over_calls(grid, R):
    got, counts = run_grid(N, grid, R, 7, runs=[(0, 1), (2, 2), (3, 6)])
    assert np.array_equal(_bits(got), _bits(oracle(N, R, 7, 2)))
    assert [c[1] for c in counts] == [1 + 0 + 2] * len(counts)


@pytest.mark.parametrize("R", [1, 2])
def test_v_rewritten_between_runs(R):
    """v changes between two runs on every rank: the second run must see the new v in its neighbours' halos too."""
    grid, seed2 = (2, 2, 1), 91
    solns = grid_solutions(N, grid, R, 2, FUSED)
    multi.connect_local(solns)
    fill(solns)
    run_all(solns, [(0, 3)])
    for s in solns:
        s.get_var("v").fill_hash(0, seed2, var_salt("v", 0), 0.05, 0.3)
    run_all(solns, [(4, 7)])
    got = gather(solns, N)
    for s in solns:
        assert s.get_option("tt_launches") == "4"
        s.close()
    ins = inputs(N, R)
    p3 = O.iso3dfd_run(ins[("p", 0)], ins[("p", 1)], ins[("v", 0)], R, 3, 2)
    p4 = O.iso3dfd_run(ins[("p", 0)], ins[("p", 1)], ins[("v", 0)], R, 4, 2)
    v2 = hash_field(seed2, var_salt("v", 0), (0, 0, 0), N, 0.05, 0.3)
    ref = O.iso3dfd_run(p4, p3, v2, R, 4, 2)[R:-R, R:-R, R:-R]
    assert np.array_equal(_bits(got), _bits(ref))


def test_mismatched_ranks_are_refused():
    """One rank asks for fused pairs, its neighbour does not: connecting them fails with both ranks named, before any launch."""
    R, grid = 1, (2, 1, 1)
    solns = grid_solutions(N, grid, R, per_rank_opts=[FUSED, {"block_steps": 2}])
    with pytest.raises(capi.YaskError) as e:
        multi.connect_local(solns)
    msg = str(e.value)
    assert "rank 0" in msg and "rank 1" in msg, msg
    for s in solns:
        assert s.get_stats().kernel_launches == 0 and s.get_option("tt_launches") == "0"
        s.close()


@pytest.mark.parametrize("stencil,R,eb", [("iso3dfd", 2, 8), ("iso3dfd_sponge", 2, 4), ("iso3dfd", 3, 4)], ids=["fp64", "sponge", "radius3"])
def test_inert_where_no_tile_exists(stencil, R, eb):
    n, grid, steps = (26, 20, 72), (2, 1, 1), 5
    a, ca = run_grid(n, grid, R, steps, opts=FUSED, stencil=stencil, eb=eb)
    b, cb = run_grid(n, grid, R, steps, opts={"block_steps": 2}, stencil=stencil, eb=eb)
    assert np.array_equal(_bits(a), _bits(b))
    assert ca == cb and all(c[1] == 0 for c in ca)


def test_block_steps_after_prepare_does_not_switch_the_path():
    R, grid, steps = 1, (2, 1, 1), 4
    solns = grid_solutions(N, grid, R, 2, FUSED)
    multi.connect_local(solns)
    for s in solns:
        s.set_option("block_steps", 1)
        s.set_option("mega_block_steps", 1)
    fill(solns)
    run_all(solns, [(0, steps - 1)])
    got = gather(solns, N)
    for s in solns:
        assert s.get_option("tt_launches") == "2"
        s.close()
    assert np.array_equal(_bits(got), _bits(oracle(N, R, steps, 2)))


# ---- processes --------------------------------------------------------------------------------------------------------------

def _single_rank(n, R, steps, seed):
    s = capi.Solution("iso3dfd", radius=R)
    s.set_overall_domain_size_vec(n)
    s.prepare_solution(0)
    fill([s], seed)
    s.run_solution(0, steps - 1)
    out = gather([s], n)
    s.close()
    return out


def _ipc_worker(rank, world, n, R, steps, seed, port, q, one_device_per_rank=False):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    dev = rank if one_device_per_rank else rank % max(1, torch.cuda.device_count())
    s = capi.Solution("iso3dfd", radius=R)
    s.set_overall_domain_size_vec(n)
    s.set_num_ranks_vec([world, 1, 1])
    s.set_rank_index_vec([rank, 0, 0])
    for k, v in FUSED.items():
        s.set_option(k, v)
    s.prepare_solution(dev)
    multi.connect(s, dist, rank, world)
    fill([s], seed)
    dist.barrier()
    s.run_solution(0, steps - 1)
    s.sync()
    p = s.get_var("p")
    f, l = p.domain_box(p.get_last_valid_step_index())
    q.put((rank, f, l, p.get_elements_in_slice(f, l), s.get_option("tt_launches")))
    dist.barrier()
    s.close()
    dist.destroy_process_group()


def _run_processes(n, R, steps, world, port, one_device_per_rank):
    import torch.multiprocessing as mp
    seed = 23
    ref = _single_rank(n, R, steps, seed)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_ipc_worker, args=(r, world, n, R, steps, seed, port, q, one_device_per_rank)) for r in range(world)]
    for pr in procs:
        pr.start()
    out = np.zeros(n, np.float32)
    for _ in range(world):
        rank, f, l, a, tl = q.get(timeout=240)
        out[f[1]:l[1] + 1, f[2]:l[2] + 1, f[3]:l[3] + 1] = a
        assert tl == str(steps // 2)
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))


@pytest.mark.parametrize("R", [1, 2])
def test_two_processes_cuda_ipc(R):
    _run_processes((96, 32, 64), R, 5, 2, 29571 + R, False)


def test_one_physical_device_per_rank():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs 2 CUDA devices, found {torch.cuda.device_count()}")
    _run_processes((192, 64, 256), 2, 6, 2, 29575, True)


@pytest.mark.parametrize("R", [1, 2])
def test_harness_two_ranks_fused_pairs(R):
    """The reference's command line: -nrx 2 -bt 2 -Mbt 2, one process per rank; -validate passes and the report shows the
    wave-front steps."""
    from tests.test_cpp_api import _run_ranks
    exe = os.path.join(ROOT, "yask_b200", "bin", f"yask_kernel.iso3dfd_r{R}.b200.exe")
    if not os.path.exists(exe):
        pytest.skip("harness not built")
    outs = _run_ranks(exe, ["-g", "96", "-nrx", "2", "-bt", "2", "-Mbt", "2", "-validate"], 2, 29581 + R)
    for rc, o, e in outs:
        assert rc == 0, o[-2000:] + e[-2000:]
    assert "TEST PASSED" in outs[0][1], outs[0][1][-2000:]
    assert [l for l in outs[0][1].splitlines() if "num-wave-front-steps" in l][0].split()[-1] == "2"
