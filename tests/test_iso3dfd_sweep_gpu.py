"""GPU: control paths of the iso3dfd sweep kernels (yask_b200/csrc/yb_iso3dfd.cuh) that the small oracle tests elsewhere do not
reach, bit for bit against the CPU oracle over the GLOBAL domain:

  A. persistent CTAs that sweep several work units each: the engine option `grid` caps the grid below the unit count, so the
     producer runs ahead across unit boundaries and the ring stage and mbarrier parity carry over from one unit to the next
     (fp32 radius 1-8 and every radius-8 tile, fp64 radius 1, 2, 4-7, the temporal tile); and, without the cap, more units
     than the device has SMs;
  B. rank grids (several ranks in this process, peers wired with raw pointers): the fused peer stores and the in-kernel
     completion signal below radius 8 and at their size thresholds, split-path interiors that start off a 16-byte boundary
     in z, the exchange options, fp64 rank grids (hand-written and generated kernels), block_steps=2 on a rank grid and runs
     split over several run_solution() calls.

Inputs are hash fields of global indices (yask_b200.synth): numpy arrays loaded into one rank, or fill_hash on every rank of a
grid, so each rank's halo cells hold what the oracle sees there.
"""
import functools

import numpy as np
import pytest

from oracle import oracle as O
from yask_b200 import capi, multi
from yask_b200.synth import hash_field, var_salt

pytestmark = pytest.mark.gpu

SEED = 41
MAX_CHUNKS = 40     # ISO_MAX_CHUNKS / TT_MAX_CHUNKS: x chunks of one launch
GRIDS = [1, 2, 3, 7]
FP32_TILE = (16, 128)                      # (y, z) of the one compiled fp32 variant at radius 1-7 and of the temporal tile
FP64_TILE = (16, 64)
R8_TILES = {t: (32, 64) if t in (0, 2, 3, 6) else (16, 128) for t in range(8)}     # option `tile` at radius 8
FP64_RADII = (1, 2, 4, 5, 6, 7)            # the hand-written fp64 sweep; 3 and 8 are generated kernels


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def inputs(n, R, dtype):
    return {("p", t): hash_field(SEED, var_salt("p", t), (-R,) * 3, [i + 2 * R for i in n], -1, 1, dtype) for t in (0, 1)} | \
           {("v", 0): hash_field(SEED, var_salt("v", 0), (0, 0, 0), n, 0.05, 0.3, dtype)}


@functools.lru_cache(maxsize=None)
def _oracle(n, R, steps, mode, dtype):
    ins = inputs(n, R, np.dtype(dtype))
    return O.iso3dfd_run(ins[("p", 0)], ins[("p", 1)], ins[("v", 0)], R, steps, mode)[R:-R, R:-R, R:-R]


def oracle(n, R, steps, mode, dtype):
    return _oracle(tuple(n), R, steps, mode, np.dtype(dtype).name)


def make(n, R, dtype, fp_mode, opts):
    s = capi.Solution("iso3dfd", radius=R, elem_bytes=np.dtype(dtype).itemsize)
    s.set_overall_domain_size_vec(n)
    s.set_option("fp_mode", fp_mode)
    for k, v in opts.items():        # before prepare_solution(): block_steps sizes the storage
        s.set_option(k, v)
    return s


def result(s):
    p = s.get_var("p")
    return p.get_elements_in_slice(*p.domain_box(p.get_last_valid_step_index()))


def run_one(n, R, steps, dtype, fp_mode, opts):
    s = make(n, R, dtype, fp_mode, opts)
    s.prepare_solution(0)
    ins = inputs(n, R, dtype)
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.set_elements_in_slice(ins[("p", t)], *p.halo_box(t))
    v.set_elements_in_slice(ins[("v", 0)], *v.halo_box(0))
    s.run_solution(0, steps - 1)
    out = result(s)
    s.close()
    assert out.dtype == np.dtype(dtype)
    return out


def run_grid(n, grid, R, steps, dtype, fp_mode=2, opts=None, runs=None):
    """Every rank of `grid` in this process; `runs` = the (first, last) step ranges of successive run_solution() calls.
    Returns the global p after the last step and every rank's kernel launch count."""
    solns = []
    for r in range(grid[0] * grid[1] * grid[2]):
        s = make(n, R, dtype, fp_mode, opts or {})
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        s.prepare_solution(0)
        solns.append(s)
    multi.connect_local(solns)
    for s in solns:
        p, v = s.get_var("p"), s.get_var("v")
        for t in (0, 1):
            p.fill_hash(t, SEED, var_salt("p", t), -1.0, 1.0)
        v.fill_hash(0, SEED, var_salt("v", 0), 0.05, 0.3)
    for first, last in runs or [(0, steps - 1)]:
        for s in solns:      # enqueue every rank before any waits: ranks wait for each other on the device
            s.run_solution(first, last)
    for s in solns:
        s.sync()
    out = np.full(n, np.nan, dtype)
    launches = []
    for s in solns:
        p = s.get_var("p")
        f, l = p.domain_box(p.get_last_valid_step_index())
        out[f[1]:l[1] + 1, f[2]:l[2] + 1, f[3]:l[3] + 1] = p.get_elements_in_slice(f, l)
        launches.append(s.get_stats().kernel_launches)
        s.close()
    return out, launches


def check_grid(n, grid, R, steps, dtype, fp_mode=2, opts=None):
    got, _ = run_grid(n, grid, R, steps, dtype, fp_mode, opts)
    assert np.array_equal(_bits(got), _bits(oracle(n, R, steps, fp_mode, dtype)))


# ---- A. persistent CTAs ------------------------------------------------------------------------------------------------

def chunk_lengths(nx, lx):
    """The engine's x chunks of a single-rank launch with option lx: ceil(nx / lx) chunks (at most MAX_CHUNKS), lengths
    differing by at most one plane."""
    nc = max(1, min(-(-nx // lx), MAX_CHUNKS, nx))
    return [nx * (c + 1) // nc - nx * c // nc for c in range(nc)]


def units(n, tile, lx):
    return -(-n[1] // tile[0]) * -(-n[2] // tile[1]) * len(chunk_lengths(n[0], lx))


# Ragged in y and z (a partial last tile in both); the chunk length, and so the sweep length n_it = chunk + 2R, differs by one
# plane between the chunks of a launch (both parities), and changes with the grid cap: lx 5 -> chunks of 4/5 planes, 7 -> 5/6,
# 3 -> 2/3.  STAGES = 5 divides few of the resulting n_it.
A32 = (23, 37, 200)
A64 = (23, 37, 100)
LX = {1: 5, 2: 7, 3: 5, 7: 3}


def check_persistent(n, R, tile, steps, dtype, fp_mode, grid, opts):
    lx = LX[grid]
    assert units(n, tile, lx) > grid      # every CTA sweeps more than one unit
    got = run_one(n, R, steps, dtype, fp_mode, {"kernel": "tma", "lx": lx, "grid": grid} | opts)
    assert np.array_equal(_bits(got), _bits(oracle(n, R, steps, fp_mode, dtype))), (R, grid, fp_mode, opts)


def _modes(radii, mode1_radius):
    return [(R, m) for R in radii for m in (0, 2)] + [(mode1_radius, 1)]


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("R,fp_mode", _modes(range(1, 8), 3))
def test_persistent_ctas_fp32(R, fp_mode, grid):
    check_persistent(A32, R, FP32_TILE, 3, np.float32, fp_mode, grid, {})


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("fp_mode", [0, 2])
@pytest.mark.parametrize("tile", range(8))
def test_persistent_ctas_fp32_radius8_tiles(tile, fp_mode, grid):
    check_persistent(A32, 8, R8_TILES[tile], 3, np.float32, fp_mode, grid, {"tile": tile})


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("R,fp_mode", _modes(FP64_RADII, 4))
def test_persistent_ctas_fp64(R, fp_mode, grid):
    check_persistent(A64, R, FP64_TILE, 3, np.float64, fp_mode, grid, {})


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("steps,fp_mode", [(4, 2), (5, 0)])     # 5: two fused launches and one one-step sweep
@pytest.mark.parametrize("variant", [0, 1, 2, 3])
@pytest.mark.parametrize("R", [1, 2])
def test_persistent_ctas_temporal_tile(R, variant, steps, fp_mode, grid):
    check_persistent(A32, R, FP32_TILE, steps, np.float32, fp_mode, grid, {"block_steps": 2, "tt_variant": variant})


@pytest.mark.parametrize("dtype,R,n,tile", [(np.float32, 3, (80, 37, 200), FP32_TILE), (np.float64, 5, (80, 37, 100), FP64_TILE)])
def test_more_units_than_sms(dtype, R, n, tile):
    """No grid cap: 2-plane chunks make more units than the device has SMs, so the persistent grid itself wraps."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert units(n, tile, 2) > sms
    got = run_one(n, R, 3, dtype, 2, {"kernel": "tma", "lx": 2})
    assert np.array_equal(_bits(got), _bits(oracle(n, R, 3, 2, dtype)))


# ---- B. rank grids -------------------------------------------------------------------------------------------------------
# Ranks get ceil(n / ranks) planes, the last one the rest.  The x-face exchange of the fp32 sweep is fused into the sweep when a
# rank has nx >= 2R planes (peer stores) and signals the neighbours from the kernel when nx >= 4R; fp64 and every grid split
# elsewhere run the split path (exterior slabs, push, interior).

@pytest.mark.parametrize("nx_rank", ["4R+1", "3R", "2R-1"])     # peer stores + signal, peer stores only, split path
@pytest.mark.parametrize("R", range(1, 9))
def test_rank_grid_fp32_x_thresholds(R, nx_rank):
    nxr = {"4R+1": 4 * R + 1, "3R": 3 * R, "2R-1": 2 * R - 1}[nx_rank]
    check_grid((2 * nxr, 20, 72), (2, 1, 1), R, 3, np.float32)


# x3: nx = 12R+1 -> 4R+1, 4R+1, 4R-1 planes (the last rank peer-stores without signalling); z2: 35 planes per rank, so the upper
# rank's interior starts at z = R, off a 16-byte boundary unless R is a multiple of the vector width
LAYOUTS = {"x3_uneven": (lambda R: (12 * R + 1, 20, 72), (3, 1, 1), {}),
           "y2": (lambda R: (13, 37, 72), (1, 2, 1), {}),
           "z2": (lambda R: (13, 20, 70), (1, 1, 2), {}),
           "z2_tma": (lambda R: (13, 20, 70), (1, 1, 2), {"kernel": "tma"}),
           "y2z2": (lambda R: (13, 37, 70), (1, 2, 2), {}),
           "x2y2z2": (lambda R: (2 * (2 * R + 3), 24, 70), (2, 2, 2), {})}


@pytest.mark.parametrize("layout", ["x3_uneven", "y2", "z2", "z2_tma"])
@pytest.mark.parametrize("R", range(1, 9))
def test_rank_grid_fp32(R, layout):
    shape, grid, opts = LAYOUTS[layout]
    check_grid(shape(R), grid, R, 3, np.float32, opts=opts)


@pytest.mark.parametrize("R", [1, 3, 8])
def test_rank_grid_fp32_eight_ranks(R):
    shape, grid, opts = LAYOUTS["x2y2z2"]
    check_grid(shape(R), grid, R, 3, np.float32, opts=opts)


@pytest.mark.parametrize("opt", [{"dma_halo": 1}, {"fused_halo": 0}, {"overlap_comms": 0}], ids=["dma_halo", "no_fused_halo", "no_overlap"])
@pytest.mark.parametrize("R", [2, 5])
def test_rank_grid_fp32_exchange_options(R, opt):
    check_grid((12 * R + 5, 20, 72), (3, 1, 1), R, 3, np.float32, opts=opt)      # 4R+2, 4R+2, 4R+1 planes: all signal


def test_rank_grid_several_boundary_units_per_cta_before_the_signal():
    R, n = 4, (2 * (4 * 4 + 1), 37, 200)
    assert -(-n[1] // FP32_TILE[0]) * -(-n[2] // FP32_TILE[1]) > 3      # boundary units per rank (one x neighbour each)
    check_grid(n, (2, 1, 1), R, 3, np.float32, opts={"grid": 3})


@pytest.mark.parametrize("layout", ["x3_uneven", "z2", "z2_tma", "y2z2"])
@pytest.mark.parametrize("R", FP64_RADII)
def test_rank_grid_fp64(R, layout):
    shape, grid, opts = LAYOUTS[layout]
    check_grid(shape(R), grid, R, 3, np.float64, opts=opts)


def test_rank_grid_fp64_eight_ranks():
    shape, grid, opts = LAYOUTS["x2y2z2"]
    check_grid(shape(5), grid, 5, 3, np.float64, opts=opts)


@pytest.mark.parametrize("grid", [(2, 1, 1), (1, 1, 2)])
@pytest.mark.parametrize("R", [3, 8])
def test_rank_grid_fp64_generated(R, grid):
    n = (26, 20, 70) if grid[0] == 2 else (13, 20, 70)
    check_grid(n, grid, R, 3, np.float64)


@pytest.mark.parametrize("R", [1, 2])
def test_rank_grid_block_steps_2(R):
    """The temporal tile is a single-rank path: on a rank grid block_steps=2 keeps one launch per step and the same bits."""
    n, grid, steps = (2 * (4 * R + 1), 20, 72), (2, 1, 1), 5
    got, launches = run_grid(n, grid, R, steps, np.float32, opts={"block_steps": 2})
    _, one_step = run_grid(n, grid, R, steps, np.float32)
    assert np.array_equal(_bits(got), _bits(oracle(n, R, steps, 2, np.float32)))
    assert launches == one_step


@pytest.mark.parametrize("dtype,R,layout", [(np.float32, 3, "x3_uneven"), (np.float64, 5, "z2")])
def test_rank_grid_runs_split_over_calls(dtype, R, layout):
    shape, grid, opts = LAYOUTS[layout]
    n = shape(R)
    got, _ = run_grid(n, grid, R, 5, dtype, opts=opts, runs=[(0, 1), (2, 4)])
    assert np.array_equal(_bits(got), _bits(oracle(n, R, 5, 2, dtype)))
