"""GPU: control paths of the hand-written average-of-points engine (yask_b200/csrc/yb_avepts.cu, yb_avepts.cuh) that the small
oracle tests in test_avepts_gpu.py do not reach, bit for bit against the CPU oracle (tests/avepts_oracle.py), halo cells included:

  A. persistent CTAs that sweep several work units each (option `grid` below the unit count): ragged domains with a partial last
     y tile, z tile and vector; x chunks one plane apart in length, so the ring phase (2R+1+PF slots) carries over between units;
  B. thin and tiny domains on one rank under kernel=direct, auto (which must pick the direct kernel) and tma;
  C. rank grids at every radius (several ranks in this process): the whole form, the split form with x, y and z exterior slabs,
     rank sizes at R (the minimum), 2R-1 and just past 2R plus one 16-byte vector, no overlap, runs split over two calls;
  D. slots past 2^31 elements (three oracle windows, tests/large_domain.py);
  E. fp_mode 0, 1 and 2 give the same bits.

Every case asserts which kernel ran (the read-only option gen_sweep_launches counts the sweep launches) and how many launches
the run made.  The fp32 default radii (3axis 4, 3axis_with_diags 4, 3plane 3, cube 2) are the emitter-generated form, tested by
test_generated_matrix_gpu.py, and are left out here.
"""
import functools
import itertools

import numpy as np
import pytest

from tests import avepts_oracle as A
from tests.large_domain import TWO31, bits, storage_bytes, three_windows
from yask_b200 import capi, multi
from yask_b200.synth import hash_field, var_salt

pytestmark = pytest.mark.gpu

SEED = 53
GRIDS = [1, 2, 3, 7]
MAX_CHUNKS = 40                       # AVP_MAX_CHUNKS
TZ = {4: 64, 8: 32}                   # z points of a sweep tile (16 rows in y)
VW = {4: 4, 8: 2}                     # points per 16-byte vector
HAND = [(s, R, eb) for s in A.SHAPES for R in range(1, 9) for eb in (4, 8) if eb == 8 or R != A.DEFAULT_RADIUS[s]]


def _dt(eb):
    return np.float32 if eb == 4 else np.float64


def inputs(n, R, eb):
    return [hash_field(SEED, var_salt("A", t), (-R,) * 3, [i + 2 * R for i in n], -1, 1, _dt(eb)) for t in (0, 1)]


@functools.lru_cache(maxsize=None)
def oracle(n, shape, R, eb, steps):
    """A at step `steps` over the global domain and its halo."""
    ins = inputs(n, R, eb)
    return A.run(ins[0], ins[1], shape, R, steps)


def make(shape, n, R, eb, opts):
    s = capi.Solution(shape, radius=R, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    for k, v in opts.items():
        s.set_option(k, v)
    return s


def run_one(shape, n, R, eb, steps, opts):
    """One rank, inputs loaded with their halos; returns A with its halo, sweep launches and kernel launches."""
    s = make(shape, n, R, eb, opts)
    try:
        s.prepare_solution(0)
        a = s.get_var("A")
        for t, x in enumerate(inputs(n, R, eb)):
            a.set_elements_in_slice(x, *a.halo_box(t))
        s.run_solution(0, steps - 1)
        got = a.get_elements_in_slice(*a.halo_box(a.get_last_valid_step_index()))
        return got, int(s.get_option("gen_sweep_launches")), s.get_stats().kernel_launches
    finally:
        s.close()


def check_one(shape, n, R, eb, steps, opts, sweeps):
    got, sw, kl = run_one(shape, n, R, eb, steps, opts)
    assert got.dtype == _dt(eb)
    assert np.array_equal(bits(got), bits(oracle(tuple(n), shape, R, eb, steps))), (shape, n, R, eb, opts)
    assert (sw, kl) == (sweeps, steps), (shape, n, R, eb, opts, sw, kl)


# ---- A. persistent CTAs ------------------------------------------------------------------------------------------------------
# nx = 23: lx 5 -> chunks of 4/5 planes, 7 -> 5/6, 3 -> 2/3; 37 rows = 2 tiles + 5; 203 fp32 = 3 tiles of 64 + 11 (2 vectors and
# 3 points), 101 fp64 = 3 tiles of 32 + 5 (2 vectors and 1 point).
A_N = {4: (23, 37, 203), 8: (23, 37, 101)}
LX = {1: 5, 2: 7, 3: 5, 7: 3}


def chunk_lengths(nx, lx):
    nc = max(1, min(-(-nx // lx), MAX_CHUNKS, nx))
    return [nx * (c + 1) // nc - nx * c // nc for c in range(nc)]


def units(n, eb, lx):
    return -(-n[1] // 16) * -(-n[2] // TZ[eb]) * len(chunk_lengths(n[0], lx))


# every hand-written (shape, radius, precision) with a grid cycling over the radii, and every grid for fp64 radius 8 (one plane of
# prefetch, PF = 1, where the other tiles have 2)
A_CASES = [(s, R, eb, GRIDS[(R + i) % 4]) for i, s in enumerate(A.SHAPES) for R in range(1, 9) for eb in (4, 8)
           if (s, R, eb) in HAND] + \
          [(s, 8, 8, g) for i, s in enumerate(A.SHAPES) for g in GRIDS if g != GRIDS[(8 + i) % 4]]


@pytest.mark.parametrize("shape,R,eb,grid", A_CASES, ids=[f"{s}-r{r}-fp{8 * e}-g{g}" for s, r, e, g in A_CASES])
def test_persistent_ctas(shape, R, eb, grid):
    n, lx = A_N[eb], LX[grid]
    cl = chunk_lengths(n[0], lx)
    assert max(cl) - min(cl) == 1 and units(n, eb, lx) > grid
    check_one(shape, n, R, eb, 2, {"kernel": "tma", "lx": lx, "grid": grid}, sweeps=2)


# ---- B. thin and tiny domains ------------------------------------------------------------------------------------------------
def tiny(R):
    """Thinner than R in every dim (1 where R is 1)."""
    return (max(1, R - 1), max(1, R // 2), max(1, R - 2))


B_DOMAINS = ["1x5x7", "3x1x200", "40x7x15", "5x40x3", "tiny"]


@pytest.mark.parametrize("kernel", ["direct", "auto", "tma"])
@pytest.mark.parametrize("dom", B_DOMAINS)
@pytest.mark.parametrize("shape,R,eb", HAND, ids=[f"{s}-r{r}-fp{8 * e}" for s, r, e in HAND])
def test_thin_domains(shape, R, eb, dom, kernel):
    n = tiny(R) if dom == "tiny" else tuple(int(x) for x in dom.split("x"))
    assert n[1] < 8 or n[2] < 16          # kernel=auto sends every one of these to the direct kernel
    check_one(shape, n, R, eb, 2, {"kernel": kernel}, sweeps=2 if kernel == "tma" else 0)


# ---- C. rank grids -------------------------------------------------------------------------------------------------------------
def _neighbours(idx, grid, l1):
    """Neighbour directions of rank idx that a var of L1 norm l1 exchanges with."""
    out = 0
    for d in itertools.product((-1, 0, 1), repeat=3):
        if any(d) and sum(map(abs, d)) <= l1 and all(0 <= i + k < g for i, k, g in zip(idx, d, grid)):
            out += 1
    return out


def _boxes(size, idx, grid, R, eb, split):
    """The boxes one step of a rank launches (halo_run_stage): the whole rank, or the exterior slabs of every split dim and then
    the interior; slab widths in z are rounded up to whole 16-byte vectors."""
    whole = [(0, x) for x in size]
    if not split:
        return [whole]
    inner = [list(b) for b in whole]
    for d in range(3):
        if grid[d] <= 1:
            continue
        al = VW[eb] if d == 2 else 1
        if idx[d] > 0:
            inner[d][0] += -(-R // al) * al
        if idx[d] < grid[d] - 1:
            inner[d][1] = max(0, inner[d][1] - R) // al * al
        if inner[d][1] - inner[d][0] < 1:
            return [whole]
    boxes, cur = [], [list(b) for b in whole]
    for d in range(3):
        if inner[d][0] > whole[d][0]:
            boxes.append([tuple(c) for c in cur[:d]] + [(whole[d][0], inner[d][0])] + [tuple(c) for c in cur[d + 1:]])
        if inner[d][1] < whole[d][1]:
            boxes.append([tuple(c) for c in cur[:d]] + [(inner[d][1], whole[d][1])] + [tuple(c) for c in cur[d + 1:]])
        cur[d] = inner[d]
    return boxes + [[tuple(c) for c in cur]]


def _is_sweep(box, kernel):
    ny, nz = box[1][1] - box[1][0], box[2][1] - box[2][0]
    return kernel == "tma" or (kernel == "auto" and ny >= 8 and nz >= 16)


def expected_launches(shape, n, R, eb, grid, rank, opts, steps):
    """(sweep launches, kernel launches) of one rank: stencil boxes per step, plus one halo push per exchanging neighbour for each
    dirty slot: both slots in the first exchange of the first run_solution() call (fill_hash marks them), then one per step.  A
    later call's first exchange finds nothing dirty, so the counts do not depend on how the steps are split over calls."""
    idx = multi.grid_coords(rank, grid)
    size = [-(-x // g) if i < g - 1 else x - -(-x // g) * (g - 1) for x, g, i in zip(n, grid, idx)]
    # an x neighbour takes the fused branch, which this engine runs as the whole form; without one, or with fused_halo=0, the
    # split form runs unless overlap_comms=0
    split = opts.get("overlap_comms", 1) != 0 and (grid[0] == 1 or opts.get("fused_halo", 1) == 0)
    boxes = [b for b in _boxes(size, idx, grid, R, eb, split) if all(e > s for s, e in b)]
    kernel = opts.get("kernel", "auto")
    sweeps = sum(_is_sweep(b, kernel) for b in boxes) * steps
    pushes = _neighbours(idx, grid, A.L1_NORM[shape]) * (2 + steps)
    return sweeps, len(boxes) * steps + pushes


def run_grid(shape, n, R, eb, grid, opts, runs):
    solns = []
    try:
        for r in range(int(np.prod(grid))):
            s = make(shape, n, R, eb, opts)
            s.set_num_ranks_vec(grid)
            s.set_rank_index_vec(multi.grid_coords(r, grid))
            s.prepare_solution(0)
            solns.append(s)
        multi.connect_local(solns)
        for s in solns:
            a = s.get_var("A")
            for t in (0, 1):
                a.fill_hash(t, SEED, var_salt("A", t), -1.0, 1.0)
        for first, last in runs:
            for s in solns:       # every rank enqueued before any waits: ranks wait for each other on the device
                s.run_solution(first, last)
        for s in solns:
            s.sync()
        out = np.full(n, np.nan, _dt(eb))
        counts = []
        for s in solns:
            a = s.get_var("A")
            f, l = a.domain_box(a.get_last_valid_step_index())
            out[f[1]:l[1] + 1, f[2]:l[2] + 1, f[3]:l[3] + 1] = a.get_elements_in_slice(f, l)
            counts.append((int(s.get_option("gen_sweep_launches")), s.get_stats().kernel_launches))
        return out, counts
    finally:
        for s in solns:
            s.close()


def check_grid(shape, n, R, eb, grid, opts, steps=3, runs=None):
    got, counts = run_grid(shape, n, R, eb, grid, opts, runs or [(0, steps - 1)])
    ref = oracle(tuple(n), shape, R, eb, steps)[R:-R, R:-R, R:-R]
    assert np.array_equal(bits(got), bits(ref)), (shape, n, R, eb, grid, opts)
    want = [expected_launches(shape, n, R, eb, grid, r, opts, steps) for r in range(int(np.prod(grid)))]
    assert counts == want, (shape, n, R, eb, grid, opts, counts, want)


# layout: (grid, options); the smallest rank of every split dim gets `size` points, the others one more
LAYOUTS = {"x2": ((2, 1, 1), {}),                                  # whole form (x splits never take the split path here)
           "x2_split": ((2, 1, 1), {"fused_halo": 0}),             # split form: x exterior slabs
           "x3_split": ((3, 1, 1), {"fused_halo": 0}),
           "y2": ((1, 2, 1), {}),
           "z2": ((1, 1, 2), {}),
           "z2_tma": ((1, 1, 2), {"kernel": "tma"}),
           "xyz2": ((2, 2, 2), {})}
SIZES = {"R": lambda R, eb: R, "2R-1": lambda R, eb: 2 * R - 1, "2R+vec+1": lambda R, eb: 2 * R + VW[eb] + 1}
BASE = (9, 20, 70)         # unsplit dims: a partial y tile; z: a partial tile and a partial vector in both precisions


def grid_domain(grid, size):
    return tuple(g * size + g - 1 if g > 1 else b for g, b in zip(grid, BASE))


C_CASES = [(s, R, eb, lay, sz) for s, R, eb in HAND for lay in LAYOUTS for sz in SIZES
           if lay != "xyz2" or s != "3axis"]        # 3axis exchanges with face neighbours only


@pytest.mark.parametrize("shape,R,eb,layout,size", C_CASES, ids=[f"{s}-r{r}-fp{8 * e}-{l}-{z}" for s, r, e, l, z in C_CASES])
def test_rank_grid(shape, R, eb, layout, size):
    grid, opts = LAYOUTS[layout]
    check_grid(shape, grid_domain(grid, SIZES[size](R, eb)), R, eb, grid, opts)


OPT_CASES = [("cube", 5, 4), ("3axis_with_diags", 8, 8), ("3plane", 2, 4), ("3axis", 7, 8)]


@pytest.mark.parametrize("layout", ["x3_split", "z2_tma", "xyz2"])
@pytest.mark.parametrize("shape,R,eb", OPT_CASES, ids=[f"{s}-r{r}-fp{8 * e}" for s, r, e in OPT_CASES])
def test_rank_grid_no_overlap(shape, R, eb, layout):
    grid, opts = LAYOUTS[layout]
    if layout == "xyz2" and shape == "3axis":
        grid = (2, 2, 1)
    check_grid(shape, grid_domain(grid, 2 * R + VW[eb] + 1), R, eb, grid, dict(opts, overlap_comms=0))


@pytest.mark.parametrize("layout", ["x2", "x3_split", "z2"])
@pytest.mark.parametrize("shape,R,eb", OPT_CASES, ids=[f"{s}-r{r}-fp{8 * e}" for s, r, e in OPT_CASES])
def test_rank_grid_runs_split_over_calls(shape, R, eb, layout):
    grid, opts = LAYOUTS[layout]
    check_grid(shape, grid_domain(grid, 2 * R - 1), R, eb, grid, opts, steps=5, runs=[(0, 1), (2, 4)])


def test_too_thin_rank_grid_is_refused_by_every_rank():
    """prepare_solution() refuses a grid whose smallest rank is thinner than the halo on every rank, before any device work."""
    R, grid, n = 8, (2, 1, 1), (15, 20, 70)          # ranks of 8 and 7 planes
    for r in range(2):
        s = make("cube", n, R, 4, {})
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        with pytest.raises(capi.YaskError, match="local-domain size of 7 in 'x' dim is less than minimum size of 8"):
            s.prepare_solution(0)
        assert not s.is_prepared()
        s.close()


# ---- D. past 2^31 elements per slot --------------------------------------------------------------------------------------------
MARGIN = 2 << 30
D_CASES = [("3axis_with_diags", 8, 4, 2, {"kernel": "tma"}), ("3axis_with_diags", 8, 4, 2, {"kernel": "direct"}),
           ("cube", 1, 8, 2, {}), ("3plane", 5, 4, 2, {}), ("3axis", 1, 4, 4, {"block_steps": 2})]


@pytest.mark.parametrize("shape,R,eb,steps,opts", D_CASES, ids=["diags-r8-sweep", "diags-r8-direct", "cube-r1-fp64", "3plane-r5",
                                                                "3axis-r1-tt"])
def test_past_2_31(shape, R, eb, steps, opts):
    import torch
    n = (1300, 1300, 1300)
    m = steps * R
    size = [32 + m] * 3
    s = make(shape, n, R, eb, opts)
    need = storage_bytes(s)
    free, _ = torch.cuda.mem_get_info()
    if free < need + MARGIN:
        s.close()
        pytest.skip(f"needs {need / 1e9:.1f} GB of device memory plus a 2 GB margin, {free / 1e9:.1f} GB free")
    info = s.get_var("A").info
    assert info.slot_elems > TWO31
    wins = three_windows(info, n, size, m)
    try:
        s.prepare_solution(0)
        a = s.get_var("A")
        for t in (0, 1):
            a.fill_hash(t, SEED, var_salt("A", t), -1.0, 1.0)
        s.run_solution(0, steps - 1)
        tl = a.get_last_valid_step_index()
        got = [a.get_elements_in_slice(*w.kept_box(tl)) for w in wins]
        sw, tt, kl = int(s.get_option("gen_sweep_launches")), int(s.get_option("tt_launches")), s.get_stats().kernel_launches
    finally:
        s.close()
    if opts.get("block_steps") == 2:
        assert (sw, tt, kl) == (0, steps // 2, steps // 2)
    else:
        assert (sw, tt, kl) == (0 if opts.get("kernel") == "direct" else steps, 0, steps)
    for g, w in zip(got, wins):
        ins = [hash_field(SEED, var_salt("A", t), [x - R for x in w.lo], [x + 2 * R for x in w.size], -1, 1, _dt(eb)) for t in (0, 1)]
        ref = A.run(ins[0], ins[1], shape, R, steps)[R:-R, R:-R, R:-R][w.kept_slices()]
        assert np.array_equal(bits(g), bits(ref)), (shape, R, eb, opts, w.lo)


# ---- E. FP modes -----------------------------------------------------------------------------------------------------------------
E_CASES = [(s, R, eb) for s, R in (("3axis", 3), ("3axis_with_diags", 6), ("3plane", 5), ("cube", 4)) for eb in (4, 8)]


@pytest.mark.parametrize("shape,R,eb", E_CASES, ids=[f"{s}-r{r}-fp{8 * e}" for s, r, e in E_CASES])
def test_fp_modes_give_the_same_bits(shape, R, eb):
    n = A_N[eb]
    for mode in (0, 1, 2):
        check_one(shape, n, R, eb, 2, {"fp_mode": mode}, sweeps=2)
