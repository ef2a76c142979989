"""Point sources and receivers on the device, bit for bit against the reference API loop on the same inputs:

    for t in steps: run_solution(t, t); add_to_element(amp[u - t0][i], [u, *src_i]) in list order; trace[u - t0r][j] = get_element

(u = t + 1, or t - 1 for a reverse solution), with one-element slices of the C ABI and the rounding of add_to_element.  Every
var a stage writes and every trace row is compared.  Each case names the schedule rule it exercises."""
import numpy as np
import pytest

from tests.golden.ranges import RANGES
from tests.helpers import range_of
from yask_b200 import capi, multi
from yask_b200.synth import var_salt

pytestmark = pytest.mark.gpu
SEED = 41


def make(stencil, n, radius=0, eb=4, opts=(), grid=None, rank=0):
    s = capi.Solution(stencil, radius=radius, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    if grid:
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(rank, grid))
    for k, v in opts:
        s.set_option(k, v)
    s.prepare_solution(0)
    return s


def fill(s, stencil, first_steps):
    rg = RANGES[stencil]
    for v in s.get_vars():
        vi = v.info
        name = vi.name.decode()
        lo, hi = range_of(rg, name)
        for t in (first_steps[:vi.step_alloc] if vi.has_step else [0]):
            v.fill_hash(t, SEED, var_salt(name, t), lo, hi)


def amp_table(nrows, n, dtype):
    a = np.random.default_rng(3).uniform(-0.5, 0.5, size=(nrows, n))
    a[0, 0] = 1.0 / 3.0                     # not representable in fp32: the rounding of the add matters
    return a


def calls(first, last, splits):
    """The run as several run_solution() calls: `splits` = steps of each call."""
    step = 1 if last >= first else -1
    ts = list(range(first, last + step, step))
    out, k = [], 0
    for n in splits or [len(ts)]:
        out.append((ts[k], ts[k + n - 1]))
        k += n
    assert k == len(ts)
    return out


def outputs(s):
    """{(var, step): domain box} of every written var at every valid step."""
    out = {}
    for v in s.get_vars():
        vi = v.info
        if not vi.is_output:
            continue
        for t in range(vi.first_valid_step, vi.last_valid_step + 1):
            out[(vi.name.decode(), t)] = v.get_elements_in_slice(*v.domain_box(t))
    return out


def loop_oracle(s, first, last, off, src, rcv):
    """The reference API loop on solution `s`: one step per call, the adds and reads through one-element slices."""
    dt = np.float32 if s.get_element_bytes() == 4 else np.float64
    step = 1 if last >= first else -1
    trace = None
    if rcv:
        trace = np.zeros((rcv[3], len(rcv[1])), dt)
    for t in range(first, last + step, step):
        s.run_solution(t, t)
        u = t + off
        if src and 0 <= u - src[2] < len(src[3]):
            var = s.get_var(src[0])
            for i, p in enumerate(src[1]):
                idx = [u] + list(p)
                cur = var.get_elements_in_slice(idx, idx).reshape(-1)[0]
                var.set_elements_in_slice(np.array([dt(cur) + dt(src[3][u - src[2]][i])], dt), idx, idx)
        if rcv and 0 <= u - rcv[2] < rcv[3]:
            var = s.get_var(rcv[0])
            for j, p in enumerate(rcv[1]):
                idx = [u] + list(p)
                trace[u - rcv[2], j] = var.get_elements_in_slice(idx, idx).reshape(-1)[0]
    return trace


def same(a, b):
    it = np.uint32 if a.dtype == np.float32 else np.uint64
    return a.shape == b.shape and np.array_equal(a.view(it), b.view(it))


def placement(n):
    """Sources on a corner, an edge, a face and inside (one point three times); receivers on corners, faces and the sources."""
    lo, hi, mid = [0] * len(n), [m - 1 for m in n], [m // 2 for m in n]
    edge = [0] + [m - 1 for m in n[1:]]
    face = list(mid)
    face[-1] = 0
    src = [mid, lo, edge, mid, face, hi, mid]
    rcv = [hi, lo, mid, face, [m // 3 for m in n], edge] + [[(7 * k + 3) % m for m in n] for k in range(10)]
    return src, rcv


def check_case(stencil, n, steps, radius=0, eb=4, opts=(), src_var=None, rcv_var=None, reverse=False, splits=None,
               short_table=True, rcv_mid=True, expect_launches=True):
    first, last, off = (steps, 1, -1) if reverse else (0, steps - 1, 1)
    fill_steps = list(range(steps, steps + 4)) if reverse else [0, 1, 2, 3]
    src_pts, rcv_pts = placement(n)
    s = make(stencil, n, radius, eb, opts)
    dt = np.float32 if s.get_element_bytes() == 4 else np.float64
    out_var = [v.get_name() for v in s.get_vars() if v.info.is_output][0]
    src_var, rcv_var = src_var or out_var, rcv_var or out_var
    nrows = steps - 2 if short_table else steps          # a table shorter than the run
    t0 = first + off
    t0r = t0 + off * (2 if rcv_mid else 0)               # a receiver window that starts mid-run
    nrows_r = steps
    amp = amp_table(nrows, len(src_pts), dt)
    if reverse:
        t0, t0r = last + off, last + off                  # rows count upwards from the last step computed
        amp = amp_table(steps, len(src_pts), dt)
    src = (src_var, src_pts, t0, amp)
    rcv = (rcv_var, rcv_pts, t0r, nrows_r)
    fill(s, stencil, fill_steps)
    s.set_sources(src_var, src_pts, t0, amp)
    s.set_receivers(rcv_var, rcv_pts, t0r, nrows_r)
    for a, b in calls(first, last, splits):
        s.run_solution(a, b)
    traces, owned = s.get_traces()
    got = outputs(s)
    launches = int(s.get_option("point_launches"))
    tt = s.get_option("tt_launches") if ("block_steps", 2) in opts else "0"
    s.close()
    o = make(stencil, n, radius, eb, opts)
    fill(o, stencil, fill_steps)
    ref_tr = loop_oracle(o, first, last, off, src, rcv)
    ref = outputs(o)
    o.close()
    assert owned.all()
    assert same(traces, ref_tr), np.argwhere(traces != ref_tr)[:5]
    assert got.keys() == ref.keys()
    for k in ref:
        assert same(got[k], ref[k]), k
    assert tt == "0"                                      # no pair ever runs while points are set
    if expect_launches:
        us = [t + off for t in range(first, last + (1 if last >= first else -1), 1 if last >= first else -1)]
        want = sum(1 for u in us if 0 <= u - t0 < len(amp) or 0 <= u - t0r < nrows_r)
        assert launches == want, (launches, want)


# single rank: the point launch follows the step's last stage on the one-step path
@pytest.mark.parametrize("stencil,n,steps,radius,eb,opts,src_var,rcv_var,reverse,splits", [
    ("iso3dfd", (40, 36, 64), 6, 8, 4, (), None, None, False, None),                         # resident radius-8 sweep
    ("iso3dfd", (40, 36, 64), 5, 8, 4, (("kernel", "direct"),), None, None, False, None),
    ("iso3dfd", (40, 36, 64), 7, 8, 4, (), None, None, False, [2, 1, 4]),                    # several run_solution() calls
    ("iso3dfd", (32, 28, 48), 5, 4, 8, (), None, None, False, None),                         # fp64
    ("iso3dfd_sponge", (30, 26, 48), 5, 3, 4, (), None, None, False, None),
    ("3axis", (30, 20, 64), 5, 1, 8, (), None, None, False, None),                           # hand-written fp64
    ("3axis", (30, 20, 64), 5, 0, 0, (), None, None, False, None),                           # generated, default radius
    ("awp_elastic", (21, 19, 40), 4, 0, 0, (), "stress_xx", "vel_x", False, None),           # two stages
    ("wave2d", (37, 50), 5, 0, 0, (), "e", "u", False, None),                                # 2-D
    ("test_reverse_2d", (37, 50), 5, 0, 0, (), None, None, True, None),                      # reverse run
], ids=["iso-r8", "iso-r8-direct", "iso-r8-split-calls", "iso-fp64-r4", "sponge-r3", "3axis-fp64-r1", "3axis-gen",
        "awp_elastic", "wave2d", "reverse-2d"])
def test_single_rank_matches_loop(stencil, n, steps, radius, eb, opts, src_var, rcv_var, reverse, splits):
    check_case(stencil, n, steps, radius, eb, opts, src_var, rcv_var, reverse, splits)


def test_in_run_tuner_with_points():
    """The tuner times each step with its point launch inside."""
    check_case("iso3dfd", (40, 36, 64), 6, 8, 4, (("auto_tune", 1),))


def test_block_steps_fall_back_and_resume():
    """iso3dfd radius 1 with block_steps=2: points make every step a one-step launch (tt_launches stays 0); once they are
    cleared the pairs come back and the run still equals the loop."""
    opts = (("block_steps", 2), ("tt_variant", 0))
    check_case("iso3dfd", (40, 24, 160), 6, 1, 4, opts)
    n, src_pts = (40, 24, 160), [[5, 5, 5], [20, 12, 80]]
    s = make("iso3dfd", n, 1, 4, opts)
    fill(s, "iso3dfd", [0, 1])
    amp = amp_table(4, 2, np.float32)
    s.set_sources("p", src_pts, 1, amp)
    s.run_solution(0, 3)
    assert s.get_option("tt_launches") == "0"
    s.clear_points()
    s.run_solution(4, 7)
    assert int(s.get_option("tt_launches")) == 2
    got = outputs(s)
    s.close()
    o = make("iso3dfd", n, 1, 4, opts)
    fill(o, "iso3dfd", [0, 1])
    loop_oracle(o, 0, 3, 1, ("p", src_pts, 1, amp), None)
    loop_oracle(o, 4, 7, 1, None, None)
    ref = outputs(o)
    o.close()
    for k in ref:
        assert same(got[k], ref[k]), k


def test_past_2_31_elements_per_slot():
    """64-bit slot offsets: sources and receivers beyond element 2^31 of a slot (iso3dfd fp32 radius 8)."""
    from tests.large_domain import crossing_index
    n, steps = (1100, 1024, 1984), 2
    s = make("iso3dfd", n)
    p = s.get_var("p")
    xc = int(crossing_index(p.info))
    assert p.info.slot_elems > 1 << 31 and xc < n[0] - 2
    src_pts = [[xc + 1, 17, 1000], [xc + 1, 17, 1000], [n[0] - 1, n[1] - 1, n[2] - 1]]
    rcv_pts = src_pts + [[xc, 3, 5], [2, 2, 2]]
    amp = amp_table(steps, len(src_pts), np.float32)
    fill(s, "iso3dfd", [0, 1])
    s.set_sources("p", src_pts, 1, amp)
    s.set_receivers("p", rcv_pts, 1, steps)
    s.run_solution(0, steps - 1)
    traces, _ = s.get_traces()
    boxes = [([t] + [max(0, c - 2) for c in q], [t] + [min(m - 1, c + 2) for c, m in zip(q, n)]) for q in rcv_pts for t in (1, 2)]
    got = [p.get_elements_in_slice(f, l) for f, l in boxes]
    s.close()
    o = make("iso3dfd", n)
    fill(o, "iso3dfd", [0, 1])
    ref_tr = loop_oracle(o, 0, steps - 1, 1, ("p", src_pts, 1, amp), ("p", rcv_pts, 1, steps))
    op = o.get_var("p")
    ref = [op.get_elements_in_slice(f, l) for f, l in boxes]
    o.close()
    assert same(traces, ref_tr)
    for a, b in zip(got, ref):
        assert same(a, b)


# rank grids in one process, against the loop on one rank over the global domain
def grid_case(n, grid, radius, src_pts, rcv_pts, steps, opts=()):
    world = int(np.prod(grid))
    amp = amp_table(steps, len(src_pts), np.float32)
    solns = [make("iso3dfd", n, radius, 4, opts, grid, r) for r in range(world)]
    multi.connect_local(solns)
    for s in solns:
        fill(s, "iso3dfd", [0, 1])
        s.set_sources("p", src_pts, 1, amp)
        s.set_receivers("p", rcv_pts, 1, steps)
    for s in solns:             # enqueue every rank first: ranks wait for each other on the device
        s.run_solution(0, steps - 1)
    for s in solns:
        s.sync()
    out = {t: np.zeros(n, np.float32) for t in (steps - 1, steps)}
    traces = np.zeros((steps, len(rcv_pts)), np.float32)
    cover = np.zeros(len(rcv_pts), int)
    launches = []
    for s in solns:
        p = s.get_var("p")
        for t in out:
            f, l = p.domain_box(t)
            out[t][f[1]:l[1] + 1, f[2]:l[2] + 1, f[3]:l[3] + 1] = p.get_elements_in_slice(f, l)
        tr, owned = s.get_traces()
        traces[:, owned] = tr[:, owned]
        cover += owned
        launches.append(int(s.get_option("point_launches")))
        s.close()
    o = make("iso3dfd", n, radius)
    fill(o, "iso3dfd", [0, 1])
    ref_tr = loop_oracle(o, 0, steps - 1, 1, ("p", src_pts, 1, amp), ("p", rcv_pts, 1, steps))
    p = o.get_var("p")
    ref = {t: p.get_elements_in_slice(*p.domain_box(t)) for t in out}
    o.close()
    assert (cover == 1).all()
    assert same(traces, ref_tr)
    for t in out:
        assert same(out[t], ref[t]), t
    # every rank launches at most twice per step (split form: exterior and interior points), the ranks together at least once
    assert all(0 <= k <= 2 * steps for k in launches) and sum(launches) >= steps


GRID_CASES = [((2, 1, 1), (75, 40, 64), "x-halo-yields"), ((2, 1, 1), (75, 40, 64), "x-just-outside"),
              ((1, 2, 1), (40, 75, 64), "y-exterior"), ((2, 2, 1), (75, 61, 64), "x-halo-yields"),
              ((2, 2, 1), (75, 61, 64), "y-exterior")]


@pytest.mark.parametrize("radius", [8, 2])
@pytest.mark.parametrize("grid,n,rule", GRID_CASES, ids=["x".join(map(str, g)) + "-" + r for g, _, r in GRID_CASES])
def test_rank_grid_matches_single_rank_loop(grid, n, rule, radius):
    """x-halo-yields: a source within the x halo width of the x interface makes the owning rank run the split form instead of
    the fused x exchange; x-just-outside: one plane farther, injected after the fused launch; y-exterior: a source in a
    y-exterior slab, injected before the pushes of the split form (or of the fused form's y exchange)."""
    x_if = (n[0] + grid[0] - 1) // grid[0]          # first x of rank 1 in x (uneven split)
    y_if = (n[1] + grid[1] - 1) // grid[1]
    mid = [x_if // 2, n[1] // 3, n[2] // 2]
    if rule == "x-halo-yields":
        src = [[x_if - radius, mid[1], mid[2]], [x_if + radius - 1, mid[1], 7]]
    elif rule == "x-just-outside":
        src = [[x_if - radius - 1, mid[1], mid[2]], [x_if + radius, mid[1], 7]]
    else:
        src = [[mid[0], y_if - 1, mid[2]], [mid[0], y_if, 9]]
    src = src + [src[0]]                             # one point twice
    rcv = src + [[0, 0, 0], [n[0] - 1, n[1] - 1, n[2] - 1], [x_if - 1, y_if - 1, 5], [min(x_if, n[0] - 1), min(y_if, n[1] - 1), 5]]
    grid_case(n, grid, radius, src, rcv, 4)
