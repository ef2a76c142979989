"""Weighted point sources and receivers (between grid points) on the device, bit for bit against the reference API loop on the
same inputs:

    for t in steps: run_solution(t, t)
                    for each source i, entry q with w != 0: var(u, idx[i][q]) = dt(var) + dt(w[i][q] * amp[u - t0][i])
                    for each receiver j: acc = 0.0; for each entry q with w != 0: acc = acc + w[j][q] * var(u, idx[j][q])
                                         trace[u - t0r][j] = dt(acc)

(u = t + 1, or t - 1 for a reverse solution).  The adds go through one-element slices of the C ABI; the receiver sums are formed
in IEEE double, one rounded multiply and one rounded add per entry, in entry order, from the field the loop read back.  Every var
a stage writes and every trace row is compared.  Rank grids run in one process and must equal the single-rank run."""
import numpy as np
import pytest

from tests.golden.ranges import RANGES
from tests.helpers import range_of
from yask_b200 import capi, multi
from yask_b200.synth import var_salt

pytestmark = pytest.mark.gpu
SEED = 43


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


def amp_table(nrows, n):
    a = np.random.default_rng(3).uniform(-0.5, 0.5, size=(nrows, n))
    a[0, 0] = 1.0 / 3.0                     # not representable in fp32: the rounding of the add matters
    return a


def calls(first, last, splits):
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


def same(a, b):
    it = np.uint32 if a.dtype == np.float32 else np.uint64
    return a.shape == b.shape and np.array_equal(a.view(it), b.view(it))


def receiver_sums(field, idx, w, dt):
    """acc = +0.0; acc = acc + w * double(v) per entry in order (numpy: one rounded op each, no FMA); dt(acc)."""
    acc = np.zeros(len(idx), np.float64)
    for q in range(idx.shape[1]):
        v = field[tuple(idx[:, q, d].clip(0, field.shape[d] - 1) for d in range(idx.shape[2]))].astype(np.float64)
        acc = np.where(w[:, q] != 0, acc + w[:, q] * v, acc)
    return acc.astype(dt)


def loop_oracle(s, first, last, off, src, rcv):
    """The reference API loop: one step per call, the source adds through one-element slices, the receivers from the field."""
    dt = np.float32 if s.get_element_bytes() == 4 else np.float64
    step = 1 if last >= first else -1
    trace = np.zeros((rcv[4], len(rcv[1])), dt) if rcv else None
    for t in range(first, last + step, step):
        s.run_solution(t, t)
        u = t + off
        if src and 0 <= u - src[3] < len(src[4]):
            var, idx, w = s.get_var(src[0]), src[1], src[2]
            for i in range(len(idx)):
                for q in range(idx.shape[1]):
                    if w[i, q] == 0:
                        continue
                    at = [u] + idx[i, q].tolist()
                    cur = var.get_elements_in_slice(at, at).reshape(-1)[0]
                    a = float(w[i, q]) * float(src[4][u - src[3]][i])
                    var.set_elements_in_slice(np.array([dt(cur) + dt(a)], dt), at, at)
        if rcv and 0 <= u - rcv[3] < rcv[4]:
            var = s.get_var(rcv[0])
            field = var.get_elements_in_slice(*var.domain_box(u))
            trace[u - rcv[3]] = receiver_sums(field, rcv[1], rcv[2], dt)
    return trace


def placement(n):
    """Trilinear sources between points, on a grid point, on the last plane, and two sharing support points; trilinear
    receivers on the sources, between points, on corners and the last plane."""
    nd = len(n)
    mid = [m / 2 + 0.25 for m in n]
    src = [mid, [m // 3 for m in n], [m - 1.0 for m in n], [m / 2 + 0.75 for m in n], [1.5] * nd, mid]
    rcv = [mid, [m - 1.0 for m in n], [0.0] * nd, [m / 2 + 0.5 for m in n], [1.25] * nd, [m - 1.5 for m in n]]
    rng = np.random.default_rng(9)
    rcv += rng.uniform(0, np.array(n) - 1, size=(12, nd)).tolist()
    return src, rcv


def check_case(stencil, n, steps, radius=0, eb=4, opts=(), src_var=None, rcv_var=None, reverse=False, splits=None):
    first, last, off = (steps, 1, -1) if reverse else (0, steps - 1, 1)
    fill_steps = list(range(steps, steps + 4)) if reverse else [0, 1, 2, 3]
    src_pos, rcv_pos = placement(n)
    sidx, sw = capi.trilinear(src_pos)
    ridx, rw = capi.trilinear(rcv_pos)
    s = make(stencil, n, radius, eb, opts)
    out_var = [v.get_name() for v in s.get_vars() if v.info.is_output][0]
    src_var, rcv_var = src_var or out_var, rcv_var or out_var
    t0 = first + off
    t0r = t0 + 2 * off                       # a receiver window that starts mid-run
    amp = amp_table(steps - 2, len(src_pos))  # a table shorter than the run
    if reverse:
        t0 = t0r = last + off
        amp = amp_table(steps, len(src_pos))
    src = (src_var, sidx, sw, t0, amp)
    rcv = (rcv_var, ridx, rw, t0r, steps)
    fill(s, stencil, fill_steps)
    s.set_sources_weighted(src_var, sidx, sw, t0, amp)
    s.set_receivers_weighted(rcv_var, ridx, rw, t0r, steps)
    for a, b in calls(first, last, splits):
        s.run_solution(a, b)
    traces, owned = s.get_traces()
    got = outputs(s)
    launches = int(s.get_option("point_launches"))
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
    us = [t + off for t in range(first, last + off, off)]
    want = sum((0 <= u - t0 < len(amp)) + (0 <= u - t0r < steps) for u in us)    # one launch per weighted kernel
    assert launches == want, (launches, want)


CASES = [
    ("iso3dfd", (40, 36, 64), 6, 8, 4, None, None, False, None),              # resident radius-8 sweep, fp32
    ("iso3dfd", (32, 28, 48), 5, 2, 8, None, None, False, None),              # fp64
    ("iso3dfd", (40, 36, 64), 7, 8, 4, None, None, False, [2, 1, 4]),         # several run_solution() calls
    ("awp_elastic", (21, 19, 40), 4, 0, 0, "stress_xx", "vel_x", False, None),  # two stages, in-place vars
    ("wave2d", (37, 50), 5, 0, 0, "e", "u", False, None),                     # 2-D: 4-entry supports
    ("test_reverse_2d", (37, 50), 5, 0, 0, None, None, True, None),           # reverse run
]


@pytest.mark.parametrize("stencil,n,steps,radius,eb,src_var,rcv_var,reverse,splits", CASES,
                         ids=["iso-r8", "iso-r2-fp64", "iso-r8-split-calls", "awp_elastic", "wave2d", "reverse-2d"])
def test_single_rank_matches_loop(stencil, n, steps, radius, eb, src_var, rcv_var, reverse, splits):
    check_case(stencil, n, steps, radius, eb, (), src_var, rcv_var, reverse, splits)


@pytest.mark.parametrize("eb", [4, 8])
def test_one_entry_of_weight_one_is_the_on_grid_set(eb):
    """k = 1, w = 1: 1.0 * a == a and T(0.0 + 1.0 * double(v)) == v, so the bits are those of set_sources / set_receivers."""
    n, steps = (40, 36, 64), 5
    src = [[20, 18, 32], [0, 0, 0], [20, 18, 32], [39, 35, 63]]
    rcv = [[21, 18, 32], [20, 18, 32], [0, 1, 0], [30, 30, 30]]
    amp = amp_table(steps - 1, len(src))
    res = []
    for weighted in (False, True):
        s = make("iso3dfd", n, 2 if eb == 8 else 8, eb)
        fill(s, "iso3dfd", [0, 1])
        if weighted:
            s.set_sources_weighted("p", np.array(src)[:, None, :], np.ones((len(src), 1)), 1, amp)
            s.set_receivers_weighted("p", np.array(rcv)[:, None, :], np.ones((len(rcv), 1)), 2, steps)
        else:
            s.set_sources("p", src, 1, amp)
            s.set_receivers("p", rcv, 2, steps)
        s.run_solution(0, steps - 1)
        res.append((s.get_traces()[0], outputs(s)))
        s.close()
    (ta, fa), (tb, fb) = res
    assert same(ta, tb)
    assert fa.keys() == fb.keys() and all(same(fa[k], fb[k]) for k in fa)


def test_many_receivers_reach_many_ctas():
    """100 000 trilinear receivers (391 CTAs of 256 threads) against the sums formed from the loop's fields."""
    n, steps = (64, 60, 128), 3
    rng = np.random.default_rng(21)
    pos = rng.uniform(0, np.array(n) - 1, size=(100_000, 3))
    idx, w = capi.trilinear(pos)
    sidx, sw = capi.trilinear([[30.5, 29.25, 64.75]])
    amp = amp_table(steps, 1)
    s = make("iso3dfd", n)
    fill(s, "iso3dfd", [0, 1])
    s.set_sources_weighted("p", sidx, sw, 1, amp)
    s.set_receivers_weighted("p", idx, w, 1, steps)
    s.run_solution(0, steps - 1)
    traces, _ = s.get_traces()
    s.close()
    o = make("iso3dfd", n)
    fill(o, "iso3dfd", [0, 1])
    ref = loop_oracle(o, 0, steps - 1, 1, ("p", sidx, sw, 1, amp), ("p", idx, w, 1, steps))
    o.close()
    assert same(traces, ref), np.argwhere(traces != ref)[:5]


def test_past_2_31_elements_per_slot():
    """64-bit offsets: support entries beyond element 2^31 of a slot (iso3dfd fp32 radius 8)."""
    from tests.large_domain import crossing_index
    n, steps = (1100, 1024, 1984), 2
    s = make("iso3dfd", n)
    p = s.get_var("p")
    xc = int(crossing_index(p.info))
    assert p.info.slot_elems > 1 << 31 and xc < n[0] - 2
    src_pos = [[xc + 0.5, 17.25, 1000.5], [xc + 1.0, 17.0, 1000.0], [n[0] - 1.0, n[1] - 1.0, n[2] - 1.5]]
    rcv_pos = src_pos + [[xc - 0.5, 3.5, 5.5], [2.5, 2.0, 2.25]]
    sidx, sw = capi.trilinear(src_pos)
    ridx, rw = capi.trilinear(rcv_pos)
    amp = amp_table(steps, len(src_pos))
    fill(s, "iso3dfd", [0, 1])
    s.set_sources_weighted("p", sidx, sw, 1, amp)
    s.set_receivers_weighted("p", ridx, rw, 1, steps)
    s.run_solution(0, steps - 1)
    traces, _ = s.get_traces()
    boxes = [([t] + [max(0, int(c) - 2) for c in q], [t] + [min(m - 1, int(c) + 3) for c, m in zip(q, n)]) for q in rcv_pos for t in (1, 2)]
    got = [p.get_elements_in_slice(f, l) for f, l in boxes]
    s.close()
    o = make("iso3dfd", n)
    fill(o, "iso3dfd", [0, 1])
    op = o.get_var("p")
    ref_tr = np.zeros((steps, len(rcv_pos)), np.float32)
    for t in range(steps):                  # the loop, with the receivers read one element at a time
        o.run_solution(t, t)
        u = t + 1
        for i in range(len(src_pos)):
            for q in range(8):
                if sw[i, q] != 0:
                    at = [u] + sidx[i, q].tolist()
                    cur = op.get_elements_in_slice(at, at).reshape(-1)[0]
                    op.set_elements_in_slice(np.array([np.float32(cur) + np.float32(float(sw[i, q]) * float(amp[t][i]))], np.float32), at, at)
        for j in range(len(rcv_pos)):
            acc = 0.0
            for q in range(8):
                if rw[j, q] != 0:
                    at = [u] + ridx[j, q].tolist()
                    acc = acc + float(rw[j, q]) * float(op.get_elements_in_slice(at, at).reshape(-1)[0])
            ref_tr[t, j] = np.float32(acc)
    ref = [op.get_elements_in_slice(f, l) for f, l in boxes]
    o.close()
    assert same(traces, ref_tr)
    for a, b in zip(got, ref):
        assert same(a, b)


# rank grids in one process, against the single-rank run of the same sets
def merged_run(stencil, n, steps, radius, eb, grid, src, rcv):
    """Run on `grid` (None: one rank); return every written var's last two steps over the global domain and the traces merged
    by the owned masks."""
    world = int(np.prod(grid)) if grid else 1
    solns = [make(stencil, n, radius, eb, (), grid, r) for r in range(world)]
    if grid:
        multi.connect_local(solns)
    for s in solns:
        fill(s, stencil, [0, 1, 2, 3])
        s.set_sources_weighted(*src)
        s.set_receivers_weighted(*rcv)
    for s in solns:             # enqueue every rank first: ranks wait for each other on the device
        s.run_solution(0, steps - 1)
    for s in solns:
        s.sync()
    dt = np.float32 if solns[0].get_element_bytes() == 4 else np.float64
    fields, traces, cover = {}, np.zeros((rcv[4], len(rcv[2])), dt), np.zeros(len(rcv[2]), int)
    for s in solns:
        for v in s.get_vars():
            vi = v.info
            if not vi.is_output:
                continue
            for t in (vi.last_valid_step - 1, vi.last_valid_step):
                if t < vi.first_valid_step:
                    continue
                f, l = v.domain_box(t)
                a = fields.setdefault((vi.name.decode(), t), np.zeros(n, dt))
                a[tuple(slice(f[k + 1], l[k + 1] + 1) for k in range(len(n)))] = v.get_elements_in_slice(f, l)
        tr, owned = s.get_traces()
        traces[:, owned] = tr[:, owned]
        cover += owned
        s.close()
    return fields, traces, cover


GRID_CASES = [
    # iso3dfd 2x1x1: a source within the x halo of the interface (the owner runs the split form) and receivers straddling it
    ("iso3dfd", (75, 40, 64), 8, 4, (2, 1, 1), "p", "p"),
    ("iso3dfd", (40, 75, 64), 8, 4, (1, 2, 1), "p", "p"),
    ("iso3dfd", (40, 36, 128), 8, 4, (1, 1, 2), "p", "p"),
    ("iso3dfd", (75, 40, 64), 2, 8, (2, 1, 1), "p", "p"),
    # awp_elastic: receivers straddling the interface on a stress var (written by the last of two stages, in place)
    ("awp_elastic", (42, 19, 40), 0, 0, (2, 1, 1), "stress_xx", "stress_xy"),
]


@pytest.mark.parametrize("stencil,n,radius,eb,grid,src_var,rcv_var", GRID_CASES,
                         ids=["iso-2x1x1", "iso-1x2x1", "iso-1x1x2", "iso-fp64-r2-2x1x1", "awp_elastic-2x1x1"])
def test_rank_grid_matches_single_rank(stencil, n, radius, eb, grid, src_var, rcv_var):
    steps = 4
    d = [k for k in range(3) if grid[k] > 1][0]
    cut = (n[d] + 1) // 2                               # first index of rank 1 in the split dim
    def at(x, z=None):
        p = [m / 3 + 0.25 for m in n]
        p[d] = x
        return p
    hw = radius if radius else 2
    src_pos = [at(cut - hw + 0.5), at(cut - 0.5), at(cut + 3.25), at(n[d] / 4 + 0.5)]
    rcv_pos = [at(cut - 0.5), at(cut - 0.01), at(cut - 1.0), at(cut + 0.5), at(cut - hw + 0.5), at(float(cut)),
               [0.0, 0.0, 0.0], [m - 1.0 for m in n], at(cut - 0.75)]
    sidx, sw = capi.trilinear(src_pos)
    ridx, rw = capi.trilinear(rcv_pos)
    amp = amp_table(steps - 1, len(src_pos))
    src = (src_var, sidx, sw, 1, amp)
    rcv = (rcv_var, ridx, rw, 1, steps)
    got, gtr, cover = merged_run(stencil, n, steps, radius, eb, grid, src, rcv)
    ref, rtr, _ = merged_run(stencil, n, steps, radius, eb, None, src, rcv)
    assert (cover == 1).all()
    assert same(gtr, rtr), np.argwhere(gtr != rtr)[:5]
    assert got.keys() == ref.keys()
    for k in ref:
        assert same(got[k], ref[k]), k


def test_yask_kernel_module_weighted_sets():
    """The yask_kernel module: yk_trilinear + yk_set_sources_weighted + yk_set_receivers_weighted equal the ctypes Solution."""
    import glob
    import os
    import subprocess
    import sys
    import textwrap
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    mod = glob.glob(os.path.join(root, "yask_b200", "lib", "python", "iso3dfd", "yask_kernel*.so"))
    if not mod:
        pytest.skip("python module not built")
    script = textwrap.dedent("""
        import struct
        import yask_kernel as yk
        steps, n = 5, (40, 36, 64)
        fac = yk.yk_factory()
        s = fac.new_solution(fac.new_env())
        s.set_overall_domain_size_vec(list(n))
        s.prepare_solution()
        s.get_var("v").set_all_elements_same(0.1)
        p = s.get_var("p")
        p.set_all_elements_same(0.0)
        p.set_element(0.25, [0, 20, 18, 32])
        sidx, sw = yk.yk_trilinear([[20.5, 18.25, 32.0]])
        ridx, rw = yk.yk_trilinear([[21.5, 18.5, 32.75], [20.0, 18.0, 32.0]])
        yk.yk_set_sources_weighted(s, "p", sidx, sw, 1, [[1.0 / 3.0]] * (steps - 1))
        yk.yk_set_receivers_weighted(s, "p", ridx, rw, 1, steps)
        s.run_solution(0, steps - 1)
        traces, owned = yk.yk_get_traces(s)
        assert all(owned) and yk.yk_get_point_launches(s) == 2 * steps - 1, yk.yk_get_point_launches(s)
        print(repr(traces))
    """)
    env = dict(os.environ, PYTHONPATH=os.path.dirname(mod[0]))
    r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    got = np.array(eval(r.stdout.strip().splitlines()[-1]), np.float32)
    s = make("iso3dfd", (40, 36, 64))
    s.get_var("v").set_all_elements_same(0.1)
    p = s.get_var("p")
    p.set_all_elements_same(0.0)
    p.set_elements_in_slice(np.array([0.25], np.float32), [0, 20, 18, 32], [0, 20, 18, 32])
    sidx, sw = capi.trilinear([[20.5, 18.25, 32.0]])
    ridx, rw = capi.trilinear([[21.5, 18.5, 32.75], [20.0, 18.0, 32.0]])
    s.set_sources_weighted("p", sidx, sw, 1, [[1.0 / 3.0]] * 4)
    s.set_receivers_weighted("p", ridx, rw, 1, 5)
    s.run_solution(0, 4)
    want, _ = s.get_traces()
    s.close()
    assert same(got, want)
