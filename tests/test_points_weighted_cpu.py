"""CPU: weighted point sources and receivers (between grid points) are planned and validated on the host -- the trilinear helper
against a numpy restatement of its formula, the refusals, ownership of every receiver by exactly one rank of a grid, and the
application order of support entries that share a grid point."""
import ctypes as C
import glob
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from yask_b200 import capi, multi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def planned(stencil="iso3dfd", n=(37, 29, 23), grid=None, rank=0, radius=0, opts=()):
    s = capi.Solution(stencil, radius=radius)
    s.set_overall_domain_size_vec(n)
    if grid:
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(rank, grid))
    for k, v in opts:
        s.set_option(k, v)
    s.plan_geometry()
    return s


def refused(fn, *words):
    with pytest.raises(capi.YaskError) as e:
        fn()
    for w in words:
        assert w in str(e.value), (w, str(e.value))


def trilinear_np(pos):
    """The formula of yb_points_trilinear, restated: per dim i = floor(p), f = p - i; entry c takes i + bit (ndd-1-d) of c in dim d
    and the weight ((1.0 * g_0) * g_1) * g_2 with g = f or 1 - f."""
    pos = np.atleast_2d(np.asarray(pos, np.float64))
    n, nd = pos.shape
    i = np.floor(pos)
    f = pos - i
    idx = np.zeros((n, 1 << nd, nd), np.int64)
    w = np.ones((n, 1 << nd), np.float64)
    for c in range(1 << nd):
        for d in range(nd):
            bit = (c >> (nd - 1 - d)) & 1
            idx[:, c, d] = i[:, d].astype(np.int64) + bit
            w[:, c] = w[:, c] * (f[:, d] if bit else 1.0 - f[:, d])
    return idx, w


@pytest.mark.parametrize("nd", [1, 2, 3])
def test_trilinear_matches_numpy_bit_for_bit(nd):
    rng = np.random.default_rng(7 + nd)
    special = [0.0, 1.0, 0.5, 2.5, -0.5, -3.25, 36.0, 35.999999999999, 511.25, 1e-17, 7.0 - 2 ** -40]
    pos = np.concatenate([rng.uniform(-50, 600, size=(200, nd)), rng.integers(-5, 40, size=(20, nd)).astype(np.float64),
                          np.array([[x] * nd for x in special]), np.array([special[k:k + nd] for k in range(len(special) - nd)])])
    idx, w = capi.trilinear(pos)
    ri, rw = trilinear_np(pos)
    assert idx.shape == (len(pos), 1 << nd, nd) and w.shape == (len(pos), 1 << nd)
    assert np.array_equal(idx, ri)
    assert np.array_equal(w.view(np.uint64), rw.view(np.uint64))
    # an integer position: one entry of weight 1 at the point itself, the others 0
    idx, w = capi.trilinear([[3.0] * nd])
    assert w[0, 0] == 1.0 and (w[0, 1:] == 0).all() and idx[0, 0].tolist() == [3] * nd
    # the weights of a point sum to 1 up to rounding, and are exact on half-integers
    idx, w = capi.trilinear([[2.5] * nd])
    assert (w == 0.5 ** nd).all()


def test_trilinear_refusals():
    refused(lambda: capi.trilinear([[1.0, np.nan, 2.0]]), "trilinear: position 0", "non-finite", "dim 1")
    refused(lambda: capi.trilinear([[1.0], [np.inf]]), "position 1", "non-finite")
    refused(lambda: capi.trilinear(np.zeros((2, 4))), "ndd 1, 2 or 3")
    L = capi.lib()
    assert L.yb_points_trilinear(3, 1, None, None, None) < 0 and b"null array" in L.yb_last_error()


def dptr(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def test_refusals_name_the_problem():
    s = planned()
    L = capi.lib()
    idx1 = np.array([[[1, 1, 1]]], np.int64)
    w1 = np.ones((1, 1))
    amp = np.ones((3, 1))
    # the C ABI itself: k < 1 and null tables
    assert L.yb_solution_set_receivers_weighted(s._h, b"p", 1, 0, dptr(idx1, C.c_int64), dptr(w1, C.c_double), 0, 3) < 0
    assert b"k = 0 support entries" in L.yb_last_error()
    assert L.yb_solution_set_receivers_weighted(s._h, b"p", 1, 1, None, dptr(w1, C.c_double), 0, 3) < 0
    assert b"null index table" in L.yb_last_error()
    assert L.yb_solution_set_sources_weighted(s._h, b"p", 1, 1, dptr(idx1, C.c_int64), None, 0, 3, dptr(amp, C.c_double)) < 0
    assert b"null weight table" in L.yb_last_error()
    assert L.yb_solution_set_sources_weighted(s._h, b"p", 1, 1, dptr(idx1, C.c_int64), dptr(w1, C.c_double), 0, 3, None) < 0
    assert b"null amplitude table" in L.yb_last_error()
    # the Python shapes
    refused(lambda: s.set_receivers_weighted("p", np.zeros((1, 0, 3), np.int64), np.zeros((1, 0)), 0, 3), "shape (n, k, 3)")
    refused(lambda: s.set_receivers_weighted("p", [[1, 1, 1]], [1.0], 0, 3), "shape (n, k, 3)")
    refused(lambda: s.set_sources_weighted("p", idx1, np.ones((1, 2)), 0, amp), "weight table of shape (1, 2)")
    refused(lambda: s.set_sources_weighted("p", idx1, w1, 0, np.ones((3, 2))), "does not match 1 source(s)")
    # weights, range, vars
    two = np.array([[[1, 1, 1], [2, 1, 1]]], np.int64)
    refused(lambda: s.set_sources_weighted("p", two, [[1.0, np.nan]], 0, amp), "point 0 entry 1 has a non-finite weight")
    refused(lambda: s.set_receivers_weighted("p", two, [[np.inf, 1.0]], 0, 3), "point 0 entry 0 has a non-finite weight")
    refused(lambda: s.set_receivers_weighted("p", np.concatenate([two, two]), [[0.5, 0.5], [0.0, -0.0]], 0, 3),
            "every weight of point 1 is 0")
    out = np.array([[[36, 1, 1], [37, 1, 1]]], np.int64)
    refused(lambda: s.set_receivers_weighted("p", out, [[0.5, 0.5]], 0, 3), "receivers: point 0 entry 1 (weight 0.5)",
            "index 37 in dim 'x'", "[0,37)")
    refused(lambda: s.set_sources_weighted("p", [[[0, -1, 0], [0, 0, 0]]], [[0.25, 0.75]], 0, amp), "sources: point 0 entry 0")
    s.set_receivers_weighted("p", out, [[1.0, 0.0]], 0, 3)          # a zero-weight entry may lie outside: it is dropped
    s.new_var("wm", ["t", "x", "y", "z", "m"])
    refused(lambda: s.set_sources_weighted("wm", idx1, w1, 0, amp), "misc dim 'm'")
    s.new_var("w4", ["t", "x", "y", "z"])
    refused(lambda: s.set_receivers_weighted("w4", idx1, w1, 0, 3), "'w4' is not written by any stage")
    refused(lambda: s.set_receivers_weighted("v", idx1, w1, 0, 3), "'v' has no step dim")
    s.close()


def test_range_waits_for_the_geometry():
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec((16, 16, 16))
    idx, w = capi.trilinear([[15.5, 3.0, 3.0]])
    s.set_receivers_weighted("p", idx, w, 0, 2)                     # not checked yet: no geometry
    refused(s.plan_geometry, "receivers: point 0 entry 4", "index 16 in dim 'x'")
    idx, w = capi.trilinear([[15.0, 15.0, 15.0]])                  # on the last plane: the outer entries weigh 0
    s.set_receivers_weighted("p", idx, w, 0, 2)
    s.plan_geometry()
    _, owned = s.get_traces()
    assert owned.tolist() == [True]
    s.close()


def test_source_var_on_a_rank_grid_must_be_written_by_the_last_stage():
    s = planned("awp_elastic", n=(24, 16, 32), grid=(2, 1, 1))
    idx, w = capi.trilinear([[5.5, 5.5, 5.5]])
    refused(lambda: s.set_sources_weighted("vel_x", idx, w, 0, np.ones((2, 1))), "source var 'vel_x' must be written by the last stage")
    s.set_sources_weighted("stress_xx", idx, w, 0, np.ones((2, 1)))
    s.close()


def test_straddling_receiver_on_a_var_not_written_by_the_last_stage():
    """awp_elastic: stage 1 writes the velocities, stage 2 the stresses.  A velocity receiver inside one rank is fine; one whose
    support crosses the x interface is refused on every rank; a stress receiver crossing it is accepted."""
    n, grid = (24, 16, 32), (2, 1, 1)
    for r in range(2):
        s = planned("awp_elastic", n=n, grid=grid, rank=r)
        idx, w = capi.trilinear([[5.5, 5.5, 5.5], [17.25, 3.0, 9.5]])
        s.set_receivers_weighted("vel_x", idx, w, 0, 2)
        idx, w = capi.trilinear([[11.5, 5.5, 5.5]])                 # x 11 | 12 is the interface
        refused(lambda: s.set_receivers_weighted("vel_x", idx, w, 0, 2), "receiver 0 straddles a rank interface",
                "'vel_x' is not written by the last stage")
        s.set_receivers_weighted("stress_xx", idx, w, 0, 2)
        _, owned = s.get_traces()
        assert owned.tolist() == [r == 0]
        s.close()


def one_slot_written_var():
    """(stencil, var) of a registered 3-D solution whose written var keeps a single step slot, if there is one."""
    for i in range(capi.lib().yb_num_stencils()):
        name = capi.lib().yb_stencil_name(i).decode()
        try:
            s = planned(name, n=(24, 24, 24))
        except capi.YaskError:
            continue
        try:
            for v in s.get_vars():
                vi = v.info
                if vi.is_output and vi.has_step and vi.step_alloc == 1:
                    return name, vi.name.decode()
        finally:
            s.close()
    return None


def test_halo_receiver_on_a_one_slot_single_stage_var():
    found = one_slot_written_var()
    if found is None:
        pytest.skip("no registered 3-D solution has a one-slot written var")
    name, var = found
    s = planned(name, n=(24, 24, 24), grid=(2, 1, 1))
    idx, w = capi.trilinear([[11.5, 5.0, 5.0]])
    with pytest.raises(capi.YaskError) as e:
        s.set_receivers_weighted(var, idx, w, 0, 2)
    s.close()
    msg = str(e.value)
    # a two-stage solution is accepted; a one-stage one with one slot is refused with the slot rule
    assert "keeps one step slot" in msg or "not written by the last stage" in msg or "halo" in msg, msg


def test_corner_receiver_on_a_face_only_var():
    """iso3dfd's p exchanges with face neighbours only: a receiver within one cell of both the x and the y interface reads a
    cell of the diagonal neighbour, which no exchange refreshes.  Every rank refuses it, naming the receiver, the entry and the
    missing edge exchange."""
    n, grid = (37, 29, 23), (2, 2, 1)
    for r in range(4):
        s = planned(n=n, grid=grid, rank=r)
        idx, w = capi.trilinear([[5.0, 5.0, 5.0], [18.5, 14.5, 7.0]])       # interfaces after x = 18 and y = 14
        refused(lambda: s.set_receivers_weighted("p", idx, w, 0, 2), "receiver 1 entry 6", "direction (1,1,0)", "edge exchange")
        idx, w = capi.trilinear([[18.5, 10.0, 7.0], [10.0, 14.5, 7.0]])     # one interface each: face exchanges
        s.set_receivers_weighted("p", idx, w, 0, 2)
        s.close()


def test_receiver_beyond_the_halo_is_refused():
    s = planned(n=(37, 29, 23), grid=(2, 1, 1), rank=1)
    idx = np.array([[[10, 3, 3], [19 + 8, 3, 3]]], np.int64)             # 9 cells past the interface; p's halo is 8
    refused(lambda: s.set_receivers_weighted("p", idx, [[0.5, 0.5]], 0, 2), "receiver 0 entry 1", "beyond var 'p''s halo of 8")
    idx = np.array([[[10, 3, 3], [19 + 7, 3, 3]]], np.int64)
    s.set_receivers_weighted("p", idx, [[0.5, 0.5]], 0, 2)
    s.close()


@pytest.mark.parametrize("fused_pair", [True, False])
def test_fused_pair_rank_grid_is_refused(fused_pair):
    opts = (("block_steps", 2), ("mega_block_steps", 2)) if fused_pair else (("block_steps", 2),)
    s = planned(n=(64, 48, 96), grid=(2, 1, 1), rank=0, radius=1, opts=opts)
    idx, w = capi.trilinear([[3.5, 3.5, 3.5]])
    if fused_pair:
        refused(lambda: s.set_sources_weighted("p", idx, w, 0, np.ones((2, 1))), "fused-pair", "mega_block_steps")
        refused(lambda: s.set_receivers_weighted("p", idx, w, 0, 2), "fused-pair")
    else:
        s.set_sources_weighted("p", idx, w, 0, np.ones((2, 1)))
        s.set_receivers_weighted("p", idx, w, 0, 2)
    s.close()


def receiver_positions(n, grid):
    """Random positions, and positions within one cell of every interface of an uneven split, on one interface at a time."""
    rng = np.random.default_rng(11)
    pos = [list(rng.uniform(0, np.array(n) - 1)) for _ in range(60)]
    for d in range(3):
        if grid[d] == 1:
            continue
        per = (n[d] + grid[d] - 1) // grid[d]
        for r in range(1, grid[d]):
            for x in (r * per - 1.0, r * per - 0.5, r * per - 0.01, float(r * per), r * per + 0.5):
                p = [m / 3 + 0.25 for m in n]
                p[d] = x
                pos.append(p)
    pos += [[0.0, 0.0, 0.0], [n[0] - 1.0, n[1] - 1.0, n[2] - 1.0]]
    # a receiver straddling two split dims needs an edge exchange: keep those out here
    def straddles(p, d):
        per = (n[d] + grid[d] - 1) // grid[d]
        return grid[d] > 1 and np.floor(p[d]) % per == per - 1 and p[d] != np.floor(p[d]) and np.floor(p[d]) < n[d] - 1
    return [p for p in pos if sum(straddles(p, d) for d in range(3)) <= 1]


@pytest.mark.parametrize("grid", [(2, 1, 1), (1, 2, 1), (1, 1, 2), (2, 2, 1), (3, 1, 1)])
def test_every_receiver_owned_by_exactly_one_rank(grid):
    n = (37, 29, 23)          # odd sizes: the last rank of a split dim is smaller
    pos = receiver_positions(n, grid)
    idx, w = capi.trilinear(pos)
    world = int(np.prod(grid))
    masks, groups = [], []
    for r in range(world):
        s = planned(n=n, grid=grid, rank=r)
        s.set_receivers_weighted("p", idx, w, 0, 3)
        s.set_sources_weighted("p", idx[-4:], w[-4:], 0, np.zeros((2, 4)))    # point_groups is read through 256 bytes
        traces, owned = s.get_traces()
        assert traces.shape == (3, len(pos))
        first, size = s.get_first_rank_domain_index_vec(), s.get_rank_domain_size_vec()
        mine = np.array([all(f <= int(np.floor(x)) < f + m for x, f, m in zip(p, first, size)) for p in pos])
        assert np.array_equal(owned, mine), r          # the rank of floor(pos), the first (nonzero) entry, owns it
        masks.append(owned)
        g = s.get_option("point_groups")
        groups += [tuple(map(int, e.split("/"))) for grp in g.split(";") if grp for e in grp.split(",")]
        s.close()
    assert np.array_equal(np.sum(masks, axis=0), np.ones(len(pos)))
    # every nonzero source entry is applied by exactly one rank
    want = sorted((i, q) for i in range(4) for q in range(8) if w[len(pos) - 4 + i, q] != 0)
    assert sorted(groups) == want


def test_groups_of_duplicate_support_points():
    s = planned(n=(16, 12, 20))
    idx = np.array([[[1, 1, 1], [2, 2, 2]], [[2, 2, 2], [1, 1, 1]], [[3, 3, 3], [1, 1, 1]], [[4, 4, 4], [2, 2, 2]]], np.int64)
    w = np.array([[0.5, 0.5], [0.25, 0.0], [1.0, 2.0], [0.0, 3.0]])
    s.set_sources_weighted("p", idx, w, 2, np.ones((3, 4)))
    # groups in order of first appearance, entries in (source, entry) order; zero weights are dropped
    assert s.get_option("point_groups") == "0/0,2/1;0/1,1/0,3/1;2/0"
    # k = 1: one entry per source, written i/0
    s.set_sources_weighted("p", idx[:, :1], np.ones((4, 1)), 0, np.ones((1, 4)))
    assert s.get_option("point_groups") == "0/0;1/0;2/0;3/0"
    # an on-grid set replaces it and is written as before
    s.set_sources("p", [[1, 1, 1], [1, 1, 1]], 0, np.ones((1, 2)))
    assert s.get_option("point_groups") == "0,1"
    s.clear_points()
    assert s.get_option("point_groups") == ""
    s.close()


def test_two_dim_solution():
    s = capi.Solution("wave2d")
    s.set_overall_domain_size_vec((20, 30))
    s.plan_geometry()
    idx, w = capi.trilinear([[3.5, 28.25], [19.0, 0.0]])
    assert idx.shape == (2, 4, 2)
    s.set_sources_weighted("e", idx, w, 0, np.ones((2, 2)))
    s.set_receivers_weighted("u", idx, w, 1, 3)
    refused(lambda: s.set_receivers_weighted("u", np.zeros((1, 4, 3), np.int64), np.ones((1, 4)), 1, 3), "(n, k, 2)")
    _, owned = s.get_traces()
    assert owned.tolist() == [True, True]
    assert s.get_option("point_groups") == "0/0;0/1;0/2;0/3;1/0"
    s.close()


MOD = glob.glob(os.path.join(ROOT, "yask_b200", "lib", "python", "iso3dfd", "yask_kernel*.so"))


@pytest.mark.skipif(not MOD, reason="python module not built")
def test_yask_kernel_trilinear_matches_capi():
    script = textwrap.dedent("""
        import yask_kernel as yk
        idx, w = yk.yk_trilinear([[1.25, 2.5, 3.0], [-0.5, 0.0, 7.75]])
        print(repr((idx, w)))
        try:
            yk.yk_trilinear([[float("nan"), 1.0, 1.0]])
            raise SystemExit("a NaN position was accepted")
        except RuntimeError as e:
            assert "non-finite" in str(e), e
    """)
    env = dict(os.environ, PYTHONPATH=os.path.dirname(MOD[0]))
    r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    idx, w = eval(r.stdout.strip())
    ri, rw = capi.trilinear([[1.25, 2.5, 3.0], [-0.5, 0.0, 7.75]])
    assert idx == ri.tolist() and w == rw.tolist()
