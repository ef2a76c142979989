"""CPU: point sources and receivers are planned and validated on the host, before anything reaches a device -- refusals,
the fused-pair rank-grid refusal, ownership of every point by exactly one rank of a grid, and the list order of several
sources on one point."""
import itertools

import numpy as np
import pytest

from yask_b200 import capi, multi


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


def test_refusals_name_the_problem():
    s = planned()
    amp = np.ones((3, 1))
    refused(lambda: s.set_sources("nope", [[1, 1, 1]], 0, amp), "'nope' not found")
    refused(lambda: s.set_sources("v", [[1, 1, 1]], 0, amp), "'v' has no step dim")        # iso3dfd's velocity: no step dim
    s.new_var("w2", ["t", "x", "y"])
    refused(lambda: s.set_receivers("w2", [[1, 1, 1]], 0, 3), "'w2' lacks domain dim 'z'")
    s.new_var("wm", ["t", "x", "y", "z", "m"])
    refused(lambda: s.set_sources("wm", [[1, 1, 1]], 0, amp), "misc dim 'm'")
    s.new_var("w4", ["t", "x", "y", "z"])
    refused(lambda: s.set_sources("w4", [[1, 1, 1]], 0, amp), "'w4' is not written by any stage")
    refused(lambda: s.set_sources("p", [[37, 0, 0]], 0, amp), "outside the overall domain [0,37)", "dim 'x'")
    refused(lambda: s.set_receivers("p", [[0, -1, 0]], 0, 3), "outside the overall domain [0,29)", "halo")   # a halo cell
    refused(lambda: s.set_receivers("p", [[0, 0, 23 + 4]], 0, 3), "outside the overall domain")               # a pad cell
    refused(lambda: s.set_sources("p", [[1, 1]], 0, amp), "3 domain index")
    refused(lambda: s.set_sources("p", [[1, 1, 1], [2, 2, 2]], 0, amp), "does not match 2 source point(s)")
    refused(lambda: s.set_sources("p", [[1, 1, 1]], 0, np.ones(4)), "does not match")
    refused(lambda: s.set_option("point_launches", 3), "read-only")
    # a refused set leaves nothing behind; a valid one is accepted
    assert s.get_option("point_launches") == "0" and s.get_option("point_groups") == ""
    s.set_sources("p", [[36, 28, 22]], 0, amp)
    assert s.get_option("point_groups") == "0"
    s.close()


def test_checks_wait_for_the_geometry():
    """Before the rank geometry is known only the var and the shapes can be checked; the range is checked once it is."""
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec((16, 16, 16))
    refused(lambda: s.set_sources("v", [[1, 1, 1]], 0, np.ones((1, 1))), "no step dim")
    s.set_sources("p", [[99, 0, 0]], 0, np.ones((1, 1)))
    refused(s.plan_geometry, "sources: point 0 has index 99 in dim 'x'", "outside the overall domain [0,16)")
    s.set_sources("p", [[15, 0, 0]], 0, np.ones((1, 1)))          # the geometry is known now: checked at once
    refused(lambda: s.set_receivers("p", [[0, 16, 0]], 0, 2), "receivers: point 0", "outside the overall domain")
    s.close()


@pytest.mark.parametrize("radius", [1, 2])
def test_fused_pair_rank_grid_is_refused(radius):
    s = planned(n=(64, 48, 96), grid=(2, 1, 1), rank=0, radius=radius, opts=(("block_steps", 2), ("mega_block_steps", 2)))
    refused(lambda: s.set_sources("p", [[3, 3, 3]], 0, np.ones((2, 1))), "fused-pair", "mega_block_steps")
    refused(lambda: s.set_receivers("p", [[3, 3, 3]], 0, 2), "fused-pair")
    s.close()
    # the same grid exchanging once per step, and one rank with pairs, take points
    for opts, grid in ((((("block_steps", 2),)), (2, 1, 1)), ((("block_steps", 2), ("mega_block_steps", 2)), None)):
        s = planned(n=(64, 48, 96), grid=grid, rank=0, radius=radius, opts=opts)
        s.set_sources("p", [[3, 3, 3]], 0, np.ones((2, 1)))
        s.close()


def grid_points(n):
    """Corners, faces, edges, both sides of every rank interface of an uneven split, and random points."""
    rng = np.random.default_rng(5)
    pts = [list(c) for c in itertools.product(*[(0, m - 1) for m in n])]
    for d in range(len(n)):
        for x in (0, n[d] // 2 - 1, n[d] // 2, (n[d] + 1) // 2, n[d] - 1):
            p = [m // 3 for m in n]
            p[d] = x
            pts.append(p)
    pts += rng.integers(0, n, size=(20, len(n))).tolist()
    return pts


@pytest.mark.parametrize("grid", [(2, 1, 1), (1, 2, 1), (2, 2, 2), (3, 1, 2)])
def test_every_point_owned_by_exactly_one_rank(grid):
    n = (37, 29, 23)         # odd sizes: the last rank of a split dim is smaller
    pts = grid_points(n)
    world = int(np.prod(grid))
    masks, groups = [], []
    for r in range(world):
        s = planned(n=n, grid=grid, rank=r)
        s.set_receivers("p", pts, 0, 4)
        s.set_sources("p", pts, 0, np.zeros((2, len(pts))))
        traces, owned = s.get_traces()
        assert traces.shape == (4, len(pts))
        first = s.get_first_rank_domain_index_vec()
        size = s.get_rank_domain_size_vec()
        mine = np.array([all(f <= x < f + m for x, f, m in zip(p, first, size)) for p in pts])
        assert np.array_equal(owned, mine), r          # halo copies of a neighbour's points are not owned
        masks.append(owned)
        g = s.get_option("point_groups")
        groups += [int(i) for grp in g.split(";") if grp for i in grp.split(",")]
        s.close()
    assert np.array_equal(np.sum(masks, axis=0), np.ones(len(pts)))      # the masks cover every receiver once
    assert sorted(groups) == list(range(len(pts)))                       # every source applied by one rank


def test_duplicate_sources_keep_list_order():
    s = planned(n=(16, 12, 20))
    pts = [[1, 2, 3], [4, 4, 4], [1, 2, 3], [0, 0, 0], [1, 2, 3], [4, 4, 4]]
    s.set_sources("p", pts, 2, np.ones((3, len(pts))))
    assert s.get_option("point_groups") == "0,2,4;1,5;3"
    s.clear_points()
    assert s.get_option("point_groups") == ""
    s.close()


def test_one_and_two_dim_solutions():
    s = capi.Solution("wave2d")
    s.set_overall_domain_size_vec((20, 30))
    s.plan_geometry()
    s.set_sources("e", [[0, 29], [19, 0]], 0, np.ones((2, 2)))
    s.set_receivers("u", [[5, 5]], 1, 3)
    refused(lambda: s.set_receivers("u", [[5, 5, 5]], 1, 3), "2 domain index")
    _, owned = s.get_traces()
    assert owned.tolist() == [True]
    s.close()
    s = capi.Solution("test_1d")
    s.set_overall_domain_size_vec((50,))
    s.plan_geometry()
    var = [v.get_name() for v in s.get_vars() if v.info.is_output][0]
    s.set_sources(var, [3, 49, 3], 0, np.ones((1, 3)))
    assert s.get_option("point_groups") == "0,2;1"
    s.close()
