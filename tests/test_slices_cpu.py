"""CPU: slice recorders are validated and planned on the host, before anything reaches a device -- refusals that name the
problem, frame shapes, the fused-pair rank-grid refusal, and each point of a decimated box owned by exactly one rank of an
uneven grid."""
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
    box = ([1, 1, 1], [5, 5, 5])
    refused(lambda: s.add_slice("nope", *box, 0, 3), "'nope' not found")
    refused(lambda: s.add_slice("v", *box, 0, 3), "'v' has no step dim")           # iso3dfd's velocity: no step dim
    s.new_var("w2", ["t", "x", "y"])
    refused(lambda: s.add_slice("w2", *box, 0, 3), "'w2' lacks domain dim 'z'")
    s.new_var("wm", ["t", "x", "y", "z", "m"])
    refused(lambda: s.add_slice("wm", *box, 0, 3), "misc dim 'm'")
    s.new_var("w4", ["t", "x", "y", "z"])
    refused(lambda: s.add_slice("w4", *box, 0, 3), "'w4' is not written by any stage")
    refused(lambda: s.add_slice("p", [0, 0, 0], [37, 3, 3], 0, 3), "outside the overall domain [0,37)", "dim 'x'")
    refused(lambda: s.add_slice("p", [0, -1, 0], [3, 3, 3], 0, 3), "outside the overall domain [0,29)", "halo")   # a halo cell
    refused(lambda: s.add_slice("p", [0, 0, 0], [3, 3, 23 + 4], 0, 3), "outside the overall domain")              # a pad cell
    refused(lambda: s.add_slice("p", [4, 0, 0], [3, 3, 3], 0, 3), "first index 4 is past last index 3 in dim 'x'")
    refused(lambda: s.add_slice("p", *box, 0, 3, stride=[1, 0, 1]), "stride 0 in dim 'y' is less than 1")
    refused(lambda: s.add_slice("p", *box, 0, 3, stride=[1, 1, -2]), "stride -2 in dim 'z' is less than 1")
    refused(lambda: s.add_slice("p", *box, 0, 3, every=0), "every = 0 is less than 1")
    refused(lambda: s.add_slice("p", *box, 0, 0), "nrows = 0 is less than 1")
    refused(lambda: s.add_slice("p", [1, 1], [2, 2], 0, 3), "3 domain index")
    refused(lambda: s.set_option("slice_launches", 3), "read-only")
    refused(lambda: s.get_slice_frames(0), "no slice recorder 0")
    # a refused recorder leaves nothing behind; a valid one is accepted and gets id 0
    assert s.get_option("slice_launches") == "0"
    assert s.add_slice("p", [0, 0, 0], [36, 28, 22], 0, 3) == 0
    assert s.add_slice("p", [1, 2, 3], [1, 2, 3], 5, 1) == 1
    s.clear_slices()
    assert s.add_slice("p", [1, 2, 3], [1, 2, 3], 5, 1) == 0          # ids restart after clear_slices()
    s.close()


def test_frames_past_a_64_bit_byte_count_are_refused():
    """nrows x box points x element bytes must fit a 64-bit count: a product that wraps would size the frames wrongly."""
    s = planned()
    refused(lambda: s.add_slice("p", [0, 0, 0], [36, 28, 22], 0, 2 ** 61), "rows of the decimated box (37 x 29 x 23 points)",
            "overflow")
    refused(lambda: s.add_slice("p", [0, 0, 0], [0, 0, 0], 0, 2 ** 62), "overflow")      # 1 point, 4-byte elements
    # 2^62 bytes fit the count: accepted here, and refused by prepare when the device cannot allocate them
    assert s.add_slice("p", [0, 0, 0], [0, 0, 0], 0, 2 ** 60) == 0
    s.close()


def test_checks_wait_for_the_geometry():
    """Before the rank geometry is known only the var and the arguments can be checked; the range is checked once it is."""
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec((16, 16, 16))
    refused(lambda: s.add_slice("v", [1, 1, 1], [2, 2, 2], 0, 1), "no step dim")
    s.add_slice("p", [0, 0, 0], [99, 0, 0], 0, 1)
    refused(s.plan_geometry, "slice: box [0, 99] in dim 'x'", "outside the overall domain [0,16)")
    s.clear_slices()
    s.plan_geometry()
    refused(lambda: s.add_slice("p", [0, 16, 0], [0, 16, 0], 0, 2), "dim 'y'", "outside the overall domain")
    s.close()


@pytest.mark.parametrize("radius", [1, 2])
def test_fused_pair_rank_grid_is_refused(radius):
    """Refused on every rank of the grid, from plan_geometry() on, whether the recorder comes before or after it."""
    grid, n = (2, 1, 1), (64, 48, 96)
    opts = (("block_steps", 2), ("mega_block_steps", 2))
    for r in range(2):
        s = planned(n=n, grid=grid, rank=r, radius=radius, opts=opts)
        refused(lambda: s.add_slice("p", [3, 3, 3], [40, 3, 90], 0, 2), "fused-pair", "mega_block_steps")
        s.close()
        s = capi.Solution("iso3dfd", radius=radius)
        s.set_overall_domain_size_vec(n)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        for k, v in opts:
            s.set_option(k, v)
        s.add_slice("p", [3, 3, 3], [40, 3, 90], 0, 2)
        refused(s.plan_geometry, "fused-pair")
        s.close()
    # the same grid exchanging once per step, and one rank with pairs, take recorders
    for o, g in (((("block_steps", 2),), grid), (opts, None)):
        s = planned(n=n, grid=g, rank=0, radius=radius, opts=o)
        s.add_slice("p", [3, 3, 3], [40, 3, 90], 0, 2)
        s.close()


@pytest.mark.parametrize("first,last,stride", [
    ([0, 0, 0], [36, 28, 22], [1, 1, 1]),
    ([3, 1, 5], [36, 28, 22], [2, 3, 4]),
    ([3, 1, 5], [35, 27, 21], [2, 3, 4]),
    ([10, 0, 0], [10, 28, 22], [1, 1, 1]),
    ([0, 0, 7], [36, 28, 7], [1, 2, 1]),
    ([5, 5, 5], [5, 5, 5], [7, 7, 7]),
    ([0, 0, 0], [36, 28, 22], [40, 30, 25]),
])
def test_frame_shapes(first, last, stride):
    s = planned()
    rid = s.add_slice("p", first, last, 0, 4, stride=stride)
    frames, owned = s.get_slice_frames(rid)
    want = tuple((b - a) // k + 1 for a, b, k in zip(first, last, stride))
    assert frames.shape == (4,) + want and frames.dtype == np.float32
    assert owned.shape == want and owned.all()
    assert not frames.any()
    s.close()


def decimated_mask(first, last, stride, lo, size):
    """The points of the decimated box inside the rank box [lo, lo + size), per dim, as a boolean array."""
    axes = []
    for a, b, k, o, m in zip(first, last, stride, lo, size):
        g = np.arange(a, b + 1, k)
        axes.append((g >= o) & (g < o + m))
    out = np.ones([len(a) for a in axes], bool)
    for d, a in enumerate(axes):
        out &= a.reshape([-1 if k == d else 1 for k in range(len(axes))])
    return out


BOXES = [([0, 0, 0], [36, 28, 22], [1, 1, 1]),          # the whole domain
         ([1, 2, 3], [36, 27, 22], [2, 3, 4]),          # decimated, odd first: the phase differs between ranks
         ([17, 0, 0], [20, 28, 22], [3, 1, 1]),         # crosses the x interface of an uneven 2-way split
         ([0, 13, 0], [36, 16, 22], [5, 2, 1]),         # crosses the y interface
         ([18, 14, 11], [18, 14, 11], [1, 1, 1]),       # one point
         ([0, 0, 9], [36, 28, 9], [7, 5, 1])]           # a z-plane


@pytest.mark.parametrize("grid", [(2, 1, 1), (3, 1, 1), (1, 2, 1), (2, 2, 2)])
def test_ownership_on_uneven_grids(grid):
    n = (37, 29, 23)              # odd sizes: the last rank of a split dim is smaller
    world = int(np.prod(grid))
    for first, last, stride in BOXES:
        masks = []
        for r in range(world):
            s = planned(n=n, grid=grid, rank=r)
            rid = s.add_slice("p", first, last, 0, 2, stride=stride)
            frames, owned = s.get_slice_frames(rid)
            want = decimated_mask(first, last, stride, s.get_first_rank_domain_index_vec(), s.get_rank_domain_size_vec())
            assert np.array_equal(owned, want), (r, first, stride)
            masks.append(owned)
            s.close()
        total = np.sum(masks, axis=0)
        assert (total == 1).all(), (first, stride)        # disjoint, and together the whole decimated box


def test_recorders_before_the_geometry_are_planned_with_it():
    grid, n = (2, 1, 1), (37, 29, 23)
    for r in range(2):
        s = capi.Solution("iso3dfd")
        s.set_overall_domain_size_vec(n)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        rid = s.add_slice("p", [1, 0, 0], [36, 28, 22], 0, 1, stride=[3, 1, 1])
        refused(lambda: s.get_slice_frames(rid), "rank geometry is not known yet")
        s.plan_geometry()
        _, owned = s.get_slice_frames(rid)
        lo, m = s.get_first_rank_domain_index_vec(), s.get_rank_domain_size_vec()
        assert np.array_equal(owned, decimated_mask([1, 0, 0], [36, 28, 22], [3, 1, 1], lo, m))
        s.close()


def test_one_and_two_dim_solutions():
    s = capi.Solution("wave2d")
    s.set_overall_domain_size_vec((20, 30))
    s.plan_geometry()
    rid = s.add_slice("u", [1, 0], [19, 29], 0, 3, stride=[2, 3])
    frames, owned = s.get_slice_frames(rid)
    assert frames.shape == (3, 10, 10) and owned.all()
    refused(lambda: s.add_slice("u", [1, 0, 0], [19, 29, 0], 0, 3), "2 domain index")
    s.close()
    s = capi.Solution("test_1d")
    s.set_overall_domain_size_vec((50,))
    s.set_num_ranks_vec((2,))
    s.set_rank_index_vec((1,))
    s.plan_geometry()
    var = [v.get_name() for v in s.get_vars() if v.info.is_output][0]
    rid = s.add_slice(var, [3], [49], 0, 2, stride=[4])
    frames, owned = s.get_slice_frames(rid)
    assert frames.shape == (2, 12)
    assert owned.tolist() == [g >= 25 for g in range(3, 50, 4)]
    s.close()
