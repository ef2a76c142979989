"""CPU: slice correlators and injectors fed from a recorder are checked on the host before anything reaches a device -- each
refusal names the field that differs, ids restart after clear, and the image's shape and owned mask follow the rank grid from
plan_geometry() on."""
import ctypes as C

import numpy as np
import pytest

from tests.test_slice_injectors_cpu import planned, refused
from yask_b200 import capi, multi

BOX = ([1, 1, 1], [30, 20, 17])


def source(n=(37, 29, 23), grid=None, rank=0, eb=4, box=BOX, nrows=4, stride=None, stencil="iso3dfd", var="p"):
    """A planned solution with one recorder (id 0): on a host without a device its frames never exist."""
    s = planned(stencil, n=n, grid=grid, rank=rank, eb=eb)
    assert s.add_slice(var, *box, 0, nrows, stride=stride) == 0
    return s


def test_correlator_refusals_name_the_problem():
    s, src = planned(), source()
    cor = s.add_slice_correlator
    refused(lambda: cor("nope", *BOX, 0, 4), "slice correlator", "'nope' not found")
    refused(lambda: cor("v", *BOX, 0, 4), "'v' has no step dim")
    refused(lambda: cor("p", *BOX, 0, 4, every=0), "slice correlator", "every = 0 is less than 1")
    refused(lambda: cor("p", *BOX, 0, 0), "nrows = 0 is less than 1")
    refused(lambda: cor("p", [0, 0, 0], [37, 3, 3], 0, 4), "slice correlator", "outside the overall domain [0,37)", "dim 'x'")
    refused(lambda: cor("p", *BOX, 0, 4, stride=[1, 0, 1]), "stride 0 in dim 'y' is less than 1")
    refused(lambda: cor("p", *BOX, 0, 4, reverse=2), "reverse = 2 is not 0 or 1")
    refused(lambda: cor("p", *BOX, 0, 4, src=src, src_id=1), "src_id 1 is not a slice recorder")
    refused(lambda: cor("p", *BOX, 0, 4, src=src, src_id=-1), "src_id -1 is not a slice recorder")
    refused(lambda: cor("p", *BOX, 0, 4, src=src, src_id=0, reverse=-1), "reverse = -1 is not 0 or 1")
    refused(lambda: cor("p", [1, 1, 2], [30, 20, 17], 0, 4, src=src, src_id=0), "box [2, 17] in dim 'z' differs from recorder 0's box [1, 17]")
    refused(lambda: cor("p", [1, 1, 1], [30, 19, 17], 0, 4, src=src, src_id=0), "box [1, 19] in dim 'y' differs")
    refused(lambda: cor("p", *BOX, 0, 4, src=src, src_id=0, stride=[2, 1, 1]), "stride 2 in dim 'x' differs from recorder 0's stride 1")
    refused(lambda: cor("p", *BOX, 0, 5, src=src, src_id=0), "nrows = 5 is more than the 4 rows of recorder 0")
    refused(lambda: cor("p", *BOX, 0, 4, src=src, src_id=0), "source solution 'iso3dfd' is not prepared", "recorder 0 has no frames")
    refused(lambda: cor("p", *BOX, 0, 4, src=src), "needs src_id")
    refused(lambda: s.set_option("slice_correlator_launches", 3), "read-only")
    # a refused correlator leaves nothing behind; nrows below the recorder's and both row orders pass every check but the frames'
    assert s.get_option("slice_correlator_launches") == "0"
    refused(lambda: cor("p", *BOX, 2, 3, src=src, src_id=0, reverse=True, every=3), "is not prepared")
    assert cor("p", *BOX, 0, 4) == 0
    s.close()
    src.close()


def test_mismatched_solutions_are_refused():
    src = source()
    for eb, want in ((8, "element bytes 8 differ from the source solution's 4"),):
        s = planned(eb=eb)
        refused(lambda: s.add_slice_correlator("p", *BOX, 0, 4, src=src, src_id=0), want)
        s.close()
    s = planned("wave2d", n=(37, 29))
    refused(lambda: s.add_slice_correlator("u", [1, 1], [30, 20], 0, 4, src=src, src_id=0), "2 domain dims differ from the source solution's 3")
    s.close()
    s = planned(n=(37, 29, 24))
    refused(lambda: s.add_slice_correlator("p", *BOX, 0, 4, src=src, src_id=0), "overall domain size 24 in dim 'z' differs from the source solution's 23")
    s.close()
    src.close()
    # rank grids: the same grid and index on both sides, with the recorder's owned part
    n, grid = (37, 29, 23), (2, 1, 1)
    for r in range(2):
        src = source(n=n, grid=grid, rank=r)
        s = planned(n=n)
        refused(lambda: s.add_slice_correlator("p", *BOX, 0, 4, src=src, src_id=0), "num_ranks 1 in dim 'x' differs from the source solution's 2")
        s.close()
        s = planned(n=n, grid=grid, rank=1 - r)
        refused(lambda: s.add_slice_correlator("p", *BOX, 0, 4, src=src, src_id=0), f"rank index {1 - r} in dim 'x' differs from the source solution's {r}")
        s.close()
        s = planned(n=n, grid=(1, 2, 1), rank=r)
        refused(lambda: s.add_slice_correlator("p", *BOX, 0, 4, src=src, src_id=0), "num_ranks 1 in dim 'x' differs")
        s.close()
        s = planned(n=n, grid=grid, rank=r)
        refused(lambda: s.add_slice_correlator("p", *BOX, 0, 4, src=src, src_id=0), "is not prepared")
        s.close()
        src.close()


def test_geometry_is_needed_on_both_sides():
    src = source()
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec((37, 29, 23))
    refused(lambda: s.add_slice_correlator("p", *BOX, 0, 4, src=src, src_id=0), "this solution has no rank geometry yet")
    refused(lambda: s.add_slice_injector_from("p", *BOX, 0, 4, src, 0), "slice injector", "this solution has no rank geometry yet")
    s.plan_geometry()
    bare = capi.Solution("iso3dfd")
    bare.set_overall_domain_size_vec((37, 29, 23))
    bare.add_slice("p", *BOX, 0, 4)
    refused(lambda: s.add_slice_correlator("p", *BOX, 0, 4, src=bare, src_id=0), "the source solution has no rank geometry yet")
    # an autocorrelation needs neither: it is planned with the geometry, as a recorder is
    assert bare.add_slice_correlator("p", *BOX, 0, 4) == 0
    for x in (s, src, bare):
        x.close()


def test_injector_from_refusals():
    s, src = planned(), source()
    inj = s.add_slice_injector_from
    refused(lambda: inj("p", *BOX, 0, 4, src, 0, mode="replace"), "unknown mode 'replace'")
    refused(lambda: inj("p", *BOX, 0, 4, src, 3), "slice injector", "src_id 3 is not a slice recorder")
    refused(lambda: inj("p", *BOX, 0, 4, src, 0, stride=[1, 1, 2]), "slice injector", "stride 2 in dim 'z' differs")
    refused(lambda: inj("p", *BOX, 0, 9, src, 0), "nrows = 9 is more than the 4 rows of recorder 0")
    refused(lambda: inj("p", *BOX, 0, 4, src, 0, reverse=3), "reverse = 3 is not 0 or 1")
    refused(lambda: inj("p", *BOX, 0, 4, src, 0), "slice injector", "is not prepared")
    assert s.get_option("slice_injector_groups") == ""
    # the C ABI checks the mode and the source itself
    f, l, st = (C.c_int64 * 3)(*BOX[0]), (C.c_int64 * 3)(*BOX[1]), (C.c_int64 * 3)(1, 1, 1)
    rid = C.c_int64(-1)
    assert capi.lib().yb_solution_add_slice_injector_from(s._h, b"p", f, l, st, 0, 1, 2, 7, src._h, 0, 0, C.byref(rid)) < 0
    assert "unknown mode 7" in capi.lib().yb_last_error().decode()
    assert capi.lib().yb_solution_add_slice_injector_from(s._h, b"p", f, l, st, 0, 1, 2, 0, None, 0, 0, C.byref(rid)) < 0
    assert "null source solution" in capi.lib().yb_last_error().decode()
    assert capi.lib().yb_solution_add_slice_correlator(s._h, b"p", f, l, st, 0, 1, 2, None, 0, 5, C.byref(rid)) < 0
    assert "reverse = 5 is not 0 or 1" in capi.lib().yb_last_error().decode()
    s.close()
    src.close()


def test_ids_restart_after_clear_and_are_separate():
    s = planned()
    assert s.add_slice("p", *BOX, 0, 3) == 0
    assert s.add_slice_correlator("p", *BOX, 0, 3) == 0
    assert s.add_slice_correlator("p", [0, 0, 0], [36, 28, 22], 1, 5, stride=[2, 2, 2], every=2) == 1
    assert s.add_slice_injector("p", *BOX, 0, np.zeros((1, 30, 20, 17), np.float32)) == 0
    assert s.add_slice("p", *BOX, 0, 3) == 1
    s.clear_slice_correlators()
    assert s.add_slice_correlator("p", *BOX, 0, 3) == 0              # ids restart after clear_slice_correlators()
    s.clear_slices()
    s.clear_slice_injectors()
    assert s.add_slice_correlator("p", *BOX, 0, 3) == 1              # and the other clears leave the correlators alone
    refused(lambda: s.get_correlator_image(2), "no slice correlator 2")
    s.close()


@pytest.mark.parametrize("radius", [1, 2])
def test_fused_pair_rank_grid_is_refused(radius):
    grid, n = (2, 1, 1), (64, 48, 96)
    opts = (("block_steps", 2), ("mega_block_steps", 2))
    box = ([3, 3, 3], [40, 3, 90])
    for r in range(2):
        s = planned(n=n, grid=grid, rank=r, radius=radius, opts=opts)
        refused(lambda: s.add_slice_correlator("p", *box, 0, 2), "slice correlators", "fused-pair", "mega_block_steps")
        s.close()
        s = capi.Solution("iso3dfd", radius=radius)
        s.set_overall_domain_size_vec(n)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        for k, v in opts:
            s.set_option(k, v)
        s.add_slice_correlator("p", *box, 0, 2)
        refused(s.plan_geometry, "slice correlators", "fused-pair")
        s.close()
    for o, g in (((("block_steps", 2),), grid), (opts, None)):
        s = planned(n=n, grid=g, rank=0, radius=radius, opts=o)
        s.add_slice_correlator("p", *box, 0, 2)
        s.close()


@pytest.mark.parametrize("grid,n", [((3, 1, 1), (37, 29, 23)), ((2, 3, 1), (37, 29, 23)), ((1, 2, 2), (20, 29, 23)), ((3,), (50,))])
def test_image_shape_and_owned_mask_on_uneven_grids(grid, n):
    """Every point of the decimated box is owned by exactly one rank, the one whose domain holds it; the phase comes from the
    global first."""
    nd = len(n)
    first, last, stride = [1, 2, 0][:nd], [m - 1 for m in n], [2, 3, 5][:nd]
    shape = tuple((b - a) // k + 1 for a, b, k in zip(first, last, stride))
    count = np.zeros(shape, int)
    for r in range(int(np.prod(grid))):
        s = planned("test_1d" if nd == 1 else "iso3dfd", n=n, grid=grid, rank=r)
        var = "p" if nd == 3 else [v.get_name() for v in s.get_vars() if v.info.is_output][0]
        assert s.add_slice_correlator(var, first, last, 0, 1, stride=stride) == 0
        img, owned = s.get_correlator_image(0)
        assert img.shape == shape and owned.shape == shape and not img.any()
        lo = s.get_first_rank_domain_index_vec()
        hi = [capi.lib().yb_get_last_rank_domain_index(s._h, d) for d in range(nd)]
        g = np.meshgrid(*[np.arange(a, b + 1, k) for a, b, k in zip(first, last, stride)], indexing="ij")
        want = np.ones(shape, bool)
        for d in range(nd):
            want &= (g[d] >= lo[d]) & (g[d] <= hi[d])
        assert np.array_equal(owned, want), r
        count += owned
        s.close()
    assert (count == 1).all()
