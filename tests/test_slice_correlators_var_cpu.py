"""CPU: correlators whose b is a var of another solution (add_slice_correlator_var) are checked on the host before anything
reaches a device.  Each refusal names the field, and the checks run in a fixed order: the source is another solution, its var
passes the var rules, then element bytes, domain dims, overall domain, rank grid and rank index, and last that the source is
prepared (which needs a device)."""
import ctypes as C

import pytest

from tests.test_slice_injectors_cpu import planned, refused
from yask_b200 import capi

BOX = ([1, 1, 1], [30, 20, 17])


def test_refusals_in_order():
    s, src = planned(), planned()
    cor = s.add_slice_correlator_var
    # the consumer's own box, window and var come first, as for every correlator
    refused(lambda: cor("nope", *BOX, 0, 4, src, "p"), "slice correlator", "'nope' not found")
    refused(lambda: cor("p", *BOX, 0, 0, src, "p"), "nrows = 0 is less than 1")
    refused(lambda: cor("p", *BOX, 0, 4, src, "p", image_dtype="float16"), "image type float16 is not allowed")
    # 1. the source is another solution
    refused(lambda: cor("p", *BOX, 0, 4, s, "p"), "slice correlator: src:", "another solution, not this one")
    refused(lambda: cor("p", *BOX, 0, 4, None, "p"), "slice correlator: src:", "null source solution")
    # 2. its var exists and passes the var rules; this comes before a mismatch of the solutions
    refused(lambda: cor("p", *BOX, 0, 4, src, "nope"), "slice correlator: src_var:", "'nope' not found in solution 'iso3dfd'")
    refused(lambda: cor("p", *BOX, 0, 4, src, "v"), "src_var:", "'v' has no step dim")
    s8 = planned(eb=8)
    refused(lambda: s8.add_slice_correlator_var("p", *BOX, 0, 4, src, "v"), "src_var:", "'v' has no step dim")
    # 3. element bytes, before the domain dims
    refused(lambda: s8.add_slice_correlator_var("p", *BOX, 0, 4, src, "p"), "element bytes 8 differ from the source solution's 4")
    w8 = planned("wave2d", n=(37, 29))
    refused(lambda: s8.add_slice_correlator_var("p", *BOX, 0, 4, w8, "u"), "element bytes 8 differ from the source solution's 4")
    # 4. the domain dims
    w = planned("wave2d", n=(37, 29))
    refused(lambda: w.add_slice_correlator_var("u", [1, 1], [30, 20], 0, 4, src, "p"), "2 domain dims differ from the source solution's 3")
    # 5. the overall domain, before the rank grid
    big = planned(n=(37, 29, 24), grid=(2, 1, 1))
    refused(lambda: big.add_slice_correlator_var("p", *BOX, 0, 4, src, "p"),
            "overall domain size 24 in dim 'z' differs from the source solution's 23")
    # 6. the source is prepared: the last check a host without a device reaches
    refused(lambda: cor("p", *BOX, 0, 4, src, "p"), "source solution 'iso3dfd' is not prepared")
    refused(lambda: cor("p", *BOX, 2, 4, src, "p", src_t0=7, every=3, stride=[2, 1, 3], image_dtype="float64"), "is not prepared")
    # a refused correlator leaves nothing behind
    assert s.get_option("slice_correlator_launches") == "0"
    refused(lambda: s.get_correlator_image(0), "no slice correlator 0")
    for x in (s, src, s8, w8, w, big):
        x.close()


def test_rank_grid_and_index_must_match():
    n, grid = (37, 29, 23), (2, 1, 1)
    for r in range(2):
        src = planned(n=n, grid=grid, rank=r)
        s = planned(n=n)
        refused(lambda: s.add_slice_correlator_var("p", *BOX, 0, 4, src, "p"), "num_ranks 1 in dim 'x' differs from the source solution's 2 (rank grid)")
        s.close()
        s = planned(n=n, grid=grid, rank=1 - r)
        refused(lambda: s.add_slice_correlator_var("p", *BOX, 0, 4, src, "p"), f"rank index {1 - r} in dim 'x' differs from the source solution's {r}")
        s.close()
        s = planned(n=n, grid=(1, 2, 1), rank=r)
        refused(lambda: s.add_slice_correlator_var("p", *BOX, 0, 4, src, "p"), "num_ranks 1 in dim 'x' differs")
        s.close()
        s = planned(n=n, grid=grid, rank=r)
        refused(lambda: s.add_slice_correlator_var("p", *BOX, 0, 4, src, "p"), "is not prepared")
        s.close()
        src.close()


def test_storage_may_differ():
    """Pads, halos and another stencil of the same dims pass every check a host can make: only the source's preparation is missing."""
    s = planned()
    for src in (planned("iso3dfd_sponge"), planned(radius=2), planned(opts=(("block_steps", 2),))):
        refused(lambda: s.add_slice_correlator_var("p", *BOX, 0, 4, src, "p"), "is not prepared")
        src.close()
    src = capi.Solution("iso3dfd")
    src.set_overall_domain_size_vec((37, 29, 23))
    for d, m in enumerate((20, 24, 40)):
        capi._chk(capi.lib().yb_set_min_pad_size(src._h, d, m))
    src.plan_geometry()
    refused(lambda: s.add_slice_correlator_var("p", *BOX, 0, 4, src, "p"), "is not prepared")
    src.close()
    s.close()


def test_geometry_is_needed_on_both_sides():
    src = planned()
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec((37, 29, 23))
    refused(lambda: s.add_slice_correlator_var("p", *BOX, 0, 4, src, "p"), "this solution has no rank geometry yet")
    s.plan_geometry()
    bare = capi.Solution("iso3dfd")
    bare.set_overall_domain_size_vec((37, 29, 23))
    refused(lambda: s.add_slice_correlator_var("p", *BOX, 0, 4, bare, "p"), "the source solution has no rank geometry yet")
    for x in (s, src, bare):
        x.close()


@pytest.mark.parametrize("radius", [1, 2])
def test_fused_pair_rank_grid_is_refused(radius):
    """A consumer on a rank grid in fused-pair mode is refused from plan_geometry() on, before the source is looked at further."""
    grid, n = (2, 1, 1), (64, 48, 96)
    opts = (("block_steps", 2), ("mega_block_steps", 2))
    box = ([3, 3, 3], [40, 3, 90])
    for r in range(2):
        src = planned(n=n, grid=grid, rank=r, radius=radius)
        s = planned(n=n, grid=grid, rank=r, radius=radius, opts=opts)
        refused(lambda: s.add_slice_correlator_var("p", *box, 0, 2, src, "p"), "slice correlators", "fused-pair", "mega_block_steps")
        s.close()
        # without the pair mode, only the source's preparation is missing
        s = planned(n=n, grid=grid, rank=r, radius=radius, opts=opts[:1])
        refused(lambda: s.add_slice_correlator_var("p", *box, 0, 2, src, "p"), "is not prepared")
        s.close()
        src.close()


def test_ids_are_shared_with_the_other_correlators():
    """A refused var correlator takes no id: the frame correlators and autocorrelations keep counting from where they were."""
    s, src = planned(), planned()
    assert s.add_slice_correlator("p", *BOX, 0, 3) == 0
    refused(lambda: s.add_slice_correlator_var("p", *BOX, 0, 3, src, "p"), "is not prepared")
    assert s.add_slice_correlator("p", *BOX, 1, 2, every=2) == 1
    s.clear_slice_correlators()
    refused(lambda: s.add_slice_correlator_var("p", *BOX, 0, 3, src, "p"), "is not prepared")
    assert s.add_slice_correlator("p", *BOX, 0, 3) == 0
    s.close()
    src.close()


def test_c_abi_checks_its_arguments():
    s, src = planned(), planned()
    f, l, st = (C.c_int64 * 3)(*BOX[0]), (C.c_int64 * 3)(*BOX[1]), (C.c_int64 * 3)(1, 1, 1)
    rid = C.c_int64(-1)
    L = capi.lib()
    assert L.yb_solution_add_slice_correlator_var(s._h, b"p", f, l, st, 0, 1, 2, src._h, None, 0, 0, C.byref(rid)) < 0
    assert "src_var: null var name" in L.yb_last_error().decode()
    assert L.yb_solution_add_slice_correlator_var(s._h, b"p", f, l, st, 0, 1, 2, None, b"p", 0, 0, C.byref(rid)) < 0
    assert "null source solution" in L.yb_last_error().decode()
    assert L.yb_solution_add_slice_correlator_var(s._h, b"p", f, l, st, 0, 1, 2, src._h, b"p", 0, 9, C.byref(rid)) < 0
    assert "unknown image type 9" in L.yb_last_error().decode()
    assert rid.value == -1
    s.close()
    src.close()
