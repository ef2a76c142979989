"""CPU: slice injectors are validated, planned and grouped on the host, before anything reaches a device -- refusals that name the
problem and leave nothing behind, ids, the fused-pair and last-stage rank-grid refusals, and the launch groups that keep id
order where boxes on one var overlap."""
import ctypes as C

import numpy as np
import pytest

from yask_b200 import capi, multi


def planned(stencil="iso3dfd", n=(37, 29, 23), grid=None, rank=0, radius=0, eb=4, opts=()):
    s = capi.Solution(stencil, radius=radius, elem_bytes=eb)
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


def frames(first, last, nrows=2, stride=None):
    stride = stride or [1] * len(first)
    return np.zeros((nrows,) + tuple((b - a) // k + 1 for a, b, k in zip(first, last, stride)), np.float32)


def test_refusals_name_the_problem():
    s = planned()
    box = ([1, 1, 1], [5, 5, 5])
    fr = frames(*box)
    inj = s.add_slice_injector
    refused(lambda: inj("nope", *box, 0, fr), "slice injector", "'nope' not found")
    refused(lambda: inj("v", *box, 0, fr), "'v' has no step dim")             # iso3dfd's velocity: no step dim
    s.new_var("w2", ["t", "x", "y"])
    refused(lambda: inj("w2", *box, 0, fr), "'w2' lacks domain dim 'z'")
    s.new_var("wm", ["t", "x", "y", "z", "m"])
    refused(lambda: inj("wm", *box, 0, fr), "misc dim 'm'")
    s.new_var("w4", ["t", "x", "y", "z"])
    refused(lambda: inj("w4", *box, 0, fr), "'w4' is not written by any stage")
    refused(lambda: inj("p", [0, 0, 0], [37, 3, 3], 0, frames([0, 0, 0], [37, 3, 3])), "outside the overall domain [0,37)", "dim 'x'")
    refused(lambda: inj("p", [0, -1, 0], [3, 3, 3], 0, frames([0, -1, 0], [3, 3, 3])), "outside the overall domain [0,29)", "halo")
    refused(lambda: inj("p", [0, 0, 0], [3, 3, 27], 0, frames([0, 0, 0], [3, 3, 27])), "outside the overall domain")   # a pad cell
    refused(lambda: inj("p", [4, 0, 0], [3, 3, 3], 0, np.zeros((2, 1, 4, 4), np.float32)), "first index 4 is past last index 3 in dim 'x'")
    refused(lambda: inj("p", *box, 0, fr, stride=[1, 0, 1]), "stride 0 in dim 'y' is less than 1")
    refused(lambda: inj("p", *box, 0, fr, stride=[1, 1, -2]), "stride -2 in dim 'z' is less than 1")
    refused(lambda: inj("p", *box, 0, fr, every=0), "every = 0 is less than 1")
    refused(lambda: inj("p", *box, 0, fr[:0]), "nrows = 0 is less than 1")
    refused(lambda: inj("p", [1, 1], [2, 2], 0, fr), "first needs 3 domain index")
    refused(lambda: inj("p", *box, 0, fr, stride=[1, 1]), "stride needs 3 domain index")
    refused(lambda: inj("p", *box, 0, fr[:, :, :, :4]), "frames of shape (2, 5, 5, 4)", "expected (nrows, 5, 5, 5)")
    refused(lambda: inj("p", *box, 0, fr[0]), "expected (nrows, 5, 5, 5)")
    refused(lambda: inj("p", *box, 0, frames(*box, stride=[1, 2, 1])), "expected (nrows, 5, 5, 5)")
    refused(lambda: inj("p", *box, 0, fr, mode="replace"), "unknown mode 'replace'")
    refused(lambda: inj("p", *box, 0, fr.astype(np.complex64)), "not real numbers")
    refused(lambda: s.set_option("slice_injector_groups", "0"), "read-only")
    refused(lambda: s.set_option("slice_injector_launches", 3), "read-only")
    # the C ABI checks the mode itself
    f, l, st = (C.c_int64 * 3)(*box[0]), (C.c_int64 * 3)(*box[1]), (C.c_int64 * 3)(1, 1, 1)
    rid = C.c_int64(-1)
    assert capi.lib().yb_solution_add_slice_injector(s._h, b"p", f, l, st, 0, 1, 2, 7, fr.ctypes.data, C.byref(rid)) < 0
    assert "unknown mode 7" in capi.lib().yb_last_error().decode()
    assert capi.lib().yb_solution_add_slice_injector(s._h, b"p", f, l, st, 0, 1, 2, 0, None, C.byref(rid)) < 0
    assert "null frames" in capi.lib().yb_last_error().decode()
    # a refused injector leaves nothing behind
    assert s.get_option("slice_injector_groups") == "" and s.get_option("slice_injector_launches") == "0"
    assert inj("p", *box, 0, fr) == 0
    assert s.get_option("slice_injector_groups") == "0"
    s.close()


def test_frames_past_a_64_bit_byte_count_are_refused():
    """nrows x box points x element bytes must fit a 64-bit count; the check comes before the frames are read."""
    s = planned()
    f, l, st = (C.c_int64 * 3)(0, 0, 0), (C.c_int64 * 3)(36, 28, 22), (C.c_int64 * 3)(1, 1, 1)
    one = np.zeros(1, np.float32)
    rid = C.c_int64(-1)
    for hi, nrows in (((36, 28, 22), 2 ** 61), ((0, 0, 0), 2 ** 62)):
        l = (C.c_int64 * 3)(*hi)
        assert capi.lib().yb_solution_add_slice_injector(s._h, b"p", f, l, st, 0, 1, nrows, 0, one.ctypes.data, C.byref(rid)) < 0
        msg = capi.lib().yb_last_error().decode()
        assert "slice injector" in msg and "overflow a 64-bit byte count" in msg, msg
    assert s.get_option("slice_injector_groups") == ""
    s.close()


def test_ids_restart_after_clear_and_are_separate_from_recorders():
    s = planned()
    box = ([1, 1, 1], [5, 5, 5])
    assert s.add_slice("p", *box, 0, 3) == 0
    assert s.add_slice_injector("p", *box, 0, frames(*box)) == 0
    assert s.add_slice_injector("p", [7, 7, 7], [9, 9, 9], 0, frames([7, 7, 7], [9, 9, 9]), mode="set") == 1
    assert s.add_slice("p", *box, 0, 3) == 1
    s.clear_slice_injectors()
    assert s.get_option("slice_injector_groups") == ""
    assert s.add_slice_injector("p", *box, 0, frames(*box)) == 0          # ids restart after clear_slice_injectors()
    assert s.add_slice("p", *box, 0, 3) == 2                              # the recorders keep theirs
    s.clear_slices()
    assert s.add_slice_injector("p", *box, 0, frames(*box)) == 1           # and clear_slices() leaves the injectors alone
    s.close()


def test_checks_wait_for_the_geometry():
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec((16, 16, 16))
    s.add_slice_injector("p", [0, 0, 0], [99, 0, 0], 0, np.zeros((1, 100, 1, 1)))
    refused(s.plan_geometry, "slice injector: box [0, 99] in dim 'x'", "outside the overall domain [0,16)")
    s.clear_slice_injectors()
    s.plan_geometry()
    s.close()


@pytest.mark.parametrize("radius", [1, 2])
def test_fused_pair_rank_grid_is_refused(radius):
    """Refused on every rank of the grid, from plan_geometry() on, whether the injector comes before or after it."""
    grid, n = (2, 1, 1), (64, 48, 96)
    opts = (("block_steps", 2), ("mega_block_steps", 2))
    box = ([3, 3, 3], [40, 3, 90])
    for r in range(2):
        s = planned(n=n, grid=grid, rank=r, radius=radius, opts=opts)
        refused(lambda: s.add_slice_injector("p", *box, 0, frames(*box)), "slice injectors", "fused-pair", "mega_block_steps")
        assert s.get_option("slice_injector_groups") == ""
        s.close()
        s = capi.Solution("iso3dfd", radius=radius)
        s.set_overall_domain_size_vec(n)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        for k, v in opts:
            s.set_option(k, v)
        s.add_slice_injector("p", *box, 0, frames(*box))
        refused(s.plan_geometry, "fused-pair")
        s.close()
    # the same grid exchanging once per step, and one rank with pairs, take injectors
    for o, g in (((("block_steps", 2),), grid), (opts, None)):
        s = planned(n=n, grid=g, rank=0, radius=radius, opts=o)
        s.add_slice_injector("p", *box, 0, frames(*box))
        s.close()


def test_rank_grid_needs_a_var_of_the_last_stage():
    """awp_elastic's velocities are written by its first stage: on a rank grid they would be exchanged before an injection, so
    they are refused there on every rank; its stresses (last stage) are taken, and one rank takes the velocities too."""
    n, grid = (41, 19, 40), (2, 1, 1)
    box = ([3, 3, 3], [30, 3, 30])
    for r in range(2):
        s = planned("awp_elastic", n=n, grid=grid, rank=r, eb=0)
        refused(lambda: s.add_slice_injector("vel_x", *box, 0, frames(*box)), "on a rank grid", "'vel_x'", "last stage")
        assert s.add_slice_injector("stress_xx", *box, 0, frames(*box)) == 0
        s.close()
        s = capi.Solution("awp_elastic", elem_bytes=0)
        s.set_overall_domain_size_vec(n)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        s.add_slice_injector("vel_x", *box, 0, frames(*box))
        refused(s.plan_geometry, "last stage")
        s.close()
    s = planned("awp_elastic", n=n, eb=0)
    assert s.add_slice_injector("vel_x", *box, 0, frames(*box)) == 0
    s.close()


@pytest.mark.parametrize("boxes,want", [
    # disjoint boxes on one var share a launch
    ([("p", [0, 0, 0], [3, 3, 3], None), ("p", [4, 0, 0], [8, 3, 3], None), ("p", [0, 10, 0], [36, 12, 22], None)], "0,1,2"),
    # an overlap ends the group; the next group starts afresh
    ([("p", [0, 0, 0], [5, 5, 5], None), ("p", [5, 5, 5], [9, 9, 9], None), ("p", [20, 0, 0], [25, 3, 3], None),
      ("p", [0, 0, 0], [0, 0, 0], None)], "0;1,2,3"),
    # an overlap with any earlier member of the group, not only the last one
    ([("p", [0, 0, 0], [5, 5, 5], None), ("p", [10, 0, 0], [12, 5, 5], None), ("p", [3, 3, 3], [4, 4, 4], None)], "0,1;2"),
    # the same box twice: each in its own launch, in id order
    ([("p", [1, 1, 1], [9, 9, 9], None)] * 3, "0;1;2"),
    # a strided pair whose bounding boxes overlap, though no point is shared
    ([("p", [0, 0, 0], [20, 0, 0], [2, 1, 1]), ("p", [1, 0, 0], [21, 0, 0], [2, 1, 1])], "0;1"),
    # the bounding box ends at the last decimated point: [0, 20] with stride 7 stops at 14
    ([("p", [0, 0, 0], [20, 0, 0], [7, 1, 1]), ("p", [15, 0, 0], [20, 0, 0], None)], "0,1"),
])
def test_launch_groups(boxes, want):
    s = planned()
    for var, f, l, st in boxes:
        s.add_slice_injector(var, f, l, 0, frames(f, l, stride=st), stride=st)
    assert s.get_option("slice_injector_groups") == want
    s.close()


def test_launch_groups_by_var():
    """The same box on two vars shares a launch: they write different storage."""
    s = planned("awp_elastic", n=(21, 19, 40), eb=0)
    box = ([2, 2, 2], [10, 10, 10])
    for var in ("stress_xx", "stress_yy", "stress_xx"):
        s.add_slice_injector(var, *box, 0, frames(*box))
    assert s.get_option("slice_injector_groups") == "0,1;2"
    s.clear_slice_injectors()
    assert s.get_option("slice_injector_groups") == ""
    s.close()


def test_groups_are_the_same_on_every_rank():
    grid, n = (2, 2, 1), (37, 29, 23)
    texts = []
    for r in range(4):
        s = planned(n=n, grid=grid, rank=r)
        s.add_slice_injector("p", [0, 0, 5], [36, 28, 5], 0, frames([0, 0, 5], [36, 28, 5]))
        s.add_slice_injector("p", [17, 13, 0], [20, 16, 22], 0, frames([17, 13, 0], [20, 16, 22]))
        s.add_slice_injector("p", [0, 0, 5], [10, 10, 5], 0, frames([0, 0, 5], [10, 10, 5]))   # meets 0, which is done
        texts.append(s.get_option("slice_injector_groups"))
        s.close()
    assert texts == ["0;1,2"] * 4


def test_one_and_two_dim_solutions():
    s = planned("wave2d", n=(20, 30))
    assert s.add_slice_injector("u", [1, 0], [19, 29], 0, np.zeros((3, 10, 10)), stride=[2, 3]) == 0
    refused(lambda: s.add_slice_injector("u", [1, 0, 0], [19, 29, 0], 0, np.zeros((3, 10, 10, 1))), "2 domain index")
    s.close()
    s = planned("test_1d", n=(50,), grid=(2,), rank=1)
    var = [v.get_name() for v in s.get_vars() if v.info.is_output][0]
    assert s.add_slice_injector(var, [3], [49], 0, np.zeros((2, 12)), stride=[4], mode="set") == 0
    s.close()
