"""CPU: the storage plan of the average-of-points temporal tile (option block_steps / -bt 2, yask_b200/csrc/yb_avepts_tt.cuh).
  * block_steps=2 on a tiled entry -- 3axis at radius 1 and 2, fp32 and fp64 -- plans the spare pair of slots of A (4 in all) and
    pads at least 2R deep below the origin in x and y, 2 HZ in z (HZ = R rounded up to whole 16-byte vectors);
  * it plans the reference's 2 slots where there is no tile: the other shapes (slower with pairs, README), other radii,
    kernel=direct, a rank grid, block_steps=1;
  * the option reads back; tt_launches is read-only.
"""
import pytest

from yask_b200 import capi

TILED = [("3axis", r, eb) for r in (1, 2) for eb in (4, 8)]


def _plan(shape, R, eb, opts, grid=(1, 1, 1), n=(40, 33, 70)):
    s = capi.Solution(shape, radius=R, elem_bytes=eb)
    try:
        s.set_overall_domain_size_vec(n)
        s.set_num_ranks_vec(grid)
        for k, v in opts.items():
            s.set_option(k, v)
        s.plan_geometry()
        a = s.get_var("A").info
        return a.storage_bytes // (a.slot_elems * a.elem_bytes), a
    finally:
        s.close()


@pytest.mark.parametrize("shape,R,eb", TILED, ids=[f"{s}-r{r}-fp{8 * e}" for s, r, e in TILED])
def test_tiled_entry_plans_spare_slots_and_pads(shape, R, eb):
    slots, a = _plan(shape, R, eb, {"block_steps": 2})
    assert slots == 4 and a.step_alloc == 2
    vw = 16 // eb
    hz = (R + vw - 1) // vw * vw
    for d in range(1, 4):       # dims 1..3 after the step dim: x, y, z
        dm = a.dims[d]
        assert dm.left_halo == dm.right_halo == R
        assert dm.left_pad >= (2 * hz if d == 3 else 2 * R)
    assert _plan(shape, R, eb, {})[0] == 2
    assert _plan(shape, R, eb, {"block_steps": 1})[0] == 2


@pytest.mark.parametrize("shape,R,eb,opts,grid", [
    ("3axis_with_diags", 1, 4, {}, (1, 1, 1)), ("3axis_with_diags", 2, 8, {}, (1, 1, 1)), ("3plane", 1, 4, {}, (1, 1, 1)),
    ("cube", 1, 8, {}, (1, 1, 1)), ("3plane", 2, 4, {}, (1, 1, 1)), ("3plane", 2, 8, {}, (1, 1, 1)), ("cube", 2, 8, {}, (1, 1, 1)),
    ("3axis", 3, 4, {}, (1, 1, 1)), ("3axis_with_diags", 5, 8, {}, (1, 1, 1)),
    ("3axis", 1, 4, {"kernel": "direct"}, (1, 1, 1)), ("3axis", 2, 8, {"gen_sweep": 0}, (1, 1, 1)),
    ("3axis", 1, 4, {}, (2, 1, 1)), ("3axis", 2, 8, {}, (2, 1, 1)), ("3axis", 1, 8, {}, (2, 2, 1))],
    ids=["diags-r1", "diags-r2-fp64", "3plane-r1", "cube-r1-fp64", "3plane-r2", "3plane-r2-fp64", "cube-r2-fp64", "3axis-r3", "diags-r5-fp64", "direct", "gen_sweep0", "3axis-2x1x1",
         "3axis-r2-fp64-2x1x1", "3axis-r1-fp64-2x2x1"])
def test_no_tile_keeps_two_slots(shape, R, eb, opts, grid):
    assert _plan(shape, R, eb, dict(opts, block_steps=2), grid=grid)[0] == 2


def test_options_read_back():
    s = capi.Solution("3axis", radius=1, elem_bytes=4)
    try:
        assert s.get_option("block_steps") == "1" and s.get_option("tt_launches") == "0"
        s.set_option("block_steps", 2)
        assert s.get_option("block_steps") == "2"
        with pytest.raises(capi.YaskError):
            s.set_option("tt_launches", 5)
        with pytest.raises(capi.YaskError):
            s.set_option("mega_block_steps", 2)      # no fused rank-grid mode for these shapes
    finally:
        s.close()
