"""CPU: the option that forces the generated kernels' 64-bit form, and the sizes tests/test_generated_wide_gpu.py runs at the
switch between the two forms.

  * the pinned "below" / "at" sizes (tests/large_domain.py: SWITCH_SIZES) straddle 2^31 elements as intended, read from
    plan_geometry(): a change of the padding fails here instead of silently moving the GPU cases off the edge;
  * gen_wide is accepted by set_option() on every unprepared generated solution, and refused as unknown by the hand-written
    engines.
"""
import pytest

from tests import generated_cases as G
from tests.large_domain import SWITCH_SIZES, TWO31, elem_offset
from yask_b200 import capi


def planned(name, n):
    """(largest var slot's VarInfo, its first domain dim) of solution `name` planned at size n."""
    s = capi.Solution(name, elem_bytes=0)
    s.set_overall_domain_size_vec(n)
    s.plan_geometry()
    vi = max((v.info for v in s.get_vars()), key=lambda i: i.slot_elems)
    d0 = [vi.dims[i] for i in range(vi.num_dims) if vi.dims[i].kind == 1][0]
    s.close()
    return vi, d0


@pytest.mark.parametrize("side", ["below", "at"])
@pytest.mark.parametrize("name", sorted(SWITCH_SIZES))
def test_switch_sizes_straddle_2_31(name, side):
    n = SWITCH_SIZES[name][side == "at"]
    vi, d0 = planned(name, n)
    plane = d0.stride
    if side == "below":
        assert TWO31 - plane <= vi.slot_elems < TWO31, (n, vi.slot_elems, plane)
    else:
        assert TWO31 <= vi.slot_elems < TWO31 + plane, (n, vi.slot_elems, plane)
    # the one-step x reach of the stencil is the whole x pad, so the high corner reads the slot's last plane: past 2^31 at
    # the "at" size, within a plane of it below
    reach = G.x_halo(G.ir_of(name))
    assert reach == d0.left_pad == d0.right_pad, (reach, d0.left_pad, d0.right_pad)
    far = elem_offset(vi, [n[0] - 1 + reach] + [m - 1 for m in n[1:]])
    assert far < vi.slot_elems
    if side == "below":
        assert TWO31 - plane < far < TWO31, (n, far)
    else:
        assert far >= TWO31, (n, far)
        # and 2^31 falls inside that plane's domain rows, not in its pads: the high corner window's reads straddle it
        assert elem_offset(vi, [n[0] - 1 + reach] + [0] * (len(n) - 1)) < TWO31


def test_gen_wide_is_accepted_before_prepare():
    for r in G.ROWS:
        s = r.solution()
        s.set_overall_domain_size_vec(r.n)
        for v in (1, 0, 1):
            s.set_option("gen_wide", v)
        assert s.get_option("gen_wide") == "1", r.name
        s.plan_geometry()
        s.close()


@pytest.mark.parametrize("stencil,radius,eb", [("iso3dfd", 8, 4), ("iso3dfd_sponge", 4, 4), ("3axis", 2, 8)],
                         ids=["iso3dfd", "iso3dfd_sponge-r4", "3axis-fp64-r2"])
def test_hand_written_engines_do_not_know_gen_wide(stencil, radius, eb):
    s = capi.Solution(stencil, radius=radius, elem_bytes=eb)
    with pytest.raises(capi.YaskError) as e:
        s.set_option("gen_wide", 1)
    assert "unknown option 'gen_wide'" in str(e.value), str(e.value)
    s.close()
