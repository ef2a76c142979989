"""iso3dfd temporal tile on rank grids (block_steps=2 with mega_block_steps=2, the reference's -bt 2 -Mbt 2), what can be checked
without a GPU:

  * the kernel's own sweep code in the CTA emulator (tests/emul/tt_emul_ranks.cpp: the back end of tt_emul.cpp) on ONE RANK's
    sub-box of a global domain: its step-1 ring past a rank interface is computed from halos that hold p(t) 2R deep, p(t-1) and v R deep -- what the deep halo exchange
    delivers (faces; edges of p(t) R deep) -- and both steps must equal the oracle's global result over the sub-box, bit for bit;
  * the storage plan_geometry() reports on rank grids: the spare pair of slots and the pads on both sides of every split dim;
  * the options: -Mbt through the C++ API's command line, the reference's minimum rank size, and where the option is inert.

Reference behaviour being matched: wave-front extensions of the halos by angle * (wf_steps - 1) = R and exchanges once per
wave-front (/root/reference/src/kernel/lib/setup.cpp:717-781); temporal blocking never changes results."""
import ctypes
import glob
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests.test_temporal_cpu import _coef32
from yask_b200.synth import hash_field, var_salt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


_LIB = None


def emul_ranks():
    """The rank emulator, compiled by g++ (flags of tests/emul/Makefile) into a temporary directory on first use."""
    global _LIB
    if _LIB is None:
        d = tempfile.mkdtemp(prefix="tt_emul_ranks_")
        try:
            so = os.path.join(d, "libtt_emul_ranks.so")
            subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", so,
                            os.path.join(ROOT, "tests", "emul", "tt_emul_ranks.cpp"), "-lm"], check=True)
            _LIB = ctypes.CDLL(so)
        finally:
            shutil.rmtree(d, ignore_errors=True)      # the loaded library stays mapped
        _LIB.tt_emul_run_ext.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 9 + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2
        _LIB.tt_emul_run_ext.restype = ctypes.c_int
    return _LIB


def _provided(n, pad, lo_if, hi_if, face_if, face_gl, edge, corner):
    """Mask over a local padded array (n + 2 pad per dim): cells a rank holds real data in.  Per dim, o = distance past the domain
    (0 inside); a cell past one side is held up to `face_if` / `face_gl` deep on an interface / global side; past two sides
    (an edge) up to `edge` deep in both (0: not held); past three sides (a corner) only with `corner` and only where every
    side is global, up to `edge` deep."""
    o, g = [], []
    for d in range(3):
        c = np.arange(-pad[d], n[d] + pad[d])
        od = np.where(c < 0, -c, np.where(c >= n[d], c - n[d] + 1, 0))
        side_if = np.where(c < 0, lo_if[d], np.where(c >= n[d], hi_if[d], False))
        sh = [1, 1, 1]
        sh[d] = -1
        o.append(od.reshape(sh))
        g.append(side_if.reshape(sh))
    k = sum((od > 0).astype(int) for od in o)
    face = np.ones_like(k, dtype=bool)
    for od, si in zip(o, g):
        face &= (od == 0) | (od <= np.where(si, face_if, face_gl))
    within_edge = np.ones_like(k, dtype=bool)
    all_global = np.ones_like(k, dtype=bool)
    for od, si in zip(o, g):
        within_edge &= od <= edge
        all_global &= ~((od > 0) & si)
    return (k == 0) | ((k == 1) & face) | ((k == 2) & within_edge & (edge > 0)) | ((k == 3) & within_edge & all_global & corner)


def run_rank(radius, variant, mode, gn, b, e, grid, nchunks, lazy, seed=7, p_depth=2, p_edges=True):
    """Emulate the fused launch of the rank that owns [b, e) of the global domain gn, its p(t) halo p_depth * R deep past an
    interface (and R deep along edges with `p_edges`).  Returns (got1, got2, ref1, ref2)."""
    R = radius
    gp = [hash_field(seed, var_salt("p", t), (-R,) * 3, [x + 2 * R for x in gn], -1, 1) for t in (0, 1)]
    gv = hash_field(seed, var_salt("v", 0), (0, 0, 0), gn, 0.05, 0.3)
    n = [e[d] - b[d] for d in range(3)]
    lo_if = [b[d] > 0 for d in range(3)]
    hi_if = [e[d] < gn[d] for d in range(3)]
    ppad, vpad = (2 * R, 2 * R, 8), (R, R, 4)

    def local(src, org, pad, mask):
        """Local padded array: src (global array whose element 0 sits at global index org) where `mask`, NaN elsewhere."""
        a = np.full([n[d] + 2 * pad[d] for d in range(3)], np.nan, np.float32)
        idx = [np.arange(b[d] - pad[d], e[d] + pad[d]) - org for d in range(3)]
        ok = [(i >= 0) & (i < src.shape[d]) for d, i in enumerate(idx)]
        sub = src[np.ix_(*[np.clip(i, 0, src.shape[d] - 1) for d, i in enumerate(idx)])]
        m = mask & ok[0][:, None, None] & ok[1][None, :, None] & ok[2][None, None, :]
        a[m] = sub[m]
        return a

    # p(t): 2R deep past an interface (faces), R deep past the global boundary (the user's halo cells), edges R deep
    cur = local(gp[1], -R, ppad, _provided(n, ppad, lo_if, hi_if, p_depth * R, R, R if p_edges else 0, False))
    # p(t-1): R deep faces; edges and corners only where every side is global (never read otherwise)
    prev = local(gp[0], -R, ppad, _provided(n, ppad, lo_if, hi_if, R, R, 0, True) | _global_box(n, ppad, lo_if, hi_if, R))
    # v: no halo; R deep past an interface (the deep exchange at the start of a run)
    v = local(gv, 0, vpad, _provided(n, vpad, lo_if, hi_if, R, 0, 0, False))
    out1, out2 = prev.copy(), cur.copy()
    lo = [R if lo_if[d] else 0 for d in range(3)]       # TTParams::ext_lo / ext_hi
    hi = [R if hi_if[d] else 0 for d in range(3)]
    i3 = lambda x: ctypes.cast((ctypes.c_int * 3)(*x), ctypes.c_void_p)
    rc = emul_ranks().tt_emul_run_ext(R, variant, mode, prev.ctypes.data, cur.ctypes.data, v.ctypes.data, out1.ctypes.data,
                                      out2.ctypes.data, i3(n), i3(ppad), i3(vpad), _coef32(R).ctypes.data, grid, nchunks, int(lazy),
                                      i3(lo), i3(hi))
    assert rc == 0, f"emulator protocol error {rc}"
    dom = tuple(slice(ppad[d], ppad[d] + n[d]) for d in range(3))
    for o, src in ((out1, prev), (out2, cur)):       # only the rank's own points are stored
        m = np.ones(o.shape, dtype=bool)
        m[dom] = False
        assert np.array_equal(o[m].view(np.uint32), src[m].view(np.uint32))
    sub = tuple(slice(b[d], e[d]) for d in range(3))
    ref1 = O.iso3dfd_run(gp[1], gp[0], gv, R, 1, mode)[R:-R, R:-R, R:-R][sub]
    ref2 = O.iso3dfd_run(gp[1], gp[0], gv, R, 2, mode)[R:-R, R:-R, R:-R][sub]
    return out1[dom], out2[dom], ref1, ref2


def _global_box(n, pad, lo_if, hi_if, R):
    """Cells within R of the domain on every axis where each side they lie past is global (the user's halo box there)."""
    m = np.ones([n[d] + 2 * pad[d] for d in range(3)], dtype=bool)
    for d in range(3):
        c = np.arange(-pad[d], n[d] + pad[d])
        ok = ((c >= 0) & (c < n[d])) | ((c < 0) & (c >= -R) & (not lo_if[d])) | ((c >= n[d]) & (c < n[d] + R) & (not hi_if[d]))
        sh = [1, 1, 1]
        sh[d] = -1
        m &= ok.reshape(sh)
    return m


def check_rank(*a, **k):
    g1, g2, r1, r2 = run_rank(*a, **k)
    assert np.array_equal(g1.view(np.uint32), np.ascontiguousarray(r1).view(np.uint32)), "p(t+1) differs from the oracle"
    assert np.array_equal(g2.view(np.uint32), np.ascontiguousarray(r2).view(np.uint32)), "p(t+2) differs from the oracle"


# (global domain, rank box [b, e)): interfaces on one side, the other, both; y and z interfaces; an x+y corner rank.  z sizes are
# ragged (not whole 16-byte vectors) where a z interface is.
POSITIONS = {
    "x_lower": ((24, 20, 40), (12, 0, 0), (24, 20, 40)),
    "x_upper": ((24, 20, 40), (0, 0, 0), (12, 20, 40)),
    "x_both": ((24, 20, 40), (8, 0, 0), (16, 20, 40)),
    "y_lower": ((12, 26, 40), (0, 13, 0), (12, 26, 40)),
    "z_upper": ((12, 20, 42), (0, 0, 0), (12, 20, 21)),
    "z_lower": ((12, 20, 42), (0, 0, 21), (12, 20, 42)),
    "xy_corner": ((24, 26, 40), (12, 13, 0), (24, 26, 40)),
    "xyz_inner": ((24, 26, 42), (8, 9, 12), (16, 17, 30)),
}


@pytest.mark.parametrize("lazy", [0, 1])
@pytest.mark.parametrize("variant", [0, 2, 4, 5])     # the four compiled forms (tt_variant 0-3)
@pytest.mark.parametrize("radius", [1, 2])
@pytest.mark.parametrize("pos", list(POSITIONS))
def test_rank_subbox_matches_global_oracle(pos, radius, variant, lazy):
    gn, b, e = POSITIONS[pos]
    check_rank(radius, variant, 2, gn, b, e, 2, 2, lazy)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("variant", [1, 3])            # small tiles (4 x 16): interfaces cut through many tiles and rounds
@pytest.mark.parametrize("radius", [1, 2])
@pytest.mark.parametrize("pos", ["x_both", "xy_corner", "z_upper", "xyz_inner"])
def test_rank_subbox_small_tiles_and_fp_modes(pos, radius, variant, mode):
    gn, b, e = POSITIONS[pos]
    for lazy in (0, 1):
        check_rank(radius, variant, mode, gn, b, e, 3, 3, lazy)


@pytest.mark.parametrize("radius", [1, 2])
def test_rank_subbox_needs_the_deep_halo(radius):
    """The sub-box check is sharp: with p(t) only R deep past the interface (the one-step halo), step 2 differs from the oracle."""
    gn, b, e = POSITIONS["x_lower"]
    g1, g2, r1, r2 = run_rank(radius, 0, 2, gn, b, e, 2, 2, 0, p_depth=1)
    assert not np.array_equal(g2.view(np.uint32), np.ascontiguousarray(r2).view(np.uint32))


@pytest.mark.parametrize("radius", [1, 2])
def test_rank_subbox_needs_the_edge_halo(radius):
    """...and at a rank with interfaces in two dims, p(t) is needed R deep along their edge too: step 1 past one interface reads
    points past the other.  Hence the deep exchange also sends to edge neighbours (as the reference does with wave-fronts)."""
    gn, b, e = POSITIONS["xy_corner"]
    g1, g2, r1, r2 = run_rank(radius, 0, 2, gn, b, e, 2, 2, 0, p_edges=False)
    assert not np.array_equal(g2.view(np.uint32), np.ascontiguousarray(r2).view(np.uint32))


# ---- storage plan on rank grids ------------------------------------------------------------------------------------------------

def _plan(radius, grid, opts, n=(64, 48, 96), rank=(0, 0, 0), stencil="iso3dfd", eb=4):
    from yask_b200 import capi
    s = capi.Solution(stencil, radius=radius, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    s.set_num_ranks_vec(grid)
    s.set_rank_index_vec(rank)
    for k, v in opts.items():
        s.set_option(k, v)
    s.plan_geometry()
    p, v = s.get_var("p").info, s.get_var("v").info
    s.close()
    slots = p.storage_bytes // (p.slot_elems * p.elem_bytes)
    return slots, p, v


FUSED = {"block_steps": 2, "mega_block_steps": 2}


@pytest.mark.parametrize("grid,rank", [((2, 1, 1), (0, 0, 0)), ((2, 1, 1), (1, 0, 0)), ((1, 2, 2), (0, 1, 0)), ((2, 2, 2), (1, 1, 1))])
@pytest.mark.parametrize("radius", [1, 2])
def test_plan_geometry_fused_rank_grid(radius, grid, rank):
    slots, p, v = _plan(radius, grid, FUSED, rank=rank)
    assert slots == 4 and p.step_alloc == 2
    for d in range(3):      # p: dims 1..3 after the step dim; v: dims 0..2
        reach_p, reach_v = (8, 4) if d == 2 else (2 * radius, radius)
        assert p.dims[d + 1].left_pad >= reach_p and v.dims[d].left_pad >= reach_v
        if grid[d] > 1:
            assert p.dims[d + 1].right_pad >= reach_p and v.dims[d].right_pad >= reach_v


@pytest.mark.parametrize("radius", [1, 2])
def test_plan_geometry_rank_grid_without_mega_block_steps(radius):
    """block_steps=2 alone on a rank grid: the reference's two slots, as prepare allocates them (one launch per step)."""
    for grid in ((2, 1, 1), (1, 2, 2)):
        slots, p, v = _plan(radius, grid, {"block_steps": 2})
        assert slots == 2
        slots, p, v = _plan(radius, grid, {})
        assert slots == 2


@pytest.mark.parametrize("radius", [1, 2])
def test_plan_geometry_single_rank_unchanged(radius):
    """mega_block_steps changes nothing on one rank: same slots and pads as block_steps=2 alone."""
    a = _plan(radius, (1, 1, 1), {"block_steps": 2})
    b = _plan(radius, (1, 1, 1), FUSED)
    assert a[0] == b[0] == 4
    for x, y in ((a[1], b[1]), (a[2], b[2])):
        assert x.storage_bytes == y.storage_bytes
        for d in range(x.num_dims):
            assert (x.dims[d].left_pad, x.dims[d].right_pad) == (y.dims[d].left_pad, y.dims[d].right_pad)


@pytest.mark.parametrize("opts,radius,eb,stencil", [(FUSED, 3, 4, "iso3dfd"), (FUSED, 2, 8, "iso3dfd"), (FUSED, 2, 4, "iso3dfd_sponge"),
                                                     (dict(FUSED, kernel="direct"), 2, 4, "iso3dfd")],
                         ids=["radius3", "fp64", "sponge", "direct"])
def test_plan_geometry_inert_where_no_tile_exists(opts, radius, eb, stencil):
    slots, _, _ = _plan(radius, (2, 1, 1), opts, stencil=stencil, eb=eb)
    assert slots == 2


@pytest.mark.parametrize("radius", [1, 2])
def test_rank_domain_below_2r_is_refused(radius):
    """The reference's minimum rank size with wave-fronts: halo + wave-front extension = 2R in a split dim."""
    from yask_b200 import capi
    s = capi.Solution("iso3dfd", radius=radius)
    s.set_overall_domain_size_vec((64, 2 * (2 * radius - 1), 96))
    s.set_num_ranks_vec((1, 2, 1))
    for k, v in FUSED.items():
        s.set_option(k, v)
    with pytest.raises(capi.YaskError) as e:
        s.plan_geometry()
    assert f"local-domain size of {2 * radius - 1} in 'y' dim is less than minimum size of {2 * radius}" in str(e.value)
    s.close()
    # without mega_block_steps the same grid plans (one exchange per step needs R only)
    assert _plan(radius, (1, 2, 1), {"block_steps": 2}, n=(64, 2 * (2 * radius - 1), 96))[0] == 2


def test_generated_solutions_refuse_mega_block_steps():
    """Generated engines have no fused rank-grid mode: they refuse the key as they refuse every key they do not know."""
    from yask_b200 import capi
    s = capi.Solution("awp")
    with pytest.raises(capi.YaskError):
        s.set_option("mega_block_steps", 2)
    s.close()


def test_tt_launches_is_read_only():
    from yask_b200 import capi
    s = capi.Solution("iso3dfd", radius=1)
    assert s.get_option("tt_launches") == "0"
    assert s.get_option("mega_block_steps") == "1"
    with pytest.raises(capi.YaskError):
        s.set_option("tt_launches", 3)
    s.set_option("mega_block_steps", 2)
    assert s.get_option("mega_block_steps") == "2"
    s.close()


# ---- -Mbt through the C++ API's command line -----------------------------------------------------------------------------------

MODS = sorted(glob.glob(os.path.join(ROOT, "yask_b200", "lib", "python", "iso3dfd_r1", "yask_kernel*.so")))


@pytest.mark.skipif(not MODS, reason="python modules not built (pybind11 missing?)")
def test_mbt_command_line_option():
    script = r'''
import yask_kernel as yk
kfac = yk.yk_factory()
soln = kfac.new_solution(kfac.new_env())
assert soln.apply_command_line_options("-bt 2 -Mbt 2 -mbt 3") == ""
assert " -Mbt 2" in soln.get_command_line_values(), soln.get_command_line_values()
print("OK")
'''
    env = dict(os.environ, PYTHONPATH=os.path.dirname(MODS[0]), CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == "OK", r.stdout + r.stderr
