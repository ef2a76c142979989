"""Every emitter-generated solution in its 64-bit addressing form (option gen_wide=1, yb_gen.cuh: MODE | GEN_WIDE), which the
engine otherwise runs only where a var slot holds 2^31 elements or more, and both forms at the switch point between them.

The matrix of tests/test_generated_matrix_gpu.py again, every case with gen_wide=1 and the solution reporting "1":
  A. every row x gen_sweep {1, 0} x (fp_mode 0 vs the uncontracted oracle, fp_mode 2 vs the oracle contracted like GCC),
     bit for bit, with nothing outside the domain changed and the same launch counts as the 32-bit form;
  B. the sweep kernels at the row's gen_sweep_lx and at gen_sweep_lx = 1;
  C. the direct kernels' knobs gen_pf (the L2 prefetch forms its addresses with gen_pos) and gen_l2_mb;
  D. the offline and in-run tuners;
  E. uneven rank grids (exterior slabs on the direct kernels, the interior on the sweep kernels) against one rank in the
     32-bit form, in both FP modes;
  F. awp_elastic and test_2d with sources, receivers, a slice recorder and a slice injector, against the 32-bit form.

Switch point: 3axis (sweep and direct kernels) and test_2d at a size whose largest slot lies just below 2^31 elements and one
just at or above it (tests/large_domain.py: SWITCH_SIZES), each checked against the oracle at its low and high corners.  These
need about 17 GB each and skip, naming the amount, when the device has less free memory than that plus a 2 GB margin.
"""
import numpy as np
import pytest

from tests import generated_cases as G
from tests.large_domain import SWITCH_SIZES, TWO31, Window, bits, fill_gen, gen_reach, gen_window_ref
from tests.test_generated_matrix_gpu import MODES, SWEEP_ROWS, TUNE_STEPS, collect, fill, n_sweep_parts, run_and_check
from tests.test_large_domain_gpu import _need
from yask_b200 import capi, multi

pytestmark = pytest.mark.gpu

WIDE = (("gen_wide", 1),)


def reports_wide(s):
    assert s.get_option("gen_wide") == "1", "the solution does not run its kernels' 64-bit form"


# ---- A. the matrix ------------------------------------------------------------------------------------------------------
MATRIX = [pytest.param(r.name, sweep, fm, c, id=f"{r.name}-{'sweep' if sweep else 'direct'}-fp_mode{fm}")
          for r in G.ROWS for fm, c in MODES for sweep in (1, 0)]


@pytest.mark.parametrize("name,sweep,fp_mode,contract", MATRIX)
def test_wide_matrix(name, sweep, fp_mode, contract):
    r = G.BY_NAME[name]
    run_and_check(name, fp_mode, contract, opts=WIDE + (("gen_sweep", sweep),), before_load=reports_wide,
                  sweep_launches=n_sweep_parts(name) * r.steps * sweep)


# ---- B. sweep chunking --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lx", ["row", 1])
@pytest.mark.parametrize("name", SWEEP_ROWS)
def test_wide_sweep_chunking(name, lx):
    r = G.BY_NAME[name]
    lx = r.lx if lx == "row" else lx
    run_and_check(name, 2, 1, opts=WIDE + (("gen_sweep", 1), ("gen_sweep_lx", lx)), before_load=reports_wide,
                  sweep_launches=n_sweep_parts(name) * r.steps)


# ---- C. direct-kernel knobs ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knob", [("gen_pf", 0), ("gen_pf", 3), ("gen_l2_mb", 1), ("gen_l2_mb", 0)], ids=lambda k: f"{k[0]}={k[1]}")
@pytest.mark.parametrize("name", G.KNOB_ROWS)
def test_wide_direct_kernel_knobs(name, knob):
    run_and_check(name, 2, 1, opts=WIDE + (("gen_sweep", 0), knob), before_load=reports_wide, sweep_launches=0)


# ---- D. tuners ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", G.TUNER_ROWS)
def test_wide_offline_tuner_then_exact(name):
    def tune(s):
        reports_wide(s)
        rep = s.run_auto_tuner_now()
        assert "best: gen_pf=" in rep and rep.count("ms/step") == 13, rep
        reports_wide(s)
    run_and_check(name, 2, 1, opts=WIDE, before_load=tune, after_run=reports_wide)


@pytest.mark.parametrize("name", G.TUNER_ROWS)
def test_wide_in_run_tuner_exact(name):
    def enable(s):
        reports_wide(s)
        s.reset_auto_tuner(True)

    def done(s):
        assert not s.is_auto_tuner_enabled()
        assert s.auto_tuner_report().count("ms/step") == 4
        reports_wide(s)
    nsw = run_and_check(name, 2, 1, opts=WIDE, steps=TUNE_STEPS, before_load=enable, after_run=done)
    if G.sweep_tiles(name):
        assert nsw >= 3 * 3 * n_sweep_parts(name), nsw


# ---- E. rank grids ------------------------------------------------------------------------------------------------------
def run_grid(r, grid, fp_mode, wide):
    """tests/test_generated_matrix_gpu.py's run_grid with gen_wide = `wide` on every rank."""
    world = int(np.prod(grid))
    solns = []
    for k in range(world):
        s = r.solution()
        s.set_overall_domain_size_vec(r.n)
        if world > 1:
            s.set_num_ranks_vec(grid)
            s.set_rank_index_vec(multi.grid_coords(k, grid))
        s.set_option("fp_mode", fp_mode)
        s.set_option("gen_wide", wide)
        s.prepare_solution(0)
        assert s.get_option("gen_wide") == str(wide)
        solns.append(s)
    if world > 1:
        multi.connect_local(solns)
    for s in solns:
        fill(s, r.name)
    for s in solns:
        s.run_solution(0, r.steps - 1)
    for s in solns:
        s.sync()
    out = collect(solns, r.n)
    for s in solns:
        s.close()
    return out


@pytest.mark.parametrize("fp_mode", [0, 2])
@pytest.mark.parametrize("name", [r.name for r in G.grid_rows()])
def test_wide_rank_grid_uneven(name, fp_mode):
    r = G.BY_NAME[name]
    one = run_grid(r, (1,) * len(r.n), fp_mode, 0)
    got = run_grid(r, r.grid, fp_mode, 1)
    assert set(got) == set(one) and len(got) == sum(1 for v in G.ir_of(name)["vars"] if v["is_output"])
    for vn in one:
        assert got[vn][0] == one[vn][0], vn
        bad = int((bits(got[vn][1]) != bits(one[vn][1])).sum())
        assert bad == 0, f"{name} grid {r.grid} fp_mode {fp_mode}: {vn}: {bad} elements differ from one rank in the 32-bit form"


# ---- F. device features around the kernels ------------------------------------------------------------------------------
# (row, source var, receiver / recorder var, injector var)
FEATURE_ROWS = [("awp_elastic", "stress_xx", "vel_x", "vel_y"), ("test_2d", "A", "A", "A")]
FEATURE_STEPS = 4


def run_features(name, src, rcv, inj, wide):
    """FEATURE_STEPS steps of row `name` with on-grid sources and receivers (corners and centre), a decimated recorder over
    the whole domain and an injector adding into a plane, in fp_mode 2; everything it produced, for comparison."""
    r = G.BY_NAME[name]
    n, nd, steps = r.n, len(r.n), FEATURE_STEPS
    rng = np.random.default_rng(29)
    s = r.solution()
    s.set_overall_domain_size_vec(n)
    s.set_option("gen_wide", wide)
    s.prepare_solution(0)
    assert s.get_option("gen_wide") == str(wide)
    fill(s, name)
    pts = [[0] * nd, [m - 1 for m in n], [m // 2 for m in n], [1] + [m - 2 for m in n[1:]]]
    s.set_sources(src, pts, 0, rng.uniform(-1, 1, (steps, len(pts))))
    s.set_receivers(rcv, pts, 0, steps)
    rid = s.add_slice(rcv, [0] * nd, [m - 1 for m in n], 0, steps, stride=[2] * nd)
    plane_f, plane_l = [n[0] // 3] + [0] * (nd - 1), [n[0] // 3] + [m - 1 for m in n[1:]]
    s.add_slice_injector(inj, plane_f, plane_l, 1, rng.uniform(-0.5, 0.5, (steps - 1, 1) + tuple(n[1:])))
    s.run_solution(0, steps - 1)
    s.sync()
    out = {"vars": collect([s], n), "traces": s.get_traces(), "frames": s.get_slice_frames(rid)}
    out["counts"] = {k: s.get_option(k) for k in ("point_launches", "slice_launches", "slice_injector_launches", "gen_sweep_launches")}
    s.close()
    return out


@pytest.mark.parametrize("name,src,rcv,inj", FEATURE_ROWS, ids=[f[0] for f in FEATURE_ROWS])
def test_wide_with_points_and_slices(name, src, rcv, inj):
    narrow = run_features(name, src, rcv, inj, 0)
    wide = run_features(name, src, rcv, inj, 1)
    assert wide["counts"] == narrow["counts"], (wide["counts"], narrow["counts"])
    c = narrow["counts"]
    assert int(c["point_launches"]) > 0 and int(c["slice_launches"]) > 0 and int(c["slice_injector_launches"]) > 0, c
    for what in ("traces", "frames"):
        (a, oa), (b, ob) = wide[what], narrow[what]
        assert oa.all() and ob.all(), what
        assert np.abs(b).max() > 0 and np.array_equal(bits(a), bits(b)), f"{name}: {what} differ between the forms"
    assert set(wide["vars"]) == set(narrow["vars"])
    for vn, (tl, a) in narrow["vars"].items():
        assert wide["vars"][vn][0] == tl and np.array_equal(bits(wide["vars"][vn][1]), bits(a)), f"{name}: {vn} differs between the forms"


# ---- the switch point ---------------------------------------------------------------------------------------------------
# (IR name and solution, steps, forms): gen_wide=0 set explicitly must not keep the 32-bit form at the "at" size
SWITCH_CASES = [
    ("3axis", 2, ({"gen_sweep": 1}, {"gen_sweep": 0, "gen_wide": 0})),
    ("test_2d", 3, ({}, {"gen_wide": 0})),
]


def corner_windows(n, size, m):
    """The windows at the low and the high corner of the domain: the high corner's x neighbours lie in the last pad planes,
    the elements of a slot with the largest positions."""
    nd = len(n)
    return [Window(n, [0] * nd, size, m), Window(n, [a - s for a, s in zip(n, size)], size, m)]


@pytest.mark.parametrize("side", ["below", "at"])
@pytest.mark.parametrize("name,steps,forms", SWITCH_CASES, ids=[c[0] for c in SWITCH_CASES])
def test_switch_point(name, steps, forms, side):
    seed = 71
    n = SWITCH_SIZES[name][side == "at"]
    m = steps * gen_reach(name)
    size = [32 + m] * len(n)
    wins = corner_windows(n, size, m)
    sums = []
    for opts in forms:
        s = capi.Solution(name, elem_bytes=0)
        s.set_overall_domain_size_vec(n)
        for k, v in opts.items():
            s.set_option(k, v)
        _need(s)
        vi = max((v.info for v in s.get_vars()), key=lambda i: i.slot_elems)
        assert (vi.slot_elems >= TWO31) == (side == "at"), (n, vi.slot_elems)
        try:
            s.prepare_solution(0)
            assert s.get_option("gen_wide") == ("1" if side == "at" else "0"), (name, side, opts)
            fill_gen(s, name, seed)
            s.run_solution(0, steps - 1)
            launched = int(s.get_option("gen_sweep_launches"))
            assert (launched > 0) == (opts.get("gen_sweep", 1) == 1 and len(n) == 3), (name, opts, launched)
            got, cs = [], {}
            for var in s.get_vars():
                v = var.info
                if not v.is_output:
                    continue
                vn, tl = v.name.decode(), v.last_valid_step
                cs[vn] = var.checksum(tl)
                got.append((vn, tl, [var.get_elements_in_slice(*w.kept_box(tl)) for w in wins]))
        finally:
            s.close()
        sums.append(cs)
        for i, w in enumerate(wins):
            ref = gen_window_ref(name, w, seed, steps, 1)
            for vn, tl, arrs in got:
                assert ref[vn][0] == tl
                assert np.array_equal(bits(arrs[i]), bits(ref[vn][1])), (name, side, opts, vn, w.lo)
    assert all(c == sums[0] for c in sums), f"{name} {side}: the forms disagree"
