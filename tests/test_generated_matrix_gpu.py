"""Every emitter-generated solution (tests/generated_cases.py: one row per name in manifest.json) against the CPU oracle on
boxes that span several tiles of both launch forms:
  A. every row x gen_sweep {1, 0} x (fp_mode 0 vs the uncontracted oracle, fp_mode 2 vs the oracle contracted like GCC),
     bit for bit, with nothing outside the domain changed;
  B. the sweep kernels at the row's gen_sweep_lx (a short last chunk) and at gen_sweep_lx = 1;
  C. the direct kernels' knobs gen_pf and gen_l2_mb (y-chunked CTA order with a shorter last chunk);
  D. the offline and in-run tuners;
  E. uneven rank grids against one rank in both FP modes, and for the FSG rows against the oracle."""
import functools

import numpy as np
import pytest

from oracle import oracle as O
from tests import generated_cases as G
from tests.golden.ranges import RANGES
from tests.helpers import field_ulps, range_of
from tests.test_generated_gpu import MATH_FUNC_STENCILS, MATH_ULPS, load_inputs, synth_inputs
from yask_b200 import multi
from yask_b200.synth import var_salt

pytestmark = pytest.mark.gpu

SEED = 17
MODES = [(0, 0), (2, 1)]     # (fp_mode, oracle contraction): strict, and the default mode with GCC's fused products
SWEEP_ROWS = [r.name for r in G.ROWS if G.sweep_tiles(r.name)]


@functools.lru_cache(maxsize=2)
def oracle_case(name, steps, contract):
    """Inputs over every var's halo box (all step slots) and the oracle's result; the matrix runs a row's four forms in
    a row, so the last two (row, mode) pairs are kept."""
    r = G.BY_NAME[name]
    ins, ir = synth_inputs(name, r.n, SEED)
    return ins, ir, O.gen_run(name, r.n, steps, ins, contract=contract)


def bits(a):
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def ring_mask(v, ir, shape):
    """True on the halo ring of a var's halo box (misc dims whole), False on its domain."""
    vd = [d for d in v["dims"] if d != ir["step_dim"]]
    m = np.ones(shape, bool)
    m[tuple(slice(v["halo"][d][0], shape[i] - v["halo"][d][1]) if d in v["halo"] else slice(None) for i, d in enumerate(vd))] = False
    return m


def run_and_check(name, fp_mode, contract, opts=(), steps=None, sweep_launches=None, before_load=None, after_run=None):
    """Runs row `name` on one rank with `opts`, then checks it against the oracle:
      * every written var bit for bit on the domain (test_func_1d: device libm within MATH_ULPS field-ulps);
      * the halo ring of every API-visible var, in every step slot, unchanged; read-only vars unchanged everywhere;
      * kernel launches == parts x steps, and sweep-kernel launches == `sweep_launches` (when given)."""
    r = G.BY_NAME[name]
    steps = steps or r.steps
    ins, ir, ref = oracle_case(name, steps, contract)
    s = r.solution()
    s.set_overall_domain_size_vec(r.n)
    s.set_option("fp_mode", fp_mode)
    for k, v in opts:
        s.set_option(k, v)
    s.prepare_solution(0)
    if before_load:
        before_load(s)
    load_inputs(s, ins)
    s.run_solution(0, steps - 1)
    if after_run:
        after_run(s)
    st = s.get_stats()
    nsw = int(s.get_option("gen_sweep_launches"))
    irv = {v["name"]: v for v in ir["vars"]}
    got_out, seen = {}, set()
    for v in s.get_vars():
        vi = v.info
        vn = vi.name.decode()
        seen.add(vn)
        alloc = vi.step_alloc if vi.has_step else 1
        for t in (range(vi.first_valid_step, vi.last_valid_step + 1) if vi.has_step else [0]):
            got = v.get_elements_in_slice(*v.halo_box(t))
            init = np.asarray(ins[(vn, t % alloc)])
            assert got.shape == init.shape, (vn, got.shape, init.shape)
            if vn not in ref:
                assert np.array_equal(bits(got), bits(init)), f"{name}: read-only var {vn} changed (step {t})"
                continue
            m = ring_mask(irv[vn], ir, got.shape)
            assert np.array_equal(bits(got[m]), bits(init[m])), \
                f"{name}: halo of {vn} changed in step slot {t % alloc}: {int((bits(got[m]) != bits(init[m])).sum())} elements"
            if t == vi.last_valid_step:
                got_out[vn] = (t, got[~m], m)
    s.close()
    assert seen == {v["name"] for v in ir["vars"] if not v.get("scratch")}
    assert set(got_out) == set(ref), (sorted(got_out), sorted(ref))
    for vn, (tl, got, m) in got_out.items():
        want = ref[vn][1][~m]
        assert ref[vn][0] == tl, (vn, ref[vn][0], tl)
        if name in MATH_FUNC_STENCILS:
            assert field_ulps(got, want) <= MATH_ULPS, (vn, field_ulps(got, want))
        else:
            bad = int((bits(got) != bits(want)).sum())
            assert bad == 0, f"{name}: {vn}: {bad} of {got.size} domain elements differ from the oracle"
    assert st.kernel_launches == G.n_parts(ir) * steps, (st.kernel_launches, G.n_parts(ir), steps)
    if sweep_launches is not None:
        assert nsw == sweep_launches, f"{name}: {nsw} sweep-kernel launches, expected {sweep_launches}"
    return nsw


def n_sweep_parts(name):
    return len(G.sweep_tiles(name))


# ---- A. the matrix ------------------------------------------------------------------------------------------------------
MATRIX = [pytest.param(r.name, sweep, fm, c, id=f"{r.name}-{'sweep' if sweep else 'direct'}-fp_mode{fm}")
          for r in G.ROWS for fm, c in MODES for sweep in (1, 0)]


@pytest.mark.parametrize("name,sweep,fp_mode,contract", MATRIX)
def test_generated_matrix(name, sweep, fp_mode, contract):
    """gen_sweep = 1 must take the sweep kernel of every part that has one (each step), gen_sweep = 0 none."""
    r = G.BY_NAME[name]
    run_and_check(name, fp_mode, contract, opts=(("gen_sweep", sweep),), sweep_launches=n_sweep_parts(name) * r.steps * sweep)


# ---- B. sweep chunking --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lx", ["row", 1])
@pytest.mark.parametrize("name", SWEEP_ROWS)
def test_sweep_chunking(name, lx):
    """The row's chunk length leaves a last chunk shorter than the x halo; lx = 1 refills the whole x reach every plane."""
    r = G.BY_NAME[name]
    lx = r.lx if lx == "row" else lx
    run_and_check(name, 2, 1, opts=(("gen_sweep", 1), ("gen_sweep_lx", lx)), sweep_launches=n_sweep_parts(name) * r.steps)


# ---- C. direct-kernel knobs ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knob", [("gen_pf", 0), ("gen_pf", 3), ("gen_l2_mb", 1), ("gen_l2_mb", 0)], ids=lambda k: f"{k[0]}={k[1]}")
@pytest.mark.parametrize("name", G.KNOB_ROWS)
def test_direct_kernel_knobs(name, knob):
    """gen_l2_mb = 1 runs the 3-D rows' direct kernels in y chunks with a shorter last one (tests/test_generated_matrix_cpu.py
    checks the sizes); every setting computes the same bits."""
    run_and_check(name, 2, 1, opts=(("gen_sweep", 0), knob), sweep_launches=0)


# ---- D. tuners ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", G.TUNER_ROWS)
def test_offline_tuner_then_exact(name):
    """run_auto_tuner_now() times gen_pf x gen_l2_mb on the vars' storage (data not preserved) and clears the stats;
    the inputs loaded afterwards give the oracle's bits."""
    def tune(s):
        rep = s.run_auto_tuner_now()
        assert "best: gen_pf=" in rep and rep.count("ms/step") == 13, rep
        assert s.get_stats().num_steps_done == 0
    run_and_check(name, 2, 1, before_load=tune)


TUNE_STEPS = 4 * 3 + 1       # 4 variants x (1 cold + 2 timed) steps, then one step with the chosen variant


@pytest.mark.parametrize("name", G.TUNER_ROWS)
def test_in_run_tuner_exact(name):
    """reset_auto_tuner(True): each step runs the next untried variant (sweep with the cost-model chunking, lx 64, lx 128,
    direct) until all 4 have their samples; the result over those steps is the oracle's."""
    def enable(s):
        s.reset_auto_tuner(True)

    def done(s):
        assert not s.is_auto_tuner_enabled()
        rep = s.auto_tuner_report()
        assert rep.count("ms/step") == 4 and "<- best" in rep, rep
    nsw = run_and_check(name, 2, 1, steps=TUNE_STEPS, before_load=enable, after_run=done)
    if G.sweep_tiles(name):
        assert nsw >= 3 * 3 * n_sweep_parts(name), nsw


# ---- E. rank grids ------------------------------------------------------------------------------------------------------
def fill(s, name):
    for v in s.get_vars():
        vi = v.info
        lo, hi = range_of(RANGES[name], vi.name.decode())
        for t in (range(vi.step_alloc) if vi.has_step else [0]):
            v.fill_hash(t, SEED, var_salt(vi.name.decode(), t), lo, hi)


def collect(solns, n):
    """Every output var over the global domain, assembled from the ranks' pieces."""
    out = {}
    for s in solns:
        for v in s.get_vars():
            vi = v.info
            if not vi.is_output:
                continue
            f, l = v.domain_box(vi.last_valid_step)
            shape, sl = [], []
            for k in range(vi.num_dims):
                d = vi.dims[k]
                if d.kind == 0:
                    continue
                if d.kind == 1:
                    shape.append(n[d.domain_index])
                    sl.append(slice(f[k], l[k] + 1))
                else:
                    shape.append(d.domain_size)
                    sl.append(slice(0, d.domain_size))
            a = out.setdefault(vi.name.decode(), (vi.last_valid_step, np.zeros(shape, v.dtype)))[1]
            a[tuple(sl)] = v.get_elements_in_slice(f, l).reshape([x.stop - x.start for x in sl])
    return out


def run_grid(r, grid, fp_mode):
    world = int(np.prod(grid))
    solns = []
    for k in range(world):
        s = r.solution()
        s.set_overall_domain_size_vec(r.n)
        if world > 1:
            s.set_num_ranks_vec(grid)
            s.set_rank_index_vec(multi.grid_coords(k, grid))
        s.set_option("fp_mode", fp_mode)
        s.prepare_solution(0)
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


GRID_ORACLE = {r.name for r in G.ROWS if r.name.startswith("fsg")}     # the FSG rows (fsg_abc and friends: sub-domain parts)


@pytest.mark.parametrize("fp_mode", [0, 2])
@pytest.mark.parametrize("name", [r.name for r in G.grid_rows()])
def test_generated_rank_grid_uneven(name, fp_mode):
    """Thin exterior slabs take the direct kernels, the interior the sweep kernels: in fp_mode 2 both forms' contraction
    meets inside one result.  Bit for bit against one rank; the FSG rows also against the oracle in fp_mode 2."""
    r = G.BY_NAME[name]
    ir = G.ir_of(name)
    one = run_grid(r, (1,) * len(r.n), fp_mode)
    got = run_grid(r, r.grid, fp_mode)
    assert set(got) == set(one) and len(got) == sum(1 for v in ir["vars"] if v["is_output"])
    for vn in one:
        assert got[vn][0] == one[vn][0], vn
        bad = int((bits(got[vn][1]) != bits(one[vn][1])).sum())
        assert bad == 0, f"{name} grid {r.grid} fp_mode {fp_mode}: {vn}: {bad} elements differ from one rank"
    if fp_mode == 2 and name in GRID_ORACLE:
        _, _, ref = oracle_case(name, r.steps, 1)
        irv = {v["name"]: v for v in ir["vars"]}
        for vn, (tl, a) in got.items():
            want = ref[vn][1]
            want = want[~ring_mask(irv[vn], ir, want.shape)].reshape(a.shape)
            assert ref[vn][0] == tl and np.array_equal(bits(a), bits(want)), f"{name}: {vn} differs from the oracle"
