"""GPU: iso3dfd_sponge on the hand-written iso3dfd sweep in its sponge form (fp32 radius 1-7, fp64 radius 1, 2, 3, 4, 5, 7, 8),
bit for bit:
  * against the reference's builds (tests/golden/iso3dfd_sponge-r<r>*.npz, iso3dfd_sponge-fp64-r<r>*.npz) with the TMA and the
    direct kernel,
  * against the sponge oracle (tests/sponge_oracle.py) at ragged sizes in every FP mode, with several chunk lengths and
    persistent CTAs that sweep several work units,
  * TMA against direct at 512^3 (fp32) and 256^3 (fp64), cr == 1 against plain iso3dfd, halo cells and the cr vars untouched,
  * rank grids in one process against one rank (fused peer stores with and without the in-kernel signal, the split path),
  * block_steps=2, the offline tuner, the command-line harness (-validate) and the iso3dfd_sponge Python module.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from tests.helpers import contract_mode_of, golden_cases, load_golden, regen_inputs
from tests.sponge_oracle import iso3dfd_sponge_run
from yask_b200 import capi, multi
from yask_b200.synth import hash_field, var_salt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP32_RADII = (1, 2, 3, 4, 5, 6, 7)
FP64_RADII = (1, 2, 3, 4, 5, 7, 8)
PREC_RADII = [(4, r) for r in FP32_RADII] + [(8, r) for r in FP64_RADII]
# the new fixtures only (the generated fp64 radius-6 solution has fixtures of its own, iso3dfd_sponge-fp64-r6*)
CASES = [p for r in (2, 4, 7) for p in golden_cases(f"iso3dfd_sponge-r{r}")] + \
        [p for r in (3, 4, 8) for p in golden_cases(f"iso3dfd_sponge-fp64-r{r}")]
CR = ("cr_x", "cr_y", "cr_z")


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _dt(eb):
    return np.float32 if eb == 4 else np.float64


def inputs(n, seed, R, eb, cr=True):
    dt = _dt(eb)
    ins = {("p", t): hash_field(seed, var_salt("p", t), (-R,) * 3, [i + 2 * R for i in n], -1, 1, dt) for t in (0, 1)}
    ins[("v", 0)] = hash_field(seed, var_salt("v", 0), (0, 0, 0), n, 0.05, 0.3, dt)
    for d, name in enumerate(CR):
        ins[(name, 0)] = hash_field(seed, var_salt(name, 0), (0,), (n[d],), 0.92, 1.0, dt) if cr else np.ones(n[d], dt)
    return ins


def make(n, R, eb, fp_mode=2, opts=None, name="iso3dfd_sponge"):
    s = capi.Solution(name, radius=R, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    s.set_option("fp_mode", fp_mode)
    for k, v in (opts or {}).items():
        s.set_option(k, v)
    return s


def load(s, ins):
    p = s.get_var("p")
    for t in (0, 1):
        p.set_elements_in_slice(ins[("p", t)], *p.halo_box(t))
    for name in [v.get_name() for v in s.get_vars()][1:]:      # v, then cr_x, cr_y, cr_z (plain iso3dfd: v only)
        var = s.get_var(name)
        var.set_elements_in_slice(ins[(name, 0)], *var.halo_box(0))


def result(s):
    p = s.get_var("p")
    return p.get_elements_in_slice(*p.domain_box(p.get_last_valid_step_index()))


def run(n, steps, ins, R, eb, fp_mode=2, opts=None):
    s = make(n, R, eb, fp_mode, opts)
    s.prepare_solution(0)
    assert s.get_element_bytes() == eb
    load(s, ins)
    s.run_solution(0, steps - 1)
    out = result(s)
    s.close()
    return out


def oracle(ins, R, steps, mode):
    return iso3dfd_sponge_run(ins[("p", 0)], ins[("p", 1)], ins[("v", 0)], ins[("cr_x", 0)], ins[("cr_y", 0)], ins[("cr_z", 0)],
                              R, steps, mode)[R:-R, R:-R, R:-R]


def test_hand_written_form_serves_every_new_radius():
    for eb, R in PREC_RADII:
        s = make((40, 24, 64), R, eb, 2, {"kernel": "tma"})      # the generated engine has no option `kernel`
        s.prepare_solution(0)
        assert s.get_option("resident") == "0"
        s.close()


@pytest.mark.parametrize("kernel", ["tma", "direct"])
@pytest.mark.parametrize("path", CASES, ids=[os.path.basename(p)[:-4] for p in CASES])
def test_bit_exact_vs_reference_fixture(path, kernel):
    meta, arrays = load_golden(path)
    R = int(meta["ref_tag"].split("-r")[1].split("-")[0].split(".")[0])
    eb = 8 if "fp64" in meta["ref_tag"] else 4
    ins = regen_inputs(meta)
    got = run(meta["n"], meta["steps"], ins, R, eb, contract_mode_of(meta["ref_tag"]), {"kernel": kernel})
    ref = arrays[f"p.t{meta['vars']['p']['steps'][1]}"]
    assert got.dtype == _dt(eb) and np.array_equal(_bits(got), _bits(ref))


# ragged sizes: nx < 4R, y not a multiple of the 16-row tile, z over several tiles (128 wide in fp32, 64 in fp64) and not a
# multiple of them, z shorter than a tile
RAGGED = [(9, 20, 40), (21, 17, 300), (40, 33, 70), (5, 16, 64)]


@pytest.mark.parametrize("fp_mode", [0, 1, 2])
@pytest.mark.parametrize("eb,R", PREC_RADII)
def test_vs_oracle_ragged(eb, R, fp_mode):
    for i, n in enumerate(RAGGED):
        steps = 2 + i % 2
        ins = inputs(n, 100 + R, R, eb)
        got = run(n, steps, ins, R, eb, fp_mode, {"kernel": "tma"})
        assert np.array_equal(_bits(got), _bits(oracle(ins, R, steps, fp_mode))), (n, R, eb, fp_mode)


# chunk lengths (sweeps of both parities) x persistent grids of 1-3 CTAs, each sweeping several work units
@pytest.mark.parametrize("grid", [1, 2, 3])
@pytest.mark.parametrize("lx", [3, 16, 50])
@pytest.mark.parametrize("eb,R", [(4, 1), (4, 4), (4, 7), (8, 3), (8, 8)])
def test_chunk_lengths_and_persistent_grid(eb, R, lx, grid):
    n = (61, 23, 200)
    ins = inputs(n, 5, R, eb)
    got = run(n, 2, ins, R, eb, 2, {"kernel": "tma", "lx": lx, "grid": grid})
    assert np.array_equal(_bits(got), _bits(oracle(ins, R, 2, 2)))


def _fill_hash(s, seed):
    p = s.get_var("p")
    for t in (0, 1):
        p.fill_hash(t, seed, var_salt("p", t), -1.0, 1.0)
    s.get_var("v").fill_hash(0, seed, var_salt("v", 0), 0.05, 0.3)
    for name in CR:
        s.get_var(name).fill_hash(0, seed, var_salt(name, 0), 0.92, 1.0)


@pytest.mark.parametrize("eb,R", [(4, 1), (4, 4), (4, 7), (8, 3), (8, 8)])
def test_tma_equals_direct_large(eb, R):
    n = (512,) * 3 if eb == 4 else (256,) * 3
    outs = []
    for kernel in ("tma", "direct"):
        s = make(n, R, eb, 2, {"kernel": kernel})
        s.prepare_solution(0)
        _fill_hash(s, 3)
        s.run_solution(0, 1)
        outs.append(result(s))
        s.close()
    assert np.array_equal(_bits(outs[0]), _bits(outs[1]))
    assert np.isfinite(outs[0]).all()


@pytest.mark.parametrize("eb,R", [(4, 2), (4, 7), (8, 3), (8, 8)])
def test_cr_one_is_plain_iso3dfd(eb, R):
    n, steps = (30, 21, 140), 3
    ins = inputs(n, 17, R, eb, cr=False)
    got = run(n, steps, ins, R, eb)
    s = capi.Solution("iso3dfd", radius=R, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    s.prepare_solution(0)
    load(s, ins)
    s.run_solution(0, steps - 1)
    ref = result(s)
    s.close()
    assert np.array_equal(_bits(got), _bits(ref))


@pytest.mark.parametrize("eb,R", [(4, 2), (4, 5), (8, 4), (8, 7)])
def test_halo_cells_and_cr_untouched(eb, R):
    n = (20, 19, 150)
    ins = inputs(n, 9, R, eb)
    s = make(n, R, eb, 2, {"kernel": "tma"})
    s.prepare_solution(0)
    load(s, ins)
    s.run_solution(0, 2)
    p = s.get_var("p")
    for t in range(p.get_first_valid_step_index(), p.get_last_valid_step_index() + 1):
        full = p.get_elements_in_slice(*p.halo_box(t))
        src = ins[("p", t % 2)]
        inner = np.ones(full.shape, bool)
        inner[R:-R, R:-R, R:-R] = False
        assert np.array_equal(_bits(full[inner]), _bits(src[inner])), t
    for name in CR:
        var = s.get_var(name)
        assert np.array_equal(_bits(var.get_elements_in_slice(*var.halo_box(0))), _bits(ins[(name, 0)])), name
    s.close()


def run_grid(n, R, eb, grid, steps=3, seed=21, opts=None):
    solns = []
    for r in range(grid[0] * grid[1] * grid[2]):
        s = make(n, R, eb, 2, opts)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        s.prepare_solution(0)
        solns.append(s)
    if len(solns) > 1:
        multi.connect_local(solns)
    for s in solns:
        _fill_hash(s, seed)      # hash data of global indices, cr vars included
    for s in solns:
        s.run_solution(0, steps - 1)
    for s in solns:
        s.sync()
    out = np.zeros(n, _dt(eb))
    for s in solns:
        p = s.get_var("p")
        f, l = p.domain_box(p.get_last_valid_step_index())
        out[f[1]:l[1] + 1, f[2]:l[2] + 1, f[3]:l[3] + 1] = p.get_elements_in_slice(f, l)
        s.close()
    return out


# fp32: per-rank nx = 4R+1 (fused peer stores and the in-kernel signal) and 3R (in [2R, 4R): fused stores, no signal) on 2x1x1;
# uneven 3x1x1, 1x2x1 and 1x1x2.  fp64: the exterior / interior split.
GRIDS = [(4, R, (2 * (4 * R + 1), 24, 140), (2, 1, 1)) for R in (1, 4, 7)] + \
        [(4, R, (2 * 3 * R, 24, 140), (2, 1, 1)) for R in (2, 4, 7)] + \
        [(4, 3, (47, 20, 100), (3, 1, 1)), (4, 5, (40, 48, 96), (1, 2, 1)), (4, 2, (24, 20, 160), (1, 1, 2)),
         (4, 7, (30, 20, 200), (1, 1, 2)),
         (8, 3, (40, 24, 96), (2, 1, 1)), (8, 8, (48, 24, 96), (2, 1, 1)), (8, 5, (30, 40, 70), (1, 2, 1)),
         (8, 7, (30, 20, 160), (1, 1, 2))]


@pytest.mark.parametrize("eb,R,n,grid", GRIDS, ids=[f"fp{8 * e}-r{r}-{'x'.join(map(str, g))}-nx{n[0]}" for e, r, n, g in GRIDS])
def test_rank_grid_matches_single_rank(eb, R, n, grid):
    ref = run_grid(n, R, eb, (1, 1, 1))
    out = run_grid(n, R, eb, grid)
    assert np.array_equal(_bits(out), _bits(ref))


@pytest.mark.parametrize("eb,R", [(4, 1), (4, 2), (8, 3)])
def test_block_steps_2_same_bits(eb, R):
    n = (40, 24, 160)
    ins = inputs(n, 12, R, eb)
    s = make(n, R, eb, 2, {"block_steps": 2})
    s.prepare_solution(0)
    load(s, ins)
    s.run_solution(0, 3)
    got = result(s)
    launches = s.get_stats().kernel_launches
    s.close()
    assert launches == 4       # one step per sweep: the sponge form has no temporal tile
    assert np.array_equal(_bits(got), _bits(oracle(ins, R, 4, 2)))


@pytest.mark.parametrize("eb,R", [(4, 4), (8, 4), (8, 8)])
def test_auto_tuner_keeps_results_exact(eb, R):
    n = (96, 40, 130)
    ins = inputs(n, 31, R, eb)
    s = make(n, R, eb)
    s.prepare_solution(0)
    report = s.run_auto_tuner_now()
    if eb == 8:
        assert "lx=" in report and "best" in report
    load(s, ins)
    s.run_solution(0, 2)
    got = result(s)
    s.close()
    assert np.array_equal(_bits(got), _bits(oracle(ins, R, 3, 2)))


@pytest.mark.parametrize("lib", ["iso3dfd_sponge_r4", "iso3dfd_sponge_r4_fp64"])
def test_harness_validate(lib):
    exe = os.path.join(ROOT, "yask_b200", "bin", f"yask_kernel.{lib}.b200.exe")
    r = subprocess.run([exe, "-g", "96", "-validate"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    # the hand-written sweep against its one-thread-per-point kernel (not the generated solutions' check)
    assert "TEST PASSED: 0 mismatch(es) between the sweep and the direct kernel" in r.stdout and "YASK DONE" in r.stdout, r.stdout[-2000:]



# the iso3dfd_sponge Python module at hand-written radii (YASK_B200_RADIUS / YASK_B200_ELEM_BYTES), against the oracle
@pytest.mark.parametrize("eb,R", [(4, 4), (8, 3)])
def test_python_module_runs(eb, R):
    mod = os.path.join(ROOT, "yask_b200", "lib", "python", "iso3dfd_sponge")
    n, steps = (24, 20, 40), 3
    ins = inputs(n, 44, R, eb)
    code = r'''
import sys
import numpy as np
import yask_kernel as yk
n, steps, dt = (24, 20, 40), 3, np.dtype(sys.argv[1])
ins = np.load(sys.argv[2])
fac = yk.yk_factory()
s = fac.new_solution(fac.new_env())
for d, k in zip(s.get_domain_dim_names(), n):
    s.set_overall_domain_size(d, k)
s.prepare_solution()
def box(v, t):
    names = v.get_dim_names()
    f = [t if d == "t" else v.get_first_rank_domain_index(d) - v.get_left_halo_size(d) for d in names]
    l = [t if d == "t" else v.get_last_rank_domain_index(d) + v.get_right_halo_size(d) for d in names]
    return f, l
for v in s.get_vars():
    for t in ([0, 1] if "t" in v.get_dim_names() else [0]):
        a = np.ascontiguousarray(ins[f"{v.get_name()}.t{t}"], dtype=dt)
        assert v.set_elements_in_slice(a.data, *box(v, t)) == a.size
s.run_solution(0, steps - 1)
p = s.get_var("p")
tl = p.get_last_valid_step_index()
f = [tl] + [p.get_first_rank_domain_index(d) for d in "xyz"]
l = [tl] + [p.get_last_rank_domain_index(d) for d in "xyz"]
out = np.zeros([b - a + 1 for a, b in zip(f, l)][1:], dt)
assert p.get_elements_in_slice(out.data, f, l) == out.size
np.save(sys.argv[3], out)
print("ok", s.get_name(), s.get_element_bytes(), p.get_left_halo_size("x"))
'''
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.npz"), os.path.join(d, "out.npy")
        np.savez(src, **{f"{k[0]}.t{k[1]}": a for k, a in ins.items()})
        env = dict(os.environ, PYTHONPATH=mod, YASK_B200_RADIUS=str(R), YASK_B200_ELEM_BYTES=str(eb))
        r = subprocess.run([sys.executable, "-c", code, np.dtype(_dt(eb)).name, src, dst], capture_output=True, text=True,
                           timeout=300, env=env)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        assert r.stdout.split() == ["ok", "iso3dfd_sponge", str(eb), str(R)]
        got = np.load(dst)
    assert np.array_equal(_bits(got), _bits(oracle(ins, R, steps, 2)))
