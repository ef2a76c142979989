"""GPU: double-precision iso3dfd on the hand-written fp64 sweep (radius 1, 2, 4, 5, 6, 7), bit for bit:
  * against the reference's fp64 builds (tests/golden/iso3dfd-fp64-r<r>*.npz) with the TMA and the direct kernel,
  * against the CPU oracle at ragged sizes in every FP mode and a few sweep chunk lengths,
  * TMA against direct at 512^3, halo cells untouched, rank grids, block_steps=2 and the offline tuner,
  * through the command-line harness (-validate) and the Python module of the iso3dfd_r4_fp64 library.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import contract_mode_of, golden_cases, load_golden, regen_inputs
from yask_b200 import capi, multi
from yask_b200.synth import hash_field, var_salt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP64_RADII = (1, 2, 4, 5, 6, 7)
CASES = [p for r in FP64_RADII for p in golden_cases(f"iso3dfd-fp64-r{r}")]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def inputs(n, seed, R):
    return {("p", t): hash_field(seed, var_salt("p", t), (-R,) * 3, [i + 2 * R for i in n], -1, 1, np.float64) for t in (0, 1)} | \
           {("v", 0): hash_field(seed, var_salt("v", 0), (0, 0, 0), n, 0.05, 0.3, np.float64)}


def make(n, R, fp_mode=2, opts=None):
    s = capi.Solution("iso3dfd", radius=R, elem_bytes=8)
    s.set_overall_domain_size_vec(n)
    s.set_option("fp_mode", fp_mode)
    for k, v in (opts or {}).items():
        s.set_option(k, v)
    return s


def load(s, ins):
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.set_elements_in_slice(ins[("p", t)], *p.halo_box(t))
    v.set_elements_in_slice(ins[("v", 0)], *v.halo_box(0))


def result(s):
    p = s.get_var("p")
    return p.get_elements_in_slice(*p.domain_box(p.get_last_valid_step_index()))


def run(n, steps, ins, R, fp_mode=2, opts=None):
    s = make(n, R, fp_mode, opts)
    s.prepare_solution(0)
    assert s.get_element_bytes() == 8
    load(s, ins)
    s.run_solution(0, steps - 1)
    out = result(s)
    s.close()
    return out


def oracle(ins, R, steps, mode):
    return O.iso3dfd_run(ins[("p", 0)], ins[("p", 1)], ins[("v", 0)], R, steps, mode)[R:-R, R:-R, R:-R]


@pytest.mark.parametrize("kernel", ["tma", "direct"])
@pytest.mark.parametrize("path", CASES, ids=[os.path.basename(p)[:-4] for p in CASES])
def test_bit_exact_vs_reference_fixture(path, kernel):
    meta, arrays = load_golden(path)
    R = int(meta["ref_tag"].split("-r")[1].split("-")[0].split(".")[0])
    ins = regen_inputs(meta)
    got = run(meta["n"], meta["steps"], ins, R, contract_mode_of(meta["ref_tag"]), {"kernel": kernel})
    ref = arrays[f"p.t{meta['vars']['p']['steps'][1]}"]
    assert got.dtype == np.float64 and np.array_equal(_bits(got), _bits(ref))


# ragged sizes: nz < 64, nz not a multiple of 64, ny not a multiple of 16, nx < 4R
RAGGED = [(9, 20, 40), (21, 17, 130), (40, 33, 70), (5, 16, 64)]


@pytest.mark.parametrize("fp_mode", [0, 1, 2])
@pytest.mark.parametrize("R", FP64_RADII)
def test_vs_oracle_ragged(R, fp_mode):
    for i, n in enumerate(RAGGED):
        steps = 2 + i % 2
        ins = inputs(n, 100 + R, R)
        ref = oracle(ins, R, steps, fp_mode)
        got = run(n, steps, ins, R, fp_mode, {"kernel": "tma"})
        assert np.array_equal(_bits(got), _bits(ref)), (n, R, fp_mode)


@pytest.mark.parametrize("lx", [3, 16, 50])
@pytest.mark.parametrize("R", [1, 4, 7])
def test_chunk_lengths(R, lx):
    n = (61, 23, 100)
    ins = inputs(n, 5, R)
    got = run(n, 2, ins, R, 2, {"kernel": "tma", "lx": lx})
    assert np.array_equal(_bits(got), _bits(oracle(ins, R, 2, 2)))


@pytest.mark.parametrize("R", [1, 4, 7])
def test_tma_equals_direct_512(R):
    n = (512, 512, 512)
    outs = []
    for kernel in ("tma", "direct"):
        s = make(n, R, 2, {"kernel": kernel})
        s.prepare_solution(0)
        p, v = s.get_var("p"), s.get_var("v")
        for t in (0, 1):
            p.fill_hash(t, 3, var_salt("p", t), -1.0, 1.0)
        v.fill_hash(0, 3, var_salt("v", 0), 0.05, 0.3)
        s.run_solution(0, 1)
        outs.append(result(s))
        s.close()
    assert np.array_equal(_bits(outs[0]), _bits(outs[1]))
    assert np.isfinite(outs[0]).all()


@pytest.mark.parametrize("R", [2, 5])
def test_halo_cells_untouched(R):
    n = (20, 19, 70)
    ins = inputs(n, 9, R)
    s = make(n, R, 2, {"kernel": "tma"})
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
    s.close()


@pytest.mark.parametrize("grid", [(2, 1, 1), (1, 2, 1)])
@pytest.mark.parametrize("R", [1, 4])
def test_rank_grid_matches_single_rank(R, grid):
    n, steps, seed = (64, 48, 96), 3, 21

    def fill(s):
        p, v = s.get_var("p"), s.get_var("v")
        for t in (0, 1):
            p.fill_hash(t, seed, var_salt("p", t), -1.0, 1.0)
        v.fill_hash(0, seed, var_salt("v", 0), 0.05, 0.3)

    s = make(n, R)
    s.prepare_solution(0)
    fill(s)
    s.run_solution(0, steps - 1)
    ref = result(s)
    s.close()
    world = grid[0] * grid[1] * grid[2]
    solns = []
    for r in range(world):
        s = make(n, R)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        s.prepare_solution(0)
        solns.append(s)
    multi.connect_local(solns)
    for s in solns:
        fill(s)
    for s in solns:
        s.run_solution(0, steps - 1)
    for s in solns:
        s.sync()
    out = np.zeros(n, np.float64)
    for s in solns:
        p = s.get_var("p")
        f, l = p.domain_box(p.get_last_valid_step_index())
        out[f[1]:l[1] + 1, f[2]:l[2] + 1, f[3]:l[3] + 1] = p.get_elements_in_slice(f, l)
        s.close()
    assert np.array_equal(_bits(out), _bits(ref))


@pytest.mark.parametrize("R", [1, 2])
def test_block_steps_2_same_bits(R):
    n = (40, 24, 160)
    ins = inputs(n, 12, R)
    s = make(n, R, 2, {"block_steps": 2})
    s.prepare_solution(0)
    load(s, ins)
    s.run_solution(0, 3)
    got = result(s)
    launches = s.get_stats().kernel_launches
    s.close()
    assert launches == 4       # one step per sweep: fp64 has no temporal tile
    assert np.array_equal(_bits(got), _bits(oracle(ins, R, 4, 2)))


def test_auto_tuner_keeps_results_exact():
    R, n = 4, (96, 40, 130)
    ins = inputs(n, 31, R)
    s = make(n, R)
    s.prepare_solution(0)
    report = s.run_auto_tuner_now()
    assert "lx=" in report and "best" in report
    load(s, ins)
    s.run_solution(0, 2)
    got = result(s)
    s.close()
    assert np.array_equal(_bits(got), _bits(oracle(ins, R, 3, 2)))


def test_harness_validate():
    exe = os.path.join(ROOT, "yask_b200", "bin", "yask_kernel.iso3dfd_r4_fp64.b200.exe")
    r = subprocess.run([exe, "-g", "96", "-validate"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    # the hand-written sweep against the one-thread-per-point kernel (not the generated solutions' check)
    assert "TEST PASSED: 0 mismatch(es) between the sweep and the direct kernel" in r.stdout and "YASK DONE" in r.stdout, r.stdout[-2000:]


def test_python_module_reports_8_bytes_and_runs():
    mod = os.path.join(ROOT, "yask_b200", "lib", "python", "iso3dfd_r4_fp64")
    code = r'''
import numpy as np
import yask_kernel as yk
fac = yk.yk_factory()
env = fac.new_env()
s = fac.new_solution(env)
assert s.get_element_bytes() == 8, s.get_element_bytes()
for d in s.get_domain_dim_names():
    s.set_overall_domain_size(d, 48)
s.prepare_solution()
for v in s.get_vars():
    v.set_all_elements_same(0.25)
s.run_solution(0, 1)
p = s.get_var("p")
print("ok", s.get_element_bytes(), p.get_element([1, 5, 5, 5]))
'''
    env = dict(os.environ, PYTHONPATH=mod)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert r.stdout.split()[:2] == ["ok", "8"]
