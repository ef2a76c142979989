"""GPU: 3axis, 3axis_with_diags, 3plane and cube at radius 1..8 in fp32 and fp64 on the hand-written average-of-points sweep
(yask_b200/csrc/yb_avepts.cuh).
  * sweep and direct kernels bit-exact against the unmodified reference built at other radii, both builds (tests/golden/<shape>-r*);
  * against the oracle (tests/avepts_oracle.py) for every shape x radius 1-8 x fp32/fp64 on ragged domains, 1-3 steps, fp_mode 0
    and 2;
  * sweep == direct by checksum at a size the oracle cannot reach; halo cells untouched;
  * rank grids equal to one rank bit for bit; the harness's -validate and the shapes' Python modules with YASK_B200_RADIUS.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from tests import avepts_oracle as A
from tests.helpers import golden_cases, load_golden, regen_inputs
from yask_b200 import capi, multi
from yask_b200.synth import hash_field, var_salt

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [p for s in A.SHAPES for r in (1, 2, 5, 8) for p in golden_cases(f"{s}-r{r}")] + \
        [p for s in A.SHAPES for r in (2, 8) for p in golden_cases(f"{s}-fp64-r{r}")]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _dt(eb):
    return np.float32 if eb == 4 else np.float64


def inputs(n, seed, R, eb):
    return [hash_field(seed, var_salt("A", t), (-R,) * 3, [i + 2 * R for i in n], -1, 1, _dt(eb)) for t in (0, 1)]


def make(shape, n, R, eb, opts=None):
    s = capi.Solution(shape, radius=R, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    for k, v in (opts or {}).items():
        s.set_option(k, v)
    return s


def result(s, halo=False):
    a = s.get_var("A")
    t = a.get_last_valid_step_index()
    return a.get_elements_in_slice(*(a.halo_box(t) if halo else a.domain_box(t)))


def run(shape, n, steps, ins, R, eb, opts=None, halo=False):
    s = make(shape, n, R, eb, opts)
    s.prepare_solution(0)
    a = s.get_var("A")
    for t in (0, 1):
        a.set_elements_in_slice(ins[t], *a.halo_box(t))
    s.run_solution(0, steps - 1)
    out = result(s, halo)
    s.close()
    return out


def test_hand_written_form_takes_kernel_option():
    for shape in A.SHAPES:
        for R, eb in ((1, 4), (8, 4), (A.DEFAULT_RADIUS[shape], 8)):
            s = make(shape, (24, 24, 64), R, eb, {"kernel": "tma"})     # the generated engines have no option `kernel`
            s.prepare_solution(0)
            assert s.get_option("kernel") == "tma"
            s.close()


@pytest.mark.parametrize("kernel", ["tma", "direct"])
@pytest.mark.parametrize("path", CASES, ids=[os.path.basename(p)[:-4] for p in CASES])
def test_bit_exact_vs_reference_fixture(path, kernel):
    meta, arrays = load_golden(path)
    shape = meta["ref_tag"].split("-")[0]
    R = int(meta["ref_tag"].split("-r")[1].split("-")[0].split(".")[0])
    eb = 8 if "fp64" in meta["ref_tag"] else 4
    ins = regen_inputs(meta)
    # cube radius 2 in fp32 is the generated form: its sweep and direct kernels (option gen_sweep)
    opts = {"gen_sweep": int(kernel == "tma")} if eb == 4 and R == A.DEFAULT_RADIUS[shape] else {"kernel": kernel}
    got = run(shape, meta["n"], meta["steps"], [ins[("A", 0)], ins[("A", 1)]], R, eb, opts)
    ref = arrays[f"A.t{meta['vars']['A']['steps'][1]}"]
    assert got.dtype == _dt(eb) and np.array_equal(_bits(got), _bits(ref))


# ragged: y not a multiple of the 16-row tile, z over several tiles (64 wide in fp32, 32 in fp64) and not a multiple of 4, nx small
RAGGED = [(9, 21, 70), (17, 17, 131)]


@pytest.mark.parametrize("fp_mode", [0, 2])
@pytest.mark.parametrize("eb", [4, 8])
@pytest.mark.parametrize("R", range(1, 9))
@pytest.mark.parametrize("shape", A.SHAPES)
def test_vs_oracle_ragged(shape, R, eb, fp_mode):
    opts = {"fp_mode": fp_mode}
    if eb == 8 or R != A.DEFAULT_RADIUS[shape]:     # (the default radius in fp32 is the generated form, which has no `kernel`)
        opts["kernel"] = "tma"
    for i, n in enumerate(RAGGED):
        steps = 1 + (R + i) % 3
        ins = inputs(n, 100 + R, R, eb)
        got = run(shape, n, steps, ins, R, eb, opts, halo=True)
        ref = A.run(ins[0], ins[1], shape, R, steps)
        assert np.array_equal(_bits(got), _bits(ref)), (shape, n, R, eb, fp_mode)    # halo cells untouched too


# chunk lengths x persistent grids of 1-3 CTAs, each sweeping several work units
@pytest.mark.parametrize("grid", [1, 3])
@pytest.mark.parametrize("lx", [3, 50])
@pytest.mark.parametrize("shape,R,eb", [("3axis", 1, 4), ("cube", 3, 4), ("3plane", 8, 8), ("3axis_with_diags", 5, 8)])
def test_chunk_lengths_and_persistent_grid(shape, R, eb, lx, grid):
    n = (61, 23, 100)
    ins = inputs(n, 5, R, eb)
    got = run(shape, n, 2, ins, R, eb, {"kernel": "tma", "lx": lx, "grid": grid})
    assert np.array_equal(_bits(got), _bits(A.run(ins[0], ins[1], shape, R, 2)[R:-R, R:-R, R:-R]))


def _fill_hash(s, seed):
    a = s.get_var("A")
    for t in (0, 1):
        a.fill_hash(t, seed, var_salt("A", t), -1.0, 1.0)


@pytest.mark.parametrize("shape,R,eb", [(s, r, e) for s in A.SHAPES for r, e in ((8, 4), (3, 8))])
def test_tma_equals_direct_large(shape, R, eb):
    n = (256, 200, 300) if shape != "cube" else (96, 200, 300)
    sums = []
    for kernel in ("tma", "direct"):
        s = make(shape, n, R, eb, {"kernel": kernel})
        s.prepare_solution(0)
        _fill_hash(s, 3)
        s.run_solution(0, 1)
        a = s.get_var("A")
        sums.append(a.checksum(a.get_last_valid_step_index()))
        s.close()
    assert sums[0] == sums[1]


def run_grid(shape, n, R, eb, grid, steps=3, seed=21):
    solns = []
    for r in range(grid[0] * grid[1] * grid[2]):
        s = make(shape, n, R, eb)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        s.prepare_solution(0)
        solns.append(s)
    if len(solns) > 1:
        multi.connect_local(solns)
    for s in solns:
        _fill_hash(s, seed)
    for s in solns:
        s.run_solution(0, steps - 1)
    for s in solns:
        s.sync()
    out = np.zeros(n, _dt(eb))
    for s in solns:
        a = s.get_var("A")
        f, l = a.domain_box(a.get_last_valid_step_index())
        out[f[1]:l[1] + 1, f[2]:l[2] + 1, f[3]:l[3] + 1] = a.get_elements_in_slice(f, l)
        s.close()
    return out


# cube (corners) and 3axis_with_diags (edges) on face, edge and corner neighbours; 3axis on a z split
GRIDS = [(s, R, eb, g) for s in ("cube", "3axis_with_diags") for R, eb in ((3, 4), (2, 8))
         for g in ((2, 1, 1), (1, 2, 1), (1, 1, 2), (2, 2, 2))] + [("3axis", 1, 4, (1, 1, 2)), ("3plane", 5, 4, (2, 2, 1))]


@pytest.mark.parametrize("shape,R,eb,grid", GRIDS, ids=[f"{s}-r{r}-fp{8 * e}-{'x'.join(map(str, g))}" for s, r, e, g in GRIDS])
def test_rank_grid_matches_single_rank(shape, R, eb, grid):
    n = (32, 40, 96)
    ref = run_grid(shape, n, R, eb, (1, 1, 1))
    out = run_grid(shape, n, R, eb, grid)
    assert np.array_equal(_bits(out), _bits(ref))


def test_auto_tuner_keeps_results_exact():
    n, R, eb = (96, 40, 130), 2, 8
    ins = inputs(n, 31, R, eb)
    s = make("cube", n, R, eb)
    s.prepare_solution(0)
    report = s.run_auto_tuner_now()
    assert "lx=" in report and "best" in report
    a = s.get_var("A")
    for t in (0, 1):
        a.set_elements_in_slice(ins[t], *a.halo_box(t))
    s.run_solution(0, 2)
    got = result(s)
    s.close()
    assert np.array_equal(_bits(got), _bits(A.run(ins[0], ins[1], "cube", R, 3)[R:-R, R:-R, R:-R]))


@pytest.mark.parametrize("lib", ["3axis_r1", "3axis_with_diags_r2", "3plane_r1", "cube_r1_fp64"])
def test_harness_validate(lib):
    exe = os.path.join(ROOT, "yask_b200", "bin", f"yask_kernel.{lib}.b200.exe")
    r = subprocess.run([exe, "-g", "96", "-validate"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "TEST PASSED: 0 mismatch(es)" in r.stdout and "YASK DONE" in r.stdout, r.stdout[-2000:]


MODULE_SCRIPT = r'''
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
a = s.get_var("A")
for t in (0, 1):
    f = [t] + [a.get_first_rank_domain_index(d) - a.get_left_halo_size(d) for d in "xyz"]
    l = [t] + [a.get_last_rank_domain_index(d) + a.get_right_halo_size(d) for d in "xyz"]
    v = np.ascontiguousarray(ins[f"A.t{t}"], dtype=dt)
    assert a.set_elements_in_slice(v.data, f, l) == v.size
s.run_solution(0, steps - 1)
tl = a.get_last_valid_step_index()
f = [tl] + [a.get_first_rank_domain_index(d) for d in "xyz"]
l = [tl] + [a.get_last_rank_domain_index(d) for d in "xyz"]
out = np.zeros([b - c + 1 for c, b in zip(f, l)][1:], dt)
assert a.get_elements_in_slice(out.data, f, l) == out.size
np.save(sys.argv[3], out)
print("ok", s.get_name(), s.get_element_bytes(), a.get_left_halo_size("x"))
'''


@pytest.mark.parametrize("shape,R,eb", [("3axis", 1, 4), ("cube", 3, 8)])
def test_python_module_runs(shape, R, eb):
    mod = os.path.join(ROOT, "yask_b200", "lib", "python", shape)
    n, steps = (24, 20, 40), 3
    ins = inputs(n, 44, R, eb)
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.npz"), os.path.join(d, "out.npy")
        np.savez(src, **{f"A.t{t}": a for t, a in enumerate(ins)})
        env = dict(os.environ, PYTHONPATH=mod, YASK_B200_RADIUS=str(R), YASK_B200_ELEM_BYTES=str(eb))
        r = subprocess.run([sys.executable, "-c", MODULE_SCRIPT, np.dtype(_dt(eb)).name, src, dst], capture_output=True,
                           text=True, timeout=300, env=env)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        assert r.stdout.split() == ["ok", shape, str(eb), str(R)]
        got = np.load(dst)
    assert np.array_equal(_bits(got), _bits(A.run(ins[0], ins[1], shape, R, steps)[R:-R, R:-R, R:-R]))
