"""GPU: the average-of-points temporal tile (option block_steps / -bt 2; yask_b200/csrc/yb_avepts_tt.cuh): two steps per sweep for
3axis at radius 1 and 2, fp32 and fp64.  Every comparison is bit for bit.
  * the unmodified reference's fixtures: two steps are one fused launch;
  * the oracle (tests/avepts_oracle.py) on ragged domains that cross the tile edges in y and z, a short last x chunk, 1-4 and 7
    steps, fp_mode 0 and 2: both valid steps with their halo cells, and one launch per pair plus one for an odd step;
  * halo cells of the two slots that differ: split runs equal one run of one step per sweep (step 1 takes its boundary values from
    the halo of the slot of t+1; the last pair of a run stores its intermediate step);
  * persistent grids, a size the oracle cannot reach, the offline tuner;
  * block_steps=2 where there is no tile (3axis_with_diags, 3plane and cube, which were slower with pairs; other radii;
    kernel=direct; a rank grid) changes nothing;
  * the harness's -bt 2 -validate and the Python module's set_block_size("t", 2).
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
from yask_b200.synth import var_salt

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILED = [("3axis", r, eb) for r in (1, 2) for eb in (4, 8)]
TILED_IDS = [f"{s}-r{r}-fp{8 * e}" for s, r, e in TILED]
PAIRS = {"block_steps": 2, "kernel": "tma"}


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _dt(eb):
    return np.float32 if eb == 4 else np.float64


def inputs(n, seed, R, eb):
    from yask_b200.synth import hash_field
    return [hash_field(seed, var_salt("A", t), (-R,) * 3, [i + 2 * R for i in n], -1, 1, _dt(eb)) for t in (0, 1)]


def prepared(shape, n, R, eb, opts, ins=None):
    s = capi.Solution(shape, radius=R, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    for k, v in opts.items():
        s.set_option(k, v)
    s.prepare_solution(0)
    if ins is not None:
        a = s.get_var("A")
        for t in (0, 1):
            a.set_elements_in_slice(ins[t], *a.halo_box(t))
    return s


def valid_steps(s):
    """Both valid steps of A, halo cells included: (older, newer)."""
    a = s.get_var("A")
    tl = a.get_last_valid_step_index()
    return [a.get_elements_in_slice(*a.halo_box(t)) for t in (tl - 1, tl)]


def slots(s):
    a = s.get_var("A").info
    return a.storage_bytes // (a.slot_elems * a.elem_bytes)


# ---- 1. the reference's fixtures ----------------------------------------------------------------------------------------------
FIXTURES = [p for r in (1, 2) for p in golden_cases(f"3axis-r{r}")]


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p)[:-4] for p in FIXTURES])
def test_bit_exact_vs_reference_fixture(path):
    meta, arrays = load_golden(path)
    shape = meta["ref_tag"].split("-")[0]
    R = int(meta["ref_tag"].split("-r")[1].split("-")[0].split(".")[0])
    ins = regen_inputs(meta)
    assert meta["steps"] == 2
    s = prepared(shape, meta["n"], R, 4, PAIRS, [ins[("A", 0)], ins[("A", 1)]])
    s.run_solution(0, 1)
    a = s.get_var("A")
    got = a.get_elements_in_slice(*a.domain_box(a.get_last_valid_step_index()))
    launches, tt = s.get_stats().kernel_launches, s.get_option("tt_launches")
    s.close()
    assert tt == "1" and launches == 1
    assert np.array_equal(_bits(got), _bits(arrays[f"A.t{meta['vars']['A']['steps'][1]}"]))


# ---- 2. the oracle ------------------------------------------------------------------------------------------------------------
# y crosses the 16-row tile; z crosses the 64-element (fp32) / 32-element (fp64) tile and ends in a partial 16-byte vector in both;
# lx = 5 splits x = 13 into chunks of 4, 4 and 5 planes
RAGGED, LX = (13, 21, 67), 5


@pytest.mark.parametrize("fp_mode", [0, 2])
@pytest.mark.parametrize("shape,R,eb", TILED, ids=TILED_IDS)
def test_vs_oracle_ragged(shape, R, eb, fp_mode):
    ins = inputs(RAGGED, 200 + R, R, eb)
    for steps in (1, 2, 3, 4, 7):
        s = prepared(shape, RAGGED, R, eb, dict(PAIRS, fp_mode=fp_mode, lx=LX), ins)
        assert slots(s) == 4
        s.run_solution(0, steps - 1)
        got = valid_steps(s)
        launches, tt = s.get_stats().kernel_launches, int(s.get_option("tt_launches"))
        s.close()
        assert launches == steps // 2 + steps % 2 and tt == steps // 2, (steps, launches, tt)
        for k, g in enumerate(got):
            ref = A.run(ins[0], ins[1], shape, R, steps - 1 + k)
            assert np.array_equal(_bits(g), _bits(ref)), (shape, R, eb, fp_mode, steps, k)


# ---- 3. halo cells of the slot of t+1, the intermediate step of the last pair -----------------------------------------------------
@pytest.mark.parametrize("shape,R,eb", TILED, ids=TILED_IDS)
def test_split_runs_equal_one_step_per_sweep(shape, R, eb):
    n = (19, 23, 45)
    ins = inputs(n, 300 + R, R, eb)         # the two slots' halo cells hold different values
    s = prepared(shape, n, R, eb, PAIRS, ins)
    for a, b in ((0, 1), (2, 4), (5, 5)):
        s.run_solution(a, b)
    got, tt = valid_steps(s), s.get_option("tt_launches")
    s.close()
    r = prepared(shape, n, R, eb, {"kernel": "tma"}, ins)
    r.run_solution(0, 5)
    ref = valid_steps(r)
    r.close()
    assert tt == "2"
    for g, e in zip(got, ref):
        assert np.array_equal(_bits(g), _bits(e))
    assert np.array_equal(_bits(ref[1]), _bits(A.run(ins[0], ins[1], shape, R, 6)))


# ---- 4. persistent grids ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", [1, 3])
@pytest.mark.parametrize("lx", [3, 50])
@pytest.mark.parametrize("shape,R,eb", TILED, ids=TILED_IDS)
def test_chunk_lengths_and_persistent_grid(shape, R, eb, lx, grid):
    n = (61, 23, 100)
    ins = inputs(n, 5, R, eb)
    s = prepared(shape, n, R, eb, dict(PAIRS, lx=lx, grid=grid), ins)
    s.run_solution(0, 3)
    got, tt = valid_steps(s), s.get_option("tt_launches")
    s.close()
    assert tt == "2"
    for k, g in enumerate(got):
        assert np.array_equal(_bits(g), _bits(A.run(ins[0], ins[1], shape, R, 3 + k)))


# ---- 5. a size the oracle cannot reach ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,R,eb", TILED, ids=TILED_IDS)
def test_pairs_equal_one_step_per_sweep_large(shape, R, eb):
    n, steps = (256, 300, 520), 4 + TILED.index((shape, R, eb)) % 2
    sums = []
    for opts in (PAIRS, {"kernel": "tma"}):
        s = prepared(shape, n, R, eb, opts)
        a = s.get_var("A")
        for t in (0, 1):
            a.fill_hash(t, 7, var_salt("A", t), -1.0, 1.0)
        s.run_solution(0, steps - 1)
        tl = a.get_last_valid_step_index()
        sums.append((a.checksum(tl - 1), a.checksum(tl), s.get_option("tt_launches")))
        s.close()
    assert sums[0][2] == str(steps // 2) and sums[1][2] == "0"
    assert sums[0][:2] == sums[1][:2]


# ---- 6. the offline tuner -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,R,eb", [("3axis", 1, 4), ("3axis", 2, 8)])
def test_auto_tuner_times_both_paths(shape, R, eb):
    n = (96, 40, 130)
    ins = inputs(n, 31, R, eb)
    s = prepared(shape, n, R, eb, {"block_steps": 2})
    report = s.run_auto_tuner_now()
    assert "one step per sweep" in report and "two steps per sweep" in report and "best" in report, report
    assert s.get_option("block_steps") in ("1", "2")
    a = s.get_var("A")
    for t in (0, 1):
        a.set_elements_in_slice(ins[t], *a.halo_box(t))
    s.run_solution(0, 4)
    got = valid_steps(s)
    s.close()
    for k, g in enumerate(got):
        assert np.array_equal(_bits(g), _bits(A.run(ins[0], ins[1], shape, R, 4 + k)))


# ---- 7. no tile: block_steps=2 changes nothing ---------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,R,eb,opts", [("3axis_with_diags", 1, 4, {}), ("3axis_with_diags", 2, 8, {}), ("3plane", 1, 4, {}),
                                            ("cube", 1, 8, {}), ("3plane", 2, 4, {}), ("cube", 2, 8, {}), ("3axis", 3, 4, {}),
                                            ("3axis", 1, 4, {"kernel": "direct"}), ("3axis", 2, 8, {"kernel": "direct"})],
                         ids=["diags-r1", "diags-r2-fp64", "3plane-r1", "cube-r1-fp64", "3plane-r2", "cube-r2-fp64", "3axis-r3",
                              "3axis-r1-direct", "3axis-r2-fp64-direct"])
def test_block_steps_without_tile_is_inert(shape, R, eb, opts):
    n = (19, 23, 45)
    ins = inputs(n, 400 + R, R, eb)
    s = prepared(shape, n, R, eb, dict(opts, block_steps=2), ins)
    nslots = slots(s)
    s.run_solution(0, 3)
    got, tt = valid_steps(s), s.get_option("tt_launches")
    s.close()
    assert nslots == 2 and tt == "0"
    for k, g in enumerate(got):
        assert np.array_equal(_bits(g), _bits(A.run(ins[0], ins[1], shape, R, 3 + k)))


def _run_grid(shape, n, R, eb, grid, opts, steps=4):
    solns = []
    for r in range(grid[0] * grid[1] * grid[2]):
        s = capi.Solution(shape, radius=R, elem_bytes=eb)
        s.set_overall_domain_size_vec(n)
        s.set_num_ranks_vec(grid)
        s.set_rank_index_vec(multi.grid_coords(r, grid))
        for k, v in opts.items():
            s.set_option(k, v)
        s.prepare_solution(0)
        solns.append(s)
    if len(solns) > 1:
        multi.connect_local(solns)
    for s in solns:
        a = s.get_var("A")
        for t in (0, 1):
            a.fill_hash(t, 23, var_salt("A", t), -1.0, 1.0)
    for s in solns:
        s.run_solution(0, steps - 1)
    for s in solns:
        s.sync()
    out = np.zeros(n, _dt(eb))
    info = []
    for s in solns:
        a = s.get_var("A")
        f, l = a.domain_box(a.get_last_valid_step_index())
        out[f[1]:l[1] + 1, f[2]:l[2] + 1, f[3]:l[3] + 1] = a.get_elements_in_slice(f, l)
        info.append((slots(s), s.get_option("tt_launches")))
        s.close()
    return out, info


@pytest.mark.parametrize("shape,R,eb", [("3axis", 1, 4), ("3axis", 2, 8)])
def test_block_steps_on_rank_grid_is_inert(shape, R, eb):
    n = (32, 40, 96)
    ref, _ = _run_grid(shape, n, R, eb, (1, 1, 1), {})
    out, info = _run_grid(shape, n, R, eb, (2, 2, 1), {"block_steps": 2})
    assert info == [(2, "0")] * 4
    assert np.array_equal(_bits(out), _bits(ref))


# ---- 8. the harness and the Python module -------------------------------------------------------------------------------------
@pytest.mark.parametrize("lib", ["3axis_r1", "cube_r1_fp64"])
def test_harness_bt2_validate(lib):
    """3axis_r1 runs the tile; on cube_r1_fp64, which has none, -bt 2 is accepted and changes nothing."""
    exe = os.path.join(ROOT, "yask_b200", "bin", f"yask_kernel.{lib}.b200.exe")
    r = subprocess.run([exe, "-g", "96", "-bt", "2", "-validate"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "TEST PASSED: 0 mismatch(es)" in r.stdout and "YASK DONE" in r.stdout, r.stdout[-2000:]
    assert [l for l in r.stdout.splitlines() if "num-temporal-block-steps" in l][0].split()[-1] == "2"


MODULE_SCRIPT = r'''
import sys
import numpy as np
import yask_kernel as yk
n, steps, dt = (24, 20, 40), 4, np.dtype(sys.argv[1])
ins = np.load(sys.argv[2])
fac = yk.yk_factory()
s = fac.new_solution(fac.new_env())
for d, k in zip(s.get_domain_dim_names(), n):
    s.set_overall_domain_size(d, k)
s.set_block_size("t", 2)
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
print("ok", s.get_block_size("t"), a.get_num_storage_bytes() // (4 if dt == np.float32 else 8))
'''


@pytest.mark.parametrize("shape,R,eb", [("3axis", 2, 4), ("3axis", 1, 8)])
def test_python_module_set_block_size(shape, R, eb):
    mod = os.path.join(ROOT, "yask_b200", "lib", "python", shape)
    n, steps = (24, 20, 40), 4
    ins = inputs(n, 44, R, eb)
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.npz"), os.path.join(d, "out.npy")
        np.savez(src, **{f"A.t{t}": a for t, a in enumerate(ins)})
        env = dict(os.environ, PYTHONPATH=mod, YASK_B200_RADIUS=str(R), YASK_B200_ELEM_BYTES=str(eb))
        r = subprocess.run([sys.executable, "-c", MODULE_SCRIPT, np.dtype(_dt(eb)).name, src, dst], capture_output=True,
                           text=True, timeout=300, env=env)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        words = r.stdout.split()
        got = np.load(dst)
    # the spare pair of slots was allocated: 4 slots of at least (n + 2R) points each
    assert words[:2] == ["ok", "2"] and int(words[2]) >= 4 * np.prod([k + 2 * R for k in n])
    assert np.array_equal(_bits(got), _bits(A.run(ins[0], ins[1], shape, R, steps)[R:-R, R:-R, R:-R]))
