"""GPU: solutions run on domains past 2^31 elements per var slot, bit for bit.

Each case fills the whole domain on the device with fill_hash (a hash of global indices), runs a few steps in the default FP
mode and compares three windows with the CPU oracle run over the same windows (tests/large_domain.py): one at the low corner,
one straddling the x plane where the element offset crosses 2^31 and one at the high corner.  A case needs tens of GB; it is
skipped, with the amount in the reason, when the device has less free memory than that plus a 2 GB margin.
"""
import os
import re
import subprocess

import numpy as np
import pytest

from tests.large_domain import (TWO31, bits, fill_gen, fill_iso, gen_reach, gen_window_ref, iso_window_ref, storage_bytes,
                                three_windows)
from yask_b200 import capi

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MARGIN = 2 << 30


def _need(s):
    """Skip unless the device has room for the solution's vars plus the margin; returns the bytes they need."""
    import torch
    need = storage_bytes(s)
    free, _ = torch.cuda.mem_get_info()
    if free < need + MARGIN:
        s.close()
        pytest.skip(f"needs {need / 1e9:.1f} GB of device memory plus a 2 GB margin, {free / 1e9:.1f} GB free")
    return need


def _main_info(s):
    vi = max((v.info for v in s.get_vars()), key=lambda i: i.slot_elems)
    assert vi.slot_elems > TWO31
    return vi


def _gen_solution(stencil, radius, eb, n, opts):
    s = capi.Solution(stencil, radius=radius, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    for k, v in opts.items():
        s.set_option(k, v)
    return s


# (registry name of the oracle's IR, solution, radius, elem_bytes, size, steps, forms)
GEN_CASES = [
    ("3axis", "3axis", 0, 0, (1300, 1300, 1300), 2, ({"gen_sweep": 1}, {"gen_sweep": 0})),
    ("iso3dfd_sponge", "iso3dfd_sponge", 8, 4, (1300, 1300, 1300), 2, ({"gen_sweep": 1}, {"gen_sweep": 0})),
    ("test_2d", "test_2d", 0, 0, (47000, 47000), 3, ({},)),
    ("iso3dfd_fp64", "iso3dfd", 8, 8, (1300, 1300, 1300), 2, ({},)),
]


@pytest.mark.parametrize("ir_name,stencil,radius,eb,n,steps,forms", GEN_CASES, ids=[c[0] for c in GEN_CASES])
def test_generated_past_2_31(ir_name, stencil, radius, eb, n, steps, forms):
    seed = 61
    m = steps * gen_reach(ir_name)
    size = [32 + m] * len(n)
    sums = []
    for opts in forms:
        s = _gen_solution(stencil, radius, eb, n, opts)
        _need(s)
        wins = three_windows(_main_info(s), n, size, m)
        assert s.get_option("fp_mode") == "2"
        try:
            s.prepare_solution(0)
            fill_gen(s, ir_name, seed)
            s.run_solution(0, steps - 1)
            # the sweep form (the default) really ran its TMA sweep kernels at this size, the direct form none (a 2-D solution
            # has no sweep kernels: they stream full-rank 3-D vars)
            launched = int(s.get_option("gen_sweep_launches"))
            assert (launched > 0) == (opts.get("gen_sweep", 1) == 1 and len(n) == 3), (ir_name, opts, launched)
            got, cs = [], {}
            for var in s.get_vars():
                vi = var.info
                if not vi.is_output:
                    continue
                name, tl = vi.name.decode(), vi.last_valid_step
                cs[name] = var.checksum(tl)
                got.append((name, tl, [var.get_elements_in_slice(*w.kept_box(tl)) for w in wins]))
        finally:
            s.close()      # the next case needs the memory even when this one fails
        sums.append(cs)
        for i, w in enumerate(wins):
            ref = gen_window_ref(ir_name, w, seed, steps, 1)
            for name, tl, arrs in got:
                assert ref[name][0] == tl
                assert np.array_equal(bits(arrs[i]), bits(ref[name][1])), (ir_name, opts, name, w.lo)
    assert all(c == sums[0] for c in sums), f"{ir_name}: the sweep and the direct kernels disagree"


# (radius, elem_bytes, size, steps, forms); the fp32 radius-8 default is the resident ring, radius 2 with block_steps=2 the
# temporal tile
ISO_CASES = [
    (8, 4, (1300, 1300, 1300), 2, ({}, {"kernel": "direct"})),
    (4, 8, (1300, 1300, 1300), 2, ({},)),
    (2, 4, (1300, 1300, 1300), 4, ({"block_steps": 2},)),
]


@pytest.mark.parametrize("R,eb,n,steps,forms", ISO_CASES, ids=["fp32-r8", "fp64-r4", "fp32-r2-tt"])
def test_hand_written_iso3dfd_past_2_31(R, eb, n, steps, forms):
    seed = 67
    dt = np.float32 if eb == 4 else np.float64
    m = steps * R
    size = [32 + m] * 3
    sums = []
    for opts in forms:
        s = _gen_solution("iso3dfd", R, eb, n, opts)
        _need(s)
        p = s.get_var("p")
        h = p.info.dims[1].left_halo
        wins = three_windows(_main_info(s), n, size, m)
        try:
            s.prepare_solution(0)
            assert s.get_element_bytes() == eb and s.get_option("fp_mode") == "2"
            if "kernel" not in opts and "block_steps" not in opts and R == 8 and eb == 4:
                assert s.get_option("resident") == "1"
            fill_iso(s, seed)
            s.run_solution(0, steps - 1)
            tl = p.get_last_valid_step_index()
            got = [p.get_elements_in_slice(*w.kept_box(tl)) for w in wins]
            sums.append(p.checksum(tl))
            st = s.get_stats()
        finally:
            s.close()
        if opts.get("block_steps") == 2:
            assert st.kernel_launches == steps // 2, "the temporal tile did not take the fused path"
        for g, w in zip(got, wins):
            assert np.array_equal(bits(g), bits(iso_window_ref(w, seed, R, h, steps, 2, dt))), (R, eb, opts, w.lo)
    assert all(c == sums[0] for c in sums)


def test_harness_past_2_31():
    """The command-line harness (C++ API) runs a 3axis domain past 2^31 elements per slot and reports a throughput."""
    n = 1300
    s = capi.Solution("3axis", elem_bytes=0)
    s.set_overall_domain_size_vec((n, n, n))
    _need(s)
    _main_info(s)
    s.close()
    exe = os.path.join(ROOT, "yask_b200", "bin", "yask_kernel.3axis.b200.exe")
    r = subprocess.run([exe, "-g", str(n), "-num_trials", "1", "-trial_steps", "2"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-2000:])
    assert re.search(r"best-throughput \(num-points/sec\):\s+[0-9.]+[KMGT]?", r.stdout), r.stdout[-3000:]
