"""Slice recorders through the reference-style APIs users already have: the `yask_kernel` Python module and the C++ functions it
binds (yask_b200/include/yask_b200_slices.hpp).  The frames of one run_solution() call must equal, bit for bit, the reference API
loop run_solution(t) / get_elements_in_slice of the same module."""
import glob
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOD = glob.glob(os.path.join(ROOT, "yask_b200", "lib", "python", "iso3dfd", "yask_kernel*.so"))

SCRIPT = textwrap.dedent("""
    import struct
    import numpy as np
    import yask_kernel as yk

    steps, n = 6, (40, 36, 64)
    fac, env = yk.yk_factory(), None

    def solution():
        global env
        env = env or fac.new_env()
        s = fac.new_solution(env)
        s.set_overall_domain_size_vec(list(n))
        s.prepare_solution()
        s.get_var("v").set_all_elements_same(0.1)
        p = s.get_var("p")
        p.set_all_elements_same(0.0)
        p.set_element(0.25, [0, 20, 18, 32])
        p.set_element(-0.5, [1, 21, 17, 30])
        return s

    a = solution()
    first, last, stride = [20, 0, 1], [20, 35, 63], [1, 2, 3]
    rid = yk.yk_add_slice(a, "p", first, last, 2, 2, stride, 2)        # p(2) and p(4)
    assert rid == 0
    a.run_solution(0, steps - 1)
    frames, shape, owned = yk.yk_get_slice_frames(a, rid)
    assert list(shape) == [2, 1, 18, 21] and all(owned), shape
    assert yk.yk_get_slice_launches(a) == 2, yk.yk_get_slice_launches(a)

    b = solution()
    p = b.get_var("p")
    ref = []
    for t in range(steps):
        b.run_solution(t)
        if t + 1 in (2, 4):
            buf = np.zeros((1, 36, 63), np.float32)
            p.get_elements_in_slice(buf, [t + 1] + first, [t + 1] + last)
            ref += buf[:, ::2, ::3].reshape(-1).tolist()
    bits = lambda xs: [struct.pack("<f", x) for x in xs]
    assert bits(frames) == bits(ref)
    try:
        yk.yk_add_slice(a, "p", [1, 2], [3, 4], 0, 1)
        raise SystemExit("a 2-index box was accepted")
    except RuntimeError as e:
        assert "3 domain indices" in str(e), e
    yk.yk_clear_slices(a)
    print("slices api ok")
""")


@pytest.mark.skipif(not MOD, reason="python module not built")
def test_yask_kernel_slices_match_reference_loop():
    env = dict(os.environ, PYTHONPATH=os.path.dirname(MOD[0]))
    r = subprocess.run([sys.executable, "-c", SCRIPT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "slices api ok" in r.stdout
