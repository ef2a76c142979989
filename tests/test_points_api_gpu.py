"""Point sources and receivers through the reference-style APIs users already have: the `yask_kernel` Python module and the
C++ functions it binds (yask_b200/include/yask_b200_points.hpp).  One shot runs in one run_solution() call and must equal,
bit for bit, the reference API loop run_solution(t) / add_to_element / get_element of the same module."""
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
    src = [[20, 18, 32], [0, 0, 0], [20, 18, 32], [39, 35, 63]]
    rcv = [[21, 18, 32], [20, 18, 32], [0, 1, 0], [30, 30, 30]]
    amp = np.random.default_rng(2).uniform(-1, 1, size=(steps - 1, len(src))).tolist()
    amp[0][0] = 1.0 / 3.0
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
        p.set_element(0.25, [0, 5, 5, 5])
        return s

    a = solution()
    yk.yk_set_sources(a, "p", src, 1, amp)
    yk.yk_set_receivers(a, "p", rcv, 1, steps)
    a.run_solution(0, steps - 1)
    traces, owned = yk.yk_get_traces(a)
    assert all(owned) and yk.yk_get_point_launches(a) == steps, yk.yk_get_point_launches(a)
    got = [a.get_var("p").get_element([steps] + q) for q in rcv + src]

    b = solution()
    p = b.get_var("p")
    ref = []
    for t in range(steps):
        b.run_solution(t)
        if t < steps - 1:
            for i, q in enumerate(src):
                p.add_to_element(amp[t][i], [t + 1] + q)
        ref.append([p.get_element([t + 1] + q) for q in rcv])
    want = [p.get_element([steps] + q) for q in rcv + src]
    bits = lambda rows: [struct.pack("<f", x) for r in rows for x in r]
    assert bits(traces) == bits(ref), (traces, ref)
    assert bits([got]) == bits([want]), (got, want)
    try:
        yk.yk_set_sources(a, "p", [[1, 2]], 0, [[1.0]])
        raise SystemExit("a 2-index point was accepted")
    except RuntimeError as e:
        assert "3 domain dims" in str(e), e
    yk.yk_clear_points(a)
    print("points api ok")
""")


@pytest.mark.skipif(not MOD, reason="python module not built")
def test_yask_kernel_points_match_reference_loop():
    env = dict(os.environ, PYTHONPATH=os.path.dirname(MOD[0]))
    r = subprocess.run([sys.executable, "-c", SCRIPT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "points api ok" in r.stdout
