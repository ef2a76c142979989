"""CPU oracle of iso3dfd_sponge at any radius, fp32 or fp64 (test infrastructure only).

A sponge step is the iso3dfd step of the pinned C oracle (oracle/yask_oracle.c, through oracle.iso3dfd_run) followed by the
reference's last statement, next_p *= cr_x(x) * cr_y(y) * cr_z(z) (/root/reference/src/stencils/Iso3dfdStencil.cpp:212-249),
evaluated as the generated code does: ((p * cr_x) * cr_y) * cr_z, three rounded multiplies in the element type.  numpy rounds
each elementwise product exactly once, and no addition follows, so the same holds in every contraction mode.
"""
import numpy as np

from oracle import oracle as O


def iso3dfd_sponge_run(p0, p1, v, crx, cry, crz, R, steps, mode):
    """p0 / p1: API steps 0 and 1 of p over (nx+2h, ny+2h, nz+2h), halo h >= R; v: (nx, ny, nz); crx / cry / crz: (nx,), (ny,),
    (nz,).  mode: the oracle's contraction mode (0 strict, 1 canonical FMA, 2 the reference's default build).  Returns the final p
    (domain + untouched halo) after `steps` steps; the inputs are not modified."""
    nx, ny, nz = v.shape
    h = (p0.shape[0] - nx) // 2
    dt = p0.dtype
    crx, cry, crz = (np.asarray(c, dtype=dt) for c in (crx, cry, crz))
    assert crx.shape == (nx,) and cry.shape == (ny,) and crz.shape == (nz,)
    cur, prev = p0, p1
    for _ in range(steps):
        nxt = O.iso3dfd_run(cur, prev, v, R, 1, mode)      # p(t+1) over p(t-1)'s storage (and its halo cells)
        d = nxt[h:h + nx, h:h + ny, h:h + nz]
        d[...] = ((d * crx[:, None, None]) * cry[None, :, None]) * crz[None, None, :]
        cur, prev = nxt, cur
    return cur
