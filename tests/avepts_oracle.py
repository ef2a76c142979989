"""CPU oracle of the four average-of-points stencils (3axis, 3axis_with_diags, 3plane, cube) at any radius, fp32 or fp64 (test
infrastructure only).

The reference defines them in /root/reference/src/stencils/SimpleStencils.cpp: AvePtsStencil::define (lines 61-75) starts from
the centre point, adds the points of the shape (AxisStencil::add_points 83-103, DiagStencil 122-151, PlaneStencil 170-213,
CubeStencil 232-255) and multiplies the sum by 1.0 / pts.  Its compiler front-end flattens the chain of `v += a + b + ...` into
ONE left-to-right sum in the order the points are written (oracle/gen/s3axis.gen.h shows it at radius 4), so a step here is a
chain of elementwise numpy additions in the element type, each rounded once, then one rounded multiply by the constant.  No
product feeds an addition, so every contraction mode gives these bits.

The constant takes the 16-significant-digit print/parse round trip of every constant in the reference's generated source
(/root/reference/src/compiler/lib/Cpp.cpp:39-53), then is rounded to the element type.
"""
import numpy as np

SHAPES = ("3axis", "3axis_with_diags", "3plane", "cube")
# The radius each shape is generated at (the reference's defaults, SimpleStencils.cpp:106, 154, 216, 258).
DEFAULT_RADIUS = {"3axis": 4, "3axis_with_diags": 4, "3plane": 3, "cube": 2}
# Largest L1 distance of a read: which neighbour ranks a halo exchange reaches (faces, edges, corners).
L1_NORM = {"3axis": 1, "3axis_with_diags": 2, "3plane": 2, "cube": 3}


def points(shape, R):
    """(dx, dy, dz) of every point read, in the order the reference adds them; the centre first."""
    level = SHAPES.index(shape)
    pts = [(0, 0, 0)]
    for r in range(1, R + 1):
        pts += [(-r, 0, 0), (r, 0, 0), (0, -r, 0), (0, r, 0), (0, 0, -r), (0, 0, r)]
    if level >= 1:
        for r in range(1, R + 1):
            pts += [(-r, -r, 0), (r, -r, 0), (-r, r, 0), (r, r, 0),
                    (-r, 0, -r), (r, 0, r), (-r, 0, r), (r, 0, -r),
                    (0, -r, -r), (0, r, r), (0, -r, r), (0, r, -r)]
    if level >= 2:
        for r in range(1, R + 1):
            for m in range(r + 1, R + 1):
                pts += [(-r, -m, 0), (-m, -r, 0), (r, m, 0), (m, r, 0), (-r, m, 0), (-m, r, 0), (r, -m, 0), (m, -r, 0),
                        (-r, 0, -m), (-m, 0, -r), (r, 0, m), (m, 0, r), (-r, 0, m), (-m, 0, r), (r, 0, -m), (m, 0, -r),
                        (0, -r, -m), (0, -m, -r), (0, r, m), (0, m, r), (0, -r, m), (0, -m, r), (0, r, -m), (0, m, -r)]
    if level >= 3:
        for rx in range(1, R + 1):
            for ry in range(1, R + 1):
                for rz in range(1, R + 1):
                    pts += [(rx, ry, rz), (rx, -ry, -rz), (rx, ry, -rz), (rx, -ry, rz),
                            (-rx, ry, rz), (-rx, -ry, -rz), (-rx, ry, -rz), (-rx, -ry, rz)]
    return pts


def npoints(shape, R):
    """1 + 6R (+ 12R diagonals) (+ 12R(R-1) in-plane) (+ 8R^3 octant points)."""
    level = SHAPES.index(shape)
    return 1 + 6 * R + (12 * R if level >= 1 else 0) + (12 * R * (R - 1) if level >= 2 else 0) + (8 * R ** 3 if level >= 3 else 0)


def scale(shape, R, dtype):
    """1 / pts as the reference's generated code holds it: printed with 16 significant digits, parsed, rounded to dtype."""
    return np.dtype(dtype).type(float("%.15e" % (1.0 / npoints(shape, R))))


def step(a, shape, R):
    """One step over the interior of `a` (domain + halo R in every dim): returns the domain's new values."""
    nx, ny, nz = (s - 2 * R for s in a.shape)

    def sh(dx, dy, dz):
        return a[R + dx:R + dx + nx, R + dy:R + dy + ny, R + dz:R + dz + nz]

    acc = None
    for d in points(shape, R):
        acc = sh(*d).copy() if acc is None else acc + sh(*d)
    return acc * scale(shape, R, a.dtype)


def run(a0, a1, shape, R, steps):
    """a0 / a1: API steps 0 and 1 of A over (n + 2R) in every dim (a1 supplies the halo cells of the odd steps' slot).  Returns
    A at step `steps` with its halo, as the reference's two-slot storage holds it; the inputs are not modified."""
    slots = [a0.copy(), a1.copy()]
    for s in range(steps):
        new = step(slots[s % 2], shape, R)
        slots[(s + 1) % 2][R:-R, R:-R, R:-R] = new
    return slots[steps % 2]
