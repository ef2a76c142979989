"""CPU: the minimum rank size of a rank grid (yask_b200/csrc/yb_core.cu, check_min_rank_size).

Every rank of a split dim must be at least as wide as the widest halo, in that dim, of the solution's vars; a thinner rank could
not send its neighbours the planes their halos read.  plan_geometry() (and prepare_solution(), before any device work) refuses
such a grid with the reference's message (/root/reference/src/kernel/lib/setup.cpp:764-772), on EVERY rank of the grid -- also
the ranks that are wide enough themselves -- so that no rank is prepared alongside a refused neighbour.  Checked here:
  * a smallest rank of (max halo - 1) is refused on every rank, in 2- and 3-rank splits of each domain dim;
  * exactly the max halo is accepted, evenly and unevenly split;
  * an unsplit dim thinner than the halo is accepted;
  * the rank grids the rest of the suite runs still plan on every rank.
Solutions: iso3dfd at radius 1-8 in both precisions, the average-of-points shapes, iso3dfd_sponge, and generated solutions with
uneven halos (awp_elastic), misc dims (ssg2), two domain dims (wave2d) and one (test_1d).
"""
import math
import re

import pytest

from tests import generated_cases as G
from yask_b200 import capi, multi

# (stencil, radius, elem_bytes); radius 0 = the generated solution's own
SOLUTIONS = [("iso3dfd", r, eb) for r in range(1, 9) for eb in (4, 8)] + \
            [(s, r, eb) for s in ("3axis", "3axis_with_diags", "3plane", "cube") for r, eb in ((1, 4), (5, 4), (8, 8), (0, 4))] + \
            [("iso3dfd_sponge", 8, 4), ("iso3dfd_sponge", 3, 8),
             ("awp_elastic", 0, 4), ("ssg2", 0, 4), ("wave2d", 0, 4), ("test_1d", 0, 4)]
IDS = [f"{s}-r{r}-fp{8 * eb}" for s, r, eb in SOLUTIONS]


def _solution(stencil, radius, eb, n, grid, rank):
    s = capi.Solution(stencil, radius=radius, elem_bytes=eb)
    s.set_overall_domain_size_vec(n)
    s.set_num_ranks_vec(grid)
    s.set_rank_index_vec(rank)
    return s


def max_halos(stencil, radius, eb):
    """{domain dim name: widest halo of any var in it}, read from one rank's plan."""
    s = capi.Solution(stencil, radius=radius, elem_bytes=eb)
    try:
        names = s.get_domain_dim_names()
        s.set_overall_domain_size_vec([64] * len(names))
        s.plan_geometry()
        h = dict.fromkeys(names, 0)
        for v in s.get_vars():
            vi = v.info
            for i in range(vi.num_dims):
                d = vi.dims[i]
                if d.kind == 1:
                    name = d.name.decode()
                    h[name] = max(h[name], d.left_halo, d.right_halo)
        return names, h
    finally:
        s.close()


def plan_all(stencil, radius, eb, n, grid):
    """Plans every rank of the grid; returns the error message of each (None where it plans)."""
    out = []
    for r in range(math.prod(grid)):
        s = _solution(stencil, radius, eb, n, grid, multi.grid_coords(r, grid))
        try:
            s.plan_geometry()
            out.append(None)
        except capi.YaskError as e:
            out.append(str(e))
        finally:
            s.close()
    return out


def _sizes(names, h, d, nranks, smallest):
    """Overall size with `nranks` ranks in dim d whose last rank gets `smallest` points and the others one more (or exactly
    `smallest` each when even); every other dim is wide."""
    n = [2 * h[x] + 24 for x in names]
    n[d] = nranks * smallest + nranks - 1
    return n


def _grid(names, d, nranks):
    g = [1] * len(names)
    g[d] = nranks
    return g


@pytest.mark.parametrize("stencil,radius,eb", SOLUTIONS, ids=IDS)
def test_rank_thinner_than_halo_is_refused_on_every_rank(stencil, radius, eb):
    names, h = max_halos(stencil, radius, eb)
    checked = 0
    for d, name in enumerate(names):
        if h[name] < 2:          # a rank of (halo - 1) points would be empty
            continue
        for nranks in (2, 3):
            n = _sizes(names, h, d, nranks, h[name] - 1)
            assert -(-n[d] // nranks) == h[name]       # the other ranks are exactly as wide as the halo
            errs = plan_all(stencil, radius, eb, n, _grid(names, d, nranks))
            want = (f"local-domain size of {h[name] - 1} in '{name}' dim is less than minimum size of {h[name]}, "
                    "which is based on stencil halos")
            assert all(e is not None and want in e for e in errs), (name, nranks, errs)
            checked += 1
    assert checked or max(h.values()) < 2


@pytest.mark.parametrize("stencil,radius,eb", SOLUTIONS, ids=IDS)
def test_rank_as_wide_as_halo_plans(stencil, radius, eb):
    names, h = max_halos(stencil, radius, eb)
    for d, name in enumerate(names):
        if h[name] < 1:
            continue
        for nranks in (2, 3):
            n = _sizes(names, h, d, nranks, h[name])         # uneven: the last rank is exactly the halo
            assert plan_all(stencil, radius, eb, n, _grid(names, d, nranks)) == [None] * nranks, (name, nranks, n)
            n[d] = nranks * h[name]                          # even
            assert plan_all(stencil, radius, eb, n, _grid(names, d, nranks)) == [None] * nranks, (name, nranks, n)


@pytest.mark.parametrize("stencil,radius,eb", SOLUTIONS, ids=IDS)
def test_unsplit_dim_thinner_than_halo_plans(stencil, radius, eb):
    names, h = max_halos(stencil, radius, eb)
    if len(names) < 2:
        pytest.skip("one domain dim: nothing left unsplit")
    for d, name in enumerate(names):
        split = (d + 1) % len(names)
        n = [2 * h[x] + 24 for x in names]
        n[d] = 1
        assert plan_all(stencil, radius, eb, n, _grid(names, split, 2)) == [None, None], (name, n)


def test_message_names_the_smallest_rank():
    """Rank sizes given per rank (all ranks alike) are checked too, and the message gives the rank size and the halo."""
    s = capi.Solution("iso3dfd", radius=8, elem_bytes=4)
    try:
        s.set_rank_domain_size_vec((7, 40, 40))
        s.set_num_ranks_vec((2, 1, 1))
        with pytest.raises(capi.YaskError, match=re.escape("local-domain size of 7 in 'x' dim is less than minimum size of 8")):
            s.plan_geometry()
        s.set_rank_domain_size_vec((8, 40, 40))
        s.plan_geometry()
    finally:
        s.close()


# ---- the rank grids the suite runs ---------------------------------------------------------------------------------------------
# (stencil, radius, elem_bytes, overall size, grid) of the rank-grid tests outside generated_cases.py, at their thinnest
SUITE_GRIDS = [
    ("iso3dfd", 0, 4, (150, 40, 64), (4, 1, 1)), ("iso3dfd", 0, 4, (64, 64, 128), (2, 2, 2)),
    ("iso3dfd", 0, 4, (37, 29, 23), (3, 1, 2)), ("iso3dfd", 0, 4, (37, 29, 23), (2, 2, 2)),
    ("iso3dfd", 2, 4, (22, 34, 70), (2, 2, 2)), ("iso3dfd", 2, 4, (64, 6, 96), (1, 2, 1)),
    ("awp_elastic", 0, 4, (24, 24, 48), (2, 2, 2)), ("ssg", 0, 8, (41, 16, 32), (3, 1, 1)),
    ("awp_abc", 0, 4, (24, 20, 36), (1, 2, 3)), ("tti", 0, 4, (36, 36, 48), (2, 2, 2)),
    ("cube", 0, 4, (32, 32, 64), (2, 2, 2)), ("test_scratch_boundary_1d", 0, 4, (256,), (4,)),
    ("swe2d", 0, 4, (48, 64), (2, 2)), ("iso3dfd_sponge", 3, 4, (47, 20, 100), (3, 1, 1)),
    ("iso3dfd_sponge", 7, 8, (30, 20, 160), (1, 1, 2)),
] + [("iso3dfd", r, eb, (2 * (2 * r - 1), 20, 72), (2, 1, 1)) for r in range(1, 9) for eb in (4, 8)] + \
    [("iso3dfd", r, 4, (2 * (2 * r + 3), 24, 70), (2, 2, 2)) for r in (1, 3, 8)] + \
    [(s, r, eb, (32, 40, 96), g) for s in ("cube", "3axis_with_diags") for r, eb in ((3, 4), (2, 8))
     for g in ((2, 1, 1), (1, 2, 1), (1, 1, 2), (2, 2, 2))]


@pytest.mark.parametrize("stencil,radius,eb,n,grid", SUITE_GRIDS)
def test_suite_rank_grids_still_plan(stencil, radius, eb, n, grid):
    assert plan_all(stencil, radius, eb, n, grid) == [None] * math.prod(grid)


@pytest.mark.parametrize("name", [r.name for r in G.ROWS if r.grid])
def test_generated_case_grids_still_plan(name):
    r = G.BY_NAME[name]
    assert plan_all(r.stencil, r.radius, r.elem_bytes, r.n, r.grid) == [None] * math.prod(r.grid)
