"""The table of tests/generated_cases.py, checked without a GPU: it covers manifest.json exactly, every row's size crosses
the tile edges of both launch forms (computed from the generated sources, not restated by hand), the direct-kernel knob
rows really chunk y at gen_l2_mb = 1, and the oracle runs every row in both contraction modes within a time budget."""
import time

import numpy as np
import pytest

from oracle import oracle as O
from tests import generated_cases as G
from tests.test_generated_gpu import synth_inputs

ROW_IDS = [r.name for r in G.ROWS]


def test_table_covers_the_manifest_exactly():
    """Every generated solution has exactly one row, so a solution added later cannot ship without GPU coverage."""
    names = [r.name for r in G.ROWS]
    assert len(names) == len(set(names)), "duplicate rows"
    assert set(names) == set(G.manifest()), (sorted(set(G.manifest()) - set(names)), sorted(set(names) - set(G.manifest())))
    for r in G.ROWS:
        m = G.manifest()[r.name]
        assert (r.stencil, r.radius, r.elem_bytes) == (m["stencil"], m["radius"], m["elem_bytes"]), r.name


def test_sweep_tiles_are_parsed():
    """16 solutions have sweep kernels today, with tile shapes 8x128, 8x64, 4x128 and 4x64."""
    tiles = {r.name: G.sweep_tiles(r.name) for r in G.ROWS}
    with_sweep = [n for n, t in tiles.items() if t]
    assert len(with_sweep) >= 16, with_sweep
    assert {(ty, tz) for t in tiles.values() for ty, tz, _ in t.values()} >= {(8, 128), (8, 64), (4, 128), (4, 64)}
    for n in with_sweep:
        parts = {p["name"] for st in G.ir_of(n)["stages"] for p in st["parts"]}
        assert set(tiles[n]) <= parts, n
    # rows with sweep kernels carry a chunk length; the others do not pretend to
    assert {r.name for r in G.ROWS if r.lx} == set(with_sweep)


@pytest.mark.parametrize("name", ROW_IDS)
def test_row_crosses_the_tile_edges(name):
    r = G.BY_NAME[name]
    ir = G.ir_of(name)
    assert len(r.n) == len(ir["domain_dims"]) and 2 <= r.steps <= 4
    bz, _, _ = G.direct_block()
    rpb = G.rows_per_block(r.elem_bytes)
    # direct kernels: a CTA is GEN_BZ points of the unit-stride dim x (GEN_BY * gen_np) rows x 1 plane
    nz = r.n[-1]
    assert nz > bz and nz % bz != 0, f"{name}: unit-stride extent {nz} vs {bz}-point blocks"
    if len(r.n) > 1:
        ny = r.n[-2]
        assert ny % rpb != 0, f"{name}: y extent {ny} is a whole number of {rpb}-row blocks"
    if len(r.n) == 3:
        assert 2e5 <= np.prod(r.n) <= 5e5, f"{name}: {np.prod(r.n)} points"
    # sweep kernels: partial tiles in y and z, a partial vector in the last z tile, three or more x chunks with a short last
    vec = 16 // r.elem_bytes
    for part, (ty, tz, vw) in G.sweep_tiles(name).items():
        nx, ny, nz = r.n
        assert ny >= 2 * ty + 1 and ny % ty != 0, f"{name}/{part}: y {ny} vs {ty}-row tiles"
        assert nz >= tz + 32 and nz % tz != 0, f"{name}/{part}: z {nz} vs {tz}-point tiles"
        assert (nz % tz) % vec != 0 and (vw == 1 or (nz % tz) % vw != 0), f"{name}/{part}: z remainder {nz % tz} is whole vectors"
        assert nx >= 12, f"{name}: x {nx} below the sweep kernels' minimum"
        c, last = G.chunks(nx, r.lx)
        assert c >= 3 and last < r.lx, f"{name}: x {nx} at gen_sweep_lx {r.lx}: {c} chunks, last {last}"
        hx = G.x_halo(ir)
        assert hx <= 1 or last < hx, f"{name}: last chunk {last} is not shorter than the x halo {hx}"
    # *_abc rows: the interior and the boundary parts both get points
    if name.endswith("_abc") and name.startswith("fsg"):
        assert min(r.n) > 40, f"{name}: {r.n} leaves no interior 20 points from each boundary"


@pytest.mark.parametrize("name", [r.name for r in G.grid_rows()])
def test_rank_grid_splits_unevenly(name):
    r = G.BY_NAME[name]
    assert len(r.grid) == len(r.n) and np.prod(r.grid) > 1
    assert G.uneven_split(r.n, r.grid), f"{name}: grid {r.grid} divides {r.n} evenly"
    hx = max(max(v["halo"].get(d, [0, 0])) for v in G.ir_of(name)["vars"] for d in G.ir_of(name)["domain_dims"])
    assert min(x // g for x, g in zip(r.n, r.grid)) > hx, f"{name}: a rank is thinner than the halo"


def test_grid_rows_cover_what_the_older_rank_grid_test_leaves():
    names = {r.name for r in G.grid_rows()}
    want = {r.name for r in G.ROWS if len(r.n) > 1 and r.name not in G.GRID_COVERED} | set(G.GRID_1D)
    assert names == want and len(names) >= 27


@pytest.mark.parametrize("name", [n for n in G.KNOB_ROWS if len(G.BY_NAME[n].n) == 3])
def test_l2_chunking_size_really_chunks(name):
    """At gen_l2_mb = 1 the direct kernels of these rows run in y chunks, the last one shorter: the y-chunked CTA order of
    gen_block_coords (yb_gen.cuh:140-152) with its `min(ychunk, nyb - y0)` branch.  G.direct_ychunks restates
    yb_gen.cu:388-406; if the engine's formula changes, this names the row that no longer chunks."""
    r = G.BY_NAME[name]
    ch = G.direct_ychunks(name, r.n, 1)
    assert ch
    for part, (nyb, ychunk) in ch.items():
        assert -(-nyb // ychunk) >= 2, f"{name}/{part}: nyb {nyb}, ychunk {ychunk}: one chunk"
        assert nyb % ychunk != 0, f"{name}/{part}: nyb {nyb} is a whole number of {ychunk}-block chunks"
    # gen_l2_mb = 0 turns the chunking off: one chunk of every y block
    assert all(nyb == yc for nyb, yc in G.direct_ychunks(name, r.n, 0).values())


def test_direct_ychunks_matches_the_engine_at_512():
    """DESIGN's worked example: ssg fp64 at 512^3 chunks y at the default 16 MB budget."""
    ch = G.direct_ychunks("ssg", (512, 512, 512), 16)
    assert all(yc < nyb for nyb, yc in ch.values()), ch


ORACLE_BUDGET_S = 10.0      # per row, both contraction modes (this file's GPU twin runs each row's oracle twice)


@pytest.mark.parametrize("name", ROW_IDS)
def test_oracle_runs_each_row_in_budget(name):
    r = G.BY_NAME[name]
    ins, ir = synth_inputs(name, r.n, 3)
    t0 = time.perf_counter()
    outs = [O.gen_run(name, r.n, r.steps, ins, contract=c) for c in (0, 1)]
    dt = time.perf_counter() - t0
    assert dt < ORACLE_BUDGET_S, f"{name}: {dt:.2f} s"
    written = {v["name"] for v in ir["vars"] if v["is_output"]}
    assert set(outs[0]) >= written and set(outs[1]) == set(outs[0])
    for name_, (tl, a) in outs[0].items():
        assert np.isfinite(a).all(), name_
