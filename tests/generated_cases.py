"""One row per emitter-generated solution (yask_b200/csrc/gen/manifest.json) for the matrix tests
(tests/test_generated_matrix_cpu.py checks the rows, tests/test_generated_matrix_gpu.py runs them).

A row says how to construct the solution, a ragged size that crosses the tile edges of both launch forms, a step count,
a sweep chunk length (option gen_sweep_lx) that leaves a short last chunk, and a rank grid that splits a dim unevenly.
The launch geometry the rows are checked against is read back from the sources: the sweep tiles from the generated
kernels' comments, the direct kernels' CTA shape from yb_gen.cuh."""
import json
import math
import os
import re
from dataclasses import dataclass

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "yask_b200", "csrc")
GEN = os.path.join(CSRC, "gen")


@dataclass(frozen=True)
class Row:
    name: str              # key in manifest.json (and csrc/gen/<name>.json, the oracle's IR)
    stencil: str           # capi.Solution(stencil, radius=radius, elem_bytes=elem_bytes) selects the generated kernels
    radius: int
    elem_bytes: int
    n: tuple               # overall domain size, in the solution's domain-dim order
    steps: int
    lx: int = 0            # gen_sweep_lx of the sweep tests (rows with sweep kernels only)
    grid: tuple = ()       # rank grid of the rank-grid test

    def solution(self):
        from yask_b200 import capi
        return capi.Solution(self.stencil, radius=self.radius, elem_bytes=self.elem_bytes)


# fp32 3-D rows with sweep kernels: 8 (or 4) rows x 128 z tiles -> y 27 (3 tiles + 3 rows, 4-row direct blocks + 3),
# z 163 (1 tile + 35 = 8 vectors + 3 points); x = 3 chunks + a last chunk shorter than the x halo.
# fp64 rows: 8 (or 4) rows x 64 z tiles, 2-row direct blocks -> y odd, z 141 or 205 (2 or 3 tiles + an odd remainder).
# *_abc rows: every dim above 40, so that the interior (20 points from each boundary) and the boundary parts both run.
ROWS = [
    Row("3axis", "3axis", 0, 4, (48, 27, 163), 3, lx=15, grid=(1, 2, 1)),
    Row("3axis_with_diags", "3axis_with_diags", 0, 4, (49, 27, 163), 2, lx=16, grid=(1, 2, 1)),
    Row("3plane", "3plane", 0, 4, (50, 27, 163), 2, lx=16, grid=(3, 1, 1)),
    Row("awp", "awp", 0, 4, (49, 27, 163), 2, lx=16, grid=(3, 1, 1)),
    Row("awp_abc", "awp_abc", 0, 4, (45, 43, 141), 2, grid=(3, 1, 1)),
    Row("awp_elastic", "awp_elastic", 0, 4, (49, 27, 163), 3, lx=16, grid=(3, 1, 1)),
    Row("awp_elastic_abc", "awp_elastic_abc", 0, 4, (43, 45, 139), 2, grid=(1, 3, 1)),
    Row("box_filter", "box_filter", 0, 4, (203, 389), 2, grid=(3, 1)),
    Row("cube", "cube", 0, 4, (49, 27, 163), 2, lx=12, grid=(3, 1, 1)),
    Row("fsg", "fsg", 0, 4, (43, 35, 141), 2, grid=(3, 1, 1)),
    Row("fsg2", "fsg2", 0, 4, (41, 39, 131), 2, grid=(3, 1, 1)),
    Row("fsg2_abc", "fsg2_abc", 0, 4, (47, 45, 139), 2, grid=(3, 1, 1)),
    Row("fsg_abc", "fsg_abc", 0, 4, (45, 51, 150), 2, grid=(2, 1, 1)),
    Row("fsg_merged", "fsg_merged", 0, 4, (41, 35, 145), 2, grid=(3, 1, 1)),
    Row("fsg_merged_abc", "fsg_merged_abc", 0, 4, (44, 43, 137), 2, grid=(1, 3, 1)),
    Row("gaussian_filter", "gaussian_filter", 0, 4, (101, 263), 3, grid=(3, 1)),
    Row("iso3dfd_fp64", "iso3dfd", 0, 8, (79, 21, 141), 2, lx=24, grid=(3, 1, 1)),
    Row("iso3dfd_fp64_r3", "iso3dfd", 3, 8, (74, 41, 141), 3, lx=24, grid=(3, 1, 1)),
    Row("iso3dfd_sponge", "iso3dfd_sponge", 0, 4, (65, 27, 163), 2, lx=20, grid=(3, 1, 1)),
    Row("iso3dfd_sponge_fp64_r6", "iso3dfd_sponge", 6, 8, (65, 23, 141), 2, lx=20, grid=(3, 1, 1)),
    Row("ssg", "ssg", 0, 8, (51, 21, 205), 2, lx=16, grid=(3, 1, 1)),
    Row("ssg2", "ssg2", 0, 4, (40, 39, 133), 2, grid=(3, 1, 1)),
    Row("ssg_merged", "ssg_merged", 0, 4, (43, 51, 141), 2, grid=(3, 1, 1)),
    Row("swe2d", "swe2d", 0, 4, (67, 301), 2, grid=(3, 1)),
    Row("test_1d", "test_1d", 0, 4, (1237,), 3, grid=(3,)),
    Row("test_2d", "test_2d", 0, 4, (101, 263), 3, grid=(3, 1)),
    Row("test_3d", "test_3d", 0, 4, (51, 27, 163), 3, lx=16, grid=(2, 1, 1)),
    Row("test_boundary_1d", "test_boundary_1d", 0, 4, (1001,), 3, grid=(3,)),
    Row("test_boundary_2d", "test_boundary_2d", 0, 4, (67, 301), 3, grid=(1, 3)),
    Row("test_boundary_3d", "test_boundary_3d", 0, 4, (41, 43, 133), 3, grid=(3, 1, 1)),
    Row("test_func_1d", "test_func_1d", 0, 4, (1103,), 3, grid=(3,)),
    Row("test_partial_3d", "test_partial_3d", 0, 4, (51, 27, 163), 2, lx=16, grid=(1, 2, 1)),
    Row("test_reverse_2d", "test_reverse_2d", 0, 4, (103, 263), 3, grid=(3, 1)),
    Row("test_scratch_1d", "test_scratch_1d", 0, 4, (1237,), 3, grid=(3,)),
    Row("test_scratch_2d", "test_scratch_2d", 0, 4, (101, 263), 3, grid=(3, 1)),
    Row("test_scratch_3d", "test_scratch_3d", 0, 4, (41, 39, 135), 3, grid=(3, 1, 1)),
    Row("test_scratch_boundary_1d", "test_scratch_boundary_1d", 0, 4, (1237,), 3, grid=(3,)),
    Row("test_scratch_stages_1d", "test_scratch_stages_1d", 0, 4, (1001,), 3, grid=(3,)),
    Row("test_stages_1d", "test_stages_1d", 0, 4, (1103,), 3, grid=(3,)),
    Row("test_stages_2d", "test_stages_2d", 0, 4, (101, 263), 3, grid=(3, 1)),
    Row("test_stages_3d", "test_stages_3d", 0, 4, (49, 27, 163), 3, lx=16, grid=(3, 1, 1)),
    Row("test_step_cond_1d", "test_step_cond_1d", 0, 4, (1001,), 4, grid=(3,)),
    Row("test_stream_1d", "test_stream_1d", 0, 4, (1237,), 3, grid=(3,)),
    Row("test_stream_2d", "test_stream_2d", 0, 4, (101, 263), 3, grid=(1, 3)),
    Row("test_stream_3d", "test_stream_3d", 0, 4, (49, 27, 163), 3, lx=16, grid=(3, 1, 1)),
    Row("tti", "tti", 0, 4, (49, 27, 163), 2, lx=16, grid=(3, 1, 1)),
    Row("wave2d", "wave2d", 0, 4, (101, 263), 3, grid=(3, 1)),
]
BY_NAME = {r.name: r for r in ROWS}


def manifest():
    return json.load(open(os.path.join(GEN, "manifest.json")))


def ir_of(name):
    return json.load(open(os.path.join(GEN, f"{name}.json")))


def gen_source(name):
    """csrc/gen/<name>.gen.cuh (names that start with a digit get an 's' prefix: they are C++ identifiers)."""
    return os.path.join(GEN, ("s" + name if name[0].isdigit() else name) + ".gen.cuh")


_TILE = re.compile(r"// sweep kernel of part '(\w+)' \(yb_gen_sweep\.cuh\):[^\n]*? tile (\d+) rows x (\d+) z[^\n]*\n"
                   r"[^\n]*\n[^\n]*\n[^\n]*\n[^\n]*constexpr int VW = (\d+),")


def sweep_tiles(name):
    """{part name: (TY, TZ, VW)} of the part's sweep kernel: tile rows, tile z points and z points per consumer thread,
    from the generated kernel's comment and its constants.  Empty when the solution has no sweep kernel."""
    return {m.group(1): (int(m.group(2)), int(m.group(3)), int(m.group(4))) for m in _TILE.finditer(open(gen_source(name)).read())}


def direct_block():
    """(GEN_BZ, GEN_BY, {elem_bytes: gen_np}) of the direct kernels' CTA, read from yb_gen.cuh."""
    src = open(os.path.join(CSRC, "yb_gen.cuh")).read()
    bz = int(re.search(r"#define YB_GEN_BZ (\d+)", src).group(1))
    by = int(re.search(r"#define YB_GEN_BY (\d+)", src).group(1))
    m = re.search(r"gen_np\(int elem_bytes\) \{ return elem_bytes == 4 \? (\d+) : (\d+); \}", src)
    return bz, by, {4: int(m.group(1)), 8: int(m.group(2))}


def rows_per_block(elem_bytes):
    _, by, np_ = direct_block()
    return by * np_[elem_bytes]


def n_parts(ir):
    return sum(len(st["parts"]) for st in ir["stages"])


def x_halo(ir):
    """The solution's x halo: the largest halo any var has in its first domain dim (the engine pads every var to it)."""
    d0 = ir["domain_dims"][0]
    return max(max(v["halo"].get(d0, [0, 0])) for v in ir["vars"])


# ---- the direct kernels' y chunking (yb_gen.cu:388-406), restated ----------------------------------------------------
def _pad_alloc(ir, k, n, align_elems):
    """Allocated extent of domain dim k: every var is padded to the largest halo any var has there (yb_gen.cu:446-448);
    the unit-stride dim's left pad and pitch are rounded up to 128 bytes (yb_core.cu:102-110)."""
    d = ir["domain_dims"][k]
    u = max(max(v["halo"].get(d, [0, 0])) for v in ir["vars"])
    if k != len(ir["domain_dims"]) - 1:
        return u + n[k] + u
    pl = -(-u // align_elems) * align_elems
    return -(-(pl + n[k] + u) // align_elems) * align_elems


def _launch_box(part, n):
    """Launch box of a non-scratch part over one rank holding the whole domain: the domain cut to the part's sub-domain
    bounds ([lo, hi] per kernel slot, each end relative to 0 / the first / the last index)."""
    sh = 3 - len(n)
    nn = [1] * sh + list(n)
    b, e = [0, 0, 0], nn[:]
    bounds = (part.get("cond") or {}).get("bounds") or {}
    for k, (lo, hi) in bounds.items():
        k = int(k)
        res = lambda kind, off: {"GF": 0, "GL": nn[k] - 1}.get(kind, 0) + off
        if lo:
            b[k] = max(b[k], res(*lo))
        if hi:
            e[k] = min(e[k], res(*hi) + 1)
    return b, e


def direct_ychunks(name, n, l2_mb):
    """Per non-scratch part of a 3-D solution: (nyb, ychunk) of its direct kernel at option gen_l2_mb = l2_mb, as
    GenEngine::launch (yb_gen.cu:388-406) computes them: the y chunk keeps (2 x halo + 1) x planes of every distinct
    full-rank var the part touches within the L2 budget, at least 4 y blocks, and the chunks are equalised."""
    ir = ir_of(name)
    eb = ir["elem_bytes"]
    rpb = rows_per_block(eb)
    dd = ir["domain_dims"]
    assert len(dd) == 3, "the direct kernels chunk y only in 3-D solutions (GenParams::SX is 0 otherwise)"
    align = 128 // eb
    sy = _pad_alloc(ir, 2, n, align)                          # y stride = pitch of the unit-stride z dim
    span = 2 * x_halo(ir) + 1
    vars_ = {v["name"]: v for v in ir["vars"]}
    out = {}
    for st in ir["stages"]:
        for p in st["parts"]:
            if p.get("scratch"):
                continue
            b, e = _launch_box(p, n)
            nyb = -(-(e[1] - b[1]) // rpb)
            nxb = e[0] - b[0]
            distinct = set()
            for a in p["accesses"]:
                v = vars_[a["var"]]
                vd = [d for d in v["dims"] if d != ir["step_dim"]]
                if [d for d in vd if d in dd] != dd:
                    continue                                  # not a full-rank var in the solution's dim order
                alloc = v["alloc_t"] if v["dims"] and v["dims"][0] == ir["step_dim"] else 1
                distinct.add((a["var"], a["toff"] % alloc, tuple(a.get("misc", []))))     # distinct storage
            ychunk = nyb
            if l2_mb > 0 and nxb > 1:
                rows = int(l2_mb * 1048576.0 / (sy * eb * span * max(len(distinct), 1)))
                yc = max(rows // rpb, 4)
                if yc < nyb:
                    nch = -(-nyb // yc)
                    ychunk = -(-nyb // nch)
            out[p["name"]] = (nyb, ychunk)
    return out


# ---- which rows each GPU test uses --------------------------------------------------------------------------------------
# Direct-kernel knobs: one row per tile family (fp32 8x128, fp64 4x64 and 8x64, a 2-D and a 1-D solution), fsg_abc and
# ssg_merged.  The 3-D ones are sized so that gen_l2_mb = 1 chunks y with a shorter last chunk (checked on the CPU).
KNOB_ROWS = ["awp_elastic", "ssg", "iso3dfd_fp64_r3", "test_2d", "test_1d", "fsg_abc", "ssg_merged"]
# Tuners: a 3-D fp32 row, an fp64 row and fsg_abc
TUNER_ROWS = ["awp_elastic", "iso3dfd_fp64_r3", "fsg_abc"]
# Rank grids: the solutions tests/test_generated_gpu.py::test_generated_rank_grid_matches_single_rank already runs on grids
GRID_COVERED = {"awp_elastic", "ssg", "awp", "tti", "cube", "awp_elastic_abc", "awp_abc", "ssg2", "test_2d", "test_scratch_3d",
                "test_scratch_2d", "test_scratch_boundary_1d", "test_stages_2d", "wave2d", "swe2d"}
GRID_1D = ["test_boundary_1d", "test_stream_1d", "test_stages_1d"]


def grid_rows():
    return [r for r in ROWS if r.name not in GRID_COVERED and (len(r.n) > 1 or r.name in GRID_1D)]


def uneven_split(n, grid):
    return any(g > 1 and x % g != 0 for x, g in zip(n, grid))


def chunks(nx, lx):
    """(number of sweep chunks, length of the last one) of an x extent nx at gen_sweep_lx = lx."""
    c = math.ceil(nx / lx)
    return c, nx - (c - 1) * lx
