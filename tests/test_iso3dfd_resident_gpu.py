"""GPU: the resident-plane form of the radius-8 fp32 iso3dfd sweep (option `resident`, iso3dfd_tma3_kernel in
yask_b200/csrc/yb_iso3dfd.cuh), at both of its tile shapes (tile 6: 32x64, tile 7: 16x128), bit for bit against the CPU oracle:
every FP mode on ragged domains and on chunks shorter than the radius, persistent CTAs that sweep several units, rank grids with
the fused x exchange and with the split path, halo cells, the generation-2 sweep at 512^3 and the offline tuner.
"""
import numpy as np
import pytest

from tests.test_iso3dfd_sweep_gpu import R8_TILES, _bits, check_grid, inputs, oracle, run_one, units
from yask_b200 import capi
from yask_b200.synth import var_salt

pytestmark = pytest.mark.gpu

R = 8
TILES = (6, 7)


def resident(tile):
    return {"kernel": "tma", "tile": tile, "resident": 1}


def test_option_reported():
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec((32, 32, 64))
    s.prepare_solution(0)
    for tile, res, want in [(7, 1, "1"), (6, 1, "1"), (7, 0, "0"), (5, 1, "0")]:
        s.set_option("tile", tile)
        s.set_option("resident", res)
        assert s.get_option("resident") == want, (tile, res)
    s.close()
    for r, eb in [(4, 4), (4, 8)]:           # no resident form: accepted, ignored, reported as 0
        s = capi.Solution("iso3dfd", radius=r, elem_bytes=eb)
        s.set_option("resident", 1)
        s.set_overall_domain_size_vec((32, 32, 64))
        s.prepare_solution(0)
        assert s.get_option("resident") == "0"
        s.close()


@pytest.mark.parametrize("lx", [0, 4, 7])           # 4, 7: chunks shorter than R
@pytest.mark.parametrize("n", [(9, 8, 16), (17, 33, 65), (40, 37, 150)])
@pytest.mark.parametrize("fp_mode", [0, 1, 2])
@pytest.mark.parametrize("tile", TILES)
def test_bit_exact_vs_oracle(tile, fp_mode, n, lx):
    got = run_one(n, R, 3, np.float32, fp_mode, resident(tile) | {"lx": lx})
    assert np.array_equal(_bits(got), _bits(oracle(n, R, 3, fp_mode, np.float32)))


@pytest.mark.parametrize("grid,lx", [(1, 5), (2, 7), (3, 5), (7, 3)])
@pytest.mark.parametrize("tile", TILES)
def test_persistent_ctas(tile, grid, lx):
    n = (23, 37, 200)
    assert units(n, R8_TILES[tile], lx) > grid
    got = run_one(n, R, 3, np.float32, 2, resident(tile) | {"lx": lx, "grid": grid})
    assert np.array_equal(_bits(got), _bits(oracle(n, R, 3, 2, np.float32)))


@pytest.mark.parametrize("tile", TILES)
def test_more_units_than_sms(tile):
    import torch
    n = (80, 70, 200)
    assert units(n, R8_TILES[tile], 2) > torch.cuda.get_device_properties(0).multi_processor_count
    got = run_one(n, R, 3, np.float32, 2, resident(tile) | {"lx": 2})
    assert np.array_equal(_bits(got), _bits(oracle(n, R, 3, 2, np.float32)))


@pytest.mark.parametrize("nx_rank", [4 * R + 1, 2 * R])        # peer stores + in-kernel signal; peer stores only
@pytest.mark.parametrize("ranks", [2, 3])
@pytest.mark.parametrize("tile", TILES)
def test_rank_grid_fused_x_exchange(tile, ranks, nx_rank):
    check_grid((ranks * nx_rank, 20, 72), (ranks, 1, 1), R, 3, np.float32, opts={"tile": tile, "resident": 1})


@pytest.mark.parametrize("tile", TILES)
def test_rank_grid_split_path(tile):
    check_grid((13, 20, 70), (1, 1, 2), R, 3, np.float32, opts={"tile": tile, "resident": 1})


@pytest.mark.parametrize("tile", TILES)
def test_halo_cells_untouched(tile):
    n = (20, 19, 70)
    ins = inputs(n, R, np.float32)
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec(n)
    for k, v in resident(tile).items():
        s.set_option(k, v)
    s.prepare_solution(0)
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.set_elements_in_slice(ins[("p", t)], *p.halo_box(t))
    v.set_elements_in_slice(ins[("v", 0)], *v.halo_box(0))
    s.run_solution(0, 2)
    for t in range(p.get_first_valid_step_index(), p.get_last_valid_step_index() + 1):
        full = p.get_elements_in_slice(*p.halo_box(t))
        src = ins[("p", t % 2)]
        inner = np.ones(full.shape, bool)
        inner[R:-R, R:-R, R:-R] = False
        assert np.array_equal(_bits(full[inner]), _bits(src[inner])), t
    s.close()


def _checksum_512(opts):
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec((512, 512, 512))
    for k, v in opts.items():
        s.set_option(k, v)
    s.prepare_solution(0)
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.fill_hash(t, 5, var_salt("p", t), -1.0, 1.0)
    v.fill_hash(0, 5, var_salt("v", 0), 0.05, 0.3)
    s.run_solution(0, 3)
    c = p.checksum(p.get_last_valid_step_index())
    s.close()
    return c


@pytest.mark.parametrize("tile", TILES)
def test_same_bits_as_generation_2_at_512(tile):
    assert _checksum_512(resident(tile)) == _checksum_512({"kernel": "tma", "tile": tile, "resident": 0})


def test_offline_tuner_keeps_bits():
    n, steps = (64, 48, 160), 2
    s = capi.Solution("iso3dfd")
    s.set_overall_domain_size_vec(n)
    s.prepare_solution(0)
    rep = s.run_auto_tuner_now()
    assert rep.count("resident=1") >= 2 and "best: tile=" in rep and " resident=" in rep.split("best:")[1], rep
    assert s.get_option("resident") in ("0", "1")
    ins = inputs(n, R, np.float32)
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.set_elements_in_slice(ins[("p", t)], *p.halo_box(t))
    v.set_elements_in_slice(ins[("v", 0)], *v.halo_box(0))
    s.run_solution(0, steps - 1)
    got = p.get_elements_in_slice(*p.domain_box(p.get_last_valid_step_index()))
    s.close()
    assert np.array_equal(_bits(got), _bits(oracle(n, R, steps, 2, np.float32)))
