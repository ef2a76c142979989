"""CPU: frame and image types of slice recorders, injectors and correlators -- the refusals, the rounding the Python call applies
to host frames (restated here with exact rational arithmetic), the 64-bit byte count at the frame type's size, and frames and
owned masks of typed recorders on a planned rank grid."""
import math
from fractions import Fraction

import numpy as np
import pytest

from tests.test_slices_cpu import decimated_mask, planned, refused
from yask_b200 import capi


def planned64(n=(37, 29, 23)):
    s = capi.Solution("iso3dfd", radius=4, elem_bytes=8)
    s.set_overall_domain_size_vec(n)
    s.plan_geometry()
    return s


BOX = ([1, 1, 1], [5, 5, 5])


def test_refusals_name_the_type_and_the_element_type():
    s = planned()
    refused(lambda: s.add_slice("p", *BOX, 0, 3, dtype="float64"), "slice: frame type float64", "element type float32")
    refused(lambda: s.add_slice_injector("p", *BOX, 0, np.zeros((2, 5, 5, 5)), dtype=np.float64), "slice injector: frame type float64",
            "element type float32")
    refused(lambda: s.add_slice_correlator("p", *BOX, 0, 3, image_dtype="float16"), "slice correlator: image type float16",
            "element type float32")
    refused(lambda: s.add_slice("p", *BOX, 0, 3, dtype="int8"), "slice: unknown dtype 'int8'")
    refused(lambda: s.add_slice("p", *BOX, 0, 3, dtype=np.complex64), "slice: unknown dtype")
    refused(lambda: s.add_slice_correlator("p", *BOX, 0, 3, image_dtype="bf16"), "slice correlator: unknown image_dtype 'bf16'")
    # the C ABI refuses a number outside YB_TYPE_*
    lo, hi = (capi.C.c_int64 * 3)(*BOX[0]), (capi.C.c_int64 * 3)(*BOX[1])
    assert capi.lib().yb_solution_add_slice_typed(s._h, b"p", lo, hi, None, 0, 1, 3, 9, None) != 0
    assert "slice: unknown frame type 9" in capi.lib().yb_last_error().decode()
    # nothing was left behind: the first valid recorder and correlator get id 0, in each allowed type
    assert [s.add_slice("p", *BOX, 0, 3, dtype=d) for d in ("float16", "bfloat16", np.float32, None)] == [0, 1, 2, 3]
    assert [s.add_slice_correlator("p", *BOX, 0, 3, image_dtype=d) for d in ("float64", "float32", None)] == [0, 1, 2]
    s.close()
    s = planned64()
    refused(lambda: s.add_slice("p", *BOX, 0, 3, dtype="float16"), "slice: frame type float16", "element type float64")
    refused(lambda: s.add_slice("p", *BOX, 0, 3, dtype="bfloat16"), "slice: frame type bfloat16", "element type float64")
    refused(lambda: s.add_slice_injector("p", *BOX, 0, np.zeros((2, 5, 5, 5)), dtype="float16"), "slice injector: frame type float16")
    refused(lambda: s.add_slice_correlator("p", *BOX, 0, 3, image_dtype="float32"), "slice correlator: image type float32",
            "element type float64")
    assert s.add_slice("p", *BOX, 0, 3, dtype="float32") == 0
    assert s.add_slice_correlator("p", *BOX, 0, 3, image_dtype=np.float64) == 0
    s.close()


def test_frames_and_images_come_back_in_their_types():
    """Before prepare: zeros of the frame type (bf16 as float32), and the image type, from the type queries."""
    s = planned()
    want = {"float16": np.float16, "bfloat16": np.float32, "float32": np.float32}
    for i, d in enumerate(want):
        assert s.add_slice("p", [0, 0, 0], [36, 28, 0], 0, 2, stride=[2, 2, 1], dtype=d) == i
        frames, owned = s.get_slice_frames(i)
        assert frames.dtype == want[d] and frames.shape == (2, 19, 15, 1) and owned.all() and not frames.any()
    for i, d in enumerate((None, "float64")):
        s.add_slice_correlator("p", *BOX, 0, 3, image_dtype=d)
        assert s.get_correlator_image(i)[0].dtype == (np.float32 if d is None else np.float64)
    s.close()


def test_byte_count_uses_the_frame_size():
    """nrows x box x sizeof(F) must fit a 64-bit count: a one-point box with 3 * 2^60 rows overflows at 4 bytes, not at 2."""
    s = planned()
    nrows = 3 << 60
    refused(lambda: s.add_slice("p", [0, 0, 0], [0, 0, 0], 0, nrows), "of 4-byte elements overflow a 64-bit byte count")
    refused(lambda: s.add_slice("p", [0, 0, 0], [0, 0, 0], 0, nrows, dtype="float32"), "overflow")
    assert s.add_slice("p", [0, 0, 0], [0, 0, 0], 0, nrows, dtype="bfloat16") == 0
    assert s.add_slice("p", [0, 0, 0], [0, 0, 0], 0, nrows, dtype="float16") == 1
    refused(lambda: s.add_slice("p", [0, 0, 0], [0, 0, 0], 0, 3 << 61, dtype="float16"), "of 2-byte elements overflow")
    s.close()
    s = planned64()
    refused(lambda: s.add_slice("p", [0, 0, 0], [0, 0, 0], 0, 3 << 59), "of 8-byte elements overflow")
    assert s.add_slice("p", [0, 0, 0], [0, 0, 0], 0, 3 << 59, dtype="float32") == 0
    s.close()


@pytest.mark.parametrize("grid", [(2, 1, 1), (2, 2, 1)])
def test_owned_mask_of_typed_recorders_on_a_rank_grid(grid):
    n = (37, 29, 23)
    first, last, stride = [1, 2, 3], [36, 27, 22], [2, 3, 4]
    world = int(np.prod(grid))
    for d in ("float16", "bfloat16"):
        total = 0
        for r in range(world):
            s = planned(n=n, grid=grid, rank=r)
            rid = s.add_slice("p", first, last, 0, 2, stride=stride, dtype=d)
            _, owned = s.get_slice_frames(rid)
            want = decimated_mask(first, last, stride, s.get_first_rank_domain_index_vec(), s.get_rank_domain_size_vec())
            assert np.array_equal(owned, want), (r, d)
            total = total + owned
            s.close()
        assert (total == 1).all()


# ---- the rounding of host frames, restated -------------------------------------------------------------------------------

def rne(x, mant, emin, largest):
    """x rounded to nearest even into a binary format of `mant` significand bits (the hidden bit included), least normal
    exponent emin and largest finite value `largest`, by exact rational arithmetic: a Python float holding the result, +-inf
    past the range, NaN for NaN."""
    if math.isnan(x) or math.isinf(x) or x == 0:
        return x
    a = abs(Fraction(x))
    e = max(math.frexp(x)[1] - 1, emin)
    ulp = Fraction(2) ** (e - (mant - 1))
    k, rem = divmod(a, ulp)
    if rem > ulp / 2 or (rem == ulp / 2 and k % 2 == 1):
        k += 1
    r = k * ulp
    return math.copysign(math.inf if r > largest else float(r), x)


F16_MAX = Fraction(65504)
BF16_MAX = (2 - Fraction(1, 2 ** 7)) * Fraction(2) ** 127


def f32_of_bits(*bits):
    return np.array(bits, np.uint32).view(np.float32)


def crafted_f32():
    p = 2.0
    vals = [1 + p ** -11, 1 + 3 * p ** -11, 1 + p ** -8, 1 + 3 * p ** -8,          # fp16 and bf16 ties, even and odd below
            65504, 65519.996, 65520, 65536, 1e5,                                    # fp16: largest finite, first overflow
            p ** -24, p ** -25, 3 * p ** -25, p ** -14 - p ** -25, p ** -14,       # fp16 subnormals and their ties
            1e-30, 3e-39, 0.0, -0.0, math.inf, -math.inf, math.nan, 1 / 3, -2 / 3, 0.1]
    a = np.array(vals + [-v for v in vals], np.float32)
    # bf16: largest finite, the tie above it and the float below; float32 subnormals on, between and at ties of the bf16 grid
    b = f32_of_bits(0x7F7F0000, 0x7F7F8000, 0x7F7F7FFF, 0x7F7FFFFF, 0x00000001, 0x00008000, 0x00018000, 0x00028000, 0x00400000,
                    0x00010001, 0x807F8000, 0x7FC00001, 0xFF800001)
    rng = np.random.default_rng(5)
    r = (rng.uniform(1, 2, 3000) * np.exp2(rng.integers(-140, 128, 3000))).astype(np.float32) * rng.choice([-1, 1], 3000)
    return np.concatenate([a, b, r.astype(np.float32)])


def test_fp16_rounding_matches_the_restatement():
    x = crafted_f32()
    got = capi.narrow_frames(x, 4, capi.TYPE_F16)
    assert got.dtype == np.float16
    for xi, gi in zip(x.tolist(), got.tolist()):
        want = rne(xi, 11, -14, F16_MAX)
        if math.isnan(want):
            assert math.isnan(gi), xi
        else:
            assert gi == want and math.copysign(1, gi) == math.copysign(1, want), (xi, gi, want)


def test_bf16_rounding_matches_the_restatement():
    x = crafted_f32()
    bits = capi.narrow_frames(x, 4, capi.TYPE_BF16)
    assert bits.dtype == np.uint16
    got = capi.bf16_widen(bits)
    for xi, gi in zip(x.tolist(), got.tolist()):
        want = rne(xi, 8, -126, BF16_MAX)
        if math.isnan(want):
            assert math.isnan(gi), xi
        else:
            assert gi == want and math.copysign(1, gi) == math.copysign(1, want), (xi, gi, want)
    # the tie at the largest finite value goes to inf (even), the float just below it stays finite
    assert capi.bf16_widen(capi.bf16_bits(f32_of_bits(0x7F7F8000, 0x7F7F7FFF))).tolist() == [math.inf, float(BF16_MAX)]


def test_host_frames_round_to_the_element_type_first():
    """Two roundings, as documented: to T, then to F.  1 + 2^-11 + 2^-40 is above the fp16 tie, but rounds to the tie 1 + 2^-11
    in fp32, which then rounds to even: 1.0.  An fp64 solution rounds once, to float32."""
    x = np.array([1 + 2.0 ** -11 + 2.0 ** -40, 1 + 2.0 ** -8 + 2.0 ** -40])
    assert capi.narrow_frames(x[:1], 4, capi.TYPE_F16).tolist() == [1.0]
    assert capi.bf16_widen(capi.narrow_frames(x[1:], 4, capi.TYPE_BF16)).tolist() == [1.0]
    assert capi.narrow_frames(x, 8, capi.TYPE_F32).tolist() == [float(np.float32(v)) for v in x]
    assert capi.narrow_frames(x, 4, capi.TYPE_ELEM).dtype == np.float32
