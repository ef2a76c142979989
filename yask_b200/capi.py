"""ctypes binding of the C ABI (include/yask_b200.h) -- the same entry points a cgo/JNI/C++
binding of the reference's yk_* API would use.  No torch types cross this boundary.

The library is never replaced by a CPU path: if libyask_b200.so is missing this module raises,
and on a machine without a CUDA device `Solution.prepare()` raises YaskError.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("YASK_B200_LIB", os.path.join(_HERE, "lib", "libyask_b200.so"))   # env override: tuning experiments only

YB_MAX_DIMS = 5
YB_NAME_LEN = 64

FP_STRICT, FP_FMA, FP_REF_GCC = 0, 1, 2


class YaskError(RuntimeError):
    """Mirror of yask::yask_exception (/root/reference/include/yask_common_api.hpp:125-179)."""

    def __init__(self, code: int, msg: str):
        super().__init__(f"YASK error: {msg} (code {code})")
        self.code = code


class DimInfo(C.Structure):
    _fields_ = [("name", C.c_char * YB_NAME_LEN), ("kind", C.c_int32), ("domain_index", C.c_int32),
                ("rank_offset", C.c_int64), ("domain_size", C.c_int64), ("left_halo", C.c_int64), ("right_halo", C.c_int64),
                ("left_pad", C.c_int64), ("right_pad", C.c_int64), ("alloc_size", C.c_int64), ("first_misc_index", C.c_int64),
                ("stride", C.c_int64)]


class VarInfo(C.Structure):
    _fields_ = [("name", C.c_char * YB_NAME_LEN), ("num_dims", C.c_int32), ("elem_bytes", C.c_int32), ("has_step", C.c_int32),
                ("step_alloc", C.c_int32), ("first_valid_step", C.c_int64), ("last_valid_step", C.c_int64),
                ("is_output", C.c_int32), ("halo_exchange_l1_norm", C.c_int32), ("slot_elems", C.c_int64),
                ("storage_bytes", C.c_int64), ("dims", DimInfo * YB_MAX_DIMS)]


class Stats(C.Structure):
    _fields_ = [("num_elements", C.c_int64), ("num_steps_done", C.c_int64), ("num_writes_done", C.c_int64),
                ("est_fp_ops_done", C.c_int64), ("num_reads_done", C.c_int64), ("elapsed_secs", C.c_double),
                ("halo_secs", C.c_double), ("kernel_launches", C.c_int64)]


# every symbol include/yask_b200.h declares (tests check the .so exports exactly these)
ABI_SYMBOLS = [
    "yb_version_string", "yb_last_error", "yb_device_count", "yb_num_stencils", "yb_stencil_name",
    "yb_solution_create", "yb_solution_destroy", "yb_solution_name", "yb_solution_target", "yb_solution_elem_bytes",
    "yb_solution_num_domain_dims", "yb_solution_domain_dim_name", "yb_solution_step_dim_name",
    "yb_set_rank_domain_size", "yb_set_overall_domain_size", "yb_set_num_ranks", "yb_set_rank_index", "yb_set_min_pad_size",
    "yb_get_rank_domain_size", "yb_get_overall_domain_size", "yb_get_num_ranks", "yb_get_rank_index",
    "yb_get_first_rank_domain_index", "yb_get_last_rank_domain_index", "yb_set_option", "yb_get_option", "yb_set_stream",
    "yb_solution_plan_geometry", "yb_solution_prepare", "yb_solution_is_prepared", "yb_num_vars", "yb_var_index", "yb_var_info_get", "yb_var_create", "yb_var_fuse", "yb_var_set_min_pad",
    "yb_var_set_slice", "yb_var_get_slice", "yb_var_set_slice_device", "yb_var_get_slice_device", "yb_var_set_all_same",
    "yb_var_set_slice_same", "yb_var_reduce_slice", "yb_solution_auto_tune", "yb_solution_reset_auto_tuner", "yb_solution_is_auto_tuner_enabled", "yb_solution_auto_tuner_report", "yb_var_fill_hash", "yb_var_fill_hash_shifted", "yb_var_checksum", "yb_var_device_ptr", "yb_copy_to_host", "yb_solution_run", "yb_solution_sync",
    "yb_get_stats", "yb_clear_stats", "yb_solution_set_sources", "yb_solution_set_receivers", "yb_solution_get_traces",
    "yb_solution_clear_points", "yb_solution_set_sources_weighted", "yb_solution_set_receivers_weighted", "yb_points_trilinear",
    "yb_solution_add_slice", "yb_solution_get_slice_frames", "yb_solution_clear_slices",
    "yb_solution_add_slice_injector", "yb_solution_clear_slice_injectors", "yb_solution_add_slice_injector_from",
    "yb_solution_add_slice_correlator", "yb_solution_get_correlator_image", "yb_solution_clear_slice_correlators",
    "yb_solution_add_slice_typed", "yb_solution_add_slice_injector_typed", "yb_solution_add_slice_correlator_typed",
    "yb_solution_get_slice_frame_type", "yb_solution_get_correlator_image_type", "yb_solution_add_slice_correlator_var",
    "yb_halo_export_size", "yb_halo_export", "yb_halo_import", "yb_halo_finalize",
    "yb_exchange_halos", "yb_comm_env_rank", "yb_comm_env_world", "yb_comm_env_local_rank", "yb_comm_init", "yb_comm_rank", "yb_comm_world",
    "yb_comm_barrier", "yb_comm_allgather", "yb_comm_sum_i64", "yb_comm_max_f64", "yb_comm_finalize", "yb_halo_connect",
]

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        p, i64, i32 = C.c_void_p, C.c_int64, C.c_int
        L.yb_version_string.restype = C.c_char_p
        L.yb_last_error.restype = C.c_char_p
        L.yb_stencil_name.restype = C.c_char_p
        L.yb_stencil_name.argtypes = [i32]
        L.yb_solution_create.argtypes = [C.POINTER(p), C.c_char_p, i32, i32]
        L.yb_solution_destroy.argtypes = [p]
        for nm in ("yb_solution_name", "yb_solution_target", "yb_solution_step_dim_name"):
            getattr(L, nm).restype = C.c_char_p
            getattr(L, nm).argtypes = [p]
        L.yb_solution_domain_dim_name.restype = C.c_char_p
        L.yb_solution_domain_dim_name.argtypes = [p, i32]
        L.yb_solution_elem_bytes.argtypes = [p]
        L.yb_solution_num_domain_dims.argtypes = [p]
        for nm in ("yb_set_rank_domain_size", "yb_set_overall_domain_size", "yb_set_num_ranks", "yb_set_rank_index",
                   "yb_set_min_pad_size"):
            getattr(L, nm).argtypes = [p, i32, i64]
        for nm in ("yb_get_rank_domain_size", "yb_get_overall_domain_size", "yb_get_num_ranks", "yb_get_rank_index",
                   "yb_get_first_rank_domain_index", "yb_get_last_rank_domain_index"):
            getattr(L, nm).argtypes = [p, i32]
            getattr(L, nm).restype = i64
        L.yb_set_option.argtypes = [p, C.c_char_p, C.c_char_p]
        L.yb_get_option.argtypes = [p, C.c_char_p, C.c_char_p, C.c_size_t]
        L.yb_solution_auto_tune.argtypes = [p, C.c_char_p, C.c_size_t]
        L.yb_solution_reset_auto_tuner.argtypes = [p, i32]
        L.yb_solution_is_auto_tuner_enabled.argtypes = [p]
        L.yb_solution_auto_tuner_report.argtypes = [p, C.c_char_p, C.c_size_t]
        L.yb_set_stream.argtypes = [p, p]
        L.yb_solution_plan_geometry.argtypes = [p]
        L.yb_solution_prepare.argtypes = [p, i32]
        L.yb_solution_is_prepared.argtypes = [p]
        L.yb_num_vars.argtypes = [p]
        L.yb_var_index.argtypes = [p, C.c_char_p]
        L.yb_var_info_get.argtypes = [p, i32, C.POINTER(VarInfo)]
        L.yb_var_create.argtypes = [p, C.c_char_p, i32, C.POINTER(C.c_char_p), C.POINTER(i64)]
        L.yb_var_set_min_pad.argtypes = [p, i32, i32, i64, i64]
        L.yb_var_fuse.argtypes = [p, i32, p, i32]
        for nm in ("yb_var_set_slice", "yb_var_get_slice", "yb_var_set_slice_device", "yb_var_get_slice_device"):
            getattr(L, nm).argtypes = [p, i32, p, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64)]
        L.yb_var_set_all_same.argtypes = [p, i32, C.c_double]
        L.yb_var_set_slice_same.argtypes = [p, i32, C.c_double, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64)]
        L.yb_var_reduce_slice.argtypes = [p, i32, C.POINTER(i64), C.POINTER(i64), C.POINTER(C.c_double), C.POINTER(i64)]
        L.yb_var_fill_hash.argtypes = [p, i32, i64, C.c_uint32, C.c_uint32, C.c_double, C.c_double]
        L.yb_var_fill_hash_shifted.argtypes = [p, i32, i64, C.c_uint32, C.c_uint32, C.c_double, C.c_double, C.POINTER(i64)]
        L.yb_var_checksum.argtypes = [p, i32, i64, C.POINTER(C.c_uint64)]
        L.yb_var_device_ptr.argtypes = [p, i32, i64, C.POINTER(p)]
        L.yb_solution_run.argtypes = [p, i64, i64]
        L.yb_solution_sync.argtypes = [p]
        L.yb_get_stats.argtypes = [p, C.POINTER(Stats)]
        L.yb_clear_stats.argtypes = [p]
        L.yb_solution_set_sources.argtypes = [p, C.c_char_p, i64, C.POINTER(i64), i64, i64, C.POINTER(C.c_double)]
        L.yb_solution_set_receivers.argtypes = [p, C.c_char_p, i64, C.POINTER(i64), i64, i64]
        L.yb_solution_get_traces.argtypes = [p, p, C.POINTER(C.c_uint8)]
        L.yb_solution_clear_points.argtypes = [p]
        L.yb_solution_set_sources_weighted.argtypes = [p, C.c_char_p, i64, i64, C.POINTER(i64), C.POINTER(C.c_double), i64, i64,
                                                       C.POINTER(C.c_double)]
        L.yb_solution_set_receivers_weighted.argtypes = [p, C.c_char_p, i64, i64, C.POINTER(i64), C.POINTER(C.c_double), i64, i64]
        L.yb_points_trilinear.argtypes = [i32, i64, C.POINTER(C.c_double), C.POINTER(i64), C.POINTER(C.c_double)]
        L.yb_solution_add_slice.argtypes = [p, C.c_char_p, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64), i64, i64, i64, C.POINTER(i64)]
        L.yb_solution_get_slice_frames.argtypes = [p, i64, p, C.POINTER(C.c_uint8)]
        L.yb_solution_clear_slices.argtypes = [p]
        L.yb_solution_add_slice_injector.argtypes = [p, C.c_char_p, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64), i64, i64, i64, i32, p,
                                                     C.POINTER(i64)]
        L.yb_solution_clear_slice_injectors.argtypes = [p]
        L.yb_solution_add_slice_injector_from.argtypes = [p, C.c_char_p, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64), i64, i64, i64, i32,
                                                          p, i64, i32, C.POINTER(i64)]
        L.yb_solution_add_slice_correlator.argtypes = [p, C.c_char_p, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64), i64, i64, i64, p, i64,
                                                       i32, C.POINTER(i64)]
        L.yb_solution_get_correlator_image.argtypes = [p, i64, p, C.POINTER(C.c_uint8)]
        L.yb_solution_clear_slice_correlators.argtypes = [p]
        L.yb_solution_add_slice_typed.argtypes = [p, C.c_char_p, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64), i64, i64, i64, i32,
                                                  C.POINTER(i64)]
        L.yb_solution_add_slice_injector_typed.argtypes = [p, C.c_char_p, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64), i64, i64, i64,
                                                           i32, i32, p, C.POINTER(i64)]
        L.yb_solution_add_slice_correlator_typed.argtypes = [p, C.c_char_p, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64), i64, i64, i64,
                                                             p, i64, i32, i32, C.POINTER(i64)]
        L.yb_solution_add_slice_correlator_var.argtypes = [p, C.c_char_p, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64), i64, i64, i64,
                                                           p, C.c_char_p, i64, i32, C.POINTER(i64)]
        L.yb_solution_get_slice_frame_type.argtypes = [p, i64, C.POINTER(i32)]
        L.yb_solution_get_correlator_image_type.argtypes = [p, i64, C.POINTER(i32)]
        L.yb_halo_export_size.argtypes = [p, C.POINTER(C.c_size_t)]
        L.yb_halo_export.argtypes = [p, p, C.c_size_t]
        L.yb_halo_import.argtypes = [p, i64, p, C.c_size_t]
        L.yb_halo_finalize.argtypes = [p]
        L.yb_exchange_halos.argtypes = [p]
        L.yb_comm_init.argtypes = [i32, i32, C.c_char_p]
        L.yb_comm_allgather.argtypes = [p, C.c_size_t, p]
        L.yb_comm_sum_i64.argtypes = [i64, C.POINTER(i64)]
        L.yb_comm_max_f64.argtypes = [C.c_double, C.POINTER(C.c_double)]
        L.yb_halo_connect.argtypes = [p]
        _lib = L
    return _lib


def _chk(rc: int) -> int:
    if rc < 0:
        raise YaskError(rc, lib().yb_last_error().decode())
    return rc


def device_count() -> int:
    return lib().yb_device_count()


def version() -> str:
    return lib().yb_version_string().decode()


def trilinear(pos):
    """Trilinear support of real-valued positions in global index units: pos (n, ndd) -> (idx (n, 2^ndd, ndd) int64,
    w (n, 2^ndd) float64), entry c taking floor(p_d) + bit (ndd - 1 - d) of c in dim d, its weight the product over d, left to
    right, of f_d or 1 - f_d (yb_points_trilinear).  An integer position gets one entry of weight 1, the rest 0."""
    a = np.asarray(pos, dtype=np.float64)
    if a.ndim == 1:
        a = a.reshape(1, -1)
    if a.ndim != 2 or not 1 <= a.shape[1] <= 3 or a.shape[0] < 1:
        raise YaskError(-1, f"trilinear: expected positions of shape (n, ndd) with ndd 1, 2 or 3, got shape {a.shape}")
    a = np.ascontiguousarray(a)
    n, nd = a.shape
    idx = np.zeros((n, 1 << nd, nd), np.int64)
    w = np.zeros((n, 1 << nd), np.float64)
    _chk(lib().yb_points_trilinear(nd, n, a.ctypes.data_as(C.POINTER(C.c_double)), idx.ctypes.data_as(C.POINTER(C.c_int64)),
                                   w.ctypes.data_as(C.POINTER(C.c_double))))
    return idx, w


# Frame and image types of the slice calls (YB_TYPE_* of include/yask_b200.h).  numpy has no bfloat16: bf16 frames cross the
# C ABI as uint16 bit patterns and come back widened exactly to float32.
TYPE_ELEM, TYPE_F64, TYPE_F32, TYPE_F16, TYPE_BF16 = 0, 1, 2, 3, 4
SLICE_TYPES = {"float64": TYPE_F64, "float32": TYPE_F32, "float16": TYPE_F16, "bfloat16": TYPE_BF16}


def slice_type(what: str, field: str, dtype) -> int:
    """YB_TYPE_* of a dtype argument: None (the element type), "float16", "bfloat16", "float32", "float64" or a numpy dtype."""
    if dtype is None:
        return TYPE_ELEM
    if isinstance(dtype, str) and dtype in SLICE_TYPES:
        return SLICE_TYPES[dtype]
    try:
        name = np.dtype(dtype).name
    except TypeError:
        name = None
    if name in ("float64", "float32", "float16"):
        return SLICE_TYPES[name]
    raise YaskError(-1, f"{what}: unknown {field} {dtype!r} (expected 'float16', 'bfloat16', 'float32' or 'float64')")


def bf16_bits(a) -> np.ndarray:
    """float32 values -> bfloat16 bit patterns (uint16): IEEE round to nearest even, overflow to +-inf, subnormals kept, NaN a
    (quiet) NaN."""
    f = np.ascontiguousarray(a, np.float32)
    u = f.view(np.uint32)
    out = ((u + np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1))) >> np.uint32(16)).astype(np.uint16)
    nan = np.isnan(f)
    out[nan] = ((u[nan] >> np.uint32(16)) | np.uint32(0x40)).astype(np.uint16)
    return out


def bf16_widen(bits) -> np.ndarray:
    """bfloat16 bit patterns (uint16) -> float32, exactly."""
    return (np.asarray(bits, np.uint16).astype(np.uint32) << np.uint32(16)).view(np.float32)


def narrow_frames(a, elem_bytes: int, ftype: int) -> np.ndarray:
    """What a host-fed injector's frames hold: the real array rounded to the element type T, then by RNE to the frame type
    (bf16 as uint16 bit patterns)."""
    t = np.ascontiguousarray(a, dtype=np.float32 if elem_bytes == 4 else np.float64)
    with np.errstate(over="ignore"):
        if ftype == TYPE_BF16:
            return bf16_bits(t.astype(np.float32))
        if ftype == TYPE_F16:
            return t.astype(np.float16)
        if ftype == TYPE_F32:
            return t.astype(np.float32)
        if ftype == TYPE_F64:
            return t.astype(np.float64)
    return t


def _arr(vals: Sequence[int]):
    return (C.c_int64 * len(vals))(*[int(v) for v in vals])


class Var:
    """Handle to one var of a Solution; method names follow yk_var (aux/yk_var_api.hpp)."""

    def __init__(self, soln: "Solution", index: int):
        self.soln, self.index = soln, index

    @property
    def info(self) -> VarInfo:
        vi = VarInfo()
        _chk(lib().yb_var_info_get(self.soln._h, self.index, C.byref(vi)))
        return vi

    def get_name(self) -> str:
        return self.info.name.decode()

    def get_dim_names(self):
        vi = self.info
        return [vi.dims[i].name.decode() for i in range(vi.num_dims)]

    @property
    def dtype(self):
        return np.float32 if self.info.elem_bytes == 4 else np.float64

    def _box(self, step, with_halo: bool):
        vi = self.info
        first, last = [], []
        for i in range(vi.num_dims):
            d = vi.dims[i]
            if d.kind == 0:
                first.append(step)
                last.append(step)
            elif d.kind == 2:
                first.append(d.first_misc_index)
                last.append(d.first_misc_index + d.domain_size - 1)
            else:
                first.append(d.rank_offset - (d.left_halo if with_halo else 0))
                last.append(d.rank_offset + d.domain_size - 1 + (d.right_halo if with_halo else 0))
        return first, last

    def halo_box(self, step=0):
        """(first, last) global indices of the rank's domain+halo box at API step `step`."""
        return self._box(step, True)

    def domain_box(self, step=0):
        return self._box(step, False)

    def set_elements_in_slice(self, buf: np.ndarray, first, last) -> int:
        a = np.ascontiguousarray(buf, dtype=self.dtype)
        n = C.c_int64(0)
        _chk(lib().yb_var_set_slice(self.soln._h, self.index, a.ctypes.data, _arr(first), _arr(last), C.byref(n)))
        assert n.value == a.size, (n.value, a.size)
        return n.value

    def get_elements_in_slice(self, first, last) -> np.ndarray:
        vi = self.info
        shape = [int(l - f + 1) for f, l in zip(first, last)]
        out = np.empty(shape, dtype=self.dtype)
        n = C.c_int64(0)
        _chk(lib().yb_var_get_slice(self.soln._h, self.index, out.ctypes.data, _arr(first), _arr(last), C.byref(n)))
        if vi.has_step and shape[0] == 1:
            out = out.reshape(shape[1:])
        return out

    def set_all_elements_same(self, val: float):
        _chk(lib().yb_var_set_all_same(self.soln._h, self.index, float(val)))

    def set_elements_in_slice_same(self, val: float, first, last) -> int:
        n = C.c_int64(0)
        _chk(lib().yb_var_set_slice_same(self.soln._h, self.index, float(val), _arr(first), _arr(last), C.byref(n)))
        return n.value

    def reduce_elements_in_slice(self, first, last) -> dict:
        """yk_var::reduce_elements_in_slice with every reduction requested: computed on the device in double."""
        out = (C.c_double * 5)()
        n = C.c_int64(0)
        _chk(lib().yb_var_reduce_slice(self.soln._h, self.index, _arr(first), _arr(last), out, C.byref(n)))
        return {"num": n.value, "sum": out[0], "sum_squares": out[1], "product": out[2], "max": out[3], "min": out[4]}

    def fill_hash(self, step: int, seed: int, salt: int, lo: float, hi: float, shift: Sequence[int] | None = None):
        """Hash field over the rank's halo box of `step`; `shift` (per solution domain dim) moves the window of global
        indices the values are drawn from."""
        if shift is None:
            _chk(lib().yb_var_fill_hash(self.soln._h, self.index, int(step), seed & 0xFFFFFFFF, salt & 0xFFFFFFFF, lo, hi))
        else:
            _chk(lib().yb_var_fill_hash_shifted(self.soln._h, self.index, int(step), seed & 0xFFFFFFFF, salt & 0xFFFFFFFF, lo, hi,
                                                _arr(list(shift) + [0] * (3 - len(shift)))))

    def fuse_vars(self, source: "Var"):
        """yk_var::fuse_vars: this var becomes another reference to `source`'s device storage."""
        _chk(lib().yb_var_fuse(self.soln._h, self.index, source.soln._h, source.index))

    def checksum(self, step: int) -> int:
        out = C.c_uint64(0)
        _chk(lib().yb_var_checksum(self.soln._h, self.index, int(step), C.byref(out)))
        return out.value

    def device_ptr(self, step: int = 0) -> int:
        out = C.c_void_p()
        _chk(lib().yb_var_device_ptr(self.soln._h, self.index, int(step), C.byref(out)))
        return out.value

    def get_first_valid_step_index(self):
        return self.info.first_valid_step

    def get_last_valid_step_index(self):
        return self.info.last_valid_step


class Solution:
    """Mirror of yk_solution for the hot path (aux/yk_solution_api.hpp): sizes, prepare, vars, run, stats."""

    def __init__(self, stencil: str = "iso3dfd", radius: int = 0, elem_bytes: int = 4):
        h = C.c_void_p()
        _chk(lib().yb_solution_create(C.byref(h), stencil.encode(), radius, elem_bytes))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            lib().yb_solution_destroy(self._h)
            self._h = None

    end_solution = close

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def get_name(self):
        return lib().yb_solution_name(self._h).decode()

    def get_target(self):
        return lib().yb_solution_target(self._h).decode()

    def get_element_bytes(self):
        return lib().yb_solution_elem_bytes(self._h)

    def get_domain_dim_names(self):
        return [lib().yb_solution_domain_dim_name(self._h, i).decode() for i in range(lib().yb_solution_num_domain_dims(self._h))]

    def get_step_dim_name(self):
        return lib().yb_solution_step_dim_name(self._h).decode()

    def _dim(self, dim):
        return dim if isinstance(dim, int) else self.get_domain_dim_names().index(dim)

    def set_overall_domain_size_vec(self, n):
        for d, v in enumerate(n):
            _chk(lib().yb_set_overall_domain_size(self._h, d, int(v)))

    def set_rank_domain_size_vec(self, n):
        for d, v in enumerate(n):
            _chk(lib().yb_set_rank_domain_size(self._h, d, int(v)))

    def set_num_ranks_vec(self, n):
        for d, v in enumerate(n):
            _chk(lib().yb_set_num_ranks(self._h, d, int(v)))

    def set_rank_index_vec(self, n):
        for d, v in enumerate(n):
            _chk(lib().yb_set_rank_index(self._h, d, int(v)))

    def get_rank_domain_size_vec(self):
        return [lib().yb_get_rank_domain_size(self._h, d) for d in range(len(self.get_domain_dim_names()))]

    def get_overall_domain_size_vec(self):
        return [lib().yb_get_overall_domain_size(self._h, d) for d in range(len(self.get_domain_dim_names()))]

    def get_first_rank_domain_index_vec(self):
        return [lib().yb_get_first_rank_domain_index(self._h, d) for d in range(len(self.get_domain_dim_names()))]

    def set_option(self, key: str, value):
        _chk(lib().yb_set_option(self._h, key.encode(), str(value).encode()))

    def run_auto_tuner_now(self) -> str:
        """Offline auto-tuner: times the engine's launch variants, keeps the fastest; var contents are not preserved."""
        buf = C.create_string_buffer(8192)
        _chk(lib().yb_solution_auto_tune(self._h, buf, 8192))
        return buf.value.decode()

    def reset_auto_tuner(self, enable: bool = True):
        _chk(lib().yb_solution_reset_auto_tuner(self._h, 1 if enable else 0))

    def is_auto_tuner_enabled(self) -> bool:
        return bool(lib().yb_solution_is_auto_tuner_enabled(self._h))

    def auto_tuner_report(self) -> str:
        buf = C.create_string_buffer(8192)
        _chk(lib().yb_solution_auto_tuner_report(self._h, buf, 8192))
        return buf.value.decode()

    def get_option(self, key: str) -> str:
        buf = C.create_string_buffer(256)
        _chk(lib().yb_get_option(self._h, key.encode(), buf, 256))
        return buf.value.decode()

    def set_stream(self, cuda_stream: int):
        _chk(lib().yb_set_stream(self._h, C.c_void_p(cuda_stream)))

    def plan_geometry(self):
        _chk(lib().yb_solution_plan_geometry(self._h))

    def prepare_solution(self, device: int = 0):
        _chk(lib().yb_solution_prepare(self._h, device))

    def get_num_vars(self):
        return lib().yb_num_vars(self._h)

    def get_var(self, name: str) -> Var:
        return Var(self, _chk(lib().yb_var_index(self._h, name.encode())))

    def new_fixed_size_var(self, name: str, dims, sizes) -> Var:
        names = (C.c_char_p * len(dims))(*[d.encode() for d in dims])
        return Var(self, _chk(lib().yb_var_create(self._h, name.encode(), len(dims), names, _arr(sizes))))

    def new_var(self, name: str, dims) -> Var:
        names = (C.c_char_p * len(dims))(*[d.encode() for d in dims])
        return Var(self, _chk(lib().yb_var_create(self._h, name.encode(), len(dims), names, None)))

    def get_vars(self):
        return [Var(self, i) for i in range(self.get_num_vars())]

    def run_solution(self, first_step: int, last_step: int | None = None):
        _chk(lib().yb_solution_run(self._h, first_step, first_step if last_step is None else last_step))

    def sync(self):
        _chk(lib().yb_solution_sync(self._h))

    def get_stats(self) -> Stats:
        st = Stats()
        _chk(lib().yb_get_stats(self._h, C.byref(st)))
        return st

    def clear_stats(self):
        _chk(lib().yb_clear_stats(self._h))

    # point sources and receivers (yb_solution_set_sources / set_receivers / get_traces / clear_points)
    def _points(self, idx, what: str) -> np.ndarray:
        nd = len(self.get_domain_dim_names())
        a = np.asarray(idx, dtype=np.int64)
        if a.ndim == 1 and nd == 1:
            a = a.reshape(-1, 1)
        if a.ndim != 2 or a.shape[1] != nd or a.shape[0] < 1:
            raise YaskError(-1, f"{what}: expected a list of points with {nd} domain index(es) each "
                                f"({', '.join(self.get_domain_dim_names())}), got shape {a.shape}")
        return np.ascontiguousarray(a)

    def set_sources(self, var: str, idx, t0: int, amp):
        """Add amp[u - t0][i] to var(u, idx[i]) (list order, element-type rounding) after every step u a run computes with
        0 <= u - t0 < len(amp).  idx: N points of global domain indices; amp: (nrows, N)."""
        pts = self._points(idx, "sources")
        a = np.asarray(amp, dtype=np.float64)
        if a.ndim != 2 or a.shape[1] != pts.shape[0]:
            raise YaskError(-1, f"sources: amplitude table of shape {a.shape} does not match {pts.shape[0]} source point(s): "
                                f"expected (nrows, {pts.shape[0]})")
        a = np.ascontiguousarray(a)
        _chk(lib().yb_solution_set_sources(self._h, var.encode(), pts.shape[0], pts.ctypes.data_as(C.POINTER(C.c_int64)),
                                           int(t0), a.shape[0], a.ctypes.data_as(C.POINTER(C.c_double))))

    def set_receivers(self, var: str, idx, t0: int, nrows: int):
        """Record var(u, idx[j]) into trace row u - t0 after every step u a run computes with 0 <= u - t0 < nrows."""
        pts = self._points(idx, "receivers")
        _chk(lib().yb_solution_set_receivers(self._h, var.encode(), pts.shape[0], pts.ctypes.data_as(C.POINTER(C.c_int64)),
                                             int(t0), int(nrows)))
        self._nrcv, self._nrows_r = pts.shape[0], int(nrows)

    def _weighted(self, idx, w, what: str):
        nd = len(self.get_domain_dim_names())
        a = np.asarray(idx, dtype=np.int64)
        ww = np.asarray(w, dtype=np.float64)
        if a.ndim != 3 or a.shape[2] != nd or a.shape[0] < 1 or a.shape[1] < 1:
            raise YaskError(-1, f"{what}: expected an index table of shape (n, k, {nd}) -- k support entries of {nd} domain "
                                f"index(es) ({', '.join(self.get_domain_dim_names())}) per point -- got shape {a.shape}")
        if ww.shape != a.shape[:2]:
            raise YaskError(-1, f"{what}: weight table of shape {ww.shape} does not match the index table: expected {a.shape[:2]}")
        return np.ascontiguousarray(a), np.ascontiguousarray(ww)

    def set_sources_weighted(self, var: str, idx, w, t0: int, amp):
        """Add w[i][q] * amp[u - t0][i] to var(u, idx[i][q]) for every source i in list order and every entry q in order with
        w[i][q] != 0, after every step u a run computes with 0 <= u - t0 < len(amp).  idx: (N, k, ndd) global domain indices;
        w: (N, k); amp: (nrows, N)."""
        pts, ww = self._weighted(idx, w, "weighted sources")
        a = np.asarray(amp, dtype=np.float64)
        if a.ndim != 2 or a.shape[1] != pts.shape[0]:
            raise YaskError(-1, f"weighted sources: amplitude table of shape {a.shape} does not match {pts.shape[0]} source(s): "
                                f"expected (nrows, {pts.shape[0]})")
        a = np.ascontiguousarray(a)
        _chk(lib().yb_solution_set_sources_weighted(self._h, var.encode(), pts.shape[0], pts.shape[1],
                                                    pts.ctypes.data_as(C.POINTER(C.c_int64)), ww.ctypes.data_as(C.POINTER(C.c_double)),
                                                    int(t0), a.shape[0], a.ctypes.data_as(C.POINTER(C.c_double))))

    def set_receivers_weighted(self, var: str, idx, w, t0: int, nrows: int):
        """Record the sum over q in order of w[j][q] * var(u, idx[j][q]) (in double, each product and sum rounded, then rounded
        to the element type) into trace row u - t0 after every step u a run computes with 0 <= u - t0 < nrows."""
        pts, ww = self._weighted(idx, w, "weighted receivers")
        _chk(lib().yb_solution_set_receivers_weighted(self._h, var.encode(), pts.shape[0], pts.shape[1],
                                                      pts.ctypes.data_as(C.POINTER(C.c_int64)), ww.ctypes.data_as(C.POINTER(C.c_double)),
                                                      int(t0), int(nrows)))
        self._nrcv, self._nrows_r = pts.shape[0], int(nrows)

    def get_traces(self):
        """(traces, owned): traces (nrows, M) in the element dtype, owned[j] True for the receivers this rank records."""
        dt = np.float32 if self.get_element_bytes() == 4 else np.float64
        m, nrows = getattr(self, "_nrcv", 0), getattr(self, "_nrows_r", 0)
        out = np.zeros((nrows, m), dtype=dt)
        owned = np.zeros(m, dtype=np.uint8)
        _chk(lib().yb_solution_get_traces(self._h, out.ctypes.data if self.is_prepared() else None,
                                          owned.ctypes.data_as(C.POINTER(C.c_uint8))))
        return out, owned.astype(bool)

    def clear_points(self):
        _chk(lib().yb_solution_clear_points(self._h))
        self._nrcv = self._nrows_r = 0

    # slice recorders (yb_solution_add_slice / get_slice_frames / clear_slices)
    def add_slice(self, var: str, first, last, t0: int, nrows: int, stride=None, every: int = 1, dtype=None) -> int:
        """Record the box first[d], first[d] + stride[d], ... <= last[d] (global domain indices) of var(u) into frame row
        (u - t0) // every after every step u a run computes with u - t0 a multiple of `every` and the row below nrows.
        dtype: the frame type ("float16", "bfloat16", "float32", "float64" or a numpy dtype; None: the element type), each
        element rounded to it to nearest even.  Returns the recorder's id."""
        ftype = slice_type("slice", "dtype", dtype)
        nd = len(self.get_domain_dim_names())
        f, l = np.atleast_1d(np.asarray(first, np.int64)), np.atleast_1d(np.asarray(last, np.int64))
        st = np.ones(nd, np.int64) if stride is None else np.atleast_1d(np.asarray(stride, np.int64))
        for what, a in (("first", f), ("last", l), ("stride", st)):
            if a.shape != (nd,):
                raise YaskError(-1, f"slice: {what} needs {nd} domain index(es) ({', '.join(self.get_domain_dim_names())}), "
                                    f"got {a.tolist()}")
        rid = C.c_int64(-1)
        _chk(lib().yb_solution_add_slice_typed(self._h, var.encode(), _arr(f.tolist()), _arr(l.tolist()), _arr(st.tolist()),
                                               int(t0), int(every), int(nrows), ftype, C.byref(rid)))
        if not hasattr(self, "_slices"):
            self._slices = {}
        self._slices[rid.value] = (tuple(int(x) for x in (l - f) // np.maximum(st, 1) + 1), int(nrows))
        return rid.value

    def get_slice_frames(self, rid: int):
        """(frames, owned): frames (nrows, *box_shape) in the frame type (bfloat16 widened exactly to float32), owned
        (box_shape) True for the points this rank records; the others stay 0."""
        shape, nrows = getattr(self, "_slices", {}).get(rid, ((0,), 0))
        ftype = self._slice_type(lib().yb_solution_get_slice_frame_type, rid)
        out = np.zeros((nrows,) + shape, dtype=self._TYPE_DTYPES[ftype])
        owned = np.zeros(shape, dtype=np.uint8)
        _chk(lib().yb_solution_get_slice_frames(self._h, int(rid), out.ctypes.data if self.is_prepared() else None,
                                                owned.ctypes.data_as(C.POINTER(C.c_uint8))))
        return (bf16_widen(out) if ftype == TYPE_BF16 else out), owned.astype(bool)

    _TYPE_DTYPES = {TYPE_F64: np.float64, TYPE_F32: np.float32, TYPE_F16: np.float16, TYPE_BF16: np.uint16}

    def _slice_type(self, query, sid: int) -> int:
        """The resolved frame or image type of recorder or correlator `sid`, or the element type when there is none (the
        getters then refuse it themselves)."""
        t = C.c_int(0)
        if query(self._h, int(sid), C.byref(t)) != 0:
            return TYPE_F32 if self.get_element_bytes() == 4 else TYPE_F64
        return t.value

    def clear_slices(self):
        _chk(lib().yb_solution_clear_slices(self._h))
        self._slices = {}

    # slice injectors (yb_solution_add_slice_injector / clear_slice_injectors)
    INJECT_MODES = {"add": 0, "set": 1}        # YB_INJECT_ADD, YB_INJECT_SET

    def add_slice_injector(self, var: str, first, last, t0: int, frames, stride=None, every: int = 1, mode: str = "add",
                           dtype=None) -> int:
        """After every step u a run computes with u - t0 a multiple of `every` and r = (u - t0) // every below len(frames), set
        (mode "set") or add frames[r] to (mode "add", one add in the element type) var(u) at the box first[d], first[d] +
        stride[d], ... <= last[d] (global domain indices).  frames: (nrows, *box_shape); a real array of another dtype is rounded
        to the element type.  dtype: the frame type the engine holds them in (as add_slice): the frames rounded to the element
        type are rounded again, to nearest even, to it, and widened exactly on the device.  The frames are copied.  Returns the
        injector's id."""
        ftype = slice_type("slice injector", "dtype", dtype)
        nd = len(self.get_domain_dim_names())
        f, l = np.atleast_1d(np.asarray(first, np.int64)), np.atleast_1d(np.asarray(last, np.int64))
        st = np.ones(nd, np.int64) if stride is None else np.atleast_1d(np.asarray(stride, np.int64))
        for what, a in (("first", f), ("last", l), ("stride", st)):
            if a.shape != (nd,):
                raise YaskError(-1, f"slice injector: {what} needs {nd} domain index(es) ({', '.join(self.get_domain_dim_names())}), "
                                    f"got {a.tolist()}")
        if mode not in self.INJECT_MODES:
            raise YaskError(-1, f"slice injector: unknown mode {mode!r} (expected 'add' or 'set')")
        fr = np.asarray(frames)
        if np.iscomplexobj(fr) or not (np.issubdtype(fr.dtype, np.floating) or np.issubdtype(fr.dtype, np.integer)):
            raise YaskError(-1, f"slice injector: frames of dtype {fr.dtype} are not real numbers")
        box = tuple(int(x) for x in (l - f) // np.maximum(st, 1) + 1)
        # an empty box or a stride below 1 is left to the engine, which names it
        if (l >= f).all() and (st >= 1).all() and (fr.ndim != nd + 1 or tuple(fr.shape[1:]) != box):
            raise YaskError(-1, f"slice injector: frames of shape {fr.shape} do not match the decimated box: expected "
                                f"(nrows, {', '.join(str(b) for b in box)})")
        fr = narrow_frames(fr, self.get_element_bytes(), ftype)
        rid = C.c_int64(-1)
        _chk(lib().yb_solution_add_slice_injector_typed(self._h, var.encode(), _arr(f.tolist()), _arr(l.tolist()), _arr(st.tolist()),
                                                        int(t0), int(every), fr.shape[0] if fr.ndim else 0, self.INJECT_MODES[mode], ftype,
                                                        fr.ctypes.data, C.byref(rid)))
        return rid.value

    def clear_slice_injectors(self):
        _chk(lib().yb_solution_clear_slice_injectors(self._h))

    def _box(self, what, first, last, stride):
        nd = len(self.get_domain_dim_names())
        f, l = np.atleast_1d(np.asarray(first, np.int64)), np.atleast_1d(np.asarray(last, np.int64))
        st = np.ones(nd, np.int64) if stride is None else np.atleast_1d(np.asarray(stride, np.int64))
        for name, a in (("first", f), ("last", l), ("stride", st)):
            if a.shape != (nd,):
                raise YaskError(-1, f"{what}: {name} needs {nd} domain index(es) ({', '.join(self.get_domain_dim_names())}), "
                                    f"got {a.tolist()}")
        return f, l, st

    def add_slice_injector_from(self, var: str, first, last, t0: int, nrows: int, src: "Solution", src_id: int, reverse: bool = False,
                                stride=None, every: int = 1, mode: str = "add") -> int:
        """add_slice_injector with the frames of recorder src_id of solution src (which may be this one), read on the device with
        no copy: row r reads recorder row nrows - 1 - r when reverse, else r.  Returns the injector's id."""
        f, l, st = self._box("slice injector", first, last, stride)
        if mode not in self.INJECT_MODES:
            raise YaskError(-1, f"slice injector: unknown mode {mode!r} (expected 'add' or 'set')")
        rid = C.c_int64(-1)
        _chk(lib().yb_solution_add_slice_injector_from(self._h, var.encode(), _arr(f.tolist()), _arr(l.tolist()), _arr(st.tolist()),
                                                       int(t0), int(every), int(nrows), self.INJECT_MODES[mode], src._h, int(src_id),
                                                       int(reverse), C.byref(rid)))
        return rid.value

    # slice correlators (yb_solution_add_slice_correlator / get_correlator_image / clear_slice_correlators)
    def add_slice_correlator(self, var: str, first, last, t0: int, nrows: int, src: "Solution" = None, src_id: int = None,
                             reverse: bool = False, stride=None, every: int = 1, image_dtype=None) -> int:
        """After every step u a run computes with u - t0 a multiple of `every` and r = (u - t0) // every below nrows, add
        var(u) * b to the image at the box first[d], first[d] + stride[d], ... <= last[d], the product and the sum each rounded to
        the element type.  b is var(u) with no src (the illumination), else row r (nrows - 1 - r when reverse) of recorder src_id
        of solution src (which may be this one), read in its frame type.  image_dtype "float64" in an fp32 solution holds the
        image in double: image + double(var) * double(b), the product exact.  Returns the correlator's id."""
        itype = slice_type("slice correlator", "image_dtype", image_dtype)
        f, l, st = self._box("slice correlator", first, last, stride)
        if src is not None and src_id is None:
            raise YaskError(-1, "slice correlator: a source solution needs src_id, the id of one of its recorders")
        rid = C.c_int64(-1)
        _chk(lib().yb_solution_add_slice_correlator_typed(self._h, var.encode(), _arr(f.tolist()), _arr(l.tolist()), _arr(st.tolist()),
                                                          int(t0), int(every), int(nrows), None if src is None else src._h,
                                                          0 if src_id is None else int(src_id), int(reverse), itype, C.byref(rid)))
        if not hasattr(self, "_correlators"):
            self._correlators = {}
        self._correlators[rid.value] = tuple(int(x) for x in (l - f) // np.maximum(st, 1) + 1)
        return rid.value

    def add_slice_correlator_var(self, var: str, first, last, t0: int, nrows: int, src: "Solution", src_var: str, src_t0: int = None,
                                 stride=None, every: int = 1, image_dtype=None) -> int:
        """add_slice_correlator whose b is var src_var of another prepared solution src on the same device, at the paired step:
        when row r is due at step u, image += var(u) * src_var(src_t0 + (u - t0)) (src_t0 defaults to t0).  For a source wavefield
        rebuilt backwards in time beside the adjoint run: alternating one-step runs of the two enqueue with no host sync and run
        in the order they were called.  A run whose due steps pair with steps outside src_var's valid window, as src's calls have
        left it, is refused before it changes anything.  Returns the correlator's id (shared with the other correlators)."""
        itype = slice_type("slice correlator", "image_dtype", image_dtype)
        f, l, st = self._box("slice correlator", first, last, stride)
        rid = C.c_int64(-1)
        _chk(lib().yb_solution_add_slice_correlator_var(self._h, var.encode(), _arr(f.tolist()), _arr(l.tolist()), _arr(st.tolist()),
                                                        int(t0), int(every), int(nrows), None if src is None else src._h,
                                                        None if src_var is None else src_var.encode(),
                                                        int(t0 if src_t0 is None else src_t0), itype, C.byref(rid)))
        if not hasattr(self, "_correlators"):
            self._correlators = {}
        self._correlators[rid.value] = tuple(int(x) for x in (l - f) // np.maximum(st, 1) + 1)
        return rid.value

    def get_correlator_image(self, cid: int):
        """(image, owned): image (box_shape) in the image type, owned (box_shape) True for the points this rank holds; the
        others stay 0."""
        shape = getattr(self, "_correlators", {}).get(cid, (0,))
        out = np.zeros(shape, dtype=self._TYPE_DTYPES[self._slice_type(lib().yb_solution_get_correlator_image_type, cid)])
        owned = np.zeros(shape, dtype=np.uint8)
        _chk(lib().yb_solution_get_correlator_image(self._h, int(cid), out.ctypes.data if self.is_prepared() else None,
                                                    owned.ctypes.data_as(C.POINTER(C.c_uint8))))
        return out, owned.astype(bool)

    def clear_slice_correlators(self):
        _chk(lib().yb_solution_clear_slice_correlators(self._h))
        self._correlators = {}

    def is_prepared(self) -> bool:
        return bool(lib().yb_solution_is_prepared(self._h))

    # multi-GPU plumbing (yb_halo_*)
    def halo_export(self) -> bytes:
        n = C.c_size_t(0)
        _chk(lib().yb_halo_export_size(self._h, C.byref(n)))
        buf = C.create_string_buffer(n.value)
        _chk(lib().yb_halo_export(self._h, buf, n.value))
        return buf.raw

    def halo_import(self, peer_rank: int, blob: bytes):
        _chk(lib().yb_halo_import(self._h, peer_rank, blob, len(blob)))

    def halo_finalize(self):
        _chk(lib().yb_halo_finalize(self._h))

    def exchange_halos(self):
        _chk(lib().yb_exchange_halos(self._h))
