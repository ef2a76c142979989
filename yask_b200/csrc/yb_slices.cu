// Slice recorders on the device (yb_slices.h): receiver planes, decimated snapshots and field dumps every k steps, recorded
// inside run_solution() by one many-CTA launch per step, instead of the reference API loop run_solution(t, t) /
// get_elements_in_slice, which pays a synchronous device-to-host copy per frame and loses the temporal tile's pairs.  Slice
// injectors write boxes back the same way (plane-wave and areal sources, boundary replay, time-varying Dirichlet data), instead of
// the loop run_solution(t, t) / get_elements_in_slice / set_elements_in_slice.  Slice correlators accumulate the imaging condition
// image += var(u) * b into an image on the device, b being var(u) itself, a recorder's frame or a var of another solution at a
// paired step, instead of the loop run_solution(t, t) / get_elements_in_slice / host arithmetic.
#include <stdio.h>
#include <string.h>

#include <algorithm>

#include "yb_box.cuh"
#include "yb_points.h"
#include "yb_slices.h"

namespace yb {

namespace {

// One recorder as the kernel sees it.  The frames stay put while the recorder is set; the var's storage and slot bias may not:
// fuse_vars on a prepared solution replaces the storage, and the offline tuner's pair trials move the bias.  A run never moves
// either (no fused pair runs while a recorder is set), so slices_begin_run re-uploads a table that is out of date before the
// run enqueues anything.
struct SliceDesc {
    const char* var_base;           // Var::dev
    long long slot_bytes;
    int alloc, bias, step_off;      // Var::slot_of(u) = imod(u, alloc) + bias
    long long t0, every, nrows;
    BoxDev box;                     // this rank's part: element offset of its first point, decimated strides
    char* frames;                   // nrows x box.total elements (correlators: null for an autocorrelation)
    char* image;                    // correlators: box.total elements
    int rev;                        // row r reads frame row nrows - 1 - r
    int lanes_log2;                 // correlators: threads per row of the unit-stride dim, a power of two up to 256
    // injectors: YB_INJECT_ADD / SET, and the rank-local coordinates of the first owned point and their step per box index
    // (dims right-aligned as in box), which the split form's selection tests against the interior box
    int mode;
    long long loc0[4], lstep[4];
    int ftype, itype;               // YB_TYPE_* of the frames and (correlators) of the image; never YB_TYPE_ELEM
    // correlators with a var link (b_var): b is element b_off + c0 * b_vs[0] + c1 * b_vs[1] + c2 * b_vs[2] + i * b_vs[3] of the
    // source var's slot imod(u + b_shift, b_alloc) + b_bias (b_slot_bytes each) at box index (c0, c1, c2, i)
    const char* b_base;
    long long b_slot_bytes, b_shift, b_off, b_vs[4];
    int b_var, b_alloc, b_bias;
};

// A 16-bit frame element, held as its bit pattern.
struct Half { unsigned short bits; };
struct BHalf { unsigned short bits; };

// N_F: IEEE round-to-nearest-even narrowing of an element to a frame type, in inline PTX without .ftz.  The engine builds with
// -ftz=true, under which nvcc's own f64 -> f32 conversion flushes subnormal results; these keep subnormal inputs and results,
// turn finite values beyond F's range into +-inf and keep NaN a NaN.
template <typename F, typename T> __device__ __forceinline__ F narrow(T v) { return v; }
template <> __device__ __forceinline__ float narrow<float, double>(double v) {
    float o;
    asm("cvt.rn.f32.f64 %0, %1;" : "=f"(o) : "d"(v));
    return o;
}
template <> __device__ __forceinline__ Half narrow<Half, float>(float v) {
    Half o;
    asm("cvt.rn.f16.f32 %0, %1;" : "=h"(o.bits) : "f"(v));
    return o;
}
template <> __device__ __forceinline__ BHalf narrow<BHalf, float>(float v) {
    BHalf o;
    asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(o.bits) : "f"(v));
    return o;
}

// Exact widening of a frame element to float or double (inline PTX for f32 -> f64: no .ftz, so subnormal inputs are kept).
__device__ __forceinline__ float wide_f(float v) { return v; }
__device__ __forceinline__ float wide_f(Half h) {
    float o;
    asm("cvt.f32.f16 %0, %1;" : "=f"(o) : "h"(h.bits));
    return o;
}
__device__ __forceinline__ float wide_f(BHalf h) { return __uint_as_float(unsigned(h.bits) << 16); }
__device__ __forceinline__ double wide_d(double v) { return v; }
__device__ __forceinline__ double wide_d(float v) {
    double o;
    asm("cvt.f64.f32 %0, %1;" : "=d"(o) : "f"(v));
    return o;
}
template <typename T, typename F> __device__ __forceinline__ T widen(F v) {
    if constexpr (sizeof(T) == 4) return wide_f(v);
    else return wide_d(v);
}

// f(F{}) with the frame element type F that `type` names among those a solution of element type T allows (the add call refused
// every other): fp32 solutions f32, f16, bf16; fp64 solutions f64, f32.  `type` is one descriptor's, so the branch is uniform
// across a CTA.
template <typename T, typename Fn> __device__ __forceinline__ void with_frame_type(int type, Fn&& f) {
    if constexpr (sizeof(T) == 4) {
        if (type == YB_TYPE_F16) f(Half{});
        else if (type == YB_TYPE_BF16) f(BHalf{});
        else f(float{});
    } else {
        if (type == YB_TYPE_F32) f(float{});
        else f(double{});
    }
}

__host__ __device__ __forceinline__ bool row_due(long long u, long long t0, long long every, long long nrows, long long& row) {
    const long long k = u - t0;
    if (k < 0 || k % every != 0) return false;
    row = k / every;
    return row < nrows;
}

// blockIdx.y walks the recorders, blockIdx.x and the threads the dense points of one, the unit-stride dim fastest (box_offset):
// x- and y-planes and stride-1 boxes are coalesced.  Offsets are 64-bit: a slot may hold more than 2^31 elements.
template <typename T>
__global__ void __launch_bounds__(256) slices_kernel(const SliceDesc* __restrict__ table, int nrec, long long t) {
    for (int r = blockIdx.y; r < nrec; r += gridDim.y) {
        const SliceDesc& d = table[r];
        const long long u = t + d.step_off;
        long long row;
        if (!row_due(u, d.t0, d.every, d.nrows, row)) continue;
        const BoxDev b = d.box;
        long long slot = u % d.alloc;
        slot = (slot < 0 ? slot + d.alloc : slot) + d.bias;
        const T* __restrict__ src = reinterpret_cast<const T*>(d.var_base + slot * d.slot_bytes);
        with_frame_type<T>(d.ftype, [&](auto tag) {
            using F = decltype(tag);
            F* __restrict__ dst = reinterpret_cast<F*>(d.frames) + row * b.total;
            long long coord[4];
            for (long long i = blockIdx.x * 256ll + threadIdx.x; i < b.total; i += gridDim.x * 256ll) dst[i] = narrow<F>(src[box_offset(b, i, coord)]);
        });
    }
}

// the rounding of add_to_element: one add in the element type
__device__ __forceinline__ float add_elem(float v, float a) { return __fadd_rn(v, a); }
__device__ __forceinline__ double add_elem(double v, double a) { return __dadd_rn(v, a); }

// which points of one injecting launch: PTS_ALL, or those outside (PTS_EXTERIOR) or inside (PTS_INTERIOR) the rank-local box
struct InjectSel {
    int sel;
    long long ib[4], ie[4];         // right-aligned like BoxDev
};

// The dual of slices_kernel, with its layout: blockIdx.y walks the injectors table[first .. first + n) (one launch group, so no
// two of them write one element), blockIdx.x and the threads the dense points of one, the unit-stride dim fastest; the frame row
// is read contiguously.  Each point belongs to one thread: no atomics.
template <typename T>
__global__ void __launch_bounds__(256) slice_injectors_kernel(const SliceDesc* __restrict__ table, int first, int n, long long t, InjectSel q) {
    for (int r = first + blockIdx.y; r < first + n; r += gridDim.y) {
        const SliceDesc& d = table[r];
        const long long u = t + d.step_off;
        long long row;
        if (!row_due(u, d.t0, d.every, d.nrows, row)) continue;
        const BoxDev b = d.box;
        long long slot = u % d.alloc;
        slot = (slot < 0 ? slot + d.alloc : slot) + d.bias;
        T* __restrict__ dst = reinterpret_cast<T*>(const_cast<char*>(d.var_base) + slot * d.slot_bytes);
        const bool set = d.mode == YB_INJECT_SET;
        with_frame_type<T>(d.ftype, [&](auto tag) {
            using F = decltype(tag);
            const F* __restrict__ src = reinterpret_cast<const F*>(d.frames) + (d.rev ? d.nrows - 1 - row : row) * b.total;
            long long coord[4];
            for (long long i = blockIdx.x * 256ll + threadIdx.x; i < b.total; i += gridDim.x * 256ll) {
                const long long o = box_offset(b, i, coord);
                if (q.sel != PTS_ALL) {
                    bool in = true;
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const long long c = d.loc0[k] + coord[k] * d.lstep[k];
                        in = in && c >= q.ib[k] && c < q.ie[k];
                    }
                    if (in != (q.sel == PTS_INTERIOR)) continue;
                }
                const T f = widen<T>(src[i]);
                dst[o] = set ? f : add_elem(dst[o], f);
            }
        });
    }
}

// the imaging condition's rounding: the product and the sum each rounded, never fused
__device__ __forceinline__ float mul_add_rn(float img, float v, float b) { return __fadd_rn(img, __fmul_rn(v, b)); }
__device__ __forceinline__ double mul_add_rn(double img, double v, double b) { return __dadd_rn(img, __dmul_rn(v, b)); }
// a double image of an fp32 solution: img + double(v) * double(b), the product exact and the sum rounded
__device__ __forceinline__ double mul_add_rn(double img, float v, float b) { return __dadd_rn(img, __dmul_rn(wide_d(v), wide_d(b))); }

// blockIdx.y walks the correlators (each writes only its own image, so all the due ones share a launch).  blockIdx.x and the
// threads walk rows of the unit-stride dim, 2^lanes_log2 threads per row: a row's storage offset is computed once, with the two
// 64-bit divisions that split the row index, and the lanes step along it, so a full-volume correlator reads var, frame and image
// contiguously and stays bound by memory, not by per-point index arithmetic.  Offsets are 64-bit: a slot may hold more than 2^31
// elements.  Var links (b_var) are left to slice_correlators_var_kernel.
template <typename T>
__global__ void __launch_bounds__(256) slice_correlators_kernel(const SliceDesc* __restrict__ table, int n, long long t) {
    for (int r = blockIdx.y; r < n; r += gridDim.y) {
        const SliceDesc& d = table[r];
        const long long u = t + d.step_off;
        long long row;
        if (d.b_var || !row_due(u, d.t0, d.every, d.nrows, row)) continue;
        const BoxDev b = d.box;
        long long slot = u % d.alloc;
        slot = (slot < 0 ? slot + d.alloc : slot) + d.bias;
        const T* __restrict__ var = reinterpret_cast<const T*>(d.var_base + slot * d.slot_bytes) + b.off;
        const int lg = d.lanes_log2, lanes = 1 << lg;
        const long long len = b.n[3], vs = b.vs[3], rows = b.n[0] * b.n[1] * b.n[2], per = 256 >> lg;
        const int lane = threadIdx.x & (lanes - 1);
        // the frame type F (an autocorrelation has no frames: its descriptor names T) and the image type I: T or, in an fp32
        // solution, double
        with_frame_type<T>(d.ftype, [&](auto ftag) {
            using F = decltype(ftag);
            const F* __restrict__ src = d.frames ? reinterpret_cast<const F*>(d.frames) + (d.rev ? d.nrows - 1 - row : row) * b.total : nullptr;
            auto walk = [&](auto itag) {
                using I = decltype(itag);
                I* __restrict__ img = reinterpret_cast<I*>(d.image);
                for (long long q = blockIdx.x * per + (threadIdx.x >> lg); q < rows; q += gridDim.x * per) {
                    const long long q1 = q / b.n[2], c2 = q - q1 * b.n[2];
                    const long long c0 = q1 / b.n[1], c1 = q1 - c0 * b.n[1];
                    const T* __restrict__ vrow = var + c0 * b.vs[0] + c1 * b.vs[1] + c2 * b.vs[2];
                    const long long o = q * len;
                    if (src) {
                        for (long long i = lane; i < len; i += lanes) img[o + i] = mul_add_rn(img[o + i], vrow[i * vs], widen<T>(src[o + i]));
                    } else {
                        for (long long i = lane; i < len; i += lanes) {
                            const T v = vrow[i * vs];
                            img[o + i] = mul_add_rn(img[o + i], v, v);
                        }
                    }
                }
            };
            if (sizeof(T) == 4 && d.itype == YB_TYPE_F64) walk(double{});
            else walk(T{});
        });
    }
}

__device__ __forceinline__ long long slot_at(long long u, int alloc, int bias) {
    const long long c = u % alloc;
    return (c < 0 ? c + alloc : c) + bias;
}

// The var links of the table (b_var): slice_correlators_kernel's row walk, with b read in T from the source var's step slot of
// the paired step through the descriptor's strides, so the source may store its var with other pads, halos and slots.  A kernel
// of its own: the second set of 64-bit row strides does not fit in slice_correlators_kernel's 64 registers.
template <typename T>
__global__ void __launch_bounds__(256) slice_correlators_var_kernel(const SliceDesc* __restrict__ table, int n, long long t) {
    for (int r = blockIdx.y; r < n; r += gridDim.y) {
        const SliceDesc& d = table[r];
        const long long u = t + d.step_off;
        long long row;
        if (!d.b_var || !row_due(u, d.t0, d.every, d.nrows, row)) continue;
        const BoxDev b = d.box;
        const T* __restrict__ var = reinterpret_cast<const T*>(d.var_base + slot_at(u, d.alloc, d.bias) * d.slot_bytes) + b.off;
        const T* __restrict__ src = reinterpret_cast<const T*>(d.b_base + slot_at(u + d.b_shift, d.b_alloc, d.b_bias) * d.b_slot_bytes) + d.b_off;
        const int lg = d.lanes_log2, lanes = 1 << lg;
        const long long len = b.n[3], vs = b.vs[3], bs = d.b_vs[3], rows = b.n[0] * b.n[1] * b.n[2], per = 256 >> lg;
        const int lane = threadIdx.x & (lanes - 1);
        auto walk = [&](auto itag) {
            using I = decltype(itag);
            I* __restrict__ img = reinterpret_cast<I*>(d.image);
            for (long long q = blockIdx.x * per + (threadIdx.x >> lg); q < rows; q += gridDim.x * per) {
                const long long q1 = q / b.n[2], c2 = q - q1 * b.n[2];
                const long long c0 = q1 / b.n[1], c1 = q1 - c0 * b.n[1];
                const T* __restrict__ vrow = var + c0 * b.vs[0] + c1 * b.vs[1] + c2 * b.vs[2];
                const T* __restrict__ brow = src + c0 * d.b_vs[0] + c1 * d.b_vs[1] + c2 * d.b_vs[2];
                const long long o = q * len;
                for (long long i = lane; i < len; i += lanes) img[o + i] = mul_add_rn(img[o + i], vrow[i * vs], brow[i * bs]);
            }
        };
        if (sizeof(T) == 4 && d.itype == YB_TYPE_F64) walk(double{});
        else walk(T{});
    }
}

// The x grid is a grid-stride cap: 8 CTAs per SM is two waves at the 4 CTAs of 256 threads per SM that the kernels' 64 registers
// allow (slice_correlators_var_kernel<float>, at 76, fits 3).  y: the hardware limit of gridDim.y; more recorders are walked by the y loop.
constexpr int CTAS_PER_SM = 8, MAX_GRID_Y = 65535;

// A device buffer freed with cudaFree on its device by its last holder: a recorder's frames outlive the recorder, and its solution,
// while a consumer holds them.
std::shared_ptr<void> device_buffer(void* ptr, int device) {
    return std::shared_ptr<void>(ptr, [device](void* q) {
        int cur = -1;
        const bool had = cudaGetDevice(&cur) == cudaSuccess;
        cudaSetDevice(device);
        cudaFree(q);
        if (had) cudaSetDevice(cur);
    });
}

void release(SliceRec& r) {
    r.frames.reset();
    r.image.reset();
    r.link.reset();
    r.uploaded_bias = -1;
    r.uploaded_base = nullptr;
}

SlicesState* new_state(SliceKind kind) {
    SlicesState* p = new SlicesState();
    p->kind = kind;
    p->what = kind == SLICE_INJECT ? "slice injector" : kind == SLICE_CORRELATE ? "slice correlator" : "slice";
    return p;
}

const char* plural(const SlicesState& p) {
    return p.kind == SLICE_INJECT ? "slice injectors" : p.kind == SLICE_CORRELATE ? "slice correlators" : "slice recorders";
}

bool active(const SlicesState* p) { return p && !p->recs.empty(); }

// A consumer of a recorder's frames against the recorder (FrameLink): the same box and stride, at most its rows, and the same
// owned part of the box on this rank -- the same overall domain, rank grid and rank index -- on the same device.  Each refusal
// names the field that differs.
int check_link(const Solution& s, const SlicesState& p, const SliceRec& r) {
    const FrameLink& l = *r.link;
    const long long id = l.src_id;
    for (int k = 0; k < s.ndd; k++) {
        const char* dn = s.spec.domain_dims[k].c_str();
        if (r.first[k] != l.first[k] || r.last[k] != l.last[k])
            return set_error(YB_EINVAL, "%s: box [%lld, %lld] in dim '%s' differs from recorder %lld's box [%lld, %lld]", p.what, (long long)r.first[k],
                             (long long)r.last[k], dn, id, (long long)l.first[k], (long long)l.last[k]);
        if (r.stride[k] != l.stride[k])
            return set_error(YB_EINVAL, "%s: stride %lld in dim '%s' differs from recorder %lld's stride %lld", p.what, (long long)r.stride[k], dn,
                             id, (long long)l.stride[k]);
    }
    if (r.nrows > l.nrows)
        return set_error(YB_EINVAL, "%s: nrows = %lld is more than the %lld rows of recorder %lld", p.what, (long long)r.nrows, (long long)l.nrows, id);
    if (!geometry_known(s)) return 0;           // checked again at plan_geometry / prepare
    for (int k = 0; k < s.ndd; k++) {
        const char* dn = s.spec.domain_dims[k].c_str();
        if (s.overall_size[k] != l.overall[k])
            return set_error(YB_EINVAL, "%s: overall domain size %lld in dim '%s' differs from the source solution's %lld", p.what,
                             (long long)s.overall_size[k], dn, (long long)l.overall[k]);
        if (s.num_ranks[k] != l.num_ranks[k])
            return set_error(YB_EINVAL, "%s: num_ranks %lld in dim '%s' differs from the source solution's %lld (rank grid)", p.what,
                             (long long)s.num_ranks[k], dn, (long long)l.num_ranks[k]);
        if (s.rank_index[k] != l.rank_index[k])
            return set_error(YB_EINVAL, "%s: rank index %lld in dim '%s' differs from the source solution's %lld", p.what,
                             (long long)s.rank_index[k], dn, (long long)l.rank_index[k]);
        if (r.own_k0[k] != l.own_k0[k] || r.own_n[k] != l.own_n[k])
            return set_error(YB_EINVAL, "%s: owned part (first %lld, count %lld) in dim '%s' differs from recorder %lld's (first %lld, count %lld)",
                             p.what, (long long)r.own_k0[k], (long long)r.own_n[k], dn, id, (long long)l.own_k0[k], (long long)l.own_n[k]);
    }
    if (s.device >= 0 && s.device != l.device)
        return set_error(YB_EINVAL, "%s: device %d differs from the source solution's device %d", p.what, s.device, l.device);
    return 0;
}

// A var link's source against the consumer s, attach checks 3 to 7 of yb_solution_add_slice_correlator_var in their order: element
// bytes, domain dims, then (both with their rank geometry) overall domain, rank grid and rank index, then that src is prepared,
// and on a consumer with a device, the device.  Each refusal names the field that differs.
int check_var_src(const Solution& s, const char* what, const Solution& src) {
    if (src.spec.elem_bytes != s.spec.elem_bytes)
        return set_error(YB_EINVAL, "%s: element bytes %d differ from the source solution's %d", what, s.spec.elem_bytes, src.spec.elem_bytes);
    if (src.ndd != s.ndd)
        return set_error(YB_EINVAL, "%s: %d domain dims differ from the source solution's %d", what, s.ndd, src.ndd);
    for (int k = 0; k < s.ndd; k++)
        if (src.spec.domain_dims[k] != s.spec.domain_dims[k])
            return set_error(YB_EINVAL, "%s: domain dim %d '%s' differs from the source solution's '%s'", what, k, s.spec.domain_dims[k].c_str(),
                             src.spec.domain_dims[k].c_str());
    if (!geometry_known(s)) return set_error(YB_ESTATE, "%s: this solution has no rank geometry yet (plan_geometry / prepare_solution)", what);
    if (!geometry_known(src))
        return set_error(YB_ESTATE, "%s: the source solution has no rank geometry yet (plan_geometry / prepare_solution)", what);
    for (int k = 0; k < s.ndd; k++)
        if (s.overall_size[k] != src.overall_size[k])
            return set_error(YB_EINVAL, "%s: overall domain size %lld in dim '%s' differs from the source solution's %lld", what,
                             (long long)s.overall_size[k], s.spec.domain_dims[k].c_str(), (long long)src.overall_size[k]);
    for (int k = 0; k < s.ndd; k++)
        if (s.num_ranks[k] != src.num_ranks[k])
            return set_error(YB_EINVAL, "%s: num_ranks %lld in dim '%s' differs from the source solution's %lld (rank grid)", what,
                             (long long)s.num_ranks[k], s.spec.domain_dims[k].c_str(), (long long)src.num_ranks[k]);
    for (int k = 0; k < s.ndd; k++)
        if (s.rank_index[k] != src.rank_index[k])
            return set_error(YB_EINVAL, "%s: rank index %lld in dim '%s' differs from the source solution's %lld", what,
                             (long long)s.rank_index[k], s.spec.domain_dims[k].c_str(), (long long)src.rank_index[k]);
    if (!src.prepared)
        return set_error(YB_ESTATE, "%s: the source solution '%s' is not prepared, so its vars have no storage yet", what, src.spec.name.c_str());
    if (s.device >= 0 && s.device != src.device)
        return set_error(YB_EINVAL, "%s: device %d differs from the source solution's device %d", what, s.device, src.device);
    return 0;
}

// A var link at plan and prepare: the source still exists and still passes check_var_src.
int check_var_link(const Solution& s, const SlicesState& p, const SliceRec& r) {
    const FrameLink& l = *r.link;
    if (!l.src)
        return set_error(YB_ESTATE, "%s: the source solution '%s' of var '%s' was destroyed", p.what, l.src_name.c_str(),
                         s.vars[r.var].spec.name.c_str());
    return check_var_src(s, p.what, *l.src);
}

// this rank's part of one recorder, injector or correlator; refuses a box outside the overall domain, on a rank grid an injector
// into a var the last stage does not write (it must land before that stage's exchange, as a source does), and a consumer whose
// part differs from its recorder's (check_link)
int plan_one(const Solution& s, const SlicesState& p, SliceRec& r) {
    const Var& v = s.vars[r.var];
    if (p.kind == SLICE_INJECT && s.multi_rank()) {
        bool last = false;
        for (int o : s.spec.stages.back().outputs) last = last || o == r.var;
        if (!last)
            return set_error(YB_EUNSUPPORTED, "%s: on a rank grid the var '%s' must be written by the last stage of '%s'", p.what,
                             v.spec.name.c_str(), s.spec.name.c_str());
    }
    r.own_off = 0;
    r.own_elems = 1;
    for (int k = 0; k < s.ndd; k++) {
        if (r.first[k] < 0 || r.last[k] >= s.overall_size[k])
            return set_error(YB_ERANGE, "%s: box [%lld, %lld] in dim '%s' is outside the overall domain [0,%lld) (halo and pad cells are refused)",
                             p.what, (long long)r.first[k], (long long)r.last[k], s.spec.domain_dims[k].c_str(), (long long)s.overall_size[k]);
        // owned decimated indices: first + k * stride inside [lo, hi]; the phase comes from the global first
        const int64_t lo = s.rank_offset[k], hi = lo + s.rank_size[k] - 1, st = r.stride[k];
        const int64_t k0 = r.first[k] >= lo ? 0 : (lo - r.first[k] + st - 1) / st;
        const int64_t k1 = hi < r.first[k] ? -1 : std::min(r.count[k] - 1, (hi - r.first[k]) / st);
        r.own_k0[k] = k0;
        r.own_n[k] = std::max<int64_t>(0, k1 - k0 + 1);
        r.own_elems *= r.own_n[k];
        const Dim* d = v.domain_dim(k);
        r.own_off += (r.first[k] + k0 * st - lo + d->pad_l) * d->stride;
    }
    return r.link ? (r.link->var_link ? check_var_link(s, p, r) : check_link(s, p, r)) : 0;
}

// rank-local coordinate of the first owned point in domain dim k (the last one is that + (own_n[k] - 1) * stride[k])
int64_t own_loc0(const Solution& s, const SliceRec& r, int k) { return r.first[k] + r.own_k0[k] * r.stride[k] - s.rank_offset[k]; }

int elem_type(const Solution& s) { return s.spec.elem_bytes == 4 ? YB_TYPE_F32 : YB_TYPE_F64; }

int type_bytes(int type) { return type == YB_TYPE_F64 ? 8 : type == YB_TYPE_F32 ? 4 : 2; }

const char* type_name(int type) {
    return type == YB_TYPE_F64 ? "float64" : type == YB_TYPE_F32 ? "float32" : type == YB_TYPE_F16 ? "float16" : "bfloat16";
}

// The frame type (image = false) or image type of a new recorder, injector or correlator: YB_TYPE_ELEM is the element type;
// otherwise refused unless the table of include/yask_b200.h allows it in this solution.
int resolve_type(const Solution& s, const char* what, int type, bool image, int& out) {
    const int et = elem_type(s);
    const char* field = image ? "image" : "frame";
    if (type == YB_TYPE_ELEM) {
        out = et;
        return 0;
    }
    if (type < YB_TYPE_F64 || type > YB_TYPE_BF16)
        return set_error(YB_EINVAL, "%s: unknown %s type %d (YB_TYPE_ELEM, YB_TYPE_F64, YB_TYPE_F32, YB_TYPE_F16 or YB_TYPE_BF16)", what,
                         field, type);
    const bool ok = image ? type == YB_TYPE_F64 || type == et : et == YB_TYPE_F32 ? type != YB_TYPE_F64 : type == YB_TYPE_F64 || type == YB_TYPE_F32;
    if (!ok)
        return set_error(YB_EINVAL, "%s: %s type %s is not allowed in a solution of element type %s (allowed: %s)", what, field,
                         type_name(type), type_name(et),
                         image ? (et == YB_TYPE_F32 ? "float32, float64" : "float64")
                               : (et == YB_TYPE_F32 ? "float32, float16, bfloat16" : "float64, float32"));
    out = type;
    return 0;
}

// a correlator's threads per row of the unit-stride dim of `len` points: the power of two at or above it, up to the CTA's 256
int lanes_log2(int64_t len) {
    int lg = 0;
    while (lg < 8 && (int64_t(1) << lg) < len) lg++;
    return lg;
}

// the source var of a var link whose source still exists, else null
const Var* link_var(const SliceRec& r) {
    return r.link && r.link->var_link && r.link->src ? &r.link->src->vars[size_t(r.link->src_var)] : nullptr;
}

SliceDesc describe(const Solution& s, const SliceRec& r) {
    const Var& v = s.vars[r.var];
    SliceDesc d{};
    d.var_base = static_cast<const char*>(v.dev);
    d.slot_bytes = (long long)v.slot_elems * v.elem_bytes;
    d.alloc = v.step_alloc();
    d.bias = v.slot_bias;
    d.step_off = r.step_off;
    d.t0 = r.t0; d.every = r.every; d.nrows = r.nrows;
    d.box.nd = s.ndd;
    d.box.off = r.own_off;
    d.box.total = r.own_elems;
    d.mode = r.mode;
    for (int i = 0; i < 4; i++) { d.box.n[i] = 1; d.box.vs[i] = 0; d.loc0[i] = 0; d.lstep[i] = 0; }
    for (int k = 0; k < s.ndd; k++) {
        d.box.n[4 - s.ndd + k] = r.own_n[k];
        d.box.vs[4 - s.ndd + k] = v.domain_dim(k)->stride * r.stride[k];
        d.loc0[4 - s.ndd + k] = own_loc0(s, r, k);
        d.lstep[4 - s.ndd + k] = r.stride[k];
    }
    d.frames = static_cast<char*>(r.frames.get());
    d.image = static_cast<char*>(r.image.get());
    d.rev = r.rev;
    d.lanes_log2 = lanes_log2(d.box.n[3]);
    d.ftype = r.ftype;
    d.itype = r.itype;
    // a var link: b from the source var, with the consumer's rank geometry (check_var_src) but its own pads, strides and slots;
    // none once the source is gone (slices_begin_run then refuses every run)
    if (!r.link || !r.link->var_link) return d;
    d.b_var = 1;
    const Var* bv = link_var(r);
    if (!bv) return d;
    d.b_base = static_cast<const char*>(bv->dev);
    d.b_slot_bytes = (long long)bv->slot_elems * bv->elem_bytes;
    d.b_alloc = bv->step_alloc();
    d.b_bias = bv->slot_bias;
    d.b_shift = r.link->src_shift;
    for (int k = 0; k < s.ndd; k++) {
        const Dim* bd = bv->domain_dim(k);
        d.b_off += (r.first[k] + r.own_k0[k] * r.stride[k] - s.rank_offset[k] + bd->pad_l) * bd->stride;
        d.b_vs[4 - s.ndd + k] = bd->stride * r.stride[k];
    }
    return d;
}

// The owned part of `rows` rows of the whole decimated box as contiguous runs of the last dim: f(element index of the run in
// rows x the whole box, its index in rows x the owned part, length).
template <typename F>
void owned_runs(const Solution& s, const SliceRec& r, int64_t rows, F f) {
    int64_t cnt[3] = {1, 1, 1}, k0[3] = {0, 0, 0}, kn[3] = {1, 1, 1};
    for (int k = 0; k < s.ndd; k++) { cnt[k] = r.count[k]; k0[k] = r.own_k0[k]; kn[k] = r.own_n[k]; }
    size_t dense = 0;
    for (int64_t row = 0; row < rows; row++)
        for (int64_t a = 0; a < kn[0]; a++)
            for (int64_t b = 0; b < kn[1]; b++, dense += size_t(kn[2]))
                f(((size_t(row) * cnt[0] + k0[0] + a) * cnt[1] + k0[1] + b) * cnt[2] + k0[2], dense, size_t(kn[2]));
}

// Recorders: zeroed frames.  Injectors: this rank's part of the caller's frames, after which the host copy is dropped (the
// geometry is fixed once a solution is prepared); one fed from a recorder holds that recorder's frames already.  Correlators: a
// zeroed image of one frame (their source frames, if any, are a recorder's).
int alloc_frames(const Solution& s, const SlicesState& p, SliceRec& r) {
    const bool corr = p.kind == SLICE_CORRELATE;
    std::shared_ptr<void>& buf = corr ? r.image : r.frames;
    const int64_t rows = corr ? 1 : r.nrows;
    const size_t eb = size_t(type_bytes(corr ? r.itype : r.ftype));
    const size_t bytes = size_t(rows) * size_t(r.own_elems) * eb;
    if (buf || (r.link && !corr)) return 0;
    if (!bytes) {
        std::vector<char>().swap(r.host_frames);
        return 0;
    }
    void* d = nullptr;
    cudaError_t e = cudaMalloc(&d, bytes);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        return set_error(YB_ENOMEM, "%s: cannot allocate %zu bytes of %s (%lld rows x %lld owned points) on device %d: %s", p.what, bytes,
                         corr ? "image" : "frames", (long long)rows, (long long)r.own_elems, s.device, cudaGetErrorString(e));
    }
    try {
        buf = device_buffer(d, s.device);
    } catch (const std::exception&) {
        return set_error(YB_ENOMEM, "%s: cannot hold %zu bytes of device memory", p.what, bytes);
    }
    if (p.kind != SLICE_INJECT) {
        YB_CUDA(cudaMemset(d, 0, bytes));
        return 0;
    }
    std::vector<char> dense(bytes);
    owned_runs(s, r, r.nrows, [&](size_t whole, size_t own, size_t n) { memcpy(dense.data() + own * eb, r.host_frames.data() + whole * eb, n * eb); });
    YB_CUDA(cudaMemcpy(d, dense.data(), bytes, cudaMemcpyHostToDevice));
    std::vector<char>().swap(r.host_frames);
    return 0;
}

// (re)write the device table; the caller has synchronized the stream.  The table is reallocated only when recorders were
// added (add_slice, prepare), so the refresh at the start of a run copies and never allocates.
int upload_table(Solution& s, SlicesState& p) {
    std::vector<SliceDesc> t;
    for (auto& r : p.recs) {
        t.push_back(describe(s, r));
        r.uploaded_bias = s.vars[r.var].slot_bias;
        r.uploaded_base = s.vars[r.var].dev;
        if (const Var* bv = link_var(r)) {
            r.uploaded_src_bias = bv->slot_bias;
            r.uploaded_src_base = bv->dev;
        }
    }
    if (t.empty()) return 0;
    YB_CUDA(cudaDeviceGetAttribute(&p.num_sms, cudaDevAttrMultiProcessorCount, s.device));
    if (t.size() > p.table_cap) {
        if (p.d_table) cudaFree(p.d_table);
        p.d_table = nullptr;
        p.table_cap = 0;
        YB_CUDA(cudaMalloc(&p.d_table, t.size() * sizeof(SliceDesc)));
        p.table_cap = t.size();
    }
    YB_CUDA(cudaMemcpy(p.d_table, t.data(), t.size() * sizeof(SliceDesc), cudaMemcpyHostToDevice));
    return 0;
}

// Launch groups of the injectors, in id order: a new group starts at injector j when the bounding box of its decimated box meets
// that of an earlier member of the current group on the same var, so that no two injectors of one launch write one element and
// the later id still applies last.  Global boxes only: every rank forms the same groups.
void plan_groups(SlicesState& p) {
    p.group_first.assign(1, 0);
    for (size_t j = 0; j < p.recs.size(); j++) {
        const SliceRec& b = p.recs[j];
        bool meets = false;
        for (size_t m = size_t(p.group_first.back()); m < j && !meets; m++) {
            const SliceRec& a = p.recs[m];
            meets = a.var == b.var;
            for (int k = 0; k < 3 && meets; k++)
                meets = a.first[k] <= b.first[k] + (b.count[k] - 1) * b.stride[k] && b.first[k] <= a.first[k] + (a.count[k] - 1) * a.stride[k];
        }
        if (meets) p.group_first.push_back(int(j));
    }
    if (!p.recs.empty()) p.group_first.push_back(int(p.recs.size()));
}

int check_mode(const Solution& s, const SlicesState& p) {
    if (fused_pair_rank_grid(s))
        return set_error(YB_EUNSUPPORTED, "%s are not supported on a rank grid in fused-pair mode (block_steps=2 with "
                                          "mega_block_steps=2): its halos are exchanged once per pair of steps, and the state after the first "
                                          "step of a pair is never stored", plural(p));
    return 0;
}

int plan_state(Solution& s, SlicesState* p) {
    if (!active(p)) return 0;
    if (int rc = check_mode(s, *p)) return rc;
    for (auto& r : p->recs)
        if (int rc = plan_one(s, *p, r)) return rc;
    return 0;
}

int prepare_state(Solution& s, SlicesState* p) {
    if (!active(p)) return 0;
    if (int rc = plan_state(s, p)) return rc;
    for (auto& r : p->recs)
        if (int rc = alloc_frames(s, *p, r)) return rc;
    return upload_table(s, *p);
}

// A var link's pairings in a run of steps first .. last: the due steps u of the run form an arithmetic sequence, and so do their
// source steps u + src_shift, so the first and last due steps bound them against the source var's valid window (as the source's
// host calls have enqueued it: the source cannot advance while this run is in flight).  Checked in run order.
int check_pairs(const Solution& s, const SlicesState& p, size_t id, const SliceRec& r, int64_t first, int64_t last) {
    const FrameLink& l = *r.link;
    if (!l.src)
        return set_error(YB_ESTATE, "%s %zu: its source solution '%s' was destroyed; no run is possible until clear_slice_correlators()",
                         p.what, id, l.src_name.c_str());
    const Var& bv = l.src->vars[size_t(l.src_var)];
    const int64_t lo = std::min(first, last) + r.step_off, hi = std::max(first, last) + r.step_off;
    const int64_t k0 = std::max<int64_t>(0, lo - r.t0 <= 0 ? 0 : (lo - r.t0 + r.every - 1) / r.every);
    const int64_t k1 = hi < r.t0 ? -1 : std::min<int64_t>(r.nrows - 1, (hi - r.t0) / r.every);
    if (k0 > k1) return 0;
    const int64_t ua = r.t0 + k0 * r.every, ub = r.t0 + k1 * r.every;
    const int64_t order[2] = {last >= first ? ua : ub, last >= first ? ub : ua};
    for (int64_t u : order) {
        const int64_t w = u + l.src_shift;
        if (w < bv.first_valid_step || w > bv.last_valid_step())
            return set_error(YB_ERANGE, "%s %zu: step %lld pairs with step %lld of var '%s' of the source solution '%s', outside its valid "
                             "steps [%lld, %lld]", p.what, id, (long long)u, (long long)w, bv.spec.name.c_str(), l.src_name.c_str(),
                             (long long)bv.first_valid_step, (long long)bv.last_valid_step());
    }
    return 0;
}

int begin_run_state(Solution& s, SlicesState* p, int64_t first, int64_t last) {
    if (!active(p)) return 0;
    if (int rc = check_mode(s, *p)) return rc;
    bool moved = false;
    for (size_t i = 0; i < p->recs.size(); i++) {
        const SliceRec& r = p->recs[i];
        if (r.link && r.link->var_link)
            if (int rc = check_pairs(s, *p, i, r, first, last)) return rc;
    }
    for (auto& r : p->recs) {
        moved = moved || r.uploaded_bias != s.vars[r.var].slot_bias || r.uploaded_base != s.vars[r.var].dev;
        if (const Var* bv = link_var(r)) moved = moved || r.uploaded_src_bias != bv->slot_bias || r.uploaded_src_base != bv->dev;
    }
    if (!moved) return 0;
    YB_CUDA(cudaStreamSynchronize(s.stream()));
    return upload_table(s, *p);
}

// Does an injecting launch with selection `sel` have any of r's owned points to write?  The owned part's rank-local bounding box
// against the interior box (a stride may step over the interior: then the launch finds nothing, which is harmless).
bool selects(const Solution& s, const SliceRec& r, int sel, const Box& interior) {
    if (sel == PTS_ALL) return true;
    bool inside = true, meets = true;
    for (int k = 0; k < s.ndd; k++) {
        const int64_t lo = own_loc0(s, r, k), hi = lo + (r.own_n[k] - 1) * r.stride[k];
        inside = inside && lo >= interior.b[k] && hi < interior.e[k];
        meets = meets && hi >= interior.b[k] && lo < interior.e[k];
    }
    return sel == PTS_INTERIOR ? meets : !inside;
}

}  // namespace

void slices_free(SlicesState* p) {
    if (!p) return;
    for (auto& r : p->recs) release(r);
    if (p->d_table) cudaFree(p->d_table);
    delete p;
}

FrameLink::~FrameLink() {
    if (!written && !read) return;
    int cur = -1;
    const bool had = cudaGetDevice(&cur) == cudaSuccess;
    cudaSetDevice(device);
    if (written) cudaEventDestroy(written);
    if (read) cudaEventDestroy(read);
    if (had) cudaSetDevice(cur);
}

void slices_preload() {
    preload_kernel((const void*)slices_kernel<float>);
    preload_kernel((const void*)slices_kernel<double>);
    preload_kernel((const void*)slice_injectors_kernel<float>);
    preload_kernel((const void*)slice_injectors_kernel<double>);
    preload_kernel((const void*)slice_correlators_kernel<float>);
    preload_kernel((const void*)slice_correlators_kernel<double>);
    preload_kernel((const void*)slice_correlators_var_kernel<float>);
    preload_kernel((const void*)slice_correlators_var_kernel<double>);
}

bool slices_active(const Solution& s) { return active(s.slices); }

bool slice_injectors_active(const Solution& s) { return active(s.injectors); }

bool slice_correlators_active(const Solution& s) { return active(s.correlators); }

int slices_plan(Solution& s) {
    for (SlicesState* p : {s.slices, s.injectors, s.correlators})
        if (int rc = plan_state(s, p)) return rc;
    return 0;
}

int slices_prepare(Solution& s) {
    for (SlicesState* p : {s.slices, s.injectors, s.correlators})
        if (int rc = prepare_state(s, p)) return rc;
    return 0;
}

int slices_begin_run(Solution& s, int64_t first_step, int64_t last_step) {
    for (SlicesState* p : {s.slices, s.injectors, s.correlators})
        if (int rc = begin_run_state(s, p, first_step, last_step)) return rc;
    return 0;
}

void slices_source_gone(Solution& s) {
    if (s.slices)
        for (const auto& w : s.slices->readers)
            if (auto l = w.lock())
                if (l->var_link) l->src = nullptr;
}

int slices_var_write_waits(Solution& s) {
    if (s.slices)
        for (const auto& w : s.slices->readers)
            if (auto l = w.lock())
                if (l->var_link) YB_CUDA(cudaStreamWaitEvent(s.stream(), l->read, 0));
    return 0;
}

int slices_var_write_records(Solution& s) {
    if (s.slices)
        for (const auto& w : s.slices->readers)
            if (auto l = w.lock())
                if (l->var_link) YB_CUDA(cudaEventRecord(l->written, s.stream()));
    return 0;
}

int slices_run_waits(Solution& s, cudaStream_t st) {
    for (SlicesState* p : {s.injectors, s.correlators})
        if (active(p))
            for (const SliceRec& r : p->recs)
                if (r.link && r.link->written) YB_CUDA(cudaStreamWaitEvent(st, r.link->written, 0));
    if (s.slices)
        for (const auto& w : s.slices->readers)
            if (auto l = w.lock()) YB_CUDA(cudaStreamWaitEvent(st, l->read, 0));
    return 0;
}

int slices_run_records(Solution& s, cudaStream_t st) {
    for (SlicesState* p : {s.injectors, s.correlators})
        if (active(p))
            for (const SliceRec& r : p->recs)
                if (r.link && r.link->read) YB_CUDA(cudaEventRecord(r.link->read, st));
    if (s.slices)
        for (const auto& w : s.slices->readers)
            if (auto l = w.lock()) YB_CUDA(cudaEventRecord(l->written, st));
    return 0;
}

int slices_launch(Solution& s, int64_t t, cudaStream_t st) {
    if (!slices_active(s)) return 0;
    SlicesState& p = *s.slices;
    int64_t most = 0;
    for (auto& r : p.recs) {
        long long row;
        if (r.own_elems && row_due(t + r.step_off, r.t0, r.every, r.nrows, row)) most = std::max(most, r.own_elems);
    }
    if (!most) return 0;
    const dim3 grid(unsigned(std::min<int64_t>((most + 255) / 256, int64_t(p.num_sms) * CTAS_PER_SM)), unsigned(std::min<size_t>(p.recs.size(), MAX_GRID_Y)));
    const SliceDesc* table = static_cast<const SliceDesc*>(p.d_table);
    if (s.spec.elem_bytes == 4) slices_kernel<float><<<grid, 256, 0, st>>>(table, int(p.recs.size()), t);
    else slices_kernel<double><<<grid, 256, 0, st>>>(table, int(p.recs.size()), t);
    YB_CUDA(cudaGetLastError());
    p.launches++;
    return 1;
}

int slice_correlators_launch(Solution& s, int64_t t, cudaStream_t st) {
    if (!slice_correlators_active(s)) return 0;
    SlicesState& p = *s.correlators;
    int64_t most[2] = {0, 0};         // frame and autocorrelation correlators; var links
    for (auto& r : p.recs) {
        long long row;
        if (!r.own_elems || !row_due(t + r.step_off, r.t0, r.every, r.nrows, row)) continue;
        // the CTAs this correlator's rows fill, 256 >> lanes_log2 rows per CTA
        const int64_t len = r.own_n[s.ndd - 1], per = 256 >> lanes_log2(len);
        int64_t& m = most[r.link && r.link->var_link];
        m = std::max(m, (r.own_elems / len + per - 1) / per);
    }
    const SliceDesc* table = static_cast<const SliceDesc*>(p.d_table);
    const int n = int(p.recs.size());
    int launched = 0;
    for (int k = 0; k < 2; k++) {
        if (!most[k]) continue;
        const dim3 grid(unsigned(std::min<int64_t>(most[k], int64_t(p.num_sms) * CTAS_PER_SM)), unsigned(std::min(n, MAX_GRID_Y)));
        if (s.spec.elem_bytes == 4) (k ? slice_correlators_var_kernel<float> : slice_correlators_kernel<float>)<<<grid, 256, 0, st>>>(table, n, t);
        else (k ? slice_correlators_var_kernel<double> : slice_correlators_kernel<double>)<<<grid, 256, 0, st>>>(table, n, t);
        YB_CUDA(cudaGetLastError());
        p.launches++;
        launched++;
    }
    return launched;
}

int slice_injectors_launch(Solution& s, int64_t t, int sel, const Box& interior, cudaStream_t st) {
    if (!slice_injectors_active(s)) return 0;
    SlicesState& p = *s.injectors;
    InjectSel q{};
    q.sel = sel;
    for (int i = 0; i < 4; i++) { q.ib[i] = 0; q.ie[i] = 1; }
    for (int k = 0; k < s.ndd; k++) { q.ib[4 - s.ndd + k] = interior.b[k]; q.ie[4 - s.ndd + k] = interior.e[k]; }
    const SliceDesc* table = static_cast<const SliceDesc*>(p.d_table);
    int launched = 0;
    for (size_t g = 0; g + 1 < p.group_first.size(); g++) {
        const int g0 = p.group_first[g], g1 = p.group_first[g + 1];
        int64_t most = 0;
        for (int j = g0; j < g1; j++) {
            const SliceRec& r = p.recs[size_t(j)];
            long long row;
            if (r.own_elems && row_due(t + r.step_off, r.t0, r.every, r.nrows, row) && selects(s, r, sel, interior)) most = std::max(most, r.own_elems);
        }
        if (!most) continue;
        const dim3 grid(unsigned(std::min<int64_t>((most + 255) / 256, int64_t(p.num_sms) * CTAS_PER_SM)), unsigned(std::min(g1 - g0, MAX_GRID_Y)));
        if (s.spec.elem_bytes == 4) slice_injectors_kernel<float><<<grid, 256, 0, st>>>(table, g0, g1 - g0, t, q);
        else slice_injectors_kernel<double><<<grid, 256, 0, st>>>(table, g0, g1 - g0, t, q);
        YB_CUDA(cudaGetLastError());
        p.launches++;
        launched++;
    }
    return launched;
}

bool slice_injectors_x_range(const Solution& s, int64_t t, int64_t& x0, int64_t& x1) {
    if (!slice_injectors_active(s)) return false;
    bool any = false;
    for (const SliceRec& r : s.injectors->recs) {
        long long row;
        if (!r.own_elems || !row_due(t + r.step_off, r.t0, r.every, r.nrows, row)) continue;
        const int64_t lo = own_loc0(s, r, 0), hi = lo + (r.own_n[0] - 1) * r.stride[0];
        x0 = any ? std::min(x0, lo) : lo;
        x1 = any ? std::max(x1, hi) : hi;
        any = true;
    }
    return any;
}

std::string slice_injector_groups_text(const Solution& s) {
    std::string out;
    if (!slice_injectors_active(s)) return out;
    const std::vector<int>& gf = s.injectors->group_first;
    for (size_t g = 0; g + 1 < gf.size(); g++) {
        if (g) out += ';';
        for (int j = gf[g]; j < gf[g + 1]; j++) out += (j > gf[g] ? "," : "") + std::to_string(j);
    }
    return out;
}

}  // namespace yb

using namespace yb;

#define SOL(s) reinterpret_cast<Solution*>(s)

// The checks shared by recorders and injectors: the var, the box, the window and a 64-bit byte count of the frames of the whole
// box (which bound every rank's share).  Fills r up to the window; `bytes`: nrows x the decimated box in bytes.
static int new_rec(Solution* s, const char* what, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                   int64_t t0, int64_t every, int64_t nrows, int frame_type, SliceRec& r, int64_t& bytes) {
    if (!first || !last) return set_error(YB_EINVAL, "%s: null box", what);
    if (int rc = point_var(*s, what, var, r.var, r.step_off)) return rc;
    if (int rc = resolve_type(*s, what, frame_type, false, r.ftype)) return rc;
    r.itype = elem_type(*s);
    const int fb = type_bytes(r.ftype);
    for (int k = 0; k < s->ndd; k++) {
        const char* dn = s->spec.domain_dims[k].c_str();
        r.first[k] = first[k];
        r.last[k] = last[k];
        r.stride[k] = stride ? stride[k] : 1;
        if (r.first[k] > r.last[k])
            return set_error(YB_EINVAL, "%s: first index %lld is past last index %lld in dim '%s'", what, (long long)r.first[k], (long long)r.last[k], dn);
        if (r.stride[k] < 1) return set_error(YB_EINVAL, "%s: stride %lld in dim '%s' is less than 1", what, (long long)r.stride[k], dn);
        r.count[k] = (r.last[k] - r.first[k]) / r.stride[k] + 1;
    }
    if (every < 1) return set_error(YB_EINVAL, "%s: every = %lld is less than 1", what, (long long)every);
    if (nrows < 1) return set_error(YB_EINVAL, "%s: nrows = %lld is less than 1", what, (long long)nrows);
    int64_t points = 1;
    bool over = false;
    for (int k = 0; k < s->ndd; k++) over = over || __builtin_mul_overflow(points, r.count[k], &points);
    over = over || __builtin_mul_overflow(points, nrows, &bytes) || __builtin_mul_overflow(bytes, int64_t(fb), &bytes);
    if (over)
        return set_error(YB_ERANGE, "%s: %lld rows of the decimated box (%lld x %lld x %lld points) of %d-byte elements overflow a 64-bit "
                         "byte count", what, (long long)nrows, (long long)r.count[0], (long long)r.count[1], (long long)r.count[2], fb);
    r.t0 = t0; r.every = every; r.nrows = nrows;
    return 0;
}

// Append r to *pp (created on first use): planned now when the rank geometry is known; on a prepared solution its frames (a
// correlator's image) are allocated and the table uploaded now too -- never by run_solution() -- after the work that may read the
// old table.
static int install(Solution* s, SlicesState*& pp, SliceKind kind, SliceRec&& r, int64_t* id) {
    if (!pp) pp = new_state(kind);
    SlicesState& p = *pp;
    if (geometry_known(*s)) {
        if (int rc = check_mode(*s, p)) return rc;
        if (int rc = plan_one(*s, p, r)) return rc;
    }
    if (s->prepared) {
        YB_CUDA(cudaSetDevice(s->device));
        YB_CUDA(cudaStreamSynchronize(s->stream()));
        if (int rc = alloc_frames(*s, p, r)) return rc;
        p.recs.push_back(std::move(r));
        if (int rc = upload_table(*s, p)) {
            release(p.recs.back());
            p.recs.pop_back();
            return rc;
        }
    } else {
        p.recs.push_back(std::move(r));
    }
    if (kind == SLICE_INJECT) plan_groups(p);
    if (id) *id = int64_t(p.recs.size()) - 1;
    return 0;
}

// Point r (its box and window filled by new_rec) at the frames of recorder src_id of solution src, read in forward or reversed
// row order.  Every check but the source's frames is made first, so that a planned source shows each refusal; then r holds the
// frames, and when src is another solution, the events that order the two streams (created here: run_solution() allocates
// nothing).
static int attach(Solution* s, SlicesState*& pp, SliceKind kind, SliceRec& r, yb_solution* src_, int64_t src_id, int reverse) {
    if (!pp) pp = new_state(kind);
    const SlicesState& p = *pp;
    if (reverse != 0 && reverse != 1) return set_error(YB_EINVAL, "%s: reverse = %d is not 0 or 1", p.what, reverse);
    r.rev = reverse;
    Solution* src = SOL(src_);
    if (!src) return set_error(YB_EINVAL, "%s: null source solution", p.what);
    if (!slices_active(*src) || src_id < 0 || src_id >= int64_t(src->slices->recs.size()))
        return set_error(YB_EINVAL, "%s: src_id %lld is not a slice recorder of the source solution '%s'", p.what, (long long)src_id,
                         src->spec.name.c_str());
    if (src->spec.elem_bytes != s->spec.elem_bytes)
        return set_error(YB_EINVAL, "%s: element bytes %d differ from the source solution's %d", p.what, s->spec.elem_bytes, src->spec.elem_bytes);
    if (src->ndd != s->ndd)
        return set_error(YB_EINVAL, "%s: %d domain dims differ from the source solution's %d", p.what, s->ndd, src->ndd);
    if (!geometry_known(*s)) return set_error(YB_ESTATE, "%s: this solution has no rank geometry yet (plan_geometry / prepare_solution)", p.what);
    if (!geometry_known(*src))
        return set_error(YB_ESTATE, "%s: the source solution has no rank geometry yet (plan_geometry / prepare_solution)", p.what);
    const SliceRec& q = src->slices->recs[size_t(src_id)];
    auto link = std::make_shared<FrameLink>();
    link->device = src->device;
    link->elem_bytes = src->spec.elem_bytes;
    link->ftype = q.ftype;
    link->ndd = src->ndd;
    link->src_id = src_id;
    link->nrows = q.nrows;
    for (int k = 0; k < 3; k++) {
        link->first[k] = q.first[k]; link->last[k] = q.last[k]; link->stride[k] = q.stride[k];
        link->overall[k] = src->overall_size[k]; link->num_ranks[k] = src->num_ranks[k]; link->rank_index[k] = src->rank_index[k];
        link->own_k0[k] = q.own_k0[k]; link->own_n[k] = q.own_n[k];
    }
    r.link = link;
    r.ftype = link->ftype;
    if (int rc = check_mode(*s, p)) return rc;
    if (int rc = plan_one(*s, p, r)) return rc;
    if (!src->prepared)
        return set_error(YB_ESTATE, "%s: the source solution '%s' is not prepared, so recorder %lld has no frames yet", p.what,
                         src->spec.name.c_str(), (long long)src_id);
    r.frames = q.frames;
    if (src == s) return 0;                     // one stream
    YB_CUDA(cudaSetDevice(src->device));
    YB_CUDA(cudaEventCreateWithFlags(&link->written, cudaEventDisableTiming));
    YB_CUDA(cudaEventCreateWithFlags(&link->read, cudaEventDisableTiming));
    YB_CUDA(cudaEventRecord(link->written, src->stream()));     // the source's runs enqueued so far
    auto& readers = src->slices->readers;
    readers.erase(std::remove_if(readers.begin(), readers.end(), [](const std::weak_ptr<FrameLink>& w) { return w.expired(); }), readers.end());
    readers.push_back(link);
    return 0;
}

static int clear_state(Solution* s, SlicesState*& p, SliceKind kind) {
    if (!p) return 0;
    if (s->prepared) {
        YB_CUDA(cudaSetDevice(s->device));
        YB_CUDA(cudaStreamSynchronize(s->stream()));
    }
    const int64_t launches = p->launches;
    // the var links of consumers of this solution's vars stay ordered against its runs
    std::vector<std::weak_ptr<FrameLink>> keep;
    for (const auto& w : p->readers)
        if (auto l = w.lock())
            if (l->var_link) keep.push_back(w);
    slices_free(p);
    p = new_state(kind);
    p->launches = launches;
    p->readers = std::move(keep);
    return 0;
}

// `rows` rows of the whole decimated box of r into out from `dev` (rows x this rank's part; null when nothing was allocated), 0
// where this rank owns no point, and the owned mask.  `out` may be null: the mask only, which needs no device.
static int copy_out(Solution* s, const SliceRec& r, const void* dev, int64_t rows, int type, void* out, uint8_t* owned) {
    size_t box = 1;
    for (int k = 0; k < s->ndd; k++) box *= size_t(r.count[k]);
    if (owned) {
        memset(owned, 0, box);
        owned_runs(*s, r, 1, [&](size_t whole, size_t, size_t n) { memset(owned + whole, 1, n); });
    }
    if (!out) return 0;
    const size_t eb = size_t(type_bytes(type));
    memset(out, 0, size_t(rows) * box * eb);
    if (!dev) return 0;
    std::vector<char> dense(size_t(rows) * size_t(r.own_elems) * eb);
    YB_CUDA(cudaSetDevice(s->device));
    YB_CUDA(cudaMemcpyAsync(dense.data(), dev, dense.size(), cudaMemcpyDeviceToHost, s->stream()));
    YB_CUDA(cudaStreamSynchronize(s->stream()));
    owned_runs(*s, r, rows, [&](size_t whole, size_t own, size_t n) { memcpy(static_cast<char*>(out) + whole * eb, dense.data() + own * eb, n * eb); });
    return 0;
}

extern "C" {

int yb_solution_add_slice_typed(yb_solution* s_, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                int64_t t0, int64_t every, int64_t nrows, int frame_type, int64_t* id) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    SliceRec r;
    int64_t bytes = 0;
    if (int rc = new_rec(s, "slice", var, first, last, stride, t0, every, nrows, frame_type, r, bytes)) return rc;
    return install(s, s->slices, SLICE_RECORD, std::move(r), id);
}

int yb_solution_add_slice(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                          int64_t t0, int64_t every, int64_t nrows, int64_t* id) {
    return yb_solution_add_slice_typed(s, var, first, last, stride, t0, every, nrows, YB_TYPE_ELEM, id);
}

int yb_solution_add_slice_injector_typed(yb_solution* s_, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                         int64_t t0, int64_t every, int64_t nrows, int mode, int frame_type, const void* frames, int64_t* id) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    const char* what = "slice injector";
    SliceRec r;
    int64_t bytes = 0;
    if (int rc = new_rec(s, what, var, first, last, stride, t0, every, nrows, frame_type, r, bytes)) return rc;
    if (mode != YB_INJECT_ADD && mode != YB_INJECT_SET)
        return set_error(YB_EINVAL, "%s: unknown mode %d (YB_INJECT_ADD = %d or YB_INJECT_SET = %d)", what, mode, YB_INJECT_ADD, YB_INJECT_SET);
    if (!frames) return set_error(YB_EINVAL, "%s: null frames", what);
    r.mode = mode;
    try {
        r.host_frames.assign(static_cast<const char*>(frames), static_cast<const char*>(frames) + bytes);
    } catch (const std::exception&) {
        return set_error(YB_ENOMEM, "%s: cannot copy %lld bytes of frames on the host", what, (long long)bytes);
    }
    return install(s, s->injectors, SLICE_INJECT, std::move(r), id);
}

int yb_solution_add_slice_injector(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                   int64_t t0, int64_t every, int64_t nrows, int mode, const void* frames, int64_t* id) {
    return yb_solution_add_slice_injector_typed(s, var, first, last, stride, t0, every, nrows, mode, YB_TYPE_ELEM, frames, id);
}

int yb_solution_add_slice_injector_from(yb_solution* s_, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                        int64_t t0, int64_t every, int64_t nrows, int mode, yb_solution* src, int64_t src_id, int reverse,
                                        int64_t* id) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    const char* what = "slice injector";
    SliceRec r;
    int64_t bytes = 0;
    if (int rc = new_rec(s, what, var, first, last, stride, t0, every, nrows, YB_TYPE_ELEM, r, bytes)) return rc;
    if (mode != YB_INJECT_ADD && mode != YB_INJECT_SET)
        return set_error(YB_EINVAL, "%s: unknown mode %d (YB_INJECT_ADD = %d or YB_INJECT_SET = %d)", what, mode, YB_INJECT_ADD, YB_INJECT_SET);
    r.mode = mode;
    if (int rc = attach(s, s->injectors, SLICE_INJECT, r, src, src_id, reverse)) return rc;
    return install(s, s->injectors, SLICE_INJECT, std::move(r), id);
}

int yb_solution_add_slice_correlator_typed(yb_solution* s_, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                           int64_t t0, int64_t every, int64_t nrows, yb_solution* src, int64_t src_id, int reverse,
                                           int image_type, int64_t* id) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    const char* what = "slice correlator";
    SliceRec r;
    int64_t bytes = 0;
    if (int rc = new_rec(s, what, var, first, last, stride, t0, every, nrows, YB_TYPE_ELEM, r, bytes)) return rc;
    if (int rc = resolve_type(*s, what, image_type, true, r.itype)) return rc;
    if (src) {
        if (int rc = attach(s, s->correlators, SLICE_CORRELATE, r, src, src_id, reverse)) return rc;
    } else if (reverse != 0 && reverse != 1) {
        return set_error(YB_EINVAL, "slice correlator: reverse = %d is not 0 or 1", reverse);
    }
    return install(s, s->correlators, SLICE_CORRELATE, std::move(r), id);
}

int yb_solution_add_slice_correlator(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                     int64_t t0, int64_t every, int64_t nrows, yb_solution* src, int64_t src_id, int reverse, int64_t* id) {
    return yb_solution_add_slice_correlator_typed(s, var, first, last, stride, t0, every, nrows, src, src_id, reverse, YB_TYPE_ELEM, id);
}

int yb_solution_add_slice_correlator_var(yb_solution* s_, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                         int64_t t0, int64_t every, int64_t nrows, yb_solution* src_, const char* src_var, int64_t src_t0,
                                         int image_type, int64_t* id) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    const char* what = "slice correlator";
    SliceRec r;
    int64_t bytes = 0;
    if (int rc = new_rec(s, what, var, first, last, stride, t0, every, nrows, YB_TYPE_ELEM, r, bytes)) return rc;
    if (int rc = resolve_type(*s, what, image_type, true, r.itype)) return rc;
    Solution* src = SOL(src_);
    if (!src) return set_error(YB_EINVAL, "%s: src: null source solution", what);
    if (src == s) return set_error(YB_EINVAL, "%s: src: the source solution must be another solution, not this one", what);
    int src_vi = -1, src_off = 0;
    if (int rc = point_var(*src, "slice correlator: src_var", src_var, src_vi, src_off)) return rc;
    if (!s->correlators) s->correlators = new_state(SLICE_CORRELATE);
    if (int rc = check_mode(*s, *s->correlators)) return rc;
    if (int rc = check_var_src(*s, what, *src)) return rc;
    auto link = std::make_shared<FrameLink>();
    link->device = src->device;
    link->elem_bytes = src->spec.elem_bytes;
    link->ndd = src->ndd;
    link->var_link = true;
    link->src = src;
    link->src_var = src_vi;
    link->src_shift = src_t0 - t0;
    link->src_name = src->spec.name;
    r.link = link;
    if (int rc = plan_one(*s, *s->correlators, r)) return rc;
    // the events that order the two streams, created here (run_solution() allocates nothing)
    YB_CUDA(cudaSetDevice(src->device));
    YB_CUDA(cudaEventCreateWithFlags(&link->written, cudaEventDisableTiming));
    YB_CUDA(cudaEventCreateWithFlags(&link->read, cudaEventDisableTiming));
    YB_CUDA(cudaEventRecord(link->written, src->stream()));     // the source's work enqueued so far
    if (!src->slices) src->slices = new_state(SLICE_RECORD);    // holds the readers even with no recorder
    auto& readers = src->slices->readers;
    readers.erase(std::remove_if(readers.begin(), readers.end(), [](const std::weak_ptr<FrameLink>& w) { return w.expired(); }), readers.end());
    readers.push_back(link);
    return install(s, s->correlators, SLICE_CORRELATE, std::move(r), id);
}

int yb_solution_get_slice_frame_type(yb_solution* s_, int64_t id, int* type) {
    Solution* s = SOL(s_);
    if (!s || !type) return set_error(YB_EINVAL, "null solution or type");
    if (!slices_active(*s) || id < 0 || id >= int64_t(s->slices->recs.size()))
        return set_error(YB_EINVAL, "get_slice_frame_type: no slice recorder %lld", (long long)id);
    *type = s->slices->recs[size_t(id)].ftype;
    return 0;
}

int yb_solution_get_correlator_image_type(yb_solution* s_, int64_t id, int* type) {
    Solution* s = SOL(s_);
    if (!s || !type) return set_error(YB_EINVAL, "null solution or type");
    if (!slice_correlators_active(*s) || id < 0 || id >= int64_t(s->correlators->recs.size()))
        return set_error(YB_EINVAL, "get_correlator_image_type: no slice correlator %lld", (long long)id);
    *type = s->correlators->recs[size_t(id)].itype;
    return 0;
}

int yb_solution_get_slice_frames(yb_solution* s_, int64_t id, void* out, uint8_t* owned) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (!slices_active(*s) || id < 0 || id >= int64_t(s->slices->recs.size()))
        return set_error(YB_EINVAL, "get_slice_frames: no slice recorder %lld", (long long)id);
    if (!geometry_known(*s)) return set_error(YB_ESTATE, "get_slice_frames: the rank geometry is not known yet (plan_geometry / prepare_solution)");
    SliceRec& r = s->slices->recs[size_t(id)];
    if (!s->prepared)
        if (int rc = plan_one(*s, *s->slices, r)) return rc;
    return copy_out(s, r, r.frames.get(), r.nrows, r.ftype, out, owned);
}

int yb_solution_get_correlator_image(yb_solution* s_, int64_t id, void* out, uint8_t* owned) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (!slice_correlators_active(*s) || id < 0 || id >= int64_t(s->correlators->recs.size()))
        return set_error(YB_EINVAL, "get_correlator_image: no slice correlator %lld", (long long)id);
    if (!geometry_known(*s)) return set_error(YB_ESTATE, "get_correlator_image: the rank geometry is not known yet (plan_geometry / prepare_solution)");
    SliceRec& r = s->correlators->recs[size_t(id)];
    if (!s->prepared)
        if (int rc = plan_one(*s, *s->correlators, r)) return rc;
    return copy_out(s, r, r.image.get(), 1, r.itype, out, owned);
}

int yb_solution_clear_slices(yb_solution* s_) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    return clear_state(s, s->slices, SLICE_RECORD);
}

int yb_solution_clear_slice_injectors(yb_solution* s_) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    return clear_state(s, s->injectors, SLICE_INJECT);
}

int yb_solution_clear_slice_correlators(yb_solution* s_) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    return clear_state(s, s->correlators, SLICE_CORRELATE);
}

}  // extern "C"
