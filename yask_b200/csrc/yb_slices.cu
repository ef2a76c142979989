// Slice recorders on the device (yb_slices.h): receiver planes, decimated snapshots and field dumps every k steps, recorded
// inside run_solution() by one many-CTA launch per step, instead of the reference API loop run_solution(t, t) /
// get_elements_in_slice, which pays a synchronous device-to-host copy per frame and loses the temporal tile's pairs.
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
    char* frames;                   // nrows x box.total elements
};

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
        T* __restrict__ dst = reinterpret_cast<T*>(d.frames) + row * b.total;
        long long coord[4];
        for (long long i = blockIdx.x * 256ll + threadIdx.x; i < b.total; i += gridDim.x * 256ll) dst[i] = src[box_offset(b, i, coord)];
    }
}

// The x grid is a grid-stride cap: 8 CTAs per SM is two waves at the 4 CTAs of 256 threads per SM that the kernel's 56
// registers allow.  y: the hardware limit of gridDim.y; more recorders are walked by the y loop.
constexpr int CTAS_PER_SM = 8, MAX_GRID_Y = 65535;

const char* const WHAT = "slice";

void release(SliceRec& r) {
    if (r.d_frames) cudaFree(r.d_frames);
    r.d_frames = nullptr;
    r.uploaded_bias = -1;
    r.uploaded_base = nullptr;
}

// this rank's part of one recorder; refuses a box outside the overall domain
int plan_one(const Solution& s, SliceRec& r) {
    const Var& v = s.vars[r.var];
    r.own_off = 0;
    r.own_elems = 1;
    for (int k = 0; k < s.ndd; k++) {
        if (r.first[k] < 0 || r.last[k] >= s.overall_size[k])
            return set_error(YB_ERANGE, "%s: box [%lld, %lld] in dim '%s' is outside the overall domain [0,%lld) (halo and pad cells are refused)",
                             WHAT, (long long)r.first[k], (long long)r.last[k], s.spec.domain_dims[k].c_str(), (long long)s.overall_size[k]);
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
    return 0;
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
    for (int i = 0; i < 4; i++) { d.box.n[i] = 1; d.box.vs[i] = 0; }
    for (int k = 0; k < s.ndd; k++) {
        d.box.n[4 - s.ndd + k] = r.own_n[k];
        d.box.vs[4 - s.ndd + k] = v.domain_dim(k)->stride * r.stride[k];
    }
    d.frames = static_cast<char*>(r.d_frames);
    return d;
}

size_t frame_bytes(const Solution& s, const SliceRec& r) { return size_t(r.nrows) * size_t(r.own_elems) * s.spec.elem_bytes; }

int alloc_frames(const Solution& s, SliceRec& r) {
    const size_t bytes = frame_bytes(s, r);
    if (!bytes || r.d_frames) return 0;
    cudaError_t e = cudaMalloc(&r.d_frames, bytes);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        r.d_frames = nullptr;
        return set_error(YB_ENOMEM, "%s: cannot allocate %zu bytes of frames (%lld rows x %lld owned points) on device %d: %s", WHAT, bytes,
                         (long long)r.nrows, (long long)r.own_elems, s.device, cudaGetErrorString(e));
    }
    YB_CUDA(cudaMemset(r.d_frames, 0, bytes));
    return 0;
}

// (re)write the device table; the caller has synchronized the stream.  The table is reallocated only when recorders were
// added (add_slice, prepare), so the refresh at the start of a run copies and never allocates.
int upload_table(Solution& s) {
    SlicesState& p = *s.slices;
    std::vector<SliceDesc> t;
    for (auto& r : p.recs) {
        t.push_back(describe(s, r));
        r.uploaded_bias = s.vars[r.var].slot_bias;
        r.uploaded_base = s.vars[r.var].dev;
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

}  // namespace

void slices_free(SlicesState* p) {
    if (!p) return;
    for (auto& r : p->recs) release(r);
    if (p->d_table) cudaFree(p->d_table);
    delete p;
}

void slices_preload() {
    preload_kernel((const void*)slices_kernel<float>);
    preload_kernel((const void*)slices_kernel<double>);
}

bool slices_active(const Solution& s) { return s.slices && !s.slices->recs.empty(); }

static int check_mode(const Solution& s) {
    if (fused_pair_rank_grid(s))
        return set_error(YB_EUNSUPPORTED, "slice recorders are not supported on a rank grid in fused-pair mode (block_steps=2 with "
                                          "mega_block_steps=2): its halos are exchanged once per pair of steps, and the state after the first "
                                          "step of a pair is never stored");
    return 0;
}

int slices_plan(Solution& s) {
    if (!slices_active(s)) return 0;
    if (int rc = check_mode(s)) return rc;
    for (auto& r : s.slices->recs)
        if (int rc = plan_one(s, r)) return rc;
    return 0;
}

int slices_prepare(Solution& s) {
    if (!slices_active(s)) return 0;
    if (int rc = slices_plan(s)) return rc;
    for (auto& r : s.slices->recs)
        if (int rc = alloc_frames(s, r)) return rc;
    return upload_table(s);
}

int slices_begin_run(Solution& s) {
    if (!slices_active(s)) return 0;
    if (int rc = check_mode(s)) return rc;
    bool moved = false;
    for (auto& r : s.slices->recs) moved = moved || r.uploaded_bias != s.vars[r.var].slot_bias || r.uploaded_base != s.vars[r.var].dev;
    if (!moved) return 0;
    YB_CUDA(cudaStreamSynchronize(s.stream()));
    return upload_table(s);
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

}  // namespace yb

using namespace yb;

extern "C" {

#define SOL(s) reinterpret_cast<Solution*>(s)

int yb_solution_add_slice(yb_solution* s_, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                          int64_t t0, int64_t every, int64_t nrows, int64_t* id) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (!first || !last) return set_error(YB_EINVAL, "%s: null box", WHAT);
    SliceRec r;
    if (int rc = point_var(*s, WHAT, var, r.var, r.step_off)) return rc;
    for (int k = 0; k < s->ndd; k++) {
        const char* dn = s->spec.domain_dims[k].c_str();
        r.first[k] = first[k];
        r.last[k] = last[k];
        r.stride[k] = stride ? stride[k] : 1;
        if (r.first[k] > r.last[k])
            return set_error(YB_EINVAL, "%s: first index %lld is past last index %lld in dim '%s'", WHAT, (long long)r.first[k], (long long)r.last[k], dn);
        if (r.stride[k] < 1) return set_error(YB_EINVAL, "%s: stride %lld in dim '%s' is less than 1", WHAT, (long long)r.stride[k], dn);
        r.count[k] = (r.last[k] - r.first[k]) / r.stride[k] + 1;
    }
    if (every < 1) return set_error(YB_EINVAL, "%s: every = %lld is less than 1", WHAT, (long long)every);
    if (nrows < 1) return set_error(YB_EINVAL, "%s: nrows = %lld is less than 1", WHAT, (long long)nrows);
    // the frames of the whole box, which bound every rank's share, must be addressable (byte counts and row offsets)
    int64_t points = 1, bytes = 0;
    bool over = false;
    for (int k = 0; k < s->ndd; k++) over = over || __builtin_mul_overflow(points, r.count[k], &points);
    over = over || __builtin_mul_overflow(points, nrows, &bytes) || __builtin_mul_overflow(bytes, int64_t(s->spec.elem_bytes), &bytes);
    if (over)
        return set_error(YB_ERANGE, "%s: %lld rows of the decimated box (%lld x %lld x %lld points) of %d-byte elements overflow a 64-bit "
                         "byte count", WHAT, (long long)nrows, (long long)r.count[0], (long long)r.count[1], (long long)r.count[2],
                         s->spec.elem_bytes);
    r.t0 = t0; r.every = every; r.nrows = nrows;
    if (geometry_known(*s)) {
        if (int rc = check_mode(*s)) return rc;
        if (int rc = plan_one(*s, r)) return rc;
    }
    if (!s->slices) s->slices = new SlicesState();
    SlicesState& p = *s->slices;
    if (s->prepared) {
        // frames are allocated here or at prepare, never by run_solution(); the table in use may still be read by queued work
        YB_CUDA(cudaSetDevice(s->device));
        YB_CUDA(cudaStreamSynchronize(s->stream()));
        if (int rc = alloc_frames(*s, r)) return rc;
        p.recs.push_back(r);
        if (int rc = upload_table(*s)) {
            release(p.recs.back());
            p.recs.pop_back();
            return rc;
        }
    } else {
        p.recs.push_back(r);
    }
    if (id) *id = int64_t(p.recs.size()) - 1;
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
        if (int rc = plan_one(*s, r)) return rc;
    const int nd = s->ndd;
    int64_t cnt[3] = {1, 1, 1}, k0[3] = {0, 0, 0}, kn[3] = {1, 1, 1};
    for (int k = 0; k < nd; k++) { cnt[k] = r.count[k]; k0[k] = r.own_k0[k]; kn[k] = r.own_n[k]; }
    const size_t box = size_t(cnt[0] * cnt[1] * cnt[2]);
    if (owned) {
        memset(owned, 0, box);
        for (int64_t a = 0; a < kn[0]; a++)
            for (int64_t b = 0; b < kn[1]; b++)
                memset(owned + ((k0[0] + a) * cnt[1] + k0[1] + b) * cnt[2] + k0[2], 1, size_t(kn[2]));
    }
    if (!out) return 0;
    const size_t eb = size_t(s->spec.elem_bytes);
    memset(out, 0, size_t(r.nrows) * box * eb);
    if (!r.d_frames) return 0;
    std::vector<char> dense(frame_bytes(*s, r));
    YB_CUDA(cudaSetDevice(s->device));
    YB_CUDA(cudaMemcpyAsync(dense.data(), r.d_frames, dense.size(), cudaMemcpyDeviceToHost, s->stream()));
    YB_CUDA(cudaStreamSynchronize(s->stream()));
    const char* src = dense.data();
    for (int64_t row = 0; row < r.nrows; row++)
        for (int64_t a = 0; a < kn[0]; a++)
            for (int64_t b = 0; b < kn[1]; b++, src += size_t(kn[2]) * eb)
                memcpy(static_cast<char*>(out) + ((size_t(row) * cnt[0] + k0[0] + a) * cnt[1] + k0[1] + b) * cnt[2] * eb + size_t(k0[2]) * eb, src,
                       size_t(kn[2]) * eb);
    return 0;
}

int yb_solution_clear_slices(yb_solution* s_) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (!s->slices) return 0;
    if (s->prepared) {
        YB_CUDA(cudaSetDevice(s->device));
        YB_CUDA(cudaStreamSynchronize(s->stream()));
    }
    const int64_t launches = s->slices->launches;
    slices_free(s->slices);
    s->slices = new SlicesState();
    s->slices->launches = launches;
    return 0;
}

}  // extern "C"
