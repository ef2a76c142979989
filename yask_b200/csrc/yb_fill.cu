// Device-side data movement helpers: strided-box <-> dense-buffer copies (the engine's
// equivalent of YkVarBase::get/set_elements_in_slice, /root/reference/src/kernel/lib/yk_var.hpp:1222-1300),
// constant fills (set_all_elements_same, yk_var.hpp:1786-1793), the synthetic hash-field
// generator (yask_b200/synth.py) and an order-independent checksum.
#include "yb_box.cuh"
#include "yb_core.h"

namespace yb {

namespace {

__host__ BoxDev to_dev(const BoxCopy& bc) {
    BoxDev b;
    b.nd = bc.nd;
    b.total = 1;
    for (int i = 0; i < 4; i++) {
        b.n[i] = i < bc.nd ? bc.n[i] : 1;
        b.vs[i] = i < bc.nd ? bc.var_stride[i] : 0;
        b.total *= b.n[i];
    }
    b.off = bc.var_off;
    return b;
}

template <typename T>
__global__ void box_copy_kernel(T* __restrict__ var, T* __restrict__ dense, BoxDev b, bool to_var) {
    long long coord[4];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < b.total; i += (long long)gridDim.x * blockDim.x) {
        long long o = box_offset(b, i, coord);
        if (to_var) var[o] = dense[i];
        else dense[i] = var[o];
    }
}

template <typename T>
__global__ void box_fill_kernel(T* __restrict__ var, BoxDev b, T value) {
    long long coord[4];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < b.total; i += (long long)gridDim.x * blockDim.x)
        var[box_offset(b, i, coord)] = value;
}

template <typename T>
__global__ void fill_all_kernel(T* __restrict__ p, long long n, T value) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = value;
}

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
    x += 0x9E3779B97F4A7C15ull;
    x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 27; x *= 0x94D049BB133111EBull;
    x ^= x >> 31;
    return x;
}

// key of a global index triple; must match yask_b200/synth.py::hash_field
__device__ __forceinline__ unsigned long long index_key(long long i0, long long i1, long long i2) {
    const unsigned long long OFF = 1ull << 19, M = 0xFFFFFull;
    return (((unsigned long long)i0 + OFF) & M) << 40 | (((unsigned long long)i1 + OFF) & M) << 20 | (((unsigned long long)i2 + OFF) & M);
}

struct G0 { long long g[3]; long long lead; };   // lead: global index of the 4th (outermost) dim, if any

// global index triple of box coordinate `coord` (box has nd <= 3 dims, left-padded with index 0)
__device__ __forceinline__ void global_triple(const BoxDev& b, const G0& g0, const long long* coord, long long* g) {
    g[0] = g[1] = g[2] = 0;
    // box dims occupy the LAST nd positions of coord[4]; map them to the last nd of the triple
    for (int k = 0; k < b.nd && k < 3; k++) {
        int cd = 3 - k;          // coord index (from the end)
        int gd = 2 - k;          // triple index (from the end)
        g[gd] = g0.g[gd] + coord[cd];
    }
}

template <typename T>
__global__ void hash_fill_kernel(T* __restrict__ var, BoxDev b, G0 g0, unsigned long long seedsalt, double lo, double hi) {
    long long coord[4], g[3];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < b.total; i += (long long)gridDim.x * blockDim.x) {
        long long o = box_offset(b, i, coord);
        global_triple(b, g0, coord, g);
        unsigned long long ss = seedsalt;
        if (b.nd == 4) {   // 4-D var: the leading index perturbs the salt (yask_b200/synth.py::hash_field)
            const unsigned long long salt = (seedsalt + (unsigned long long)(g0.lead + coord[0]) * 0x9E3779B1ull) & 0xFFFFFFFFull;
            ss = (seedsalt & 0xFFFFFFFF00000000ull) | salt;
        }
        unsigned long long key = index_key(g[0], g[1], g[2]) ^ (ss * 0xD6E8FEB86659FD93ull);
        unsigned long long h = splitmix64(key);
        double u = __dmul_rn((double)(h >> 40), 1.0 / 16777216.0);
        double val = __dadd_rn(lo, __dmul_rn(hi - lo, u));
        var[o] = (T)val;
    }
}

template <typename T>
__global__ void checksum_kernel(const T* __restrict__ var, BoxDev b, G0 g0, unsigned long long* out) {
    long long coord[4], g[3];
    unsigned long long acc = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < b.total; i += (long long)gridDim.x * blockDim.x) {
        long long o = box_offset(b, i, coord);
        global_triple(b, g0, coord, g);
        unsigned long long bits;
        if (sizeof(T) == 4) bits = (unsigned long long)__float_as_uint((float)var[o]);
        else bits = (unsigned long long)__double_as_longlong((double)var[o]);
        acc += splitmix64(index_key(g[0], g[1], g[2]) ^ (bits * 0x9E3779B97F4A7C15ull));
    }
    for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
    if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}

// ---- reductions over a strided box (yk_var::reduce_elements_in_slice, aux/yk_var_api.hpp:984-1048, 1050-1110) --------
// All five results are accumulated in double, in a FIXED order (grid-stride per thread, shuffle tree per warp,
// warp 0 over the warps, one final block over the per-block partials), so a given box always reduces to the same bits.
__device__ __forceinline__ void red_init(RedVals& r) {
    r.sum = 0.0; r.sumsq = 0.0; r.prod = 1.0;
    r.mx = -__longlong_as_double(0x7ff0000000000000ll);
    r.mn = __longlong_as_double(0x7ff0000000000000ll);
}
__device__ __forceinline__ void red_merge(RedVals& a, const RedVals& b) {
    a.sum += b.sum; a.sumsq += b.sumsq; a.prod *= b.prod;
    a.mx = fmax(a.mx, b.mx); a.mn = fmin(a.mn, b.mn);
}
__device__ __forceinline__ RedVals red_shfl(const RedVals& r, int delta) {
    RedVals o;
    o.sum = __shfl_down_sync(0xffffffffu, r.sum, delta);
    o.sumsq = __shfl_down_sync(0xffffffffu, r.sumsq, delta);
    o.prod = __shfl_down_sync(0xffffffffu, r.prod, delta);
    o.mx = __shfl_down_sync(0xffffffffu, r.mx, delta);
    o.mn = __shfl_down_sync(0xffffffffu, r.mn, delta);
    return o;
}
// block-wide merge; the result is valid in thread 0
__device__ __forceinline__ void red_block(RedVals& r) {
    __shared__ RedVals wsum[8];
    for (int d = 16; d > 0; d >>= 1) { RedVals o = red_shfl(r, d); red_merge(r, o); }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) wsum[w] = r;
    __syncthreads();
    if (w == 0) {
        RedVals t;
        red_init(t);
        if (threadIdx.x < (blockDim.x >> 5)) t = wsum[threadIdx.x];
        for (int d = 4; d > 0; d >>= 1) { RedVals o = red_shfl(t, d); red_merge(t, o); }
        r = t;
    }
}
template <typename T>
__global__ void __launch_bounds__(256) box_reduce_kernel(const T* __restrict__ var, BoxDev b, RedVals* __restrict__ partial) {
    long long coord[4];
    RedVals r;
    red_init(r);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < b.total; i += (long long)gridDim.x * blockDim.x) {
        const double v = (double)var[box_offset(b, i, coord)];
        r.sum += v; r.sumsq += v * v; r.prod *= v;
        r.mx = fmax(r.mx, v); r.mn = fmin(r.mn, v);
    }
    red_block(r);
    if (threadIdx.x == 0) partial[blockIdx.x] = r;
}
__global__ void __launch_bounds__(256) reduce_final_kernel(const RedVals* __restrict__ partial, int n, RedVals* __restrict__ out) {
    RedVals r;
    red_init(r);
    for (int i = threadIdx.x; i < n; i += blockDim.x) red_merge(r, partial[i]);
    red_block(r);
    if (threadIdx.x == 0) *out = r;
}

// Grid cap of the grid-stride kernels, a constant rather than a multiple of the SM count: the reduction's partition into
// per-block partial sums, and so the rounding of its result, is then the same on every device.
constexpr int MAX_GRID = 2368;

int grid_for(long long total) {
    long long g = (total + 255) / 256;
    if (g > MAX_GRID) g = MAX_GRID;
    if (g < 1) g = 1;
    return int(g);
}

// The dense box has its dims right-aligned in a 4-entry array so that coord[3] is unit stride.
BoxDev right_align(const BoxCopy& bc) {
    BoxCopy r{};
    r.nd = bc.nd;
    r.var_off = bc.var_off;
    BoxDev b;
    b.nd = bc.nd;
    b.off = bc.var_off;
    b.total = 1;
    for (int i = 0; i < 4; i++) { b.n[i] = 1; b.vs[i] = 0; }
    for (int k = 0; k < bc.nd; k++) {
        b.n[4 - bc.nd + k] = bc.n[k];
        b.vs[4 - bc.nd + k] = bc.var_stride[k];
        b.total *= bc.n[k];
    }
    (void)r;
    return b;
}

}  // namespace

int launch_box_copy(void* var_slot, void* dense, const BoxCopy& bc, int elem_bytes, bool to_var, cudaStream_t st) {
    BoxDev b = right_align(bc);
    if (b.total == 0) return 0;
    if (elem_bytes == 4) box_copy_kernel<float><<<grid_for(b.total), 256, 0, st>>>((float*)var_slot, (float*)dense, b, to_var);
    else box_copy_kernel<double><<<grid_for(b.total), 256, 0, st>>>((double*)var_slot, (double*)dense, b, to_var);
    YB_CUDA(cudaGetLastError());
    return 0;
}

int launch_box_fill(void* var_slot, const BoxCopy& bc, int elem_bytes, double value, cudaStream_t st) {
    BoxDev b = right_align(bc);
    if (b.total == 0) return 0;
    if (elem_bytes == 4) box_fill_kernel<float><<<grid_for(b.total), 256, 0, st>>>((float*)var_slot, b, (float)value);
    else box_fill_kernel<double><<<grid_for(b.total), 256, 0, st>>>((double*)var_slot, b, value);
    YB_CUDA(cudaGetLastError());
    return 0;
}

int launch_fill_all(void* ptr, int64_t n, int elem_bytes, double value, cudaStream_t st) {
    if (n == 0) return 0;
    if (elem_bytes == 4) fill_all_kernel<float><<<grid_for(n), 256, 0, st>>>((float*)ptr, n, (float)value);
    else fill_all_kernel<double><<<grid_for(n), 256, 0, st>>>((double*)ptr, n, value);
    YB_CUDA(cudaGetLastError());
    return 0;
}

int launch_hash_fill(void* var_slot, const BoxCopy& bc, const int64_t* g0, int elem_bytes, uint32_t seed, uint32_t salt,
                     double lo, double hi, cudaStream_t st) {
    BoxDev b = right_align(bc);
    if (b.total == 0) return 0;
    if (bc.nd > 4) return set_error(YB_EUNSUPPORTED, "hash fill supports at most 4 non-step dims");
    G0 g;
    for (int i = 0; i < 3; i++) g.g[i] = g0[i];
    g.lead = g0[3];
    unsigned long long ss = ((unsigned long long)seed << 32) | (unsigned long long)salt;
    if (elem_bytes == 4) hash_fill_kernel<float><<<grid_for(b.total), 256, 0, st>>>((float*)var_slot, b, g, ss, lo, hi);
    else hash_fill_kernel<double><<<grid_for(b.total), 256, 0, st>>>((double*)var_slot, b, g, ss, lo, hi);
    YB_CUDA(cudaGetLastError());
    return 0;
}

int reduce_scratch_entries() { return MAX_GRID + 1; }

// partial: device array of reduce_scratch_entries() RedVals; the result lands in partial[0] ... [last entry]
int launch_box_reduce(const void* var_slot, const BoxCopy& bc, int elem_bytes, RedVals* partial, cudaStream_t st) {
    BoxDev b = right_align(bc);
    const int g = grid_for(b.total);
    RedVals* out = partial + (reduce_scratch_entries() - 1);
    if (elem_bytes == 4) box_reduce_kernel<float><<<g, 256, 0, st>>>((const float*)var_slot, b, partial);
    else box_reduce_kernel<double><<<g, 256, 0, st>>>((const double*)var_slot, b, partial);
    YB_CUDA(cudaGetLastError());
    reduce_final_kernel<<<1, 256, 0, st>>>(partial, g, out);
    YB_CUDA(cudaGetLastError());
    return 0;
}

int launch_checksum(const void* var_slot, const BoxCopy& bc, const int64_t* g0, int elem_bytes, unsigned long long* dev_out,
                    cudaStream_t st) {
    BoxDev b = right_align(bc);
    if (bc.nd > 3) return set_error(YB_EUNSUPPORTED, "checksum supports at most 3 non-step dims");
    YB_CUDA(cudaMemsetAsync(dev_out, 0, sizeof(unsigned long long), st));
    if (b.total == 0) return 0;
    G0 g;
    for (int i = 0; i < 3; i++) g.g[i] = g0[i];
    g.lead = 0;
    if (elem_bytes == 4) checksum_kernel<float><<<grid_for(b.total), 256, 0, st>>>((const float*)var_slot, b, g, dev_out);
    else checksum_kernel<double><<<grid_for(b.total), 256, 0, st>>>((const double*)var_slot, b, g, dev_out);
    YB_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace yb
