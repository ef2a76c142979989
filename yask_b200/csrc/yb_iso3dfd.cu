// iso3dfd engine: spec (what the reference compiler derives from
// /root/reference/src/stencils/Iso3dfdStencil.cpp, SURVEY.md Appendix A), FD coefficients,
// TMA tensor maps and kernel launch logic.
#include <math.h>

#include <algorithm>
#include <vector>
#include <stdio.h>
#include <stdlib.h>

#include "yb_core.h"
#include "yb_iso3dfd.cuh"
#include "yb_iso3dfd_tiles.h"
#include "yb_iso3dfd_tt.cuh"

namespace yb {

// ---- FD coefficients ----------------------------------------------------------------------------------
// Fornberg's recurrence with the same operation order as the reference
// (/root/reference/src/contrib/coefficients/fd_coeff.cpp:53-101, called through
// get_center_fd_coefficients, /root/reference/src/common/fd_coeff2.cpp:49-57), then the x3 centre
// weight and /50^2 scaling of Iso3dfdStencil.cpp:68-88, then the 16-significant-digit print/parse
// round trip every constant takes through the reference's generated source (Cpp.cpp:39-53).
static void center_fd_coeffs(int order, int radius, std::vector<double>& out) {
    const int np = 2 * radius + 1;
    std::vector<double> pts(np);
    for (int i = 0; i < np; i++) pts[i] = double(i - radius);
    // w[m][n][k]: weight of point k for derivative m using points 0..n
    std::vector<double> w(size_t(order + 1) * np * np, 0.0);
    auto W = [&](int m, int n, int k) -> double& { return w[(size_t(m) * np + n) * np + k]; };
    W(0, 0, 0) = 1.0;
    double c1 = 1.0;
    for (int n = 1; n < np; n++) {
        double c2 = 1.0;
        const int mmax = std::min(n, order);
        for (int k = 0; k < n; k++) {
            const double c3 = pts[n] - pts[k];
            c2 = c2 * c3;
            for (int m = 0; m <= mmax; m++) {
                double t = (pts[n] - 0.0) * W(m, n - 1, k);
                if (m > 0) t -= m * W(m - 1, n - 1, k);
                t *= 1.0 / c3;
                if (t == 0.0) t = 0.0;
                W(m, n, k) = t;
            }
        }
        for (int m = 0; m <= mmax; m++) {
            double t = 0.0;
            if (m > 0) t += m * W(m - 1, n - 1, n - 1);
            t -= (pts[n - 1] - 0.0) * W(m, n - 1, n - 1);
            t *= c1 / c2;
            if (t == 0.0) t = 0.0;
            W(m, n, n) = t;
        }
        c1 = c2;
    }
    out.resize(np);
    for (int i = 0; i < np; i++) out[i] = W(order, np - 1, i);
}

static double const_roundtrip(double v) {
    if (double(int(v)) == v) return v;
    char buf[64];
    snprintf(buf, sizeof buf, "%.15e", v);
    return strtod(buf, nullptr);
}

void iso3dfd_coeffs(int radius, double* c) {
    std::vector<double> full;
    center_fd_coeffs(2, radius, full);
    const double d2 = 50.0 * 50.0;
    for (int i = 0; i <= 2 * radius; i++) {
        if (i == radius) full[i] *= 3.0;
        full[i] /= d2;
    }
    for (int r = 0; r <= radius; r++) c[r] = const_roundtrip(full[radius + r]);
}

// sponge: iso3dfd_sponge (/root/reference/src/stencils/Iso3dfdStencil.cpp:212-249), iso3dfd with an absorbing boundary: three 1-D
// vars cr_x(x), cr_y(y), cr_z(z) after p and v, as the generated solution declares them (no halo, not written), and
// p(t+1) *= cr_x * cr_y * cr_z.
StencilSpec iso3dfd_spec(int radius, int elem_bytes, bool sponge) {
    StencilSpec sp;
    sp.name = sponge ? "iso3dfd_sponge" : "iso3dfd";
    sp.description = sponge ? "isotropic 3-D finite-difference wave equation with an absorbing sponge boundary, order 2*radius in space"
                            : "isotropic 3-D finite-difference wave equation, 2nd order in time, order 2*radius in space";
    sp.domain_dims = {"x", "y", "z"};
    sp.radius = radius;
    sp.elem_bytes = elem_bytes;
    VarSpec p;
    p.name = "p";
    p.step_alloc = 2;   // write-back of t+1 over t-1 (SURVEY.md Appendix A)
    p.is_output = true;
    p.l1_norm = 1;
    DimSpec t; t.name = "t"; t.kind = DIM_STEP;
    p.dims.push_back(t);
    const char* dn[3] = {"x", "y", "z"};
    for (int d = 0; d < 3; d++) {
        DimSpec ds; ds.name = dn[d]; ds.kind = DIM_DOMAIN; ds.domain_index = d; ds.halo_l = ds.halo_r = radius;
        p.dims.push_back(ds);
    }
    VarSpec v;
    v.name = "v";
    v.step_alloc = 1;
    for (int d = 0; d < 3; d++) {
        DimSpec ds; ds.name = dn[d]; ds.kind = DIM_DOMAIN; ds.domain_index = d;
        v.dims.push_back(ds);
    }
    sp.vars = {p, v};
    if (sponge) {
        for (int d = 0; d < 3; d++) {
            VarSpec cr;
            cr.name = std::string("cr_") + dn[d];
            cr.step_alloc = 1;
            DimSpec ds; ds.name = dn[d]; ds.kind = DIM_DOMAIN; ds.domain_index = d;
            cr.dims.push_back(ds);
            sp.vars.push_back(cr);
        }
    }
    StageSpec st;
    st.name = "stage_1";
    st.outputs = {0};
    st.inputs = sponge ? std::vector<int>{0, 1, 2, 3, 4} : std::vector<int>{0, 1};
    // reference compiler counts for radius r: reads 6r+3, writes 1, fp ops 7r+5 (r=8: 51/1/61); the sponge reads its three
    // factors and multiplies by them: reads 6r+6, fp ops 7r+8 (r=8: 54/1/64, the generated part's counts)
    st.reads = 6 * radius + (sponge ? 6 : 3);
    st.writes = 1;
    st.fp_ops = 7 * radius + (sponge ? 8 : 5);
    sp.stages = {st};
    return sp;
}

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// 3-D tiled map over one step slot of a var (dims x,y,z; z unit stride) with box (bz, by, 1); FLOAT32 or FLOAT64 elements.
int make_map(CUtensorMap* map, const Var& v, int slot, int bz, int by) {
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) return set_error(YB_ECUDA, "cuTensorMapEncodeTiled not available from the driver");
    const Dim* dx = v.domain_dim(0);
    const Dim* dy = v.domain_dim(1);
    const Dim* dz = v.domain_dim(2);
    cuuint64_t gdim[3] = {cuuint64_t(dz->alloc), cuuint64_t(dy->alloc), cuuint64_t(dx->alloc)};
    const cuuint64_t eb = cuuint64_t(v.elem_bytes);
    cuuint64_t gstr[2] = {cuuint64_t(dy->stride) * eb, cuuint64_t(dx->stride) * eb};
    cuuint32_t box[3] = {cuuint32_t(bz), cuuint32_t(by), 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(map, v.elem_bytes == 8 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT64 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, v.slot_ptr(slot), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(YB_ECUDA, "cuTensorMapEncodeTiled failed with code %d", int(r));
    return 0;
}

}  // namespace

// 3-D tiled map over one step slot of a full-rank var of any element size (generated sweep kernels, yb_gen.cu).
int make_var_tensor_map(void* map_, const Var& v, int slot, int box_z, int box_y) {
    CUtensorMap* map = static_cast<CUtensorMap*>(map_);
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) return set_error(YB_ECUDA, "cuTensorMapEncodeTiled not available from the driver");
    const Dim* dx = v.domain_dim(0);
    const Dim* dy = v.domain_dim(1);
    const Dim* dz = v.domain_dim(2);
    if (!dx || !dy || !dz || dz->stride != 1) return set_error(YB_EUNSUPPORTED, "tensor map: var '%s' is not a full-rank 3-D var", v.spec.name.c_str());
    const cuuint64_t eb = cuuint64_t(v.elem_bytes);
    cuuint64_t gdim[3] = {cuuint64_t(dz->alloc), cuuint64_t(dy->alloc), cuuint64_t(dx->alloc)};
    cuuint64_t gstr[2] = {cuuint64_t(dy->stride) * eb, cuuint64_t(dx->stride) * eb};
    cuuint32_t box[3] = {cuuint32_t(box_z), cuuint32_t(box_y), 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(map, v.elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, v.slot_ptr(slot), gdim, gstr,
                     box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(YB_ECUDA, "cuTensorMapEncodeTiled failed with code %d (var '%s')", int(r), v.spec.name.c_str());
    return 0;
}

namespace {

template <class T, int PW, int U>
TileCfg cfg_tile(const char* name) {
    return TileCfg{true, name, T::TY, T::TZ, T::HP, T::HROWS, T::THREADS + 128 * PW, T::SMEM_BYTES,
                   {iso3dfd_tma2_kernel<T, 0, PW, U>, iso3dfd_tma2_kernel<T, 1, PW, U>, iso3dfd_tma2_kernel<T, 2, PW, U>,
                    iso3dfd_tma2_kernel<T, 3, PW, U>}};
}

// Compiled variants of the sweep kernel for radius 8 (option `tile`): tile shape x producer warpgroup x planes per trip.
constexpr int NTILES = 8;
constexpr int DEFAULT_TILE = 7;
const TileCfg& tile_cfg(int i) {
    static const TileCfg cfgs[NTILES] = {
        cfg_tile<IsoTile2<8, 16, 16, 5>, 0, 1>("32x64, in-loop producer"),
        cfg_tile<IsoTile2<8, 8, 32, 5>, 0, 1>("16x128, in-loop producer"),
        cfg_tile<IsoTile2<8, 16, 16, 5>, 1, 1>("32x64 + producer warpgroup"),
        cfg_tile<IsoTile2<8, 16, 16, 5>, 0, 2>("32x64, 2 planes per trip"),
        cfg_tile<IsoTile2<8, 8, 32, 5>, 1, 1>("16x128 + producer warpgroup"),
        cfg_tile<IsoTile2<8, 8, 32, 5>, 0, 2>("16x128, 2 planes per trip"),
        cfg_tile<IsoTile2<8, 16, 16, 5>, 1, 2>("32x64 + producer warpgroup, 2 planes per trip"),
        cfg_tile<IsoTile2<8, 8, 32, 5>, 1, 2>("16x128 + producer warpgroup, 2 planes per trip"),
    };
    return cfgs[i];
}

// Resident-plane form (option `resident`, iso3dfd_tma3_kernel) of the radius-8 producer-warpgroup, 2-planes-per-trip variants:
// same tile shapes, so it shares their tensor maps.  Rings within the 227 KB opt-in: 16x128 (18 KB slots) 10 slots = 1 plane of
// prefetch; 32x64 (15 KB slots) 12 slots = 3 planes; both with 2 stages of p(t-1) / v.  nullptr for the other tiles.
template <class T>
TileCfg cfg_resident(const char* name) {
    return TileCfg{true, name, T::TY, T::TZ, T::HP, T::HROWS, T::THREADS + 128, T::SMEM_BYTES,
                   {iso3dfd_tma3_kernel<T, 0>, iso3dfd_tma3_kernel<T, 1>, iso3dfd_tma3_kernel<T, 2>, iso3dfd_tma3_kernel<T, 3>}};
}
const TileCfg* resident_cfg(int tile) {
    static const TileCfg cfgs[2] = {cfg_resident<IsoTile3<8, 16, 16, 12, 2>>("32x64 resident planes, 12 slots"),
                                    cfg_resident<IsoTile3<8, 8, 32, 10, 2>>("16x128 resident planes, 10 slots")};
    return tile == 6 ? &cfgs[0] : tile == 7 ? &cfgs[1] : nullptr;
}

// ---- temporal tile (yb_iso3dfd_tt.cuh): compiled variants per radius and FP mode ----
typedef void (*TTKernelFn)(const TTMaps, const TTParams);
struct TTCfg {
    const char* name;
    int ty, tz, iy, iz, s1y, s1z, threads, warm;   // warm = 4R warm-up iterations per chunk
    uint32_t smem;
    TTKernelFn fn[3];
};
template <class T>
TTCfg tt_cfg(const char* name) {
    return TTCfg{name, T::TY, T::TZ, T::IY, T::IZ, T::S1Y, T::S1Z, T::THREADS, 4 * T::R, T::SMEM_BYTES,
                 {iso3dfd_tt2_kernel<T, 0>, iso3dfd_tt2_kernel<T, 1>, iso3dfd_tt2_kernel<T, 2>}};
}
// Variants per radius (option tt_variant): 0 = every neighbour read from shared memory, 1 = x neighbours of
// both steps in register queues (38 % fewer shared-memory loads, smaller rings, one more plane of prefetch).
constexpr int TT_VARIANTS = 4;       // 2, 3 = forms 0, 1 with 512 threads (16 warps per SM to hide the shared-memory latency)
const TTCfg* tt_radius_cfg(int radius, int variant) {
    static const TTCfg cfgs[TT_MAX_R][TT_VARIANTS] = {
        {tt_cfg<TTile<1, 16, 128, 3, 256, 0>>("r1 2 steps, tile 16x128, 3 planes ahead"),
         tt_cfg<TTile<1, 16, 128, 3, 256, 1>>("r1 2 steps, tile 16x128, 3 planes ahead, x queues"),
         tt_cfg<TTile<1, 16, 128, 3, 512, 0>>("r1 2 steps, tile 16x128, 3 planes ahead, 512 threads"),
         tt_cfg<TTile<1, 16, 128, 3, 512, 1>>("r1 2 steps, tile 16x128, 3 planes ahead, x queues, 512 threads")},
        {tt_cfg<TTile<2, 16, 128, 2, 256, 0>>("r2 2 steps, tile 16x128, 2 planes ahead"),
         tt_cfg<TTile<2, 16, 128, 3, 256, 1>>("r2 2 steps, tile 16x128, 3 planes ahead, x queues"),
         tt_cfg<TTile<2, 16, 128, 2, 512, 0>>("r2 2 steps, tile 16x128, 2 planes ahead, 512 threads"),
         tt_cfg<TTile<2, 16, 128, 3, 512, 1>>("r2 2 steps, tile 16x128, 3 planes ahead, x queues, 512 threads")}};
    return (radius >= 1 && radius <= TT_MAX_R && variant >= 0 && variant < TT_VARIANTS) ? &cfgs[radius - 1][variant] : nullptr;
}

// Copies a box of cells from one step slot to another (same geometry): keeps the halo cells of the extra storage
// slots of a temporally tiled var equal to those of the slot two steps earlier -- what the reference's two-slot storage
// gives by construction (p(t+2) lives in the memory of p(t), halo cells included).
__global__ void slot_box_copy_kernel(float* dst, const float* src, long long sx, long long sy, int bx, int by, int bz, int ex, int ey, int ez) {
    const long long n = (long long)ex * ey * ez;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int z = int(i % ez);
        const long long r = i / ez;
        const int y = int(r % ey), x = int(r / ey);
        const long long o = (long long)(bx + x) * sx + (long long)(by + y) * sy + (bz + z);
        dst[o] = src[o];
    }
}

struct IsoEngine : Engine {
    int radius = 8;
    bool f64 = false;              // 8-byte elements: the double-precision sweep (iso_radius_cfg_f64), one compiled variant per radius
    bool sponge = false;           // iso3dfd_sponge: the SP form of the sweep (iso_sponge_cfg / iso_sponge_cfg_f64) and direct kernels
    double coef[ISO_MAX_R + 1] = {0};
    std::string kernel = "auto";   // auto | tma | direct
    int tile = DEFAULT_TILE;       // index into tile_cfg(): 16x128, producer warpgroup, 2 planes per trip
    bool resident = true;          // tiles 6 and 7 at radius 8 in fp32: their resident-plane form (resident_cfg())
    int lx = 0;                    // planes per sweep chunk (0 = choose per launch)
    int grid_override = 0;
    int num_sms = 148;
    bool attr_set[NTILES + 2][4] = {};    // [cfg_index()][FP mode]
    // L2 policy of the sweep: both p(t) streams evict_last (a plane is fetched halo-less 8 sweep steps before it is fetched
    // with its halo, and its halo rows are the neighbouring tiles' centre rows), p(t-1) / v evict_first (streamed once), results
    // leave with streaming stores
    int pol_c = 2, pol_h = 2, pol_pv = 1, st_cs = 1;
    bool mem_probe = false;      // debug: fp_mode=3 style memory-only kernel
    int peer_probe = 0;          // debug: see IsoParams::peer_probe
    IsoMaps maps[NTILES][4];       // [tile][slot of p(t)]; p(t-1) is its partner (slot ^ 1) in the live pair of slots
    bool maps_ok = false;
    // temporal tile: option block_steps (the reference's -bt).  It needs two storage slots beyond the two the API sees
    // (Var::extra_slots), so it must be asked for before prepare_solution(); later changes only switch the launch path.
    int block_steps = 1;
    bool tt_ok = false;            // extra slots allocated and tensor maps built
    TTMaps tt_maps[4];             // [slot of p(t)]; the variants of one radius share their box shapes
    int tt_variant = -1;           // option tt_variant: index into tt_radius_cfg(); -1 = the engine's choice (tt_var())
    // The shared-memory form at both radii.  Radius 2, 1024^3, H100 80GB HBM3: 5.53-5.59 against 6.10 ms/step for the register-queue
    // form in three interleaved runs of each at a 700 W power limit (5.66 against 6.37 in one run at 400 W); radius 1: within 3 % of
    // the fastest form in one run
    int tt_var() const { return tt_variant >= 0 ? tt_variant : 0; }
    bool tt_attr_set[TT_VARIANTS][3] = {};

    int set_option(Solution& s, const std::string& k, const std::string& v) override {
        if (k == "kernel") {
            if (v != "auto" && v != "tma" && v != "direct") return YB_EINVAL;
            kernel = v;
        } else if (k == "tile") {
            int t = atoi(v.c_str());
            if (t < 0 || t >= NTILES) return YB_EINVAL;
            tile = t;
        }
        else if (k == "resident") { resident = atoi(v.c_str()) != 0; }
        else if (k == "lx") { lx = std::max(0, atoi(v.c_str())); }
        else if (k == "grid") { grid_override = std::max(0, atoi(v.c_str())); }
        else if (k == "mem_probe") { mem_probe = atoi(v.c_str()) != 0; }
        else if (k == "peer_probe") { peer_probe = atoi(v.c_str()); }
        else if (k == "pol_c") { pol_c = atoi(v.c_str()); }
        else if (k == "pol_h") { pol_h = atoi(v.c_str()); }
        else if (k == "pol_pv") { pol_pv = atoi(v.c_str()); }
        else if (k == "st_cs") { st_cs = atoi(v.c_str()) != 0; }
        else if (k == "tt_variant") {
            const int t = atoi(v.c_str());
            if (t < -1 || t >= TT_VARIANTS) return YB_EINVAL;
            tt_variant = t;
        }
        else if (k == "block_steps") {
            block_steps = std::max(1, atoi(v.c_str()));
            if (!s.prepared && s.vars.size() >= 2) {
                const bool on = block_steps >= 2 && s.spec.radius <= TT_MAX_R && s.spec.elem_bytes == 4 && !is_sponge(s.spec);
                s.vars[0].extra_slots = on ? 2 : 0;
                if (on) {
                    // the tile's boxes reach 2R rows / planes (p) and R rows / planes, one 16-byte vector in z (v) below the
                    // domain origin: pad that far, so that no TMA coordinate is ever negative (boxes that stick out at the
                    // upper end are zero-filled by the hardware, as in the one-step kernels on ragged domains)
                    const int R = s.spec.radius;
                    for (Dim& d : s.vars[0].dims)
                        if (d.spec.kind == DIM_DOMAIN) d.min_pad_l = std::max<int64_t>(d.min_pad_l, d.spec.domain_index == 2 ? 8 : 2 * R);
                    for (Dim& d : s.vars[1].dims)
                        if (d.spec.kind == DIM_DOMAIN) d.min_pad_l = std::max<int64_t>(d.min_pad_l, d.spec.domain_index == 2 ? 4 : R);
                }
            }
        }
        else return YB_EINVAL;
        return 0;
    }
    bool get_option(const Solution& s, const std::string& k, std::string& v) const override {
        if (k == "kernel") v = kernel;
        else if (k == "tile") v = std::to_string(tile);
        else if (k == "resident") v = (s.spec.radius == 8 && s.spec.elem_bytes == 4 && resident && resident_cfg(tile)) ? "1" : "0";
        else if (k == "lx") v = std::to_string(lx);
        else if (k == "grid") v = std::to_string(grid_override);
        else if (k == "block_steps") v = std::to_string(block_steps);
        else if (k == "tt_variant") v = std::to_string(tt_var());
        else return false;
        return true;
    }

    // iso3dfd_sponge has no temporal tile: block_steps=2 runs one step per sweep, as in fp64
    static bool is_sponge(const StencilSpec& sp) { return sp.name == "iso3dfd_sponge"; }

    int prepare(Solution& s) override {
        radius = s.spec.radius;
        if (radius < 1 || radius > ISO_MAX_R) return set_error(YB_EUNSUPPORTED, "iso3dfd radius must be in 1..%d", ISO_MAX_R);
        if (s.spec.elem_bytes != 4 && s.spec.elem_bytes != 8) return set_error(YB_EUNSUPPORTED, "iso3dfd: elements must be 4 or 8 bytes");
        f64 = s.spec.elem_bytes == 8;
        sponge = is_sponge(s.spec);
        if (sponge && (f64 ? !iso_sponge_cfg_f64(radius) : !iso_sponge_cfg(radius)))
            return set_error(YB_EUNSUPPORTED, "iso3dfd_sponge: the hand-written sweep serves radius 1-7 in fp32 and 1, 2, 3, 4, 5, 7 and 8 "
                                              "in fp64 (fp32 radius 8 and fp64 radius 6 are generated)");
        if (f64 && !sponge && !iso_radius_cfg_f64(radius))
            return set_error(YB_EUNSUPPORTED, "iso3dfd fp64: the hand-written sweep serves radius 1, 2, 4, 5, 6 and 7 (3 and 8 are generated)");
        iso3dfd_coeffs(radius, coef);
        cudaDeviceProp prop;
        YB_CUDA(cudaGetDeviceProperties(&prop, s.device));
        num_sms = prop.multiProcessorCount;
        maps_ok = false;
        tt_ok = false;
        const int nsl = s.vars[0].nslots();
        if (nsl > 4) return set_error(YB_EUNSUPPORTED, "iso3dfd: at most 4 storage slots of p");
        if (prop.major >= 9 && f64) {
            const TileCfgT<double>& c = sweep_cfg<double>();
            for (int cur = 0; cur < nsl; cur++)
                if (int rc = make_maps(s, c, cur, maps[0][cur])) return rc;
            maps_ok = true;
            for (int m = 0; m < 3; m++) preload_kernel((const void*)c.fn[m]);
        } else if (prop.major >= 9 && (radius == 8 || iso_radius_cfg(radius))) {
            const Var& p = s.vars[0];
            const Var& v = s.vars[1];
            for (int tl = 0; tl < (radius == 8 ? NTILES : 1); tl++) {
                const TileCfg& c = radius == 8 ? tile_cfg(tl) : sweep_cfg<float>();
                for (int cur = 0; cur < nsl; cur++)
                    if (int rc = make_maps(s, c, cur, maps[tl][cur])) return rc;
            }
            maps_ok = true;
            // (the temporal tile computes plain iso3dfd: never for a sponge solution, whatever gave p its spare slots)
            if (const TTCfg* tc = (p.extra_slots == 2 && nsl == 4 && !sponge) ? tt_radius_cfg(radius, 0) : nullptr) {
                for (int cur = 0; cur < nsl; cur++) {
                    TTMaps& m = tt_maps[cur];
                    if (int rc = make_map(&m.pin, p, cur, tc->iz, tc->iy)) return rc;
                    if (int rc = make_map(&m.prev, p, cur ^ 1, tc->s1z, tc->s1y)) return rc;
                    if (int rc = make_map(&m.v, v, 0, tc->s1z, tc->s1y)) return rc;
                }
                tt_ok = true;
                for (int vr = 0; vr < TT_VARIANTS; vr++)
                    for (int m = 0; m < 3; m++) preload_kernel((const void*)tt_radius_cfg(radius, vr)->fn[m]);
                preload_kernel((const void*)slot_box_copy_kernel);
            }
            const TileCfg& c = sweep_cfg<float>();
            for (int m = 0; m < 4; m++) preload_kernel((const void*)c.fn[m]);
        }
        if (sponge) {
            const void* fns[2][3] = {{(const void*)iso3dfd_direct_kernel<float, 0, true>, (const void*)iso3dfd_direct_kernel<float, 1, true>,
                                      (const void*)iso3dfd_direct_kernel<float, 2, true>},
                                     {(const void*)iso3dfd_direct_kernel<double, 0, true>, (const void*)iso3dfd_direct_kernel<double, 1, true>,
                                      (const void*)iso3dfd_direct_kernel<double, 2, true>}};
            for (int m = 0; m < 3; m++) preload_kernel(fns[f64][m]);
        } else if (f64) {
            preload_kernel((const void*)iso3dfd_direct_kernel<double, 0>);
            preload_kernel((const void*)iso3dfd_direct_kernel<double, 1>);
            preload_kernel((const void*)iso3dfd_direct_kernel<double, 2>);
        } else {
            preload_kernel((const void*)iso3dfd_direct_kernel<float, 0>);
            preload_kernel((const void*)iso3dfd_direct_kernel<float, 1>);
            preload_kernel((const void*)iso3dfd_direct_kernel<float, 2>);
        }
        return 0;
    }

    // Tensor maps of one sweep variant with p(t) in slot `cur`.
    template <class E>
    static int make_maps(const Solution& s, const TileCfgT<E>& c, int cur, IsoMaps& m) {
        const Var& p = s.vars[0];
        const Var& v = s.vars[1];
        if (int rc = make_map(&m.h, p, cur, c.hp, c.hrows)) return rc;
        if (int rc = make_map(&m.c, p, cur, c.tz, c.ty)) return rc;
        if (int rc = make_map(&m.p, p, cur ^ 1, c.tz, c.ty)) return rc;
        return make_map(&m.v, v, 0, c.tz, c.ty);
    }

    // The sweep variant a launch uses: the selected tile (in its resident-plane form where it has one and `resident` is on) at
    // radius 8, the one compiled variant at other radii, in fp64 and for iso3dfd_sponge (which has no fp32 radius-8 form).
    bool resident_on() const { return radius == 8 && !f64 && !sponge && resident && resident_cfg(tile); }
    template <class E>
    const TileCfgT<E>& sweep_cfg() const {
        if constexpr (sizeof(E) == 8) return sponge ? *iso_sponge_cfg_f64(radius) : *iso_radius_cfg_f64(radius);
        else if (sponge) return *iso_sponge_cfg(radius);
        else return radius != 8 ? *iso_radius_cfg(radius) : resident_on() ? *resident_cfg(tile) : tile_cfg(tile);
    }
    // Row of attr_set: the tile at radius 8 (NTILES + 0 / 1: resident forms of tiles 6 / 7), 0 otherwise.
    int cfg_index() const { return radius != 8 ? 0 : resident_on() ? NTILES + (tile == 7) : tile; }

    template <class E>
    void fill_params(const Solution& s, int64_t t, const Box& box, IsoParamsT<E>& P) const {
        const Var& p = s.vars[0];
        const Var& v = s.vars[1];
        const int cur = p.slot_of(t);
        const Dim *px = p.domain_dim(0), *py = p.domain_dim(1), *pz = p.domain_dim(2);
        const Dim *vx = v.domain_dim(0), *vy = v.domain_dim(1), *vz = v.domain_dim(2);
        // p(t+1) is written over p(t-1) (/root/reference/src/compiler/lib/Var.cpp:435-464): slot_of(t+1) == slot_of(t-1)
        P.out = reinterpret_cast<E*>(p.slot_ptr(p.slot_of(t + 1))) + p.origin_offset();
        P.prev = reinterpret_cast<const E*>(p.slot_ptr(p.slot_of(t - 1))) + p.origin_offset();
        P.cur = reinterpret_cast<const E*>(p.slot_ptr(cur)) + p.origin_offset();
        P.vel = reinterpret_cast<const E*>(v.slot_ptr(0)) + v.origin_offset();
        P.out_sx = px->stride; P.out_sy = py->stride;
        P.v_sx = vx->stride; P.v_sy = vy->stride;
        P.nx = int(px->domain); P.ny = int(py->domain); P.nz = int(pz->domain);
        P.x_begin = int(box.b[0]); P.x_end = int(box.e[0]);
        P.y_begin = int(box.b[1]); P.y_end = int(box.e[1]);
        P.z_begin = int(box.b[2]); P.z_end = int(box.e[2]);
        P.pad_x = int(px->pad_l); P.pad_y = int(py->pad_l); P.pad_z = int(pz->pad_l);
        P.vpad_x = int(vx->pad_l); P.vpad_y = int(vy->pad_l); P.vpad_z = int(vz->pad_l);
        P.pol_c = pol_c; P.pol_h = pol_h; P.pol_pv = pol_pv; P.st_cs = st_cs; P.peer_probe = peer_probe;
        for (int r = 0; r <= ISO_MAX_R; r++) P.c[r] = r <= radius ? E(coef[r]) : E(0);    // fp64: the round-tripped doubles as they are
        P.cr_x = P.cr_y = P.cr_z = nullptr;
        if (sponge) {       // vars 2, 3, 4: cr_x, cr_y, cr_z, each at its domain origin
            P.cr_x = reinterpret_cast<const E*>(s.vars[2].slot_ptr(0)) + s.vars[2].origin_offset();
            P.cr_y = reinterpret_cast<const E*>(s.vars[3].slot_ptr(0)) + s.vars[3].origin_offset();
            P.cr_z = reinterpret_cast<const E*>(s.vars[4].slot_ptr(0)) + s.vars[4].origin_offset();
        }
    }

    int launch(Solution& s, int, int64_t t, const Box& box, cudaStream_t st) override {
        if (box.empty()) return 0;
        return f64 ? launch_sweep<double>(s, t, box, st) : launch_sweep<float>(s, t, box, st);
    }

    template <class E>
    int launch_sweep(Solution& s, int64_t t, const Box& box, cudaStream_t st) {
        const Var& p = s.vars[0];
        const int cur = p.slot_of(t);
        IsoParamsT<E> P{};
        fill_params(s, t, box, P);
        int mode = s.fp_mode;
        bool use_tma = maps_ok && kernel != "direct";
        if (kernel == "auto") {
            // thin slabs in y/z (halo faces) are not worth a tile sweep
            if (box.e[1] - box.b[1] < 8 || box.e[2] - box.b[2] < 16) use_tma = false;
        }
        if (kernel == "tma" && !maps_ok) return set_error(YB_EUNSUPPORTED, "the tiled TMA kernel needs sm_90+");
        // TMA box loads whose z start is off a 16-byte boundary fault on an H100 (halo_run_stage never asks for such a box)
        if (use_tma && (box.b[2] * int64_t(sizeof(E))) % 16 != 0) {
            if (kernel == "tma") return set_error(YB_EUNSUPPORTED, "the tiled TMA kernel needs boxes that start on a 16-byte boundary in z");
            use_tma = false;
        }
        if (use_tma) {
            const int ti = (radius == 8 && !f64 && !sponge) ? tile : 0;      // tensor maps; other radii, fp64 and sponge: one compiled variant
            const int ai = cfg_index();
            const TileCfgT<E>& c = sweep_cfg<E>();
            if (mem_probe && c.fn[3]) mode = 3;
            // fused halo exchange: only for whole-domain launches of a kernel that implements the peer stores
            P.peer_lo = P.peer_hi = nullptr;
            bool fused = s.fused_x.var == 0 && c.fused_ok && mode != 3 && box.b[0] == 0 && box.e[0] == P.nx && P.nx >= 2 * radius;
            // in-kernel completion signal: needs room for boundary-first chunks; the copy-engine path exists only with it
            const bool sig = fused && s.fused_x.counter != nullptr && P.nx >= 4 * radius;
            if (fused && s.fused_x.dma && !sig) fused = false;
            const bool nb_lo = fused && s.fused_x.lo != nullptr, nb_hi = fused && s.fused_x.hi != nullptr;   // x neighbours
            if (fused) {
                if (!s.fused_x.dma) {        // the kernel stores the boundary planes into the neighbours itself
                    P.peer_lo = static_cast<E*>(s.fused_x.lo);
                    P.peer_hi = static_cast<E*>(s.fused_x.hi);
                }
                s.fused_x.used = true;
            }
            P.nty = int((box.e[1] - box.b[1] + c.ty - 1) / c.ty);
            P.ntz = int((box.e[2] - box.b[2] + c.tz - 1) / c.tz);
            const int64_t ntile = int64_t(P.nty) * P.ntz;
            const int gmax = grid_override > 0 ? grid_override : num_sms;
            // x chunks of equal length.  With an in-kernel completion signal the chunk that starts at plane 0 and the chunk
            // that ends at plane nx-1 (swept downwards) are numbered first, so that every CTA computes -- and stores into the
            // neighbours -- the boundary planes at the very start of its first sweeps.
            const int64_t ib = box.b[0], ie = box.e[0];
            const int64_t nxb = ie - ib;
            const int min_nc = (sig && nb_lo && nb_hi) ? 2 : 1;
            const int64_t max_nc = std::min<int64_t>(ISO_MAX_CHUNKS, sig ? nxb / radius : nxb);
            int nc_best = min_nc;
            if (lx > 0) {
                nc_best = int(std::max<int64_t>(min_nc, std::min<int64_t>((nxb + lx - 1) / lx, max_nc)));
            } else {
                // Pick the chunk count that minimises (rounds of units per CTA) x (chunk length + queue
                // warm-up): long chunks amortise the 2R warm-up planes, short ones balance the last round.
                double best = 1e30;
                for (int64_t nc = min_nc; nc <= max_nc; nc++) {
                    const int64_t l = (nxb + nc - 1) / nc;
                    const int64_t rounds = (ntile * nc + gmax - 1) / gmax;
                    const double cost = double(rounds) * (double(l) + 2 * radius * 0.4);
                    if (cost < best * 0.999) { best = cost; nc_best = int(nc); }
                }
            }
            int nb = 0, nsig = 0;
            {
                const int nc = nc_best;      // balanced partition: chunk lengths differ by at most one plane (all >= R when signalling)
                std::vector<int> order;
                if (sig && nb_lo) order.push_back(0);
                if (sig && nb_hi && !(nc == 1 && nb_lo)) order.push_back(nc - 1);
                nsig = int(order.size());
                for (int c = 0; c < nc; c++)
                    if (std::find(order.begin(), order.end(), c) == order.end()) order.push_back(c);
                for (int c : order) {
                    const int64_t x0 = ib + nxb * c / nc, x1 = ib + nxb * (c + 1) / nc;
                    const bool down = sig && nb_hi && c == nc - 1 && !(nc == 1 && nb_lo);
                    P.cx0[nb] = int(down ? x1 - 1 : x0); P.clen[nb] = int(x1 - x0); P.cdir[nb] = down ? -1 : 1;
                    nb++;
                }
            }
            P.nchunks = nb;
            P.sig_units = 0; P.sig_total = 0; P.sig_counter = nullptr; P.sig_flag_lo = P.sig_flag_hi = nullptr; P.sig_epoch = 0;
            const int64_t nunits = int64_t(P.nty) * P.ntz * P.nchunks;
            int grid = int(std::min<int64_t>(nunits, gmax));
            if (sig) {
                P.sig_units = int(ntile) * nsig;
                P.sig_total = unsigned(grid) * unsigned(c.ty * c.tz / (2 * IsoVec<E>::N) / 32);   // consumer warps: 2 vectors per thread
                P.sig_counter = s.fused_x.counter;
                P.sig_flag_lo = s.fused_x.flag_lo; P.sig_flag_hi = s.fused_x.flag_hi;
                P.sig_epoch = s.fused_x.epoch;
                s.fused_x.signalled = true;
            }
            if (!attr_set[ai][mode]) {
                YB_CUDA(cudaFuncSetAttribute(c.fn[mode], cudaFuncAttributeMaxDynamicSharedMemorySize, int(c.smem)));
                attr_set[ai][mode] = true;
            }
            c.fn[mode]<<<grid, c.threads, c.smem, st>>>(maps[ti][cur], P);
        } else {
            dim3 blk(128, 1, 1);
            dim3 grd(unsigned((box.e[2] - box.b[2] + 127) / 128), unsigned(box.e[1] - box.b[1]), unsigned(box.e[0] - box.b[0]));
            if (grd.y > 65535 || grd.z > 65535) return set_error(YB_EUNSUPPORTED, "direct kernel: domain too large in x or y");
            if (sponge) {
                switch (mode) {
                    case 0: iso3dfd_direct_kernel<E, 0, true><<<grd, blk, 0, st>>>(P, radius); break;
                    case 1: iso3dfd_direct_kernel<E, 1, true><<<grd, blk, 0, st>>>(P, radius); break;
                    default: iso3dfd_direct_kernel<E, 2, true><<<grd, blk, 0, st>>>(P, radius); break;
                }
            } else {
                switch (mode) {
                    case 0: iso3dfd_direct_kernel<E, 0><<<grd, blk, 0, st>>>(P, radius); break;
                    case 1: iso3dfd_direct_kernel<E, 1><<<grd, blk, 0, st>>>(P, radius); break;
                    default: iso3dfd_direct_kernel<E, 2><<<grd, blk, 0, st>>>(P, radius); break;
                }
            }
        }
        YB_CUDA(cudaGetLastError());
        return 1;
    }

    // ---- temporal tile -------------------------------------------------------------------------------------------
    int fused_steps(const Solution& s) const override {
        return (tt_ok && block_steps >= 2 && kernel != "direct" && !s.multi_rank()) ? 2 : 1;
    }

    // Halo cells of the spare pair of slots take those of the live pair, so that whichever pair a fused launch reads holds
    // the halo cells the reference's two slots would (kernels never write halo cells; the API may, between runs).
    int begin_run(Solution& s, int64_t, cudaStream_t st) override {
        const Var& p = s.vars[0];
        if (p.extra_slots != 2 || !p.dev) return 0;
        const Dim* d[3] = {p.domain_dim(0), p.domain_dim(1), p.domain_dim(2)};
        int64_t lo[3], hi[3], db[3], de[3];     // halo box and domain box in alloc coordinates
        for (int k = 0; k < 3; k++) {
            db[k] = d[k]->pad_l; de[k] = d[k]->pad_l + d[k]->domain;
            lo[k] = db[k] - d[k]->spec.halo_l; hi[k] = de[k] + d[k]->spec.halo_r;
        }
        for (int pair = 0; pair < 2; pair++) {
            const float* src = reinterpret_cast<const float*>(p.slot_ptr(p.slot_bias + pair));
            float* dst = reinterpret_cast<float*>(p.slot_ptr((p.slot_bias ^ 2) + pair));
            // shell = x slabs over the whole (y,z) halo box, y slabs over the domain's x range, z slabs over the domain's x and y ranges
            const int64_t slabs[6][6] = {{lo[0], db[0], lo[1], hi[1], lo[2], hi[2]}, {de[0], hi[0], lo[1], hi[1], lo[2], hi[2]},
                                         {db[0], de[0], lo[1], db[1], lo[2], hi[2]}, {db[0], de[0], de[1], hi[1], lo[2], hi[2]},
                                         {db[0], de[0], db[1], de[1], lo[2], db[2]}, {db[0], de[0], db[1], de[1], de[2], hi[2]}};
            for (auto& b : slabs) {
                const int64_t ex = b[1] - b[0], ey = b[3] - b[2], ez = b[5] - b[4];
                if (ex <= 0 || ey <= 0 || ez <= 0) continue;
                const int64_t n = ex * ey * ez;
                const int grid = int(std::min<int64_t>((n + 255) / 256, 16 * num_sms));
                slot_box_copy_kernel<<<grid, 256, 0, st>>>(dst, src, d[0]->stride, d[1]->stride, int(b[0]), int(b[2]), int(b[4]), int(ex), int(ey), int(ez));
            }
        }
        YB_CUDA(cudaGetLastError());
        return 0;
    }

    // Steps t+1 and t+2 in one sweep (iso3dfd_tt2_kernel): reads the live pair of slots (p(t-1), p(t)), writes p(t+1) / p(t+2)
    // into the partners of p(t-1) / p(t) in the spare pair, which then becomes the live one.
    int launch_steps(Solution& s, int64_t t, int nsteps, const Box& box, cudaStream_t st) override {
        if (nsteps != 2 || !tt_ok) return set_error(YB_EUNSUPPORTED, "iso3dfd: no temporal tile for %d steps in this configuration", nsteps);
        if (box.empty()) return 0;
        const int vr = tt_var();
        const TTCfg& c = *tt_radius_cfg(radius, vr);
        Var& p = s.vars[0];
        const Var& v = s.vars[1];
        const Dim *px = p.domain_dim(0), *py = p.domain_dim(1), *pz = p.domain_dim(2);
        const Dim *vx = v.domain_dim(0), *vy = v.domain_dim(1), *vz = v.domain_dim(2);
        for (int k = 0; k < 3; k++)
            if (box.b[k] != 0 || box.e[k] != p.domain_dim(k)->domain) return set_error(YB_EUNSUPPORTED, "iso3dfd: the temporal tile runs on the whole rank domain");
        TTParams P{};
        const int cur = p.slot_of(t), prev = p.slot_of(t - 1);      // prev == cur ^ 1 (tensor maps)
        P.out1 = reinterpret_cast<float*>(p.slot_ptr(prev ^ 2)) + p.origin_offset();
        P.out2 = reinterpret_cast<float*>(p.slot_ptr(cur ^ 2)) + p.origin_offset();
        P.vel = reinterpret_cast<const float*>(v.slot_ptr(0)) + v.origin_offset();
        P.p_sx = px->stride; P.p_sy = py->stride; P.v_sx = vx->stride; P.v_sy = vy->stride;
        P.nx = int(px->domain); P.ny = int(py->domain); P.nz = int(pz->domain);
        P.pad_x = int(px->pad_l); P.pad_y = int(py->pad_l); P.pad_z = int(pz->pad_l);
        P.vpad_x = int(vx->pad_l); P.vpad_y = int(vy->pad_l); P.vpad_z = int(vz->pad_l);
        for (int r = 0; r <= TT_MAX_R; r++) P.c[r] = r <= radius ? float(coef[r]) : 0.f;
        P.pol_p = pol_h; P.st_cs = st_cs;       // same options (pol_h, st_cs) and defaults as the one-step kernel's haloed p(t) stream / stores
        P.nty = (P.ny + c.ty - 1) / c.ty;
        P.ntz = (P.nz + c.tz - 1) / c.tz;
        // x chunks of (almost) equal length: minimise (rounds of units per CTA) x (chunk length + warm-up iterations;
        // those of the first 2R only load, the next 2R only run step 1)
        const int64_t ntile = int64_t(P.nty) * P.ntz;
        const int gmax = grid_override > 0 ? grid_override : num_sms;
        const int64_t max_nc = std::min<int64_t>(TT_MAX_CHUNKS, P.nx);
        int nc_best = 1;
        if (lx > 0) nc_best = int(std::max<int64_t>(1, std::min<int64_t>((P.nx + lx - 1) / lx, max_nc)));
        else {
            double best = 1e30;
            for (int64_t nc = 1; nc <= max_nc; nc++) {
                const int64_t l = (P.nx + nc - 1) / nc;
                const int64_t rounds = (ntile * nc + gmax - 1) / gmax;
                const double cost = double(rounds) * (double(l) + c.warm * 0.4);
                if (cost < best * 0.999) { best = cost; nc_best = int(nc); }
            }
        }
        P.nchunks = nc_best;
        for (int k = 0; k < nc_best; k++) {
            const int64_t x0 = int64_t(P.nx) * k / nc_best, x1 = int64_t(P.nx) * (k + 1) / nc_best;
            P.cx0[k] = int(x0); P.clen[k] = int(x1 - x0);
        }
        const int64_t nunits = ntile * P.nchunks;
        const int grid = int(std::min<int64_t>(nunits, gmax));
        const int mode = std::min(std::max(s.fp_mode, 0), 2);
        if (!tt_attr_set[vr][mode]) {
            YB_CUDA(cudaFuncSetAttribute(c.fn[mode], cudaFuncAttributeMaxDynamicSharedMemorySize, int(c.smem)));
            tt_attr_set[vr][mode] = true;
        }
        c.fn[mode]<<<grid, c.threads, c.smem, st>>>(tt_maps[cur], P);
        YB_CUDA(cudaGetLastError());
        p.slot_bias ^= 2;       // steps t+1, t+2 (and every later access, stream-ordered) live in the other pair now
        return 1;
    }

    // In-run tuner: the same variants as the offline tuner, one per step of a live run.
    static constexpr int TUNE_TILES[6] = {7, 6, 5, 4, 1, 0};
    static constexpr int TUNE_LXS[3] = {0, 256, 512};
    int tune_variants(const Solution&) const override { return (maps_ok && radius == 8 && !f64 && !sponge && kernel != "direct") ? 18 : 0; }
    void tune_select(Solution& s, int v) override {
        tile = TUNE_TILES[v / 3]; lx = TUNE_LXS[v % 3];
        s.options["tile"] = std::to_string(tile);
        s.options["lx"] = std::to_string(lx);
        preload_kernel((const void*)sweep_cfg<float>().fn[s.fp_mode]);
    }
    std::string tune_describe(const Solution&, int v) const override {
        char b[160];
        snprintf(b, sizeof b, "tile=%d (%s) lx=%d", TUNE_TILES[v / 3], tile_cfg(TUNE_TILES[v / 3]).name, TUNE_LXS[v % 3]);
        return b;
    }

    // Offline tuner of a solution that has a temporal tile: one step per sweep against two steps per sweep in each compiled form,
    // timed per STEP over the whole rank box; the fastest stays selected (block_steps / tt_variant).  All compute the same bits.
    int auto_tune_temporal(Solution& s, cudaStream_t st, std::string& report) {
        Box whole;
        for (int d = 0; d < 3; d++) { whole.b[d] = 0; whole.e[d] = s.rank_size[d]; }
        int64_t t = s.vars[0].last_valid_step();
        if (int rc = begin_run(s, t, st)) return rc;
        const int keep_bs = block_steps, keep_var = tt_variant;
        const int dflt_var = tt_var();
        double best = 1e30;
        int best_bs = 1, best_var = tt_var();
        char line[200];
        report.clear();
        for (int cand = 0; cand <= TT_VARIANTS; cand++) {
            double ms;
            if (cand == 0) {
                ms = time_launches(st, 4, [&]() { return launch(s, 0, t++, whole, st); });
                snprintf(line, sizeof line, " one step per sweep: %.4f ms/step\n", ms);
            } else {
                tt_variant = cand - 1;
                ms = time_launches(st, 3, [&]() { const int rc = launch_steps(s, t, 2, whole, st); t += 2; return rc; }) / 2;
                snprintf(line, sizeof line, " two steps per sweep, %s: %.4f ms/step\n", tt_radius_cfg(radius, tt_variant)->name, ms);
            }
            if (ms < 0) { block_steps = keep_bs; tt_variant = keep_var; return set_error(YB_ECUDA, "auto-tuner: a trial launch failed"); }
            report += line;
            if (ms < best) { best = ms; best_bs = cand == 0 ? 1 : 2; best_var = cand == 0 ? dflt_var : cand - 1; }
        }
        block_steps = best_bs; tt_variant = best_var;
        snprintf(line, sizeof line, "best: block_steps=%d tt_variant=%d (%.4f ms/step)\n", block_steps, tt_variant, best);
        report += line;
        s.options["block_steps"] = std::to_string(block_steps);
        s.options["tt_variant"] = std::to_string(tt_variant);
        return 0;
    }

    // Offline tuner: the compiled sweep variants (tile shape, producer warpgroup, planes per trip, resident planes) x sweep
    // chunk lengths, timed over the whole rank box; the analogue of the reference's block-size search
    // (/root/reference/src/kernel/lib/auto_tuner.cpp) for the knobs this engine has.  fp64 has one variant per radius: only
    // the chunk length is searched.  iso3dfd_sponge keeps the same behaviour: fp64 searches the chunk length, fp32 (radius 1-7)
    // has nothing to tune.
    int auto_tune(Solution& s, cudaStream_t st, std::string& report) override {
        if (tt_ok && kernel != "direct" && !s.multi_rank()) return auto_tune_temporal(s, st, report);
        if (!maps_ok || (radius != 8 && !f64) || kernel == "direct") { report = "iso3dfd: no tiled variants to tune for this configuration"; return 0; }
        Box whole;
        for (int d = 0; d < 3; d++) { whole.b[d] = 0; whole.e[d] = s.rank_size[d]; }
        if (whole.e[1] < 8 || whole.e[2] < 16) { report = "iso3dfd: domain too thin for the tiled kernel"; return 0; }
        const int64_t t0 = s.vars[0].last_valid_step();
        // (tile, resident) pairs; resident = 1 only where the tile has a resident-plane form
        const std::vector<std::pair<int, bool>> forms =
            f64 ? std::vector<std::pair<int, bool>>{{tile, false}}
                : std::vector<std::pair<int, bool>>{{7, true}, {6, true}, {7, false}, {6, false}, {5, false}, {4, false}, {1, false}, {0, false}};
        const int lxs[] = {0, 256, 512, 1024};   // planes per interior chunk (0 = cost model)
        const int keep_tile = tile, keep_lx = lx;
        const bool keep_res = resident;
        double best = 1e30;
        int best_tile = tile, best_lx = lx;
        bool best_res = resident;
        char line[160];
        report.clear();
        for (const auto& [ti, res] : forms)
            for (int l : lxs) {
                if (l > whole.e[0]) continue;
                tile = ti; resident = res; lx = l;
                int64_t t = t0;
                const double ms = time_launches(st, 3, [&]() { return launch(s, 0, t++, whole, st); });
                if (ms < 0) { tile = keep_tile; resident = keep_res; lx = keep_lx; return set_error(YB_ECUDA, "auto-tuner: a trial launch failed"); }
                snprintf(line, sizeof line, " tile=%d resident=%d (%s) lx=%d: %.4f ms/step\n", ti, int(resident_on()), f64 ? sweep_cfg<double>().name : sweep_cfg<float>().name, l, ms);
                report += line;
                if (ms < best) { best = ms; best_tile = ti; best_res = res; best_lx = l; }
            }
        tile = best_tile; resident = best_res; lx = best_lx;
        snprintf(line, sizeof line, "best: tile=%d resident=%d lx=%d (%.4f ms/step)\n", tile, int(resident_on()), lx, best);
        report += line;
        s.options["tile"] = std::to_string(tile);
        s.options["resident"] = resident ? "1" : "0";
        s.options["lx"] = std::to_string(lx);
        return 0;
    }
};

}  // namespace

std::unique_ptr<Engine> make_iso3dfd_engine() { return std::unique_ptr<Engine>(new IsoEngine()); }

}  // namespace yb
