// Average-of-points engine: 3axis, 3axis_with_diags, 3plane and cube at any radius 1..8 in fp32 and fp64 (yb_avepts.cuh).  The
// registry (yb_stencils.cpp) routes here every radius and precision the emitter-generated kernels do not serve.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <string>

#include "yb_avepts_tiles.h"
#include "yb_chunk_plan.h"
#include "yb_core.h"

namespace yb {

namespace {
const char* const kShapes[4] = {"3axis", "3axis_with_diags", "3plane", "cube"};
}

int avepts_shape(const std::string& name) {
    for (int i = 0; i < 4; i++)
        if (name == kShapes[i]) return i;
    return -1;
}

// 1 + 6R axis points, + 12R diagonal points, + 12R(R-1) in-plane points, + 8R^3 octant points
int64_t avepts_points(int shape, int R) {
    return 1 + 6 * R + (shape >= AVP_DIAGS ? 12 * R : 0) + (shape >= AVP_PLANE ? 12 * R * (R - 1) : 0) +
           (shape >= AVP_CUBE ? 8 * int64_t(R) * R * R : 0);
}

// The generated solution's declaration (yask_b200/csrc/gen/<shape>.json): one var A(t, x, y, z), two step slots, halo R in every
// domain dim, the L1 norm of its farthest read (faces for 3axis, edges for the diagonals and planes, corners for the cube); one
// stage that reads pts points and does pts - 1 additions and one multiply.
StencilSpec avepts_spec(int shape, int radius, int elem_bytes) {
    static const int l1[4] = {1, 2, 2, 3};
    StencilSpec sp;
    sp.name = kShapes[shape];
    sp.description = "average of the points of a symmetric 3-D shape of the given radius";
    sp.domain_dims = {"x", "y", "z"};
    sp.radius = radius;
    sp.elem_bytes = elem_bytes;
    VarSpec a;
    a.name = "A";
    a.step_alloc = 2;
    a.is_output = true;
    a.l1_norm = l1[shape];
    DimSpec t; t.name = "t"; t.kind = DIM_STEP;
    a.dims.push_back(t);
    const char* dn[3] = {"x", "y", "z"};
    for (int d = 0; d < 3; d++) {
        DimSpec ds; ds.name = dn[d]; ds.kind = DIM_DOMAIN; ds.domain_index = d; ds.halo_l = ds.halo_r = radius;
        a.dims.push_back(ds);
    }
    sp.vars = {a};
    StageSpec st;
    st.name = "stage_1";
    st.outputs = {0};
    st.inputs = {0};
    st.reads = avepts_points(shape, radius);
    st.writes = 1;
    st.fp_ops = st.reads;
    sp.stages = {st};
    return sp;
}

namespace {

template <class E>
const AvpCfgT<E>* sweep_cfg(int shape, int R) {
    if (R < 1 || R > AVP_MAX_R) return nullptr;
    switch (shape) {
        case AVP_3AXIS: return &avp_table<AVP_3AXIS, E>()[R - 1];
        case AVP_DIAGS: return &avp_table<AVP_DIAGS, E>()[R - 1];
        case AVP_PLANE: return &avp_table<AVP_PLANE, E>()[R - 1];
        case AVP_CUBE: return &avp_table<AVP_CUBE, E>()[R - 1];
    }
    return nullptr;
}

// The temporal tile of (shape, radius, element size), or null where block_steps has no effect.
template <class E>
const AvpTTCfgT<E>* tt_cfg(int shape, int R) {
    if (R < 1 || R > AVP_TT_MAX_R) return nullptr;
    const AvpTTCfgT<E>* t = nullptr;
    switch (shape) {
        case AVP_3AXIS: t = avp_tt_table<AVP_3AXIS, E>(); break;
        case AVP_DIAGS: t = avp_tt_table<AVP_DIAGS, E>(); break;
        case AVP_PLANE: t = avp_tt_table<AVP_PLANE, E>(); break;
        case AVP_CUBE: t = avp_tt_table<AVP_CUBE, E>(); break;
        default: return nullptr;
    }
    return t[R - 1].fn ? &t[R - 1] : nullptr;
}
bool has_tt(const StencilSpec& sp) {
    const int shape = avepts_shape(sp.name);
    return sp.elem_bytes == 8 ? tt_cfg<double>(shape, sp.radius) != nullptr : tt_cfg<float>(shape, sp.radius) != nullptr;
}

template <class E>
using AvpDirectFn = void (*)(AvpParamsT<E>, int);
template <class E>
AvpDirectFn<E> direct_fn(int shape) {
    static const AvpDirectFn<E> fns[4] = {avepts_direct_kernel<E, AVP_3AXIS>, avepts_direct_kernel<E, AVP_DIAGS>,
                                          avepts_direct_kernel<E, AVP_PLANE>, avepts_direct_kernel<E, AVP_CUBE>};
    return fns[shape];
}

// 1/pts through the 16-significant-digit print/parse round trip of the reference's generated constants
// (/root/reference/src/compiler/lib/Cpp.cpp:39-53)
double scale_of(int shape, int R) {
    char buf[64];
    snprintf(buf, sizeof buf, "%.15e", 1.0 / double(avepts_points(shape, R)));
    return strtod(buf, nullptr);
}

struct AvpEngine : Engine {
    int shape = 0, radius = 1;
    bool f64 = false;
    std::string kernel = "auto";   // auto | tma | direct
    int lx = 0;                    // planes per sweep chunk (0 = cost model)
    int grid_override = 0;
    int gmax = 132;                // resident CTAs of the sweep kernel over the device
    int tt_gmax = 132;             // the same for the temporal tile
    int num_sms = 132;
    bool maps_ok = false, attr_set = false;
    CUtensorMap maps[4];           // A(t) in each storage slot (4 with the temporal tile's spare pair)
    // Temporal tile: option block_steps (the reference's -bt).  Its spare pair of slots is planned at prepare (plan_storage), so the
    // option must be set before prepare_solution(); later changes only switch the launch path.  One rank only.
    int block_steps = 1;
    int64_t tt_launches = 0;       // read-only option tt_launches: fused launches since prepare
    int64_t sweep_launches = 0;    // read-only option gen_sweep_launches (the generated engines' name): one-step sweeps since prepare
    bool tt_ok = false;            // spare slots allocated and tensor maps built
    CUtensorMap tt_maps[4];        // A(t) in each storage slot, the tile's boxes

    int set_option(Solution&, const std::string& k, const std::string& v) override {
        if (k == "block_steps") {
            block_steps = std::max(1, atoi(v.c_str()));
        } else if (k == "kernel") {
            if (v != "auto" && v != "tma" && v != "direct") return YB_EINVAL;
            kernel = v;
        } else if (k == "gen_sweep") {     // the generated engines' switch between their sweep and direct kernels
            kernel = atoi(v.c_str()) != 0 ? "auto" : "direct";
        } else if (k == "lx") {
            lx = std::max(0, atoi(v.c_str()));
        } else if (k == "grid") {
            grid_override = std::max(0, atoi(v.c_str()));
        } else {
            return YB_EINVAL;
        }
        return 0;
    }
    bool get_option(const Solution&, const std::string& k, std::string& v) const override {
        if (k == "kernel") v = kernel;
        else if (k == "gen_sweep") v = kernel == "direct" ? "0" : "1";
        else if (k == "lx") v = std::to_string(lx);
        else if (k == "grid") v = std::to_string(grid_override);
        else if (k == "block_steps") v = std::to_string(block_steps);
        else if (k == "tt_launches") v = std::to_string(tt_launches);
        else if (k == "gen_sweep_launches") v = std::to_string(sweep_launches);
        else return false;
        return true;
    }

    template <class E>
    const AvpCfgT<E>& cfg() const { return *sweep_cfg<E>(shape, radius); }

    // The temporal tile's storage on one rank: the spare pair of slots of A, and pads as deep as the tile's boxes of A(t) reach
    // below the origin (2R rows / planes, 2 HZ columns), so that no TMA coordinate is negative.  Boxes that stick out at the upper
    // end are zero-filled by the hardware, as in the one-step sweep.
    void plan_storage(Solution& s) override {
        Var& a = s.vars[0];
        if (a.dev) return;
        a.extra_slots = 0;
        if (block_steps < 2 || kernel == "direct" || s.multi_rank() || !has_tt(s.spec)) return;
        a.extra_slots = 2;
        const int R = s.spec.radius, vw = 16 / s.spec.elem_bytes;
        for (Dim& d : a.dims)
            if (d.spec.kind == DIM_DOMAIN)
                d.min_pad_l = std::max<int64_t>(d.min_pad_l, d.spec.domain_index == 2 ? 2 * ((R + vw - 1) / vw * vw) : 2 * R);
    }

    int prepare(Solution& s) override {
        shape = avepts_shape(s.spec.name);
        radius = s.spec.radius;
        if (shape < 0 || radius < 1 || radius > AVP_MAX_R)
            return set_error(YB_EUNSUPPORTED, "%s: the hand-written sweep serves radius 1-%d", s.spec.name.c_str(), AVP_MAX_R);
        if (s.spec.elem_bytes != 4 && s.spec.elem_bytes != 8) return set_error(YB_EUNSUPPORTED, "%s: elements must be 4 or 8 bytes", s.spec.name.c_str());
        f64 = s.spec.elem_bytes == 8;
        maps_ok = attr_set = tt_ok = false;
        tt_launches = sweep_launches = 0;
        cudaDeviceProp prop;
        YB_CUDA(cudaGetDeviceProperties(&prop, s.device));
        num_sms = prop.multiProcessorCount;
        if (s.vars[0].nslots() > 4) return set_error(YB_EUNSUPPORTED, "%s: at most 4 storage slots of A", s.spec.name.c_str());
        if (prop.major >= 9) {
            if (int rc = f64 ? build<double>(s) : build<float>(s)) return rc;
            maps_ok = true;
        }
        preload_kernel(f64 ? (const void*)direct_fn<double>(shape) : (const void*)direct_fn<float>(shape));
        return 0;
    }

    template <class E>
    int build(const Solution& s) {
        const AvpCfgT<E>& c = cfg<E>();
        const Var& a = s.vars[0];
        const int nsl = a.nslots();
        for (int slot = 0; slot < nsl; slot++)
            if (int rc = make_var_tensor_map(&maps[slot], a, slot, c.hp, c.hrows)) return rc;
        YB_CUDA(cudaFuncSetAttribute(c.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(c.smem)));
        int per_sm = 0;
        YB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, c.fn, c.threads, c.smem));
        gmax = std::max(1, per_sm) * num_sms;
        attr_set = true;
        const AvpTTCfgT<E>* tc = tt_cfg<E>(shape, radius);
        if (tc && a.extra_slots == 2 && nsl == 4) {
            for (int slot = 0; slot < nsl; slot++)
                if (int rc = make_var_tensor_map(&tt_maps[slot], a, slot, tc->ip, tc->irows)) return rc;
            YB_CUDA(cudaFuncSetAttribute(tc->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(tc->smem)));
            per_sm = 0;
            YB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tc->fn, tc->threads, tc->smem));
            tt_gmax = std::max(1, per_sm) * num_sms;
            preload_halo_shell_copy(int(sizeof(E)));
            tt_ok = true;
        }
        return 0;
    }

    int launch(Solution& s, int, int64_t t, const Box& box, cudaStream_t st) override {
        if (box.empty()) return 0;
        return f64 ? launch_t<double>(s, t, box, st) : launch_t<float>(s, t, box, st);
    }

    template <class E>
    int launch_t(Solution& s, int64_t t, const Box& box, cudaStream_t st) {
        const Var& a = s.vars[0];
        const Dim *dx = a.domain_dim(0), *dy = a.domain_dim(1), *dz = a.domain_dim(2);
        AvpParamsT<E> P{};
        P.out = reinterpret_cast<E*>(a.slot_ptr(a.slot_of(t + 1))) + a.origin_offset();
        P.cur = reinterpret_cast<const E*>(a.slot_ptr(a.slot_of(t))) + a.origin_offset();
        P.sx = dx->stride; P.sy = dy->stride;
        P.x_begin = int(box.b[0]); P.x_end = int(box.e[0]);
        P.y_begin = int(box.b[1]); P.y_end = int(box.e[1]);
        P.z_begin = int(box.b[2]); P.z_end = int(box.e[2]);
        P.pad_x = int(dx->pad_l); P.pad_y = int(dy->pad_l); P.pad_z = int(dz->pad_l);
        P.scale = E(scale_of(shape, radius));
        if (kernel == "tma" && !maps_ok) return set_error(YB_EUNSUPPORTED, "the tiled TMA kernel needs sm_90+");
        bool use_tma = maps_ok && kernel != "direct";
        // thin slabs in y / z (halo faces of a rank grid) are not worth a tile sweep
        if (kernel == "auto" && (box.e[1] - box.b[1] < 8 || box.e[2] - box.b[2] < 16)) use_tma = false;
        // TMA boxes must start on a 16-byte boundary in z
        if (use_tma && (box.b[2] * int64_t(sizeof(E))) % 16 != 0) {
            if (kernel == "tma") return set_error(YB_EUNSUPPORTED, "the tiled TMA kernel needs boxes that start on a 16-byte boundary in z");
            use_tma = false;
        }
        if (use_tma) {
            const AvpCfgT<E>& c = cfg<E>();
            P.nty = int((box.e[1] - box.b[1] + c.ty - 1) / c.ty);
            P.ntz = int((box.e[2] - box.b[2] + c.tz - 1) / c.tz);
            const int64_t ntile = int64_t(P.nty) * P.ntz;
            const int g = grid_override > 0 ? grid_override : gmax;
            const int64_t nxb = box.e[0] - box.b[0];
            P.nchunks = chunk_count(nxb, ntile, g, lx, 2 * radius, 1, std::min<int64_t>(AVP_MAX_CHUNKS, nxb));
            chunk_partition(box.b[0], nxb, P.nchunks, false, false, P.cx0, P.clen, nullptr);
            const int grid = int(std::min<int64_t>(ntile * P.nchunks, g));
            c.fn<<<grid, c.threads, c.smem, st>>>(maps[a.slot_of(t)], P);
            sweep_launches++;
        } else {
            dim3 grd(unsigned((box.e[2] - box.b[2] + 127) / 128), unsigned(box.e[1] - box.b[1]), unsigned(box.e[0] - box.b[0]));
            if (grd.y > 65535 || grd.z > 65535) return set_error(YB_EUNSUPPORTED, "direct kernel: domain too large in x or y");
            direct_fn<E>(shape)<<<grd, 128, 0, st>>>(P, radius);
        }
        YB_CUDA(cudaGetLastError());
        return 1;
    }

    // ---- temporal tile -------------------------------------------------------------------------------------------
    int fused_steps(const Solution& s) const override {
        return (tt_ok && block_steps >= 2 && kernel != "direct" && !s.multi_rank()) ? 2 : 1;
    }

    int begin_run(Solution& s, int64_t, cudaStream_t st) override { return copy_halo_shells(s.vars[0], num_sms, st); }

    // Steps t+1 and t+2 in one sweep (avepts_tt2_kernel) over the whole rank domain: reads A(t) from the live pair of slots, writes
    // A(t+2) into the partner of A(t)'s slot in the spare pair -- and A(t+1) into the partner of its slot when the launch ends the
    // run -- then makes the spare pair the live one.
    int launch_steps(Solution& s, int64_t t, int nsteps, bool ends_run, const Box& box, cudaStream_t st) override {
        if (nsteps != 2 || !tt_ok) return set_error(YB_EUNSUPPORTED, "%s: no temporal tile for %d steps in this configuration", s.spec.name.c_str(), nsteps);
        if (box.empty()) return 0;
        for (int k = 0; k < 3; k++)
            if (box.b[k] != 0 || box.e[k] != s.rank_size[k]) return set_error(YB_EUNSUPPORTED, "%s: the temporal tile runs on the whole rank domain", s.spec.name.c_str());
        const int rc = f64 ? launch_tt<double>(s, t, ends_run, box, st) : launch_tt<float>(s, t, ends_run, box, st);
        if (rc < 0) return rc;
        tt_launches++;
        s.vars[0].slot_bias ^= 2;       // steps t+1, t+2 (and every later access, stream-ordered) live in the other pair now
        return 1;
    }

    template <class E>
    int launch_tt(Solution& s, int64_t t, bool ends_run, const Box& box, cudaStream_t st) {
        const AvpTTCfgT<E>& c = *tt_cfg<E>(shape, radius);
        const Var& a = s.vars[0];
        const Dim *dx = a.domain_dim(0), *dy = a.domain_dim(1), *dz = a.domain_dim(2);
        const int cur = a.slot_of(t), nxt = a.slot_of(t + 1);         // nxt == cur ^ 1
        auto at = [&](int slot) { return reinterpret_cast<E*>(a.slot_ptr(slot)) + a.origin_offset(); };
        AvpTTParamsT<E> P{};
        P.out = at(cur ^ 2);
        P.cur = at(cur);
        P.out1 = ends_run ? at(nxt ^ 2) : nullptr;
        P.halo1 = at(nxt);
        P.sx = dx->stride; P.sy = dy->stride;
        P.x_begin = 0; P.x_end = int(box.e[0]);
        P.y_begin = 0; P.y_end = int(box.e[1]);
        P.z_begin = 0; P.z_end = int(box.e[2]);
        P.pad_x = int(dx->pad_l); P.pad_y = int(dy->pad_l); P.pad_z = int(dz->pad_l);
        P.scale = E(scale_of(shape, radius));
        P.nty = int((box.e[1] + c.ty - 1) / c.ty);
        P.ntz = int((box.e[2] + c.tz - 1) / c.tz);
        const int64_t ntile = int64_t(P.nty) * P.ntz;
        const int g = grid_override > 0 ? grid_override : tt_gmax;
        const int64_t nx = box.e[0];
        // a chunk loads 4R planes and computes 2R step-1 planes before its first result
        P.nchunks = chunk_count(nx, ntile, g, lx, 4 * radius, 1, std::min<int64_t>(AVP_MAX_CHUNKS, nx));
        chunk_partition(0, nx, P.nchunks, false, false, P.cx0, P.clen, nullptr);
        const int grid = int(std::min<int64_t>(ntile * P.nchunks, g));
        c.fn<<<grid, c.threads, c.smem, st>>>(tt_maps[cur], P);
        YB_CUDA(cudaGetLastError());
        return 1;
    }

    // Offline tuner: the sweep's chunk length, timed over the whole rank box; then, where the temporal tile is built, one step per
    // sweep against two (block_steps), at that chunk length.  Every candidate computes the same bits.
    int auto_tune(Solution& s, cudaStream_t st, std::string& report) override {
        Box whole;
        for (int d = 0; d < 3; d++) { whole.b[d] = 0; whole.e[d] = s.rank_size[d]; }
        if (!maps_ok || kernel == "direct" || whole.e[1] < 8 || whole.e[2] < 16) {
            report = s.spec.name + ": no tiled variants to tune for this configuration";
            return 0;
        }
        const int keep_lx = lx, keep_bs = block_steps;
        int64_t t = s.vars[0].last_valid_step();
        double best_ms = 1e30;
        int best = 0;
        char line[160];
        report.clear();
        for (int l : {0, 32, 64, 128, 256, 512}) {
            if (l > whole.e[0]) continue;
            lx = l;
            const double ms = time_launches(st, 3, [&]() { return launch(s, 0, t++, whole, st); });
            if (ms < 0) { lx = keep_lx; return set_error(YB_ECUDA, "auto-tuner: a trial launch failed"); }
            snprintf(line, sizeof line, " one step per sweep, lx=%d: %.4f ms/step\n", l, ms);
            report += line;
            if (ms < best_ms) { best_ms = ms; best = l; }
        }
        lx = best;
        if (tt_ok && !s.multi_rank()) {
            if (int rc = begin_run(s, t, st)) return rc;
            const double ms = time_launches(st, 3, [&]() { const int rc = launch_steps(s, t, 2, false, whole, st); t += 2; return rc; }) / 2;
            if (ms < 0) { lx = keep_lx; block_steps = keep_bs; return set_error(YB_ECUDA, "auto-tuner: a trial launch failed"); }
            snprintf(line, sizeof line, " two steps per sweep, lx=%d: %.4f ms/step\n", lx, ms);
            report += line;
            block_steps = ms < best_ms ? 2 : 1;
            best_ms = std::min(best_ms, ms);
            s.options["block_steps"] = std::to_string(block_steps);
        }
        snprintf(line, sizeof line, "best: lx=%d block_steps=%d (%.4f ms/step)\n", lx, block_steps, best_ms);
        report += line;
        s.options["lx"] = std::to_string(lx);
        return 0;
    }
};

}  // namespace

std::unique_ptr<Engine> make_avepts_engine() { return std::unique_ptr<Engine>(new AvpEngine()); }

}  // namespace yb
