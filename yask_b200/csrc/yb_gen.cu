// Engine for emitter-generated solutions: turns a GenStencil table into a StencilSpec and launches
// one kernel per part and stage (the reference runs the parts of a stage back to back over each
// micro-block, /root/reference/src/kernel/lib/context.cpp:1158; parts of a stage are independent).
#include <algorithm>
#include <cstring>
#include <map>

#include "yb_core.h"
#include "yb_gen_sweep.cuh"
// generated solutions: declarations + table (each solution is compiled in its own translation unit)
#include "gen/gen_all.inc"

namespace yb {

using namespace gen;

namespace {

typedef void (*DescribeFn)(GenStencil&);
struct GenEntry { const char* name; DescribeFn describe; };
const GenEntry kGen[] = {YB_GEN_TABLE};

VarSpec var_spec_of(const GenStencil& g, const GenVar& gv) {
    VarSpec v;
    v.name = gv.name;
    v.step_alloc = gv.alloc_t;
    v.is_output = gv.is_output;
    v.l1_norm = gv.l1_norm;
    for (auto* dn : gv.dims) {
        DimSpec d;
        d.name = dn;
        if (g.step_dim == dn) { d.kind = DIM_STEP; }
        else {
            d.kind = DIM_MISC;
            for (size_t k = 0; k < g.domain_dims.size(); k++)
                if (g.domain_dims[k] == dn) { d.kind = DIM_DOMAIN; d.domain_index = int(k); d.halo_l = gv.halo_l[k]; d.halo_r = gv.halo_r[k]; }
            if (d.kind == DIM_MISC) {
                const size_t di = v.dims.size();
                d.misc_first = gv.misc_first[di];
                d.misc_size = std::max(1, gv.misc_size[di]);
            }
        }
        v.dims.push_back(d);
    }
    return v;
}

struct GenEngine : Engine {
    GenStencil g;
    // Scratch vars (MAKE_SCRATCH_VAR in the DSL) are engine-internal: one HBM array each over the rank domain plus the
    // var's halo, in the solution's shared padded geometry.  (The reference keeps one micro-block-sized copy per
    // thread, /root/reference/src/kernel/lib/setup.cpp:807-; a GPU launch covers the whole rank box at once.)
    std::vector<Var> scratch;
    int nreg = 0;      // g.vars[0..nreg) are the API-visible vars, the rest scratch
    ~GenEngine() override {
        for (auto& v : scratch)
            if (v.dev) cudaFree(v.dev);
        for (auto& kv : sweep_maps) cudaFree(kv.second);
    }
    const Var& var_of(const Solution& s, int gi) const { return gi < nreg ? s.vars[gi] : scratch[gi - nreg]; }
    // option gen_pf (or env YB_GEN_PF): L2 prefetch distance in x planes (0 = off) of the direct kernels.
    int pf_dist = 1;
    GenEngine() {
        if (const char* e = getenv("YB_GEN_PF")) pf_dist = std::max(0, atoi(e));
        if (const char* e = getenv("YB_GEN_L2_MB")) l2_mb = std::max(0, atoi(e));
        if (const char* e = getenv("YB_GEN_SWEEP")) sweep = atoi(e) != 0;
    }
    int sweep = 1;     // option gen_sweep (env YB_GEN_SWEEP): 1 (default) = TMA-staged sweep kernels where a part has one and the
                       // launch box allows; 0 = direct kernels everywhere
    int sweep_lx = 0;    // option gen_sweep_lx: x planes per sweep chunk (0 = cost model)
    int sweep_min_x = 12;  // shorter boxes (exterior slabs of a rank grid) take the direct kernels
    int num_sms = 148;
    std::map<const void*, bool> sweep_attr;   // kernels whose dynamic shared-memory limit has been raised
    // tensor maps of a part's streams live in device memory, one array per combination of step slots (they depend only on
    // the vars' storage, fixed after prepare)
    std::map<std::pair<const GenPart*, std::string>, void*> sweep_maps;
    void free_sweep_maps() {
        for (auto& kv : sweep_maps) cudaFree(kv.second);
        sweep_maps.clear();
    }
    bool wide = false;   // kernels in their 64-bit addressing form (prepare); option gen_wide reads it back
    bool force_wide = false;   // option gen_wide = 1: the 64-bit form at any size (0: only where a slot needs it)
    int l2_mb = 16;    // option gen_l2_mb (env YB_GEN_L2_MB): L2 budget of one y chunk's sweep working set (0 = no chunking)
    int set_option(Solution&, const std::string& key, const std::string& value) override {
        if (key == "gen_wide") { force_wide = atoi(value.c_str()) != 0; return 0; }
        if (key == "gen_pf") { pf_dist = std::max(0, atoi(value.c_str())); return 0; }
        if (key == "gen_l2_mb") { l2_mb = std::max(0, atoi(value.c_str())); return 0; }
        if (key == "gen_sweep") { sweep = atoi(value.c_str()) != 0; return 0; }
        if (key == "gen_sweep_lx") { sweep_lx = std::max(0, atoi(value.c_str())); return 0; }
        return YB_EINVAL;
    }
    int prepare(Solution& s) override {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, s.device) == cudaSuccess) num_sms = prop.multiProcessorCount;
        if (s.spec.elem_bytes != g.elem_bytes)
            return set_error(YB_EUNSUPPORTED, "solution '%s' was generated for %d-byte elements", g.name.c_str(), g.elem_bytes);
        // the kernels' addressing form (GenFnPair): 64-bit element positions once a var slot holds 2^31 elements or
        // more, the 32-bit form below that (scratch vars share the solution's geometry, so the API-visible vars decide);
        // option gen_wide = 1 takes the 64-bit form at any size, so that it can be checked on small domains
        wide = force_wide;
        for (auto& v : s.vars) wide = wide || v.slot_elems >= (int64_t(1) << 31);
        sweep_launches = 0;
        for (auto& st : g.stages)
            for (auto& p : st.parts)
                if (int(p.acc.size()) > GEN_MAX_ACC) return set_error(YB_EUNSUPPORTED, "part '%s' touches too many vars", p.name);
        for (auto& st : g.stages)
            for (auto& p : st.parts)
                for (int m = 0; m < 2; m++) {
                    preload_kernel((const void*)p.fn[g.elem_bytes == 8 ? 1 : 0][m].pick(wide));
                    preload_kernel((const void*)p.sweep.fn[g.elem_bytes == 8 ? 1 : 0][m].pick(wide));
                }
        for (auto& v : scratch)
            if (v.dev) cudaFree(v.dev);
        scratch.clear();
        free_sweep_maps();
        for (auto& gv : g.vars) {
            if (!gv.is_scratch) continue;
            Var v;
            v.spec = var_spec_of(g, gv);
            v.elem_bytes = g.elem_bytes;
            for (auto& ds : v.spec.dims) { Dim d; d.spec = ds; v.dims.push_back(d); }
            compute_var_geometry(s, v);
            YB_CUDA(cudaMalloc(&v.dev, v.bytes()));
            YB_CUDA(cudaMemsetAsync(v.dev, 0, v.bytes(), s.stream()));
            scratch.push_back(std::move(v));
        }
        return 0;
    }
    // Sizes the generated kernels cannot address, refused before anything is allocated (Engine::check_geometry):
    //  * a dimension: launch boxes and point coordinates are int (GenParams::xb..ze, GEN_KERNEL_BEGIN), so a domain dim and
    //    its pads must span fewer than 2^31 elements -- what bounds a 1-D solution, or the unit-stride dim of a 2-D one;
    //  * the neighbour offsets: the kernels form each point's position in 64 bits where the slots need it, but add the
    //    offsets dx*SX + dy*SY + dz (int SX, SY: GenParams) in 32 bits (yb_gen.cuh, GEN_POS).  |dy*SY + dz| < SX, so
    //    (x halo + 1) x-planes of a 3-D var must stay below 2^31 elements: that bounds the y*z extent, not the size of a var;
    //  * the launch grids: one 1-D grid per part, fewer than 2^31 CTAs (direct kernels, and sweep kernels at their longest
    //    chunking, one plane per chunk).
    int check_geometry(const Solution& s) const override {
        const int64_t lim = int64_t(1) << 31;
        const int sh = 3 - s.ndd;
        int64_t ext[3] = {1, 1, 1};   // per kernel slot: largest extent of any var, pads included
        for (auto& v : s.vars)
            for (auto& d : v.dims) {
                if (d.spec.kind != DIM_DOMAIN) continue;
                if (d.alloc >= lim)
                    return set_error(YB_EUNSUPPORTED,
                                     "var '%s': dim '%s' spans %lld elements with its pads (domain %lld); the generated kernels "
                                     "index a dimension with 32-bit ints, limit 2^31 - 1 elements",
                                     v.spec.name.c_str(), d.spec.name.c_str(), (long long)d.alloc, (long long)d.domain);
                ext[d.spec.domain_index + sh] = std::max(ext[d.spec.domain_index + sh], d.alloc);
            }
        if (s.ndd == 3)
            for (auto& v : s.vars) {
                const Dim* d0 = v.domain_dim(0);
                if (!d0 || !v.domain_dim(1) || !v.domain_dim(2)) continue;
                const int64_t reach = std::max(d0->pad_l, d0->pad_r) + 1;
                if (reach * d0->stride >= lim)
                    return set_error(YB_EUNSUPPORTED,
                                     "var '%s': %lld x-planes of %lld elements (x halo + 1) reach 2^31 elements, the limit of the "
                                     "generated kernels' 32-bit neighbour offsets; reduce the y*z extent (%lld x %lld)",
                                     v.spec.name.c_str(), (long long)reach, (long long)d0->stride,
                                     (long long)v.domain_dim(1)->domain, (long long)v.domain_dim(2)->domain);
            }
        auto cdiv = [](int64_t a, int64_t b) { return (a + b - 1) / b; };
        const int64_t direct = cdiv(ext[2], GEN_BZ) * cdiv(ext[1], GEN_BY * gen_np(g.elem_bytes)) * cdiv(ext[0], GEN_BX);
        int64_t grid = direct;
        for (auto& st : g.stages)
            for (auto& p : st.parts)
                if (p.sweep.ty > 0 && p.sweep.tz > 0)
                    grid = std::max(grid, cdiv(ext[2], p.sweep.tz) * cdiv(ext[1], p.sweep.ty) * ext[0]);
        if (grid >= lim)
            return set_error(YB_EUNSUPPORTED, "domain %lld x %lld x %lld (pads included) needs a launch grid of %lld CTAs; the "
                             "generated kernels' 1-D grids take fewer than 2^31", (long long)ext[0], (long long)ext[1],
                             (long long)ext[2], (long long)grid);
        return 0;
    }
    // Read-only option gen_sweep_launches: sweep-kernel launches since prepare (which parts took the TMA sweep form).
    // Option gen_wide on a prepared solution: the addressing form its kernels run, "1" (64-bit) or "0" (32-bit).
    int64_t sweep_launches = 0;
    bool get_option(const Solution& s, const std::string& key, std::string& v) const override {
        if (key == "gen_wide" && s.prepared) { v = wide ? "1" : "0"; return true; }
        if (key != "gen_sweep_launches") return false;
        v = std::to_string(sweep_launches);
        return true;
    }
    // In-run tuner: sweep kernels with the cost-model chunking or fixed chunk lengths, and the direct kernels.
    int tune_variants(const Solution&) const override { return 4; }
    void tune_select(Solution& s, int v) override {
        sweep = v < 3 ? 1 : 0;
        sweep_lx = v == 1 ? 64 : (v == 2 ? 128 : 0);
        s.options["gen_sweep"] = std::to_string(sweep);
        s.options["gen_sweep_lx"] = std::to_string(sweep_lx);
    }
    std::string tune_describe(const Solution&, int v) const override {
        static const char* d[4] = {"gen_sweep=1 gen_sweep_lx=0 (cost model)", "gen_sweep=1 gen_sweep_lx=64", "gen_sweep=1 gen_sweep_lx=128", "gen_sweep=0 (direct kernels)"};
        return d[v];
    }

    // Offline tuner: L2 prefetch distance x sweep-chunk budget, timed over one full step of the rank box.
    int auto_tune(Solution& s, cudaStream_t st, std::string& report) override {
        Box whole;
        for (int d = 0; d < 3; d++) { whole.b[d] = 0; whole.e[d] = d < s.ndd ? s.rank_size[d] : 1; }
        const int pfs[] = {0, 1, 2};
        const int l2s[] = {0, 8, 16, 32};
        const int keep_pf = pf_dist, keep_l2 = l2_mb;
        double best = 1e30;
        int best_pf = pf_dist, best_l2 = l2_mb;
        char line[128];
        report.clear();
        int64_t t = 0;
        for (auto& v : s.vars) t = std::max(t, v.last_valid_step());
        for (int pf : pfs)
            for (int l2 : l2s) {
                pf_dist = pf; l2_mb = l2;
                const double ms = time_launches(st, 2, [&]() {
                    int n = 0;
                    for (size_t sg = 0; sg < g.stages.size(); sg++) {
                        const int rc = launch(s, int(sg), t, whole, st);
                        if (rc < 0) return rc;
                        n += rc;
                    }
                    return n;
                });
                if (ms < 0) { pf_dist = keep_pf; l2_mb = keep_l2; return set_error(YB_ECUDA, "auto-tuner: a trial launch failed"); }
                snprintf(line, sizeof line, " gen_pf=%d gen_l2_mb=%d: %.4f ms/step\n", pf, l2, ms);
                report += line;
                if (ms < best) { best = ms; best_pf = pf; best_l2 = l2; }
            }
        pf_dist = best_pf; l2_mb = best_l2;
        snprintf(line, sizeof line, "best: gen_pf=%d gen_l2_mb=%d (%.4f ms/step)\n", pf_dist, l2_mb, best);
        report += line;
        s.options["gen_pf"] = std::to_string(pf_dist);
        s.options["gen_l2_mb"] = std::to_string(l2_mb);
        return 0;
    }

    int launch(Solution& s, int stage, int64_t t, const Box& box, cudaStream_t st) override {
        if (box.empty()) return 0;
        const GenStage& gs = g.stages[stage];
        int n = 0;
        std::vector<char> scratch_written(scratch.size(), 0);
        for (auto& p : gs.parts) {
            GenParams P{};
            P.t = t;
            // The solution's domain dims are right-aligned into the kernel's (x,y,z) slots: slot k holds domain dim
            // k - sh, so the unit-stride dim always lands in slot z (1-D/2-D solutions leave the outer slots empty).
            const int sh = 3 - s.ndd;
            // shrink the launch box to the part's sub-domain (IF_DOMAIN), expressed over global indices
            // (the reference intersects with per-part bounding boxes, setup.cpp:1235-1498)
            Box pb;
            for (int k = 0; k < 3; k++) {
                const int d = k - sh;
                pb.b[k] = d >= 0 ? box.b[d] - p.wh_l[k] : 0;
                pb.e[k] = d >= 0 ? box.e[d] + p.wh_r[k] : 1;
                P.off[k] = d >= 0 ? s.rank_offset[d] : 0;
                P.gfirst[k] = 0;
                P.glast[k] = d >= 0 ? s.overall_size[d] - 1 : 0;
                const auto& bd = p.bound[k];
                auto resolve = [&](int kind, int off) { return (kind == 2 ? P.glast[k] : (kind == 1 ? P.gfirst[k] : 0)) + off; };
                if (bd.lo_kind >= 0) pb.b[k] = std::max<int64_t>(pb.b[k], resolve(bd.lo_kind, bd.lo_off) - P.off[k]);
                if (bd.hi_kind >= 0) pb.e[k] = std::min<int64_t>(pb.e[k], resolve(bd.hi_kind, bd.hi_off) - P.off[k] + 1);
            }
            if (pb.empty()) continue;
            P.xb = int(pb.b[0]); P.xe = int(pb.e[0]);
            P.yb = int(pb.b[1]); P.ye = int(pb.e[1]);
            P.zb = int(pb.b[2]); P.ze = int(pb.e[2]);
            P.SX = P.SY = 0;
            for (size_t k = 0; k < p.acc.size(); k++) {
                const Var& v = var_of(s, p.acc[k].var);
                const int slot = v.slot_of(t + p.acc[k].toff);
                int64_t moff = 0;      // constant misc-dim indices select a sub-array
                int mi = 0;
                for (auto& d : v.dims)
                    if (d.spec.kind == DIM_MISC) moff += (p.acc[k].misc[mi++] - d.spec.misc_first) * d.stride;
                P.ptr[k] = v.slot_ptr(slot) + size_t(v.origin_offset() + moff) * v.elem_bytes;
                const Dim* d0 = sh <= 0 ? v.domain_dim(0 - sh) : nullptr;
                const Dim* d1 = sh <= 1 ? v.domain_dim(1 - sh) : nullptr;
                const Dim* d2 = v.domain_dim(2 - sh);
                P.sx[k] = d0 ? d0->stride : 0;
                P.sy[k] = d1 ? d1->stride : 0;
                P.sz[k] = d2 ? d2->stride : 0;
                // full-rank var declared in the solution's dim order: must share the solution-wide geometry (a var that
                // permutes the dims -- H(y, z, x) -- is addressed through its own strides; the emitter gives it mask 15)
                bool in_order = true;
                int last_di = -1;
                for (auto& d : v.dims)
                    if (d.spec.kind == DIM_DOMAIN) { in_order = in_order && d.spec.domain_index > last_di; last_di = d.spec.domain_index; }
                if (d0 && d1 && d2 && in_order) {
                    if (P.SX == 0) { P.SX = int(d0->stride); P.SY = int(d1->stride); }
                    if (d0->stride != P.SX || d1->stride != P.SY || d2->stride != 1)
                        return set_error(YB_EUNSUPPORTED, "var '%s' does not share the solution's padded geometry", v.spec.name.c_str());
                }
            }
            // A scratch var whose first writer in this stage is conditional starts from zero
            // (/root/reference/src/kernel/lib/stencil_calc.cpp:85-109).
            if (p.is_scratch)
                for (int o : p.outs) {
                    const int si = p.acc[o].var - nreg;
                    if (si < 0 || scratch_written[si]) continue;
                    scratch_written[si] = 1;
                    if (p.conditional) YB_CUDA(cudaMemsetAsync(scratch[si].dev, 0, scratch[si].bytes(), st));
                }
            // Sweep variant: TMA-staged shared-memory planes (yb_gen_sweep.cuh), for whole-box launches of parts that have one.
            const int fi = g.elem_bytes == 8 ? 1 : 0, mi = s.fp_mode == 0 ? 0 : 1;
            // (TMA boxes and the consumers' 128-bit accesses need the box to start on a 16-byte boundary in z)
            if (sweep && p.sweep.fn[fi][mi].narrow && P.SX != 0 && pb.e[0] - pb.b[0] >= sweep_min_x && pb.e[2] - pb.b[2] >= 32 &&
                pb.b[2] % (16 / g.elem_bytes) == 0) {
                GenSweepParams SP;
                memset(&SP, 0, sizeof SP);
                SP.g = P;
                const GenSweep& sw = p.sweep;
                bool first = true;
                std::string key;
                for (size_t k = 0; k < sw.streams.size(); k++) {
                    const GenSweepStream& ss = sw.streams[k];
                    const Var& v = var_of(s, p.acc[ss.acc].var);
                    const Dim *d0 = v.domain_dim(0), *d1 = v.domain_dim(1), *d2 = v.domain_dim(2);
                    if (!d0 || !d1 || !d2) return set_error(YB_EUNSUPPORTED, "sweep kernel: var '%s' is not full rank", v.spec.name.c_str());
                    if (first) { SP.px = int(d0->pad_l); SP.py = int(d1->pad_l); SP.pz = int(d2->pad_l); first = false; }
                    if (d0->pad_l != SP.px || d1->pad_l != SP.py || d2->pad_l != SP.pz)
                        return set_error(YB_EUNSUPPORTED, "sweep kernel: var '%s' does not share the solution's padded geometry", v.spec.name.c_str());
                    key.push_back(char('0' + v.slot_of(t + p.acc[ss.acc].toff)));
                }
                auto mk = std::make_pair(&p, key);
                auto it = sweep_maps.find(mk);
                if (it == sweep_maps.end()) {
                    std::vector<CUtensorMap> hm(sw.streams.size());
                    for (size_t k = 0; k < sw.streams.size(); k++) {
                        const GenSweepStream& ss = sw.streams[k];
                        const Var& v = var_of(s, p.acc[ss.acc].var);
                        if (int rc = make_var_tensor_map(&hm[k], v, v.slot_of(t + p.acc[ss.acc].toff), ss.pz, ss.rows)) return rc;
                    }
                    void* dm = nullptr;
                    YB_CUDA(cudaMalloc(&dm, hm.size() * sizeof(CUtensorMap)));
                    YB_CUDA(cudaMemcpy(dm, hm.data(), hm.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice));
                    it = sweep_maps.emplace(mk, dm).first;
                }
                SP.maps = static_cast<const CUtensorMap*>(it->second);
                SP.nzb = int((pb.e[2] - pb.b[2] + sw.tz - 1) / sw.tz);
                SP.nyb = int((pb.e[1] - pb.b[1] + sw.ty - 1) / sw.ty);
                const int64_t nxb = pb.e[0] - pb.b[0];
                if (sweep_lx > 0) {
                    SP.lx = int(std::min<int64_t>(sweep_lx, nxb));
                } else {
                    // chunk count that minimises (waves of CTAs) x (chunk length + pipeline fill): long chunks amortise the
                    // x reach re-read at every chunk start, short ones fill the last wave
                    const int64_t slots = int64_t(num_sms) * sw.occ, tiles = int64_t(SP.nzb) * SP.nyb;
                    double best = 1e30;
                    int64_t best_l = nxb;
                    for (int64_t nc = 1; nc <= 64 && nc <= nxb; nc++) {
                        const int64_t l = (nxb + nc - 1) / nc;
                        const int64_t waves = (tiles * nc + slots - 1) / slots;
                        const double cost = double(waves) * (double(l) + 8.0);
                        if (cost < best * 0.999) { best = cost; best_l = l; }
                    }
                    SP.lx = int(best_l);
                }
                SP.nchunks = int((nxb + SP.lx - 1) / SP.lx);
                GenSweepFn sfn = sw.fn[fi][mi].pick(wide);
                if (!sweep_attr[(const void*)sfn]) {
                    YB_CUDA(cudaFuncSetAttribute((const void*)sfn, cudaFuncAttributeMaxDynamicSharedMemorySize, sw.smem));
                    sweep_attr[(const void*)sfn] = true;
                }
                const int64_t nb = int64_t(SP.nzb) * SP.nyb * SP.nchunks;
                if (nb >= (int64_t(1) << 31)) return set_error(YB_EUNSUPPORTED, "domain too large for the sweep kernels");
                sfn<<<unsigned(nb), sw.threads, sw.smem, st>>>(SP);
                YB_CUDA(cudaGetLastError());
                sweep_launches++;
                n++;
                continue;
            }
            // L2 prefetch list: full-rank vars the part only reads (distinct storage)
            P.npf = 0;
            P.pfd = pf_dist;
            if (pf_dist > 0 && P.SX != 0) {
                for (size_t k = 0; k < p.acc.size(); k++) {
                    if (P.sx[k] != P.SX || P.sy[k] != P.SY || P.sz[k] != 1) continue;
                    if (std::find(p.outs.begin(), p.outs.end(), int(k)) != p.outs.end()) continue;
                    bool dup = false;
                    for (int q = 0; q < P.npf; q++) dup = dup || P.ptr[P.pf[q]] == P.ptr[k];
                    if (!dup) P.pf[P.npf++] = (unsigned char)k;
                }
            }
            GenKernelFn fn = p.fn[g.elem_bytes == 8 ? 1 : 0][s.fp_mode == 0 ? 0 : 1].pick(wide);
            const int rows_per_block = GEN_BY * gen_np(g.elem_bytes);
            P.nzb = int((pb.e[2] - pb.b[2] + GEN_BZ - 1) / GEN_BZ);
            P.nyb = int((pb.e[1] - pb.b[1] + rows_per_block - 1) / rows_per_block);
            P.nxb = int((pb.e[0] - pb.b[0] + GEN_BX - 1) / GEN_BX);
            // y chunk: keep (x span of the stencil) planes of every full-rank var of the part within the L2 budget
            P.ychunk = P.nyb;
            if (l2_mb > 0 && P.SX != 0 && P.nxb > 1) {
                int nfull = 0;
                for (size_t k = 0; k < p.acc.size(); k++) {
                    if (P.sx[k] != P.SX) continue;
                    bool dup = false;
                    for (size_t q = 0; q < k; q++) dup = dup || P.ptr[q] == P.ptr[k];
                    nfull += !dup;
                }
                const int64_t span = 2 * std::max<int64_t>(s.spec.uniform_pad[std::max(0, 0 - sh)], 0) + 1;
                const double row_bytes = double(P.SY) * g.elem_bytes * double(span) * std::max(nfull, 1);
                int64_t rows = int64_t(double(l2_mb) * 1048576.0 / row_bytes);
                int64_t yc = std::max<int64_t>(rows / rows_per_block, 4);
                if (yc < P.nyb) {
                    // equalise the chunks
                    const int64_t nch = (P.nyb + yc - 1) / yc;
                    P.ychunk = int((P.nyb + nch - 1) / nch);
                }
            }
            const int64_t nblocks = int64_t(P.nzb) * P.nyb * P.nxb;
            if (nblocks >= (int64_t(1) << 31)) return set_error(YB_EUNSUPPORTED, "domain too large for the generated kernels");
            fn<<<unsigned(nblocks), GEN_BLOCK, 0, st>>>(P);
            YB_CUDA(cudaGetLastError());
            n++;
        }
        return n;
    }
};

}  // namespace

int gen_registry_size() { return int(sizeof(kGen) / sizeof(kGen[0])); }
const char* gen_registry_name(int i) { return kGen[i].name; }

int gen_registry_create(const std::string& name, int elem_bytes, StencilSpec& spec, std::unique_ptr<Engine>& eng) {
    for (auto& e : kGen) {
        if (name != e.name) continue;
        auto ge = std::unique_ptr<GenEngine>(new GenEngine());
        e.describe(ge->g);
        const GenStencil& g = ge->g;
        if (elem_bytes != 0 && elem_bytes != g.elem_bytes)
            return set_error(YB_EUNSUPPORTED, "solution '%s' is generated for %d-byte elements (asked for %d)", e.name, g.elem_bytes, elem_bytes);
        spec = StencilSpec();
        spec.name = g.name;
        spec.description = "generated from the reference DSL definition by yask_b200/emitter";
        spec.step_dim = g.step_dim;
        spec.domain_dims = g.domain_dims;
        spec.elem_bytes = g.elem_bytes;
        ge->nreg = 0;
        bool seen_scratch = false;
        for (auto& gv : g.vars) {
            if (gv.is_scratch) { seen_scratch = true; continue; }     // scratch vars come last in the table
            if (seen_scratch) return set_error(YB_EINVAL, "generated table of '%s': scratch var before a regular var", e.name);
            spec.vars.push_back(var_spec_of(g, gv));
            ge->nreg++;
        }
        // one padded geometry for all vars: pad every dim to the largest halo any var has there
        for (auto& gv : g.vars)
            for (size_t k = 0; k < g.domain_dims.size() && k < 3; k++)
                spec.uniform_pad[k] = std::max<int64_t>(spec.uniform_pad[k], std::max(gv.halo_l[k], gv.halo_r[k]));
        for (auto& gs : g.stages) {
            StageSpec st;
            st.name = gs.name;
            for (auto& p : gs.parts) {
                st.fp_ops += p.fp_ops; st.reads += p.reads; st.writes += p.writes;
                for (int o : p.outs)
                    if (p.acc[o].var < ge->nreg) {
                        st.outputs.push_back(p.acc[o].var);
                        if (p.acc[o].toff != 0) st.out_step_off = p.acc[o].toff;    // +1, or -1 for reverse-time solutions
                    }
                for (auto& a : p.acc)
                    if (a.var < ge->nreg) st.inputs.push_back(a.var);
            }
            spec.stages.push_back(st);
        }
        eng = std::move(ge);
        return 0;
    }
    return YB_EINVAL;
}

}  // namespace yb
