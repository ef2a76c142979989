// C ABI of libyask_b200 (include/yask_b200.h): solution life cycle, rank geometry, var storage in
// HBM, slice copies, the run loop and stats.  Host-side counterpart of the reference's
// StencilContext (/root/reference/src/kernel/lib/{context,soln_apis,setup}.cpp) -- integer
// bookkeeping only; all arithmetic happens in the engines' CUDA kernels.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>

#include "yb_core.h"
#include "yb_halo.h"
#include "yb_points.h"
#include "yb_slices.h"

namespace yb {

static thread_local char g_err[1024] = "";

int set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
    return code;
}

Solution::~Solution() {
    if (device >= 0) {
        cudaSetDevice(device);
        halo_free(halo); halo = nullptr;
        for (auto& v : vars) {
            if (v.store) v.store.reset();          // frees when this was the last var sharing the allocation
            else if (v.dev) cudaFree(v.dev);
            v.dev = nullptr;
        }
        for (auto& pe : pending_events) { cudaEventDestroy(pe.first); cudaEventDestroy(pe.second); }
        if (stage_dev) cudaFree(stage_dev);
        if (stage_host) cudaFreeHost(stage_host);
        if (own_stream) cudaStreamDestroy(own_stream);
        if (comm_stream) cudaStreamDestroy(comm_stream);
    }
    slices_source_gone(*this);   // consumers of this solution's vars (var links) refuse to run from now on
    points_free(points);     // device tables are released on `device`, selected above
    slices_free(slices);
    slices_free(injectors);
    slices_free(correlators);
}

static int check_dim(const Solution* s, int dim) {
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (dim < 0 || dim >= s->ndd) return set_error(YB_EINVAL, "domain dim index %d out of range [0,%d)", dim, s->ndd);
    return 0;
}
static int check_var(const Solution* s, int var) {
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (var < 0 || var >= int(s->vars.size())) return set_error(YB_EINVAL, "var index %d out of range", var);
    return 0;
}

// ---- geometry (setup_rank + update_var_info + YkVarBase::resize) ------------------------------------
// Per-rank sizes follow /root/reference/src/kernel/lib/setup.cpp:462-503: when only the overall
// size is given, every rank gets ceil(overall/nranks) and the last one the remainder.
static int compute_rank_geometry(Solution& s) {
    for (int d = 0; d < s.ndd; d++) {
        int64_t nr = s.num_ranks[d], ri = s.rank_index[d];
        if (nr < 1) return set_error(YB_EINVAL, "num_ranks must be >= 1");
        if (ri < 0 || ri >= nr) return set_error(YB_EINVAL, "rank index %lld out of range [0,%lld)", (long long)ri, (long long)nr);
        int64_t rs = s.req_rank_size[d], os = s.req_overall_size[d];
        if (rs > 0 && os <= 0) {
            // rank size given: all ranks are assumed to use the same size
            s.rank_size[d] = rs;
            s.overall_size[d] = rs * nr;
            s.rank_offset[d] = rs * ri;
        } else if (os > 0) {
            int64_t per = (os + nr - 1) / nr;
            int64_t last = os - per * (nr - 1);
            if (last <= 0) return set_error(YB_EINVAL, "overall size %lld too small for %lld ranks", (long long)os, (long long)nr);
            if (rs > 0 && rs * nr != os && nr > 1)
                return set_error(YB_EINVAL, "rank size and overall size are inconsistent in dim %d", d);
            s.rank_size[d] = (rs > 0 && nr == 1) ? os : (ri == nr - 1 ? last : per);
            s.overall_size[d] = os;
            s.rank_offset[d] = per * ri;
        } else {
            return set_error(YB_EINVAL, "domain size of dim '%s' was not set", s.spec.domain_dims[d].c_str());
        }
    }
    return 0;
}

// Every rank of a split dim must be at least as wide as the widest halo of the solution's vars in that dim, or a halo exchange
// would have to send planes it does not own (/root/reference/src/kernel/lib/setup.cpp:709-713, 764-772).  The test is on the
// grid's smallest rank -- the last one, which takes the remainder -- so that every rank refuses the grid, not only the thin one:
// a rank prepared alongside a refused neighbour would wait for it forever in its first exchange.
static int check_min_rank_size(const Solution& s) {
    for (int d = 0; d < s.ndd; d++) {
        const int64_t nr = s.num_ranks[d];
        if (nr <= 1) continue;
        int64_t halo = 0;
        for (const Var& v : s.vars)
            if (!v.spec.user_var)
                if (const Dim* dd = v.domain_dim(d)) halo = std::max({halo, dd->spec.halo_l, dd->spec.halo_r});
        const int64_t os = s.overall_size[d];
        const int64_t smallest = std::min(s.rank_size[d], os - (os + nr - 1) / nr * (nr - 1));
        if (smallest < halo)
            return set_error(YB_EINVAL, "local-domain size of %lld in '%s' dim is less than minimum size of %lld, which is based on stencil "
                                        "halos and temporal wave-front sizes", (long long)smallest, s.spec.domain_dims[d].c_str(), (long long)halo);
    }
    return 0;
}

void compute_var_geometry(Solution& s, Var& v) {
    const int align_elems = 128 / v.elem_bytes;  // 128-B rows
    int nd = int(v.dims.size());
    int last_domain = -1;
    for (int i = 0; i < nd; i++)
        if (v.dims[i].spec.kind == DIM_DOMAIN) last_domain = i;
    for (int i = 0; i < nd; i++) {
        Dim& d = v.dims[i];
        if (d.spec.kind == DIM_STEP) {
            if (v.spec.fixed_size) v.spec.step_alloc = int(v.spec.fixed_sizes[i]);
            d.domain = v.spec.step_alloc; d.alloc = d.domain; d.stride = 0; continue;
        }
        if (d.spec.kind == DIM_MISC) { d.domain = d.spec.misc_size; d.alloc = d.domain; d.pad_l = d.pad_r = 0; continue; }
        int dd = d.spec.domain_index;
        d.domain = s.rank_size[dd];
        d.rank_offset = s.rank_offset[dd];
        if (v.spec.fixed_size) { d.domain = v.spec.fixed_sizes[i]; d.rank_offset = 0; }
        int64_t pl = std::max({d.spec.halo_l, d.min_pad_l, s.min_pad[dd], s.spec.uniform_pad[dd]});
        int64_t pr = std::max({d.spec.halo_r, d.min_pad_r, s.min_pad[dd], s.spec.uniform_pad[dd]});
        if (i == last_domain) {
            // unit-stride dim: domain origin on a 128-B boundary, pitch a multiple of 128 B
            pl = (pl + align_elems - 1) / align_elems * align_elems;
            int64_t a = pl + d.domain + pr;
            a = (a + align_elems - 1) / align_elems * align_elems;
            pr = a - pl - d.domain;
        }
        d.pad_l = pl; d.pad_r = pr;
        d.alloc = pl + d.domain + pr;
    }
    // Storage order: domain dims innermost (declared order, last one unit-stride), misc dims outside them -- a var
    // with misc dims is an array of identically shaped domain boxes (the reference's default "outer misc" layout).
    int64_t stride = 1;
    for (int pass = 0; pass < 2; pass++)
        for (int i = nd - 1; i >= 0; i--) {
            Dim& d = v.dims[i];
            if (d.spec.kind == DIM_STEP) continue;
            if ((pass == 0) != (d.spec.kind == DIM_DOMAIN)) continue;
            d.stride = stride;
            stride *= d.alloc;
        }
    v.slot_elems = std::max<int64_t>(stride, 1);
    // keep every slot 256-B aligned
    int64_t a256 = 256 / v.elem_bytes;
    v.slot_elems = (v.slot_elems + a256 - 1) / a256 * a256;
    v.first_valid_step = 0;
}

// device storage of a var, owned through Var::store
static cudaError_t alloc_var_storage(Var& v) {
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, std::max<size_t>(v.bytes(), 256));
    if (e != cudaSuccess) return e;
    v.store = std::shared_ptr<void>(p, [](void* q) { cudaFree(q); });
    v.dev = p;
    return cudaSuccess;
}

static int ensure_stage(Solution& s, size_t bytes) {
    if (s.stage_bytes >= bytes) return 0;
    if (s.stage_dev) cudaFree(s.stage_dev);
    s.stage_dev = nullptr; s.stage_bytes = 0;
    YB_CUDA(cudaMalloc(&s.stage_dev, bytes));
    s.stage_bytes = bytes;
    return 0;
}

// Resolve a [first,last] slice (global indices, step first) into step range + BoxCopy.
struct Slice {
    int64_t t0 = 0, t1 = 0;
    BoxCopy bc{};
    int64_t elems_per_step = 1;
    int64_t g0[4] = {0, 0, 0, 0};   // global index of the box origin: last three dims, then the leading 4th dim
};

static int resolve_slice(const Solution& s, const Var& v, const int64_t* first, const int64_t* last, bool check_steps, Slice& sl) {
    int nd = int(v.dims.size());
    int k = 0;
    sl.bc.nd = 0; sl.bc.var_off = 0; sl.elems_per_step = 1;
    int nns = nd - (v.has_step() ? 1 : 0);
    if (nns > 4) return set_error(YB_EUNSUPPORTED, "var '%s': more than 4 non-step dims", v.spec.name.c_str());
    for (int i = 0; i < nd; i++) {
        const Dim& d = v.dims[i];
        int64_t f = first[i], l = last[i];
        if (l < f) return set_error(YB_ERANGE, "var '%s' dim '%s': last index %lld < first %lld", v.spec.name.c_str(), d.spec.name.c_str(), (long long)l, (long long)f);
        if (d.spec.kind == DIM_STEP) {
            if (check_steps && (f < v.first_valid_step || l > v.last_valid_step()))
                return set_error(YB_ERANGE, "var '%s': step indices [%lld,%lld] outside the valid steps [%lld,%lld]", v.spec.name.c_str(),
                                 (long long)f, (long long)l, (long long)v.first_valid_step, (long long)v.last_valid_step());
            if (l - f + 1 > v.step_alloc())
                return set_error(YB_ERANGE, "var '%s': step range longer than the %d allocated steps", v.spec.name.c_str(), v.step_alloc());
            sl.t0 = f; sl.t1 = l;
            continue;
        }
        int64_t lo, hi;  // first/last local (allocated) global index
        if (d.spec.kind == DIM_DOMAIN) { lo = d.rank_offset - d.pad_l; hi = d.rank_offset + d.domain + d.pad_r - 1; }
        else { lo = d.spec.misc_first; hi = d.spec.misc_first + d.domain - 1; }
        if (f < lo || l > hi)
            return set_error(YB_ERANGE, "var '%s' dim '%s': indices [%lld,%lld] outside the allocation [%lld,%lld]", v.spec.name.c_str(),
                             d.spec.name.c_str(), (long long)f, (long long)l, (long long)lo, (long long)hi);
        sl.bc.n[k] = l - f + 1;
        sl.bc.var_stride[k] = d.stride;
        sl.bc.var_off += (f - lo) * d.stride;
        sl.elems_per_step *= sl.bc.n[k];
        k++;
    }
    sl.bc.nd = k;
    // global index triple of the box origin (left padded with 0)
    int kk = 0;
    for (int i = 0; i < nd; i++) {
        if (v.dims[i].spec.kind == DIM_STEP) continue;
        if (k <= 3) sl.g0[3 - k + kk] = first[i];
        else if (k == 4) { if (kk == 0) sl.g0[3] = first[i]; else sl.g0[kk - 1] = first[i]; }
        kk++;
    }
    (void)s;
    return 0;
}

static int slice_copy(Solution& s, int var, void* buf, const int64_t* first, const int64_t* last, int64_t* n_done, bool to_var, bool buf_on_device) {
    if (int rc = check_var(&s, var)) return rc;
    if (!s.prepared) return set_error(YB_ESTATE, "var storage is not allocated: call prepare_solution first");
    if (!buf) return set_error(YB_EINVAL, "null buffer");
    Var& v = s.vars[var];
    Slice sl;
    // writes do not check the step window (set_element semantics); reads do.
    if (int rc = resolve_slice(s, v, first, last, !to_var, sl)) return rc;
    YB_CUDA(cudaSetDevice(s.device));
    cudaStream_t st = s.stream();
    const int eb = v.elem_bytes;
    int64_t done = 0;
    // chunk along the outermost box dim so the staging buffer stays bounded
    const size_t CHUNK = size_t(256) << 20;
    if (to_var)
        if (int rc = slices_var_write_waits(s)) return rc;
    for (int64_t t = sl.t0; t <= sl.t1; t++) {
        char* slot = v.slot_ptr(v.slot_of(t));
        char* hb = static_cast<char*>(buf) + size_t(t - sl.t0) * sl.elems_per_step * eb;
        if (buf_on_device) {
            if (int rc = launch_box_copy(slot, hb, sl.bc, eb, to_var, st)) return rc;
        } else if (sl.bc.nd == 0) {
            if (to_var) YB_CUDA(cudaMemcpyAsync(slot + sl.bc.var_off * eb, hb, eb, cudaMemcpyHostToDevice, st));
            else YB_CUDA(cudaMemcpyAsync(hb, slot + sl.bc.var_off * eb, eb, cudaMemcpyDeviceToHost, st));
            YB_CUDA(cudaStreamSynchronize(st));
        } else {
            int64_t inner = sl.elems_per_step / sl.bc.n[0];
            int64_t rows_per_chunk = std::max<int64_t>(1, int64_t(CHUNK / std::max<size_t>(1, size_t(inner) * eb)));
            rows_per_chunk = std::min(rows_per_chunk, sl.bc.n[0]);
            if (int rc = ensure_stage(s, size_t(rows_per_chunk) * inner * eb)) return rc;
            for (int64_t r0 = 0; r0 < sl.bc.n[0]; r0 += rows_per_chunk) {
                int64_t nr = std::min(rows_per_chunk, sl.bc.n[0] - r0);
                BoxCopy bc = sl.bc;
                bc.n[0] = nr;
                bc.var_off += r0 * sl.bc.var_stride[0];
                size_t nb = size_t(nr) * inner * eb;
                char* hchunk = hb + size_t(r0) * inner * eb;
                if (to_var) {
                    YB_CUDA(cudaMemcpyAsync(s.stage_dev, hchunk, nb, cudaMemcpyHostToDevice, st));
                    if (int rc = launch_box_copy(slot, s.stage_dev, bc, eb, true, st)) return rc;
                } else {
                    if (int rc = launch_box_copy(slot, s.stage_dev, bc, eb, false, st)) return rc;
                    YB_CUDA(cudaMemcpyAsync(hchunk, s.stage_dev, nb, cudaMemcpyDeviceToHost, st));
                }
                YB_CUDA(cudaStreamSynchronize(st));  // staging buffer is reused
            }
        }
        done += sl.elems_per_step;
        if (to_var) v.update_valid_step(t);
    }
    if (to_var)
        if (int rc = slices_var_write_records(s)) return rc;
    if (to_var && s.halo) halo_mark_dirty(s, var);
    if (n_done) *n_done = done;
    return 0;
}

}  // namespace yb

using namespace yb;

// ===============================================================================================
// C ABI
// ===============================================================================================
extern "C" {

const char* yb_version_string(void) { return "4.05.04-b200.r1"; }
const char* yb_last_error(void) { return g_err; }

int yb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
int yb_num_stencils(void) { return registry_size(); }
const char* yb_stencil_name(int i) { return registry_name(i); }

int yb_solution_create(yb_solution** out, const char* stencil, int radius, int elem_bytes) {
    if (!out || !stencil) return set_error(YB_EINVAL, "null argument");
    *out = nullptr;
    auto s = std::make_unique<Solution>();
    if (elem_bytes != 0 && elem_bytes != 4 && elem_bytes != 8) return set_error(YB_EINVAL, "element bytes must be 4 or 8");
    if (int rc = registry_create(stencil, radius, elem_bytes, s->spec, s->engine)) return rc;
    s->ndd = int(s->spec.domain_dims.size());
    for (auto& vs : s->spec.vars) {
        Var v;
        v.spec = vs;
        v.elem_bytes = s->spec.elem_bytes;
        for (auto& ds : vs.dims) { Dim d; d.spec = ds; v.dims.push_back(d); }
        s->vars.push_back(std::move(v));
    }
    *out = reinterpret_cast<yb_solution*>(s.release());
    return 0;
}

#define SOL(s) reinterpret_cast<Solution*>(s)
#define CSOL(s) reinterpret_cast<const Solution*>(s)

int yb_solution_destroy(yb_solution* s) {
    delete SOL(s);
    return 0;
}
const char* yb_solution_name(const yb_solution* s) { return s ? CSOL(s)->spec.name.c_str() : ""; }
const char* yb_solution_target(const yb_solution*) { return "sm_90a"; }
int yb_solution_elem_bytes(const yb_solution* s) { return s ? CSOL(s)->spec.elem_bytes : 0; }
int yb_solution_num_domain_dims(const yb_solution* s) { return s ? CSOL(s)->ndd : 0; }
const char* yb_solution_domain_dim_name(const yb_solution* s, int i) {
    if (check_dim(CSOL(s), i)) return "";
    return CSOL(s)->spec.domain_dims[i].c_str();
}
const char* yb_solution_step_dim_name(const yb_solution* s) { return s ? CSOL(s)->spec.step_dim.c_str() : ""; }

static int not_prepared(Solution* s, const char* what) {
    if (s->prepared) return set_error(YB_ESTATE, "%s is not allowed after prepare_solution()", what);
    return 0;
}

int yb_set_rank_domain_size(yb_solution* s_, int dim, int64_t n) {
    Solution* s = SOL(s_);
    if (int rc = check_dim(s, dim)) return rc;
    if (int rc = not_prepared(s, "set_rank_domain_size")) return rc;
    if (n < 0) return set_error(YB_EINVAL, "domain size must not be negative");
    s->req_rank_size[dim] = n;            // 0 = derive from the overall size (settings.cpp:196-200)
    if (n > 0) s->req_overall_size[dim] = 0;
    return 0;
}
int yb_set_overall_domain_size(yb_solution* s_, int dim, int64_t n) {
    Solution* s = SOL(s_);
    if (int rc = check_dim(s, dim)) return rc;
    if (int rc = not_prepared(s, "set_overall_domain_size")) return rc;
    if (n < 0) return set_error(YB_EINVAL, "domain size must not be negative");
    s->req_overall_size[dim] = n;         // 0 = derive from the rank size
    if (n > 0) s->req_rank_size[dim] = 0;
    return 0;
}
int yb_set_num_ranks(yb_solution* s_, int dim, int64_t n) {
    Solution* s = SOL(s_);
    if (int rc = check_dim(s, dim)) return rc;
    if (int rc = not_prepared(s, "set_num_ranks")) return rc;
    if (n < 1) return set_error(YB_EINVAL, "number of ranks must be positive");
    s->num_ranks[dim] = n;
    return 0;
}
int yb_set_rank_index(yb_solution* s_, int dim, int64_t i) {
    Solution* s = SOL(s_);
    if (int rc = check_dim(s, dim)) return rc;
    if (int rc = not_prepared(s, "set_rank_index")) return rc;
    s->rank_index[dim] = i;
    return 0;
}
int yb_set_min_pad_size(yb_solution* s_, int dim, int64_t n) {
    Solution* s = SOL(s_);
    if (int rc = check_dim(s, dim)) return rc;
    if (int rc = not_prepared(s, "set_min_pad_size")) return rc;
    if (n < 0) return set_error(YB_EINVAL, "pad must be non-negative");
    s->min_pad[dim] = n;
    return 0;
}
int64_t yb_get_rank_domain_size(const yb_solution* s, int dim) {
    if (check_dim(CSOL(s), dim)) return -1;
    return CSOL(s)->rank_size[dim] > 0 ? CSOL(s)->rank_size[dim] : CSOL(s)->req_rank_size[dim];
}
int64_t yb_get_overall_domain_size(const yb_solution* s, int dim) {
    if (check_dim(CSOL(s), dim)) return -1;
    return CSOL(s)->overall_size[dim] > 0 ? CSOL(s)->overall_size[dim] : CSOL(s)->req_overall_size[dim];
}
int64_t yb_get_num_ranks(const yb_solution* s, int dim) { return check_dim(CSOL(s), dim) ? -1 : CSOL(s)->num_ranks[dim]; }
int64_t yb_get_rank_index(const yb_solution* s, int dim) { return check_dim(CSOL(s), dim) ? -1 : CSOL(s)->rank_index[dim]; }
int64_t yb_get_first_rank_domain_index(const yb_solution* s, int dim) { return check_dim(CSOL(s), dim) ? -1 : CSOL(s)->rank_offset[dim]; }
int64_t yb_get_last_rank_domain_index(const yb_solution* s, int dim) {
    return check_dim(CSOL(s), dim) ? -1 : CSOL(s)->rank_offset[dim] + CSOL(s)->rank_size[dim] - 1;
}

int yb_set_option(yb_solution* s_, const char* key, const char* value) {
    Solution* s = SOL(s_);
    if (!s || !key || !value) return set_error(YB_EINVAL, "null argument");
    std::string k = key, v = value;
    if (k == "fp_mode") {
        int m = atoi(value);
        if (m < 0 || m > 2) return set_error(YB_EINVAL, "fp_mode must be 0, 1 or 2");
        s->fp_mode = m;
    } else if (k == "auto_tune") {
        s->tuner = Solution::InRunTuner();
        s->tuner.enabled = atoi(value) != 0;
    } else if (k == "point_launches" || k == "point_groups" || k == "slice_launches" || k == "slice_injector_groups" ||
               k == "slice_injector_launches" || k == "slice_correlator_launches") {
        return set_error(YB_EINVAL, "option '%s' is read-only", key);
    } else if (k == "overlap_comms" || k == "min_exterior" || k == "fused_halo" || k == "dma_halo") {
        // consumed by the halo engine at run time
    } else if (s->engine->set_option(*s, k, v) != 0) {
        return set_error(YB_EINVAL, "unknown option '%s'", key);
    }
    s->options[k] = v;
    return 0;
}
int yb_get_option(const yb_solution* s_, const char* key, char* value, size_t n) {
    const Solution* s = CSOL(s_);
    if (!s || !key || !value || !n) return set_error(YB_EINVAL, "null argument");
    std::string v;
    if (std::string(key) == "fp_mode") v = std::to_string(s->fp_mode);
    else if (std::string(key) == "point_launches") v = std::to_string(s->points ? s->points->launches : 0);   // read-only
    else if (std::string(key) == "point_groups") v = points_groups_text(*s);                                    // read-only
    else if (std::string(key) == "slice_launches") v = std::to_string(s->slices ? s->slices->launches : 0);   // read-only
    else if (std::string(key) == "slice_injector_groups") v = slice_injector_groups_text(*s);                   // read-only
    else if (std::string(key) == "slice_injector_launches") v = std::to_string(s->injectors ? s->injectors->launches : 0);   // read-only
    else if (std::string(key) == "slice_correlator_launches") v = std::to_string(s->correlators ? s->correlators->launches : 0);   // read-only
    else if (!s->engine->get_option(*s, key, v)) {
        auto it = s->options.find(key);
        if (it == s->options.end()) return set_error(YB_EINVAL, "unknown option '%s'", key);
        v = it->second;
    }
    snprintf(value, n, "%s", v.c_str());
    return 0;
}
int yb_set_stream(yb_solution* s_, void* st) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    s->user_stream = static_cast<cudaStream_t>(st);
    s->use_user_stream = true;
    return 0;
}

// Spare storage slots serve the temporal tile.  A rank grid drops them unless the engine keeps them for its fused rank-grid
// mode (Engine::plan_storage), which also pads for the deeper halos of that mode.
static void plan_storage(Solution& s) {
    if (s.multi_rank()) for (auto& v : s.vars) if (!v.dev) v.extra_slots = 0;
    s.engine->plan_storage(s);
}

int yb_solution_plan_geometry(yb_solution* s_) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (s->prepared) return 0;
    if (int rc = compute_rank_geometry(*s)) return rc;
    if (int rc = check_min_rank_size(*s)) return rc;
    plan_storage(*s);
    for (auto& v : s->vars) compute_var_geometry(*s, v);
    s->geometry_planned = true;
    if (int rc = s->engine->check_geometry(*s)) return rc;
    if (points_active(*s))
        if (int rc = points_plan(*s)) return rc;          // point sets given before the geometry are checked now
    return slices_plan(*s);                               // and so are slice recorders, injectors and correlators
}

int yb_solution_prepare(yb_solution* s_, int device) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (s->prepared) return set_error(YB_ESTATE, "solution already prepared");
    int ndev = yb_device_count();
    if (ndev <= 0) return set_error(YB_ECUDA, "no CUDA device available: the yask_b200 engine has no CPU fallback");
    if (device < 0 || device >= ndev) return set_error(YB_EINVAL, "device %d out of range [0,%d)", device, ndev);
    if (int rc = compute_rank_geometry(*s)) return rc;
    if (int rc = check_min_rank_size(*s)) return rc;
    s->geometry_planned = true;
    plan_storage(*s);
    // a size the kernels cannot address is refused before any storage is allocated
    for (auto& v : s->vars)
        if (!v.dev) compute_var_geometry(*s, v);
    if (int rc = s->engine->check_geometry(*s)) return rc;
    if (int rc = slices_plan(*s)) return rc;
    YB_CUDA(cudaSetDevice(device));
    s->device = device;
    if (!s->own_stream) YB_CUDA(cudaStreamCreateWithFlags(&s->own_stream, cudaStreamNonBlocking));
    if (!s->comm_stream) YB_CUDA(cudaStreamCreateWithFlags(&s->comm_stream, cudaStreamNonBlocking));
    for (auto& v : s->vars) {
        const int64_t fvs = v.first_valid_step;
        const size_t had = v.dev ? v.bytes() : 0;
        compute_var_geometry(*s, v);
        if (v.dev) {
            // storage came from fuse_vars before prepare: it must fit the geometry this solution needs
            if (v.bytes() != had) return set_error(YB_EINVAL, "var '%s' was fused with storage of %zu bytes but this solution needs %zu", v.spec.name.c_str(), had, v.bytes());
            v.first_valid_step = fvs;
            continue;
        }
        YB_CUDA(alloc_var_storage(v));
        // the reference zero-initialises storage (alloc.cpp); halo cells outside the global domain
        // keep whatever the user wrote there.
        YB_CUDA(cudaMemsetAsync(v.dev, 0, v.bytes(), s->stream()));
    }
    if (int rc = s->engine->prepare(*s)) return rc;
    points_preload();
    slices_preload();
    if (s->multi_rank()) {
        if (int rc = halo_prepare(*s)) return rc;
    }
    if (int rc = slices_prepare(*s)) return rc;       // frames and images of the slices added before prepare
    if (s->slices) s->slices->launches = 0;
    if (s->injectors) s->injectors->launches = 0;
    if (s->correlators) s->correlators->launches = 0;
    YB_CUDA(cudaStreamSynchronize(s->stream()));
    s->prepared = true;
    memset(&s->stats, 0, sizeof s->stats);
    if (s->points) {
        // the point tables follow the final geometry; a set this geometry refuses is reported by the first run
        s->points->stale = true;
        s->points->launches = 0;
        if (points_begin_run(*s) == YB_ECUDA) return YB_ECUDA;
    }
    return 0;
}
int yb_solution_is_prepared(const yb_solution* s) { return s && CSOL(s)->prepared; }

int yb_num_vars(const yb_solution* s) { return s ? int(CSOL(s)->vars.size()) : 0; }
int yb_var_index(const yb_solution* s, const char* name) {
    if (!s || !name) return set_error(YB_EINVAL, "null argument");
    for (size_t i = 0; i < CSOL(s)->vars.size(); i++)
        if (CSOL(s)->vars[i].spec.name == name) return int(i);
    return set_error(YB_EINVAL, "var '%s' not found in solution '%s'", name, CSOL(s)->spec.name.c_str());
}

int yb_var_info_get(const yb_solution* s_, int var, yb_var_info* out) {
    const Solution* s = CSOL(s_);
    if (int rc = check_var(s, var)) return rc;
    if (!out) return set_error(YB_EINVAL, "null output");
    const Var& v = s->vars[var];
    memset(out, 0, sizeof *out);
    snprintf(out->name, YB_NAME_LEN, "%s", v.spec.name.c_str());
    out->num_dims = int(v.dims.size());
    out->elem_bytes = v.elem_bytes;
    out->has_step = v.has_step();
    out->step_alloc = v.step_alloc();
    out->first_valid_step = v.first_valid_step;
    out->last_valid_step = v.last_valid_step();
    out->is_output = v.spec.is_output;
    out->halo_exchange_l1_norm = v.spec.l1_norm;
    out->slot_elems = v.slot_elems;
    out->storage_bytes = int64_t(v.bytes());
    for (int i = 0; i < out->num_dims && i < YB_MAX_DIMS; i++) {
        const Dim& d = v.dims[i];
        yb_dim_info& o = out->dims[i];
        snprintf(o.name, YB_NAME_LEN, "%s", d.spec.name.c_str());
        o.kind = d.spec.kind;
        o.domain_index = d.spec.kind == DIM_DOMAIN ? d.spec.domain_index : -1;
        o.rank_offset = d.rank_offset;
        o.domain_size = d.spec.kind == DIM_STEP ? v.step_alloc() : (d.spec.kind == DIM_MISC ? d.spec.misc_size : d.domain);
        o.left_halo = d.spec.halo_l; o.right_halo = d.spec.halo_r;
        o.left_pad = d.pad_l; o.right_pad = d.pad_r;
        o.alloc_size = d.alloc;
        o.first_misc_index = d.spec.misc_first;
        o.stride = d.stride;
    }
    return 0;
}

int yb_var_create(yb_solution* s_, const char* name, int ndims, const char* const* dim_names, const int64_t* sizes) {
    Solution* s = SOL(s_);
    if (!s || !name || (ndims > 0 && !dim_names)) return set_error(YB_EINVAL, "null argument");
    if (ndims < 0 || ndims > YB_MAX_DIMS) return set_error(YB_EINVAL, "a var may have at most %d dims", YB_MAX_DIMS);
    for (auto& v : s->vars)
        if (v.spec.name == name) return set_error(YB_EINVAL, "var '%s' already exists", name);
    Var v;
    v.spec.name = name;
    v.spec.user_var = true;
    v.spec.fixed_size = sizes != nullptr;
    v.elem_bytes = s->spec.elem_bytes;
    for (int i = 0; i < ndims; i++) {
        DimSpec d;
        d.name = dim_names[i];
        for (int j = 0; j < i; j++)
            if (d.name == dim_names[j]) return set_error(YB_EINVAL, "dim '%s' repeated in var '%s'", dim_names[i], name);
        if (d.name == s->spec.step_dim) {
            if (i != 0) return set_error(YB_EINVAL, "step dim '%s' must be the first dim of var '%s'", dim_names[i], name);
            d.kind = DIM_STEP;
        } else {
            d.kind = DIM_MISC;
            for (int k = 0; k < s->ndd; k++)
                if (d.name == s->spec.domain_dims[k]) { d.kind = DIM_DOMAIN; d.domain_index = k; }
            if (d.kind == DIM_MISC) d.misc_size = sizes ? sizes[i] : 1;
        }
        if (sizes) {
            if (sizes[i] < 1) return set_error(YB_EINVAL, "size of dim '%s' must be positive", dim_names[i]);
            v.spec.fixed_sizes.push_back(sizes[i]);
        }
        v.spec.dims.push_back(d);
    }
    v.spec.step_alloc = 1;
    for (auto& ds : v.spec.dims) { Dim d; d.spec = ds; v.dims.push_back(d); }
    if (v.spec.fixed_size) compute_var_geometry(*s, v);   // geometry of a fixed-size var is known at creation
    if (s->prepared) {
        YB_CUDA(cudaSetDevice(s->device));
        compute_var_geometry(*s, v);
        YB_CUDA(alloc_var_storage(v));
        YB_CUDA(cudaMemsetAsync(v.dev, 0, v.bytes(), s->stream()));
        if (s->halo) return set_error(YB_EUNSUPPORTED, "vars cannot be added to a prepared multi-rank solution");
    }
    s->vars.push_back(std::move(v));
    return int(s->vars.size()) - 1;
}

// yk_var::fuse_vars (/root/reference/src/kernel/lib/yk_var_apis.cpp:302-360): `var` of `s` becomes another reference to the
// storage of `src_var` of `src` (which may be the same solution).  Both must agree on element size, dims and allocation
// (is_storage_layout_identical); any storage `var` had is released; the valid-step window is taken from the source.
int yb_var_fuse(yb_solution* s_, int var, yb_solution* src_, int src_var) {
    Solution* s = SOL(s_);
    Solution* src = SOL(src_);
    if (int rc = check_var(s, var)) return rc;
    if (int rc = check_var(src, src_var)) return rc;
    Var& d = s->vars[var];
    Var& o = src->vars[src_var];
    if (&d == &o) return 0;
    if (s->halo || src->halo) return set_error(YB_EUNSUPPORTED, "fuse_vars: vars of a prepared multi-rank solution are mapped by their neighbours and cannot change storage");
    if (d.elem_bytes != o.elem_bytes || d.dims.size() != o.dims.size())
        return set_error(YB_EINVAL, "fuse_vars(): '%s' and '%s' differ in element size or number of dims", d.spec.name.c_str(), o.spec.name.c_str());
    for (size_t i = 0; i < d.dims.size(); i++)
        if (d.dims[i].spec.name != o.dims[i].spec.name || d.dims[i].spec.kind != o.dims[i].spec.kind)
            return set_error(YB_EINVAL, "fuse_vars(): dim %zu of '%s' is '%s' but '%s' in '%s'", i, d.spec.name.c_str(), d.dims[i].spec.name.c_str(),
                             o.dims[i].spec.name.c_str(), o.spec.name.c_str());
    // a var with spare slots (temporal tile) switches its live slot set at run time; a second view of the same storage would
    // not follow
    if (d.extra_slots || o.extra_slots)
        return set_error(YB_EUNSUPPORTED, "fuse_vars(): '%s' / '%s' carry spare storage slots of a temporal tile (block_steps); fuse before selecting it or not at all",
                         d.spec.name.c_str(), o.spec.name.c_str());
    if (!o.dev) {
        // source not allocated: this var becomes unallocated too (yk_var_api.hpp:1378-1383)
        if (s->prepared) return set_error(YB_ESTATE, "fuse_vars(): source var '%s' has no storage but '%s' belongs to a prepared solution", o.spec.name.c_str(), d.spec.name.c_str());
        d.store.reset(); d.dev = nullptr;
        return 0;
    }
    if (s->prepared || d.dev) {
        // geometry of `var` is known: it must match the source's allocation exactly
        bool same = d.step_alloc() == o.step_alloc() && d.extra_slots == o.extra_slots && d.slot_elems == o.slot_elems;
        for (size_t i = 0; i < d.dims.size() && same; i++)
            same = d.dims[i].alloc == o.dims[i].alloc && d.dims[i].pad_l == o.dims[i].pad_l && d.dims[i].stride == o.dims[i].stride &&
                   d.dims[i].domain == o.dims[i].domain;
        if (!same) return set_error(YB_EINVAL, "fuse_vars(): attempt to replace the storage of '%s' with the incompatible layout of '%s'", d.spec.name.c_str(), o.spec.name.c_str());
    } else {
        // not prepared yet: adopt the source's geometry now; prepare() checks that it is what the solution needs
        d.spec.step_alloc = o.spec.step_alloc;
        d.extra_slots = o.extra_slots;
        for (size_t i = 0; i < d.dims.size(); i++) {
            const DimSpec keep = d.dims[i].spec;
            d.dims[i] = o.dims[i];
            d.dims[i].spec = keep;
            d.dims[i].spec.halo_l = std::max(keep.halo_l, int64_t(0)); d.dims[i].spec.halo_r = std::max(keep.halo_r, int64_t(0));
        }
        d.slot_elems = o.slot_elems;
    }
    if (src->prepared) { cudaSetDevice(src->device); cudaStreamSynchronize(src->stream()); }
    if (!o.store) return set_error(YB_ESTATE, "fuse_vars(): storage of '%s' is not shareable", o.spec.name.c_str());
    d.store = o.store;
    d.dev = o.dev;
    d.first_valid_step = o.first_valid_step;
    if (s->prepared) {
        // tensor maps and cached pointers of the engine refer to the old storage
        YB_CUDA(cudaSetDevice(s->device));
        YB_CUDA(cudaStreamSynchronize(s->stream()));
        if (int rc = s->engine->prepare(*s)) return rc;
    }
    return 0;
}

int yb_var_set_min_pad(yb_solution* s_, int var, int dim, int64_t left, int64_t right) {
    Solution* s = SOL(s_);
    if (int rc = check_var(s, var)) return rc;
    if (int rc = not_prepared(s, "set_min_pad_size")) return rc;
    Var& v = s->vars[var];
    if (dim < 0 || dim >= int(v.dims.size()) || v.dims[dim].spec.kind != DIM_DOMAIN)
        return set_error(YB_EINVAL, "var '%s': dim %d is not a domain dim", v.spec.name.c_str(), dim);
    if (left >= 0) v.dims[dim].min_pad_l = left;
    if (right >= 0) v.dims[dim].min_pad_r = right;
    return 0;
}

int yb_var_set_slice(yb_solution* s, int var, const void* buf, const int64_t* first, const int64_t* last, int64_t* n) {
    return slice_copy(*SOL(s), var, const_cast<void*>(buf), first, last, n, true, false);
}
int yb_var_get_slice(yb_solution* s, int var, void* buf, const int64_t* first, const int64_t* last, int64_t* n) {
    return slice_copy(*SOL(s), var, buf, first, last, n, false, false);
}
int yb_var_set_slice_device(yb_solution* s, int var, const void* buf, const int64_t* first, const int64_t* last, int64_t* n) {
    return slice_copy(*SOL(s), var, const_cast<void*>(buf), first, last, n, true, true);
}
int yb_var_get_slice_device(yb_solution* s, int var, void* buf, const int64_t* first, const int64_t* last, int64_t* n) {
    return slice_copy(*SOL(s), var, buf, first, last, n, false, true);
}

int yb_var_reduce_slice(yb_solution* s_, int var, const int64_t* first, const int64_t* last, double out[5], int64_t* n_done) {
    Solution* s = SOL(s_);
    if (int rc = check_var(s, var)) return rc;
    if (!first || !last || !out) return set_error(YB_EINVAL, "null argument");
    if (!s->prepared) return set_error(YB_ESTATE, "var storage is not allocated: call prepare_solution first");
    Var& v = s->vars[var];
    Slice sl;
    if (int rc = resolve_slice(*s, v, first, last, true, sl)) return rc;
    YB_CUDA(cudaSetDevice(s->device));
    const size_t bytes = size_t(reduce_scratch_entries()) * sizeof(RedVals);
    if (int rc = ensure_stage(*s, bytes)) return rc;
    RedVals* part = static_cast<RedVals*>(s->stage_dev);
    RedVals tot{0.0, 0.0, 1.0, -HUGE_VAL, HUGE_VAL};
    for (int64_t t = sl.t0; t <= sl.t1; t++) {
        if (sl.elems_per_step == 0) break;
        if (int rc = launch_box_reduce(v.slot_ptr(v.slot_of(t)), sl.bc, v.elem_bytes, part, s->stream())) return rc;
        RedVals r;
        YB_CUDA(cudaMemcpyAsync(&r, part + (reduce_scratch_entries() - 1), sizeof r, cudaMemcpyDeviceToHost, s->stream()));
        YB_CUDA(cudaStreamSynchronize(s->stream()));
        tot.sum += r.sum; tot.sumsq += r.sumsq; tot.prod *= r.prod;
        tot.mx = std::max(tot.mx, r.mx); tot.mn = std::min(tot.mn, r.mn);
    }
    out[0] = tot.sum; out[1] = tot.sumsq; out[2] = tot.prod; out[3] = tot.mx; out[4] = tot.mn;
    if (n_done) *n_done = sl.elems_per_step * (sl.t1 - sl.t0 + 1);
    return 0;
}

int yb_var_set_all_same(yb_solution* s_, int var, double value) {
    Solution* s = SOL(s_);
    if (int rc = check_var(s, var)) return rc;
    if (!s->prepared) return set_error(YB_ESTATE, "var storage is not allocated: call prepare_solution first");
    Var& v = s->vars[var];
    YB_CUDA(cudaSetDevice(s->device));
    if (int rc = slices_var_write_waits(*s)) return rc;
    if (int rc = launch_fill_all(v.dev, v.slot_elems * v.nslots(), v.elem_bytes, value, s->stream())) return rc;
    if (int rc = slices_var_write_records(*s)) return rc;
    if (s->halo) halo_mark_dirty(*s, var);
    return 0;
}

int yb_var_set_slice_same(yb_solution* s_, int var, double value, const int64_t* first, const int64_t* last, int64_t* n_done) {
    Solution* s = SOL(s_);
    if (int rc = check_var(s, var)) return rc;
    if (!s->prepared) return set_error(YB_ESTATE, "var storage is not allocated: call prepare_solution first");
    Var& v = s->vars[var];
    Slice sl;
    if (int rc = resolve_slice(*s, v, first, last, false, sl)) return rc;
    YB_CUDA(cudaSetDevice(s->device));
    if (int rc = slices_var_write_waits(*s)) return rc;
    for (int64_t t = sl.t0; t <= sl.t1; t++) {
        if (int rc = launch_box_fill(v.slot_ptr(v.slot_of(t)), sl.bc, v.elem_bytes, value, s->stream())) return rc;
        v.update_valid_step(t);
    }
    if (int rc = slices_var_write_records(*s)) return rc;
    if (s->halo) halo_mark_dirty(*s, var);
    if (n_done) *n_done = sl.elems_per_step * (sl.t1 - sl.t0 + 1);
    return 0;
}

// first/last of the rank "halo box" (domain + halos) or domain box of a var at one step
static void var_box(const Var& v, int64_t step, bool with_halo, int64_t* first, int64_t* last) {
    for (size_t i = 0; i < v.dims.size(); i++) {
        const Dim& d = v.dims[i];
        if (d.spec.kind == DIM_STEP) { first[i] = last[i] = step; }
        else if (d.spec.kind == DIM_MISC) { first[i] = d.spec.misc_first; last[i] = d.spec.misc_first + d.domain - 1; }
        else {
            first[i] = d.rank_offset - (with_halo ? d.spec.halo_l : 0);
            last[i] = d.rank_offset + d.domain - 1 + (with_halo ? d.spec.halo_r : 0);
        }
    }
}

int yb_var_fill_hash(yb_solution* s_, int var, int64_t step, uint32_t seed, uint32_t salt, double lo, double hi) {
    return yb_var_fill_hash_shifted(s_, var, step, seed, salt, lo, hi, nullptr);
}

int yb_var_fill_hash_shifted(yb_solution* s_, int var, int64_t step, uint32_t seed, uint32_t salt, double lo, double hi,
                             const int64_t* shift) {
    Solution* s = SOL(s_);
    if (int rc = check_var(s, var)) return rc;
    if (!s->prepared) return set_error(YB_ESTATE, "var storage is not allocated: call prepare_solution first");
    Var& v = s->vars[var];
    int64_t first[YB_MAX_DIMS], last[YB_MAX_DIMS];
    var_box(v, step, true, first, last);
    Slice sl;
    if (int rc = resolve_slice(*s, v, first, last, false, sl)) return rc;
    YB_CUDA(cudaSetDevice(s->device));
    if (shift) {
        // sl.g0 holds the global index of the box origin for the LAST three non-step dims (left padded); add the shift of
        // the domain dims among them
        int nns = 0;
        for (auto& d : v.dims) nns += d.spec.kind != DIM_STEP;
        int k = 0;
        for (auto& d : v.dims) {
            if (d.spec.kind == DIM_STEP) continue;
            const int pos = nns <= 3 ? 3 - nns + k : (k == 0 ? 3 : k - 1);
            if (d.spec.kind == DIM_DOMAIN) sl.g0[pos] += shift[d.spec.domain_index];
            k++;
        }
    }
    if (int rc = slices_var_write_waits(*s)) return rc;
    if (int rc = launch_hash_fill(v.slot_ptr(v.slot_of(step)), sl.bc, sl.g0, v.elem_bytes, seed, salt, lo, hi, s->stream())) return rc;
    if (int rc = slices_var_write_records(*s)) return rc;
    v.update_valid_step(step);
    if (s->halo) halo_mark_dirty(*s, var);
    return 0;
}

int yb_var_checksum(yb_solution* s_, int var, int64_t step, uint64_t* out) {
    Solution* s = SOL(s_);
    if (int rc = check_var(s, var)) return rc;
    if (!s->prepared) return set_error(YB_ESTATE, "var storage is not allocated: call prepare_solution first");
    if (!out) return set_error(YB_EINVAL, "null output");
    Var& v = s->vars[var];
    int64_t first[YB_MAX_DIMS], last[YB_MAX_DIMS];
    var_box(v, step, false, first, last);
    Slice sl;
    if (int rc = resolve_slice(*s, v, first, last, true, sl)) return rc;
    YB_CUDA(cudaSetDevice(s->device));
    if (int rc = ensure_stage(*s, 256)) return rc;
    if (int rc = launch_checksum(v.slot_ptr(v.slot_of(step)), sl.bc, sl.g0, v.elem_bytes, (unsigned long long*)s->stage_dev, s->stream())) return rc;
    unsigned long long h = 0;
    YB_CUDA(cudaMemcpyAsync(&h, s->stage_dev, 8, cudaMemcpyDeviceToHost, s->stream()));
    YB_CUDA(cudaStreamSynchronize(s->stream()));
    *out = h;
    return 0;
}

int yb_var_device_ptr(yb_solution* s_, int var, int64_t step, void** out) {
    Solution* s = SOL(s_);
    if (int rc = check_var(s, var)) return rc;
    if (!s->prepared) return set_error(YB_ESTATE, "var storage is not allocated");
    if (!out) return set_error(YB_EINVAL, "null output");
    Var& v = s->vars[var];
    *out = v.slot_ptr(v.slot_of(step));
    return 0;
}

int yb_copy_to_host(void* host_dst, const void* dev_src, size_t bytes) {
    if (!host_dst || !dev_src) return set_error(YB_EINVAL, "null argument");
    YB_CUDA(cudaMemcpy(host_dst, dev_src, bytes, cudaMemcpyDeviceToHost));
    return 0;
}

// ---- run_solution ----------------------------------------------------------------------------------
// Mirrors /root/reference/src/kernel/lib/context.cpp:220-624.  Single rank: one launch per stage part over the whole rank box.
// Multi-rank (halo_run_stage, yb_halo.cu): for each step, for each stage: finish the previous exchange -> exterior slabs ->
// start this stage's exchange -> interior.  Multi-rank with fused steps (the reference's wave-fronts, -bt / -Mbt): one deep
// exchange at the start, then per fused launch: finish the exchange -> whole rank box -> deep exchange (halo_run_steps).
int yb_solution_run(yb_solution* s_, int64_t first_step, int64_t last_step) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (!s->prepared) return set_error(YB_ESTATE, "run_solution() called without calling prepare_solution() first");
    YB_CUDA(cudaSetDevice(s->device));
    cudaStream_t st = s->stream();
    // point tables are normally uploaded when they are set (or at prepare); before anything of this run is enqueued otherwise
    if (int rc = points_begin_run(*s)) return rc;
    if (int rc = slices_begin_run(*s, first_step, last_step)) return rc;
    if (int rc = slices_run_waits(*s, st)) return rc;     // frames shared with other solutions (yb_slices.h)
    // Timing events: pairs of finished runs are folded into the stats and recycled here, so that calling
    // run_solution(t) once per step (the reference's usual pattern) keeps a bounded number of events alive.
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    for (size_t i = 0; i < s->pending_events.size();) {
        auto& pe = s->pending_events[i];
        float ms = 0;
        if (cudaEventQuery(pe.second) == cudaSuccess && cudaEventElapsedTime(&ms, pe.first, pe.second) == cudaSuccess) {
            s->stats.elapsed_secs += double(ms) * 1e-3;
            if (!e0) { e0 = pe.first; e1 = pe.second; }
            else { cudaEventDestroy(pe.first); cudaEventDestroy(pe.second); }
            s->pending_events.erase(s->pending_events.begin() + i);
        } else {
            (void)cudaGetLastError();
            i++;
        }
    }
    if (!e0) {
        YB_CUDA(cudaEventCreate(&e0));
        if (cudaEventCreate(&e1) != cudaSuccess) { cudaEventDestroy(e0); return set_error(YB_ECUDA, "cudaEventCreate failed"); }
    }
    s->pending_events.emplace_back(e0, e1);     // owned by the solution from here on (drained by get_stats / the next run)
    YB_CUDA(cudaEventRecord(e0, st));
    YB_CUDA(cudaEventRecord(e1, st));           // placeholder so that the pair is always complete; re-recorded below
    Box whole;
    for (int d = 0; d < 3; d++) { whole.b[d] = 0; whole.e[d] = d < s->ndd ? s->rank_size[d] : 1; }
    int64_t pts = whole.points();
    int rc = 0;
    if (s->halo) rc = halo_exchange_all(*s, st);  // initial exchange of everything dirty (context.cpp:346)
    // direction from the order of the arguments, as the reference does (context.cpp:237-246)
    const int64_t step_dir = last_step >= first_step ? 1 : -1;
    if (rc >= 0) rc = s->engine->begin_run(*s, first_step, st);
    // Temporal tile (the reference's "-bt", context.cpp:657-681): a forward run goes through the engine's fused launch, `fs` steps
    // at a time; what is left over (and every other kind of run) takes the one-step path below.  A rank grid fuses steps only
    // in the mode its engine fixed at prepare; its halos are then 2R deep and exchanged once per fused launch.  Point sources
    // and slice injectors enter between two steps, and slice recorders and correlators read a step a pair would never store, so a
    // solution with any of them runs one step per launch (all are refused on a rank grid in the fused mode).
    int64_t t_first = first_step;
    const int fs = (step_dir > 0 && (s->halo || !s->tuner.enabled) && !points_active(*s) && !slices_active(*s) && !slice_injectors_active(*s) &&
                    !slice_correlators_active(*s))
                       ? s->engine->fused_steps(*s) : 1;
    if (s->halo && fs > 1 && rc >= 0 && last_step - t_first + 1 >= fs) rc = halo_exchange_deep(*s, t_first, true, st);
    while (fs > 1 && rc >= 0 && last_step - t_first + 1 >= fs) {
        const bool ends_run = t_first + fs - 1 == last_step;
        rc = s->halo ? halo_run_steps(*s, t_first, fs, st) : s->engine->launch_steps(*s, t_first, fs, ends_run, whole, st);
        if (rc < 0) break;
        s->stats.kernel_launches += rc;
        for (int k = 0; k < fs; k++) {
            for (const StageSpec& sp : s->spec.stages) {
                s->stats.num_writes_done += sp.writes * pts;
                s->stats.num_reads_done += sp.reads * pts;
                s->stats.est_fp_ops_done += sp.fp_ops * pts;
                for (int vi : sp.outputs) s->vars[vi].update_valid_step(t_first + k + sp.out_step_off);
            }
            s->stats.num_steps_done++;
        }
        t_first += fs;
    }
    for (int64_t t = t_first; t != last_step + step_dir && rc >= 0; t += step_dir) {
        // in-run auto-tuner (/root/reference/src/kernel/lib/auto_tuner.cpp, context.cpp:592-600): this step runs with the next
        // untried launch variant and is timed on its own; once every variant has its samples the fastest stays selected
        cudaEvent_t te0 = nullptr, te1 = nullptr;
        int tv = -1;
        if (s->tuner.enabled) {
            const int nv = s->engine->tune_variants(*s);
            if (nv <= 1) s->tuner.enabled = false;
            else {
                if (int(s->tuner.ms.size()) != nv) { s->tuner.ms.assign(nv, 1e30); s->tuner.tries.assign(nv, 0); s->tuner.next = 0; s->tuner.report.clear(); }
                tv = s->tuner.next;
                s->engine->tune_select(*s, tv);
                if (cudaEventCreate(&te0) == cudaSuccess && cudaEventCreate(&te1) == cudaSuccess) cudaEventRecord(te0, st);
            }
        }
        for (size_t sg = 0; sg < s->spec.stages.size() && rc >= 0; sg++) {
            if (s->halo) {
                rc = halo_run_stage(*s, int(sg), t, st);
            } else {
                rc = s->engine->launch(*s, int(sg), t, whole, st);
                if (rc > 0) s->stats.kernel_launches += rc;
            }
            const StageSpec& sp = s->spec.stages[sg];
            s->stats.num_writes_done += sp.writes * pts;
            s->stats.num_reads_done += sp.reads * pts;
            s->stats.est_fp_ops_done += sp.fp_ops * pts;
            for (int vi : sp.outputs) s->vars[vi].update_valid_step(t + sp.out_step_off);
        }
        // injectors, then sources and receivers of the step just computed (a rank grid applies them inside its last stage,
        // halo_run_stage)
        if (rc >= 0 && !s->halo) rc = slice_injectors_launch(*s, t, PTS_ALL, whole, st);
        if (rc >= 0 && !s->halo) rc = points_launch(*s, t, PTS_ALL, whole, st);
        // then the slice recorders, before the next step's first launch can overwrite an in-place var (halo_run_stage on a grid)
        if (rc >= 0 && !s->halo) rc = slices_launch(*s, t, st);
        if (rc >= 0 && !s->halo) rc = slice_correlators_launch(*s, t, st);    // which see that step's recording
        s->stats.num_steps_done++;
        if (tv >= 0 && te0 && te1) {
            cudaEventRecord(te1, st);
            float ms = 0;
            if (cudaEventSynchronize(te1) == cudaSuccess && cudaEventElapsedTime(&ms, te0, te1) == cudaSuccess) {
                auto& tu = s->tuner;
                tu.ms[tv] = std::min(tu.ms[tv], double(ms));
                if (++tu.tries[tv] >= tu.reps + 1) tu.next++;        // the first sample of a variant includes its cold start
                if (tu.next >= int(tu.ms.size())) {
                    int best = 0;
                    for (size_t i = 1; i < tu.ms.size(); i++) if (tu.ms[i] < tu.ms[best]) best = int(i);
                    char line[200];
                    for (size_t i = 0; i < tu.ms.size(); i++) {
                        snprintf(line, sizeof line, " %s: %.4f ms/step%s\n", s->engine->tune_describe(*s, int(i)).c_str(), tu.ms[i], int(i) == best ? "  <- best" : "");
                        tu.report += line;
                    }
                    s->engine->tune_select(*s, best);
                    tu.enabled = false;
                }
            }
        }
        if (te0) cudaEventDestroy(te0);
        if (te1) cudaEventDestroy(te1);
    }
    if (s->halo && rc >= 0) rc = halo_finish(*s, st);   // the last exchange completes inside the run (and its timing)
    if (s->halo && rc >= 0) rc = points_record_pending(*s, st);        // then the last step's weighted receivers
    if (int e = slices_run_records(*s, st)) return e;
    YB_CUDA(cudaEventRecord(e1, st));
    return rc < 0 ? rc : 0;
}

int yb_solution_sync(yb_solution* s_) {
    Solution* s = SOL(s_);
    if (!s || !s->prepared) return set_error(YB_ESTATE, "solution not prepared");
    YB_CUDA(cudaSetDevice(s->device));
    YB_CUDA(cudaStreamSynchronize(s->stream()));
    YB_CUDA(cudaStreamSynchronize(s->comm_stream));
    return 0;
}

static int drain_events(Solution* s) {
    for (auto& pe : s->pending_events) {
        YB_CUDA(cudaEventSynchronize(pe.second));
        float ms = 0;
        YB_CUDA(cudaEventElapsedTime(&ms, pe.first, pe.second));
        s->stats.elapsed_secs += double(ms) * 1e-3;
        cudaEventDestroy(pe.first);
        cudaEventDestroy(pe.second);
    }
    s->pending_events.clear();
    return 0;
}

int yb_get_stats(yb_solution* s_, yb_stats* out) {
    Solution* s = SOL(s_);
    if (!s || !out) return set_error(YB_EINVAL, "null argument");
    if (!s->prepared) return set_error(YB_ESTATE, "solution not prepared");
    YB_CUDA(cudaSetDevice(s->device));
    if (int rc = drain_events(s)) return rc;
    s->stats.num_elements = 1;
    for (int d = 0; d < s->ndd; d++) s->stats.num_elements *= s->overall_size[d];
    *out = s->stats;
    return 0;
}

int yb_solution_auto_tune(yb_solution* s_, char* report, size_t n) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (!s->prepared) return set_error(YB_ESTATE, "run_auto_tuner_now() called without calling prepare_solution() first");
    YB_CUDA(cudaSetDevice(s->device));
    std::string rep;
    if (int rc = s->engine->auto_tune(*s, s->stream(), rep)) return rc;
    YB_CUDA(cudaStreamSynchronize(s->stream()));
    if (report && n) snprintf(report, n, "%s", rep.c_str());
    return yb_clear_stats(s_);      // the reference clears the stats when the tuner is done (yk_solution_api.hpp:872)
}

// yk_solution::reset_auto_tuner / is_auto_tuner_enabled (aux/yk_solution_api.hpp:820-856): (re)start or stop the in-run tuner
int yb_solution_reset_auto_tuner(yb_solution* s_, int enable) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    s->tuner = Solution::InRunTuner();
    s->tuner.enabled = enable != 0;
    return 0;
}
int yb_solution_is_auto_tuner_enabled(const yb_solution* s) { return s && CSOL(s)->tuner.enabled; }
int yb_solution_auto_tuner_report(const yb_solution* s_, char* report, size_t n) {
    const Solution* s = CSOL(s_);
    if (!s || !report || !n) return set_error(YB_EINVAL, "null argument");
    snprintf(report, n, "%s", s->tuner.report.c_str());
    return 0;
}

int yb_clear_stats(yb_solution* s_) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (s->prepared) {
        YB_CUDA(cudaSetDevice(s->device));
        if (int rc = drain_events(s)) return rc;
    }
    memset(&s->stats, 0, sizeof s->stats);
    return 0;
}

}  // extern "C"
