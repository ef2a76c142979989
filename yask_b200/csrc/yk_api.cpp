// C++ host mirror of the reference's kernel API (yask_b200/include/yask_kernel_api.hpp) implemented as a
// thin adapter over the C ABI (include/yask_b200.h).  Built once per solution into
// libyask_kernel.<stencil>.b200.so (-DYK_STENCIL_NAME=<stencil>), like the reference's per-stencil
// libyask_kernel.<stencil>.<arch>.so (/root/reference/src/common/common.mk:211-216); the objects the
// factory hands out play the role of StencilContext / YkVarImpl
// (/root/reference/src/kernel/lib/{factory,soln_apis,yk_var_apis}.cpp).  Host bookkeeping only.
#include "../include/yask_kernel_api.hpp"
#include "../include/yask_b200_points.hpp"
#include "../include/yask_b200_slices.hpp"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>

extern "C" {
#include "../../include/yask_b200.h"
}

#ifndef YK_STENCIL_NAME
#define YK_STENCIL_NAME iso3dfd
#endif
#define YK_STR2(x) #x
#define YK_STR(x) YK_STR2(x)

namespace yask {

// ---- common API ----------------------------------------------------------------------------------------------
std::string yask_get_version_string() { return yb_version_string(); }
const char* yask_exception::what() const noexcept { return _msg.c_str(); }
void yask_exception::add_message(const std::string& message) { _msg.append(message); }
const char* yask_exception::get_message() const { return _msg.c_str(); }

namespace {

[[noreturn]] void fail(const std::string& m) {
    yask_exception e("YASK error: " + m);
    throw e;
}
inline int chk(int rc) {
    if (rc < 0) fail(yb_last_error());
    return rc;
}
inline idx_t chk64(idx_t v) {
    if (v < 0) fail(yb_last_error());
    return v;
}

struct StdoutOutput : yask_stdout_output { std::ostream& get_ostream() override { return std::cout; } };
struct NullBuf : std::streambuf { int overflow(int c) override { return c; } };
struct NullOutput : yask_null_output {
    NullBuf buf; std::ostream os{&buf};
    std::ostream& get_ostream() override { return os; }
};
struct StringOutput : yask_string_output {
    std::ostringstream os;
    std::ostream& get_ostream() override { return os; }
    std::string get_string() const override { return os.str(); }
    void discard() override { os.str(""); }
};
struct FileOutput : yask_file_output {
    std::string fn; std::ofstream os;
    explicit FileOutput(const std::string& f) : fn(f), os(f) { if (!os) fail("cannot open '" + f + "' for output"); }
    std::ostream& get_ostream() override { return os; }
    std::string get_filename() const override { return fn; }
    void close() override { os.close(); }
};

yask_output_ptr g_debug;
bool g_trace = false;

}  // namespace

yask_file_output_ptr yask_output_factory::new_file_output(const std::string& f) const { return std::make_shared<FileOutput>(f); }
yask_string_output_ptr yask_output_factory::new_string_output() const { return std::make_shared<StringOutput>(); }
yask_stdout_output_ptr yask_output_factory::new_stdout_output() const { return std::make_shared<StdoutOutput>(); }
yask_null_output_ptr yask_output_factory::new_null_output() const { return std::make_shared<NullOutput>(); }

void yask_print_splash(std::ostream& os, int argc, char** argv, std::string leader) {
    os << "YASK -- Yet Another Stencil Kit (yask_b200 engine), version " << yask_get_version_string() << "\n";
    if (argc > 1) {
        os << leader;
        for (int i = 0; i < argc; i++) os << (i ? " " : "") << argv[i];
        os << "\n";
    }
}

void yk_env::set_debug_output(yask_output_ptr debug) { g_debug = debug; }
void yk_env::disable_debug_output() { g_debug = std::make_shared<NullOutput>(); }
yask_output_ptr yk_env::get_debug_output() {
    if (!g_debug) g_debug = std::make_shared<StdoutOutput>();
    return g_debug;
}
void yk_env::set_trace_enabled(bool enable) { g_trace = enable; }
bool yk_env::is_trace_enabled() { return g_trace; }

namespace {

// One process = one rank = one GPU.  The ranks of a job are started by any launcher that exports rank and world size
// (torchrun, mpirun, srun, a shell loop); they meet in the library's shared-memory mailbox (yb_comm.cpp), which stands in
// for the reference's MPI communicator (/root/reference/src/kernel/lib/setup.cpp:60-139, yask_kernel_api.hpp:238-293).
struct B200Env : yk_env {
    B200Env() { chk_comm(yb_comm_init(yb_comm_env_rank(), yb_comm_env_world(), nullptr)); }
    static void chk_comm(int rc) { if (rc < 0) fail(yb_last_error()); }
    int get_num_ranks() const override { return yb_comm_world(); }
    int get_rank_index() const override { return yb_comm_rank(); }
    void global_barrier() const override { chk_comm(yb_comm_barrier()); }
    idx_t sum_over_ranks(idx_t v) const override { int64_t s = 0; chk_comm(yb_comm_sum_i64(v, &s)); return idx_t(s); }
    void assert_equality_over_ranks(idx_t v, const std::string& descr) const override {
        // setup.cpp:106-121: every rank must hold the same value
        const idx_t s = sum_over_ranks(v);
        if (s != v * idx_t(yb_comm_world())) fail("ranks disagree on " + descr + " (this rank: " + std::to_string(v) + ")");
    }
    void finalize() override { yb_comm_finalize(); }
    [[noreturn]] void exit(int code) override { std::exit(code); }
};

struct Handle {   // owns the C-ABI solution
    yb_solution* s = nullptr;
    ~Handle() { if (s) yb_solution_destroy(s); }
};

struct B200Stats : yk_stats {
    yb_stats st;
    idx_t get_num_elements() override { return st.num_elements; }
    idx_t get_num_steps_done() override { return st.num_steps_done; }
    idx_t get_num_writes_done() override { return st.num_writes_done; }
    idx_t get_est_fp_ops_done() override { return st.est_fp_ops_done; }
    double get_elapsed_secs() override { return st.elapsed_secs; }
};

struct B200Reduction : yk_var::yk_reduction_result {
    int mask = 0; idx_t n = 0; double sum = 0, sumsq = 0, prod = 1, mx = 0, mn = 0;
    int get_reduction_mask() const override { return mask; }
    idx_t get_num_elements_reduced() const override { return n; }
    double need(int bit, double v, const char* what) const {
        if (!(mask & bit)) fail(std::string(what) + " reduction was not requested in reduce_elements_in_slice()");
        return v;
    }
    double get_sum() const override { return need(yk_var::yk_sum_reduction, sum, "sum"); }
    double get_sum_squares() const override { return need(yk_var::yk_sum_squares_reduction, sumsq, "sum-of-squares"); }
    double get_product() const override { return need(yk_var::yk_product_reduction, prod, "product"); }
    double get_max() const override { return need(yk_var::yk_max_reduction, mx, "max"); }
    double get_min() const override { return need(yk_var::yk_min_reduction, mn, "min"); }
};

struct B200Var : yk_var {
    std::shared_ptr<Handle> h;
    int vi;
    std::string name;
    bool* step_wrap;                       // the owning solution's set_step_wrap() flag
    std::vector<char> raw_mirror;          // host snapshot for get_raw_storage_buffer()

    B200Var(std::shared_ptr<Handle> h_, int vi_, bool* sw) : h(h_), vi(vi_), step_wrap(sw) { name = info().name; }
    yb_var_info info() const {
        yb_var_info i;
        chk(yb_var_info_get(h->s, vi, &i));
        return i;
    }
    int pos(const yb_var_info& i, const std::string& dim, int kind_mask, const char* fn) const {
        for (int k = 0; k < i.num_dims; k++)
            if (dim == i.dims[k].name) {
                if (!((1 << i.dims[k].kind) & kind_mask)) break;
                return k;
            }
        fail(std::string("dimension '") + dim + "' is not valid for " + fn + " on var '" + name + "'");
    }
    static constexpr int STEP = 1, DOMAIN = 2, MISC = 4;
    bool prepared() const { return yb_solution_is_prepared(h->s) != 0; }

    const std::string& get_name() const override { return name; }
    int get_num_dims() const override { return info().num_dims; }
    string_vec get_dim_names() const override {
        auto i = info(); string_vec v;
        for (int k = 0; k < i.num_dims; k++) v.push_back(i.dims[k].name);
        return v;
    }
    int get_num_domain_dims() const override { auto i = info(); int n = 0; for (int k = 0; k < i.num_dims; k++) n += i.dims[k].kind == 1; return n; }
    bool is_dim_used(const std::string& dim) const override {
        auto i = info();
        for (int k = 0; k < i.num_dims; k++) if (dim == i.dims[k].name) return true;
        return false;
    }
    bool is_fixed_size() const override { return fixed; }
    bool fixed = false;

    // first/last allocated global index of dim k (SURVEY.md Appendix C)
    static idx_t first_local(const yb_var_info& i, int k) {
        const auto& d = i.dims[k];
        if (d.kind == 0) return i.first_valid_step;
        if (d.kind == 2) return d.first_misc_index;
        return d.rank_offset - d.left_pad;
    }
    static idx_t last_local(const yb_var_info& i, int k) {
        const auto& d = i.dims[k];
        if (d.kind == 0) return i.last_valid_step;
        if (d.kind == 2) return d.first_misc_index + d.domain_size - 1;
        return d.rank_offset + d.domain_size + d.right_pad - 1;
    }
    idx_t get_first_local_index(const std::string& dim) const override { auto i = info(); return first_local(i, pos(i, dim, 7, "get_first_local_index")); }
    idx_t get_last_local_index(const std::string& dim) const override { auto i = info(); return last_local(i, pos(i, dim, 7, "get_last_local_index")); }
    idx_t_vec get_first_local_index_vec() const override { auto i = info(); idx_t_vec v; for (int k = 0; k < i.num_dims; k++) v.push_back(first_local(i, k)); return v; }
    idx_t_vec get_last_local_index_vec() const override { auto i = info(); idx_t_vec v; for (int k = 0; k < i.num_dims; k++) v.push_back(last_local(i, k)); return v; }
    idx_t get_alloc_size(const std::string& dim) const override {
        auto i = info(); int k = pos(i, dim, 7, "get_alloc_size");
        return i.dims[k].kind == 0 ? i.step_alloc : i.dims[k].alloc_size;
    }
    idx_t_vec get_alloc_size_vec() const override {
        auto i = info(); idx_t_vec v;
        for (int k = 0; k < i.num_dims; k++) v.push_back(i.dims[k].kind == 0 ? i.step_alloc : i.dims[k].alloc_size);
        return v;
    }
    idx_t get_first_valid_step_index() const override { auto i = info(); if (!i.has_step) fail("var '" + name + "' does not use the step dimension"); return i.first_valid_step; }
    idx_t get_last_valid_step_index() const override { auto i = info(); if (!i.has_step) fail("var '" + name + "' does not use the step dimension"); return i.last_valid_step; }
    idx_t get_rank_domain_size(const std::string& dim) const override { auto i = info(); return i.dims[pos(i, dim, DOMAIN, "get_rank_domain_size")].domain_size; }
    idx_t_vec dom_vec(int which) const {
        auto i = info(); idx_t_vec v;
        for (int k = 0; k < i.num_dims; k++) {
            const auto& d = i.dims[k];
            if (d.kind != 1) continue;
            switch (which) {
                case 0: v.push_back(d.domain_size); break;
                case 1: v.push_back(d.rank_offset); break;
                case 2: v.push_back(d.rank_offset + d.domain_size - 1); break;
                case 3: v.push_back(d.rank_offset - d.left_halo); break;
                default: v.push_back(d.rank_offset + d.domain_size + d.right_halo - 1); break;
            }
        }
        return v;
    }
    idx_t_vec get_rank_domain_size_vec() const override { return dom_vec(0); }
    idx_t get_first_rank_domain_index(const std::string& dim) const override { auto i = info(); return i.dims[pos(i, dim, DOMAIN, "get_first_rank_domain_index")].rank_offset; }
    idx_t_vec get_first_rank_domain_index_vec() const override { return dom_vec(1); }
    idx_t get_last_rank_domain_index(const std::string& dim) const override { auto i = info(); auto& d = i.dims[pos(i, dim, DOMAIN, "get_last_rank_domain_index")]; return d.rank_offset + d.domain_size - 1; }
    idx_t_vec get_last_rank_domain_index_vec() const override { return dom_vec(2); }
    idx_t get_left_halo_size(const std::string& dim) const override { auto i = info(); return i.dims[pos(i, dim, DOMAIN, "get_left_halo_size")].left_halo; }
    idx_t get_right_halo_size(const std::string& dim) const override { auto i = info(); return i.dims[pos(i, dim, DOMAIN, "get_right_halo_size")].right_halo; }
    idx_t get_first_rank_halo_index(const std::string& dim) const override { auto i = info(); auto& d = i.dims[pos(i, dim, DOMAIN, "get_first_rank_halo_index")]; return d.rank_offset - d.left_halo; }
    idx_t_vec get_first_rank_halo_index_vec() const override { return dom_vec(3); }
    idx_t get_last_rank_halo_index(const std::string& dim) const override { auto i = info(); auto& d = i.dims[pos(i, dim, DOMAIN, "get_last_rank_halo_index")]; return d.rank_offset + d.domain_size + d.right_halo - 1; }
    idx_t_vec get_last_rank_halo_index_vec() const override { return dom_vec(4); }
    idx_t get_left_pad_size(const std::string& dim) const override { auto i = info(); return i.dims[pos(i, dim, DOMAIN, "get_left_pad_size")].left_pad; }
    idx_t get_right_pad_size(const std::string& dim) const override { auto i = info(); return i.dims[pos(i, dim, DOMAIN, "get_right_pad_size")].right_pad; }
    idx_t get_left_extra_pad_size(const std::string& dim) const override { auto i = info(); auto& d = i.dims[pos(i, dim, DOMAIN, "get_left_extra_pad_size")]; return d.left_pad - d.left_halo; }
    idx_t get_right_extra_pad_size(const std::string& dim) const override { auto i = info(); auto& d = i.dims[pos(i, dim, DOMAIN, "get_right_extra_pad_size")]; return d.right_pad - d.right_halo; }
    idx_t get_first_misc_index(const std::string& dim) const override { auto i = info(); return i.dims[pos(i, dim, MISC, "get_first_misc_index")].first_misc_index; }
    idx_t get_last_misc_index(const std::string& dim) const override { auto i = info(); auto& d = i.dims[pos(i, dim, MISC, "get_last_misc_index")]; return d.first_misc_index + d.domain_size - 1; }

    // Are the indices inside the allocation (and, unless step wrap is on, the valid steps)?
    bool local(const yb_var_info& i, const idx_t_vec& idx, bool check_step) const {
        if (int(idx.size()) != i.num_dims)
            fail("attempt to access " + std::to_string(i.num_dims) + "-D var '" + name + "' with " + std::to_string(idx.size()) + " indices");
        for (int k = 0; k < i.num_dims; k++) {
            if (i.dims[k].kind == 0 && (!check_step || *step_wrap)) continue;
            if (idx[k] < first_local(i, k) || idx[k] > last_local(i, k)) return false;
        }
        return true;
    }
    // With set_step_wrap(true) any step index addresses the slot it wraps to (imod_flr(t, alloc_t), yk_var.hpp:131-147): reads go
    // through the step of the valid window that lives in that slot (the C ABI checks the window on reads).
    idx_t_vec wrapped(const yb_var_info& i, const idx_t_vec& idx) const {
        idx_t_vec out = idx;
        if (*step_wrap && i.has_step && !out.empty()) {
            const idx_t a = i.step_alloc, f = i.first_valid_step;
            idx_t d = (out[0] - f) % a;
            if (d < 0) d += a;
            out[0] = f + d;
        }
        return out;
    }
    bool are_indices_local(const idx_t_vec& indices) const override {
        if (!prepared()) return false;
        return local(info(), indices, true);
    }
    bool are_indices_local(const idx_t_init_list& indices) const override { return are_indices_local(idx_t_vec(indices)); }
    void need_storage(const char* fn) const {
        if (!prepared()) fail(std::string("call to '") + fn + "' with no storage allocated for var '" + name + "'");
    }
    double get_element(const idx_t_vec& indices) const override {
        need_storage("get_element");
        auto i = info();
        if (!local(i, indices, true)) fail("get_element: indices " + format_indices(indices) + " are not valid for var '" + name + "'");
        double out = 0;
        const idx_t_vec w = wrapped(i, indices);
        if (i.elem_bytes == 4) { float f = 0; chk(yb_var_get_slice(h->s, vi, &f, w.data(), w.data(), nullptr)); out = f; }
        else chk(yb_var_get_slice(h->s, vi, &out, w.data(), w.data(), nullptr));
        return out;
    }
    double get_element(const idx_t_init_list& indices) const override { return get_element(idx_t_vec(indices)); }
    idx_t set_element(double val, const idx_t_vec& indices, bool strict) override {
        need_storage("set_element");
        auto i = info();
        if (!local(i, indices, false)) {   // set_element does not check the step index (yk_var_apis.cpp:392-408)
            if (strict) fail("set_element: indices " + format_indices(indices) + " are not valid for var '" + name + "'");
            return 0;
        }
        if (i.elem_bytes == 4) { float f = float(val); chk(yb_var_set_slice(h->s, vi, &f, indices.data(), indices.data(), nullptr)); }
        else chk(yb_var_set_slice(h->s, vi, &val, indices.data(), indices.data(), nullptr));
        return 1;
    }
    idx_t set_element(double val, const idx_t_init_list& indices, bool strict) override { return set_element(val, idx_t_vec(indices), strict); }
    idx_t add_to_element(double val, const idx_t_vec& indices, bool strict) override {
        need_storage("add_to_element");
        auto i = info();
        if (!local(i, indices, true)) {
            if (strict) fail("add_to_element: indices " + format_indices(indices) + " are not valid for var '" + name + "'");
            return 0;
        }
        double cur = get_element(indices);
        // same rounding as the reference: the sum is formed in the element type (yk_var.hpp:1060-1070)
        double nv = i.elem_bytes == 4 ? double(float(float(cur) + float(val))) : cur + val;
        return set_element(nv, indices, strict);
    }
    idx_t add_to_element(double val, const idx_t_init_list& indices, bool strict) override { return add_to_element(val, idx_t_vec(indices), strict); }

    static size_t slice_elems(const idx_t_vec& f, const idx_t_vec& l) {
        size_t n = 1;
        for (size_t k = 0; k < f.size(); k++) n *= size_t(l[k] - f[k] + 1);
        return n;
    }
    template <typename T>
    idx_t get_typed(T* buf, size_t buffer_size, const idx_t_vec& first, const idx_t_vec& last) const {
        need_storage("get_elements_in_slice");
        auto i = info();
        if (int(first.size()) != i.num_dims || int(last.size()) != i.num_dims) fail("get_elements_in_slice: wrong number of indices for var '" + name + "'");
        size_t n = slice_elems(first, last);
        if (buffer_size < n) fail("get_elements_in_slice: buffer of " + std::to_string(buffer_size) + " element(s) is too small for " + std::to_string(n));
        int64_t done = 0;
        idx_t_vec wf = first, wl = last;
        if (*step_wrap && i.has_step && first[0] == last[0]) { wf = wrapped(i, first); wl[0] = wf[0]; }      // one step: wrap it into the window
        if (sizeof(T) == size_t(i.elem_bytes)) { chk(yb_var_get_slice(h->s, vi, buf, wf.data(), wl.data(), &done)); return done; }
        // element-size conversion through a temporary
        std::vector<char> tmp(n * i.elem_bytes);
        chk(yb_var_get_slice(h->s, vi, tmp.data(), wf.data(), wl.data(), &done));
        for (size_t k = 0; k < n; k++) buf[k] = i.elem_bytes == 4 ? T(reinterpret_cast<float*>(tmp.data())[k]) : T(reinterpret_cast<double*>(tmp.data())[k]);
        return done;
    }
    template <typename T>
    idx_t set_typed(const T* buf, size_t buffer_size, const idx_t_vec& first, const idx_t_vec& last) {
        need_storage("set_elements_in_slice");
        auto i = info();
        if (int(first.size()) != i.num_dims || int(last.size()) != i.num_dims) fail("set_elements_in_slice: wrong number of indices for var '" + name + "'");
        size_t n = slice_elems(first, last);
        if (buffer_size < n) fail("set_elements_in_slice: buffer of " + std::to_string(buffer_size) + " element(s) is too small for " + std::to_string(n));
        int64_t done = 0;
        if (sizeof(T) == size_t(i.elem_bytes)) { chk(yb_var_set_slice(h->s, vi, buf, first.data(), last.data(), &done)); return done; }
        std::vector<char> tmp(n * i.elem_bytes);
        for (size_t k = 0; k < n; k++) {
            if (i.elem_bytes == 4) reinterpret_cast<float*>(tmp.data())[k] = float(buf[k]);
            else reinterpret_cast<double*>(tmp.data())[k] = double(buf[k]);
        }
        chk(yb_var_set_slice(h->s, vi, tmp.data(), first.data(), last.data(), &done));
        return done;
    }
    idx_t get_elements_in_slice(float* b, size_t n, const idx_t_vec& f, const idx_t_vec& l) const override { return get_typed(b, n, f, l); }
    idx_t get_elements_in_slice(double* b, size_t n, const idx_t_vec& f, const idx_t_vec& l) const override { return get_typed(b, n, f, l); }
    idx_t set_elements_in_slice(const float* b, size_t n, const idx_t_vec& f, const idx_t_vec& l) override { return set_typed(b, n, f, l); }
    idx_t set_elements_in_slice(const double* b, size_t n, const idx_t_vec& f, const idx_t_vec& l) override { return set_typed(b, n, f, l); }
    idx_t get_elements_in_slice(void* b, const idx_t_vec& f, const idx_t_vec& l) const override {
        need_storage("get_elements_in_slice");
        int64_t done = 0; chk(yb_var_get_slice(h->s, vi, b, f.data(), l.data(), &done)); return done;
    }
    idx_t set_elements_in_slice(const void* b, const idx_t_vec& f, const idx_t_vec& l) override {
        need_storage("set_elements_in_slice");
        int64_t done = 0; chk(yb_var_set_slice(h->s, vi, b, f.data(), l.data(), &done)); return done;
    }
    idx_t set_elements_in_slice(const yk_var_ptr source, const idx_t_vec& fs, const idx_t_vec& ft, const idx_t_vec& lt) override {
        if (!source) fail("set_elements_in_slice: null source var");
        idx_t_vec ls(fs);
        for (size_t k = 0; k < fs.size(); k++) ls[k] = fs[k] + (lt[k] - ft[k]);
        size_t n = slice_elems(ft, lt);
        std::vector<double> tmp(n);
        source->get_elements_in_slice(tmp.data(), n, fs, ls);
        return set_elements_in_slice(tmp.data(), n, ft, lt);
    }
    void set_all_elements_same(double val) override { need_storage("set_all_elements_same"); chk(yb_var_set_all_same(h->s, vi, val)); }
    idx_t set_elements_in_slice_same(double val, const idx_t_vec& f, const idx_t_vec& l, bool strict) override {
        need_storage("set_elements_in_slice_same");
        auto i = info();
        idx_t_vec ff(f), ll(l);
        if (!strict) {   // clip to the allocation
            for (int k = 0; k < i.num_dims; k++) {
                if (i.dims[k].kind == 0) continue;
                ff[k] = std::max(ff[k], first_local(i, k));
                ll[k] = std::min(ll[k], last_local(i, k));
                if (ll[k] < ff[k]) return 0;
            }
        }
        int64_t done = 0;
        chk(yb_var_set_slice_same(h->s, vi, val, ff.data(), ll.data(), &done));
        return done;
    }
    yk_reduction_result_ptr reduce_elements_in_slice(int mask, const idx_t_vec& f, const idx_t_vec& l, bool strict) override {
        need_storage("reduce_elements_in_slice");
        auto i = info();
        if (int(f.size()) != i.num_dims || int(l.size()) != i.num_dims) fail("reduce_elements_in_slice: wrong number of indices for var '" + name + "'");
        auto r = std::make_shared<B200Reduction>();
        r->mask = mask; r->mx = -HUGE_VAL; r->mn = HUGE_VAL;
        idx_t_vec ff(f), ll(l);
        if (!strict) {   // clip every index to the local range (check_indices, yk_var.cpp:485-545); nothing left: num 0, initial values
            for (int k = 0; k < i.num_dims; k++) {
                if (i.dims[k].kind == 0 && *step_wrap) continue;
                ff[k] = std::max(ff[k], first_local(i, k));
                ll[k] = std::min(ll[k], last_local(i, k));
                if (ll[k] < ff[k]) return r;
            }
        }
        double out[5];
        int64_t n = 0;
        chk(yb_var_reduce_slice(h->s, vi, ff.data(), ll.data(), out, &n));   // on the device, in double
        r->n = idx_t(n);
        r->sum = out[0]; r->sumsq = out[1]; r->prod = out[2]; r->mx = out[3]; r->mn = out[4];
        return r;
    }
    std::string format_indices(const idx_t_vec& indices) const override {
        auto i = info();
        if (int(indices.size()) != i.num_dims) fail("format_indices: wrong number of indices for var '" + name + "'");
        std::ostringstream os;
        for (int k = 0; k < i.num_dims; k++) os << (k ? ", " : "") << i.dims[k].name << "=" << indices[k];
        return os.str();
    }
    std::string format_indices(const idx_t_init_list& indices) const override { return format_indices(idx_t_vec(indices)); }
    int get_halo_exchange_l1_norm() const override { return info().halo_exchange_l1_norm; }
    void set_halo_exchange_l1_norm(int) override { fail("set_halo_exchange_l1_norm is not supported by the yask_b200 engine (norms come from the compiler)"); }
    bool is_dynamic_step_alloc() const override { return false; }
    bool set_numa_preferred(int) override { return false; }
    int get_numa_preferred() const override { return yask_numa_offload; }
    void set_pad(const std::string& dim, idx_t l, idx_t r, const char* fn) {
        auto i = info();
        chk(yb_var_set_min_pad(h->s, vi, pos(i, dim, DOMAIN, fn), l, r));
    }
    void set_left_min_pad_size(const std::string& dim, idx_t size) override { set_pad(dim, size, -1, "set_left_min_pad_size"); }
    void set_right_min_pad_size(const std::string& dim, idx_t size) override { set_pad(dim, -1, size, "set_right_min_pad_size"); }
    void set_min_pad_size(const std::string& dim, idx_t size) override { set_pad(dim, size, size, "set_min_pad_size"); }
    void set_left_halo_size(const std::string&, idx_t) override { fail("halo sizes of solution vars are fixed by the stencil compiler"); }
    void set_right_halo_size(const std::string&, idx_t) override { fail("halo sizes of solution vars are fixed by the stencil compiler"); }
    void set_halo_size(const std::string&, idx_t) override { fail("halo sizes of solution vars are fixed by the stencil compiler"); }
    void set_alloc_size(const std::string&, idx_t) override { fail("set_alloc_size: use new_fixed_size_var() to create a var with explicit sizes"); }
    void set_first_misc_index(const std::string&, idx_t) override { fail("set_first_misc_index is not supported by the yask_b200 engine"); }
    bool is_storage_allocated() const override { return prepared(); }
    idx_t get_num_storage_bytes() const override { return info().storage_bytes; }
    idx_t get_num_storage_elements() const override { auto i = info(); return i.slot_elems * i.step_alloc; }
    // Device storage of every var, fixed-size user vars included, is allocated by prepare_solution() on the device chosen there
    // (yk_var_api.hpp:1281-1296: "storage will be allocated" now OR by prepare_solution()); a call before it is therefore a
    // request that prepare_solution() honours, not an error -- the reference's Python API test makes exactly that call.
    void alloc_storage() override {}
    void release_storage() override {}
    bool is_storage_layout_identical(const yk_var_ptr other) const override {
        if (!other) return false;
        return get_dim_names() == other->get_dim_names() && get_alloc_size_vec() == other->get_alloc_size_vec();
    }
    void fuse_vars(yk_var_ptr source) override {
        auto src = std::dynamic_pointer_cast<B200Var>(source);
        if (!src) fail("fuse_vars(): the source var does not belong to the yask_b200 engine");
        chk(yb_var_fuse(h->s, vi, src->h->s, src->vi));
    }
    // Storage lives in HBM: hand out a HOST snapshot (refreshed on every call).  The reference documents no
    // layout guarantees for this buffer (aux/yk_var_api.hpp:1399-1437); writes to it are not propagated.
    void* get_raw_storage_buffer() override {
        if (!prepared()) return nullptr;
        auto i = info();
        // the step slots the API can see (a var with spare slots for the temporal tile keeps them out of this view)
        raw_mirror.resize(size_t(i.slot_elems) * size_t(i.has_step ? i.step_alloc : 1) * size_t(i.elem_bytes));
        void* dev = nullptr;
        chk(yb_var_device_ptr(h->s, vi, 0, &dev));
        chk(yb_solution_sync(h->s));
        chk(yb_copy_to_host(raw_mirror.data(), dev, raw_mirror.size()));   // step 0 lives in the first slot of the live set
        return raw_mirror.data();
    }
};

struct B200Solution : yk_solution {
    std::shared_ptr<Handle> h = std::make_shared<Handle>();
    std::string name, descr;
    std::map<std::string, idx_t> block_size;
    std::map<std::string, yk_var_ptr> var_cache;
    std::vector<hook_fn_t> before_prepare, after_prepare;
    std::vector<hook_fn_2idx_t> before_run, after_run;
    bool step_wrap = false;
    int device = -1;
    idx_t point_rcv = 0, point_rows = 0;   // shape of the receiver set (yk_set_receivers)
    std::vector<idx_t_vec> slice_shape;     // frames shape (nrows, box extents...) of each slice recorder (yk_add_slice)
    std::vector<idx_t_vec> correlator_shape;   // image shape (box extents...) of each slice correlator (yk_add_slice_correlator)

    // The reference fixes a solution's radius and element size when it builds the kernel library (`make stencil=iso3dfd
    // radius=2 real_bytes=8`, /root/reference/src/kernel/Makefile); here the library name carries them the same way:
    // libyask_kernel.iso3dfd_r2.b200.so (-DYK_STENCIL_NAME=iso3dfd_r2) is iso3dfd with radius 2, and a `_fp64` suffix
    // (iso3dfd_r4_fp64) selects 8-byte elements; iso3dfd_sponge_r<N>[_fp64], 3axis_r<N>[_fp64], 3axis_with_diags_r<N>[_fp64],
    // 3plane_r<N>[_fp64] and cube_r<N>[_fp64] do the same for those solutions.  YASK_B200_RADIUS and YASK_B200_ELEM_BYTES override
    // them at run time.
    static bool takes_radius(const std::string& base) {
        for (const char* n : {"iso3dfd", "iso3dfd_sponge", "3axis", "3axis_with_diags", "3plane", "cube"})
            if (base == n) return true;
        return false;
    }
    explicit B200Solution(const char* stencil_) {
        std::string stencil = stencil_;
        int radius = 0, elem_bytes = 0;
        const std::string fp64 = "_fp64";      // iso3dfd_fp64, <solution>_r<N>_fp64
        if (stencil.size() > fp64.size() && stencil.compare(stencil.size() - fp64.size(), fp64.size(), fp64) == 0) {
            const std::string base = stencil.substr(0, stencil.size() - fp64.size());
            const size_t r = base.rfind("_r");
            if (base == "iso3dfd" || (r != std::string::npos && r + 2 < base.size() && takes_radius(base.substr(0, r)) &&
                                      base.find_first_not_of("0123456789", r + 2) == std::string::npos)) {
                elem_bytes = 8;
                stencil = base;
            }
        }
        const size_t us = stencil.rfind("_r");
        if (us != std::string::npos && us + 2 < stencil.size() && takes_radius(stencil.substr(0, us)) &&
            stencil.find_first_not_of("0123456789", us + 2) == std::string::npos) {
            radius = atoi(stencil.c_str() + us + 2);
            stencil.resize(us);
        }
        if (const char* e = getenv("YASK_B200_RADIUS")) radius = atoi(e);
        if (const char* e = getenv("YASK_B200_ELEM_BYTES")) elem_bytes = atoi(e);
        chk(yb_solution_create(&h->s, stencil.c_str(), radius, elem_bytes));
        name = yb_solution_name(h->s);
        descr = "H100-native engine for solution '" + name + "'";
    }
    int dpos(const std::string& dim, const char* fn) const {
        int n = yb_solution_num_domain_dims(h->s);
        for (int k = 0; k < n; k++)
            if (dim == yb_solution_domain_dim_name(h->s, k)) return k;
        fail(std::string("dimension '") + dim + "' is not a domain dimension in " + fn + "()");
    }
    template <typename F> void set_vec(const idx_t_vec& v, F f, const char* fn) {
        int n = yb_solution_num_domain_dims(h->s);
        if (int(v.size()) != n) fail(std::string(fn) + ": expected " + std::to_string(n) + " value(s)");
        for (int k = 0; k < n; k++) chk(f(h->s, k, v[k]));
    }
    template <typename F> idx_t_vec get_vec(F f) const {
        idx_t_vec v;
        for (int k = 0; k < yb_solution_num_domain_dims(h->s); k++) v.push_back(f(h->s, k));
        return v;
    }
    const std::string& get_name() const override { return name; }
    const std::string& get_description() const override { return descr; }
    std::string get_target() const override { return yb_solution_target(h->s); }
    bool is_offloaded() const override { return true; }
    int get_element_bytes() const override { return yb_solution_elem_bytes(h->s); }
    std::string get_step_dim_name() const override { return yb_solution_step_dim_name(h->s); }
    int get_num_domain_dims() const override { return yb_solution_num_domain_dims(h->s); }
    string_vec get_domain_dim_names() const override { string_vec v; for (int k = 0; k < get_num_domain_dims(); k++) v.push_back(yb_solution_domain_dim_name(h->s, k)); return v; }
    string_vec get_misc_dim_names() const override {
        string_vec v;
        for (int i = 0; i < yb_num_vars(h->s); i++) {
            yb_var_info vi; chk(yb_var_info_get(h->s, i, &vi));
            for (int k = 0; k < vi.num_dims; k++)
                if (vi.dims[k].kind == 2 && std::find(v.begin(), v.end(), vi.dims[k].name) == v.end()) v.push_back(vi.dims[k].name);
        }
        return v;
    }
    void set_rank_domain_size(const std::string& dim, idx_t size) override { chk(yb_set_rank_domain_size(h->s, dpos(dim, "set_rank_domain_size"), size)); }
    void set_rank_domain_size_vec(const idx_t_vec& v) override { set_vec(v, yb_set_rank_domain_size, "set_rank_domain_size_vec"); }
    void set_rank_domain_size_vec(const idx_t_init_list& v) override { set_rank_domain_size_vec(idx_t_vec(v)); }
    idx_t get_rank_domain_size(const std::string& dim) const override { return yb_get_rank_domain_size(h->s, dpos(dim, "get_rank_domain_size")); }
    idx_t_vec get_rank_domain_size_vec() const override { return get_vec(yb_get_rank_domain_size); }
    void set_overall_domain_size(const std::string& dim, idx_t size) override { chk(yb_set_overall_domain_size(h->s, dpos(dim, "set_overall_domain_size"), size)); }
    void set_overall_domain_size_vec(const idx_t_vec& v) override { set_vec(v, yb_set_overall_domain_size, "set_overall_domain_size_vec"); }
    void set_overall_domain_size_vec(const idx_t_init_list& v) override { set_overall_domain_size_vec(idx_t_vec(v)); }
    idx_t get_overall_domain_size(const std::string& dim) const override { return yb_get_overall_domain_size(h->s, dpos(dim, "get_overall_domain_size")); }
    idx_t_vec get_overall_domain_size_vec() const override { return get_vec(yb_get_overall_domain_size); }
    // Block sizes steer the reference's CPU tiling only; they are recorded so that callers read back what they set.
    // The STEP block size is the exception: it is the reference's temporal blocking (-bt, context.cpp:657-681) and selects
    // the engine's temporal tile where one exists (iso3dfd radius <= 2: two steps per sweep; needs extra storage, so it has
    // to be set before prepare_solution() to take effect).  Results never depend on it.
    void set_block_size(const std::string& dim, idx_t size) override {
        if (dim != get_step_dim_name()) dpos(dim, "set_block_size");
        else (void)yb_set_option(h->s, "block_steps", std::to_string(size < 1 ? 1 : size).c_str());    // engines without one refuse: fine
        block_size[dim] = size;
    }
    // Mega-block steps of the step dim (the reference's -Mbt): engines without a fused rank-grid mode refuse the option: fine.
    void set_mega_block_steps(idx_t n) { (void)yb_set_option(h->s, "mega_block_steps", std::to_string(n < 1 ? 1 : n).c_str()); }
    void set_block_size_vec(const idx_t_vec& v) override { auto d = get_domain_dim_names(); if (v.size() != d.size()) fail("set_block_size_vec: wrong number of values"); for (size_t k = 0; k < d.size(); k++) block_size[d[k]] = v[k]; }
    void set_block_size_vec(const idx_t_init_list& v) override { set_block_size_vec(idx_t_vec(v)); }
    idx_t get_block_size(const std::string& dim) const override {
        if (dim != get_step_dim_name()) dpos(dim, "get_block_size");
        auto it = block_size.find(dim);
        return it == block_size.end() ? 0 : it->second;
    }
    idx_t_vec get_block_size_vec() const override { idx_t_vec v; for (auto& d : get_domain_dim_names()) v.push_back(get_block_size(d)); return v; }
    void set_num_ranks(const std::string& dim, idx_t num) override { chk(yb_set_num_ranks(h->s, dpos(dim, "set_num_ranks"), num)); }
    void set_num_ranks_vec(const idx_t_vec& v) override { set_vec(v, yb_set_num_ranks, "set_num_ranks_vec"); }
    void set_num_ranks_vec(const idx_t_init_list& v) override { set_num_ranks_vec(idx_t_vec(v)); }
    idx_t get_num_ranks(const std::string& dim) const override { return yb_get_num_ranks(h->s, dpos(dim, "get_num_ranks")); }
    idx_t_vec get_num_ranks_vec() const override { return get_vec(yb_get_num_ranks); }
    void set_rank_index(const std::string& dim, idx_t num) override { chk(yb_set_rank_index(h->s, dpos(dim, "set_rank_index"), num)); }
    void set_rank_index_vec(const idx_t_vec& v) override { set_vec(v, yb_set_rank_index, "set_rank_index_vec"); }
    void set_rank_index_vec(const idx_t_init_list& v) override { set_rank_index_vec(idx_t_vec(v)); }
    idx_t get_rank_index(const std::string& dim) const override { return yb_get_rank_index(h->s, dpos(dim, "get_rank_index")); }
    idx_t_vec get_rank_index_vec() const override { return get_vec(yb_get_rank_index); }
    int get_num_outer_threads() const override { return 1; }
    int get_num_inner_threads() const override { return 1; }

    // Options: the per-dim size families of the reference (settings.cpp:289-373: -g, -l, -b, -nr, -ri, -mp with an
    // optional dim suffix), the engine's own knobs, and the reference's CPU-tuning flags, which are accepted
    // and ignored.  Unrecognised arguments are returned, as the reference does.
    std::string apply_command_line_options(const string_vec& args) override {
        std::string rest;
        auto dims = get_domain_dim_names();
        static const char* ignored_bool[] = {"pre_auto_tune", "warmup", "use_shm", "exchange_halos", "force_scalar",
                                             "force_scalar_exchange", "bundle_allocs", "bind_inner_threads", "allow_addl_padding", "use_device_mpi",
                                             "print_suffixes", "trace", "validate", "find_loc"};
        static const char* ignored_val[] = {"outer_threads", "inner_threads", "max_threads", "thread_divisor", "numa_pref", "msg_rank", "min_exterior",
                                            "auto_tune_trial_secs", "auto_tune_radius", "auto_tune_targets", "mbt", "ep", "mp_extra"};
        for (size_t a = 0; a < args.size(); a++) {
            const std::string& arg = args[a];
            bool used = false;
            if (arg.size() > 1 && arg[0] == '-') {
                std::string key = arg.substr(1);
                auto take = [&]() -> std::string { if (a + 1 >= args.size()) fail("no argument for option '" + arg + "'"); return args[++a]; };
                // -[no-]overlap_comms (the reference's switch for exterior-first evaluation, settings.cpp) selects the same thing here
                if (key == "auto_tune" || key == "no-auto_tune") { chk(yb_solution_reset_auto_tuner(h->s, key[0] == 'n' ? 0 : 1)); used = true; }
                if (key == "overlap_comms" || key == "no-overlap_comms") { chk(yb_set_option(h->s, "overlap_comms", key[0] == 'n' ? "0" : "1")); used = true; }
                if (key == "bt") { set_block_size(get_step_dim_name(), atoll(take().c_str())); used = true; }     // temporal tile
                // the reference's mega-block steps (wave-front steps): on a rank grid, halos are exchanged once per that many steps.
                // Unlike the reference it does not default to -bt (there -bt alone keeps one exchange per step on a rank grid).
                if (key == "Mbt") { set_mega_block_steps(atoll(take().c_str())); used = true; }
                if (!used) for (auto* b : ignored_bool) if (key == b || key == std::string("no-") + b) used = true;
                if (!used) for (auto* v : ignored_val) if (key == v) { take(); used = true; }
                if (!used) {
                    struct Fam { const char* pfx; int (*fn)(yb_solution*, int, int64_t); };
                    static const Fam fams[] = {{"g", yb_set_overall_domain_size}, {"l", yb_set_rank_domain_size}, {"nr", yb_set_num_ranks},
                                               {"ri", yb_set_rank_index}, {"mp", yb_set_min_pad_size}};
                    for (auto& f : fams) {
                        std::string p = f.pfx;
                        if (key == p) { idx_t v = atoll(take().c_str()); for (size_t k = 0; k < dims.size(); k++) chk(f.fn(h->s, int(k), v)); used = true; break; }
                        for (size_t k = 0; k < dims.size() && !used; k++)
                            if (key == p + dims[k]) { chk(f.fn(h->s, int(k), atoll(take().c_str()))); used = true; }
                        if (used) break;
                    }
                }
                if (!used) for (const char* p : {"b", "mb", "nb", "pb", "Mb"}) {
                    std::string ps = p;
                    if (key == ps) { idx_t v = atoll(take().c_str()); if (ps == "b") for (auto& d : dims) block_size[d] = v; used = true; break; }
                    for (auto& d : dims) if (key == ps + d) { idx_t v = atoll(take().c_str()); if (ps == "b") block_size[d] = v; used = true; break; }
                    if (used) break;
                }
                if (!used) for (const char* k : {"fp_mode", "kernel", "tile", "lx", "grid", "gen_pf", "gen_l2_mb", "gen_sweep", "gen_sweep_lx", "fused_halo"})
                    if (key == k) { std::string v = take(); chk(yb_set_option(h->s, k, v.c_str())); used = true; break; }
                if (!used && key == "device") { device = atoi(take().c_str()); used = true; }
            }
            if (!used) rest += (rest.empty() ? "" : " ") + arg;
        }
        return rest;
    }
    std::string apply_command_line_options(const std::string& args) override {
        string_vec v; std::istringstream is(args); std::string t;
        while (is >> t) v.push_back(t);
        return apply_command_line_options(v);
    }
    std::string apply_command_line_options(int argc, char* argv[]) override {
        string_vec v;
        for (int i = 1; i < argc; i++) v.push_back(argv[i]);
        return apply_command_line_options(v);
    }
    std::string get_command_line_help() override {
        return " -g<dim> <n>   overall domain size        -l<dim> <n>   rank domain size\n"
               " -nr<dim> <n>  ranks in dim               -ri<dim> <n>  rank index in dim\n"
               " -mp<dim> <n>  minimum padding            -b<dim> <n>   block size (recorded; no effect on the GPU)\n"
               " -bt <n>       block steps: n >= 2 selects the temporal tile where the engine has one (iso3dfd fp32 radius <= 2;\n"
               "               3axis radius <= 2 in fp32 and fp64 on one rank)\n"
               " -Mbt <n>      mega-block steps: with -bt 2, n >= 2 runs the temporal tile on rank grids too, halos exchanged once per 2 steps\n"
               " -fp_mode 0|1|2  FP contraction mode      -kernel auto|tma|direct   -tile <n>   -lx <n>   -device <n>\n";
    }
    std::string get_command_line_values() override {
        std::ostringstream os;
        auto d = get_domain_dim_names();
        for (size_t k = 0; k < d.size(); k++)
            os << " -g" << d[k] << " " << yb_get_overall_domain_size(h->s, int(k)) << " -l" << d[k] << " " << yb_get_rank_domain_size(h->s, int(k)) << " -nr" << d[k]
               << " " << yb_get_num_ranks(h->s, int(k)) << " -ri" << d[k] << " " << yb_get_rank_index(h->s, int(k));
        char mbt[32];
        if (yb_get_option(h->s, "mega_block_steps", mbt, sizeof mbt) == 0) os << " -Mbt " << mbt;
        return os.str();
    }
    int get_num_vars() const override { return yb_num_vars(h->s); }
    yk_var_ptr make_var(int vi, bool fixed = false) {
        auto v = std::make_shared<B200Var>(h, vi, &step_wrap);
        v->fixed = fixed;
        auto it = var_cache.find(v->name);
        if (it != var_cache.end()) return it->second;
        var_cache[v->name] = v;
        return v;
    }
    yk_var_ptr get_var(const std::string& vname) override {
        int vi = yb_var_index(h->s, vname.c_str());
        if (vi < 0) fail("var '" + vname + "' not found in solution '" + name + "'");   // context.hpp:631-636
        return make_var(vi);
    }
    std::vector<yk_var_ptr> get_vars() override { std::vector<yk_var_ptr> v; for (int i = 0; i < yb_num_vars(h->s); i++) v.push_back(make_var(i)); return v; }
    void prepare_solution() override {
        for (auto& f : before_prepare) f(*this);
        // Rank grid of a multi-rank job (setup.cpp:228-256): when the caller did not choose one, split the first domain dim
        // (the outermost storage dim: its faces are contiguous planes); the position of this rank in the grid follows its
        // job rank, row-major over the domain dims.
        const int world = yb_comm_world(), rank = yb_comm_rank();
        const int ndd = yb_solution_num_domain_dims(h->s);
        int64_t grid = 1;
        for (int d = 0; d < ndd; d++) grid *= yb_get_num_ranks(h->s, d);
        if (world > 1) {
            if (grid == 1) { chk(yb_set_num_ranks(h->s, 0, world)); grid = world; }
            if (grid != world) fail("the rank grid has " + std::to_string(grid) + " ranks but the job has " + std::to_string(world));
            bool idx_set = false;
            for (int d = 0; d < ndd; d++) idx_set = idx_set || yb_get_rank_index(h->s, d) != 0;
            if (!idx_set) {
                int64_t r = rank;
                for (int d = ndd - 1; d >= 0; d--) { const int64_t n = yb_get_num_ranks(h->s, d); chk(yb_set_rank_index(h->s, d, r % n)); r /= n; }
            }
        }
        int dev = device;
        if (dev < 0) {
            dev = yb_comm_env_local_rank();
            const int ndev = yb_device_count();
            if (ndev > 0) dev %= ndev;
        }
        chk(yb_solution_prepare(h->s, dev));
        if (grid > 1) chk(yb_halo_connect(h->s));
        for (auto& f : after_prepare) f(*this);
    }
    idx_t get_first_rank_domain_index(const std::string& dim) const override { return yb_get_first_rank_domain_index(h->s, dpos(dim, "get_first_rank_domain_index")); }
    idx_t_vec get_first_rank_domain_index_vec() const override { return get_vec(yb_get_first_rank_domain_index); }
    idx_t get_last_rank_domain_index(const std::string& dim) const override { return yb_get_last_rank_domain_index(h->s, dpos(dim, "get_last_rank_domain_index")); }
    idx_t_vec get_last_rank_domain_index_vec() const override { return get_vec(yb_get_last_rank_domain_index); }
    void run_solution(idx_t first, idx_t last) override {
        for (auto& f : before_run) f(*this, first, last);
        chk(yb_solution_run(h->s, first, last));
        for (auto& f : after_run) f(*this, first, last);
    }
    void run_solution(idx_t step) override { run_solution(step, step); }
    void copy_vars_to_device() const override {}     // vars always live on the device
    void copy_vars_from_device() const override { chk(yb_solution_sync(h->s)); }
    void exchange_halos() override { chk(yb_exchange_halos(h->s)); }
    void end_solution() override { var_cache.clear(); }
    yk_stats_ptr get_stats() override {
        auto st = std::make_shared<B200Stats>();
        chk(yb_get_stats(h->s, &st->st));
        chk(yb_clear_stats(h->s));    // the reference's get_stats() also resets the counters (soln_apis.cpp:349-)
        return st;
    }
    void clear_stats() override { chk(yb_clear_stats(h->s)); }
    // in-run tuner over the engine's launch variants (the reference tunes CPU block sizes the same way, auto_tuner.cpp)
    void reset_auto_tuner(bool enable, bool) override { chk(yb_solution_reset_auto_tuner(h->s, enable ? 1 : 0)); }
    bool is_auto_tuner_enabled() const override { return yb_solution_is_auto_tuner_enabled(h->s) != 0; }
    void run_auto_tuner_now(bool verbose) override {
        // auto_tuner.cpp raises when called before prepare_solution().  What is tuned here are the engine's launch
        // variants (sweep tile / chunk length, prefetch distance, L2 chunking), not CPU block sizes.
        if (!yb_solution_is_prepared(h->s)) fail("run_auto_tuner_now() called without calling prepare_solution() first");
        char report[8192];
        chk(yb_solution_auto_tune(h->s, report, sizeof report));
        if (verbose) { auto out = yk_env::get_debug_output(); if (out) out->get_ostream() << "auto-tuner:\n" << report; }
    }
    void set_min_pad_size(const std::string& dim, idx_t size) override { chk(yb_set_min_pad_size(h->s, dpos(dim, "set_min_pad_size"), size)); min_pad[dim] = size; }
    std::map<std::string, idx_t> min_pad;
    idx_t get_min_pad_size(const std::string& dim) const override { dpos(dim, "get_min_pad_size"); auto it = min_pad.find(dim); return it == min_pad.end() ? 0 : it->second; }
    yk_var_ptr create(const std::string& vname, const string_vec& dims, const idx_t_vec* sizes) {
        std::vector<const char*> names;
        for (auto& d : dims) names.push_back(d.c_str());
        if (sizes && sizes->size() != dims.size()) fail("new_fixed_size_var: " + std::to_string(dims.size()) + " dim(s) but " + std::to_string(sizes->size()) + " size(s)");
        int vi = chk(yb_var_create(h->s, vname.c_str(), int(dims.size()), names.data(), sizes ? sizes->data() : nullptr));
        return make_var(vi, sizes != nullptr);
    }
    yk_var_ptr new_var(const std::string& vname, const string_vec& dims) override { return create(vname, dims, nullptr); }
    yk_var_ptr new_var(const std::string& vname, const std::initializer_list<std::string>& dims) override { return create(vname, string_vec(dims), nullptr); }
    yk_var_ptr new_fixed_size_var(const std::string& vname, const string_vec& dims, const idx_t_vec& sizes) override { return create(vname, dims, &sizes); }
    yk_var_ptr new_fixed_size_var(const std::string& vname, const std::initializer_list<std::string>& dims, const idx_t_init_list& sizes) override {
        idx_t_vec s(sizes);
        return create(vname, string_vec(dims), &s);
    }
    bool set_default_numa_preferred(int) override { return false; }
    int get_default_numa_preferred() const override { return yask_numa_offload; }
    void call_before_prepare_solution(hook_fn_t f) override { before_prepare.push_back(f); }
    void call_after_prepare_solution(hook_fn_t f) override { after_prepare.push_back(f); }
    void call_before_run_solution(hook_fn_2idx_t f) override { before_run.push_back(f); }
    void call_after_run_solution(hook_fn_2idx_t f) override { after_run.push_back(f); }
    void fuse_vars(yk_solution_ptr source) override {
        // every pair of vars with the same name (soln_apis.cpp:271-283)
        if (!source) fail("fuse_vars(): null source solution");
        for (auto& sv : source->get_vars())
            if (yb_var_index(h->s, sv->get_name().c_str()) >= 0) get_var(sv->get_name())->fuse_vars(sv);
    }
    void set_step_wrap(bool w) override { step_wrap = w; }
    bool get_step_wrap() const override { return step_wrap; }
    void set_debug_output(yask_output_ptr debug) override { yk_env::set_debug_output(debug); }
};

}  // namespace

yk_factory::yk_factory() {}
std::string yk_factory::get_version_string() { return yask_get_version_string(); }
yk_env_ptr yk_factory::new_env() const { return std::make_shared<B200Env>(); }
yk_env_ptr yk_factory::new_env(MPI_Comm) const { return std::make_shared<B200Env>(); }
yk_solution_ptr yk_factory::new_solution(yk_env_ptr env) const {
    if (!env) fail("new_solution() called with a null env");
    return std::make_shared<B200Solution>(YK_STR(YK_STENCIL_NAME));
}
yk_solution_ptr yk_factory::new_solution(yk_env_ptr env, const yk_solution_ptr source) const {
    auto s = new_solution(env);
    if (source) {   // copy the settings made through set_*() (factory.cpp:99-105)
        auto dims = source->get_domain_dim_names();
        for (auto& d : dims)
            if (source->get_overall_domain_size(d) > 0) s->set_overall_domain_size(d, source->get_overall_domain_size(d));
        s->set_num_ranks_vec(source->get_num_ranks_vec());
        s->set_rank_index_vec(source->get_rank_index_vec());
    }
    return s;
}

// ---- point sources and receivers (yask_b200_points.hpp) ----------------------------------------------------------
namespace {
B200Solution& b200(const yk_solution_ptr& soln) {
    auto* s = dynamic_cast<B200Solution*>(soln.get());
    if (!s) fail("point sources and receivers: not a solution of this engine");
    return *s;
}
std::vector<int64_t> flat_points(B200Solution& s, const std::vector<idx_t_vec>& idx, const char* what) {
    const size_t nd = size_t(yb_solution_num_domain_dims(s.h->s));
    std::vector<int64_t> out;
    for (size_t i = 0; i < idx.size(); i++) {
        if (idx[i].size() != nd)
            fail(std::string(what) + ": point " + std::to_string(i) + " has " + std::to_string(idx[i].size()) + " indices but the solution has " +
                 std::to_string(nd) + " domain dims");
        out.insert(out.end(), idx[i].begin(), idx[i].end());
    }
    return out;
}
}  // namespace

void yk_set_sources(yk_solution_ptr soln, const std::string& var, const std::vector<idx_t_vec>& idx, idx_t t0,
                    const std::vector<std::vector<double>>& amp) {
    B200Solution& s = b200(soln);
    const std::vector<int64_t> pts = flat_points(s, idx, "sources");
    std::vector<double> flat;
    for (size_t r = 0; r < amp.size(); r++) {
        if (amp[r].size() != idx.size())
            fail("sources: amplitude row " + std::to_string(r) + " has " + std::to_string(amp[r].size()) + " values for " + std::to_string(idx.size()) +
                 " source point(s)");
        flat.insert(flat.end(), amp[r].begin(), amp[r].end());
    }
    chk(yb_solution_set_sources(s.h->s, var.c_str(), int64_t(idx.size()), pts.data(), t0, int64_t(amp.size()), flat.data()));
}

void yk_set_receivers(yk_solution_ptr soln, const std::string& var, const std::vector<idx_t_vec>& idx, idx_t t0, idx_t nrows) {
    B200Solution& s = b200(soln);
    const std::vector<int64_t> pts = flat_points(s, idx, "receivers");
    chk(yb_solution_set_receivers(s.h->s, var.c_str(), int64_t(idx.size()), pts.data(), t0, nrows));
    s.point_rcv = idx_t(idx.size());
    s.point_rows = nrows;
}

void yk_get_traces(yk_solution_ptr soln, std::vector<std::vector<double>>& traces, std::vector<bool>& owned) {
    B200Solution& s = b200(soln);
    const size_t m = size_t(s.point_rcv), rows = size_t(s.point_rows);
    const int eb = yb_solution_elem_bytes(s.h->s);
    std::vector<char> raw(rows * m * eb);
    std::vector<uint8_t> own(m);
    chk(yb_solution_get_traces(s.h->s, yb_solution_is_prepared(s.h->s) ? raw.data() : nullptr, own.data()));
    traces.assign(rows, std::vector<double>(m, 0.0));
    for (size_t r = 0; r < rows; r++)
        for (size_t j = 0; j < m; j++)
            traces[r][j] = eb == 4 ? double(reinterpret_cast<const float*>(raw.data())[r * m + j]) : reinterpret_cast<const double*>(raw.data())[r * m + j];
    owned.assign(own.begin(), own.end());
}

void yk_clear_points(yk_solution_ptr soln) {
    B200Solution& s = b200(soln);
    chk(yb_solution_clear_points(s.h->s));
    s.point_rcv = s.point_rows = 0;
}

idx_t yk_get_point_launches(yk_solution_ptr soln) {
    char v[64];
    chk(yb_get_option(b200(soln).h->s, "point_launches", v, sizeof v));
    return idx_t(atoll(v));
}

namespace {
// n x k x ndd indices and n x k weights, flattened; every point must have the same k entries of ndd indices
void flat_weighted(B200Solution& s, const std::vector<std::vector<idx_t_vec>>& idx, const std::vector<std::vector<double>>& w, const char* what,
                   std::vector<int64_t>& pts, std::vector<double>& ws, size_t& k) {
    const size_t nd = size_t(yb_solution_num_domain_dims(s.h->s));
    if (idx.size() != w.size())
        fail(std::string(what) + ": " + std::to_string(idx.size()) + " index lists but " + std::to_string(w.size()) + " weight lists");
    k = idx.empty() ? 0 : idx[0].size();
    for (size_t i = 0; i < idx.size(); i++) {
        if (idx[i].size() != k || w[i].size() != k)
            fail(std::string(what) + ": point " + std::to_string(i) + " has " + std::to_string(idx[i].size()) + " entries and " +
                 std::to_string(w[i].size()) + " weights; point 0 has " + std::to_string(k) + " entries");
        for (size_t q = 0; q < k; q++) {
            if (idx[i][q].size() != nd)
                fail(std::string(what) + ": point " + std::to_string(i) + " entry " + std::to_string(q) + " has " + std::to_string(idx[i][q].size()) +
                     " indices but the solution has " + std::to_string(nd) + " domain dims");
            pts.insert(pts.end(), idx[i][q].begin(), idx[i][q].end());
        }
        ws.insert(ws.end(), w[i].begin(), w[i].end());
    }
}
}  // namespace

void yk_set_sources_weighted(yk_solution_ptr soln, const std::string& var, const std::vector<std::vector<idx_t_vec>>& idx,
                             const std::vector<std::vector<double>>& w, idx_t t0, const std::vector<std::vector<double>>& amp) {
    B200Solution& s = b200(soln);
    std::vector<int64_t> pts;
    std::vector<double> ws, flat;
    size_t k = 0;
    flat_weighted(s, idx, w, "weighted sources", pts, ws, k);
    for (size_t r = 0; r < amp.size(); r++) {
        if (amp[r].size() != idx.size())
            fail("weighted sources: amplitude row " + std::to_string(r) + " has " + std::to_string(amp[r].size()) + " values for " +
                 std::to_string(idx.size()) + " source(s)");
        flat.insert(flat.end(), amp[r].begin(), amp[r].end());
    }
    chk(yb_solution_set_sources_weighted(s.h->s, var.c_str(), int64_t(idx.size()), int64_t(k), pts.data(), ws.data(), t0, int64_t(amp.size()),
                                         flat.data()));
}

void yk_set_receivers_weighted(yk_solution_ptr soln, const std::string& var, const std::vector<std::vector<idx_t_vec>>& idx,
                               const std::vector<std::vector<double>>& w, idx_t t0, idx_t nrows) {
    B200Solution& s = b200(soln);
    std::vector<int64_t> pts;
    std::vector<double> ws;
    size_t k = 0;
    flat_weighted(s, idx, w, "weighted receivers", pts, ws, k);
    chk(yb_solution_set_receivers_weighted(s.h->s, var.c_str(), int64_t(idx.size()), int64_t(k), pts.data(), ws.data(), t0, nrows));
    s.point_rcv = idx_t(idx.size());
    s.point_rows = nrows;
}

void yk_trilinear(const std::vector<std::vector<double>>& pos, std::vector<std::vector<idx_t_vec>>& idx, std::vector<std::vector<double>>& w) {
    const size_t n = pos.size(), nd = n ? pos[0].size() : 0;
    std::vector<double> flat;
    for (size_t i = 0; i < n; i++) {
        if (pos[i].size() != nd)
            fail("trilinear: position " + std::to_string(i) + " has " + std::to_string(pos[i].size()) + " coordinates; position 0 has " + std::to_string(nd));
        flat.insert(flat.end(), pos[i].begin(), pos[i].end());
    }
    const size_t k = size_t(1) << std::min<size_t>(nd, 3);
    std::vector<int64_t> fi(n * k * nd);
    std::vector<double> fw(n * k);
    chk(yb_points_trilinear(int(nd), int64_t(n), flat.data(), fi.data(), fw.data()));
    idx.assign(n, std::vector<idx_t_vec>(k, idx_t_vec(nd)));
    w.assign(n, std::vector<double>(k));
    for (size_t i = 0; i < n; i++)
        for (size_t q = 0; q < k; q++) {
            for (size_t d = 0; d < nd; d++) idx[i][q][d] = fi[(i * k + q) * nd + d];
            w[i][q] = fw[i * k + q];
        }
}

// ---- slice recorders (yask_b200_slices.hpp) ------------------------------------------------------------------------
namespace {
B200Solution& b200_slices(const yk_solution_ptr& soln) {
    auto* s = dynamic_cast<B200Solution*>(soln.get());
    if (!s) fail("slice recorders: not a solution of this engine");
    return *s;
}
}  // namespace

namespace {
// YB_TYPE_* of a frame or image type name ("" is the element type)
int slice_type(const char* what, const char* field, const std::string& name) {
    if (name.empty()) return YB_TYPE_ELEM;
    if (name == "float64") return YB_TYPE_F64;
    if (name == "float32") return YB_TYPE_F32;
    if (name == "float16") return YB_TYPE_F16;
    if (name == "bfloat16") return YB_TYPE_BF16;
    fail(std::string(what) + ": unknown " + field + " '" + name + "' (expected float16, bfloat16, float32 or float64)");
    return YB_TYPE_ELEM;
}

int type_bytes(int type) { return type == YB_TYPE_F64 ? 8 : type == YB_TYPE_F32 ? 4 : 2; }

// float -> IEEE half bits, round to nearest even: overflow to +-inf, subnormal results kept, NaN a quiet NaN
uint16_t half_bits(float v) {
    uint32_t f;
    memcpy(&f, &v, 4);
    const uint32_t sign = f & 0x80000000u;
    f ^= sign;
    uint16_t o;
    if (f >= (127u + 16u) << 23) {                      // |v| >= 2^16 (inf, NaN)
        o = f > 255u << 23 ? 0x7e00 : 0x7c00;
    } else if (f < 113u << 23) {                        // |v| < 2^-14: a half subnormal or zero; adding 0.5f rounds to its grid
        const uint32_t magic = 126u << 23;
        float x, m;
        memcpy(&x, &f, 4);
        memcpy(&m, &magic, 4);
        x += m;
        uint32_t xi;
        memcpy(&xi, &x, 4);
        o = uint16_t(xi - magic);
    } else {                                            // normal: rebias, round the 13 dropped bits to nearest even
        f += (uint32_t(15 - 127) << 23) + 0xfffu + ((f >> 13) & 1u);
        o = uint16_t(f >> 13);                          // a carry past 65504 gives 0x7c00, inf
    }
    return uint16_t(o | (sign >> 16));
}

double half_value(uint16_t h) {
    const int e = (h >> 10) & 0x1f, m = h & 0x3ff;
    const double v = e == 0 ? std::ldexp(double(m), -24) : e == 31 ? (m ? NAN : INFINITY) : std::ldexp(double(m | 0x400), e - 25);
    return h & 0x8000 ? -v : v;
}

// float -> bfloat16 bits, round to nearest even (NaN a quiet NaN)
uint16_t bf16_bits(float v) {
    uint32_t f;
    memcpy(&f, &v, 4);
    if (std::isnan(v)) return uint16_t((f >> 16) | 0x40);
    return uint16_t((f + 0x7fffu + ((f >> 16) & 1u)) >> 16);
}

double bf16_value(uint16_t b) {
    const uint32_t f = uint32_t(b) << 16;
    float v;
    memcpy(&v, &f, 4);
    return v;
}

// element i of a buffer of YB_TYPE_* `type`, widened exactly to double
double widened(const std::vector<char>& raw, int type, size_t i) {
    const char* p = raw.data() + i * size_t(type_bytes(type));
    if (type == YB_TYPE_F64) { double v; memcpy(&v, p, 8); return v; }
    if (type == YB_TYPE_F32) { float v; memcpy(&v, p, 4); return v; }
    uint16_t h;
    memcpy(&h, p, 2);
    return type == YB_TYPE_F16 ? half_value(h) : bf16_value(h);
}
}  // namespace

idx_t yk_add_slice(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0, idx_t nrows,
                   const idx_t_vec& stride, idx_t every) {
    return yk_add_slice_typed(soln, var, first, last, t0, nrows, "", stride, every);
}

idx_t yk_add_slice_typed(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0, idx_t nrows,
                         const std::string& dtype, const idx_t_vec& stride, idx_t every) {
    B200Solution& s = b200_slices(soln);
    const size_t nd = size_t(yb_solution_num_domain_dims(s.h->s));
    if (first.size() != nd || last.size() != nd || (!stride.empty() && stride.size() != nd))
        fail("slice: first, last and stride need " + std::to_string(nd) + " domain indices each");
    const int type = slice_type("slice", "dtype", dtype);
    const std::vector<int64_t> f(first.begin(), first.end()), l(last.begin(), last.end()), st(stride.begin(), stride.end());
    int64_t id = -1;
    chk(yb_solution_add_slice_typed(s.h->s, var.c_str(), f.data(), l.data(), st.empty() ? nullptr : st.data(), t0, every, nrows, type, &id));
    idx_t_vec shape{nrows};
    for (size_t k = 0; k < nd; k++) shape.push_back((l[k] - f[k]) / (st.empty() ? 1 : st[k]) + 1);
    s.slice_shape.resize(size_t(id) + 1);
    s.slice_shape[size_t(id)] = shape;
    return idx_t(id);
}

void yk_get_slice_frames(yk_solution_ptr soln, idx_t id, std::vector<double>& frames, idx_t_vec& shape, std::vector<bool>& owned) {
    B200Solution& s = b200_slices(soln);
    if (id < 0 || size_t(id) >= s.slice_shape.size()) fail("get_slice_frames: no slice recorder " + std::to_string(id));
    shape = s.slice_shape[size_t(id)];
    size_t box = 1;
    for (size_t k = 1; k < shape.size(); k++) box *= size_t(shape[k]);
    const size_t n = size_t(shape[0]) * box;
    int type = 0;
    chk(yb_solution_get_slice_frame_type(s.h->s, id, &type));
    std::vector<char> raw(n * size_t(type_bytes(type)));
    std::vector<uint8_t> own(box);
    chk(yb_solution_get_slice_frames(s.h->s, id, yb_solution_is_prepared(s.h->s) ? raw.data() : nullptr, own.data()));
    frames.resize(n);
    for (size_t i = 0; i < n; i++) frames[i] = widened(raw, type, i);
    owned.assign(own.begin(), own.end());
}

void yk_clear_slices(yk_solution_ptr soln) {
    B200Solution& s = b200_slices(soln);
    chk(yb_solution_clear_slices(s.h->s));
    s.slice_shape.clear();
}

idx_t yk_get_slice_launches(yk_solution_ptr soln) {
    char v[64];
    chk(yb_get_option(b200_slices(soln).h->s, "slice_launches", v, sizeof v));
    return idx_t(atoll(v));
}

idx_t yk_add_slice_injector(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                            idx_t nrows, const std::vector<double>& frames, const idx_t_vec& stride, idx_t every, bool set) {
    return yk_add_slice_injector_typed(soln, var, first, last, t0, nrows, frames, "", stride, every, set);
}

idx_t yk_add_slice_injector_typed(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                                  idx_t nrows, const std::vector<double>& frames, const std::string& dtype, const idx_t_vec& stride,
                                  idx_t every, bool set) {
    B200Solution& s = b200_slices(soln);
    int type = slice_type("slice injector", "dtype", dtype);
    const size_t nd = size_t(yb_solution_num_domain_dims(s.h->s));
    if (first.size() != nd || last.size() != nd || (!stride.empty() && stride.size() != nd))
        fail("slice injector: first, last and stride need " + std::to_string(nd) + " domain indices each");
    const std::vector<int64_t> f(first.begin(), first.end()), l(last.begin(), last.end()), st(stride.begin(), stride.end());
    size_t n = nrows > 0 ? size_t(nrows) : 0;
    for (size_t k = 0; k < nd; k++) n *= l[k] >= f[k] && (st.empty() || st[k] > 0) ? size_t((l[k] - f[k]) / (st.empty() ? 1 : st[k]) + 1) : 0;
    if (n && frames.size() != n)
        fail("slice injector: " + std::to_string(frames.size()) + " frame values given, nrows x the decimated box is " + std::to_string(n));
    int64_t id = -1;
    const int mode = set ? YB_INJECT_SET : YB_INJECT_ADD;
    const bool f32 = yb_solution_elem_bytes(s.h->s) == 4;
    if (type == YB_TYPE_ELEM) type = f32 ? YB_TYPE_F32 : YB_TYPE_F64;
    // each value rounded to the element type, then to the frame type (a type the solution does not allow is refused below)
    std::vector<char> fr(frames.size() * size_t(type_bytes(type)));
    for (size_t i = 0; i < frames.size(); i++) {
        const double t = f32 ? double(float(frames[i])) : frames[i];
        char* p = fr.data() + i * size_t(type_bytes(type));
        if (type == YB_TYPE_F64) { memcpy(p, &t, 8); continue; }
        const float v = float(t);
        if (type == YB_TYPE_F32) { memcpy(p, &v, 4); continue; }
        const uint16_t h = type == YB_TYPE_F16 ? half_bits(v) : bf16_bits(v);
        memcpy(p, &h, 2);
    }
    chk(yb_solution_add_slice_injector_typed(s.h->s, var.c_str(), f.data(), l.data(), st.empty() ? nullptr : st.data(), t0, every, nrows, mode,
                                             type, fr.data(), &id));
    return idx_t(id);
}

void yk_clear_slice_injectors(yk_solution_ptr soln) { chk(yb_solution_clear_slice_injectors(b200_slices(soln).h->s)); }

idx_t yk_get_slice_injector_launches(yk_solution_ptr soln) {
    char v[64];
    chk(yb_get_option(b200_slices(soln).h->s, "slice_injector_launches", v, sizeof v));
    return idx_t(atoll(v));
}

namespace {
// the C ABI's box arguments of a slice call, checked against the solution's domain dims
void slice_box(B200Solution& s, const char* what, const idx_t_vec& first, const idx_t_vec& last, const idx_t_vec& stride,
               std::vector<int64_t>& f, std::vector<int64_t>& l, std::vector<int64_t>& st) {
    const size_t nd = size_t(yb_solution_num_domain_dims(s.h->s));
    if (first.size() != nd || last.size() != nd || (!stride.empty() && stride.size() != nd))
        fail(std::string(what) + ": first, last and stride need " + std::to_string(nd) + " domain indices each");
    f.assign(first.begin(), first.end());
    l.assign(last.begin(), last.end());
    st.assign(stride.begin(), stride.end());
}
}  // namespace

idx_t yk_add_slice_injector_from(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                                 idx_t nrows, yk_solution_ptr src, idx_t src_id, bool reverse, const idx_t_vec& stride, idx_t every, bool set) {
    B200Solution& s = b200_slices(soln);
    std::vector<int64_t> f, l, st;
    slice_box(s, "slice injector", first, last, stride, f, l, st);
    int64_t id = -1;
    chk(yb_solution_add_slice_injector_from(s.h->s, var.c_str(), f.data(), l.data(), st.empty() ? nullptr : st.data(), t0, every, nrows,
                                            set ? YB_INJECT_SET : YB_INJECT_ADD, b200_slices(src).h->s, src_id, reverse ? 1 : 0, &id));
    return idx_t(id);
}

idx_t yk_add_slice_correlator(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                              idx_t nrows, yk_solution_ptr src, idx_t src_id, bool reverse, const idx_t_vec& stride, idx_t every) {
    return yk_add_slice_correlator_typed(soln, var, first, last, t0, nrows, "", src, src_id, reverse, stride, every);
}

idx_t yk_add_slice_correlator_typed(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                                    idx_t nrows, const std::string& image_dtype, yk_solution_ptr src, idx_t src_id, bool reverse,
                                    const idx_t_vec& stride, idx_t every) {
    B200Solution& s = b200_slices(soln);
    std::vector<int64_t> f, l, st;
    slice_box(s, "slice correlator", first, last, stride, f, l, st);
    const int type = slice_type("slice correlator", "image_dtype", image_dtype);
    int64_t id = -1;
    chk(yb_solution_add_slice_correlator_typed(s.h->s, var.c_str(), f.data(), l.data(), st.empty() ? nullptr : st.data(), t0, every, nrows,
                                               src ? b200_slices(src).h->s : nullptr, src_id, reverse ? 1 : 0, type, &id));
    idx_t_vec shape;
    for (size_t k = 0; k < f.size(); k++) shape.push_back((l[k] - f[k]) / (st.empty() ? 1 : st[k]) + 1);
    s.correlator_shape.resize(size_t(id) + 1);
    s.correlator_shape[size_t(id)] = shape;
    return idx_t(id);
}

idx_t yk_add_slice_correlator_var(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                                  idx_t nrows, yk_solution_ptr src, const std::string& src_var, idx_t src_t0, const idx_t_vec& stride,
                                  idx_t every, const std::string& image_dtype) {
    B200Solution& s = b200_slices(soln);
    std::vector<int64_t> f, l, st;
    slice_box(s, "slice correlator", first, last, stride, f, l, st);
    const int type = slice_type("slice correlator", "image_dtype", image_dtype);
    int64_t id = -1;
    chk(yb_solution_add_slice_correlator_var(s.h->s, var.c_str(), f.data(), l.data(), st.empty() ? nullptr : st.data(), t0, every, nrows,
                                             src ? b200_slices(src).h->s : nullptr, src_var.c_str(), src_t0, type, &id));
    idx_t_vec shape;
    for (size_t k = 0; k < f.size(); k++) shape.push_back((l[k] - f[k]) / (st.empty() ? 1 : st[k]) + 1);
    s.correlator_shape.resize(size_t(id) + 1);
    s.correlator_shape[size_t(id)] = shape;
    return idx_t(id);
}

void yk_get_correlator_image(yk_solution_ptr soln, idx_t id, std::vector<double>& image, idx_t_vec& shape, std::vector<bool>& owned) {
    B200Solution& s = b200_slices(soln);
    if (id < 0 || size_t(id) >= s.correlator_shape.size()) fail("get_correlator_image: no slice correlator " + std::to_string(id));
    shape = s.correlator_shape[size_t(id)];
    size_t n = 1;
    for (idx_t e : shape) n *= size_t(e);
    int type = 0;
    chk(yb_solution_get_correlator_image_type(s.h->s, id, &type));
    std::vector<char> raw(n * size_t(type_bytes(type)));
    std::vector<uint8_t> own(n);
    chk(yb_solution_get_correlator_image(s.h->s, id, yb_solution_is_prepared(s.h->s) ? raw.data() : nullptr, own.data()));
    image.resize(n);
    for (size_t i = 0; i < n; i++) image[i] = widened(raw, type, i);
    owned.assign(own.begin(), own.end());
}

void yk_clear_slice_correlators(yk_solution_ptr soln) {
    B200Solution& s = b200_slices(soln);
    chk(yb_solution_clear_slice_correlators(s.h->s));
    s.correlator_shape.clear();
}

idx_t yk_get_slice_correlator_launches(yk_solution_ptr soln) {
    char v[64];
    chk(yb_get_option(b200_slices(soln).h->s, "slice_correlator_launches", v, sizeof v));
    return idx_t(atoll(v));
}

}  // namespace yask
