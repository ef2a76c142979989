// Python module `yask_kernel`: the reference's Python kernel API over the yask_b200 engine.
//
// The reference generates this module with SWIG from its C++ API headers
// (/root/reference/src/kernel/swig/yask_kernel_api.i, built per stencil and target by src/kernel/Makefile as
// lib/_yask_kernel.so + yask/yask_kernel.py); here the same classes -- the C++ mirror in
// yask_b200/include/yask_kernel_api.hpp, implemented by yk_api.cpp over the C ABI -- are bound with pybind11, one module
// per solution (yask_b200/lib/python/<stencil>/yask_kernel*.so), so that scripts written for the reference
// (`import yask_kernel as yk; yk.yk_factory() ...`) run unchanged.  What SWIG's interface file prescribes is kept:
//   * yask_exception surfaces as Python RuntimeError carrying get_message()            (yask_kernel_api.i:62-69)
//   * `void* buffer_ptr` arguments take any writable object with the buffer protocol   (%pybuffer_mutable_string)
//   * vectors of indices / names / vars convert from and to Python sequences            (%template vector_idx ...)
//   * global constants live in `cvar` (yask_kernel.cvar.yask_numa_local, aux/yk_solution_api.hpp:47-73)
// Host-side glue only: every call lands in the C++ mirror, which holds no compute path.
#include <pybind11/functional.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cstdint>

#include "../include/yask_kernel_api.hpp"
#include "../include/yask_b200_points.hpp"
#include "../include/yask_b200_slices.hpp"

namespace py = pybind11;
using namespace yask;

namespace {

// element count and pointer of a Python buffer that must hold the slice [first, last]
struct Buf {
    void* ptr;
    size_t elems;      // number of items of the buffer's own item size (4 or 8 bytes: the caller picks the solution's element type)
};
Buf writable(py::buffer& b, bool need_write) {
    py::buffer_info bi = b.request(need_write);
    if (bi.itemsize != 4 && bi.itemsize != 8) throw yask_exception("YASK error: the buffer must hold float32 or float64 items");
    return Buf{bi.ptr, size_t(bi.size)};
}
size_t slice_elems(const idx_t_vec& first, const idx_t_vec& last) {
    if (first.size() != last.size()) throw yask_exception("YASK error: first and last indices differ in length");
    size_t n = 1;
    for (size_t i = 0; i < first.size(); i++) n *= last[i] >= first[i] ? size_t(last[i] - first[i] + 1) : 0;
    return n;
}

}  // namespace

PYBIND11_MODULE(yask_kernel, m) {
    m.doc() = "YASK kernel API (yask_b200 engine): same classes and methods as the reference's SWIG-generated yask_kernel module";
    py::register_exception_translator([](std::exception_ptr p) {
        try {
            if (p) std::rethrow_exception(p);
        } catch (const yask_exception& e) {
            PyErr_SetString(PyExc_RuntimeError, e.get_message());
        }
    });
    m.def("yask_get_version_string", &yask_get_version_string);

    // ---- constants (SWIG: module.cvar) ----
    py::module_ cvar = m.def_submodule("cvar", "global constants of the C++ API");
    cvar.attr("yask_numa_local") = yask_numa_local;
    cvar.attr("yask_numa_interleave") = yask_numa_interleave;
    cvar.attr("yask_numa_none") = yask_numa_none;
    cvar.attr("yask_numa_offload") = yask_numa_offload;

    // ---- output objects (yask_common_api.hpp) ----
    py::class_<yask_output, yask_output_ptr>(m, "yask_output");
    py::class_<yask_file_output, yask_output, yask_file_output_ptr>(m, "yask_file_output")
        .def("get_filename", &yask_file_output::get_filename)
        .def("close", &yask_file_output::close);
    py::class_<yask_string_output, yask_output, yask_string_output_ptr>(m, "yask_string_output")
        .def("get_string", &yask_string_output::get_string)
        .def("discard", &yask_string_output::discard);
    py::class_<yask_stdout_output, yask_output, yask_stdout_output_ptr>(m, "yask_stdout_output");
    py::class_<yask_null_output, yask_output, yask_null_output_ptr>(m, "yask_null_output");
    py::class_<yask_output_factory>(m, "yask_output_factory")
        .def(py::init<>())
        .def("new_file_output", &yask_output_factory::new_file_output)
        .def("new_string_output", &yask_output_factory::new_string_output)
        .def("new_stdout_output", &yask_output_factory::new_stdout_output)
        .def("new_null_output", &yask_output_factory::new_null_output);

    // ---- factory, env, stats ----
    py::class_<yk_env, yk_env_ptr>(m, "yk_env")
        .def_static("set_debug_output", &yk_env::set_debug_output)
        .def_static("disable_debug_output", &yk_env::disable_debug_output)
        .def_static("get_debug_output", &yk_env::get_debug_output)
        .def_static("set_trace_enabled", &yk_env::set_trace_enabled)
        .def_static("is_trace_enabled", &yk_env::is_trace_enabled)
        .def("get_num_ranks", &yk_env::get_num_ranks)
        .def("get_rank_index", &yk_env::get_rank_index)
        .def("global_barrier", &yk_env::global_barrier)
        .def("sum_over_ranks", &yk_env::sum_over_ranks)
        .def("assert_equality_over_ranks", &yk_env::assert_equality_over_ranks)
        .def("finalize", &yk_env::finalize);
    py::class_<yk_stats, yk_stats_ptr>(m, "yk_stats")
        .def("get_num_elements", &yk_stats::get_num_elements)
        .def("get_num_steps_done", &yk_stats::get_num_steps_done)
        .def("get_num_writes_done", &yk_stats::get_num_writes_done)
        .def("get_est_fp_ops_done", &yk_stats::get_est_fp_ops_done)
        .def("get_elapsed_secs", &yk_stats::get_elapsed_secs);
    py::class_<yk_factory>(m, "yk_factory")
        .def(py::init<>())
        .def("get_version_string", &yk_factory::get_version_string)
        .def("new_env", [](const yk_factory& f) { return f.new_env(); })
        .def("new_solution", [](const yk_factory& f, yk_env_ptr env) { return f.new_solution(env); })
        .def("new_solution", [](const yk_factory& f, yk_env_ptr env, yk_solution_ptr src) { return f.new_solution(env, src); });

    // ---- reduction result ----
    py::class_<yk_var::yk_reduction_result, yk_var::yk_reduction_result_ptr>(m, "yk_reduction_result")
        .def("get_reduction_mask", &yk_var::yk_reduction_result::get_reduction_mask)
        .def("get_num_elements_reduced", &yk_var::yk_reduction_result::get_num_elements_reduced)
        .def("get_sum", &yk_var::yk_reduction_result::get_sum)
        .def("get_sum_squares", &yk_var::yk_reduction_result::get_sum_squares)
        .def("get_product", &yk_var::yk_reduction_result::get_product)
        .def("get_max", &yk_var::yk_reduction_result::get_max)
        .def("get_min", &yk_var::yk_reduction_result::get_min);

    // ---- var ----
    py::class_<yk_var, yk_var_ptr> var(m, "yk_var");
    var.attr("yk_sum_reduction") = int(yk_var::yk_sum_reduction);
    var.attr("yk_sum_squares_reduction") = int(yk_var::yk_sum_squares_reduction);
    var.attr("yk_product_reduction") = int(yk_var::yk_product_reduction);
    var.attr("yk_max_reduction") = int(yk_var::yk_max_reduction);
    var.attr("yk_min_reduction") = int(yk_var::yk_min_reduction);
    var.def("get_name", &yk_var::get_name)
        .def("get_num_dims", &yk_var::get_num_dims)
        .def("get_dim_names", &yk_var::get_dim_names)
        .def("get_num_domain_dims", &yk_var::get_num_domain_dims)
        .def("is_dim_used", &yk_var::is_dim_used)
        .def("is_fixed_size", &yk_var::is_fixed_size)
        .def("get_first_local_index", &yk_var::get_first_local_index)
        .def("get_first_local_index_vec", &yk_var::get_first_local_index_vec)
        .def("get_last_local_index", &yk_var::get_last_local_index)
        .def("get_last_local_index_vec", &yk_var::get_last_local_index_vec)
        .def("get_first_rank_alloc_index", &yk_var::get_first_rank_alloc_index)
        .def("get_last_rank_alloc_index", &yk_var::get_last_rank_alloc_index)
        .def("get_alloc_size", &yk_var::get_alloc_size)
        .def("get_alloc_size_vec", &yk_var::get_alloc_size_vec)
        .def("get_first_valid_step_index", &yk_var::get_first_valid_step_index)
        .def("get_last_valid_step_index", &yk_var::get_last_valid_step_index)
        .def("get_rank_domain_size", &yk_var::get_rank_domain_size)
        .def("get_rank_domain_size_vec", &yk_var::get_rank_domain_size_vec)
        .def("get_first_rank_domain_index", &yk_var::get_first_rank_domain_index)
        .def("get_first_rank_domain_index_vec", &yk_var::get_first_rank_domain_index_vec)
        .def("get_last_rank_domain_index", &yk_var::get_last_rank_domain_index)
        .def("get_last_rank_domain_index_vec", &yk_var::get_last_rank_domain_index_vec)
        .def("get_left_halo_size", &yk_var::get_left_halo_size)
        .def("get_right_halo_size", &yk_var::get_right_halo_size)
        .def("get_first_rank_halo_index", &yk_var::get_first_rank_halo_index)
        .def("get_first_rank_halo_index_vec", &yk_var::get_first_rank_halo_index_vec)
        .def("get_last_rank_halo_index", &yk_var::get_last_rank_halo_index)
        .def("get_last_rank_halo_index_vec", &yk_var::get_last_rank_halo_index_vec)
        .def("get_left_pad_size", &yk_var::get_left_pad_size)
        .def("get_right_pad_size", &yk_var::get_right_pad_size)
        .def("get_left_extra_pad_size", &yk_var::get_left_extra_pad_size)
        .def("get_right_extra_pad_size", &yk_var::get_right_extra_pad_size)
        .def("get_first_misc_index", &yk_var::get_first_misc_index)
        .def("get_last_misc_index", &yk_var::get_last_misc_index)
        .def("are_indices_local", [](const yk_var& v, const idx_t_vec& i) { return v.are_indices_local(i); })
        .def("get_element", [](const yk_var& v, const idx_t_vec& i) { return v.get_element(i); })
        .def("set_element", [](yk_var& v, double val, const idx_t_vec& i, bool strict) { return v.set_element(val, i, strict); },
             py::arg("val"), py::arg("indices"), py::arg("strict_indices") = true)
        .def("add_to_element", [](yk_var& v, double val, const idx_t_vec& i, bool strict) { return v.add_to_element(val, i, strict); },
             py::arg("val"), py::arg("indices"), py::arg("strict_indices") = true)
        .def("set_all_elements_same", &yk_var::set_all_elements_same)
        .def("set_elements_in_slice_same",
             [](yk_var& v, double val, const idx_t_vec& first, const idx_t_vec& last, bool strict) { return v.set_elements_in_slice_same(val, first, last, strict); },
             py::arg("val"), py::arg("first_indices"), py::arg("last_indices"), py::arg("strict_indices") = true)
        // buffer <-> slice: the buffer's element type must be the solution's (float or double), as with the reference's void* overloads
        .def("get_elements_in_slice",
             [](const yk_var& v, py::buffer b, const idx_t_vec& first, const idx_t_vec& last) {
                 const Buf bf = writable(b, true);
                 const size_t n = slice_elems(first, last);
                 if (bf.elems < n) throw yask_exception("YASK error: buffer too small for the requested slice");
                 return v.get_elements_in_slice(bf.ptr, first, last);
             })
        .def("set_elements_in_slice",
             [](yk_var& v, py::buffer b, const idx_t_vec& first, const idx_t_vec& last) {
                 const Buf bf = writable(b, false);
                 const size_t n = slice_elems(first, last);
                 if (bf.elems < n) throw yask_exception("YASK error: buffer too small for the requested slice");
                 return v.set_elements_in_slice(static_cast<const void*>(bf.ptr), first, last);
             })
        .def("set_elements_in_slice",
             [](yk_var& v, yk_var_ptr src, const idx_t_vec& fs, const idx_t_vec& ft, const idx_t_vec& lt) { return v.set_elements_in_slice(src, fs, ft, lt); })
        .def("reduce_elements_in_slice",
             [](yk_var& v, int mask, const idx_t_vec& first, const idx_t_vec& last, bool strict) { return v.reduce_elements_in_slice(mask, first, last, strict); },
             py::arg("reduction_mask"), py::arg("first_indices"), py::arg("last_indices"), py::arg("strict_indices") = true)
        .def("format_indices", [](const yk_var& v, const idx_t_vec& i) { return v.format_indices(i); })
        .def("get_halo_exchange_l1_norm", &yk_var::get_halo_exchange_l1_norm)
        .def("set_halo_exchange_l1_norm", &yk_var::set_halo_exchange_l1_norm)
        .def("is_dynamic_step_alloc", &yk_var::is_dynamic_step_alloc)
        .def("set_numa_preferred", &yk_var::set_numa_preferred)
        .def("get_numa_preferred", &yk_var::get_numa_preferred)
        .def("set_left_min_pad_size", &yk_var::set_left_min_pad_size)
        .def("set_right_min_pad_size", &yk_var::set_right_min_pad_size)
        .def("set_min_pad_size", &yk_var::set_min_pad_size)
        .def("set_left_halo_size", &yk_var::set_left_halo_size)
        .def("set_right_halo_size", &yk_var::set_right_halo_size)
        .def("set_halo_size", &yk_var::set_halo_size)
        .def("set_alloc_size", &yk_var::set_alloc_size)
        .def("set_first_misc_index", &yk_var::set_first_misc_index)
        .def("is_storage_allocated", &yk_var::is_storage_allocated)
        .def("get_num_storage_bytes", &yk_var::get_num_storage_bytes)
        .def("get_num_storage_elements", &yk_var::get_num_storage_elements)
        .def("alloc_storage", &yk_var::alloc_storage)
        .def("release_storage", &yk_var::release_storage)
        .def("is_storage_layout_identical", &yk_var::is_storage_layout_identical)
        .def("fuse_vars", &yk_var::fuse_vars)
        // SWIG hands out an opaque pointer object that int() turns into the address; an int serves the same scripts
        .def("get_raw_storage_buffer", [](yk_var& v) { return reinterpret_cast<std::uintptr_t>(v.get_raw_storage_buffer()); });

    // ---- solution ----
    py::class_<yk_solution, yk_solution_ptr>(m, "yk_solution")
        .def("get_name", &yk_solution::get_name)
        .def("get_description", &yk_solution::get_description)
        .def("get_target", &yk_solution::get_target)
        .def("is_offloaded", &yk_solution::is_offloaded)
        .def("get_element_bytes", &yk_solution::get_element_bytes)
        .def("get_step_dim_name", &yk_solution::get_step_dim_name)
        .def("get_num_domain_dims", &yk_solution::get_num_domain_dims)
        .def("get_domain_dim_names", &yk_solution::get_domain_dim_names)
        .def("get_misc_dim_names", &yk_solution::get_misc_dim_names)
        .def("set_rank_domain_size", &yk_solution::set_rank_domain_size)
        .def("set_rank_domain_size_vec", [](yk_solution& s, const idx_t_vec& v) { s.set_rank_domain_size_vec(v); })
        .def("get_rank_domain_size", &yk_solution::get_rank_domain_size)
        .def("get_rank_domain_size_vec", &yk_solution::get_rank_domain_size_vec)
        .def("set_overall_domain_size", &yk_solution::set_overall_domain_size)
        .def("set_overall_domain_size_vec", [](yk_solution& s, const idx_t_vec& v) { s.set_overall_domain_size_vec(v); })
        .def("get_overall_domain_size", &yk_solution::get_overall_domain_size)
        .def("get_overall_domain_size_vec", &yk_solution::get_overall_domain_size_vec)
        .def("set_block_size", &yk_solution::set_block_size)
        .def("set_block_size_vec", [](yk_solution& s, const idx_t_vec& v) { s.set_block_size_vec(v); })
        .def("get_block_size", &yk_solution::get_block_size)
        .def("get_block_size_vec", &yk_solution::get_block_size_vec)
        .def("set_num_ranks", &yk_solution::set_num_ranks)
        .def("set_num_ranks_vec", [](yk_solution& s, const idx_t_vec& v) { s.set_num_ranks_vec(v); })
        .def("get_num_ranks", &yk_solution::get_num_ranks)
        .def("get_num_ranks_vec", &yk_solution::get_num_ranks_vec)
        .def("set_rank_index", &yk_solution::set_rank_index)
        .def("set_rank_index_vec", [](yk_solution& s, const idx_t_vec& v) { s.set_rank_index_vec(v); })
        .def("get_rank_index", &yk_solution::get_rank_index)
        .def("get_rank_index_vec", &yk_solution::get_rank_index_vec)
        .def("get_num_outer_threads", &yk_solution::get_num_outer_threads)
        .def("get_num_inner_threads", &yk_solution::get_num_inner_threads)
        .def("apply_command_line_options", [](yk_solution& s, const std::string& a) { return s.apply_command_line_options(a); })
        .def("apply_command_line_options", [](yk_solution& s, const string_vec& a) { return s.apply_command_line_options(a); })
        .def("get_command_line_help", &yk_solution::get_command_line_help)
        .def("get_command_line_values", &yk_solution::get_command_line_values)
        .def("get_num_vars", &yk_solution::get_num_vars)
        .def("get_var", &yk_solution::get_var)
        .def("get_vars", &yk_solution::get_vars)
        .def("prepare_solution", &yk_solution::prepare_solution)
        .def("get_first_rank_domain_index", &yk_solution::get_first_rank_domain_index)
        .def("get_first_rank_domain_index_vec", &yk_solution::get_first_rank_domain_index_vec)
        .def("get_last_rank_domain_index", &yk_solution::get_last_rank_domain_index)
        .def("get_last_rank_domain_index_vec", &yk_solution::get_last_rank_domain_index_vec)
        .def("run_solution", [](yk_solution& s, idx_t first, idx_t last) { s.run_solution(first, last); })
        .def("run_solution", [](yk_solution& s, idx_t step) { s.run_solution(step); })
        .def("copy_vars_to_device", &yk_solution::copy_vars_to_device)
        .def("copy_vars_from_device", &yk_solution::copy_vars_from_device)
        .def("exchange_halos", &yk_solution::exchange_halos)
        .def("end_solution", &yk_solution::end_solution)
        .def("get_stats", &yk_solution::get_stats)
        .def("clear_stats", &yk_solution::clear_stats)
        .def("reset_auto_tuner", &yk_solution::reset_auto_tuner, py::arg("enable"), py::arg("verbose") = false)
        .def("is_auto_tuner_enabled", &yk_solution::is_auto_tuner_enabled)
        .def("run_auto_tuner_now", &yk_solution::run_auto_tuner_now, py::arg("verbose") = true)
        .def("set_min_pad_size", &yk_solution::set_min_pad_size)
        .def("get_min_pad_size", &yk_solution::get_min_pad_size)
        .def("new_var", [](yk_solution& s, const std::string& name, const string_vec& dims) { return s.new_var(name, dims); })
        .def("new_fixed_size_var",
             [](yk_solution& s, const std::string& name, const string_vec& dims, const idx_t_vec& sizes) { return s.new_fixed_size_var(name, dims, sizes); })
        .def("set_default_numa_preferred", &yk_solution::set_default_numa_preferred)
        .def("get_default_numa_preferred", &yk_solution::get_default_numa_preferred)
        .def("call_before_prepare_solution", &yk_solution::call_before_prepare_solution)
        .def("call_after_prepare_solution", &yk_solution::call_after_prepare_solution)
        .def("call_before_run_solution", &yk_solution::call_before_run_solution)
        .def("call_after_run_solution", &yk_solution::call_after_run_solution)
        .def("fuse_vars", &yk_solution::fuse_vars)
        .def("set_step_wrap", &yk_solution::set_step_wrap)
        .def("get_step_wrap", &yk_solution::get_step_wrap)
        .def("set_debug_output", &yk_solution::set_debug_output);

    // ---- point sources and receivers on the device (yask_b200_points.hpp; not in the reference API) ----
    m.def("yk_set_sources", &yk_set_sources, py::arg("soln"), py::arg("var"), py::arg("idx"), py::arg("t0"), py::arg("amp"));
    m.def("yk_set_receivers", &yk_set_receivers, py::arg("soln"), py::arg("var"), py::arg("idx"), py::arg("t0"), py::arg("nrows"));
    m.def("yk_get_traces", [](yk_solution_ptr s) {
        std::vector<std::vector<double>> traces;
        std::vector<bool> owned;
        yk_get_traces(s, traces, owned);
        return py::make_tuple(traces, owned);
    }, py::arg("soln"), "(traces[row][receiver] as floats, owned[receiver])");
    m.def("yk_clear_points", &yk_clear_points, py::arg("soln"));
    m.def("yk_get_point_launches", &yk_get_point_launches, py::arg("soln"));
    m.def("yk_set_sources_weighted", &yk_set_sources_weighted, py::arg("soln"), py::arg("var"), py::arg("idx"), py::arg("w"), py::arg("t0"),
          py::arg("amp"));
    m.def("yk_set_receivers_weighted", &yk_set_receivers_weighted, py::arg("soln"), py::arg("var"), py::arg("idx"), py::arg("w"), py::arg("t0"),
          py::arg("nrows"));
    m.def("yk_trilinear", [](const std::vector<std::vector<double>>& pos) {
        std::vector<std::vector<idx_t_vec>> idx;
        std::vector<std::vector<double>> w;
        yk_trilinear(pos, idx, w);
        return py::make_tuple(idx, w);
    }, py::arg("pos"), "(idx[point][entry][dim], w[point][entry]) of the trilinear support of each position");

    // ---- slice recorders on the device (yask_b200_slices.hpp; not in the reference API) ----
    m.def("yk_add_slice", &yk_add_slice, py::arg("soln"), py::arg("var"), py::arg("first"), py::arg("last"), py::arg("t0"), py::arg("nrows"),
          py::arg("stride") = idx_t_vec{}, py::arg("every") = 1);
    m.def("yk_get_slice_frames", [](yk_solution_ptr s, idx_t id) {
        std::vector<double> frames;
        idx_t_vec shape;
        std::vector<bool> owned;
        yk_get_slice_frames(s, id, frames, shape, owned);
        return py::make_tuple(frames, shape, owned);
    }, py::arg("soln"), py::arg("id"), "(frames as a flat list of floats, shape (nrows, box extents...), owned per box point)");
    m.def("yk_clear_slices", &yk_clear_slices, py::arg("soln"));
    m.def("yk_get_slice_launches", &yk_get_slice_launches, py::arg("soln"));
    // ---- slice injectors on the device (yask_b200_slices.hpp; not in the reference API) ----
    m.def("yk_add_slice_injector", &yk_add_slice_injector, py::arg("soln"), py::arg("var"), py::arg("first"), py::arg("last"), py::arg("t0"),
          py::arg("nrows"), py::arg("frames"), py::arg("stride") = idx_t_vec{}, py::arg("every") = 1, py::arg("set") = false);
    m.def("yk_clear_slice_injectors", &yk_clear_slice_injectors, py::arg("soln"));
    m.def("yk_get_slice_injector_launches", &yk_get_slice_injector_launches, py::arg("soln"));
    m.def("yk_add_slice_injector_from", &yk_add_slice_injector_from, py::arg("soln"), py::arg("var"), py::arg("first"), py::arg("last"),
          py::arg("t0"), py::arg("nrows"), py::arg("src"), py::arg("src_id"), py::arg("reverse") = false, py::arg("stride") = idx_t_vec{},
          py::arg("every") = 1, py::arg("set") = false);
    // ---- slice correlators on the device (yask_b200_slices.hpp; not in the reference API) ----
    m.def("yk_add_slice_correlator", &yk_add_slice_correlator, py::arg("soln"), py::arg("var"), py::arg("first"), py::arg("last"),
          py::arg("t0"), py::arg("nrows"), py::arg("src") = yk_solution_ptr(), py::arg("src_id") = 0, py::arg("reverse") = false,
          py::arg("stride") = idx_t_vec{}, py::arg("every") = 1);
    m.def("yk_add_slice_correlator_var", &yk_add_slice_correlator_var, py::arg("soln"), py::arg("var"), py::arg("first"), py::arg("last"),
          py::arg("t0"), py::arg("nrows"), py::arg("src"), py::arg("src_var"), py::arg("src_t0"), py::arg("stride") = idx_t_vec{},
          py::arg("every") = 1, py::arg("image_dtype") = "");
    m.def("yk_get_correlator_image", [](yk_solution_ptr s, idx_t id) {
        std::vector<double> image;
        idx_t_vec shape;
        std::vector<bool> owned;
        yk_get_correlator_image(s, id, image, shape, owned);
        return py::make_tuple(image, shape, owned);
    }, py::arg("soln"), py::arg("id"), "(image as a flat list of floats, shape (box extents...), owned per box point)");
    m.def("yk_clear_slice_correlators", &yk_clear_slice_correlators, py::arg("soln"));
    m.def("yk_get_slice_correlator_launches", &yk_get_slice_correlator_launches, py::arg("soln"));
    // ---- frame and image types of the slice calls ("float16", "bfloat16", "float32", "float64"; "" the element type) ----
    m.def("yk_add_slice_typed", &yk_add_slice_typed, py::arg("soln"), py::arg("var"), py::arg("first"), py::arg("last"), py::arg("t0"),
          py::arg("nrows"), py::arg("dtype"), py::arg("stride") = idx_t_vec{}, py::arg("every") = 1);
    m.def("yk_add_slice_injector_typed", &yk_add_slice_injector_typed, py::arg("soln"), py::arg("var"), py::arg("first"), py::arg("last"),
          py::arg("t0"), py::arg("nrows"), py::arg("frames"), py::arg("dtype"), py::arg("stride") = idx_t_vec{}, py::arg("every") = 1,
          py::arg("set") = false);
    m.def("yk_add_slice_correlator_typed", &yk_add_slice_correlator_typed, py::arg("soln"), py::arg("var"), py::arg("first"), py::arg("last"),
          py::arg("t0"), py::arg("nrows"), py::arg("image_dtype"), py::arg("src") = yk_solution_ptr(), py::arg("src_id") = 0,
          py::arg("reverse") = false, py::arg("stride") = idx_t_vec{}, py::arg("every") = 1);
}
