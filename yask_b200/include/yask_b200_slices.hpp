// Slice recorders, injectors and correlators on the device inside run_solution(): an extension of the C++ kernel API of this engine.
//
// The reference API has no such calls; its users record a receiver plane or a snapshot from the host, one step at a time:
//
//     for (idx_t t = 0; t < nt; t++) {
//         soln->run_solution(t);
//         if ((t + 1) % k == 0) p->get_elements_in_slice(frame[(t + 1) / k], {t + 1, x0, y0, z0}, {t + 1, x1, y1, z1});
//     }
//
// With the functions below the same frames come from one soln->run_solution(0, nt - 1) call, bit for bit: after every step u a
// run computes (and after that step's sources and receivers, yask_b200_points.hpp), if u - t0 is a multiple of `every` and
// r = (u - t0) / every < nrows, frame r holds var(u) at first[d], first[d] + stride[d], ... <= last[d].  They are free functions,
// not members: yk_solution keeps the reference's vtable layout.  Semantics, storage and the rank-grid rules:
// yb_solution_add_slice in include/yask_b200.h.
#pragma once
#include "yask_kernel_api.hpp"

namespace yask {

// first, last: global domain indices (x, y, z order of get_domain_dim_names()), inclusive; stride: empty for 1 in every dim.
// Returns the recorder's id (0, 1, ... until yk_clear_slices).
idx_t yk_add_slice(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0, idx_t nrows,
                   const idx_t_vec& stride = {}, idx_t every = 1);
// frames: nrows x the decimated box, row-major, the last domain dim fastest, widened to double (rows not recorded yet and points
// this rank does not own are 0); shape: (nrows, box extents...); owned: per box point, this rank records it.
void yk_get_slice_frames(yk_solution_ptr soln, idx_t id, std::vector<double>& frames, idx_t_vec& shape, std::vector<bool>& owned);
// Remove every recorder: later runs take their usual launch path again.
void yk_clear_slices(yk_solution_ptr soln);
// Recording launches since prepare_solution().
idx_t yk_get_slice_launches(yk_solution_ptr soln);

// Slice injectors, the dual of the recorders: replaces the host loop
//
//     soln->run_solution(t);  p->get_elements_in_slice(box, ...);  box[::stride] (+)= frame[r];  p->set_elements_in_slice(box, ...);
//
// After every step u a run computes, if u - t0 is a multiple of `every` and r = (u - t0) / every < nrows, frame r is set into
// (set = true) or added to (one add in the element type) var(u) at first[d], first[d] + stride[d], ... <= last[d], before that
// step's sources, receivers and recorders.  frames: nrows x the decimated box, row-major, the last domain dim fastest, given as
// doubles and rounded once to the element type.  Semantics and the rank-grid rules: yb_solution_add_slice_injector in
// include/yask_b200.h.  Returns the injector's id (0, 1, ... until yk_clear_slice_injectors; separate from the recorders').
idx_t yk_add_slice_injector(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                            idx_t nrows, const std::vector<double>& frames, const idx_t_vec& stride = {}, idx_t every = 1, bool set = false);
// Remove every injector: later runs take their usual launch path again.
void yk_clear_slice_injectors(yk_solution_ptr soln);
// Injecting launches since prepare_solution().
idx_t yk_get_slice_injector_launches(yk_solution_ptr soln);
// An injector whose frames are those of recorder src_id of solution src (which may be soln), read on the device with no copy: row
// r reads recorder row nrows - 1 - r when reverse, else r.  Checks, sharing and ordering: yb_solution_add_slice_correlator.
idx_t yk_add_slice_injector_from(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                                 idx_t nrows, yk_solution_ptr src, idx_t src_id, bool reverse = false, const idx_t_vec& stride = {},
                                 idx_t every = 1, bool set = false);

// Slice correlators, the imaging condition of a reverse-time shot: replaces the host loop
//
//     soln->run_solution(t);  p->get_elements_in_slice(box, ...);  image += frame[r] * box[::stride];
//
// After every step u a run computes, if u - t0 is a multiple of `every` and r = (u - t0) / every < nrows, image += var(u) * b at
// first[d], first[d] + stride[d], ... <= last[d], the product and the sum each rounded to the element type, after that step's
// recorders.  b is var(u) when src is null (the illumination), else row r (nrows - 1 - r when reverse) of recorder src_id of src
// (which may be soln).  Semantics and checks: yb_solution_add_slice_correlator in include/yask_b200.h.  Returns the correlator's
// id (0, 1, ... until yk_clear_slice_correlators; separate from the recorders' and injectors').
idx_t yk_add_slice_correlator(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                              idx_t nrows, yk_solution_ptr src = nullptr, idx_t src_id = 0, bool reverse = false,
                              const idx_t_vec& stride = {}, idx_t every = 1);
// A correlator whose b is var src_var of another prepared solution src on the same device at the paired step: image += var(u) *
// src_var(src_t0 + (u - t0)), for a source wavefield rebuilt backwards in time beside the adjoint run instead of stored as
// snapshots.  Semantics, checks and ordering: yb_solution_add_slice_correlator_var in include/yask_b200.h.  Shares the ids,
// getters and launch counter of the other correlators.
idx_t yk_add_slice_correlator_var(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                                  idx_t nrows, yk_solution_ptr src, const std::string& src_var, idx_t src_t0, const idx_t_vec& stride = {},
                                  idx_t every = 1, const std::string& image_dtype = "");
// image: the decimated box, row-major, the last domain dim fastest, widened to double (points this rank does not own are 0);
// shape: the box extents; owned: per box point, this rank holds it.
void yk_get_correlator_image(yk_solution_ptr soln, idx_t id, std::vector<double>& image, idx_t_vec& shape, std::vector<bool>& owned);
// Remove every correlator and free its image.
void yk_clear_slice_correlators(yk_solution_ptr soln);
// Correlating launches since prepare_solution(): one per step with a row due, and a second right after it when a correlator with a
// source var (yk_add_slice_correlator_var) has a row due too.
idx_t yk_get_slice_correlator_launches(yk_solution_ptr soln);

// Frame and image types (the typed calls): "float16", "bfloat16", "float32" or "float64"; "" is the element type.  Allowed
// combinations, rounding and storage: YB_TYPE_* and the typed calls in include/yask_b200.h.  The getters above widen every type
// to double exactly.
//
// A recorder whose frames are held in `dtype`: frame[r][pt] = var(u, pt) rounded to nearest even.
idx_t yk_add_slice_typed(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0, idx_t nrows,
                         const std::string& dtype, const idx_t_vec& stride = {}, idx_t every = 1);
// A host-fed injector whose frames are held in `dtype`: each value is rounded to the element type, then to nearest even to dtype.
idx_t yk_add_slice_injector_typed(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                                  idx_t nrows, const std::vector<double>& frames, const std::string& dtype, const idx_t_vec& stride = {},
                                  idx_t every = 1, bool set = false);
// A correlator whose image is held in `image_dtype` ("float64" in an fp32 solution: image + double(var) * double(b)).
idx_t yk_add_slice_correlator_typed(yk_solution_ptr soln, const std::string& var, const idx_t_vec& first, const idx_t_vec& last, idx_t t0,
                                    idx_t nrows, const std::string& image_dtype, yk_solution_ptr src = nullptr, idx_t src_id = 0,
                                    bool reverse = false, const idx_t_vec& stride = {}, idx_t every = 1);

}  // namespace yask
