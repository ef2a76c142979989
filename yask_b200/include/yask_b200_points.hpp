// Point sources and receivers applied on the device inside run_solution(): an extension of the C++ kernel API of this engine.
//
// The reference API has no such calls; its users inject a source wavelet and record receivers from the host, one step at a time:
//
//     for (idx_t t = 0; t < nt; t++) {
//         soln->run_solution(t);
//         p->add_to_element(w[t], {t + 1, sx, sy, sz});
//         for (j ...) trace[t][j] = p->get_element({t + 1, rx[j], ry[j], rz[j]});
//     }
//
// With the functions below the same shot is one soln->run_solution(0, nt - 1) call and gives the same bits: after every step u a
// run computes, amp[u - t0][i] is added to var(u, idx[i]) for every source in list order (rounded like add_to_element), then
// var(u, ridx[j]) is stored into traces[u - t0r][j].  They are free functions, not members: yk_solution keeps the reference's
// vtable layout.  Semantics, validation and the rank-grid rules: yb_solution_set_sources in include/yask_b200.h.
#pragma once
#include "yask_kernel_api.hpp"

namespace yask {

// idx: one vector of global domain indices (x, y, z order of get_domain_dim_names()) per source; amp: one row per step from t0,
// each with idx.size() amplitudes.  Replaces the previous source set.
void yk_set_sources(yk_solution_ptr soln, const std::string& var, const std::vector<idx_t_vec>& idx, idx_t t0,
                    const std::vector<std::vector<double>>& amp);
// Record var(u, idx[j]) into traces[u - t0][j] for t0 <= u < t0 + nrows.  Replaces the previous receiver set.
void yk_set_receivers(yk_solution_ptr soln, const std::string& var, const std::vector<idx_t_vec>& idx, idx_t t0, idx_t nrows);
// traces[row][j] (element values widened to double; rows not recorded yet are 0); owned[j]: this rank records receiver j.
void yk_get_traces(yk_solution_ptr soln, std::vector<std::vector<double>>& traces, std::vector<bool>& owned);
// Remove both sets: later runs take their usual launch path again.
void yk_clear_points(yk_solution_ptr soln);
// Point-kernel launches since prepare_solution().
idx_t yk_get_point_launches(yk_solution_ptr soln);

}  // namespace yask
