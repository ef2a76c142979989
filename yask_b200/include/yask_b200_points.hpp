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

// Weighted sets: sources and receivers between grid points (yb_solution_set_sources_weighted in include/yask_b200.h).  idx[i][q]
// is the q-th support point of point i (global domain indices) and w[i][q] its weight; every point has the same number of
// entries.  Sources add w[i][q] * amp[u - t0][i] in (i, q) order; receiver j records the double sum of w[j][q] * var(u, idx[j][q])
// rounded to the element type.  Each replaces the set of its kind.
void yk_set_sources_weighted(yk_solution_ptr soln, const std::string& var, const std::vector<std::vector<idx_t_vec>>& idx,
                             const std::vector<std::vector<double>>& w, idx_t t0, const std::vector<std::vector<double>>& amp);
void yk_set_receivers_weighted(yk_solution_ptr soln, const std::string& var, const std::vector<std::vector<idx_t_vec>>& idx,
                               const std::vector<std::vector<double>>& w, idx_t t0, idx_t nrows);
// Trilinear support of real-valued positions in global index units (yb_points_trilinear): idx[i] gets 2^ndd points, w[i] their
// weights, x varying slowest.
void yk_trilinear(const std::vector<std::vector<double>>& pos, std::vector<std::vector<idx_t_vec>>& idx, std::vector<std::vector<double>>& w);

}  // namespace yask
