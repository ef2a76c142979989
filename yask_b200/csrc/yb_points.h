// Point sources and receivers applied on the device inside run_solution() (yb_points.cu).
//
// A solution may carry one source set (a var, N global domain points, a first step t0 and an amplitude table amp[nrows][N])
// and one receiver set (a var, M global domain points, a first step t0r and nrows_r rows).  Whenever a run has computed step u,
// every source whose row u - t0 is in the table is added to var(u, point) in list order, then every receiver row u - t0r in
// range records var(u, point) -- bit for bit what the reference API loop run_solution(t, t) / add_to_element / get_element gives.
// Each rank keeps only the points of its own domain.
// Either set may instead be weighted (k support entries of grid points and double weights per point, e.g. the trilinear corners
// of a position between grid points): sources add w * amp, receivers record the double sum of w * var rounded to the element
// type (semantics in include/yask_b200.h, rank-grid rules in DESIGN.md 3.7).
#pragma once
#include "yb_core.h"

namespace yb {

struct PointSet {
    bool set = false;
    int var = -1;
    int step_off = 1;              // step the var's writing stage computes, relative to t (+1 forward, -1 reverse solutions)
    int64_t n = 0, t0 = 0, nrows = 0;
    int k = 0;                     // support entries per point of a weighted set (0: an on-grid set, one grid point per point)
    std::vector<int64_t> idx;      // n x ndd global domain indices (weighted: n x k x ndd)
    std::vector<double> w;         // weighted sets: n x k weights
    std::vector<double> amp;       // nrows x n (sources only)
};

// This rank's share of the point sets (points_plan; host only, needs the rank geometry but no device)
struct PointPlan {
    // sources grouped by point, groups in order of first appearance: group g applies the amplitude columns
    // src_col[grp_first[g] .. grp_first[g+1]) in list order
    std::vector<long long> grp_off;      // element offset of the point in a step slot of the source var
    std::vector<long long> grp_loc;      // 3 per group: rank-local domain coordinates (0 for missing dims)
    std::vector<int> grp_first, src_col;
    std::vector<double> src_w;           // weighted sources: the weight of each src_col entry ...
    std::vector<int> src_q;              // ... and its support entry (point_groups text)
    std::vector<long long> rcv_off, rcv_loc;    // weighted receivers: rcv_off per support entry, no rcv_loc
    std::vector<int> rcv_col;            // receiver list index (trace column) of each owned receiver
    std::vector<int> rcv_first;          // weighted receivers: entries rcv_first[j] .. rcv_first[j+1) of owned receiver j
    std::vector<double> rcv_w;           // weighted receivers: weight per entry
    std::vector<unsigned char> owned;    // per receiver of the list: recorded by this rank
};

struct PointsState {
    PointSet src, rcv;
    PointPlan plan;
    bool stale = true;             // plan, device tables and trace buffer are rebuilt at the next run
    std::vector<void*> dev;        // device allocations of the tables below
    long long *d_grp_off = nullptr, *d_grp_loc = nullptr, *d_rcv_off = nullptr, *d_rcv_loc = nullptr;
    int *d_grp_first = nullptr, *d_src_col = nullptr, *d_rcv_col = nullptr, *d_rcv_first = nullptr;
    double *d_amp = nullptr, *d_src_w = nullptr, *d_rcv_w = nullptr;
    int num_sms = 0;               // of the solution's device: caps the weighted kernels' grids
    bool rcv_pending = false;      // rank grid: weighted receivers of step pending_t wait for that step's last exchange
    int64_t pending_t = 0;
    void* d_trace = nullptr;       // nrows_r x M elements of the solution's type
    int64_t launches = 0;          // point-kernel launches since prepare (read-only option point_launches)
};

// which owned points one launch applies: all, those outside `interior` (exterior slabs of a rank grid) or those inside it
enum { PTS_ALL = 0, PTS_EXTERIOR = 1, PTS_INTERIOR = 2 };

void points_free(PointsState* p);
// The var of a point set or a slice recorder (`what` prefixes the messages): step dim, every domain dim, no misc dim, written by
// a stage; step_off: the step its writing stage computes, relative to t
int point_var(const Solution& s, const char* what, const char* name, int& vi, int& step_off);
bool geometry_known(const Solution& s);         // plan_geometry() or prepare_solution() has run
// a rank grid whose halos are exchanged once per pair of steps (block_steps=2 + mega_block_steps=2), known from plan_geometry()
bool fused_pair_rank_grid(const Solution& s);
void points_preload();                       // load the point kernel now (preload_kernel)
bool points_active(const Solution& s);
// refuse point sets on a rank grid whose halos are exchanged once per pair of steps (fixed at prepare on every rank)
int points_check_mode(const Solution& s);
int points_plan(Solution& s);                 // validation + ownership + grouping (host)
int points_begin_run(Solution& s);            // plan, upload and trace allocation after a change
// the point launches of step t (the step the stage loop just computed from t), in this order: weighted sources, the on-grid
// kernel, weighted receivers (deferred on a rank grid, see points_record_pending).  Returns #kernels launched or <0
int points_launch(Solution& s, int64_t t, int sel, const Box& interior, cudaStream_t st);
// rank grid: record the weighted receivers deferred by points_launch.  Called right after the wait for the step's last exchange
// (the next step's first stage, or the end of the run), so that halo cells hold the neighbours' values of that step
int points_record_pending(Solution& s, cudaStream_t st);
// read-only option point_groups: this rank's grouped source table, groups in application order separated by ';', each the
// comma-separated list indices of the sources it adds, in the order it adds them (e.g. "0,2;1"); a weighted set writes each
// entry as source/support entry (e.g. "0/3,2/0;1/0")
std::string points_groups_text(const Solution& s);
// rank-local x range [x0, x1] of the sources this rank applies at step t; false when it applies none
bool points_source_x_range(const Solution& s, int64_t t, int64_t& x0, int64_t& x1);

}  // namespace yb
