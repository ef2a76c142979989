// Point sources and receivers on the device (yb_points.h): one small launch per computed step adds the source wavelet at a
// few points and records the field at the receiver points, so that a whole shot runs in one run_solution() call instead of
// the reference API loop run_solution(t, t) / add_to_element / get_element, which pays host round trips on every step.
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <map>

#include "yb_halo.h"
#include "yb_points.h"

namespace yb {

namespace {

struct PointArgs {
    void* src_slot;                 // step slot of the source var (null: no source row this step)
    const long long* grp_off;
    const long long* grp_loc;
    const int* grp_first;
    const int* src_col;
    const double* amp_row;          // amp[u - t0]
    int ngrp;
    const void* rcv_slot;           // step slot of the receiver var (null: no receiver row this step)
    const long long* rcv_off;
    const long long* rcv_loc;
    const int* rcv_col;
    void* trace_row;                // trace[u - t0r]
    int nrcv;
    int sel;                        // PTS_*
    long long ib[3], ie[3];         // interior box (rank-local) for PTS_EXTERIOR / PTS_INTERIOR
};

template <typename A>
__device__ __forceinline__ bool selected(const A& a, const long long* loc) {
    if (a.sel == PTS_ALL) return true;
    const bool in = loc[0] >= a.ib[0] && loc[0] < a.ie[0] && loc[1] >= a.ib[1] && loc[1] < a.ie[1] && loc[2] >= a.ib[2] && loc[2] < a.ie[2];
    return a.sel == PTS_INTERIOR ? in : !in;
}

// the rounding of yk_var::add_to_element: the sum is formed in the element type
__device__ __forceinline__ float add_amp(float v, double a) { return __fadd_rn(v, __double2float_rn(a)); }
__device__ __forceinline__ double add_amp(double v, double a) { return __dadd_rn(v, a); }

// ONE CTA: a thread applies every source of one point in list order (the host grouped duplicates, so no two threads touch one
// element and no atomics reorder the adds), the CTA barrier makes the sums visible, then the receivers are read.  Offsets are
// 64-bit: a slot may hold more than 2^31 elements.
template <typename T>
__global__ void __launch_bounds__(256) points_kernel(PointArgs a) {
    if (a.src_slot) {
        T* base = static_cast<T*>(a.src_slot);
        for (int g = threadIdx.x; g < a.ngrp; g += blockDim.x) {
            if (!selected(a, a.grp_loc + 3 * g)) continue;
            T v = base[a.grp_off[g]];
            for (int k = a.grp_first[g]; k < a.grp_first[g + 1]; k++) v = add_amp(v, a.amp_row[a.src_col[k]]);
            base[a.grp_off[g]] = v;
        }
    }
    __syncthreads();
    if (a.rcv_slot) {
        const T* base = static_cast<const T*>(a.rcv_slot);
        T* out = static_cast<T*>(a.trace_row);
        for (int j = threadIdx.x; j < a.nrcv; j += blockDim.x)
            if (selected(a, a.rcv_loc + 3 * j)) out[a.rcv_col[j]] = base[a.rcv_off[j]];
    }
}

// Weighted sets (yb_solution_set_sources_weighted / set_receivers_weighted).  Both kernels are multi-CTA and grid-stride, and
// every product and sum is rounded on its own (__dmul_rn / __dadd_rn: no FMA), so the bits are those of the host formula.
struct WeightedSrcArgs {
    void* slot;                     // step slot of the source var
    const long long* grp_off;       // per group: element offset in the slot (64-bit)
    const long long* grp_loc;       // per group: rank-local coordinates (for sel)
    const int* grp_first;           // entries grp_first[g] .. grp_first[g+1) of group g, in (source, support entry) order
    const int* col;                 // per entry: amplitude column (source list index)
    const double* w;                // per entry: weight
    const double* amp_row;          // amp[u - t0]
    int ngrp;
    int sel;                        // PTS_*
    long long ib[3], ie[3];
};

struct WeightedRcvArgs {
    const void* slot;               // step slot of the receiver var
    const long long* off;           // per entry: element offset in the slot; may reach into halo cells
    const int* first;               // entries first[j] .. first[j+1) of owned receiver j, in support order
    const int* col;                 // per owned receiver: trace column
    const double* w;                // per entry: weight
    void* trace_row;                // trace[u - t0r]
    int nrcv;
};

__device__ __forceinline__ void store_elem(float* p, double v) { *p = __double2float_rn(v); }
__device__ __forceinline__ void store_elem(double* p, double v) { *p = v; }

// A thread owns one group -- every entry on one element -- so no two threads touch an element and no atomics are needed; the
// entries are added in list order: v = v + w * amp, the product in double, the sum with add_to_element's rounding.
template <typename T>
__global__ void __launch_bounds__(256) weighted_sources_kernel(WeightedSrcArgs a) {
    T* base = static_cast<T*>(a.slot);
    for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < a.ngrp; g += gridDim.x * blockDim.x) {
        if (!selected(a, a.grp_loc + 3 * g)) continue;
        const long long o = a.grp_off[g];
        T v = base[o];
        for (int e = a.grp_first[g]; e < a.grp_first[g + 1]; e++) v = add_amp(v, __dmul_rn(a.w[e], a.amp_row[a.col[e]]));
        base[o] = v;
    }
}

// A thread owns one receiver and sums its entries in order from +0.0 in double, then rounds once to the element type.
template <typename T>
__global__ void __launch_bounds__(256) weighted_receivers_kernel(WeightedRcvArgs a) {
    const T* base = static_cast<const T*>(a.slot);
    T* out = static_cast<T*>(a.trace_row);
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < a.nrcv; j += gridDim.x * blockDim.x) {
        double acc = 0.0;
        for (int e = a.first[j]; e < a.first[j + 1]; e++) acc = __dadd_rn(acc, __dmul_rn(a.w[e], double(base[a.off[e]])));
        store_elem(out + a.col[j], acc);
    }
}

constexpr int CTAS_PER_SM = 8;      // grid cap of the weighted kernels (grid-stride: the cap bounds the launch, not the result)

unsigned grid_for(const PointsState& p, size_t n) {
    return unsigned(std::min<size_t>((n + 255) / 256, size_t(std::max(p.num_sms, 1)) * CTAS_PER_SM));
}

const char* set_name(bool src) { return src ? "sources" : "receivers"; }

template <typename V>
int upload(PointsState& p, V*& dst, const std::vector<V>& src) {
    dst = nullptr;
    if (src.empty()) return 0;
    void* d = nullptr;
    YB_CUDA(cudaMalloc(&d, src.size() * sizeof(V)));
    p.dev.push_back(d);
    YB_CUDA(cudaMemcpy(d, src.data(), src.size() * sizeof(V), cudaMemcpyHostToDevice));
    dst = static_cast<V*>(d);
    return 0;
}

void release_device(PointsState& p) {
    for (void* d : p.dev) cudaFree(d);
    p.dev.clear();
    if (p.d_trace) cudaFree(p.d_trace);
    p.d_trace = nullptr;
    p.d_grp_off = p.d_grp_loc = p.d_rcv_off = p.d_rcv_loc = nullptr;
    p.d_grp_first = p.d_src_col = p.d_rcv_col = p.d_rcv_first = nullptr;
    p.d_amp = p.d_src_w = p.d_rcv_w = nullptr;
}

// Ranks of a split dim: every rank but the last holds ceil(overall / nranks) points (compute_rank_geometry)
void rank_box_of(const Solution& s, int d, int64_t g, int64_t& ri, int64_t& off, int64_t& size) {
    const int64_t nr = s.num_ranks[d], os = s.overall_size[d], per = (os + nr - 1) / nr;
    ri = std::min(g / per, nr - 1);
    off = per * ri;
    size = ri == nr - 1 ? os - per * (nr - 1) : per;
}

// Weighted receiver j on a rank grid: the owner is the rank holding its first nonzero entry; every other entry must be in the
// owner's domain or in a halo cell the owner's exchange refreshes (within the var's halo, toward a neighbour the var talks to).
// A receiver that reads halo cells needs them to stay put until it is recorded (DESIGN 3.7): its var written by the last stage
// and either two step slots or two stages.  Every rank checks every receiver, so all ranks refuse together.
int check_weighted_receiver(const Solution& s, const PointSet& ps, int64_t j, const int64_t* ri, const int64_t* roff, const int64_t* rsize) {
    const Var& v = s.vars[ps.var];
    bool halo = false;
    for (int64_t q = 0; q < ps.k; q++) {
        if (ps.w[size_t(j * ps.k + q)] == 0) continue;
        const int64_t* g = &ps.idx[size_t(j * ps.k + q) * s.ndd];
        int dir[3] = {0, 0, 0};
        for (int d = 0; d < s.ndd; d++) {
            const int64_t l = g[d] - roff[d];
            const Dim* dd = v.domain_dim(d);
            if (l < 0 && -l > dd->spec.halo_l)
                return set_error(YB_EUNSUPPORTED, "receivers: receiver %lld entry %lld lies %lld cell(s) below the first '%s' of its owner rank, "
                                                  "beyond var '%s''s halo of %lld there: a receiver may reach past a rank interface only as far as "
                                                  "the halo exchange refreshes", (long long)j, (long long)q, (long long)-l, s.spec.domain_dims[d].c_str(),
                                 v.spec.name.c_str(), (long long)dd->spec.halo_l);
            if (l >= rsize[d] && l - rsize[d] >= dd->spec.halo_r)
                return set_error(YB_EUNSUPPORTED, "receivers: receiver %lld entry %lld lies %lld cell(s) above the last '%s' of its owner rank, "
                                                  "beyond var '%s''s halo of %lld there: a receiver may reach past a rank interface only as far as "
                                                  "the halo exchange refreshes", (long long)j, (long long)q, (long long)(l - rsize[d] + 1),
                                 s.spec.domain_dims[d].c_str(), v.spec.name.c_str(), (long long)dd->spec.halo_r);
            dir[d] = l < 0 ? -1 : l >= rsize[d] ? 1 : 0;
        }
        if (!dir[0] && !dir[1] && !dir[2]) continue;
        // the neighbour in direction dir fills these cells with its pushes toward us, direction -dir
        const int back[3] = {-dir[0], -dir[1], -dir[2]};
        if (!var_talks_to(v, back))
            return set_error(YB_EUNSUPPORTED, "receivers: receiver %lld entry %lld is a halo cell of its owner rank (%lld,%lld,%lld) toward the "
                                              "neighbour in direction (%d,%d,%d), but var '%s' exchanges halos only with neighbours at most %d "
                                              "dim(s) away: this %s exchange is not done, so the receiver cannot be recorded",
                             (long long)j, (long long)q, (long long)ri[0], (long long)ri[1], (long long)ri[2], dir[0], dir[1], dir[2],
                             v.spec.name.c_str(), v.spec.l1_norm, abs(dir[0]) + abs(dir[1]) + abs(dir[2]) == 2 ? "edge" : "corner");
        halo = true;
    }
    if (!halo) return 0;
    bool last = false;
    for (int o : s.spec.stages.back().outputs) last = last || o == ps.var;
    if (!last)
        return set_error(YB_EUNSUPPORTED, "receivers: receiver %lld straddles a rank interface (it reads halo cells), and var '%s' is not "
                                          "written by the last stage of '%s': a neighbour may overwrite those cells before the step's last "
                                          "exchange, after which the receiver is recorded", (long long)j, v.spec.name.c_str(), s.spec.name.c_str());
    if (v.nslots() < 2 && s.spec.stages.size() < 2)
        return set_error(YB_EUNSUPPORTED, "receivers: receiver %lld straddles a rank interface (it reads halo cells), and var '%s' keeps one "
                                          "step slot in the one-stage solution '%s': a neighbour may push the next step into those cells before "
                                          "they are read", (long long)j, v.spec.name.c_str(), s.spec.name.c_str());
    return 0;
}

}  // namespace

// The var of a point set or a slice recorder (`what`): step dim, every domain dim, no misc dim, written by a stage.
int point_var(const Solution& s, const char* what, const char* name, int& vi, int& step_off) {
    if (!name) return set_error(YB_EINVAL, "%s: null var name", what);
    vi = -1;
    for (size_t i = 0; i < s.vars.size(); i++)
        if (s.vars[i].spec.name == name) vi = int(i);
    if (vi < 0) return set_error(YB_EINVAL, "%s: var '%s' not found in solution '%s'", what, name, s.spec.name.c_str());
    const Var& v = s.vars[vi];
    if (!v.has_step()) return set_error(YB_EINVAL, "%s: var '%s' has no step dim '%s'", what, name, s.spec.step_dim.c_str());
    for (auto& d : v.dims)
        if (d.spec.kind == DIM_MISC)
            return set_error(YB_EUNSUPPORTED, "%s: var '%s' has misc dim '%s': vars with misc dims are not supported", what, name, d.spec.name.c_str());
    for (int k = 0; k < s.ndd; k++)
        if (!v.domain_dim(k))
            return set_error(YB_EINVAL, "%s: var '%s' lacks domain dim '%s'", what, name, s.spec.domain_dims[k].c_str());
    bool written = false;
    for (auto& sp : s.spec.stages)
        for (int o : sp.outputs)
            if (o == vi) { written = true; step_off = sp.out_step_off; }
    if (!written) return set_error(YB_EINVAL, "%s: var '%s' is not written by any stage of '%s'", what, name, s.spec.name.c_str());
    return 0;
}

void points_free(PointsState* p) {
    if (!p) return;
    release_device(*p);
    delete p;
}

void points_preload() {
    preload_kernel((const void*)points_kernel<float>);
    preload_kernel((const void*)points_kernel<double>);
    preload_kernel((const void*)weighted_sources_kernel<float>);
    preload_kernel((const void*)weighted_sources_kernel<double>);
    preload_kernel((const void*)weighted_receivers_kernel<float>);
    preload_kernel((const void*)weighted_receivers_kernel<double>);
}

bool points_active(const Solution& s) { return s.points && (s.points->src.set || s.points->rcv.set); }

bool geometry_known(const Solution& s) { return s.prepared || s.geometry_planned; }

bool fused_pair_rank_grid(const Solution& s) {
    if (!geometry_known(s) || !s.multi_rank()) return false;
    // fused-pair rank grids keep the temporal tile's spare slots (Engine::plan_storage); after prepare the engine says so itself
    bool pairs = s.prepared && s.engine->fused_steps(s) > 1;
    for (auto& v : s.vars) pairs = pairs || v.extra_slots > 0;
    return pairs;
}

int points_check_mode(const Solution& s) {
    if (!points_active(s)) return 0;
    if (fused_pair_rank_grid(s))
        return set_error(YB_EUNSUPPORTED, "point sources and receivers are not supported on a rank grid in fused-pair mode (block_steps=2 with "
                                          "mega_block_steps=2): its halos are exchanged once per pair of steps, and the state between the two steps "
                                          "where a source enters is never stored");
    return 0;
}

int points_plan(Solution& s) {
    if (int rc = points_check_mode(s)) return rc;
    PointsState& p = *s.points;
    PointPlan plan;
    // entry e of a set: point e of an on-grid set, support entry e % k of point e / k of a weighted one
    auto locate = [&](const PointSet& ps, bool src, int64_t e, long long& off, long long* loc, bool& own) -> int {
        const Var& v = s.vars[ps.var];
        off = 0; own = true;
        loc[0] = loc[1] = loc[2] = 0;
        for (int k = 0; k < s.ndd; k++) {
            const int64_t g = ps.idx[size_t(e) * s.ndd + k];
            if (g < 0 || g >= s.overall_size[k]) {
                if (ps.k)
                    return set_error(YB_ERANGE, "%s: point %lld entry %lld (weight %g) has index %lld in dim '%s', outside the overall domain "
                                                "[0,%lld) (only entries of weight 0 may lie outside)", set_name(src), (long long)(e / ps.k),
                                     (long long)(e % ps.k), ps.w[size_t(e)], (long long)g, s.spec.domain_dims[k].c_str(), (long long)s.overall_size[k]);
                return set_error(YB_ERANGE, "%s: point %lld has index %lld in dim '%s', outside the overall domain [0,%lld) (halo and pad cells "
                                            "are refused)", set_name(src), (long long)e, (long long)g, s.spec.domain_dims[k].c_str(),
                                 (long long)s.overall_size[k]);
            }
            const int64_t l = g - s.rank_offset[k];
            if (l < 0 || l >= s.rank_size[k]) own = false;
            loc[k] = l;
            const Dim* d = v.domain_dim(k);
            off += (l + d->pad_l) * d->stride;
        }
        return 0;
    };
    if (p.src.set) {
        // on a rank grid the source enters before the exchange of the LAST stage; a var written earlier would already be published
        if (s.multi_rank()) {
            bool last = false;
            for (int o : s.spec.stages.back().outputs) last = last || o == p.src.var;
            if (!last)
                return set_error(YB_EUNSUPPORTED, "sources: on a rank grid the source var '%s' must be written by the last stage of '%s'",
                                 s.vars[p.src.var].spec.name.c_str(), s.spec.name.c_str());
        }
        struct Entry { int col, q; double w; };
        std::map<long long, int> group_of;
        std::vector<std::vector<Entry>> cols;
        const int64_t k = std::max(p.src.k, 1);
        for (int64_t e = 0; e < p.src.n * k; e++) {
            const double w = p.src.k ? p.src.w[size_t(e)] : 1.0;
            if (w == 0) continue;                                   // dropped: it need not lie in the domain
            long long off, loc[3];
            bool own;
            if (int rc = locate(p.src, true, e, off, loc, own)) return rc;
            if (!own) continue;
            auto it = group_of.find(off);
            if (it == group_of.end()) {
                it = group_of.emplace(off, int(cols.size())).first;
                cols.emplace_back();
                plan.grp_off.push_back(off);
                plan.grp_loc.insert(plan.grp_loc.end(), loc, loc + 3);
            }
            cols[it->second].push_back(Entry{int(e / k), int(e % k), w});
        }
        plan.grp_first.push_back(0);
        for (auto& c : cols) {
            for (const Entry& en : c) {
                plan.src_col.push_back(en.col);
                if (p.src.k) { plan.src_q.push_back(en.q); plan.src_w.push_back(en.w); }
            }
            plan.grp_first.push_back(int(plan.src_col.size()));
        }
    }
    if (p.rcv.set) {
        plan.owned.assign(size_t(p.rcv.n), 0);
        if (p.rcv.k) plan.rcv_first.push_back(0);
        for (int64_t j = 0; j < p.rcv.n; j++) {
            long long off, loc[3];
            bool own;
            if (!p.rcv.k) {
                if (int rc = locate(p.rcv, false, j, off, loc, own)) return rc;
                if (!own) continue;
                plan.owned[size_t(j)] = 1;
                plan.rcv_off.push_back(off);
                plan.rcv_loc.insert(plan.rcv_loc.end(), loc, loc + 3);
                plan.rcv_col.push_back(int(j));
                continue;
            }
            // weighted: the owner holds the first nonzero entry; offsets are taken in the owner's rank-local coordinates
            const int64_t k = p.rcv.k;
            int64_t q0 = 0;
            while (p.rcv.w[size_t(j * k + q0)] == 0) q0++;           // set_receivers_weighted refused all-zero points
            for (int64_t q = 0; q < k; q++)
                if (p.rcv.w[size_t(j * k + q)] != 0)
                    if (int rc = locate(p.rcv, false, j * k + q, off, loc, own)) return rc;
            int64_t ri[3] = {0, 0, 0}, roff[3] = {0, 0, 0}, rsize[3] = {1, 1, 1};
            bool mine = true;
            for (int d = 0; d < s.ndd; d++) {
                rank_box_of(s, d, p.rcv.idx[size_t(j * k + q0) * s.ndd + d], ri[d], roff[d], rsize[d]);
                mine = mine && ri[d] == s.rank_index[d];
            }
            if (s.multi_rank())
                if (int rc = check_weighted_receiver(s, p.rcv, j, ri, roff, rsize)) return rc;
            if (!mine) continue;
            plan.owned[size_t(j)] = 1;
            for (int64_t q = 0; q < k; q++) {
                const double w = p.rcv.w[size_t(j * k + q)];
                if (w == 0) continue;
                locate(p.rcv, false, j * k + q, off, loc, own);      // owner-local offset (loc may be negative: a halo cell)
                plan.rcv_off.push_back(off);
                plan.rcv_w.push_back(w);
            }
            plan.rcv_first.push_back(int(plan.rcv_off.size()));
            plan.rcv_col.push_back(int(j));
        }
    }
    p.plan = std::move(plan);
    return 0;
}

int points_begin_run(Solution& s) {
    if (!points_active(s)) return 0;
    if (int rc = points_check_mode(s)) return rc;
    PointsState& p = *s.points;
    p.rcv_pending = false;          // a run that failed midway leaves nothing to record in the next
    if (!p.stale) return 0;
    if (int rc = points_plan(s)) return rc;
    release_device(p);
    const PointPlan& pl = p.plan;
    if (!p.num_sms) YB_CUDA(cudaDeviceGetAttribute(&p.num_sms, cudaDevAttrMultiProcessorCount, s.device));
    if (p.src.set) {
        if (int rc = upload(p, p.d_grp_off, pl.grp_off)) return rc;
        if (int rc = upload(p, p.d_grp_loc, pl.grp_loc)) return rc;
        if (int rc = upload(p, p.d_grp_first, pl.grp_first)) return rc;
        if (int rc = upload(p, p.d_src_col, pl.src_col)) return rc;
        if (int rc = upload(p, p.d_src_w, pl.src_w)) return rc;
        if (int rc = upload(p, p.d_amp, p.src.amp)) return rc;
    }
    if (p.rcv.set) {
        if (int rc = upload(p, p.d_rcv_off, pl.rcv_off)) return rc;
        if (int rc = upload(p, p.d_rcv_loc, pl.rcv_loc)) return rc;
        if (int rc = upload(p, p.d_rcv_col, pl.rcv_col)) return rc;
        if (int rc = upload(p, p.d_rcv_first, pl.rcv_first)) return rc;
        if (int rc = upload(p, p.d_rcv_w, pl.rcv_w)) return rc;
        const size_t bytes = size_t(p.rcv.nrows) * size_t(p.rcv.n) * s.spec.elem_bytes;
        if (bytes) {
            YB_CUDA(cudaMalloc(&p.d_trace, bytes));
            YB_CUDA(cudaMemset(p.d_trace, 0, bytes));
        }
    }
    p.stale = false;
    return 0;
}

static bool in_box(const long long* loc, const Box& b) {
    for (int k = 0; k < 3; k++)
        if (loc[k] < b.b[k] || loc[k] >= b.e[k]) return false;
    return true;
}

// the weighted receiver launch of step t (rows due are checked by the caller)
static int points_record_weighted(Solution& s, int64_t t, cudaStream_t st) {
    PointsState& p = *s.points;
    const PointPlan& pl = p.plan;
    const int64_t u = t + p.rcv.step_off, row = u - p.rcv.t0;
    const Var& v = s.vars[p.rcv.var];
    WeightedRcvArgs a{};
    a.slot = v.slot_ptr(v.slot_of(u));
    a.off = p.d_rcv_off; a.first = p.d_rcv_first; a.col = p.d_rcv_col; a.w = p.d_rcv_w;
    a.trace_row = static_cast<char*>(p.d_trace) + size_t(row) * size_t(p.rcv.n) * s.spec.elem_bytes;
    a.nrcv = int(pl.rcv_col.size());
    const unsigned grid = grid_for(p, pl.rcv_col.size());
    if (s.spec.elem_bytes == 4) weighted_receivers_kernel<float><<<grid, 256, 0, st>>>(a);
    else weighted_receivers_kernel<double><<<grid, 256, 0, st>>>(a);
    YB_CUDA(cudaGetLastError());
    p.launches++;
    return 1;
}

int points_launch(Solution& s, int64_t t, int sel, const Box& interior, cudaStream_t st) {
    if (!points_active(s)) return 0;
    PointsState& p = *s.points;
    const PointPlan& pl = p.plan;
    auto wanted = [&](const long long* loc) { return sel == PTS_ALL || (sel == PTS_INTERIOR) == in_box(loc, interior); };
    PointArgs a{};
    a.sel = sel;
    for (int k = 0; k < 3; k++) { a.ib[k] = interior.b[k]; a.ie[k] = interior.e[k]; }
    int launched = 0;
    // weighted sources first: an on-grid receiver of this launch must see them
    if (p.src.set && p.src.k && !pl.grp_off.empty()) {
        const int64_t u = t + p.src.step_off, row = u - p.src.t0;
        bool any = false;
        for (size_t g = 0; g < pl.grp_off.size() && !any; g++) any = wanted(&pl.grp_loc[3 * g]);
        if (row >= 0 && row < p.src.nrows && any) {
            const Var& v = s.vars[p.src.var];
            WeightedSrcArgs w{};
            w.slot = v.slot_ptr(v.slot_of(u));
            w.grp_off = p.d_grp_off; w.grp_loc = p.d_grp_loc; w.grp_first = p.d_grp_first; w.col = p.d_src_col; w.w = p.d_src_w;
            w.amp_row = p.d_amp + row * p.src.n;
            w.ngrp = int(pl.grp_off.size());
            w.sel = sel;
            for (int k = 0; k < 3; k++) { w.ib[k] = interior.b[k]; w.ie[k] = interior.e[k]; }
            const unsigned grid = grid_for(p, pl.grp_off.size());
            if (s.spec.elem_bytes == 4) weighted_sources_kernel<float><<<grid, 256, 0, st>>>(w);
            else weighted_sources_kernel<double><<<grid, 256, 0, st>>>(w);
            YB_CUDA(cudaGetLastError());
            p.launches++;
            launched++;
        }
    }
    // weighted receivers last; a rank grid records them once the step's last exchange has arrived (points_record_pending)
    auto weighted_receivers = [&]() -> int {
        if (!p.rcv.set || !p.rcv.k || pl.rcv_col.empty()) return 0;
        const int64_t row = t + p.rcv.step_off - p.rcv.t0;
        if (row < 0 || row >= p.rcv.nrows) return 0;
        if (s.halo) {
            p.rcv_pending = true;
            p.pending_t = t;
            return 0;
        }
        return points_record_weighted(s, t, st);
    };
    int nsel = 0;
    if (p.src.set && !p.src.k && !pl.grp_off.empty()) {
        const int64_t u = t + p.src.step_off, row = u - p.src.t0;
        if (row >= 0 && row < p.src.nrows) {
            for (size_t g = 0; g < pl.grp_off.size() && !nsel; g++) nsel += wanted(&pl.grp_loc[3 * g]);
            const Var& v = s.vars[p.src.var];
            a.src_slot = v.slot_ptr(v.slot_of(u));
            a.grp_off = p.d_grp_off; a.grp_loc = p.d_grp_loc; a.grp_first = p.d_grp_first; a.src_col = p.d_src_col;
            a.amp_row = p.d_amp + row * p.src.n;
            a.ngrp = int(pl.grp_off.size());
        }
    }
    int rsel = 0;
    if (p.rcv.set && !p.rcv.k && !pl.rcv_off.empty()) {
        const int64_t u = t + p.rcv.step_off, row = u - p.rcv.t0;
        if (row >= 0 && row < p.rcv.nrows) {
            for (size_t j = 0; j < pl.rcv_off.size() && !rsel; j++) rsel += wanted(&pl.rcv_loc[3 * j]);
            const Var& v = s.vars[p.rcv.var];
            a.rcv_slot = v.slot_ptr(v.slot_of(u));
            a.rcv_off = p.d_rcv_off; a.rcv_loc = p.d_rcv_loc; a.rcv_col = p.d_rcv_col;
            a.trace_row = static_cast<char*>(p.d_trace) + size_t(row) * size_t(p.rcv.n) * s.spec.elem_bytes;
            a.nrcv = int(pl.rcv_off.size());
        }
    }
    if (nsel || rsel) {
        if (s.spec.elem_bytes == 4) points_kernel<float><<<1, 256, 0, st>>>(a);
        else points_kernel<double><<<1, 256, 0, st>>>(a);
        YB_CUDA(cudaGetLastError());
        p.launches++;
        launched++;
    }
    const int rc = weighted_receivers();
    return rc < 0 ? rc : launched + rc;
}

int points_record_pending(Solution& s, cudaStream_t st) {
    if (!points_active(s) || !s.points->rcv_pending) return 0;
    s.points->rcv_pending = false;
    return points_record_weighted(s, s.points->pending_t, st);
}

std::string points_groups_text(const Solution& s) {
    std::string out;
    if (!points_active(s)) return out;
    const PointPlan& pl = s.points->plan;
    for (size_t g = 0; g + 1 < pl.grp_first.size(); g++) {
        if (g) out += ';';
        for (int k = pl.grp_first[g]; k < pl.grp_first[g + 1]; k++) {
            out += (k > pl.grp_first[g] ? "," : "") + std::to_string(pl.src_col[k]);
            if (s.points->src.k) out += "/" + std::to_string(pl.src_q[k]);
        }
    }
    return out;
}

bool points_source_x_range(const Solution& s, int64_t t, int64_t& x0, int64_t& x1) {
    if (!points_active(s) || !s.points->src.set) return false;
    const PointsState& p = *s.points;
    const int64_t row = t + p.src.step_off - p.src.t0;
    if (row < 0 || row >= p.src.nrows || p.plan.grp_off.empty()) return false;
    x0 = x1 = p.plan.grp_loc[0];
    for (size_t g = 1; g < p.plan.grp_off.size(); g++) {
        x0 = std::min<int64_t>(x0, p.plan.grp_loc[3 * g]);
        x1 = std::max<int64_t>(x1, p.plan.grp_loc[3 * g]);
    }
    return true;
}

}  // namespace yb

using namespace yb;

extern "C" {

#define SOL(s) reinterpret_cast<Solution*>(s)

// Replace the set of its kind by `ps` (var, shape and weights already checked).  With the rank geometry known the set is checked
// now (range, ownership, mode); a prepared solution uploads it now too, so that run_solution() enqueues nothing but launches.
static int install_set(Solution* s, bool src, PointSet&& ps) {
    const bool had = s->points != nullptr;
    if (!had) s->points = new PointsState();
    PointSet keep = src ? s->points->src : s->points->rcv;
    (src ? s->points->src : s->points->rcv) = std::move(ps);
    s->points->stale = true;
    if (geometry_known(*s)) {
        if (int rc = points_plan(*s)) {
            (src ? s->points->src : s->points->rcv) = std::move(keep);
            return rc;
        }
    }
    if (s->prepared) {
        YB_CUDA(cudaSetDevice(s->device));
        YB_CUDA(cudaStreamSynchronize(s->stream()));     // the tables being replaced may still be in use
        return points_begin_run(*s);
    }
    return 0;
}

static int set_points(Solution* s, bool src, const char* var, int64_t n, const int64_t* idx, int64_t t0, int64_t nrows, const double* amp) {
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (n < 1) return set_error(YB_EINVAL, "%s: at least one point is needed (clear_points() removes a set)", set_name(src));
    if (!idx) return set_error(YB_EINVAL, "%s: null index array", set_name(src));
    if (nrows < 0) return set_error(YB_EINVAL, "%s: negative row count %lld", set_name(src), (long long)nrows);
    if (src && nrows > 0 && !amp) return set_error(YB_EINVAL, "sources: null amplitude table for %lld rows", (long long)nrows);
    if (n > int64_t(1) << 30) return set_error(YB_EINVAL, "%s: too many points", set_name(src));
    PointSet ps;
    if (int rc = point_var(*s, set_name(src), var, ps.var, ps.step_off)) return rc;
    ps.set = true;
    ps.n = n; ps.t0 = t0; ps.nrows = nrows;
    ps.idx.assign(idx, idx + size_t(n) * s->ndd);
    if (src) ps.amp.assign(amp, amp + size_t(n) * size_t(nrows));
    return install_set(s, src, std::move(ps));
}

static int set_weighted(Solution* s, bool src, const char* var, int64_t n, int64_t k, const int64_t* idx, const double* w, int64_t t0,
                        int64_t nrows, const double* amp) {
    if (!s) return set_error(YB_EINVAL, "null solution");
    const char* what = src ? "weighted sources" : "weighted receivers";
    if (n < 1) return set_error(YB_EINVAL, "%s: at least one point is needed (clear_points() removes a set)", what);
    if (k < 1) return set_error(YB_EINVAL, "%s: k = %lld support entries per point; at least one is needed", what, (long long)k);
    if (!idx) return set_error(YB_EINVAL, "%s: null index table", what);
    if (!w) return set_error(YB_EINVAL, "%s: null weight table", what);
    if (nrows < 0) return set_error(YB_EINVAL, "%s: negative row count %lld", what, (long long)nrows);
    if (src && nrows > 0 && !amp) return set_error(YB_EINVAL, "%s: null amplitude table for %lld rows", what, (long long)nrows);
    if (n > (int64_t(1) << 30) / k) return set_error(YB_EINVAL, "%s: too many support entries (%lld points x %lld)", what, (long long)n, (long long)k);
    for (int64_t i = 0; i < n; i++) {
        bool any = false;
        for (int64_t q = 0; q < k; q++) {
            const double x = w[i * k + q];
            if (!std::isfinite(x)) return set_error(YB_EINVAL, "%s: point %lld entry %lld has a non-finite weight (%g)", what, (long long)i, (long long)q, x);
            any = any || x != 0;
        }
        if (!any) return set_error(YB_EINVAL, "%s: every weight of point %lld is 0", what, (long long)i);
    }
    PointSet ps;
    if (int rc = point_var(*s, what, var, ps.var, ps.step_off)) return rc;
    ps.set = true;
    ps.n = n; ps.k = int(k); ps.t0 = t0; ps.nrows = nrows;
    ps.idx.assign(idx, idx + size_t(n) * size_t(k) * s->ndd);
    ps.w.assign(w, w + size_t(n) * size_t(k));
    if (src) ps.amp.assign(amp, amp + size_t(n) * size_t(nrows));
    return install_set(s, src, std::move(ps));
}

int yb_solution_set_sources_weighted(yb_solution* s, const char* var, int64_t n, int64_t k, const int64_t* idx, const double* w, int64_t t0,
                                     int64_t nrows, const double* amp) {
    return set_weighted(SOL(s), true, var, n, k, idx, w, t0, nrows, amp);
}

int yb_solution_set_receivers_weighted(yb_solution* s, const char* var, int64_t m, int64_t k, const int64_t* idx, const double* w,
                                       int64_t t0r, int64_t nrows_r) {
    return set_weighted(SOL(s), false, var, m, k, idx, w, t0r, nrows_r, nullptr);
}

int yb_points_trilinear(int ndd, int64_t n, const double* pos, int64_t* idx_out, double* w_out) {
    if (ndd < 1 || ndd > 3) return set_error(YB_EINVAL, "trilinear: %d dims; 1, 2 or 3 are supported", ndd);
    if (n < 1) return set_error(YB_EINVAL, "trilinear: at least one position is needed");
    if (!pos || !idx_out || !w_out) return set_error(YB_EINVAL, "trilinear: null array");
    for (int64_t i = 0; i < n * ndd; i++)
        if (!std::isfinite(pos[i]) || std::fabs(pos[i]) >= 0x1p62)
            return set_error(YB_EINVAL, "trilinear: position %lld has a non-finite or out-of-range coordinate in dim %d (%g)", (long long)(i / ndd),
                             int(i % ndd), pos[i]);
    const int k = 1 << ndd;
    for (int64_t i = 0; i < n; i++) {
        int64_t base[3];
        double f[3];
        for (int d = 0; d < ndd; d++) {
            const double fl = std::floor(pos[i * ndd + d]);
            base[d] = int64_t(fl);
            f[d] = pos[i * ndd + d] - fl;
        }
        for (int c = 0; c < k; c++) {
            double wt = 1.0;
            for (int d = 0; d < ndd; d++) {
                const int bit = (c >> (ndd - 1 - d)) & 1;
                idx_out[(i * k + c) * ndd + d] = base[d] + bit;
                wt = wt * (bit ? f[d] : 1.0 - f[d]);
            }
            w_out[i * k + c] = wt;
        }
    }
    return 0;
}

int yb_solution_set_sources(yb_solution* s, const char* var, int64_t n, const int64_t* idx, int64_t t0, int64_t nrows, const double* amp) {
    return set_points(SOL(s), true, var, n, idx, t0, nrows, amp);
}

int yb_solution_set_receivers(yb_solution* s, const char* var, int64_t m, const int64_t* idx, int64_t t0r, int64_t nrows_r) {
    return set_points(SOL(s), false, var, m, idx, t0r, nrows_r, nullptr);
}

int yb_solution_get_traces(yb_solution* s_, void* out, uint8_t* owned) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (!points_active(*s) || !s->points->rcv.set) return set_error(YB_ESTATE, "get_traces: no receivers are set");
    PointsState& p = *s->points;
    if (p.stale) {
        if (!geometry_known(*s)) return set_error(YB_ESTATE, "get_traces: the rank geometry is not known yet (plan_geometry / prepare_solution)");
        if (int rc = points_plan(*s)) return rc;
    }
    if (owned) memcpy(owned, p.plan.owned.data(), p.plan.owned.size());
    if (!out) return 0;
    const size_t bytes = size_t(p.rcv.nrows) * size_t(p.rcv.n) * s->spec.elem_bytes;
    if (p.stale || !p.d_trace) {         // nothing recorded since the last change
        memset(out, 0, bytes);
        return 0;
    }
    YB_CUDA(cudaSetDevice(s->device));
    YB_CUDA(cudaMemcpyAsync(out, p.d_trace, bytes, cudaMemcpyDeviceToHost, s->stream()));
    YB_CUDA(cudaStreamSynchronize(s->stream()));
    return 0;
}

int yb_solution_clear_points(yb_solution* s_) {
    Solution* s = SOL(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (!s->points) return 0;
    if (s->prepared) {
        YB_CUDA(cudaSetDevice(s->device));
        YB_CUDA(cudaStreamSynchronize(s->stream()));
    }
    const int64_t launches = s->points->launches;
    points_free(s->points);
    s->points = new PointsState();
    s->points->launches = launches;
    s->points->stale = false;
    return 0;
}

}  // extern "C"
