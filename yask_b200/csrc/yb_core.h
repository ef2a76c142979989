// Internal host-side data model of libyask_b200 (not part of the ABI).
//
// Mirrors, in a device-resident form, the pieces of the reference runtime that sit on the
// run_solution() path:
//   Solution  <- StencilContext + KernelSettings   (/root/reference/src/kernel/lib/context.hpp, settings.hpp:200-328)
//   Var       <- YkVarBase / YkVarBaseCore          (/root/reference/src/kernel/lib/yk_var.hpp:88-149, yk_var.cpp:206-384)
//   StencilSpec <- the generated context ctor       (emitter: /root/reference/src/compiler/lib/YaskKernel.cpp:730-)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/yask_b200.h"

namespace yb {

enum DimKind { DIM_STEP = 0, DIM_DOMAIN = 1, DIM_MISC = 2 };

// ---- compile-time description of a solution (what the reference's generated ctor encodes) ----
struct DimSpec {
    std::string name;
    int kind = DIM_DOMAIN;
    int domain_index = -1;           // 0..2 for domain dims
    int64_t halo_l = 0, halo_r = 0;  // domain dims
    int64_t misc_first = 0, misc_size = 1;
};

struct VarSpec {
    std::string name;
    std::vector<DimSpec> dims;  // declared order; step dim (if any) first
    int step_alloc = 1;         // alloc_t
    bool is_output = false;
    bool user_var = false;      // created through yb_var_create (not touched by kernels)
    bool fixed_size = false;    // user var with explicit sizes (not tied to the rank domain)
    std::vector<int64_t> fixed_sizes;
    int l1_norm = 0;            // max L1 distance of any read -> which neighbours need halos
};

struct StageSpec {
    std::string name;
    std::vector<int> outputs;  // var indices written (at t + out_step_off)
    int out_step_off = 1;      // +1; -1 for reverse-time solutions (equations defined at t-1)
    std::vector<int> inputs;   // var indices read
    int64_t fp_ops = 0, reads = 0, writes = 0;  // per point, as counted by the reference compiler
};

struct StencilSpec {
    std::string name, description;
    std::string step_dim = "t";
    std::vector<std::string> domain_dims;  // e.g. x,y,z  (last = unit stride)
    std::vector<VarSpec> vars;
    std::vector<StageSpec> stages;
    int radius = 0;
    int elem_bytes = 4;
    int64_t uniform_pad[YB_MAX_DOMAIN_DIMS] = {0, 0, 0};  // pad every var at least this much (shared geometry)
};

// ---- run-time geometry -------------------------------------------------------------------------
struct Dim {
    DimSpec spec;
    int64_t rank_offset = 0;
    int64_t domain = 1;       // rank-domain size, alloc_t or misc extent
    int64_t min_pad_l = 0, min_pad_r = 0;
    int64_t pad_l = 0, pad_r = 0;
    int64_t alloc = 1;
    int64_t stride = 0;       // elements
};

struct Var {
    VarSpec spec;
    std::vector<Dim> dims;
    int elem_bytes = 4;
    int64_t slot_elems = 0;
    int64_t first_valid_step = 0;  // local offset of the step dim
    void* dev = nullptr;           // nslots() * slot_elems elements
    // Solution vars own their storage through `store` (cudaFree on the last release): yk_var::fuse_vars makes two vars --
    // possibly of two solutions -- share one allocation (/root/reference/src/kernel/lib/yk_var_apis.cpp:334-360).
    std::shared_ptr<void> store;
    // Spare storage slots beyond the `step_alloc` steps the API can see.  A temporal tile writes steps t+1 and t+2 while
    // overlapping tiles still read the halo cells of t-1 and t, so it cannot update in place: the engine asks for a second
    // set of `step_alloc` slots (yb_iso3dfd.cu) and the fused launch ping-pongs between the two sets (`slot_bias` = first
    // slot of the live set).  Everything else -- the API's valid-step window, the wrap of step indices onto `step_alloc`
    // slots, in-place one-step launches -- sees exactly the reference's storage.
    int extra_slots = 0;
    int slot_bias = 0;
    bool has_step() const { return !dims.empty() && dims[0].spec.kind == DIM_STEP; }
    int step_alloc() const { return has_step() ? spec.step_alloc : 1; }
    int nslots() const { return has_step() ? spec.step_alloc + extra_slots : 1; }
    int64_t last_valid_step() const { return first_valid_step + step_alloc() - 1; }
    size_t bytes() const { return size_t(slot_elems) * nslots() * elem_bytes; }
    // storage slot of a step index: imod_flr(t, alloc_t) (/root/reference/src/kernel/lib/yk_var.hpp:131-147)
    int slot_of(int64_t t) const {
        int a = step_alloc();
        int64_t c = t % a;
        return int(c < 0 ? c + a : c) + slot_bias;
    }
    char* slot_ptr(int slot) const { return static_cast<char*>(dev) + size_t(slot) * slot_elems * elem_bytes; }
    // element offset (within a slot) of the var's domain origin / first misc index
    int64_t origin_offset() const {
        int64_t o = 0;
        for (auto& d : dims)
            if (d.spec.kind == DIM_DOMAIN) o += d.pad_l * d.stride;
        return o;
    }
    const Dim* domain_dim(int domain_index) const {
        for (auto& d : dims)
            if (d.spec.kind == DIM_DOMAIN && d.spec.domain_index == domain_index) return &d;
        return nullptr;
    }
    // update_valid_step (/root/reference/src/kernel/lib/yk_var.cpp:559-575)
    void update_valid_step(int64_t t) {
        if (!has_step()) return;
        if (t < first_valid_step) first_valid_step = t;
        else if (t > last_valid_step()) first_valid_step = t - step_alloc() + 1;
    }
};

// Box of rank-local domain coordinates [begin, end) per domain dim.
struct Box {
    int64_t b[YB_MAX_DOMAIN_DIMS] = {0, 0, 0};
    int64_t e[YB_MAX_DOMAIN_DIMS] = {1, 1, 1};
    bool empty() const { return b[0] >= e[0] || b[1] >= e[1] || b[2] >= e[2]; }
    int64_t points() const { return empty() ? 0 : (e[0] - b[0]) * (e[1] - b[1]) * (e[2] - b[2]); }
};

struct Solution;

// One implementation per stencil family: owns kernels, tensor maps and launch logic.
struct Engine {
    virtual ~Engine() {}
    // called by plan_geometry() and by prepare() once the rank geometry is known and before the vars' geometry is: storage that
    // depends on the rank grid (spare slots, pads).  Default: nothing.
    virtual void plan_storage(Solution&) {}
    // called by plan_geometry() and by prepare() once the vars' geometry is known and before any storage is allocated:
    // refuse a size the engine's kernels cannot address.  Default: no limit.
    virtual int check_geometry(const Solution&) const { return 0; }
    // called at the end of prepare(): build tensor maps etc.
    virtual int prepare(Solution& s) = 0;
    // launch stage `stage` of step t (computing t+1) over `box` on `stream`; returns #kernels launched or <0
    virtual int launch(Solution& s, int stage, int64_t t, const Box& box, cudaStream_t stream) = 0;
    virtual int set_option(Solution&, const std::string&, const std::string&) { return YB_EINVAL; }
    // Offline auto-tuner (yk_solution::run_auto_tuner_now): time the engine's launch variants over the rank box on
    // `stream`, keep the fastest, describe the trials in `report`.  Var contents are not preserved.  Default: nothing to tune.
    virtual int auto_tune(Solution&, cudaStream_t, std::string& report) { report = "nothing to tune"; return 0; }
    virtual bool get_option(const Solution&, const std::string&, std::string&) const { return false; }
    // In-run auto-tuner (yk_solution::reset_auto_tuner / -auto_tune): the launch variants the run loop may cycle through
    // while it executes REAL steps -- every variant computes identical bits, so tuning on live data is safe.
    virtual int tune_variants(const Solution&) const { return 0; }
    virtual void tune_select(Solution&, int /*variant*/) {}
    virtual std::string tune_describe(const Solution&, int /*variant*/) const { return ""; }
    // May stage `stage` be evaluated as several sub-box launches (exterior slabs first, interior last)?  False when the
    // result of a launch depends on what an earlier launch of the same stage wrote (scratch vars computed from vars the
    // stage updates in place).
    virtual bool can_split(const Solution&, int /*stage*/) const { return true; }
    // Temporal tiling (the reference's block steps, "-bt"; /root/reference/src/kernel/lib/context.cpp:657-681): how many
    // consecutive steps one launch_steps() call may fuse for a forward run over the whole rank box (1 = no temporal tile).
    // On a rank grid the answer is fixed at prepare, and halos are then exchanged once per fused launch (halo_run_steps):
    // every rank of the grid must give the same one (yb_halo_import checks).
    virtual int fused_steps(const Solution&) const { return 1; }
    // called once per run_solution() before the first step (first_step = t of the first launch)
    virtual int begin_run(Solution&, int64_t /*first_step*/, cudaStream_t) { return 0; }
    // all stages of steps t+1 .. t+nsteps in one go; returns #kernels launched or <0.  ends_run: step t+nsteps is the last of the
    // run_solution() call, so every step of the API's window must be stored; otherwise an engine may skip storing a step that no
    // later launch reads (the average-of-points tile keeps A(t+1) in shared memory).
    virtual int launch_steps(Solution&, int64_t /*t*/, int /*nsteps*/, bool /*ends_run*/, const Box&, cudaStream_t) { return YB_EUNSUPPORTED; }
};

struct HaloState;  // yb_halo.cu
void halo_free(HaloState*);
struct PointsState;  // yb_points.cu
void points_free(PointsState*);
struct SlicesState;  // yb_slices.cu
void slices_free(SlicesState*);

struct Solution {
    StencilSpec spec;
    std::unique_ptr<Engine> engine;
    int ndd = 3;  // number of domain dims
    // requested settings (0 = unset), reference: KernelSettings::_rank_sizes/_global_sizes/_num_ranks/_rank_indices
    int64_t req_rank_size[YB_MAX_DOMAIN_DIMS] = {0, 0, 0};
    int64_t req_overall_size[YB_MAX_DOMAIN_DIMS] = {0, 0, 0};
    int64_t num_ranks[YB_MAX_DOMAIN_DIMS] = {1, 1, 1};
    int64_t rank_index[YB_MAX_DOMAIN_DIMS] = {0, 0, 0};
    int64_t min_pad[YB_MAX_DOMAIN_DIMS] = {0, 0, 0};
    // actual (after prepare)
    int64_t rank_size[YB_MAX_DOMAIN_DIMS] = {0, 0, 0};
    int64_t overall_size[YB_MAX_DOMAIN_DIMS] = {0, 0, 0};
    int64_t rank_offset[YB_MAX_DOMAIN_DIMS] = {0, 0, 0};
    std::vector<Var> vars;
    std::map<std::string, std::string> options;
    int fp_mode = YB_FP_REF_GCC;
    bool geometry_planned = false;   // plan_geometry() has derived the rank geometry (prepare() does too)
    bool prepared = false;
    int device = -1;
    cudaStream_t own_stream = nullptr, user_stream = nullptr, comm_stream = nullptr;
    bool use_user_stream = false;
    cudaStream_t stream() const { return use_user_stream ? user_stream : own_stream; }
    // in-run auto-tuner: steps cycle through the engine's variants (reps timed steps each), the fastest is kept
    struct InRunTuner {
        bool enabled = false;
        int next = 0, reps = 2;
        std::vector<double> ms;        // best time seen per variant
        std::vector<int> tries;
        std::string report;
    } tuner;
    // stats
    yb_stats stats{};
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending_events;  // per run() call
    // staging buffer for slice copies
    void* stage_dev = nullptr;
    size_t stage_bytes = 0;
    void* stage_host = nullptr;  // pinned
    size_t stage_host_bytes = 0;
    // multi-GPU
    HaloState* halo = nullptr;   // owned; freed by halo_free()
    // point sources and receivers (yb_points.h)
    PointsState* points = nullptr;   // owned; freed by points_free()
    // slice recorders (yb_slices.h)
    SlicesState* slices = nullptr;   // owned; freed by slices_free()
    // slice injectors (yb_slices.h)
    SlicesState* injectors = nullptr;   // owned; freed by slices_free()
    // slice correlators (yb_slices.h)
    SlicesState* correlators = nullptr;   // owned; freed by slices_free()
    // Fused halo stores (set by the halo layer before a stage launch, consumed by an engine that can store its
    // boundary planes straight into the x neighbours' halo cells): element (0,0,0)-relative base pointers of the
    // OUTPUT var's step slot in the lower / upper x neighbour, or null.  The engine sets `used` if it honoured them.
    // In-kernel completion signal: when `counter` is set the engine may ALSO publish `epoch` into the x neighbours'
    // flag words itself, as soon as its boundary planes are stored (it then sets `signalled`), so that the exchange
    // overlaps the interior of the same launch.
    struct FusedX {
        void* lo = nullptr; void* hi = nullptr; int var = -1; bool used = false;
        unsigned long long* flag_lo = nullptr; unsigned long long* flag_hi = nullptr;
        unsigned long long epoch = 0; unsigned int* counter = nullptr; bool signalled = false;
        // dma: the engine only ORDERS its work (boundary planes first) and publishes `epoch` into flag_lo -- a word in LOCAL
        // memory -- when they are stored; the halo layer's side stream waits on that word and moves the planes with the copy
        // engines (yb_halo.cu).  lo / hi then merely say on which sides there is a neighbour.
        bool dma = false;
    } fused_x;
    int multi_rank() const { return int(num_ranks[0] * num_ranks[1] * num_ranks[2]) > 1; }
    ~Solution();
};

// storage geometry of one var from the solution's rank geometry (yb_core.cu)
void compute_var_geometry(Solution& s, Var& v);

// Times `reps` calls of fn() on `st` with CUDA events after one untimed call; returns ms per call (<0 on error).
template <class F>
inline double time_launches(cudaStream_t st, int reps, F fn) {
    cudaEvent_t e0, e1;
    if (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess) return -1;
    double ms = -1;
    if (fn() >= 0) {
        cudaEventRecord(e0, st);
        bool ok = true;
        for (int i = 0; i < reps && ok; i++) ok = fn() >= 0;
        cudaEventRecord(e1, st);
        float f = 0;
        if (ok && cudaEventSynchronize(e1) == cudaSuccess && cudaEventElapsedTime(&f, e0, e1) == cudaSuccess) ms = double(f) / reps;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return ms;
}

// Force the (lazily loaded) kernel `fn` into the context now.  CUDA loads a kernel at its first launch, and that load may
// need the context to go idle; a first launch issued while a halo wait kernel is spinning on a peer whose work the same
// host thread has not enqueued yet (several ranks driven from ONE process, as the in-process rank-grid tests do) would
// then never return.  Every kernel the run loop can launch is therefore touched once in prepare().
inline void preload_kernel(const void* fn) {
    if (!fn) return;
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, fn) != cudaSuccess) (void)cudaGetLastError();
}

// error plumbing
int set_error(int code, const char* fmt, ...);
#define YB_CUDA(call)                                                                              \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
            return yb::set_error(YB_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

// registry (yb_stencils.cpp)
int registry_size();
const char* registry_name(int i);
// builds spec + engine; returns 0 or error
int registry_create(const std::string& name, int radius, int elem_bytes, StencilSpec& spec, std::unique_ptr<Engine>& eng);

// CUtensorMap (passed as void* to keep <cuda.h> out of this header) over one step slot of a full-rank 3-D var,
// box (box_z, box_y, 1) -- yb_iso3dfd.cu
int make_var_tensor_map(void* map, const Var& v, int slot, int box_z, int box_y);

// Temporal tiles (Var::extra_slots == 2): copy the halo cells of the live pair of slots of `v` into the spare pair, so that the
// pair a fused launch writes holds the halo cells the reference's two slots would -- yb_iso3dfd.cu.  The copy kernel is loaded by
// preload_halo_shell_copy().
int copy_halo_shells(const Var& v, int num_sms, cudaStream_t st);
void preload_halo_shell_copy(int elem_bytes);

// engines
std::unique_ptr<Engine> make_iso3dfd_engine();
StencilSpec iso3dfd_spec(int radius, int elem_bytes, bool sponge);
// 3axis, 3axis_with_diags, 3plane, cube (yb_avepts.cu): shape index 0..3 of a solution name (-1: none of them), points read
std::unique_ptr<Engine> make_avepts_engine();
int avepts_shape(const std::string& name);
int64_t avepts_points(int shape, int radius);
StencilSpec avepts_spec(int shape, int radius, int elem_bytes);

// device utilities (yb_fill.cu)
struct BoxCopy {
    int nd;                       // number of non-step dims (<= 4)
    int64_t n[4];                 // box extents
    int64_t var_stride[4];        // element strides in var storage
    int64_t var_off;              // element offset of the box origin in the slot
};
struct RedVals { double sum, sumsq, prod, mx, mn; };
int reduce_scratch_entries();
int launch_box_reduce(const void* var_slot, const BoxCopy& bc, int elem_bytes, RedVals* partial, cudaStream_t st);
int launch_box_copy(void* var_slot, void* dense, const BoxCopy& bc, int elem_bytes, bool to_var, cudaStream_t st);
int launch_box_fill(void* var_slot, const BoxCopy& bc, int elem_bytes, double value, cudaStream_t st);
int launch_fill_all(void* ptr, int64_t n, int elem_bytes, double value, cudaStream_t st);
// hash fill over a box whose first element has global index g0[] (3 entries, missing dims = 0)
int launch_hash_fill(void* var_slot, const BoxCopy& bc, const int64_t* g0, int elem_bytes, uint32_t seed, uint32_t salt,
                     double lo, double hi, cudaStream_t st);
int launch_checksum(const void* var_slot, const BoxCopy& bc, const int64_t* g0, int elem_bytes, unsigned long long* dev_out,
                    cudaStream_t st);

}  // namespace yb
