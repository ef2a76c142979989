// Slice recorders, slice injectors and slice correlators: boxes of a var recorded from, written into, or correlated with frames
// on the device inside run_solution() (yb_slices.cu).
//
// A recorder names a var, an inclusive box [first, last] of global domain indices with a stride per dim, and a step window:
// step u (the step a run has just computed) is recorded into frame row (u - t0) / every when u - t0 is a multiple of `every` and
// that row is below nrows.  A frame row holds what get_elements_in_slice of the decimated box would read right after the
// run_solution() call that computed u -- after that step's sources and receivers (yb_points.h).  Each rank records and stores
// only its own part of the decimated box.
//
// An injector is the dual: the same box and window, and frames given by the caller.  When row r is due at step u it sets
// (YB_INJECT_SET) or adds to (YB_INJECT_ADD, one add in the element type) var(u) at every point of the decimated box, right after
// the step's stages and before its sources, receivers and recorders.  Injectors run in id order: the list is split into launch
// groups, a new group starting where an injector's box meets an earlier member's on the same var.
//
// A correlator has a recorder's box and window and accumulates var(u) * b into an image of one frame, on the device: b is var(u)
// itself (autocorrelation: the source illumination) or row r, or nrows - 1 - r (reverse), of a recorder's frames.  Correlators
// run after the step's recorders.  Injectors may read a recorder's frames the same way instead of the caller's.  A correlator may
// also read b from a var of another prepared solution on the same device, at the paired step src_t0 + (u - t0) (a var link): the
// source wavefield rebuilt backwards in time beside the adjoint run, so the shot stores no snapshots.
#pragma once
#include <memory>

#include "yb_core.h"

namespace yb {

// A recorder's frames held by a consumer (a correlator, or an injector fed from a recorder): the geometry the attach call checked,
// checked again at the consumer's prepare, and the events that order the two solutions' streams -- none when the source is the
// consumer itself.  Held by the consumer; the source keeps a weak reference (SlicesState::readers).  A var link (src non-null:
// a correlator reading a var of another solution) names the source and its var instead of a recorder; the source's destructor
// clears src (slices_source_gone), after which the consumer refuses to run until its correlators are cleared.
struct FrameLink {
    int device = -1, elem_bytes = 0, ndd = 0;
    int ftype = 0;                              // the recorder's frame type (YB_TYPE_*), which the consumer reads
    int64_t src_id = 0, nrows = 0;
    int64_t first[3] = {0, 0, 0}, last[3] = {0, 0, 0}, stride[3] = {1, 1, 1};
    int64_t overall[3] = {0, 0, 0}, num_ranks[3] = {1, 1, 1}, rank_index[3] = {0, 0, 0};
    int64_t own_k0[3] = {0, 0, 0}, own_n[3] = {0, 0, 0};
    cudaEvent_t written = nullptr;              // recorded by the source after each of its runs
    cudaEvent_t read = nullptr;                 // recorded by the consumer after each of its runs
    // var links only
    bool var_link = false;
    Solution* src = nullptr;                    // null once the source is destroyed
    int src_var = -1;
    int64_t src_shift = 0;                      // source step = consumer step u + src_shift (src_t0 - t0)
    std::string src_name;                       // the source solution's name, for messages after it is gone
    ~FrameLink();
};

struct SliceRec {
    int var = -1;
    int step_off = 1;                           // step the var's writing stage computes, relative to t
    int64_t first[3] = {0, 0, 0}, last[3] = {0, 0, 0}, stride[3] = {1, 1, 1};   // global; missing dims 0, 0, 1
    int64_t t0 = 0, every = 1, nrows = 1;
    int64_t count[3] = {1, 1, 1};               // shape of the decimated box
    // this rank's part (slices_plan): decimated indices own_k0[d] .. own_k0[d] + own_n[d] - 1 of every dim
    int64_t own_k0[3] = {0, 0, 0}, own_n[3] = {0, 0, 0};
    int64_t own_off = 0;                        // element offset of its first point in a step slot of the var
    int64_t own_elems = 0;
    // nrows x own_elems elements of the frame type: a recorder's frames, the frames an injector reads (its own, or a
    // recorder's), a correlator's source frames (null: autocorrelation).  Freed with cudaFree by the last holder.
    std::shared_ptr<void> frames;
    int ftype = 0;                              // YB_TYPE_* of the frames, resolved (a consumer of a recorder: the recorder's)
    // the var's storage and slot_bias as the device table holds them (fuse_vars and the offline tuner's pairs move them)
    const void* uploaded_base = nullptr;
    int uploaded_bias = -1;
    const void* uploaded_src_base = nullptr;    // the same of a var link's source var
    int uploaded_src_bias = -1;
    // injectors only
    int mode = 0;                               // YB_INJECT_ADD / YB_INJECT_SET
    std::vector<char> host_frames;              // the caller's frames (nrows x the whole decimated box) until uploaded
    // consumers of a recorder's frames (injectors fed from a recorder, correlators with a source)
    int rev = 0;                                // row r reads frame row nrows - 1 - r
    std::shared_ptr<FrameLink> link;
    // correlators only
    std::shared_ptr<void> image;                // own_elems elements of the image type, zeroed at allocation
    int itype = 0;                              // YB_TYPE_* of the image, resolved
};

enum SliceKind { SLICE_RECORD, SLICE_INJECT, SLICE_CORRELATE };

struct SlicesState {
    const char* what = "slice";                 // message prefix: "slice", "slice injector" or "slice correlator"
    SliceKind kind = SLICE_RECORD;
    std::vector<SliceRec> recs;
    void* d_table = nullptr;                    // one descriptor per recorder (yb_slices.cu)
    size_t table_cap = 0;                       // descriptors d_table has room for
    int num_sms = 0;                            // of the solution's device, read with the table
    int64_t launches = 0;                       // launches since prepare (read-only options slice_launches, slice_injector_launches)
    std::vector<int> group_first;               // injectors: launch group g is recs[group_first[g] .. group_first[g + 1])
    // recorders: consumers in other solutions of this one's frames or vars (var links), which this one's runs order; the var
    // links outlive clear_slices
    std::vector<std::weak_ptr<FrameLink>> readers;
};

void slices_free(SlicesState* p);
void slices_preload();                          // load the recording, injecting and correlating kernels now (preload_kernel)
bool slices_active(const Solution& s);
bool slice_injectors_active(const Solution& s);
bool slice_correlators_active(const Solution& s);
// validation + this rank's part of every recorder, injector and correlator (host only: needs the rank geometry, no device)
int slices_plan(Solution& s);
// plan, then allocate the frames of every recorder and injector, the images of the correlators, and upload the descriptor tables
// (prepare_solution)
int slices_prepare(Solution& s);
// before a run of steps first_step .. last_step enqueues anything: refuse it if a correlator's var link has lost its source or
// pairs a due step with a source step outside the source var's valid window; then refresh the descriptor tables if a var's
// storage (fuse_vars) or live slots (a temporal tile of the offline tuner) moved since they were uploaded, a var link's source
// var included; never allocates a frame buffer
int slices_begin_run(Solution& s, int64_t first_step, int64_t last_step);
// The source solution s is being destroyed: its var links' consumers lose it (FrameLink::src)
void slices_source_gone(Solution& s);
// Writes of the var-data calls into s's vars (fills, set_elements): before them s's stream waits for the last runs of the
// consumers that read its vars (var links), and after them records the event those consumers' next runs wait on.
int slices_var_write_waits(Solution& s);
int slices_var_write_records(Solution& s);
// Frames shared between two solutions: at the start of a run, before anything else is enqueued, the stream waits for the
// sources' last runs to have written the frames this solution reads, and for its consumers' last runs to have read the frames
// this solution writes; at its end the run records its own events for them.  Never allocates.
int slices_run_waits(Solution& s, cudaStream_t st);
int slices_run_records(Solution& s, cudaStream_t st);
// the recording launch of step t (the step the stage loop just computed from t): returns #kernels launched (0 or 1) or <0
int slices_launch(Solution& s, int64_t t, cudaStream_t st);
// the correlating launch of step t, right after the recording launch: one for every correlator with a row due.  Returns #kernels
// launched (0 or 1) or <0
int slice_correlators_launch(Solution& s, int64_t t, cudaStream_t st);
// the injecting launches of step t, one per launch group with a row due, in id order; sel (PTS_*) picks the points outside or
// inside `interior` (rank-local) on a rank grid's split form.  Returns #kernels launched or <0
int slice_injectors_launch(Solution& s, int64_t t, int sel, const Box& interior, cudaStream_t st);
// rank-local x range [x0, x1] of the points this rank injects at step t; false when it injects none
bool slice_injectors_x_range(const Solution& s, int64_t t, int64_t& x0, int64_t& x1);
// read-only option slice_injector_groups: the launch groups in order separated by ';', each its comma-separated ids ("0,1;2")
std::string slice_injector_groups_text(const Solution& s);

}  // namespace yb
