// Slice recorders: boxes of a var recorded on the device inside run_solution() (yb_slices.cu).
//
// A recorder names a var, an inclusive box [first, last] of global domain indices with a stride per dim, and a step window:
// step u (the step a run has just computed) is recorded into frame row (u - t0) / every when u - t0 is a multiple of `every` and
// that row is below nrows.  A frame row holds what get_elements_in_slice of the decimated box would read right after the
// run_solution() call that computed u -- after that step's sources and receivers (yb_points.h).  Each rank records and stores
// only its own part of the decimated box.
#pragma once
#include "yb_core.h"

namespace yb {

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
    void* d_frames = nullptr;                   // nrows x own_elems elements of the solution's type
    // the var's storage and slot_bias as the device table holds them (fuse_vars and the offline tuner's pairs move them)
    const void* uploaded_base = nullptr;
    int uploaded_bias = -1;
};

struct SlicesState {
    std::vector<SliceRec> recs;
    void* d_table = nullptr;                    // one descriptor per recorder (yb_slices.cu)
    size_t table_cap = 0;                       // descriptors d_table has room for
    int num_sms = 0;                            // of the solution's device, read with the table
    int64_t launches = 0;                       // recording launches since prepare (read-only option slice_launches)
};

void slices_free(SlicesState* p);
void slices_preload();                          // load the recording kernel now (preload_kernel)
bool slices_active(const Solution& s);
// validation + this rank's part of every recorder (host only: needs the rank geometry, no device)
int slices_plan(Solution& s);
// plan, then allocate the frames of every recorder and upload the descriptor table (prepare_solution)
int slices_prepare(Solution& s);
// before a run enqueues anything: refresh the descriptor table if a var's storage (fuse_vars) or live slots (a temporal tile
// of the offline tuner) moved since it was uploaded; never allocates a frame buffer
int slices_begin_run(Solution& s);
// the recording launch of step t (the step the stage loop just computed from t): returns #kernels launched (0 or 1) or <0
int slices_launch(Solution& s, int64_t t, cudaStream_t st);

}  // namespace yb
