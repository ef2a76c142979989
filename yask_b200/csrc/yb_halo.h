// Multi-GPU halo exchange over NVLink peer memory (one process per GPU, CUDA IPC).
// Replaces StencilContext::exchange_halos (/root/reference/src/kernel/lib/halo.cpp:80-491).
#pragma once
#include "yb_core.h"

namespace yb {

int halo_prepare(Solution& s);                       // allocate sync flags, neighbour table
void halo_mark_dirty(Solution& s, int var);          // host wrote into a var (dirty protocol, yk_var.cpp:122-152)
int halo_exchange_all(Solution& s, cudaStream_t st); // exchange every dirty var/step, complete in stream order
int halo_run_stage(Solution& s, int stage, int64_t t, cudaStream_t st);  // wait(previous) -> exterior -> push -> interior
int halo_finish(Solution& s, cudaStream_t st);       // enqueue the wait of the exchange still in flight (end of run_solution)
// Does var v need data from the neighbour in direction dir?  (L1-norm pruning + nonzero halo width; host only, no device state.)
bool var_talks_to(const Var& v, const int dir[3]);
// Fused rank-grid mode (Engine::fused_steps > 1 on a rank grid)
int halo_exchange_deep(Solution& s, int64_t t, bool with_inputs, cudaStream_t st);  // p(t) 2R, p(t-1) R [, v R] deep
int halo_run_steps(Solution& s, int64_t t, int nsteps, cudaStream_t st);            // wait(previous) -> fused launch -> deep exchange

}  // namespace yb
