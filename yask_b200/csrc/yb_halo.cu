// Multi-GPU halo exchange over NVLink peer memory, one process per GPU.
//
// Replaces StencilContext::exchange_halos and the MPI buffer machinery
// (/root/reference/src/kernel/lib/halo.cpp:80-491, alloc.cpp:456-1031, setup.cpp:169-524):
//   * neighbour discovery: the 3^N - 1 neighbourhood of the rank grid, pruned per var by its
//     halo-exchange L1 norm (alloc.cpp:502-522) -- iso3dfd (norm 1) talks to faces only;
//   * no pack/unpack buffers and no MPI: every rank maps its neighbours' var storage with CUDA IPC
//     (the analogue of the reference's MPI-3 shared-memory windows, alloc.cpp:214-249) and a push
//     kernel writes the sender's boundary slab straight into the receiver's halo cells;
//   * completion is a monotonically increasing epoch written into the receiver's flag word with
//     system-scope release semantics; the receiver's stream runs a one-thread wait kernel before the
//     next stage reads its halos (replaces MPI_Wait / the SimpleLock spin of settings.hpp:436-500).
//
// Geometry (alloc.cpp:693-751): to the neighbour in direction d, per dim k
//     d_k = -1 : send my FIRST  halo_r planes -> its right halo   [n_peer, n_peer + halo_r)
//     d_k = +1 : send my LAST   halo_l planes -> its left halo    [-halo_l, 0)
//     d_k =  0 : the whole domain extent in that dim.
#include <stdio.h>
#include <string.h>
#include <unistd.h>

#include <algorithm>

#include <cuda.h>

#include "yb_halo.h"
#include "yb_points.h"
#include "yb_slices.h"

namespace yb {

namespace {

constexpr uint32_t BLOB_MAGIC = 0x59423230;  // "YB20"
constexpr int MAX_VARS = 128;    // vars of one solution a blob describes (fsg_abc declares 70)
constexpr int NDIRS = 27;

struct BlobVar {
    cudaIpcMemHandle_t handle;
    uint64_t raw_ptr;     // valid only inside the exporting process
    int64_t bytes;
    int64_t slot_elems;
    // geometry of the non-step dims (declared order): the receiver's strides/pads may differ from the
    // sender's when the last rank of a dim has a smaller domain
    int32_t nd;
    int64_t pad_l[4], stride[4], domain[4];
};

struct Blob {
    uint32_t magic, version;
    int64_t pid;
    uint64_t nonce;       // identifies the exporting PROCESS (pids repeat across pid namespaces that share an IPC namespace)
    int32_t device;
    int32_t num_vars;
    int64_t rank_index[3];
    int64_t rank_size[3];
    cudaIpcMemHandle_t flags_handle;
    uint64_t flags_raw;
    int32_t fused_steps;  // steps per halo exchange (Engine::fused_steps): neighbours must agree, or they would wait for each other's epochs
    BlobVar vars[MAX_VARS];
};

// One random word per process, drawn at first use: raw device pointers of a blob are honoured only when the blob was
// exported by this very process (same nonce); everything else goes through the IPC handles.
uint64_t process_nonce() {
    static uint64_t n = 0;
    if (!n) {
        FILE* f = fopen("/dev/urandom", "rb");
        if (f) { if (fread(&n, sizeof n, 1, f) != 1) n = 0; fclose(f); }
        if (!n) n = (uint64_t(getpid()) << 32) ^ uint64_t(reinterpret_cast<uintptr_t>(&n)) ^ 0x9e3779b97f4a7c15ull;
    }
    return n;
}

inline int dir_index(const int d[3]) { return (d[0] + 1) * 9 + (d[1] + 1) * 3 + (d[2] + 1); }

struct CopyBox {        // strided box, up to 3 dims, z (last) unit stride
    long long n[3];
    long long src_stride[3];
    long long dst_stride[3];
    long long src_off, dst_off;
};

// One thread per element (or per float4 when everything is 16-B aligned).
template <typename T>
__global__ void halo_push_kernel(const T* __restrict__ src, T* __restrict__ dst, CopyBox b, int vec) {
    const long long nz = b.n[2] / vec;
    const long long total = b.n[0] * b.n[1] * nz;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long z = (i % nz) * vec;
        const long long r = i / nz;
        const long long y = r % b.n[1];
        const long long x = r / b.n[1];
        const long long so = b.src_off + x * b.src_stride[0] + y * b.src_stride[1] + z;
        const long long dof = b.dst_off + x * b.dst_stride[0] + y * b.dst_stride[1] + z;
        if (vec == 4 && sizeof(T) == 4) {
            *reinterpret_cast<float4*>(dst + dof) = *reinterpret_cast<const float4*>(src + so);
        } else if (vec == 2 && sizeof(T) == 8) {
            *reinterpret_cast<double2*>(dst + dof) = *reinterpret_cast<const double2*>(src + so);
        } else {
            dst[dof] = src[so];
        }
    }
}

__global__ void halo_signal_kernel(unsigned long long* peer_flag, unsigned long long epoch) {
    __threadfence_system();  // all earlier peer writes of this stream are ordered before the flag
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(peer_flag), "l"(epoch) : "memory");
}

__global__ void halo_wait_kernel(const unsigned long long* flags, unsigned int dir_mask, unsigned long long epoch) {
    for (int d = 0; d < NDIRS; d++) {
        if (!((dir_mask >> d) & 1u)) continue;
        unsigned long long v;
        unsigned long long spins = 0;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flags + d) : "memory");
            if (v < epoch) {
                __nanosleep(500);
                // a peer that never signals (crashed rank, mis-wired launcher) must not hang the GPU:
                // give up after ~60 s and abort the context with an error instead.
                if (++spins > 120000000ull) { printf("yask_b200: halo wait timed out (dir %d, epoch %llu, seen %llu)\n", d, epoch, v); __trap(); }
            }
        } while (v < epoch);
    }
}

// cuStreamWaitValue64 (stream memory operation): lets the side stream wait for a word the sweep kernel writes while it is
// still running.  Fetched from the driver at run time, like cuTensorMapEncodeTiled.
typedef CUresult (*StreamWaitValue64Fn)(CUstream, CUdeviceptr, cuuint64_t, unsigned int);
StreamWaitValue64Fn stream_wait_value64() {
    static StreamWaitValue64Fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuStreamWaitValue64", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<StreamWaitValue64Fn>(p);
        (void)cudaGetLastError();
    }
    return fn;
}

struct Neighbor {
    int dir[3];
    int64_t peer_linear = -1;
    bool connected = false;
    bool same_process = false;
    std::vector<char*> var_base;            // mapped peer storage per var
    std::vector<BlobVar> var_geom;          // peer geometry per var
    unsigned long long* peer_flags = nullptr;
    std::vector<void*> opened;              // handles to close
};

}  // namespace

struct HaloState {
    std::vector<Neighbor> nbrs;             // existing neighbours in the rank grid
    unsigned long long* flags = nullptr;    // my 27 epoch words (device)
    unsigned long long epoch = 0;           // exchanges completed so far
    std::vector<std::vector<char>> dirty;   // [var][slot]
    bool finalized = false;
    int device = -1;
    bool wait_pending = false;              // the neighbours' epoch `epoch` has not been waited for yet
    unsigned int wait_mask = 0;
    unsigned int* sig_counter = nullptr;    // device word: arrivals of the in-kernel boundary signal (yb_iso3dfd.cuh)
    unsigned long long* local_done = nullptr;   // device word: epoch whose boundary planes are stored (copy-engine path)
    cudaEvent_t comm_ev = nullptr;          // last work enqueued on the side stream
    cudaEvent_t ext_ev = nullptr;           // exterior launches of the current stage (the side stream's pushes follow it)
    bool comm_pending = false;
};

void halo_free(HaloState* h) {
    if (!h) return;
    for (auto& nb : h->nbrs)
        if (!nb.same_process)
            for (void* p : nb.opened) cudaIpcCloseMemHandle(p);
    if (h->flags) cudaFree(h->flags);
    if (h->sig_counter) cudaFree(h->sig_counter);
    if (h->comm_ev) cudaEventDestroy(h->comm_ev);
    if (h->ext_ev) cudaEventDestroy(h->ext_ev);
    delete h;
}

static int64_t linear_rank(const Solution& s, const int64_t idx[3]) {
    return (idx[0] * s.num_ranks[1] + idx[1]) * s.num_ranks[2] + idx[2];
}

int halo_prepare(Solution& s) {
    if (int(s.vars.size()) > MAX_VARS) return set_error(YB_EUNSUPPORTED, "more than %d vars", MAX_VARS);
    auto* h = new HaloState();
    s.halo = h;
    h->device = s.device;
    preload_kernel((const void*)halo_push_kernel<float>);
    preload_kernel((const void*)halo_push_kernel<double>);
    preload_kernel((const void*)halo_signal_kernel);
    preload_kernel((const void*)halo_wait_kernel);
    YB_CUDA(cudaMalloc(&h->flags, NDIRS * sizeof(unsigned long long)));
    YB_CUDA(cudaMemset(h->flags, 0, NDIRS * sizeof(unsigned long long)));
    YB_CUDA(cudaMalloc(&h->sig_counter, 256));
    YB_CUDA(cudaMemset(h->sig_counter, 0, 256));
    h->local_done = reinterpret_cast<unsigned long long*>(h->sig_counter) + 8;      // same allocation, its own 64-byte line
    YB_CUDA(cudaEventCreateWithFlags(&h->comm_ev, cudaEventDisableTiming));
    YB_CUDA(cudaEventCreateWithFlags(&h->ext_ev, cudaEventDisableTiming));
    h->dirty.resize(s.vars.size());
    for (size_t i = 0; i < s.vars.size(); i++) h->dirty[i].assign(s.vars[i].nslots(), 1);  // everything starts dirty (context.hpp:545-549)
    int d[3];
    for (d[0] = -1; d[0] <= 1; d[0]++)
        for (d[1] = -1; d[1] <= 1; d[1]++)
            for (d[2] = -1; d[2] <= 1; d[2]++) {
                if (!d[0] && !d[1] && !d[2]) continue;
                int64_t idx[3];
                bool ok = true;
                for (int k = 0; k < 3; k++) {
                    idx[k] = s.rank_index[k] + d[k];
                    if (idx[k] < 0 || idx[k] >= s.num_ranks[k]) ok = false;
                }
                if (!ok) continue;
                Neighbor nb;
                memcpy(nb.dir, d, sizeof d);
                nb.peer_linear = linear_rank(s, idx);
                nb.var_base.assign(s.vars.size(), nullptr);
                nb.var_geom.resize(s.vars.size());
                h->nbrs.push_back(nb);
            }
    return 0;
}

void halo_mark_dirty(Solution& s, int var) {
    if (!s.halo) return;
    for (auto& f : s.halo->dirty[var]) f = 1;
}

// Does var v need data from the neighbour in direction dir?  (L1-norm pruning + nonzero halo width.)
bool var_talks_to(const Var& v, const int dir[3]) {
    int l1 = abs(dir[0]) + abs(dir[1]) + abs(dir[2]);
    if (l1 > v.spec.l1_norm) return false;
    for (int k = 0; k < 3; k++) {
        if (!dir[k]) continue;
        const Dim* d = v.domain_dim(k);
        if (!d) return false;   // var does not span this dim: nothing to exchange that way
        // sending towards -1 fills the peer's RIGHT halo, towards +1 its LEFT halo
        if ((dir[k] < 0 ? d->spec.halo_r : d->spec.halo_l) == 0) return false;
    }
    return true;
}

// `depth` > 0: that many planes past the interface instead of the var's halo (fused rank-grid mode, halo_exchange_deep)
static int push_var_slot(Solution& s, const Neighbor& nb, int vi, int slot, cudaStream_t st, int64_t depth = 0) {
    const Var& v = s.vars[vi];
    const BlobVar& pg = nb.var_geom[vi];
    int k4 = 0;
    long long n4[4] = {1, 1, 1, 1}, ss[4] = {0, 0, 0, 0}, ds[4] = {0, 0, 0, 0};
    long long so = 0, dof = 0;
    for (auto& d : v.dims) {
        if (d.spec.kind == DIM_STEP) continue;
        if (k4 >= 4) return set_error(YB_EUNSUPPORTED, "halo exchange of vars with more than 4 non-step dims");
        long long first_src, count, first_dst;  // in rank-local domain coordinates of sender / receiver
        if (d.spec.kind == DIM_MISC) { first_src = 0; count = d.domain; first_dst = 0; }
        else {
            const int dk = nb.dir[d.spec.domain_index];
            if (dk < 0) { count = depth > 0 ? depth : d.spec.halo_r; first_src = 0; first_dst = pg.domain[k4]; }
            else if (dk > 0) { count = depth > 0 ? depth : d.spec.halo_l; first_src = d.domain - count; first_dst = -count; }
            else { count = d.domain; first_src = 0; first_dst = 0; }
            if (count > d.domain) return set_error(YB_EUNSUPPORTED, "rank domain smaller than halo in dim '%s'", d.spec.name.c_str());
            if (dk == 0 && pg.domain[k4] != d.domain) return set_error(YB_EINVAL, "neighbour has a different size in an unsplit dim");
        }
        const long long pad = d.spec.kind == DIM_MISC ? 0 : d.pad_l;
        n4[k4] = count; ss[k4] = d.stride; ds[k4] = pg.stride[k4];
        so += (first_src + pad) * d.stride;
        dof += (first_dst + pg.pad_l[k4]) * pg.stride[k4];
        k4++;
    }
    // Sort the dims by descending source stride so the innermost (unit-stride) dim is last; a 4th (outermost) dim,
    // i.e. a misc dim, is looped over on the host.
    int order[4] = {0, 1, 2, 3};
    std::sort(order, order + k4, [&](int a, int b) { return ss[a] > ss[b]; });
    const int outer = k4 > 3 ? order[0] : -1;
    const long long n_outer = outer >= 0 ? n4[outer] : 1;
    int launched = 0;
    for (long long io = 0; io < n_outer; io++) {
        CopyBox b{};
        for (int i = 0; i < 3; i++) { b.n[i] = 1; b.src_stride[i] = b.dst_stride[i] = 0; }
        const int first = outer >= 0 ? 1 : 0;
        const int nin = k4 - first;
        for (int i = 0; i < nin; i++) {
            const int d = order[first + i];
            b.n[3 - nin + i] = n4[d]; b.src_stride[3 - nin + i] = ss[d]; b.dst_stride[3 - nin + i] = ds[d];
        }
        b.src_off = so + (outer >= 0 ? io * ss[outer] : 0);
        b.dst_off = dof + (outer >= 0 ? io * ds[outer] : 0);
        const long long total = b.n[0] * b.n[1] * b.n[2];
        if (total == 0) return 0;
        if (b.src_stride[2] > 1 || b.dst_stride[2] > 1) return set_error(YB_EUNSUPPORTED, "halo push needs a unit-stride innermost dim");
        const char* src = v.slot_ptr(slot);
        char* dst = nb.var_base[vi] + size_t(slot) * pg.slot_elems * v.elem_bytes;
        int vec = 1;
        const int vw = 16 / v.elem_bytes;
        bool al = (b.n[2] % vw == 0) && (b.src_off % vw == 0) && (b.dst_off % vw == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0) &&
                  ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) && b.src_stride[2] == 1 && b.dst_stride[2] == 1;
        for (int i = 0; i < 2; i++) al = al && (b.src_stride[i] % vw == 0) && (b.dst_stride[i] % vw == 0);
        if (al) vec = vw;
        const long long work = total / vec;
        const int grid = int(std::min<long long>((work + 255) / 256, 1184));      // grid-stride copy: the cap bounds the launch, not the result
        if (v.elem_bytes == 4) halo_push_kernel<float><<<grid, 256, 0, st>>>((const float*)src, (float*)dst, b, vec);
        else halo_push_kernel<double><<<grid, 256, 0, st>>>((const double*)src, (double*)dst, b, vec);
        YB_CUDA(cudaGetLastError());
        launched++;
    }
    return launched;
}

// Enqueue the wait for the exchange that is still in flight (if any): the neighbours' epoch `h->epoch` must have
// arrived before (a) anything of this rank reads its halo cells again and (b) this rank overwrites the neighbours'
// halo cells again (WAR: a neighbour publishes its epoch only after the launches that read those cells).
static int halo_flush_wait(Solution& s, cudaStream_t st) {
    HaloState* h = s.halo;
    if (!h) return 0;
    if (h->comm_pending) {      // the side stream's copies read planes the next launch may overwrite
        YB_CUDA(cudaStreamWaitEvent(st, h->comm_ev, 0));
        h->comm_pending = false;
    }
    if (!h->wait_pending) return 0;
    halo_wait_kernel<<<1, 1, 0, st>>>(h->flags, h->wait_mask, h->epoch);
    YB_CUDA(cudaGetLastError());
    h->wait_pending = false;
    return 0;
}

// Push every dirty var/slot to the neighbours that need it and publish the next epoch.  The matching wait is left
// pending (halo_flush_wait) so that whatever the caller enqueues next overlaps the transfer.
//   skip_var:  the stage kernel already stored this var's x-face halos into the peers (fused path)
//   signalled: ... and already published the epoch to the pure x neighbours itself
//   side:      enqueue the pushes and signals on the side stream (ordered after what `st` holds now), so that the launches
//              the caller puts on `st` next -- the interior -- run while the slabs travel
static int halo_exchange_impl(Solution& s, cudaStream_t st, int skip_var, bool signalled, bool side = false) {
    HaloState* h = s.halo;
    if (!h) return 0;
    if (!h->finalized) return set_error(YB_ESTATE, "multi-rank solution: halo peers were not connected (yb_halo_import/finalize)");
    if (int rc = halo_flush_wait(s, st)) return rc;
    cudaStream_t ps = st;
    if (side && s.comm_stream && h->ext_ev) {
        YB_CUDA(cudaEventRecord(h->ext_ev, st));
        YB_CUDA(cudaStreamWaitEvent(s.comm_stream, h->ext_ev, 0));
        ps = s.comm_stream;
    }
    // Always a full handshake (even with nothing dirty): exchanges are collective, and every rank must
    // advance its epoch in lock-step with its neighbours.
    h->epoch++;
    unsigned int mask = 0;
    int launched = 0;
    for (auto& nb : h->nbrs) {
        const bool pure_x = nb.dir[0] != 0 && nb.dir[1] == 0 && nb.dir[2] == 0;
        for (size_t vi = 0; vi < s.vars.size(); vi++) {
            if (!var_talks_to(s.vars[vi], nb.dir)) continue;
            if (int(vi) == skip_var && pure_x) continue;   // done by the kernel
            for (int slot = 0; slot < s.vars[vi].nslots(); slot++) {
                if (!h->dirty[vi][slot]) continue;
                int rc = push_var_slot(s, nb, int(vi), slot, ps);
                if (rc < 0) return rc;
                launched += rc;
            }
        }
        int opp[3] = {-nb.dir[0], -nb.dir[1], -nb.dir[2]};
        // I am the peer's neighbour in direction `opp`; the peer waits on flags[dir_index(opp)]
        if (!(signalled && pure_x)) halo_signal_kernel<<<1, 1, 0, ps>>>(nb.peer_flags + dir_index(opp), h->epoch);
        mask |= 1u << dir_index(nb.dir);
    }
    YB_CUDA(cudaGetLastError());
    if (ps != st) {
        YB_CUDA(cudaEventRecord(h->comm_ev, ps));
        h->comm_pending = true;
    }
    h->wait_pending = true;
    h->wait_mask = mask;
    for (auto& dv : h->dirty)
        for (auto& f : dv) f = 0;
    s.stats.kernel_launches += launched;
    return 0;
}

// Explicit exchange (yk_solution::exchange_halos, the start and the end of run_solution): complete on return of the stream.
int halo_exchange_all(Solution& s, cudaStream_t st) {
    if (int rc = halo_exchange_impl(s, st, -1, false)) return rc;
    return halo_flush_wait(s, st);
}

int halo_finish(Solution& s, cudaStream_t st) { return halo_flush_wait(s, st); }

// Exchange of the fused rank-grid mode (the reference's wave-fronts: halos grow by the wave-front extension and are exchanged once
// per fused launch, /root/reference/src/kernel/lib/setup.cpp:717-781).  A fused launch that computes steps t+1 and t+2 reads the
// output var p(t) 2H and p(t-1) H deep past every rank interface (H = p's halo), and its inputs without a halo (v) H deep.  So:
//   face neighbours: the slot of step t 2H deep, the slot of t-1 H deep and, with `with_inputs`, every input var without a halo
//                    H deep (var_talks_to never sends those; they change only between runs);
//   edge neighbours: the slot of step t H deep -- step 1 beyond one interface reads the points beyond the other (the reference
//                    exchanges with every neighbour whenever it runs wave-fronts, alloc.cpp:504-510);
//   anything else that is dirty, as halo_exchange_impl sends it.
// Same epoch and WAR protocol as halo_exchange_impl, so every rank makes the same sequence of exchanges; the wait is left pending.
int halo_exchange_deep(Solution& s, int64_t t, bool with_inputs, cudaStream_t st) {
    HaloState* h = s.halo;
    if (!h->finalized) return set_error(YB_ESTATE, "multi-rank solution: halo peers were not connected (yb_halo_import/finalize)");
    if (int rc = halo_flush_wait(s, st)) return rc;
    const StageSpec& sp = s.spec.stages[0];
    const int pv = sp.outputs[0];
    const Var& p = s.vars[pv];
    int64_t H = 0;
    for (auto& d : p.dims)
        if (d.spec.kind == DIM_DOMAIN) H = std::max({H, d.spec.halo_l, d.spec.halo_r});
    const int newest = p.slot_of(t), older = p.slot_of(t - 1);
    auto haloless = [&](const Var& v) {
        for (auto& d : v.dims)
            if (d.spec.kind == DIM_DOMAIN && (d.spec.halo_l || d.spec.halo_r)) return false;
        return v.domain_dim(0) && v.domain_dim(1) && v.domain_dim(2);
    };
    h->epoch++;
    unsigned int mask = 0;
    int launched = 0;
    for (auto& nb : h->nbrs) {
        const int l1 = abs(nb.dir[0]) + abs(nb.dir[1]) + abs(nb.dir[2]);
        std::vector<std::pair<int, int>> sent;     // (var, slot) pushed deep to this neighbour
        auto push = [&](int vi, int slot, int64_t depth) {
            const int rc = push_var_slot(s, nb, vi, slot, st, depth);
            if (rc >= 0) { launched += rc; sent.emplace_back(vi, slot); }
            return rc;
        };
        int rc = 0;
        if (l1 == 1) {
            if (rc >= 0) rc = push(pv, newest, 2 * H);
            if (rc >= 0) rc = push(pv, older, H);
            if (with_inputs)
                for (int vi : sp.inputs)
                    if (rc >= 0 && vi != pv && haloless(s.vars[vi])) rc = push(vi, 0, H);
        } else if (l1 == 2) {
            rc = push(pv, newest, H);
        }
        for (size_t vi = 0; vi < s.vars.size() && rc >= 0; vi++) {
            if (!var_talks_to(s.vars[vi], nb.dir)) continue;
            for (int slot = 0; slot < s.vars[vi].nslots() && rc >= 0; slot++)
                if (h->dirty[vi][slot] && std::find(sent.begin(), sent.end(), std::make_pair(int(vi), slot)) == sent.end()) rc = push(int(vi), slot, 0);
        }
        if (rc < 0) return rc;
        int opp[3] = {-nb.dir[0], -nb.dir[1], -nb.dir[2]};
        halo_signal_kernel<<<1, 1, 0, st>>>(nb.peer_flags + dir_index(opp), h->epoch);
        mask |= 1u << dir_index(nb.dir);
    }
    YB_CUDA(cudaGetLastError());
    h->wait_pending = true;
    h->wait_mask = mask;
    for (auto& dv : h->dirty)
        for (auto& f : dv) f = 0;
    s.stats.kernel_launches += launched;
    return 0;
}

// `nsteps` steps from step t in ONE fused launch over the whole rank box (Engine::launch_steps), after the previous exchange has
// arrived; then the deep exchange of the two newest steps.  Returns the number of kernels launched (the exchange's pushes are
// counted by it).
int halo_run_steps(Solution& s, int64_t t, int nsteps, cudaStream_t st) {
    HaloState* h = s.halo;
    if (!h->finalized) return set_error(YB_ESTATE, "multi-rank solution: halo peers were not connected (yb_halo_import/finalize)");
    if (int rc = halo_flush_wait(s, st)) return rc;
    Box whole;
    for (int d = 0; d < 3; d++) { whole.b[d] = 0; whole.e[d] = d < s.ndd ? s.rank_size[d] : 1; }
    // the deep exchange below sends both newest steps, so every fused launch stores them (ends_run)
    const int rc = s.engine->launch_steps(s, t, nsteps, true, whole, st);
    if (rc < 0) return rc;
    for (const StageSpec& sp : s.spec.stages)
        for (int vi : sp.outputs)
            for (int k = 1; k <= nsteps; k++) h->dirty[vi][s.vars[vi].slot_of(t + k)] = 1;
    if (int e = halo_exchange_deep(s, t + nsteps, false, st)) return e;
    return rc;
}

// Is anything but `var`'s slot `slot` waiting to be pushed?  (The in-kernel signal may only be used when the kernel's
// own stores are the whole exchange.)
static bool other_dirty(const HaloState* h, int var, int slot) {
    for (size_t vi = 0; vi < h->dirty.size(); vi++)
        for (size_t sl = 0; sl < h->dirty[vi].size(); sl++)
            if (h->dirty[vi][sl] && !(int(vi) == var && int(sl) == slot)) return true;
    return false;
}

// One stage of one step on a multi-rank solution, ordered as the reference orders it
// (/root/reference/src/kernel/lib/context.cpp:378-475, halo.cpp:494-574): wait for the previous exchange, evaluate the
// EXTERIOR (the slabs the neighbours need) first, start the exchange, evaluate the interior while the halos travel.
// The wait for this exchange is enqueued in front of the next stage.  Three forms:
//   * fused (iso3dfd sweep kernel, x neighbours only): ONE launch whose first work units are the boundary planes; it
//     stores them into the neighbours' HBM as it computes them and publishes the epoch itself (IsoParams::sig_*);
//   * split: one launch per exterior slab, push kernels + epoch publication, then the interior launch;
//   * whole (domain too thin to split, stages with scratch vars, option overlap_comms=0): whole box, then push.
// Point sources and receivers (yb_points.h) are applied in the last stage of the step, and a source is in its slot before the
// exchange that publishes it: split form -- exterior points after the exterior launches, before the pushes and signals; the others
// after the interior launch; whole form -- after the launch, before the push; fused form -- after the launch, for sources farther
// than the widest x halo from every x interface (no neighbour reads them).  A rank that owns a source nearer than that runs the
// stage in the split form instead: the fused launch stores and publishes its boundary planes itself, before a source could enter.
// Both forms advance the epoch once, so the choice is the rank's own.
// Weighted receivers (yb_points.h) may read halo cells, which hold the neighbours' values of step u only once the step's last
// exchange has arrived: the last stage defers them, and they are recorded right after that wait -- at the top of the next step's
// first stage, or after halo_finish at the end of the run -- before the next step's first launch on this stream.
// Slice injectors (yb_slices.h) write the last stage's output like sources, just before them and in the same places; an injector
// row whose owned part reaches within the widest x halo of an x interface with a neighbour turns the fused form into the split
// form, as a source there does (writes_near_x_interface).  The split form injects the points outside the interior before the
// pushes and the rest after the interior launch, so every point is written once and before the exchange that publishes it.
// Slice recorders (yb_slices.h) only read: they record in the last stage, after the launch that computed the rank's last points
// and that launch's points (fused: the launch; whole: the launch; split: the interior launch), on this stream, so before the next
// step's first launch overwrites an in-place var.  They never change the form.  Slice correlators only read the var too: they
// follow the recorders in the same places.
// Does this rank write at step t, after the last stage's launch, within w planes of an x interface with a neighbour rank (point
// sources, slice injectors)?  Such a write must come before the boundary planes are published, which the fused x launch does itself.
static bool writes_near_x_interface(const Solution& s, int64_t t, int64_t w) {
    const bool lo = s.rank_index[0] > 0, hi = s.rank_index[0] < s.num_ranks[0] - 1;
    auto near = [&](int64_t x0, int64_t x1) { return (lo && x0 < w) || (hi && x1 >= s.rank_size[0] - w); };
    int64_t x0 = 0, x1 = 0;
    return (points_source_x_range(s, t, x0, x1) && near(x0, x1)) || (slice_injectors_x_range(s, t, x0, x1) && near(x0, x1));
}

int halo_run_stage(Solution& s, int stage, int64_t t, cudaStream_t st) {
    Box whole;
    for (int d = 0; d < 3; d++) { whole.b[d] = 0; whole.e[d] = d < s.ndd ? s.rank_size[d] : 1; }
    HaloState* h = s.halo;
    if (!h->finalized) return set_error(YB_ESTATE, "multi-rank solution: halo peers were not connected (yb_halo_import/finalize)");
    if (int rc = halo_flush_wait(s, st)) return rc;
    if (int rc = points_record_pending(s, st); rc < 0) return rc;       // the previous step's weighted receivers, halos now final
    const StageSpec& sp = s.spec.stages[stage];
    auto mark_outputs_dirty = [&]() {
        for (int vi : sp.outputs) h->dirty[vi][s.vars[vi].slot_of(t + sp.out_step_off)] = 1;
    };
    auto opt_off = [&](const char* key) { auto it = s.options.find(key); return it != s.options.end() && it->second == "0"; };
    const bool overlap = !opt_off("overlap_comms");
    const bool last_stage = stage + 1 == int(s.spec.stages.size());
    // the last stage's writes after its launch: injectors first, then sources (and the receivers of the points kernel)
    auto apply_points = [&](int sel, const Box& interior) {
        if (!last_stage) return 0;
        const int a = slice_injectors_launch(s, t, sel, interior, st);
        if (a < 0) return a;
        const int b = points_launch(s, t, sel, interior, st);
        return b < 0 ? b : a + b;
    };
    auto record_slices = [&]() {
        if (!last_stage) return 0;
        const int a = slices_launch(s, t, st);
        if (a < 0) return a;
        const int b = slice_correlators_launch(s, t, st);
        return b < 0 ? b : a + b;
    };
    int64_t wx = 0;         // widest x halo: the planes of an x interface the neighbour reads
    for (auto& v : s.vars)
        if (const Dim* dx = v.domain_dim(0)) wx = std::max({wx, dx->spec.halo_l, dx->spec.halo_r});
    const bool fused_ok = !opt_off("fused_halo") && !(last_stage && writes_near_x_interface(s, t, wx));

    // ---- fused path -----------------------------------------------------------------------------------------
    s.fused_x = Solution::FusedX();
    unsigned long long *fx_flag_lo = nullptr, *fx_flag_hi = nullptr;      // the neighbours' flag words (copy-engine path)
    bool only_x = !h->nbrs.empty();
    for (auto& nb : h->nbrs) only_x = only_x && nb.dir[1] == 0 && nb.dir[2] == 0;
    if (sp.outputs.size() == 1 && fused_ok) {
        const int vi = sp.outputs[0];
        const Var& v = s.vars[vi];
        const int slot = v.slot_of(t + sp.out_step_off);
        const Dim* dx = v.domain_dim(0);
        for (auto& nb : h->nbrs) {
            if (nb.dir[1] != 0 || nb.dir[2] != 0 || nb.dir[0] == 0 || !dx) continue;
            const BlobVar& pg = nb.var_geom[vi];
            // same y/z geometry on both sides (always true for pure x neighbours) and a 3-D var
            bool same = pg.nd == 3 && pg.stride[0] == v.dims[1].stride && pg.stride[1] == v.dims[2].stride && pg.stride[2] == 1 &&
                        pg.pad_l[1] == v.dims[2].pad_l && pg.pad_l[2] == v.dims[3].pad_l;
            if (!same) continue;
            char* base = nb.var_base[vi] + size_t(slot) * pg.slot_elems * v.elem_bytes;
            long long origin = pg.pad_l[0] * pg.stride[0] + pg.pad_l[1] * pg.stride[1] + pg.pad_l[2] * pg.stride[2];
            int opp[3] = {-nb.dir[0], 0, 0};
            if (nb.dir[0] < 0) {
                s.fused_x.lo = base + (origin + pg.domain[0] * pg.stride[0]) * v.elem_bytes;      // its right halo starts at its n_x
                s.fused_x.flag_lo = nb.peer_flags + dir_index(opp);
            } else {
                s.fused_x.hi = base + (origin - dx->domain * pg.stride[0]) * v.elem_bytes;          // my plane n_x-R.. -> its planes -R..
                s.fused_x.flag_hi = nb.peer_flags + dir_index(opp);
            }
            s.fused_x.var = vi;
        }
        // the kernel may publish the epoch itself when its stores are the whole exchange
        size_t n_fused = (s.fused_x.lo ? 1 : 0) + (s.fused_x.hi ? 1 : 0);
        if (s.fused_x.var >= 0 && only_x && n_fused == h->nbrs.size() && overlap && !other_dirty(h, vi, slot)) {
            s.fused_x.counter = h->sig_counter;
            s.fused_x.epoch = h->epoch + 1;
            // Copy-engine transfer (option dma_halo=1; default: the kernel's own peer stores): the kernel publishes the epoch
            // into a LOCAL word once its boundary planes are stored, the side stream waits on that word (cuStreamWaitValue64)
            // and moves the planes -- contiguous slabs of R x-planes -- with cudaMemcpyAsync over NVLink, then publishes the
            // epoch to the neighbour.
            auto dm = s.options.find("dma_halo");
            if (dm != s.options.end() && dm->second == "1" && stream_wait_value64() && s.comm_stream) {
                s.fused_x.dma = true;
                fx_flag_lo = s.fused_x.flag_lo; fx_flag_hi = s.fused_x.flag_hi;
                s.fused_x.flag_lo = h->local_done; s.fused_x.flag_hi = nullptr;
            }
        }
    }
    if (s.fused_x.var >= 0) {
        const Solution::FusedX fx = s.fused_x;
        int rc = s.engine->launch(s, stage, t, whole, st);
        if (rc < 0) return rc;
        s.stats.kernel_launches += rc;
        mark_outputs_dirty();
        const int skip = s.fused_x.used ? s.fused_x.var : -1;
        const bool signalled = s.fused_x.used && s.fused_x.signalled;
        const bool dma = signalled && fx.dma;
        s.fused_x = Solution::FusedX();
        if (int e = apply_points(PTS_ALL, whole); e < 0) return e;
        if (int e = record_slices(); e < 0) return e;
        if (dma) {
            const Var& v = s.vars[fx.var];
            const Dim* dx = v.domain_dim(0);
            const int64_t R = std::max(dx->spec.halo_l, dx->spec.halo_r);
            const size_t bytes = size_t(R) * size_t(dx->stride) * v.elem_bytes;
            const char* mine = v.slot_ptr(v.slot_of(t + sp.out_step_off)) + size_t(dx->pad_l) * dx->stride * v.elem_bytes;   // plane x = 0
            CUresult cr = stream_wait_value64()(reinterpret_cast<CUstream>(s.comm_stream), reinterpret_cast<CUdeviceptr>(h->local_done), fx.epoch,
                                                CU_STREAM_WAIT_VALUE_GEQ);
            if (cr != CUDA_SUCCESS) return set_error(YB_ECUDA, "cuStreamWaitValue64 failed with code %d", int(cr));
            // fx.lo / fx.hi are the peers' element (0,0,0)-relative bases as the kernel would index them (like `out`): plane x
            // of this rank lands at base + (x * stride) there; whole planes, pads included, are contiguous on both sides
            const size_t origin_off = size_t(v.origin_offset() - dx->pad_l * dx->stride) * v.elem_bytes;   // y/z pads inside a plane
            if (fx.lo) {
                YB_CUDA(cudaMemcpyAsync(static_cast<char*>(fx.lo) - origin_off, mine, bytes, cudaMemcpyDefault, s.comm_stream));
                halo_signal_kernel<<<1, 1, 0, s.comm_stream>>>(fx_flag_lo, fx.epoch);
            }
            if (fx.hi) {
                const size_t last = size_t(dx->domain - R) * dx->stride * v.elem_bytes;
                YB_CUDA(cudaMemcpyAsync(static_cast<char*>(fx.hi) + last - origin_off, mine + last, bytes, cudaMemcpyDefault, s.comm_stream));
                halo_signal_kernel<<<1, 1, 0, s.comm_stream>>>(fx_flag_hi, fx.epoch);
            }
            YB_CUDA(cudaGetLastError());
            YB_CUDA(cudaEventRecord(h->comm_ev, s.comm_stream));
            h->comm_pending = true;
        }
        return halo_exchange_impl(s, st, skip, signalled);
    }

    // ---- split path: exterior slabs, exchange, interior --------------------------------------------------------
    Box interior = whole;
    bool split = overlap && s.engine->can_split(s, stage);
    int64_t w[3] = {0, 0, 0};
    for (int d = 0; d < s.ndd && split; d++) {
        if (s.num_ranks[d] <= 1) continue;
        // In a unit-stride dim every box starts on a 16-byte boundary (the rank's domain origin is 128-B aligned): the TMA
        // sweep kernels need that, and a box start off it faults on an H100.  So the exterior slabs there are w rounded up
        // to whole 16-byte vectors wide -- up to 3 (fp32) or 1 (fp64) planes more -- and the interior keeps its sweep.
        int64_t al = 1;
        for (auto& v : s.vars) {
            const Dim* dd = v.domain_dim(d);
            if (!dd) continue;
            w[d] = std::max<int64_t>(w[d], std::max(dd->spec.halo_l, dd->spec.halo_r));
            if (dd->stride == 1) al = std::max<int64_t>(al, 16 / v.elem_bytes);
        }
        if (s.rank_index[d] > 0) interior.b[d] += (w[d] + al - 1) / al * al;
        if (s.rank_index[d] < s.num_ranks[d] - 1) interior.e[d] = std::max<int64_t>(0, interior.e[d] - w[d]) / al * al;
        if (interior.e[d] - interior.b[d] < 1) split = false;
    }
    if (!split) {
        int rc = s.engine->launch(s, stage, t, whole, st);
        if (rc < 0) return rc;
        s.stats.kernel_launches += rc;
        mark_outputs_dirty();
        if (int e = apply_points(PTS_ALL, whole); e < 0) return e;
        if (int e = record_slices(); e < 0) return e;
        return halo_exchange_impl(s, st, -1, false);
    }
    Box cur = whole;
    for (int d = 0; d < s.ndd; d++) {
        for (int side = 0; side < 2; side++) {
            Box slab = cur;
            if (side == 0) { if (interior.b[d] == whole.b[d]) continue; slab.e[d] = interior.b[d]; }
            else { if (interior.e[d] == whole.e[d]) continue; slab.b[d] = interior.e[d]; }
            int rc = s.engine->launch(s, stage, t, slab, st);
            if (rc < 0) return rc;
            s.stats.kernel_launches += rc;
        }
        cur.b[d] = interior.b[d]; cur.e[d] = interior.e[d];
    }
    mark_outputs_dirty();
    if (int e = apply_points(PTS_EXTERIOR, interior); e < 0) return e;
    if (int rc = halo_exchange_impl(s, st, -1, false, true)) return rc;      // pushes on the side stream, behind the exterior
    int rc = s.engine->launch(s, stage, t, interior, st);
    if (rc < 0) return rc;
    s.stats.kernel_launches += rc;
    if (int e = apply_points(PTS_INTERIOR, interior); e < 0) return e;
    if (int e = record_slices(); e < 0) return e;
    return 0;
}

}  // namespace yb

using namespace yb;

extern "C" {

int yb_halo_export_size(const yb_solution* s_, size_t* n) {
    if (!s_ || !n) return set_error(YB_EINVAL, "null argument");
    *n = sizeof(Blob);
    return 0;
}

int yb_halo_export(yb_solution* s_, void* out, size_t nbytes) {
    Solution* s = reinterpret_cast<Solution*>(s_);
    if (!s || !out) return set_error(YB_EINVAL, "null argument");
    if (!s->prepared) return set_error(YB_ESTATE, "solution not prepared");
    if (!s->halo) return set_error(YB_ESTATE, "solution has a single rank: nothing to export");
    if (nbytes < sizeof(Blob)) return set_error(YB_EINVAL, "blob buffer too small");
    YB_CUDA(cudaSetDevice(s->device));
    Blob b;
    memset(&b, 0, sizeof b);
    b.magic = BLOB_MAGIC; b.version = 4; b.pid = int64_t(getpid()); b.nonce = process_nonce(); b.device = s->device;
    b.num_vars = int(s->vars.size());
    for (int k = 0; k < 3; k++) { b.rank_index[k] = s->rank_index[k]; b.rank_size[k] = s->rank_size[k]; }
    b.fused_steps = s->engine->fused_steps(*s);
    YB_CUDA(cudaIpcGetMemHandle(&b.flags_handle, s->halo->flags));
    b.flags_raw = reinterpret_cast<uint64_t>(s->halo->flags);
    for (int i = 0; i < b.num_vars; i++) {
        const Var& v = s->vars[i];
        YB_CUDA(cudaIpcGetMemHandle(&b.vars[i].handle, v.dev));
        b.vars[i].raw_ptr = reinterpret_cast<uint64_t>(v.dev);
        b.vars[i].bytes = int64_t(v.bytes());
        b.vars[i].slot_elems = v.slot_elems;
        int k = 0;
        for (auto& d : v.dims) {
            if (d.spec.kind == DIM_STEP || k >= 4) continue;
            b.vars[i].pad_l[k] = d.spec.kind == DIM_MISC ? 0 : d.pad_l;
            b.vars[i].stride[k] = d.stride;
            b.vars[i].domain[k] = d.domain;
            k++;
        }
        b.vars[i].nd = k;
    }
    memcpy(out, &b, sizeof b);
    return 0;
}

int yb_halo_import(yb_solution* s_, int64_t peer_rank_linear, const void* blob, size_t nbytes) {
    Solution* s = reinterpret_cast<Solution*>(s_);
    if (!s || !blob) return set_error(YB_EINVAL, "null argument");
    if (!s->halo) return set_error(YB_ESTATE, "solution has a single rank");
    if (nbytes < sizeof(Blob)) return set_error(YB_EINVAL, "blob too small");
    Blob b;
    memcpy(&b, blob, sizeof b);
    if (b.magic != BLOB_MAGIC || b.num_vars != int(s->vars.size())) return set_error(YB_EINVAL, "halo blob does not match this solution");
    YB_CUDA(cudaSetDevice(s->device));
    for (auto& nb : s->halo->nbrs) {
        if (nb.peer_linear != peer_rank_linear) continue;
        for (int k = 0; k < 3; k++)
            if (b.rank_index[k] != s->rank_index[k] + nb.dir[k]) return set_error(YB_EINVAL, "blob of rank %lld has unexpected rank index", (long long)peer_rank_linear);
        const int fs = s->engine->fused_steps(*s);
        if (b.fused_steps != fs)
            return set_error(YB_EINVAL, "rank %lld exchanges halos once per %d step(s) but its neighbour rank %lld once per %d: block_steps and "
                                        "mega_block_steps must select the same mode on every rank", (long long)linear_rank(*s, s->rank_index), fs,
                             (long long)peer_rank_linear, int(b.fused_steps));
        nb.same_process = (b.nonce == process_nonce());
        for (int i = 0; i < b.num_vars; i++) nb.var_geom[i] = b.vars[i];
        if (nb.same_process) {
            // same process (single-process multi-rank tests): plain pointers; enable peer access if on another device
            if (b.device != s->device) {
                cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
                    return set_error(YB_ECUDA, "cudaDeviceEnablePeerAccess(%d) failed: %s", b.device, cudaGetErrorString(e));
                cudaGetLastError();
            }
            nb.peer_flags = reinterpret_cast<unsigned long long*>(b.flags_raw);
            for (int i = 0; i < b.num_vars; i++) nb.var_base[i] = reinterpret_cast<char*>(b.vars[i].raw_ptr);
        } else {
            void* p = nullptr;
            YB_CUDA(cudaIpcOpenMemHandle(&p, b.flags_handle, cudaIpcMemLazyEnablePeerAccess));
            nb.opened.push_back(p);
            nb.peer_flags = static_cast<unsigned long long*>(p);
            for (int i = 0; i < b.num_vars; i++) {
                void* q = nullptr;
                YB_CUDA(cudaIpcOpenMemHandle(&q, b.vars[i].handle, cudaIpcMemLazyEnablePeerAccess));
                nb.opened.push_back(q);
                nb.var_base[i] = static_cast<char*>(q);
            }
        }
        nb.connected = true;
        return 0;
    }
    return 0;  // not a neighbour: ignored
}

int yb_halo_finalize(yb_solution* s_) {
    Solution* s = reinterpret_cast<Solution*>(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (!s->halo) return 0;
    for (auto& nb : s->halo->nbrs)
        if (!nb.connected)
            return set_error(YB_ESTATE, "neighbour rank %lld (dir %d,%d,%d) was not imported", (long long)nb.peer_linear, nb.dir[0], nb.dir[1], nb.dir[2]);
    s->halo->finalized = true;
    return 0;
}

int yb_exchange_halos(yb_solution* s_) {
    Solution* s = reinterpret_cast<Solution*>(s_);
    if (!s) return set_error(YB_EINVAL, "null solution");
    if (!s->prepared) return set_error(YB_ESTATE, "exchange_halos() called before prepare_solution()");
    if (!s->halo) return 0;
    YB_CUDA(cudaSetDevice(s->device));
    int rc = halo_exchange_all(*s, s->stream());
    return rc < 0 ? rc : 0;
}

}  // extern "C"
