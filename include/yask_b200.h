/*
 * yask_b200.h -- C ABI of the H100-native stencil engine (libyask_b200.so).
 *
 * This is the drop-in boundary for the hot path of intel/yask (yk_solution::run_solution and
 * the var/geometry calls around it).  The reference has no C plugin ABI: its boundary is the
 * C++ kernel API (yk_factory / yk_env / yk_solution / yk_var / yk_stats,
 * /root/reference/include/yask_kernel_api.hpp, aux/yk_solution_api.hpp, aux/yk_var_api.hpp),
 * implemented by a per-stencil libyask_kernel.<stencil>.<arch>.so.  Each entry point below is
 * what a binding of that C++ API needs from a device engine; the C++ mirror of the reference
 * API that sits on top of it lives in yask_b200/include/yask_kernel_api.hpp (see INTEGRATION.md).
 *
 * Conventions
 *   - plain C types only; every function returns 0 on success, a negative YB_E* code on
 *     failure, and yb_last_error() returns the message for the calling thread (the C++ layer
 *     turns it into yask::yask_exception, /root/reference/include/yask_common_api.hpp:125-179).
 *   - indices are GLOBAL ("overall problem") element indices exactly as in the reference's
 *     yk_var API (aux/yk_var_api.hpp:60-183): domain index 0 is the first point of the overall
 *     domain, halo points of the first rank are negative.
 *   - dims of a var are given in the var's declared order; the step dim (if any) comes first.
 *   - all data lives in device (HBM) memory; host buffers passed to slice calls are copied.
 *   - there is NO CPU fallback: without a CUDA device yb_solution_prepare() fails.
 */
#ifndef YASK_B200_H
#define YASK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YB_MAX_DIMS 5          /* step + up to 3 domain + misc */
#define YB_MAX_DOMAIN_DIMS 3
#define YB_NAME_LEN 64

enum {
    YB_OK = 0,
    YB_EINVAL = -1,    /* bad argument / unknown name  (reference: yask_exception) */
    YB_ESTATE = -2,    /* call not legal in this state, e.g. run before prepare (context.cpp:265-266) */
    YB_ERANGE = -3,    /* index outside the allocation / invalid step (yk_var.hpp:1084-1135) */
    YB_ECUDA = -4,     /* CUDA runtime/driver error, or no device */
    YB_ENOMEM = -5,
    YB_EUNSUPPORTED = -6
};

/* FP-contraction modes of the point-update arithmetic (see oracle/yask_oracle.c). */
enum {
    YB_FP_STRICT = 0,   /* IEEE mul/add in DSL order == reference built with -ffp-contract=off */
    YB_FP_FMA = 1,      /* canonical fused form */
    YB_FP_REF_GCC = 2   /* FMA pattern of the reference's default GCC build (default) */
};

typedef struct yb_solution yb_solution;   /* opaque; mirrors yk_solution (aux/yk_solution_api.hpp:82) */

/* Per-dim geometry of one var, all in elements.  Mirrors the getters of yk_var
 * (aux/yk_var_api.hpp:185-640) and SURVEY.md Appendix C. */
typedef struct yb_dim_info {
    char name[YB_NAME_LEN];
    int32_t kind;             /* 0 = step, 1 = domain, 2 = misc */
    int32_t domain_index;     /* for kind==1: position in the solution's domain dims, else -1 */
    int64_t rank_offset;      /* global index of this rank's first domain point */
    int64_t domain_size;      /* rank domain size (kind 1); alloc_t (kind 0); misc extent (kind 2) */
    int64_t left_halo, right_halo;
    int64_t left_pad, right_pad;   /* >= halo; alloc = left_pad + domain_size + right_pad */
    int64_t alloc_size;
    int64_t first_misc_index;
    int64_t stride;           /* element stride in device storage (0 for the step dim) */
} yb_dim_info;

typedef struct yb_var_info {
    char name[YB_NAME_LEN];
    int32_t num_dims;
    int32_t elem_bytes;
    int32_t has_step;
    int32_t step_alloc;           /* number of step slots (alloc_t) */
    int64_t first_valid_step, last_valid_step;
    int32_t is_output;            /* written by the solution */
    int32_t halo_exchange_l1_norm;
    int64_t slot_elems;           /* elements per step slot (incl. pads) */
    int64_t storage_bytes;
    yb_dim_info dims[YB_MAX_DIMS];
} yb_var_info;

/* Mirrors yk_stats (aux/yk_solution_api.hpp:1300-1348). */
typedef struct yb_stats {
    int64_t num_elements;         /* overall domain points */
    int64_t num_steps_done;
    int64_t num_writes_done;
    int64_t est_fp_ops_done;
    int64_t num_reads_done;
    double elapsed_secs;          /* device time inside yb_solution_run (CUDA events) */
    double halo_secs;             /* part of elapsed spent waiting on halo exchange */
    int64_t kernel_launches;      /* stencil kernels launched since last clear */
} yb_stats;

/* ---- library ------------------------------------------------------------------------------ */
const char* yb_version_string(void);              /* yk_factory::get_version_string, yask_kernel_api.hpp:90 */
const char* yb_last_error(void);
int yb_device_count(void);                        /* number of visible CUDA devices (0 if none) */
int yb_num_stencils(void);
const char* yb_stencil_name(int i);               /* registry of built-in solutions (REGISTER_SOLUTION names) */

/* ---- solution life cycle (yk_factory::new_solution, factory.cpp:51-105) --------------------- */
/* stencil: "iso3dfd" | ... ; radius <= 0 selects the stencil's default (iso3dfd: 8);
 * elem_bytes: 4 or 8 (0 = default 4). */
int yb_solution_create(yb_solution** out, const char* stencil, int radius, int elem_bytes);
int yb_solution_destroy(yb_solution* s);          /* yk_solution::end_solution + release */
const char* yb_solution_name(const yb_solution* s);           /* get_name */
const char* yb_solution_target(const yb_solution* s);         /* get_target: "sm_90a" */
int yb_solution_elem_bytes(const yb_solution* s);             /* get_element_bytes */
int yb_solution_num_domain_dims(const yb_solution* s);        /* get_num_domain_dims */
const char* yb_solution_domain_dim_name(const yb_solution* s, int i);
const char* yb_solution_step_dim_name(const yb_solution* s);

/* ---- settings, legal before prepare (aux/yk_solution_api.hpp:187-518) ------------------------ */
int yb_set_rank_domain_size(yb_solution* s, int dim, int64_t n);     /* set_rank_domain_size */
int yb_set_overall_domain_size(yb_solution* s, int dim, int64_t n);  /* set_overall_domain_size */
int yb_set_num_ranks(yb_solution* s, int dim, int64_t n);            /* set_num_ranks */
int yb_set_rank_index(yb_solution* s, int dim, int64_t i);           /* set_rank_index */
int yb_set_min_pad_size(yb_solution* s, int dim, int64_t n);         /* set_min_pad_size */
int64_t yb_get_rank_domain_size(const yb_solution* s, int dim);
int64_t yb_get_overall_domain_size(const yb_solution* s, int dim);
int64_t yb_get_num_ranks(const yb_solution* s, int dim);
int64_t yb_get_rank_index(const yb_solution* s, int dim);
int64_t yb_get_first_rank_domain_index(const yb_solution* s, int dim);  /* valid after prepare */
int64_t yb_get_last_rank_domain_index(const yb_solution* s, int dim);
/* Engine options ("-key value" strings of apply_command_line_options, soln_apis.cpp:285-313):
 *   fp_mode = 0|1|2, kernel = auto|tma|direct, lx = <planes per sweep chunk>, ...            */
int yb_set_option(yb_solution* s, const char* key, const char* value);
int yb_get_option(const yb_solution* s, const char* key, char* value, size_t value_len);
/* Run the kernels on this CUDA stream (a cudaStream_t cast to void*; NULL = the solution's own). */
int yb_set_stream(yb_solution* s, void* cuda_stream);

/* Host-only part of prepare (setup_rank, setup.cpp:462-503): derive this rank's domain size and
 * offset from the overall size / rank grid / rank index.  Needs no device; prepare() calls it too. */
int yb_solution_plan_geometry(yb_solution* s);

/* ---- prepare: rank geometry + device allocation (prepare_solution, soln_apis.cpp:137-249) ---- */
int yb_solution_prepare(yb_solution* s, int device);
int yb_solution_is_prepared(const yb_solution* s);

/* ---- vars (yk_solution::get_var/get_vars, yk_var getters) ----------------------------------- */
int yb_num_vars(const yb_solution* s);
int yb_var_index(const yb_solution* s, const char* name);     /* <0 if unknown */
int yb_var_info_get(const yb_solution* s, int var, yb_var_info* out);
/* User-created vars (yk_solution::new_var / new_fixed_size_var, aux/yk_solution_api.hpp:994-1089): not read
 * or written by the stencil kernels.  dim names matching the step dim / a domain dim take that role, any
 * other name is a misc dim.  sizes == NULL: sized like the solution (new_var); otherwise fixed sizes (one per
 * dim: steps / domain points / misc extent).  Returns the new var's index (>= 0) or a negative error. */
int yb_var_create(yb_solution* s, const char* name, int ndims, const char* const* dim_names, const int64_t* sizes);

/* yk_var::fuse_vars (aux/yk_var_api.hpp:1370-1397; /root/reference/src/kernel/lib/yk_var_apis.cpp:334-360): `var` of `s`
 * becomes another reference to the device storage of `src_var` of `src` (the same or another solution of this process);
 * layouts must be identical; storage `var` had is released when its last user lets go. */
int yb_var_fuse(yb_solution* s, int var, yb_solution* src, int src_var);
/* Set per-var geometry before prepare (set_halo_size / set_min_pad_size, yk_var_api.hpp:1180-1290). */
int yb_var_set_min_pad(yb_solution* s, int var, int dim, int64_t left, int64_t right);

/* Slice copies between a caller-owned HOST buffer (row-major in declared dim order, last dim
 * unit stride) and device storage: yk_var::set_elements_in_slice / get_elements_in_slice
 * (aux/yk_var_api.hpp:699-751, 876-961).  first/last have num_dims entries (step first).
 * Returns the number of elements copied in *n_done (may be NULL). */
int yb_var_set_slice(yb_solution* s, int var, const void* host_buf, const int64_t* first, const int64_t* last, int64_t* n_done);
int yb_var_get_slice(yb_solution* s, int var, void* host_buf, const int64_t* first, const int64_t* last, int64_t* n_done);
/* Same, but the buffer is DEVICE memory on the solution's device (no host round trip). */
int yb_var_set_slice_device(yb_solution* s, int var, const void* dev_buf, const int64_t* first, const int64_t* last, int64_t* n_done);
int yb_var_get_slice_device(yb_solution* s, int var, void* dev_buf, const int64_t* first, const int64_t* last, int64_t* n_done);
/* yk_solution::run_auto_tuner_now (aux/yk_solution_api.hpp:858-882): times the engine's launch variants over the rank
 * domain right now (no halo exchange; var contents are NOT preserved), keeps the fastest for later run_solution()
 * calls, clears the stats.  `report` (may be NULL) receives one line per trial. */
int yb_solution_auto_tune(yb_solution* s, char* report, size_t report_len);
/* In-run tuner (yk_solution::reset_auto_tuner, is_auto_tuner_enabled, option -auto_tune; aux/yk_solution_api.hpp:820-856):
 * while enabled, every run_solution() step executes with the next untried launch variant and is timed; when all variants
 * have their samples the fastest stays selected and the tuner switches itself off.  Variants compute identical bits, so the
 * steps taken while tuning are real steps. */
int yb_solution_reset_auto_tuner(yb_solution* s, int enable);
int yb_solution_is_auto_tuner_enabled(const yb_solution* s);
int yb_solution_auto_tuner_report(const yb_solution* s, char* report, size_t report_len);
/* Reductions over a slice, on the device, accumulated in double in a fixed order: yk_var::reduce_elements_in_slice
 * (aux/yk_var_api.hpp:984-1110; /root/reference/src/kernel/lib/yk_var.hpp:1367-1450).
 * out = {sum, sum of squares, product, max, min}; *n_done = number of elements reduced (may be NULL). */
int yb_var_reduce_slice(yb_solution* s, int var, const int64_t* first, const int64_t* last, double out[5], int64_t* n_done);
/* set_all_elements_same (writes every storage element incl. pads, yk_var.hpp:1786-1793). */
int yb_var_set_all_same(yb_solution* s, int var, double value);
/* set_elements_in_slice_same. */
int yb_var_set_slice_same(yb_solution* s, int var, double value, const int64_t* first, const int64_t* last, int64_t* n_done);
/* Deterministic synthetic data on the device: value = lo + (hi-lo)*u(hash(seed, salt, global idx))
 * over the rank's halo box of API step `step` (same function as yask_b200/synth.py). */
int yb_var_fill_hash(yb_solution* s, int var, int64_t step, uint32_t seed, uint32_t salt, double lo, double hi);
/* Same, with `shift[d]` (one entry per solution domain dim; NULL = zeros) added to the global index of every point:
 * a small stand-alone solution can then hold exactly the values a window of a larger (multi-rank) problem holds --
 * bench.py's halo check recomputes the rank interfaces this way. */
int yb_var_fill_hash_shifted(yb_solution* s, int var, int64_t step, uint32_t seed, uint32_t salt, double lo, double hi,
                             const int64_t* shift);
/* Order-independent 64-bit checksum (sum of per-element bit patterns mixed with the global index)
 * over the rank-domain box of API step `step`. */
int yb_var_checksum(yb_solution* s, int var, int64_t step, uint64_t* out);
/* Raw device pointer of a step slot (get_raw_storage_buffer, yk_var_api.hpp:1399-1437). */
int yb_var_device_ptr(yb_solution* s, int var, int64_t step, void** out);

/* Plain device->host copy of `bytes` bytes (for host snapshots of raw storage). */
int yb_copy_to_host(void* host_dst, const void* dev_src, size_t bytes);

/* ---- run (yk_solution::run_solution, context.cpp:220-624) ----------------------------------- */
int yb_solution_run(yb_solution* s, int64_t first_step, int64_t last_step);
int yb_solution_sync(yb_solution* s);              /* wait for all queued device work */
int yb_get_stats(yb_solution* s, yb_stats* out);   /* get_stats (syncs) */
int yb_clear_stats(yb_solution* s);                /* clear_stats */

/* ---- point sources and receivers, applied on the device inside run_solution() ------------------------------------
 * Replaces the host loop run_solution(t, t); add_to_element(amp[t], {t+1, src}); get_element({t+1, rcv}) with one call.
 * Whenever a run has computed step u (after all its stages; u = t+1, or t-1 for a reverse solution):
 *   1. if 0 <= u - t0 < nrows: var(u, idx_i) += amp[u - t0][i] for every source i in list order, rounded as add_to_element
 *      (fp32: float(float(old) + float(amp)); fp64: old + amp);
 *   2. then, if 0 <= u - t0r < nrows_r: trace[u - t0r][j] = var(u, ridx_j) in the element type.
 * `idx` holds n (m) points of num_domain_dims GLOBAL domain indices each, row-major; every index must lie in the overall
 * domain (halo and pad cells are refused).  The var must have the step dim and every domain dim, no misc dim, and be written
 * by a stage; on a rank grid a source var must be written by the last stage.  The sets persist across runs until cleared or
 * replaced; a rank keeps only the points of its own domain.  Legal before or after prepare (checked as soon as the rank
 * geometry is known; a prepared solution synchronizes its stream and uploads the tables).  While points are set every run takes
 * one step per launch (block_steps pairs resume once they are cleared); a rank grid whose halos are exchanged once per pair of
 * steps (block_steps=2 + mega_block_steps=2) refuses them.  Read-only option point_launches: point-kernel launches since prepare. */
int yb_solution_set_sources(yb_solution* s, const char* var, int64_t n, const int64_t* idx, int64_t t0, int64_t nrows,
                            const double* amp /* nrows x n */);
int yb_solution_set_receivers(yb_solution* s, const char* var, int64_t m, const int64_t* idx, int64_t t0r, int64_t nrows_r);
/* Copy the traces (nrows_r x m elements of the solution's type; rows not recorded yet are 0) into `out` and set owned[j] = 1
 * for the receivers this rank records (0 for the others, whose columns stay 0).  `out` may be NULL: then only the mask, which
 * needs no device once the rank geometry is known (plan_geometry). */
int yb_solution_get_traces(yb_solution* s, void* out, uint8_t* owned);
int yb_solution_clear_points(yb_solution* s);      /* remove both sets */

/* Weighted sets: sources and receivers between grid points.  Each of the n sources (m receivers) has k support entries
 * (idx[i][q], w[i][q]): num_domain_dims GLOBAL domain indices (idx is n x k x num_domain_dims, row-major) and a double weight
 * (w is n x k).  A weighted set replaces the set of its kind, on-grid or weighted; the source set and the receiver set are each
 * one kind or the other, independently.  Whenever a run has computed step u (after all its stages):
 *   1. if 0 <= u - t0 < nrows: for each source i in list order, each entry q in order with w[i][q] != 0:
 *      a = w[i][q] * amp[u - t0][i] in double (one rounded multiply), added to var(u, idx[i][q]) with add_to_element's rounding
 *      (fp32: float(float(old) + float(a)); fp64: old + a);
 *   2. then, if 0 <= u - t0r < nrows_r: for each receiver j, acc = +0.0 (double), then for each entry q in order with
 *      w[j][q] != 0: acc = acc + w[j][q] * double(var(u, idx[j][q])), every multiply and add rounded on its own (no FMA);
 *      trace[u - t0r][j] = T(acc), rounded to nearest.
 * Entries of weight exactly 0 are dropped and need not lie in the domain; every other entry must.  A non-finite weight, k < 1 and
 * a point whose weights are all 0 are refused.  k = 1, w = 1 gives the bits of yb_solution_set_sources / set_receivers.
 * On a rank grid each rank adds the source entries of its own domain.  Receiver j is owned (get_traces' mask) by the rank holding
 * its first nonzero entry; every other entry must be in that rank's domain or in a halo cell its exchange refreshes (within the
 * var's halo, toward a neighbour the var exchanges with: iso3dfd's p exchanges with face neighbours only, so a receiver reaching a
 * diagonal neighbour is refused).  A receiver that reads halo cells is recorded after the step's last exchange and needs its var
 * written by the last stage, and either two step slots or two stages.  Every other rule (var, prepare, upload, pairs, fused-pair
 * rank grids, get_traces, clear_points) is that of yb_solution_set_sources.  point_launches counts one per kernel launched;
 * point_groups writes a weighted entry as i/q ("0/3,2/0;1/0"). */
int yb_solution_set_sources_weighted(yb_solution* s, const char* var, int64_t n, int64_t k, const int64_t* idx, const double* w,
                                     int64_t t0, int64_t nrows, const double* amp /* nrows x n */);
int yb_solution_set_receivers_weighted(yb_solution* s, const char* var, int64_t m, int64_t k, const int64_t* idx, const double* w,
                                       int64_t t0r, int64_t nrows_r);
/* Trilinear support of n positions of ndd (1-3) doubles each, in global index units (e.g. 511.25): k = 2^ndd entries per point,
 * idx_out n x k x ndd, w_out n x k.  Per dim d: i_d = floor(p_d), f_d = p_d - i_d.  Entry c (0 .. k-1) takes i_d + bit in dim d,
 * bit = (c >> (ndd - 1 - d)) & 1 (x varies slowest); its weight is ((1.0 * g_0) * g_1) * g_2 in double, left to right, with
 * g_d = bit ? f_d : 1.0 - f_d.  An integer position yields one entry of weight 1 and k - 1 of weight 0.  Non-finite positions
 * (and |p| >= 2^62) are refused.  Needs no solution and no device. */
int yb_points_trilinear(int ndd, int64_t n, const double* pos, int64_t* idx_out, double* w_out);

/* ---- slice recorders: boxes of a var recorded on the device inside run_solution() ----------------------------------
 * Replaces the host loop run_solution(t, t); get_elements_in_slice(frame, {u, first...}, {u, last...}) with one call, for receiver
 * planes, decimated snapshots and field dumps every k steps.  A recorder records the decimated box first[d], first[d] + stride[d],
 * ... <= last[d] (num_domain_dims GLOBAL domain indices each, inclusive, inside the overall domain: halo and pad cells are refused;
 * stride may be NULL for 1 in every dim; the phase comes from the global first, never from a rank's origin).  Whenever a run has
 * computed step u (after all its stages, and after that step's sources and receivers; u = t+1, or t-1 for a reverse solution),
 * if u - t0 is a multiple of `every` and r = (u - t0) / every is in [0, nrows): frame[r] = var(u, box) in the element type.
 * The var must have the step dim and every domain dim, no misc dim, and be written by a stage.  Each rank allocates nrows x its
 * OWNED part of the decimated box on the device: at this call on a prepared solution (which synchronizes its stream), otherwise
 * at prepare -- never in run_solution(); an allocation that fails is refused, naming the bytes.  Rows not recorded yet are 0.
 * Recorders persist across runs until cleared; *id (0, 1, ...) names this one.  While any is set every run takes one step per
 * launch (block_steps pairs resume once they are cleared); a rank grid whose halos are exchanged once per pair of steps
 * (block_steps=2 + mega_block_steps=2) refuses them.  Read-only option slice_launches: recording launches since prepare (one per
 * step in which some recorder of this rank has a row due, whatever the number of recorders). */
int yb_solution_add_slice(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                          int64_t t0, int64_t every, int64_t nrows, int64_t* id);
/* Copy the frames of recorder `id` into `out`: nrows x the full decimated box (extents (last - first) / stride + 1, domain dims in
 * order, the last fastest) of the solution's type; the points this rank does not own stay 0.  owned[] gets 1 per point of the
 * decimated box this rank records (0 elsewhere).  `out` may be NULL: then only the mask, which needs no device once the rank
 * geometry is known (plan_geometry). */
int yb_solution_get_slice_frames(yb_solution* s, int64_t id, void* out, uint8_t* owned);
int yb_solution_clear_slices(yb_solution* s);      /* remove every recorder and free its frames; ids restart at 0 */

/* ---- slice injectors: boxes written into a var on the device inside run_solution() ----------------------------------
 * The dual of a recorder, for plane-wave and areal sources, back-propagating a recorded plane, boundary replay and time-varying
 * Dirichlet data.  It replaces the host loop run_solution(t, t); get_elements_in_slice(box, {u, first...}, {u, last...});
 * box[::stride] = frame (or box[::stride] + frame); set_elements_in_slice(box) with one call, bit for bit.  The box (first, last,
 * stride), the window (t0, every, nrows) and the var rules are those of yb_solution_add_slice.  `frames` holds nrows x the
 * decimated box of the solution's element type, the last domain dim fastest; the call copies it.  Whenever a run has computed
 * step u (u = t+1, or t-1 for a reverse solution), if u - t0 is a multiple of `every` and r = (u - t0) / every is in [0, nrows),
 * then for every point pt of the decimated box:
 *   YB_INJECT_SET: var(u, pt) = frame[r][pt];
 *   YB_INJECT_ADD: var(u, pt) = T(var(u, pt) + frame[r][pt]), one add in the element type (add_to_element's rounding).
 * Within step u, after all its stages: the injectors in id order (where two on one var overlap, the later id wins or adds last),
 * then the sources, the receivers and the recorders, which so see the injection.  On a rank grid each rank writes its own part
 * of the box, and the var must be written by the last stage (as for sources); neighbours receive the values through that stage's
 * exchange.  Each rank keeps nrows x its own part on the device, allocated and uploaded at this call on a prepared solution
 * (which synchronizes its stream), otherwise at prepare -- never in run_solution().  While any injector is set every run takes
 * one step per launch (block_steps pairs resume once they are cleared); a fused-pair rank grid refuses them.  *id (0, 1, ...)
 * names the injector; ids are separate from the recorders'.  Read-only options: slice_injector_groups, the launch groups in order
 * (ids in a group separated by ',', groups by ';', e.g. "0,1;2": a group ends before an injector whose box meets that of an
 * earlier member on the same var); slice_injector_launches, injecting launches since prepare (one per group with a row due). */
enum { YB_INJECT_ADD = 0, YB_INJECT_SET = 1 };
int yb_solution_add_slice_injector(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                   int64_t t0, int64_t every, int64_t nrows, int mode, const void* frames, int64_t* id);
int yb_solution_clear_slice_injectors(yb_solution* s);   /* remove every injector and free its frames; ids restart at 0 */
/* An injector as yb_solution_add_slice_injector whose frames are those of recorder `src_id` of solution `src` (which may be `s`),
 * read on the device with no copy: row r reads recorder row reverse ? nrows - 1 - r : r, with this injector's nrows.  The
 * frames are shared as described at yb_solution_add_slice_correlator, with the same checks and the same ordering. */
int yb_solution_add_slice_injector_from(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                        int64_t t0, int64_t every, int64_t nrows, int mode, yb_solution* src, int64_t src_id, int reverse,
                                        int64_t* id);

/* ---- slice correlators: the imaging condition accumulated on the device inside run_solution() ----------------------------
 * For the adjoint run of a reverse-time shot: image(x) += S(x, u) * R(x, u) summed over the correlated steps, where S is the
 * forward wavefield kept as a recorder's frames and R the var.  It replaces the host loop run_solution(t, t);
 * get_elements_in_slice(box, {u, first...}, {u, last...}); image += frame[row] * box[::stride] with one call, bit for bit.  The
 * box (first, last, stride), the window (t0, every, nrows) and the var rules are those of yb_solution_add_slice.  The image is one
 * frame of the decimated box in the element type T, zeroed when it is allocated; each rank holds its own part.  Whenever a run
 * has computed step u, if u - t0 is a multiple of `every` and r = (u - t0) / every is in [0, nrows), then for every point pt:
 *   image[pt] = T(image[pt] + T(var(u, pt) * b[pt])), the product and the sum each rounded (no FMA),
 * where b = var(u) when `src` is NULL (autocorrelation: the source illumination), otherwise row reverse ? nrows - 1 - r : r of
 * recorder `src_id` of solution `src` (which may be `s`), as that row stands when the launch runs in stream order.  Within step
 * u: injectors, sources, receivers, recorders, then the correlators, all due ones in one launch.  Images accumulate across runs.
 * Frames shared from a recorder: the consumer holds a reference, so clear_slices on `src` or destroying `src` leaves it reading
 * the frames as they were.  Refused unless `src` has recorder src_id with this box and stride and at least nrows rows, the same
 * element bytes and domain dims, and (both with their rank geometry) the same overall domain, rank grid and rank index; then
 * unless `src` is prepared, so the frames exist; `reverse` is 0 or 1; a consumer planned before its prepare is checked again then,
 * with the device.  Between two solutions runs behave as if executed in the order the host enqueued them: a consumer's run waits
 * for the source's last run, and a source's run for the last runs of its consumers.  Images are allocated at this call on a
 * prepared solution (which synchronizes its stream), otherwise at prepare -- never in run_solution().  While any correlator is
 * set every run takes one step per launch; a fused-pair rank grid refuses them.  *id (0, 1, ...) names the correlator; ids are
 * separate from the recorders' and injectors'.  Read-only option slice_correlator_launches: correlating launches since prepare
 * (one per step in which some correlator of this rank has a row due, and a second right after it when a correlator of
 * yb_solution_add_slice_correlator_var has a row due in that step). */
int yb_solution_add_slice_correlator(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                     int64_t t0, int64_t every, int64_t nrows, yb_solution* src, int64_t src_id, int reverse, int64_t* id);
/* The image of correlator `id` as the whole decimated box in the solution's type (0 where this rank owns no point) and the owned
 * mask, as yb_solution_get_slice_frames with one row. */
int yb_solution_get_correlator_image(yb_solution* s, int64_t id, void* out, uint8_t* owned);
int yb_solution_clear_slice_correlators(yb_solution* s);   /* remove every correlator and free its image; ids restart at 0 */

/* A correlator as yb_solution_add_slice_correlator_typed whose b is var `src_var` of another prepared solution `src` on the same
 * device, read at the paired step: when row r is due at step u,
 *   image[pt] = I(image[pt] + var(u, pt) * src_var(src_t0 + (u - t0), pt)), rounded as yb_solution_add_slice_correlator_typed,
 * at the same global points.  For a reverse-time shot with no snapshots: `src` rebuilds the source wavefield backwards in time
 * beside the adjoint run `s`, and alternating one-step runs of the two enqueue with no host sync.  The two solutions may store
 * their vars differently (pads, halos, slot counts, spare temporal-tile slots, another stencil).  Ids, image, image types,
 * yb_solution_get_correlator_image, yb_solution_clear_slice_correlators and slice_correlator_launches are those of the other
 * correlators.  All due correlators of this call share one launch per step, right after the launch of the other correlators,
 * so a step in which both kinds are due takes two correlating launches.  Refused, naming the field, in this order: `src` is not another
 * solution; `src_var` is missing or breaks the var rules of yb_solution_add_slice; the element bytes differ; the domain dims
 * differ; (both with their rank geometry) the overall domain, rank grid or rank index differ; `src` is not prepared; the device
 * differs (a consumer planned before its prepare is checked again then).  Ordering: every run of `s` waits for `src`'s last run
 * and var-data writes, and every run or var-data write of `src` waits for the last run of `s`, so runs behave as if executed in
 * the order the host enqueued them.  Before a run of `s` enqueues anything, every due step u of it must pair with a step inside
 * the valid window of `src_var` as the host has enqueued `src` (yb_var_info first_valid_step .. last_valid_step); otherwise the
 * run is refused, naming the correlator, u, the paired step and the window, and changes nothing.  If `src` is destroyed, the
 * images stay readable and every run of `s` is refused until yb_solution_clear_slice_correlators. */
int yb_solution_add_slice_correlator_var(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                         int64_t t0, int64_t every, int64_t nrows, yb_solution* src, const char* src_var, int64_t src_t0,
                                         int image_type, int64_t* id);

/* ---- frame and image types of the slice calls ------------------------------------------------------------------------
 * A recorder's or a host-fed injector's frames are held in a frame type F, and a correlator's image in an image type I.
 * YB_TYPE_ELEM (the default of the untyped calls) is the solution's element type T, and leaves every bit, allocation, launch and
 * counter as the untyped call has them.  Allowed:
 *   fp32 solution: F in {float32, float16, bfloat16}, I in {float32, float64};
 *   fp64 solution: F in {float64, float32},           I = float64.
 * Every other combination is refused at the add call, naming the type and the element type.  Each narrowing is one IEEE
 * round-to-nearest-even conversion from T: finite values beyond F's range become +-inf, subnormal results are kept (the
 * conversions do not flush, though the engine runs fp32 arithmetic with FTZ), NaN stays NaN (payload unspecified).  Widening F
 * to T, and T to double, is exact.  float16 and bfloat16 elements cross this ABI as their 16-bit patterns (uint16_t). */
enum { YB_TYPE_ELEM = 0, YB_TYPE_F64 = 1, YB_TYPE_F32 = 2, YB_TYPE_F16 = 3, YB_TYPE_BF16 = 4 };
/* yb_solution_add_slice with frames of type `frame_type`: frame[r][pt] = N_F(var(u, pt)), nrows x the owned part x sizeof(F)
 * bytes per rank (the 64-bit byte-count refusal uses sizeof(F)); yb_solution_get_slice_frames copies out in F. */
int yb_solution_add_slice_typed(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                int64_t t0, int64_t every, int64_t nrows, int frame_type, int64_t* id);
/* yb_solution_add_slice_injector whose `frames` are nrows x the decimated box of type `frame_type`, widened exactly on the device:
 *   YB_INJECT_SET: var(u, pt) = T(frame[r][pt]);   YB_INJECT_ADD: var(u, pt) = T(var(u, pt) + T(frame[r][pt])), one add in T.
 * An injector or correlator fed from a recorder (yb_solution_add_slice_injector_from, yb_solution_add_slice_correlator with a
 * source) reads that recorder's frame type and takes none of its own. */
int yb_solution_add_slice_injector_typed(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                         int64_t t0, int64_t every, int64_t nrows, int mode, int frame_type, const void* frames, int64_t* id);
/* yb_solution_add_slice_correlator with an image of type `image_type` (own_elems x sizeof(I) bytes per rank); b is read in the
 * source recorder's frame type and widened exactly to T.  With I = T: image = T(image + T(var * b)) as the untyped call.  With
 * I = float64 in an fp32 solution: image = image + double(var) * double(b), the product exact and the sum rounded in double
 * (an autocorrelation: image + double(v) * double(v)).  yb_solution_get_correlator_image copies out in I. */
int yb_solution_add_slice_correlator_typed(yb_solution* s, const char* var, const int64_t* first, const int64_t* last, const int64_t* stride,
                                           int64_t t0, int64_t every, int64_t nrows, yb_solution* src, int64_t src_id, int reverse,
                                           int image_type, int64_t* id);
/* The frame type of recorder `id` and the image type of correlator `id`, resolved (never YB_TYPE_ELEM): the layout
 * yb_solution_get_slice_frames and yb_solution_get_correlator_image write. */
int yb_solution_get_slice_frame_type(yb_solution* s, int64_t id, int* type);
int yb_solution_get_correlator_image_type(yb_solution* s, int64_t id, int* type);

/* ---- multi-GPU halo exchange, one process per GPU (replaces exchange_halos, halo.cpp:80-491) --- */
/* Each rank exports an opaque blob (CUDA IPC handles of its var storage + sync flags), the
 * launcher all-gathers the blobs (torch.distributed / MPI / files) and imports every
 * neighbour's blob.  After that the boundary kernels write halos straight into the peers' HBM
 * over NVLink; no further host communication is needed. */
int yb_halo_export_size(const yb_solution* s, size_t* nbytes);
int yb_halo_export(yb_solution* s, void* blob, size_t nbytes);
int yb_halo_import(yb_solution* s, int64_t peer_rank_linear, const void* blob, size_t nbytes);
int yb_halo_finalize(yb_solution* s);              /* after all imports: ready to run */
int yb_exchange_halos(yb_solution* s);             /* yk_solution::exchange_halos (public API) */

/* ---- job rendezvous without MPI or torch (replaces the MPI set-up of setup.cpp:169-524 and the harness's
 *      yk_env::global_barrier / sum_over_ranks, yask_kernel_api.hpp:238-293) ---------------------------------------
 * One process per GPU on one node; the ranks meet in a POSIX shared-memory mailbox named after `job_key` (NULL:
 * YASK_JOB_ID, else MASTER_ADDR:MASTER_PORT + the launcher's pid).  yb_comm_env_* read the rank / world size / local
 * rank a launcher exported (YASK_*, torchrun's RANK/WORLD_SIZE/LOCAL_RANK, Open MPI, PMI, Slurm). */
int yb_comm_env_rank(void);
int yb_comm_env_world(void);
int yb_comm_env_local_rank(void);
int yb_comm_init(int rank, int world, const char* job_key);
int yb_comm_rank(void);
int yb_comm_world(void);
int yb_comm_barrier(void);
int yb_comm_allgather(const void* mine, size_t nbytes, void* all /* world * nbytes */);
int yb_comm_sum_i64(int64_t v, int64_t* out);
int yb_comm_max_f64(double v, double* out);
int yb_comm_finalize(void);
/* export -> all-gather through the communicator -> import every neighbour -> finalize, for a prepared multi-rank solution
 * whose rank-grid position matches this process's job rank (row-major over the domain dims, x slowest). */
int yb_halo_connect(yb_solution* s);

#ifdef __cplusplus
}
#endif
#endif /* YASK_B200_H */
