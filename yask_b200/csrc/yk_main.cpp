// Command-line harness for one solution: the yask_b200 counterpart of the reference's kernel driver
// (/root/reference/src/kernel/yask_main.cpp), built as bin/yask_kernel.<stencil>.b200.exe.  It uses ONLY the
// public kernel API (yask_kernel_api.hpp), accepts the reference's command lines (its CPU-tuning options are
// recognised and ignored by apply_command_line_options) and prints the same "key: value" report lines
// (yask_main.cpp:513-536, soln_apis.cpp:455-470), so log scrapers written for the reference keep working.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <iomanip>
#include <iostream>
#include <cstdint>
#include <sstream>
#include <vector>

#include "yask_kernel_api.hpp"

using namespace yask;

namespace {

const char* DIV = "───────────────────────────────────────────────────────────\n";

// engineering notation as the reference prints it ("3.12G", "17.2M"; common_utils.cpp make_num_str)
std::string num_str(double v) {
    static const char* sfx[] = {"", "K", "M", "G", "T", "P"};
    int k = 0;
    double a = std::fabs(v);
    while (a >= 1000. && k < 5) { a /= 1000.; v /= 1000.; k++; }
    std::ostringstream os;
    os << std::setprecision(4) << v << sfx[k];
    return os.str();
}

struct Trial { idx_t nsteps; double secs, pts_ps, reads_ps, writes_ps, flops; };

void usage(const char* exe, yk_solution_ptr soln) {
    std::cout << "Usage: " << exe << " [options]\n"
              << " -h | -help              this text\n"
              << " -trial_steps | -dt <n>  steps per performance trial (default 50)\n"
              << " -num_trials | -t <n>    number of trials (default 3)\n"
              << " -msg_rank <r>           rank that prints (default 0); a job of several ranks is started once per rank\n"
              << "                         (RANK / WORLD_SIZE / LOCAL_RANK as torchrun, mpirun or srun export them)\n"
              << " -warmup_steps <n>       untimed steps before the trials (default 5)\n"
              << " -init_val <x>           value every var is initialised to (default 0.1, var k gets x*(1+k/16))\n"
              << " -validate               cross-check on the device: sweep kernels (temporal tile included) against the one-thread-per-point\n"
              << "                         kernels of a second solution, every written var, element for element\n"
              << " -[no-]pre_auto_tune     time the engine's launch variants before the trials and keep the fastest (default on; 1 rank)\n"
              << "Solution options:\n" << soln->get_command_line_help();
}

}  // namespace

int main(int argc, char** argv) {
    try {
        yk_factory kfac;
        auto env = kfac.new_env();
        auto soln = kfac.new_solution(env);
        idx_t trial_steps = 50, num_trials = 3, warmup_steps = 5, msg_rank = 0;
        double init_val = 0.1, init_seed = 0.1;
        bool pre_auto_tune = true;
        bool validate = false;
        idx_t mega_block_steps = 0;      // -Mbt: steps per halo exchange of a rank grid's temporal tile (reported as num-wave-front-steps)
        // harness options first; everything else goes to the solution (as yask_main.cpp:199-259 does)
        string_vec rest;
        for (int i = 1; i < argc; i++) {
            std::string a = argv[i];
            auto val = [&]() -> std::string {
                if (i + 1 >= argc) { std::cerr << "Error: no argument for option '" << a << "'\n"; std::exit(1); }
                return argv[++i];
            };
            if (a == "-h" || a == "-help" || a == "--help") { usage(argv[0], soln); return 0; }
            // (-t and -dt are the reference's deprecated aliases of -num_trials and -trial_steps, yask_main.cpp:107-119)
            else if (a == "-trial_steps" || a == "-dt") trial_steps = atoll(val().c_str());
            else if (a == "-num_trials" || a == "-t") num_trials = atoll(val().c_str());
            else if (a == "-warmup_steps") warmup_steps = atoll(val().c_str());
            else if (a == "-msg_rank") msg_rank = atoll(val().c_str());
            else if (a == "-init_val") init_val = atof(val().c_str());
            else if (a == "-init_seed") init_seed = atof(val().c_str());   // spread of the per-var values (the reference seeds its varying sequence with it)
            else if (a == "-trial_time" || a == "-sleep") val();      // reference options with no meaning here
            else if (a == "-validate" || a == "-v") validate = true;
            else if (a == "-pre_auto_tune") pre_auto_tune = true;          // yask_main.cpp:53: on by default
            else if (a == "-no-pre_auto_tune") pre_auto_tune = false;
            else if (a == "-Mbt") { rest.push_back(a); rest.push_back(val()); mega_block_steps = atoll(rest.back().c_str()); }   // also the solution's
            else rest.push_back(a);
        }
        // only one rank of a job prints (yask_main.cpp -msg_rank)
        const int nranks = env->get_num_ranks(), my_rank = env->get_rank_index();
        std::ostringstream quiet;
        std::ostream& out = my_rank == msg_rank ? std::cout : quiet;
        out << "YASK-compatible kernel harness, solution '" << soln->get_name() << "', target " << soln->get_target()
            << ", " << soln->get_element_bytes() << "-byte elements, API version " << kfac.get_version_string() << "\n";
        std::string unused = soln->apply_command_line_options(rest);
        if (!unused.empty()) { std::cerr << "Error: extraneous parameter(s): '" << unused << "'; run with '-help' for usage.\n"; return 1; }
        if (trial_steps < 1 || num_trials < 1) { std::cerr << "Error: -trial_steps and -num_trials must be positive.\n"; return 1; }

        soln->prepare_solution();
        auto dims = soln->get_domain_dim_names();
        idx_t pts = 1;
        out << DIV << "Problem:\n";
        std::ostringstream gs, ls;
        for (auto& d : dims) {
            gs << (gs.str().empty() ? "" : " * ") << d << "=" << soln->get_overall_domain_size(d);
            ls << (ls.str().empty() ? "" : " * ") << d << "=" << soln->get_rank_domain_size(d);
            pts *= soln->get_rank_domain_size(d);
        }
        out << " global-domain-size:     " << gs.str() << "\n"
                  << " local-domain-size:      " << ls.str() << "\n"
                  << " num-ranks:              " << env->get_num_ranks() << "\n"
                  << " num-points-per-step:    " << num_str(double(pts)) << "\n";
        // the keys the reference's log tooling collects (utils/lib/YaskUtils.pm @log_keys; wording of setup.cpp:613-650,
        // soln_apis.cpp:155), so that utils/bin/yask_log_to_csv.pl reads these logs like its own
        idx_t alloc_bytes = 0;
        for (auto& v : soln->get_vars()) alloc_bytes += v->get_num_storage_bytes();
        out << "Num MPI ranks:             " << nranks << "\n"
            << "Domain size in this rank (points):          " << num_str(double(pts)) << "\n"
            << "Total allocation in this rank:              " << num_str(double(alloc_bytes)) << "B\n"
            << "Overall problem size in " << nranks << " rank(s) (points): " << num_str(double(env->sum_over_ranks(pts))) << "\n"
            << "Other settings:\n"
            << " yask-version:           " << kfac.get_version_string() << "\n"
            << " target:                 " << soln->get_target() << "\n"
            << " stencil-name:           " << soln->get_name() << "\n"
            << " stencil-description:    " << soln->get_description() << "\n"
            << " element-size:           " << soln->get_element_bytes() << "B\n"
            << " num-temporal-block-steps:  " << std::max<idx_t>(1, soln->get_block_size(soln->get_step_dim_name())) << "\n"
            << " num-wave-front-steps:      " << std::max<idx_t>(1, mega_block_steps) << "\n";

        // data: every var constant, slightly different per var (the reference's init_same pattern)
        int k = 0;
        auto var_val = [&](int kk) { return init_val * (1.0 + double(kk) * init_seed / 1.6); };
        for (auto& v : soln->get_vars()) v->set_all_elements_same(var_val(k++));

        // iso3dfd runs on the hand-written engine (option -kernel) in fp32 and, in fp64, at the radii its fp64 sweep serves;
        // fp64 at radius 3 and 8 is emitter-generated.  iso3dfd_sponge runs on it too, except at its default radius (8 in fp32, 6 in
        // fp64); the hand-written engine is the one that takes option -kernel.
        const bool sponge = soln->get_name() == "iso3dfd_sponge";
        bool hand_iso = soln->get_name() == "iso3dfd" || sponge;
        if (validate && hand_iso && (soln->get_element_bytes() == 8 || sponge)) {
            try {
                kfac.new_solution(env, soln)->apply_command_line_options("-kernel direct");
            } catch (yask_exception&) {
                hand_iso = false;
            }
        }
        if (validate && !hand_iso) {
            // Emitter-generated solutions: every stencil part has two independent launch forms -- the TMA sweep kernels and the
            // one-thread-per-point direct kernels (-gen_sweep 0), the role the reference's scalar run_ref() plays for its
            // vectorised code (/root/reference/src/kernel/lib/context.cpp:85-217, yask_main.cpp:562-644).  Same data, same steps,
            // every written var compared element for element.
            auto other = kfac.new_solution(env, soln);
            other->apply_command_line_options("-gen_sweep 0");
            other->prepare_solution();
            const bool f64 = soln->get_element_bytes() == 8;
            const std::string sd = soln->get_step_dim_name();
            std::vector<std::pair<yk_var_ptr, yk_var_ptr>> pairs;
            k = 0;
            for (auto& v : soln->get_vars()) {
                auto w = other->get_var(v->get_name());
                w->set_all_elements_same(var_val(k++));
                pairs.emplace_back(v, w);
            }
            // ripple on every var that has the step dim (the ones the solution updates), identical in both solutions: a
            // deterministic +-5 % pattern over the rank's domain box at its first valid step
            auto box_of = [&](yk_var_ptr v, idx_t t, idx_t_vec& f, idx_t_vec& l) {
                size_t n = 1;
                f.clear(); l.clear();
                for (auto& d : v->get_dim_names()) {
                    if (d == sd) { f.push_back(t); l.push_back(t); }
                    else if (std::find(dims.begin(), dims.end(), d) != dims.end()) { f.push_back(v->get_first_rank_domain_index(d)); l.push_back(v->get_last_rank_domain_index(d)); }
                    else { f.push_back(v->get_first_misc_index(d)); l.push_back(v->get_last_misc_index(d)); }
                    n *= size_t(l.back() - f.back() + 1);
                }
                return n;
            };
            k = 0;
            for (auto& pr : pairs) {
                const double base = var_val(k++);
                if (!pr.first->is_dim_used(sd) || pr.first->is_fixed_size()) continue;
                idx_t_vec f, l;
                const size_t n = box_of(pr.first, pr.first->get_first_valid_step_index(), f, l);
                std::vector<double> bd(f64 ? n : 0);
                std::vector<float> bf(f64 ? 0 : n);
                uint64_t h = 0x9E3779B97F4A7C15ull * uint64_t(k + 1 + 1000 * my_rank);
                for (size_t i = 0; i < n; i++) {
                    h ^= h << 13; h ^= h >> 7; h ^= h << 17;
                    const double val = base * (1.0 + 0.05 * (double(h >> 40) / double(1 << 24) - 0.5));
                    if (f64) bd[i] = val; else bf[i] = float(val);
                }
                for (auto* v : {&pr.first, &pr.second}) {
                    if (f64) (*v)->set_elements_in_slice(bd.data(), n, f, l); else (*v)->set_elements_in_slice(bf.data(), n, f, l);
                }
            }
            env->global_barrier();
            const idx_t vsteps = std::min<idx_t>(trial_steps, 4);
            soln->run_solution(0, vsteps - 1);
            other->run_solution(0, vsteps - 1);
            idx_t bad = 0, compared = 0;
            for (auto& pr : pairs) {
                if (!pr.first->is_dim_used(sd) || pr.first->is_fixed_size()) continue;
                idx_t_vec f, l;
                const size_t n = box_of(pr.first, pr.first->get_last_valid_step_index(), f, l);
                if (f64) {
                    std::vector<double> a(n), b(n);
                    pr.first->get_elements_in_slice(a.data(), n, f, l);
                    pr.second->get_elements_in_slice(b.data(), n, f, l);
                    for (size_t i = 0; i < n; i++) bad += !(a[i] == b[i]) && !(a[i] != a[i] && b[i] != b[i]);
                } else {
                    std::vector<float> a(n), b(n);
                    pr.first->get_elements_in_slice(a.data(), n, f, l);
                    pr.second->get_elements_in_slice(b.data(), n, f, l);
                    for (size_t i = 0; i < n; i++) bad += !(a[i] == b[i]) && !(a[i] != a[i] && b[i] != b[i]);
                }
                compared += idx_t(n);
            }
            bad = env->sum_over_ranks(bad);
            compared = env->sum_over_ranks(compared);
            other->end_solution();
            out << DIV << (bad ? "TEST FAILED: " : "TEST PASSED: ") << bad << " mismatch(es) in " << compared
                << " element(s) between the sweep kernels and the direct kernels over " << vsteps << " step(s).\n";
            soln->end_solution();
            env->finalize();
            if (!bad) out << "YASK DONE\n";
            return bad ? 1 : 0;
        }
        if (validate) {
            // the same steps with the sweep kernel and with the one-thread-per-point kernel must agree bit for bit
            auto p = soln->get_var("p");
            auto other = kfac.new_solution(env, soln);
            other->apply_command_line_options("-kernel direct");
            other->prepare_solution();
            k = 0;
            for (auto& v : other->get_vars()) v->set_all_elements_same(var_val(k++));
            // iso3dfd_sponge: a ripple in [0.95, 1] along each sponge factor (a function of the global index, the same in both
            // solutions), so that a factor taken from the wrong row, plane or vector shows up -- constant factors would only
            // check the rounding order of the three multiplies
            if (sponge) {
                for (const char* name : {"cr_x", "cr_y", "cr_z"}) {
                    yk_var_ptr vars[2] = {soln->get_var(name), other->get_var(name)};
                    const std::string d = vars[0]->get_dim_names()[0];
                    const idx_t_vec f{vars[0]->get_first_rank_domain_index(d)}, l{vars[0]->get_last_rank_domain_index(d)};
                    const size_t n = size_t(l[0] - f[0] + 1);
                    std::vector<double> bd(n);
                    std::vector<float> bf(n);
                    for (size_t i = 0; i < n; i++) {
                        bd[i] = 0.95 + 0.05 * double((f[0] + idx_t(i)) * 7919 % 101) / 100.0;
                        bf[i] = float(bd[i]);
                    }
                    for (auto& v : vars) {
                        if (soln->get_element_bytes() == 8) v->set_elements_in_slice(bd.data(), n, f, l);
                        else v->set_elements_in_slice(bf.data(), n, f, l);
                    }
                }
            }
            // a bump in the middle so that the field is not constant
            idx_t_vec mid;
            mid.push_back(0);
            for (auto& d : dims) mid.push_back(soln->get_overall_domain_size(d) / 2);
            bool mine = true;     // the bump belongs to the rank whose domain holds it
            for (size_t d = 0; d < dims.size(); d++)
                mine = mine && mid[d + 1] >= p->get_first_rank_domain_index(dims[d]) && mid[d + 1] <= p->get_last_rank_domain_index(dims[d]);
            if (mine) {
                p->set_element(1.0, mid);
                other->get_var("p")->set_element(1.0, mid);
            }
            env->global_barrier();
            const idx_t vsteps = std::min<idx_t>(trial_steps, 4);
            soln->run_solution(0, vsteps - 1);
            other->run_solution(0, vsteps - 1);
            auto q = other->get_var("p");
            idx_t tl = p->get_last_valid_step_index();
            idx_t_vec f{tl}, l{tl};
            for (auto& d : dims) { f.push_back(p->get_first_rank_domain_index(d)); l.push_back(p->get_last_rank_domain_index(d)); }
            const size_t np = size_t(pts);
            idx_t bad = 0;
            if (soln->get_element_bytes() == 8) {
                std::vector<double> a(np), b(np);
                p->get_elements_in_slice(a.data(), a.size(), f, l);
                q->get_elements_in_slice(b.data(), b.size(), f, l);
                for (size_t i = 0; i < a.size(); i++) bad += a[i] != b[i];
            } else {
                std::vector<float> a(np), b(np);
                p->get_elements_in_slice(a.data(), a.size(), f, l);
                q->get_elements_in_slice(b.data(), b.size(), f, l);
                for (size_t i = 0; i < a.size(); i++) bad += a[i] != b[i];
            }
            bad = env->sum_over_ranks(bad);
            other->end_solution();
            out << DIV << (bad ? "TEST FAILED: " : "TEST PASSED: ") << bad << " mismatch(es) between the sweep and the direct kernel over "
                      << vsteps << " step(s).\n";
            soln->end_solution();
            env->finalize();
            if (!bad) out << "YASK DONE\n";
            return bad ? 1 : 0;
        }

        // The reference tunes before the trials unless told not to (yask_main.cpp:53,440-478).  Here the tuner times the engine's
        // launch variants -- sweep tile / chunk length, direct vs sweep kernels, one or two steps per sweep where a temporal tile
        // exists -- and keeps the fastest; every variant computes the same bits.  Single-rank runs only.
        if (pre_auto_tune && nranks == 1) {
            out << DIV << "Running the auto-tuner before the trials (-no-pre_auto_tune skips it)...\n";
            soln->run_auto_tuner_now(false);
            k = 0;
            for (auto& v : soln->get_vars()) v->set_all_elements_same(var_val(k++));      // the tuner does not preserve var contents
        }
        if (warmup_steps > 0) soln->run_solution(0, warmup_steps - 1);
        idx_t first_t = warmup_steps;
        std::vector<Trial> trials;
        for (idx_t tr = 0; tr < num_trials; tr++) {
            soln->clear_stats();
            env->global_barrier();
            soln->run_solution(first_t, first_t + trial_steps - 1);
            first_t += trial_steps;
            auto st = soln->get_stats();      // waits for the device
            Trial t;
            t.nsteps = st->get_num_steps_done();
            // the ranks advance in lock-step (halo epochs); report the mean of their device times
            t.secs = nranks > 1 ? double(env->sum_over_ranks(idx_t(st->get_elapsed_secs() * 1e9))) * 1e-9 / nranks : st->get_elapsed_secs();
            t.pts_ps = double(st->get_num_elements()) * double(t.nsteps) / t.secs;
            t.writes_ps = double(st->get_num_writes_done()) / t.secs;
            t.reads_ps = 0.;
            t.flops = double(st->get_est_fp_ops_done()) / t.secs;
            trials.push_back(t);
            out << DIV << "Trial " << (tr + 1) << ":\n"
                      << " num-steps-done:               " << t.nsteps << "\n"
                      << " elapsed-time (sec):           " << num_str(t.secs) << "\n"
                      << " throughput (num-writes/sec):  " << num_str(t.writes_ps) << "\n"
                      << " throughput (est-FLOPS):       " << num_str(t.flops) << "\n"
                      << " throughput (num-points/sec):  " << num_str(t.pts_ps) << "\n";
        }
        std::vector<Trial> sorted = trials;
        std::sort(sorted.begin(), sorted.end(), [](const Trial& a, const Trial& b) { return a.pts_ps > b.pts_ps; });
        const Trial& best = sorted.front();
        const Trial& mid = sorted[sorted.size() / 2];
        double sum = 0, sum2 = 0;
        for (auto& t : trials) { sum += t.pts_ps; sum2 += t.pts_ps * t.pts_ps; }
        const double n = double(trials.size());
        const double sd = n > 2 ? std::sqrt(std::max(0., (sum2 - sum * sum / n) / (n - 1.))) : 0.;
        out << DIV << "Throughput stats across trials:\n"
                  << " num-trials:                          " << trials.size() << "\n"
                  << " min-throughput (num-points/sec):     " << num_str(sorted.back().pts_ps) << "\n"
                  << " max-throughput (num-points/sec):     " << num_str(best.pts_ps) << "\n"
                  << " ave-throughput (num-points/sec):     " << num_str(sum / n) << "\n"
                  << " std-dev-throughput (num-points/sec): " << num_str(sd) << "\n"
                  << DIV << "Performance stats of best trial:\n"
                  << " best-num-steps-done:              " << best.nsteps << "\n"
                  << " best-elapsed-time (sec):          " << num_str(best.secs) << "\n"
                  << " best-throughput (num-writes/sec): " << num_str(best.writes_ps) << "\n"
                  << " best-throughput (est-FLOPS):      " << num_str(best.flops) << "\n"
                  << " best-throughput (num-points/sec): " << num_str(best.pts_ps) << "\n"
                  << DIV << "Performance stats of 50th-percentile trial:\n"
                  << " mid-num-steps-done:               " << mid.nsteps << "\n"
                  << " mid-elapsed-time (sec):           " << num_str(mid.secs) << "\n"
                  << " mid-throughput (num-writes/sec):  " << num_str(mid.writes_ps) << "\n"
                  << " mid-throughput (est-FLOPS):       " << num_str(mid.flops) << "\n"
                  << " mid-throughput (num-points/sec):  " << num_str(mid.pts_ps) << "\n";
        soln->end_solution();
        env->finalize();
        out << "YASK DONE\n";
        return 0;
    } catch (yask_exception& e) {
        std::cerr << "YASK kernel harness: " << e.get_message() << "\n";
        return 1;
    }
}
