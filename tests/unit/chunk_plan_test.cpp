// TEST ONLY: x-chunk planning of the iso3dfd sweep launches (yask_b200/csrc/yb_chunk_plan.h, chunk_count / chunk_partition),
// with the bounds the one-step sweep and the temporal tile pass.
#include <cstdio>

#include "../../yask_b200/csrc/yb_chunk_plan.h"

#define CHECK(c) do { if (!(c)) { printf("FAILED: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

constexpr int MAX_CHUNKS = 40;      // ISO_MAX_CHUNKS / TT_MAX_CHUNKS

int main() {
    int x0[MAX_CHUNKS], len[MAX_CHUNKS], dir[MAX_CHUNKS];
    const int caps[] = {1, 7, 132, 148}, lxs[] = {0, 3, 256, 1024};
    for (int nx = 1; nx <= 600; nx += 7)
        for (int ntile : {1, 5, 64, 600})
            for (int gmax : caps)
                for (int lx : lxs)
                    for (int R = 1; R <= 8; R++)
                        for (int cfg = 0; cfg < 5; cfg++) {
                            // cfg 0, 1: no signal (box from plane 0 / plane 5); 2, 3, 4: in-kernel signal with a lower, an upper
                            // or both x neighbours (whole rank domains of at least 4R planes only, as the sweep asks)
                            const bool sig = cfg >= 2, lo = sig && cfg != 3, hi = sig && cfg != 2;
                            if (sig && nx < 4 * R) continue;
                            const int64_t b = cfg == 1 ? 5 : 0;
                            const int min_nc = (lo && hi) ? 2 : 1;
                            const int64_t max_nc = std::min<int64_t>(MAX_CHUNKS, sig ? nx / R : nx);
                            const int nc = yb::chunk_count(nx, ntile, gmax, lx, 2 * R, min_nc, max_nc);
                            CHECK(nc >= min_nc && nc <= max_nc);
                            if (lx > 0) {       // lx honoured within the bounds
                                const int64_t want = (nx + lx - 1) / lx;
                                CHECK(nc == std::max<int64_t>(min_nc, std::min<int64_t>(want, max_nc)));
                            }
                            const int nfirst = yb::chunk_partition(b, nx, nc, lo, hi, x0, len, dir);
                            // the chunks cover [b, b + nx) exactly, with lengths that differ by at most one plane
                            bool seen[2048] = {};
                            int lmin = nx, lmax = 0;
                            for (int k = 0; k < nc; k++) {
                                const int first = dir[k] > 0 ? x0[k] : x0[k] - len[k] + 1;
                                CHECK(dir[k] == 1 || dir[k] == -1);
                                for (int x = first; x < first + len[k]; x++) {
                                    CHECK(x >= b && x < b + nx && !seen[x]);
                                    seen[x] = true;
                                }
                                lmin = std::min(lmin, len[k]);
                                lmax = std::max(lmax, len[k]);
                            }
                            for (int64_t x = b; x < b + nx; x++) CHECK(seen[x]);
                            CHECK(lmax - lmin <= 1 && lmin >= 1);
                            if (!sig) {
                                CHECK(nfirst == 0);
                                for (int k = 0; k < nc; k++) CHECK(dir[k] == 1 && x0[k] == (k == 0 ? b : x0[k - 1] + len[k - 1]));
                                continue;
                            }
                            // signalling: every chunk is at least R planes long; the boundary chunks come first, the last chunk
                            // of the domain is swept downwards from plane nx - 1
                            CHECK(lmin >= R);
                            CHECK(nfirst == int(lo) + int(hi));
                            int k = 0;
                            if (lo) { CHECK(x0[k] == 0 && dir[k] == 1); k++; }
                            if (hi) { CHECK(x0[k] == nx - 1 && dir[k] == -1); k++; }
                            for (; k < nc; k++) CHECK(dir[k] == 1 && (!lo || x0[k] > 0) && (!hi || x0[k] + len[k] < nx));
                        }
    // temporal tile: warm-up 4R, no signal; the cost model prefers fewer, longer chunks as the warm-up grows
    for (int R = 1; R <= 2; R++) {
        const int nc = yb::chunk_count(1024, 64 * 8, 132, 0, 4 * R, 1, MAX_CHUNKS);
        CHECK(nc >= 1 && nc <= MAX_CHUNKS);
        CHECK(yb::chunk_partition(0, 1024, nc, false, false, x0, len, nullptr) == 0);
        CHECK(x0[0] == 0 && x0[nc - 1] + len[nc - 1] == 1024);
    }
    CHECK(yb::chunk_count(1024, 1, 132, 0, 4, 1, MAX_CHUNKS) == MAX_CHUNKS);    // one tile: as many chunks as the grid can use
    CHECK(yb::chunk_count(1024, 132 * 40, 132, 0, 4, 1, MAX_CHUNKS) == 1);      // a full grid of tiles: no splitting
    printf("OK\n");
    return 0;
}
