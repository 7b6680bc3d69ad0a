// Host-side check of the work-plan arithmetic in r2_gaussian_b200/csrc/r2x_binning.cuh (plan_chunk_for, plan_slice are
// __host__ __device__): the chunk policy per consumer and the equal-slice cut of a tile list.  Built (cross-compiled for
// sm_90a, host code run) by tests/test_plan_cpu.py; no GPU needed.
#include <cstdio>
#include <cstdlib>
#include "../../r2_gaussian_b200/csrc/r2x_binning.cuh"

using namespace r2x;

#define CHECK(cond)                                                         \
    do {                                                                    \
        if (!(cond)) {                                                      \
            printf("plan_check: FAILED %s (line %d)\n", #cond, __LINE__);   \
            return 1;                                                       \
        }                                                                   \
    } while (0)

int main() {
    // rasterizer: the staging buffer holds PLAN_CHUNK records, so that is the chunk whatever the instance count
    for (uint32_t R : {0u, 1u, 1000u, 1062151u, 40000000u}) CHECK(plan_chunk_for(R, 0, PLAN_CHUNK) == (uint32_t)PLAN_CHUNK);
    // voxelizer: a multiple of PLAN_CHUNK in [PLAN_CHUNK, VOX_CHUNK_CAP], non-decreasing in R, about R / 4096
    uint32_t prev = 0;
    for (uint32_t R = 0; R < 40000000u; R += 37717u) {
        const uint32_t c = plan_chunk_for(R, 0, VOX_CHUNK_CAP);
        CHECK(c % PLAN_CHUNK == 0 && c >= (uint32_t)PLAN_CHUNK && c <= (uint32_t)VOX_CHUNK_CAP);
        CHECK(c >= prev);
        CHECK(c == (uint32_t)VOX_CHUNK_CAP || (unsigned long long)c * 4096ull + 4096ull * PLAN_CHUNK > R);
        prev = c;
    }
    CHECK(plan_chunk_for(150000u, 0, VOX_CHUNK_CAP) == 256u);        // a TV crop keeps thousands of small items
    CHECK(plan_chunk_for(10730134u, 0, VOX_CHUNK_CAP) == 2816u);     // the 256^3 query: one item per tile (avg 327 / tile)
    // the experiment override is clamped to what the consumer can take
    CHECK(plan_chunk_for(5u, 128, PLAN_CHUNK) == 128u && plan_chunk_for(5u, 100000, PLAN_CHUNK) == (uint32_t)PLAN_CHUNK);
    CHECK(plan_chunk_for(5u, 1, VOX_CHUNK_CAP) == (uint32_t)PLAN_MIN_CHUNK && plan_chunk_for(5u, 100000, VOX_CHUNK_CAP) == (uint32_t)VOX_CHUNK_CAP);
    // equal slices: contiguous, in order, covering the list, sizes within one of each other, never above the chunk
    srand(7);
    for (int trial = 0; trial < 20000; ++trial) {
        const uint32_t start = (uint32_t)rand() % 100000u, len = (uint32_t)rand() % 20000u;
        const uint32_t C = 64u * (1u + (uint32_t)rand() % 64u);
        const int nch = len ? (int)((len - 1) / C) + 1 : 1;
        uint32_t at = start;
        int lo = 1 << 30, hi = 0;
        for (int c = 0; c < nch; ++c) {
            uint32_t b; int n;
            plan_slice(make_uint2(start, start + len), c, nch, b, n);
            CHECK(b == at && n >= 0 && (uint32_t)n <= C);
            at += (uint32_t)n;
            lo = n < lo ? n : lo; hi = n > hi ? n : hi;
        }
        CHECK(at == start + len && hi - lo <= 1);
    }
    printf("plan_check: ok\n");
    return 0;
}
