// r2x_stripes.cu -- sorting-based stripe removal of a projection stack (r2x_remove_stripes, include/r2x.h states the
// model; r2_gaussian_b200/stripes.py is the caller).
//
// Pass A (stripes_sort_kernel): a CTA owns one detector row and a tile of TW columns.  It reads each view's TW columns
// as one coalesced segment, builds (key << 32 | v) words in shared memory -- unique, so any sort of them is stable --,
// pads each column to P = next power of two >= n with ~0 (above every real word: v < 2^16), bitonic-sorts the TW
// columns together and writes the sorted keys (uint32) and views (uint16) rank-major, [H][n][W].  TW P = min(32 P, 8192)
// words, 64 KiB at most, so three CTAs fit an SM at any n up to R2X_STRIPES_MAX_VIEWS.  The steps j >= 16 of a stage
// run through shared memory, the steps j < 16 on 16 consecutive words per thread in registers.  Word i of column cl
// sits at cl P + (i ^ (((i >> 4) ^ cl) & 15 & (P - 1))): the swizzle spreads over the banks both a view's TW words
// (global load and store) and the 16-word groups of a warp's threads (register steps).
// Pass B (stripes_median_kernel): a CTA owns one (row, rank) and 256 columns.  It stages the tile's keys and the
// reflected halo, each thread finds the rank-h key of its window by counting, and writes its value to
// out[pi(k, c), r, c].  The CTAs of one row run together, so a view's row of out is assembled in L2 before it leaves.
// Pass A reads every row of `in` before pass B writes `out`, which is what makes out == in safe.  No atomics.
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_common.cuh"

namespace r2x {
namespace {

constexpr int SORT_THREADS = 256;
constexpr int SORT_WORDS = 8192;            // TW * P, 64 KiB of shared memory
constexpr int SORT_MAX_TW = 32;
constexpr int SORT_BLOCKS_PER_SM = 3;
constexpr int MED_THREADS = 256;            // = columns per pass-B tile
constexpr int MED_BLOCKS_PER_SM = 8;

__device__ __forceinline__ uint32_t stripe_key(uint32_t u) { return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ uint32_t stripe_unkey(uint32_t k) { return (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k; }

struct StripeGeom {
    int n, H, W, h;
    int P, logP, TW, logTW, tilesA, tilesB;
};

__device__ __forceinline__ int swz(int cl, int P, int i) { return cl * P + (i ^ (((i >> 4) ^ cl) & 15 & (P - 1))); }

__device__ __forceinline__ void cmp_swap(unsigned long long& a, unsigned long long& b, bool up) {
    if ((a > b) == up) {
        const unsigned long long t = a;
        a = b;
        b = t;
    }
}

// the bitonic steps j < SORT_GROUP of stages k_lo .. k_hi, each thread on SORT_GROUP consecutive words of a column held
// in registers (a whole column when P < SORT_GROUP): one shared-memory round trip instead of one per step
constexpr int SORT_GROUP = 16;
__device__ __forceinline__ void sort_register_steps(unsigned long long* sw, int P, int logP, int E, int k_lo, int k_hi) {
    const int G = P < SORT_GROUP ? P : SORT_GROUP;
    for (int g = threadIdx.x; g < E / G; g += SORT_THREADS) {
        const int cl = (g * G) >> logP, i0 = (g * G) & (P - 1);
        unsigned long long w[SORT_GROUP];
#pragma unroll
        for (int q = 0; q < SORT_GROUP; ++q)
            if (q < G) w[q] = sw[swz(cl, P, i0 + q)];
        for (int k = k_lo; k <= k_hi; k <<= 1) {
#pragma unroll
            for (int j = SORT_GROUP / 2; j >= 1; j >>= 1) {
                if (j <= (k >> 1)) {
#pragma unroll
                    for (int q = 0; q < SORT_GROUP; ++q)
                        if (!(q & j) && (q | j) < G) cmp_swap(w[q], w[q | j], ((i0 | q) & k) == 0);
                }
            }
        }
#pragma unroll
        for (int q = 0; q < SORT_GROUP; ++q)
            if (q < G) sw[swz(cl, P, i0 + q)] = w[q];
    }
    __syncthreads();
}

__global__ void __launch_bounds__(SORT_THREADS) stripes_sort_kernel(StripeGeom g, const float* __restrict__ in,
                                                                    uint32_t* __restrict__ keys,
                                                                    uint16_t* __restrict__ views) {
    extern __shared__ unsigned long long sw[];
    const int P = g.P, TW = g.TW, E = TW * P;
    const long long HW = (long long)g.H * g.W;
    const long long total = (long long)g.H * g.tilesA;
    const uint32_t* src = reinterpret_cast<const uint32_t*>(in);
    for (long long work = blockIdx.x; work < total; work += gridDim.x) {
        const int r = (int)(work / g.tilesA);
        const int c0 = (int)(work - (long long)r * g.tilesA) * TW;
        for (int e = threadIdx.x; e < E; e += SORT_THREADS) {
            const int v = e >> g.logTW, cl = e & (TW - 1);
            unsigned long long w = ~0ull;
            if (v < g.n && c0 + cl < g.W)
                w = ((unsigned long long)stripe_key(src[(size_t)v * HW + (size_t)r * g.W + c0 + cl]) << 32) |
                    (unsigned)v;
            sw[swz(cl, P, v)] = w;
        }
        __syncthreads();
        // bitonic sort of each P-long column, ascending; pairs never leave their column (j < P, columns P-aligned).
        // Steps j >= SORT_GROUP go through shared memory, the rest of each stage in registers.
        if (P > 1) sort_register_steps(sw, P, g.logP, E, 2, P < SORT_GROUP ? P : SORT_GROUP);
        for (int k = 2 * SORT_GROUP; k <= P; k <<= 1) {
            for (int j = k >> 1; j >= SORT_GROUP; j >>= 1) {
                for (int t = threadIdx.x; t < (E >> 1); t += SORT_THREADS) {
                    const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                    const int cl = lo >> g.logP, i = lo & (P - 1);
                    const int a = swz(cl, P, i), b = swz(cl, P, i + j);
                    const unsigned long long x = sw[a], y = sw[b];
                    if ((x > y) == ((i & k) == 0)) {            // k == P: every column ascending
                        sw[a] = y;
                        sw[b] = x;
                    }
                }
                __syncthreads();
            }
            sort_register_steps(sw, P, g.logP, E, k, k);
        }
        const size_t base = (size_t)r * g.n * g.W;
        for (int e = threadIdx.x; e < g.n * TW; e += SORT_THREADS) {
            const int k = e >> g.logTW, cl = e & (TW - 1);
            if (c0 + cl < g.W) {
                const unsigned long long w = sw[swz(cl, P, k)];
                const size_t o = base + (size_t)k * g.W + c0 + cl;
                keys[o] = (uint32_t)(w >> 32);
                views[o] = (uint16_t)w;
            }
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(MED_THREADS) stripes_median_kernel(StripeGeom g, const uint32_t* __restrict__ keys,
                                                                     const uint16_t* __restrict__ views,
                                                                     float* __restrict__ out) {
    __shared__ uint32_t sk[MED_THREADS + R2X_STRIPES_MAX_SIZE - 1];
    const int h = g.h, K = 2 * h + 1;
    const long long HW = (long long)g.H * g.W;
    const long long total = (long long)g.H * g.n * g.tilesB;
    uint32_t* dst = reinterpret_cast<uint32_t*>(out);
    for (long long work = blockIdx.x; work < total; work += gridDim.x) {
        const long long rk = work / g.tilesB;               // r * n + k
        const int c0 = (int)(work - rk * g.tilesB) * MED_THREADS;
        const int tw = min(MED_THREADS, g.W - c0);
        const uint32_t* row = keys + (size_t)rk * g.W;
        for (int i = threadIdx.x; i < tw + 2 * h; i += MED_THREADS) {
            int j = c0 - h + i;
            j = j < 0 ? -j - 1 : (j >= g.W ? 2 * g.W - 1 - j : j);
            sk[i] = row[j];
        }
        __syncthreads();
        const int c = threadIdx.x;
        if (c < tw) {
            const uint32_t* win = sk + c;
            uint32_t med = win[h];
            for (int m = 0; m < K; ++m) {                   // the key with <= h smaller and > h not larger
                const uint32_t x = win[m];
                int lt = 0, le = 0;
                for (int i = 0; i < K; ++i) {
                    lt += win[i] < x;
                    le += win[i] <= x;
                }
                if (lt <= h && h < le) {
                    med = x;
                    break;
                }
            }
            const long long r = rk / g.n;
            const int v = views[(size_t)rk * g.W + c0 + c];
            dst[(size_t)v * HW + (size_t)r * g.W + c0 + c] = stripe_unkey(med);
        }
        __syncthreads();
    }
}

int ilog2(int x) {
    int l = 0;
    while ((1 << l) < x) ++l;
    return l;
}

bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + nb && y < x + na;
}

}  // namespace
}  // namespace r2x

extern "C" {

size_t r2x_remove_stripes_scratch_bytes(int n, int H, int W) {
    if (n < 1 || n > R2X_STRIPES_MAX_VIEWS || H < 1 || W < 1 || (long long)H * W >= (1LL << 31)) return 0;
    return (size_t)6 * n * H * W;
}

int r2x_remove_stripes(void* stream, int n, int H, int W, int K, const float* in, float* out, void* scratch,
                       size_t scratch_bytes) {
    using namespace r2x;
    if (!in || !out || !scratch) return fail_msg(R2X_ERR_INVALID, "r2x_remove_stripes: bad pointer (NULL)");
    if (n < 1 || n > R2X_STRIPES_MAX_VIEWS)
        return fail_msg(R2X_ERR_INVALID, "r2x_remove_stripes: bad n (views must be in [1, R2X_STRIPES_MAX_VIEWS = 8192])");
    if (H < 1 || W < 1) return fail_msg(R2X_ERR_INVALID, "r2x_remove_stripes: bad shape (H, W >= 1)");
    if ((long long)H * W >= (1LL << 31)) return fail_msg(R2X_ERR_INVALID, "r2x_remove_stripes: bad shape (H * W must be < 2^31)");
    if (K < 1 || K > R2X_STRIPES_MAX_SIZE || K % 2 == 0)
        return fail_msg(R2X_ERR_INVALID, "r2x_remove_stripes: bad K (must be odd, 1 <= K <= 255)");
    const int h = K / 2;
    if (h > W) return fail_msg(R2X_ERR_INVALID, "r2x_remove_stripes: bad K (h = (K - 1) / 2 must be <= W)");
    const size_t need = r2x_remove_stripes_scratch_bytes(n, H, W);
    if (scratch_bytes < need) return fail_msg(R2X_ERR_INVALID, "r2x_remove_stripes: bad scratch (too small)");
    if ((uintptr_t)scratch % 16 != 0) return fail_msg(R2X_ERR_INVALID, "r2x_remove_stripes: bad scratch (not 16-byte aligned)");
    const size_t bytes = (size_t)n * H * W * sizeof(float);
    if (in != out && overlaps(in, bytes, out, bytes))
        return fail_msg(R2X_ERR_INVALID, "r2x_remove_stripes: bad pointers (out overlaps in without being in)");
    if (overlaps(scratch, need, in, bytes) || overlaps(scratch, need, out, bytes))
        return fail_msg(R2X_ERR_INVALID, "r2x_remove_stripes: bad scratch (overlaps in or out)");

    StripeGeom g;
    g.n = n;
    g.H = H;
    g.W = W;
    g.h = h;
    g.logP = ilog2(n);
    g.P = 1 << g.logP;
    g.TW = g.P * SORT_MAX_TW <= SORT_WORDS ? SORT_MAX_TW : SORT_WORDS / g.P;
    g.logTW = ilog2(g.TW);
    g.tilesA = (W + g.TW - 1) / g.TW;
    g.tilesB = (W + MED_THREADS - 1) / MED_THREADS;
    uint32_t* keys = static_cast<uint32_t*>(scratch);
    uint16_t* views = reinterpret_cast<uint16_t*>(keys + (size_t)n * H * W);

    int sms = 0;
    R2X_CUDA_OK(sm_count(&sms));
    const size_t smem = (size_t)g.TW * g.P * sizeof(unsigned long long);
    R2X_CUDA_OK(cudaFuncSetAttribute(stripes_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long totalA = (long long)H * g.tilesA, capA = (long long)sms * SORT_BLOCKS_PER_SM;
    stripes_sort_kernel<<<(unsigned)(totalA < capA ? totalA : capA), SORT_THREADS, smem, (cudaStream_t)stream>>>(
        g, in, keys, views);
    R2X_CUDA_OK(cudaGetLastError());
    const long long totalB = (long long)H * n * g.tilesB, capB = (long long)sms * MED_BLOCKS_PER_SM;
    stripes_median_kernel<<<(unsigned)(totalB < capB ? totalB : capB), MED_THREADS, 0, (cudaStream_t)stream>>>(
        g, keys, views, out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
