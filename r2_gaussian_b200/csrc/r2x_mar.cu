// r2x_mar.cu -- metal-trace inpainting of a projection stack (r2x_mar_inpaint, include/r2x.h states the model;
// r2_gaussian_b200/mar.py is the caller).
//
// One CTA per (view, row).  The row is staged in shared memory -- p, the clamped prior Pe when there is one, the raw
// trace flags and then their exclusive prefix count S, and the dilated trace t -- and each thread owns one run of
// K = ceil(W / MAR_THREADS) consecutive columns:
//   1. coalesced loads of p, m (t0 = m > tau, into S) and P (Pe = P > eps ? P : eps);
//   2. S = exclusive prefix count of t0 (per-thread run sums, one block scan); t[c] = S[hi + 1] - S[lo] > 0 with
//      [lo, hi] = [c - d, c + d] clipped to the row, so the dilation is exact and O(W) whatever d is;
//   3. per run, the last non-trace column and the first; a block max-scan of the former gives each run the nearest
//      non-trace column to its left, a reverse block min-scan of the latter the nearest to its right;
//   4. a left-to-right walk of the run records l for every trace column (in S's storage, which is dead by then), a
//      right-to-left walk finds r and writes the inpainted value over p's stage.  Only trace columns are written and
//      l, r are never trace columns, so no thread reads a value another thread changes;
//   5. coalesced stores of the row and the trace.
// The whole row is read before any of it is written, so out == p is safe.  No atomics: bitwise reproducible.
#include <cmath>
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_common.cuh"

namespace r2x {
namespace {

constexpr int MAR_THREADS = 256;
constexpr int MAR_WARPS = MAR_THREADS / 32;

struct MaxOp {
    __device__ int operator()(int a, int b) const { return a > b ? a : b; }
};
struct MinOp {
    __device__ int operator()(int a, int b) const { return a < b ? a : b; }
};
struct SumOp {
    __device__ int operator()(int a, int b) const { return a + b; }
};

// exclusive scan of one int per thread in thread order (REV: in reverse thread order) under an associative and
// commutative op; every thread of the CTA must call it
template <bool REV, typename Op>
__device__ __forceinline__ int block_scan_exclusive(int x, int ident, Op op, int* wsum) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = REV ? __shfl_down_sync(0xFFFFFFFFu, inc, o) : __shfl_up_sync(0xFFFFFFFFu, inc, o);
        if (REV ? lane + o < 32 : lane >= o) inc = op(inc, y);
    }
    if (lane == (REV ? 0 : 31)) wsum[warp] = inc;
    __syncthreads();
    int pre = ident;
#pragma unroll
    for (int w = 0; w < MAR_WARPS; ++w)
        if (REV ? w > warp : w < warp) pre = op(pre, wsum[w]);
    int exc = REV ? __shfl_down_sync(0xFFFFFFFFu, inc, 1) : __shfl_up_sync(0xFFFFFFFFu, inc, 1);
    if (lane == (REV ? 31 : 0)) exc = ident;
    __syncthreads();                                        // wsum is reused by the next scan
    return op(pre, exc);
}

template <bool PRIOR>
__global__ void __launch_bounds__(MAR_THREADS) mar_inpaint_kernel(int W, const float* p, const float* __restrict__ m,
                                                                  float tau, int d, const float* __restrict__ P,
                                                                  float eps, float* out, uint8_t* __restrict__ trace) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int wsum[MAR_WARPS];
    float* sp = reinterpret_cast<float*>(smem);                       // [W]   p, then the output
    float* sPe = sp + W;                                              // [W]   Pe (PRIOR only)
    int* sS = reinterpret_cast<int*>(sPe + (PRIOR ? W : 0));          // [W+1] t0, then S, then l
    uint8_t* st = reinterpret_cast<uint8_t*>(sS + W + 1);             // [W]   t
    const size_t row = (size_t)blockIdx.x * (size_t)W;
    const int tid = threadIdx.x;

    for (int c = tid; c < W; c += MAR_THREADS) {
        sp[c] = p[row + c];
        sS[c] = m[row + c] > tau ? 1 : 0;
        if (PRIOR) {
            const float v = P[row + c];
            sPe[c] = v > eps ? v : eps;
        }
    }
    __syncthreads();

    const int K = (W + MAR_THREADS - 1) / MAR_THREADS;
    const int c0 = min(tid * K, W), c1 = min(c0 + K, W);
    int tot = 0;
    for (int c = c0; c < c1; ++c) tot += sS[c];
    const int base = block_scan_exclusive<false>(tot, 0, SumOp(), wsum);   // syncs: every t0 read before S is written
    int run = base;
    for (int c = c0; c < c1; ++c) {
        const int f = sS[c];
        sS[c] = run;
        run += f;
    }
    if (tid == MAR_THREADS - 1) sS[W] = run;
    __syncthreads();

    int last_good = -1, first_good = W;
    for (int c = c0; c < c1; ++c) {
        const int lo = max(c - d, 0), hi = min(c + d, W - 1);              // d <= W: no overflow
        const bool t = sS[hi + 1] - sS[lo] > 0;
        st[c] = t ? 1 : 0;
        if (!t) {
            last_good = c;
            if (first_good == W) first_good = c;
        }
    }
    const int left = block_scan_exclusive<false>(last_good, -1, MaxOp(), wsum);   // syncs: S read before l is written
    const int right = block_scan_exclusive<true>(first_good, W, MinOp(), wsum);

    int l = left;
    for (int c = c0; c < c1; ++c) {
        if (!st[c]) l = c;
        else sS[c] = l;
    }
    int r = right;
    for (int c = c1 - 1; c >= c0; --c) {
        if (!st[c]) {
            r = c;
            continue;
        }
        const int lc = sS[c];
        float v;
        if (lc >= 0 && r < W) {
            const float ql = PRIOR ? __fdiv_rn(sp[lc], sPe[lc]) : sp[lc];
            const float qr = PRIOR ? __fdiv_rn(sp[r], sPe[r]) : sp[r];
            const float s = __fdiv_rn((float)(c - lc), (float)(r - lc));
            v = __fadd_rn(ql, __fmul_rn(s, __fsub_rn(qr, ql)));
        } else if (lc >= 0) {
            v = PRIOR ? __fdiv_rn(sp[lc], sPe[lc]) : sp[lc];
        } else if (r < W) {
            v = PRIOR ? __fdiv_rn(sp[r], sPe[r]) : sp[r];
        } else {
            if (!PRIOR) continue;                                          // a whole-trace row without a prior: p
            v = 1.0f;
        }
        sp[c] = PRIOR ? __fmul_rn(v, sPe[c]) : v;
    }
    __syncthreads();

    for (int c = tid; c < W; c += MAR_THREADS) {
        out[row + c] = sp[c];
        if (trace) trace[row + c] = st[c];
    }
}

size_t mar_smem_bytes(int W, bool prior) {
    return (size_t)W * sizeof(float) * (prior ? 2 : 1) + (size_t)(W + 1) * sizeof(int) + (size_t)W;
}

bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + nb && y < x + na;
}

}  // namespace
}  // namespace r2x

extern "C" {

int r2x_mar_inpaint(void* stream, int n, int H, int W, const float* p, const float* m, float tau, int d,
                    const float* P, float eps, float* out, uint8_t* trace) {
    using namespace r2x;
    if (!p || !m || !out) return fail_msg(R2X_ERR_INVALID, "r2x_mar_inpaint: bad pointer (NULL p, m or out)");
    if (n < 1 || H < 1 || W < 1) return fail_msg(R2X_ERR_INVALID, "r2x_mar_inpaint: bad shape (n, H, W >= 1)");
    if ((long long)n * H >= (1LL << 31)) return fail_msg(R2X_ERR_INVALID, "r2x_mar_inpaint: bad shape (n * H must be < 2^31)");
    if (W > R2X_MAR_MAX_W) return fail_msg(R2X_ERR_INVALID, "r2x_mar_inpaint: bad shape (W must be <= R2X_MAR_MAX_W = 16384)");
    if (!isfinite(tau)) return fail_msg(R2X_ERR_INVALID, "r2x_mar_inpaint: bad tau (must be finite)");
    if (!(isfinite(eps) && eps > 0.0f)) return fail_msg(R2X_ERR_INVALID, "r2x_mar_inpaint: bad eps (must be finite and > 0)");
    if (d < 0) return fail_msg(R2X_ERR_INVALID, "r2x_mar_inpaint: bad d (must be >= 0)");
    const size_t bytes = (size_t)n * H * W * sizeof(float), tbytes = (size_t)n * H * W;
    if (out != p && overlaps(out, bytes, p, bytes))
        return fail_msg(R2X_ERR_INVALID, "r2x_mar_inpaint: bad pointers (out overlaps p without being p)");
    if (overlaps(out, bytes, m, bytes) || (P && overlaps(out, bytes, P, bytes)))
        return fail_msg(R2X_ERR_INVALID, "r2x_mar_inpaint: bad pointers (out overlaps m or P)");
    if (trace && (overlaps(trace, tbytes, p, bytes) || overlaps(trace, tbytes, m, bytes) ||
                  (P && overlaps(trace, tbytes, P, bytes)) || overlaps(trace, tbytes, out, bytes)))
        return fail_msg(R2X_ERR_INVALID, "r2x_mar_inpaint: bad pointers (trace overlaps p, m, P or out)");

    const int dd = d < W ? d : W;                                          // a wider dilation changes nothing
    const size_t smem = mar_smem_bytes(W, P != nullptr);
    const unsigned grid = (unsigned)((long long)n * H);
    if (P) {
        R2X_CUDA_OK(cudaFuncSetAttribute(mar_inpaint_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        mar_inpaint_kernel<true><<<grid, MAR_THREADS, smem, (cudaStream_t)stream>>>(W, p, m, tau, dd, P, eps, out, trace);
    } else {
        R2X_CUDA_OK(cudaFuncSetAttribute(mar_inpaint_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        mar_inpaint_kernel<false><<<grid, MAR_THREADS, smem, (cudaStream_t)stream>>>(W, p, m, tau, dd, P, eps, out, trace);
    }
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
