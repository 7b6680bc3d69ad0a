// r2x_detector.cu -- the horizontal detector offset on the device (r2x_detector_offset_apply / _grad, include/r2x.h).
// A detector shifted by s pixels along u moves every projected 2-D mean by s pixels and nothing else: rays, conics and
// mu stay those of the nominal geometry.  With ndc2Pix(x) = ((x + 1) W - 1) / 2, the shift is the full projection
// whose x row (entries 0, 4, 8, 12 of the 16 floats as the torch tensors store them) gains (2 s / W) times its w row
// (entries 3, 7, 11, 15): x/w + 2 s / W.  Apply evaluates each entry in float64 and rounds it once; a zero increment is
// taken as -0.0, so s = 0 returns the matrices bit for bit (as r2x_pose_apply does).
// The gradient, with cull, radii and tile rectangles held fixed as for every per-Gaussian gradient, is
//   dL/ds = sum over views and Gaussians of dL/dpix_x = (2 / W) sum dL_dmean2D.x
// (dL_dmean2D is dL/dndc, g2x = ... 0.5 W in raster_gauss_bwd_kernel).  Two launches: a fixed grid of float64 block
// partial sums over contiguous chunks, then one block that adds the partials in order -- no atomics, bitwise
// reproducible, the result written (not accumulated).
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_common.cuh"

namespace r2x {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxBlocks = 1024;
constexpr long long kPerBlock = 8 * kThreads;   // at least this many elements per stage-one block

// one thread per (view, entry): x row += (2 s / W) w row, every other entry copied
__global__ void __launch_bounds__(kThreads) detector_offset_apply_kernel(const float* __restrict__ offset, int W, int n,
                                                                         const float* __restrict__ full,
                                                                         float* __restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 16 * n) return;
    const int k = e & 15;
    if ((k & 3) != 0) {
        out[e] = full[e];
        return;
    }
    const double d = 2.0 * (double)offset[0] / (double)W * (double)full[e + 3];
    out[e] = (float)((double)full[e] + (d == 0.0 ? -0.0 : d));
}

__host__ __device__ inline int grad_blocks(long long N) {
    const long long b = (N + kPerBlock - 1) / kPerBlock;
    return (int)(b < 1 ? 1 : (b > kMaxBlocks ? kMaxBlocks : b));
}

// block b sums the x components of elements [b chunk, (b + 1) chunk) of the N = n_views P rows of dL_dmean2D
__global__ void __launch_bounds__(kThreads) detector_offset_partial_kernel(long long N, long long chunk,
                                                                           const float* __restrict__ g,
                                                                           double* __restrict__ partial) {
    __shared__ double s[kThreads];
    const long long lo = (long long)blockIdx.x * chunk;
    const long long hi = lo + chunk < N ? lo + chunk : N;
    double acc = 0.0;
    for (long long i = lo + threadIdx.x; i < hi; i += kThreads) acc += (double)g[3 * i];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int h = kThreads / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = s[0];
}

__global__ void __launch_bounds__(kThreads) detector_offset_final_kernel(int nb, int W, const double* __restrict__ partial,
                                                                         float* __restrict__ out) {
    __shared__ double s[kThreads];
    double acc = 0.0;
    for (int i = threadIdx.x; i < nb; i += kThreads) acc += partial[i];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int h = kThreads / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = (float)(2.0 / (double)W * s[0]);
}

}  // namespace
}  // namespace r2x

extern "C" {

int r2x_detector_offset_apply(void* stream, const float* offset, int W, int n_views, const float* full_proj,
                              float* out_full_proj) {
    using namespace r2x;
    if (!offset || !full_proj || !out_full_proj) return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_apply: null pointer");
    if (W <= 0) return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_apply: W must be positive");
    if (n_views <= 0 || n_views > (1 << 26))
        return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_apply: n_views out of range");
    const int nblk = (16 * n_views + kThreads - 1) / kThreads;
    detector_offset_apply_kernel<<<nblk, kThreads, 0, (cudaStream_t)stream>>>(offset, W, n_views, full_proj,
                                                                              out_full_proj);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

size_t r2x_detector_offset_grad_scratch_bytes(int P, int n_views) {
    if (P < 0 || n_views <= 0) return 0;
    return (size_t)r2x::grad_blocks((long long)P * n_views) * sizeof(double);
}

int r2x_detector_offset_grad(void* stream, int P, int n_views, int W, const float* dL_dmean2D, float* dL_doffset,
                             void* scratch, size_t scratch_bytes) {
    using namespace r2x;
    if (!dL_doffset || !scratch || (P > 0 && !dL_dmean2D))
        return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_grad: null pointer");
    if (P < 0) return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_grad: P must be non-negative");
    if (n_views <= 0) return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_grad: n_views must be positive");
    if (W <= 0) return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_grad: W must be positive");
    const long long N = (long long)P * n_views;
    const int nb = grad_blocks(N);
    if (scratch_bytes < (size_t)nb * sizeof(double))
        return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_grad: scratch smaller than "
                                         "r2x_detector_offset_grad_scratch_bytes(P, n_views)");
    const long long chunk = (N + nb - 1) / nb;
    cudaStream_t st = (cudaStream_t)stream;
    detector_offset_partial_kernel<<<nb, kThreads, 0, st>>>(N, chunk, dL_dmean2D, (double*)scratch);
    R2X_CUDA_OK(cudaGetLastError());
    detector_offset_final_kernel<<<1, kThreads, 0, st>>>(nb, W, (const double*)scratch, dL_doffset);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
