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
// r2x_detector_offset_cost measures the offset from the projections instead: the mismatch of conjugate rays (the model
// is in include/r2x.h) for K candidate shifts, float64 samples, the same two-stage fixed-order reduction per candidate.
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

// ---- the conjugate-ray cost of candidate shifts (r2x_detector_offset_cost) ----------------------------------------
// Stage one: block (b, k) sums the samples [b chunk, (b + 1) chunk) of candidate k, thread-strided, then a fixed tree;
// stage two: one thread per candidate adds its nb chunk sums in order.  The chunk count shrinks as K grows so that the
// K nb partials stay within kCostMaxPartials.
constexpr int kCostThreads = 256;
constexpr int kCostMaxChunks = 256;
constexpr long long kCostPerBlock = 16 * kCostThreads;   // at least this many samples per stage-one block
constexpr long long kCostMaxPartials = 1LL << 20;
constexpr int kCostMaxK = 65535;                          // gridDim.y
constexpr long long kCostMaxSamples = 1LL << 62;

struct CostPartial {
    double num, den;
    long long count;
};

__host__ __device__ inline int cost_chunks(long long T, int K) {
    long long cap = kCostMaxPartials / (K > 0 ? K : 1);
    cap = cap < 1 ? 1 : (cap > kCostMaxChunks ? kCostMaxChunks : cap);
    const long long b = (T + kCostPerBlock - 1) / kCostPerBlock;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// the float64 value of `row` at fractional column c by linear interpolation; false when c is outside [0, W - 1]
__device__ __forceinline__ bool cost_lerp(const float* __restrict__ row, int W, double c, double& v) {
    if (!(c >= 0.0 && c <= (double)(W - 1))) return false;   // NaN fails too
    const double f0 = floor(c);
    const int c0 = (int)f0;
    const double f = c - f0;
    const double a = (double)row[c0];
    v = f > 0.0 ? (1.0 - f) * a + f * (double)row[c0 + 1] : a;
    return true;
}

// value of view `img` at row r0 (+ fraction fr) and column c
__device__ __forceinline__ bool cost_sample(const float* __restrict__ img, int W, int r0, double fr, double c,
                                            double& v) {
    double lo, hi;
    if (!cost_lerp(img + (long long)r0 * W, W, c, lo)) return false;
    if (fr > 0.0) {
        cost_lerp(img + (long long)(r0 + 1) * W, W, c, hi);
        lo = (1.0 - fr) * lo + fr * hi;
    }
    v = lo;
    return true;
}

__global__ void __launch_bounds__(kCostThreads) detector_offset_cost_partial_kernel(
    int mode, int H, int W, const float* __restrict__ projs, const int* __restrict__ pair_views,
    const double* __restrict__ pair_dbeta, double fan, double mid_row, int row_lo, int n_rows, long long T,
    long long chunk, const double* __restrict__ sigma, CostPartial* __restrict__ partial) {
    __shared__ double s_num[kCostThreads], s_den[kCostThreads];
    __shared__ long long s_cnt[kCostThreads];
    const int k = blockIdx.y;
    const double sg = sigma[k];
    const double centre = 0.5 * (double)(W - 1);
    const long long lo = (long long)blockIdx.x * chunk;
    const long long hi = lo + chunk < T ? lo + chunk : T;
    const long long per_pair = (long long)n_rows * W;
    const long long view = (long long)H * W;
    // cone beam: the mid-plane row, the same for every sample
    const int mr0 = (int)floor(mid_row);
    const double mfr = mid_row - (double)mr0;
    double num = 0.0, den = 0.0;
    long long cnt = 0;
    for (long long q = lo + threadIdx.x; q < hi; q += kCostThreads) {
        long long p;
        int r0;
        double fr, ci, cj;
        if (mode == 0) {
            p = q / per_pair;
            const long long rem = q - p * per_pair;
            const int m = (int)(rem % W);
            r0 = row_lo + (int)(rem / W);
            fr = 0.0;
            ci = (double)m + sg;
            cj = (double)(W - 1 - m) + sg;
        } else {
            p = q;
            const double t = fan * tan(0.5 * (M_PI - pair_dbeta[p]));
            r0 = mr0;
            fr = mfr;
            ci = centre + t + sg;
            cj = centre - t + sg;
        }
        const float* vi = projs + (long long)pair_views[2 * p] * view;
        const float* vj = projs + (long long)pair_views[2 * p + 1] * view;
        double a, b;
        if (cost_sample(vi, W, r0, fr, ci, a) && cost_sample(vj, W, r0, fr, cj, b)) {
            const double d = a - b;
            num += d * d;
            den += a * a + b * b;
            ++cnt;
        }
    }
    s_num[threadIdx.x] = num;
    s_den[threadIdx.x] = den;
    s_cnt[threadIdx.x] = cnt;
    __syncthreads();
    for (int h = kCostThreads / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) {
            s_num[threadIdx.x] += s_num[threadIdx.x + h];
            s_den[threadIdx.x] += s_den[threadIdx.x + h];
            s_cnt[threadIdx.x] += s_cnt[threadIdx.x + h];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[(long long)k * gridDim.x + blockIdx.x] = {s_num[0], s_den[0], s_cnt[0]};
}

__global__ void __launch_bounds__(kCostThreads) detector_offset_cost_final_kernel(int K, int nb,
                                                                                  const CostPartial* __restrict__ partial,
                                                                                  double* __restrict__ num,
                                                                                  double* __restrict__ den,
                                                                                  long long* __restrict__ count) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    double n = 0.0, d = 0.0;
    long long c = 0;
    for (int b = 0; b < nb; ++b) {
        const CostPartial& s = partial[(long long)k * nb + b];
        n += s.num;
        d += s.den;
        c += s.count;
    }
    num[k] = n;
    den[k] = d;
    count[k] = c;
}

// samples per candidate, or -1 when the sizes are out of range
inline long long cost_samples(int mode, int W, int n_pairs, int n_rows) {
    if (W <= 0 || n_pairs <= 0 || n_rows <= 0) return -1;
    const long long per_pair = mode == 0 ? (long long)n_rows * W : 1;
    if ((long long)n_pairs > kCostMaxSamples / per_pair) return -1;
    return (long long)n_pairs * per_pair;
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

size_t r2x_detector_offset_cost_scratch_bytes(int mode, int W, int n_pairs, int n_rows, int K) {
    using namespace r2x;
    const long long T = cost_samples(mode, W, n_pairs, n_rows);
    if (T < 0 || K <= 0 || K > kCostMaxK) return 0;
    return (size_t)K * (size_t)cost_chunks(T, K) * sizeof(CostPartial);
}

int r2x_detector_offset_cost(void* stream, int mode, int N, int H, int W, const float* projs, int n_pairs,
                             const int* pair_views, const double* pair_dbeta, double DSD, double du, double t_v,
                             int row_lo, int n_rows, int K, const double* sigma, double* num, double* den,
                             long long* count, void* scratch, size_t scratch_bytes) {
    using namespace r2x;
    if (!projs || !pair_views || !sigma || !num || !den || !count || !scratch || (mode == 1 && !pair_dbeta))
        return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: null pointer");
    if (mode != 0 && mode != 1) return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: mode must be 0 or 1");
    if (N <= 0 || H <= 0 || W <= 0)
        return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: N, H and W must be positive");
    if (n_pairs <= 0) return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: no conjugate pairs");
    if (K <= 0 || K > kCostMaxK)
        return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: K must be in [1, 65535]");
    double fan = 0.0, mid_row = 0.0;
    if (mode == 0) {
        if (n_rows <= 0 || row_lo < 0 || row_lo > H - n_rows)
            return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: rows [row_lo, row_lo + n_rows) outside the image");
    } else {
        if (n_rows != 1) return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: cone beam samples one row");
        if (!(DSD > 0.0 && du > 0.0 && DSD < 1e300 && du < 1e300))
            return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: DSD and du must be finite and positive");
        mid_row = 0.5 * (double)(H - 1) + t_v;
        if (!(mid_row >= 0.0 && mid_row <= (double)(H - 1)))
            return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: the mid-plane row (H - 1) / 2 + t_v lies "
                                             "outside the image");
        fan = DSD / du;
    }
    const long long T = cost_samples(mode, W, n_pairs, n_rows);
    if (T < 0) return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: too many samples");
    const int nb = cost_chunks(T, K);
    if (scratch_bytes < (size_t)K * nb * sizeof(CostPartial))
        return fail_msg(R2X_ERR_INVALID, "r2x_detector_offset_cost: scratch smaller than "
                                         "r2x_detector_offset_cost_scratch_bytes");
    const long long chunk = (T + nb - 1) / nb;
    cudaStream_t st = (cudaStream_t)stream;
    detector_offset_cost_partial_kernel<<<dim3(nb, K), kCostThreads, 0, st>>>(
        mode, H, W, projs, pair_views, pair_dbeta, fan, mid_row, row_lo, n_rows, T, chunk, sigma,
        (CostPartial*)scratch);
    R2X_CUDA_OK(cudaGetLastError());
    detector_offset_cost_final_kernel<<<(K + kCostThreads - 1) / kCostThreads, kCostThreads, 0, st>>>(
        K, nb, (const CostPartial*)scratch, num, den, count);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
