// Kernels around the hot path that the reference runs as ~40 small torch ops per iteration (SURVEY §8(f) rank 2):
//   * image loss  = w_l1 * mean|x - y| + w_dssim * (1 - mean SSIM(x, y)), forward AND gradient in two launches
//     (r2_gaussian/utils/loss_utils.py:37-104, train.py:118-127): 11-tap Gaussian window (sigma 1.5), zero
//     padding, C1 = 0.01^2, C2 = 0.03^2, single channel;
//   * 3-D total variation of a volume, forward and gradient in one launch (loss_utils.py:19-34, train.py:128-143);
//   * one fused Adam step over all parameter groups (torch.optim.Adam semantics as used at
//     gaussian_model.py:216, eps = 1e-15, no weight decay).
// All reductions are two-stage in a fixed order: results are bitwise reproducible.
#include <cmath>
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_binning.cuh"
#include "r2x_common.cuh"

namespace r2x {

// ------------------------------------------------------------------------------------------------
// SSIM + L1
// ------------------------------------------------------------------------------------------------
constexpr int LT = 16;            // output tile edge
constexpr int LH = 5;             // window half width
constexpr int LE = LT + 2 * LH;   // 26: tile + halo

struct SsimWindow { float g[11]; };

// The reference's 1-D window, bit for bit: torch.Tensor([exp(-(x-5)^2 / (2*1.5^2)) for x in range(11)]) divided by
// its float32 .sum() (loss_utils.py:45-52).  Hard-coded because torch's vectorised sum does not round like a
// sequential one (3.7592328 vs 3.7592325): a window that sums to 1 + 7e-8 instead of 1 - 3e-8 biases
// sigma^2 = E[x^2] - mu^2 by ~1e-7 mu^2, visible in the mean SSIM at 3e-5.  The 2-D window of the reference is
// the float32 outer product of this vector; applying it separably differs from that by rounding only.
static SsimWindow make_window() {
    static const float g[11] = {0x1.0d956cp-10f, 0x1.f1fe02p-8f, 0x1.26eb18p-5f, 0x1.bff0fep-4f, 0x1.b43c3ep-3f,
                                0x1.106560p-2f,  0x1.b43c3ep-3f, 0x1.bff0fep-4f, 0x1.26eb18p-5f, 0x1.f1fe02p-8f,
                                0x1.0d956cp-10f};
    SsimWindow w;
    for (int i = 0; i < 11; ++i) w.g[i] = g[i];
    return w;
}

// Stage 1: per pixel SSIM statistics -> the three maps the gradient needs + per-CTA partial sums.
// The *_body functions are shared by the one-image kernels and the batched ones (*_views_kernel: blockIdx.z or, for the
// reduction, blockIdx.x is the image, whose pointers are shifted before the body runs).
__device__ __forceinline__ void ssim_stats_body(int H, int W, const float* __restrict__ x, const float* __restrict__ y,
                                                const SsimWindow& win,
                                                float* __restrict__ maps,       // [3][H][W] or NULL
                                                float* __restrict__ partial) {  // [nblk][2]
    __shared__ float sx[LE][LE + 1], sy[LE][LE + 1];
    __shared__ float hx[LE][LT], hy[LE][LT], hxx[LE][LT], hyy[LE][LT], hxy[LE][LT];
    __shared__ float s_red[2][LT * LT / 32];
    const int tid = threadIdx.y * LT + threadIdx.x;
    const int x0 = blockIdx.x * LT - LH, y0 = blockIdx.y * LT - LH;
    for (int i = tid; i < LE * LE; i += LT * LT) {
        const int r = i / LE, c = i - r * LE;
        const int gx = x0 + c, gy = y0 + r;
        const bool in = gx >= 0 && gx < W && gy >= 0 && gy < H;
        sx[r][c] = in ? x[(size_t)gy * W + gx] : 0.f;
        sy[r][c] = in ? y[(size_t)gy * W + gx] : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < LE * LT; i += LT * LT) {   // horizontal pass
        const int r = i / LT, c = i - r * LT;
        float a = 0.f, b = 0.f, aa = 0.f, bb = 0.f, ab = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float u = sx[r][c + k], v = sy[r][c + k], g = win.g[k];
            a = fmaf(g, u, a); b = fmaf(g, v, b);
            aa = fmaf(g, u * u, aa); bb = fmaf(g, v * v, bb); ab = fmaf(g, u * v, ab);
        }
        hx[r][c] = a; hy[r][c] = b; hxx[r][c] = aa; hyy[r][c] = bb; hxy[r][c] = ab;
    }
    __syncthreads();
    const int c = threadIdx.x, r = threadIdx.y;
    float mu1 = 0.f, mu2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
    for (int k = 0; k < 11; ++k) {   // vertical pass
        const float g = win.g[k];
        mu1 = fmaf(g, hx[r + k][c], mu1); mu2 = fmaf(g, hy[r + k][c], mu2);
        e11 = fmaf(g, hxx[r + k][c], e11); e22 = fmaf(g, hyy[r + k][c], e22); e12 = fmaf(g, hxy[r + k][c], e12);
    }
    const int gx = blockIdx.x * LT + c, gy = blockIdx.y * LT + r;
    const bool in = gx < W && gy < H;
    const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
    const float mu1s = mu1 * mu1, mu2s = mu2 * mu2, mu12 = mu1 * mu2;
    const float s11 = e11 - mu1s, s22 = e22 - mu2s, s12 = e12 - mu12;
    const float A1 = 2.f * mu12 + C1, A2 = 2.f * s12 + C2, B1 = mu1s + mu2s + C1, B2 = s11 + s22 + C2;
    const float inv = 1.f / (B1 * B2);
    const float S = A1 * A2 * inv;
    float l1 = 0.f, ss = 0.f;
    if (in) {
        l1 = fabsf(sx[r + LH][c + LH] - sy[r + LH][c + LH]);
        ss = S;
        if (maps) {
            // dS/dE[x^2] = dS/dsigma1^2,  dS/dE[xy] = dS/dsigma12,  dS/dmu1 with the sigma terms folded in
            const float dS_ds11 = -S / B2;
            const float dS_ds12 = 2.f * A1 * inv;
            const float dS_dmu1 = 2.f * mu2 * A2 * inv - 2.f * mu1 * S / B1 - 2.f * mu1 * dS_ds11 - mu2 * dS_ds12;
            const size_t o = (size_t)gy * W + gx, n = (size_t)H * W;
            maps[o] = dS_dmu1; maps[n + o] = dS_ds11; maps[2 * n + o] = dS_ds12;
        }
    }
    // CTA sums in a fixed order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        l1 += __shfl_xor_sync(0xffffffffu, l1, o);
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
    }
    if ((tid & 31) == 0) { s_red[0][tid >> 5] = l1; s_red[1][tid >> 5] = ss; }
    __syncthreads();
    if (tid == 0) {
        float a = 0.f, b = 0.f;
        for (int w = 0; w < LT * LT / 32; ++w) { a += s_red[0][w]; b += s_red[1][w]; }
        const size_t blk = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
        partial[2 * blk] = a; partial[2 * blk + 1] = b;
    }
}

__global__ void __launch_bounds__(LT * LT) ssim_stats_kernel(int H, int W, const float* __restrict__ x,
                                                            const float* __restrict__ y, SsimWindow win,
                                                            float* __restrict__ maps, float* __restrict__ partial) {
    ssim_stats_body(H, W, x, y, win, maps, partial);
}

// image v = blockIdx.z: its maps and partials live in slab v (`slab` floats apart) of the scratch
__global__ void __launch_bounds__(LT * LT) ssim_stats_views_kernel(int H, int W, const float* __restrict__ x,
                                                                  const float* __restrict__ y, SsimWindow win,
                                                                  float* __restrict__ maps, float* __restrict__ partial,
                                                                  size_t slab) {
    const size_t v = blockIdx.z, n = (size_t)H * W;
    ssim_stats_body(H, W, x + v * n, y + v * n, win, maps ? maps + v * slab : nullptr, partial + v * slab);
}

// fixed-order final reduction of the per-CTA partials: out = {mean |x-y|, mean SSIM, total loss}
__device__ __forceinline__ void ssim_reduce_body(int nblk, const float* __restrict__ partial, float inv_n, float w_l1,
                                                 float w_dssim, float* __restrict__ out) {
    __shared__ double s_a[32], s_b[32];
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < nblk; i += 1024) { a += (double)partial[2 * i]; b += (double)partial[2 * i + 1]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if ((threadIdx.x & 31) == 0) { s_a[threadIdx.x >> 5] = a; s_b[threadIdx.x >> 5] = b; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ta = 0.0, tb = 0.0;
        for (int w = 0; w < 32; ++w) { ta += s_a[w]; tb += s_b[w]; }
        const float l1 = (float)(ta * (double)inv_n), ssim = (float)(tb * (double)inv_n);
        out[0] = l1; out[1] = ssim; out[2] = w_l1 * l1 + w_dssim * (1.f - ssim);
    }
}

__global__ void __launch_bounds__(1024) ssim_reduce_kernel(int nblk, const float* __restrict__ partial, float inv_n,
                                                           float w_l1, float w_dssim, float* __restrict__ out) {
    ssim_reduce_body(nblk, partial, inv_n, w_l1, w_dssim, out);
}

// image v = blockIdx.x -> out[3 v .. 3 v + 2]
__global__ void __launch_bounds__(1024) ssim_reduce_views_kernel(int nblk, const float* __restrict__ partial,
                                                                 size_t slab, float inv_n, float w_l1, float w_dssim,
                                                                 float* __restrict__ out) {
    ssim_reduce_body(nblk, partial + blockIdx.x * slab, inv_n, w_l1, w_dssim, out + 3 * (size_t)blockIdx.x);
}

// Stage 2: d loss / d x = w_l1 sign(x-y)/N - w_dssim/N [ conv(M1) + 2 x conv(M2) + y conv(M3) ]
__device__ __forceinline__ void ssim_grad_body(int H, int W, const float* __restrict__ x, const float* __restrict__ y,
                                               const SsimWindow& win, const float* __restrict__ maps, float w_l1,
                                               float w_dssim, float inv_n, float* __restrict__ grad) {
    __shared__ float sm[3][LE][LE + 1];
    __shared__ float hm[3][LE][LT];
    const int tid = threadIdx.y * LT + threadIdx.x;
    const int x0 = blockIdx.x * LT - LH, y0 = blockIdx.y * LT - LH;
    const size_t n = (size_t)H * W;
    for (int i = tid; i < LE * LE; i += LT * LT) {
        const int r = i / LE, c = i - r * LE;
        const int gx = x0 + c, gy = y0 + r;
        const bool in = gx >= 0 && gx < W && gy >= 0 && gy < H;
        const size_t o = (size_t)gy * W + gx;
        sm[0][r][c] = in ? maps[o] : 0.f;
        sm[1][r][c] = in ? maps[n + o] : 0.f;
        sm[2][r][c] = in ? maps[2 * n + o] : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < LE * LT; i += LT * LT) {
        const int r = i / LT, c = i - r * LT;
        float a = 0.f, b = 0.f, d = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float g = win.g[k];
            a = fmaf(g, sm[0][r][c + k], a); b = fmaf(g, sm[1][r][c + k], b); d = fmaf(g, sm[2][r][c + k], d);
        }
        hm[0][r][c] = a; hm[1][r][c] = b; hm[2][r][c] = d;
    }
    __syncthreads();
    const int c = threadIdx.x, r = threadIdx.y;
    const int gx = blockIdx.x * LT + c, gy = blockIdx.y * LT + r;
    if (gx >= W || gy >= H) return;
    float a = 0.f, b = 0.f, d = 0.f;
#pragma unroll
    for (int k = 0; k < 11; ++k) {
        const float g = win.g[k];
        a = fmaf(g, hm[0][r + k][c], a); b = fmaf(g, hm[1][r + k][c], b); d = fmaf(g, hm[2][r + k][c], d);
    }
    const size_t o = (size_t)gy * W + gx;
    const float xv = x[o], yv = y[o];
    const float diff = xv - yv;
    const float sgn = (diff > 0.f) ? 1.f : ((diff < 0.f) ? -1.f : 0.f);
    const float dssim = a + 2.f * xv * b + yv * d;
    grad[o] = inv_n * (w_l1 * sgn - w_dssim * dssim);
}

__global__ void __launch_bounds__(LT * LT) ssim_grad_kernel(int H, int W, const float* __restrict__ x,
                                                           const float* __restrict__ y, SsimWindow win,
                                                           const float* __restrict__ maps, float w_l1, float w_dssim,
                                                           float inv_n, float* __restrict__ grad) {
    ssim_grad_body(H, W, x, y, win, maps, w_l1, w_dssim, inv_n, grad);
}

__global__ void __launch_bounds__(LT * LT) ssim_grad_views_kernel(int H, int W, const float* __restrict__ x,
                                                                 const float* __restrict__ y, SsimWindow win,
                                                                 const float* __restrict__ maps, size_t slab, float w_l1,
                                                                 float w_dssim, float inv_n, float* __restrict__ grad) {
    const size_t v = blockIdx.z, n = (size_t)H * W;
    ssim_grad_body(H, W, x + v * n, y + v * n, win, maps + v * slab, w_l1, w_dssim, inv_n, grad + v * n);
}

size_t image_loss_scratch_bytes(int H, int W) {
    const size_t nblk = (size_t)((W + LT - 1) / LT) * ((H + LT - 1) / LT);
    return 256 + ((3 * (size_t)H * W * sizeof(float) + 255) & ~(size_t)255) + nblk * 2 * sizeof(float);
}

int launch_image_loss(cudaStream_t st, int H, int W, const float* image, const float* target, float w_l1,
                      float w_dssim, float* loss_out, float* grad_out, void* scratch, size_t scratch_bytes) {
    if (H <= 0 || W <= 0) return fail_msg(R2X_ERR_INVALID, "r2x_image_loss: bad H/W");
    if (!image || !target || !loss_out || !scratch) return fail_msg(R2X_ERR_INVALID, "r2x_image_loss: null pointer");
    if (scratch_bytes < image_loss_scratch_bytes(H, W)) return fail_msg(R2X_ERR_INVALID, "r2x_image_loss: scratch too small");
    static const SsimWindow win = make_window();
    const dim3 grid((W + LT - 1) / LT, (H + LT - 1) / LT), block(LT, LT);
    const int nblk = (int)(grid.x * grid.y);
    float* maps = (float*)(((size_t)scratch + 255) & ~(size_t)255);
    float* partial = (float*)((char*)maps + ((3 * (size_t)H * W * sizeof(float) + 255) & ~(size_t)255));
    const float inv_n = 1.0f / (float)((double)H * (double)W);
    ssim_stats_kernel<<<grid, block, 0, st>>>(H, W, image, target, win, grad_out ? maps : nullptr, partial);
    ssim_reduce_kernel<<<1, 1024, 0, st>>>(nblk, partial, inv_n, w_l1, w_dssim, loss_out);
    if (grad_out) ssim_grad_kernel<<<grid, block, 0, st>>>(H, W, image, target, win, maps, w_l1, w_dssim, inv_n, grad_out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

// N images: slab v of the scratch holds image v's maps [3][H][W] and then its per-CTA partials, laid out as the
// single-image scratch (so every image goes through exactly the single-image arithmetic).
static size_t image_loss_slab_bytes(int H, int W) {
    const size_t nblk = (size_t)((W + LT - 1) / LT) * ((H + LT - 1) / LT);
    return ((3 * (size_t)H * W * sizeof(float) + 255) & ~(size_t)255) + ((nblk * 2 * sizeof(float) + 255) & ~(size_t)255);
}

size_t image_loss_views_scratch_bytes(int N, int H, int W) {
    if (N < 1 || H <= 0 || W <= 0) return 0;
    return 256 + (size_t)N * image_loss_slab_bytes(H, W);
}

int launch_image_loss_views(cudaStream_t st, int N, int H, int W, const float* images, const float* targets, float w_l1,
                            float w_dssim, float* loss_out, float* grad_out, void* scratch, size_t scratch_bytes) {
    if (N < 1 || N > 65535) return fail_msg(R2X_ERR_INVALID, "r2x_image_loss_views: bad N (need 1 <= N <= 65535)");
    if (H <= 0 || W <= 0) return fail_msg(R2X_ERR_INVALID, "r2x_image_loss_views: bad H/W");
    if (!images || !targets || !loss_out || !scratch) return fail_msg(R2X_ERR_INVALID, "r2x_image_loss_views: null pointer");
    if (scratch_bytes < image_loss_views_scratch_bytes(N, H, W))
        return fail_msg(R2X_ERR_INVALID, "r2x_image_loss_views: scratch too small");
    static const SsimWindow win = make_window();
    const dim3 grid((W + LT - 1) / LT, (H + LT - 1) / LT, N), block(LT, LT);
    const int nblk = (int)(grid.x * grid.y);
    const size_t slab = image_loss_slab_bytes(H, W) / sizeof(float);
    float* maps = (float*)(((size_t)scratch + 255) & ~(size_t)255);
    float* partial = (float*)((char*)maps + ((3 * (size_t)H * W * sizeof(float) + 255) & ~(size_t)255));
    const float inv_n = 1.0f / (float)((double)H * (double)W);
    ssim_stats_views_kernel<<<grid, block, 0, st>>>(H, W, images, targets, win, grad_out ? maps : nullptr, partial, slab);
    ssim_reduce_views_kernel<<<N, 1024, 0, st>>>(nblk, partial, slab, inv_n, w_l1, w_dssim, loss_out);
    if (grad_out)
        ssim_grad_views_kernel<<<grid, block, 0, st>>>(H, W, images, targets, win, maps, slab, w_l1, w_dssim, inv_n,
                                                       grad_out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// 3-D total variation: loss = (sum|d/dx| + sum|d/dy| + sum|d/dz|) * scale ; grad by gathering the six incident
// differences of every voxel (no atomics).  vol[x][y][z], z fastest.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sgnf(float v) { return (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f); }

__global__ void __launch_bounds__(256) tv3d_kernel(int nx, int ny, int nz, const float* __restrict__ vol, float scale,
                                                   float* __restrict__ grad, float* __restrict__ partial) {
    __shared__ float s_red[8];
    const size_t n = (size_t)nx * ny * nz;
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    float acc = 0.f;
    if (i < n) {
        const int z = (int)(i % nz), y = (int)((i / nz) % ny), x = (int)(i / ((size_t)nz * ny));
        const size_t sx = (size_t)ny * nz, sy = (size_t)nz;
        const float v = vol[i];
        float g = 0.f;
        if (x + 1 < nx) { const float d = vol[i + sx] - v; acc += fabsf(d); g -= sgnf(d); }
        if (y + 1 < ny) { const float d = vol[i + sy] - v; acc += fabsf(d); g -= sgnf(d); }
        if (z + 1 < nz) { const float d = vol[i + 1] - v; acc += fabsf(d); g -= sgnf(d); }
        if (grad) {
            if (x > 0) g += sgnf(v - vol[i - sx]);
            if (y > 0) g += sgnf(v - vol[i - sy]);
            if (z > 0) g += sgnf(v - vol[i - 1]);
            grad[i] = g * scale;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += s_red[w];
        partial[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(1024) tv3d_reduce_kernel(int nblk, const float* __restrict__ partial, float scale,
                                                           float* __restrict__ out) {
    __shared__ double s_a[32];
    double a = 0.0;
    for (int i = threadIdx.x; i < nblk; i += 1024) a += (double)partial[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if ((threadIdx.x & 31) == 0) s_a[threadIdx.x >> 5] = a;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 32; ++w) t += s_a[w];
        out[0] = (float)(t * (double)scale);
    }
}

size_t tv3d_scratch_bytes(int nx, int ny, int nz) {
    const size_t n = (size_t)nx * ny * nz;
    return 256 + ((n + 255) / 256) * sizeof(float);
}

int launch_tv3d(cudaStream_t st, int nx, int ny, int nz, const float* vol, int reduction_mean, float* loss_out,
                float* grad_out, void* scratch, size_t scratch_bytes) {
    if (nx <= 0 || ny <= 0 || nz <= 0) return fail_msg(R2X_ERR_INVALID, "r2x_tv3d_loss: bad grid");
    if (!vol || !loss_out || !scratch) return fail_msg(R2X_ERR_INVALID, "r2x_tv3d_loss: null pointer");
    if (scratch_bytes < tv3d_scratch_bytes(nx, ny, nz)) return fail_msg(R2X_ERR_INVALID, "r2x_tv3d_loss: scratch too small");
    const size_t n = (size_t)nx * ny * nz;
    const int nblk = (int)((n + 255) / 256);
    float scale = 1.f;
    if (reduction_mean) {
        const double tot = (double)(nx - 1) * ny * nz + (double)nx * (ny - 1) * nz + (double)nx * ny * (nz - 1);
        scale = (float)(1.0 / tot);
    }
    float* partial = (float*)(((size_t)scratch + 255) & ~(size_t)255);
    tv3d_kernel<<<nblk, 256, 0, st>>>(nx, ny, nz, vol, scale, grad_out, partial);
    tv3d_reduce_kernel<<<1, 1024, 0, st>>>(nblk, partial, scale, loss_out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Fused Adam over up to R2X_ADAM_MAX_GROUPS parameter tensors (torch.optim.Adam, amsgrad off, no weight decay):
//   m <- m + (1-b1)(g - m);  v <- b2 v + (1-b2) g^2;  p <- p - (lr / bc1) m / (sqrt(v)/sqrt(bc2) + eps)
// ------------------------------------------------------------------------------------------------
struct AdamPack {
    r2x_adam_group g[R2X_ADAM_MAX_GROUPS];
    const float* grad2[R2X_ADAM_MAX_GROUPS];   // optional second gradient source, summed with g.grad (null = none)
    const uint32_t* guard[2];                  // optional {count, overflow} status words: any overflow -> no update
    int n;
};

__global__ void __launch_bounds__(256) adam_kernel(AdamPack pk, float one_minus_b1, float beta2, float one_minus_b2,
                                                   float eps, float inv_bc1, float inv_sqrt_bc2) {
    if ((pk.guard[0] && pk.guard[0][1]) || (pk.guard[1] && pk.guard[1][1])) return;
    const r2x_adam_group gr = pk.g[blockIdx.y];
    const float* __restrict__ g2 = pk.grad2[blockIdx.y];
    const float step_size = gr.lr * inv_bc1;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < gr.numel; i += (long long)gridDim.x * 256) {
        const float g = g2 ? gr.grad[i] + g2[i] : gr.grad[i];
        float m = gr.exp_avg[i], v = gr.exp_avg_sq[i];
        m = fmaf(one_minus_b1, g - m, m);
        v = fmaf(one_minus_b2, g * g, beta2 * v);
        gr.exp_avg[i] = m;
        gr.exp_avg_sq[i] = v;
        const float denom = sqrtf(v) * inv_sqrt_bc2 + eps;
        gr.param[i] = gr.param[i] - step_size * (m / denom);
    }
}

int launch_adam(cudaStream_t st, int ngroups, const r2x_adam_group* groups, double beta1, double beta2, double eps,
                long long step, const float* const* grads2, const uint32_t* guard0, const uint32_t* guard1) {
    if (ngroups < 0 || ngroups > R2X_ADAM_MAX_GROUPS) return fail_msg(R2X_ERR_INVALID, "r2x_adam_step: too many groups");
    if (step < 1) return fail_msg(R2X_ERR_INVALID, "r2x_adam_step: step counts from 1");
    if (ngroups == 0) return 0;
    AdamPack pk{};
    pk.n = ngroups;
    pk.guard[0] = guard0;
    pk.guard[1] = guard1;
    long long maxn = 0;
    for (int i = 0; i < ngroups; ++i) {
        pk.g[i] = groups[i];
        pk.grad2[i] = grads2 ? grads2[i] : nullptr;
        if (groups[i].numel < 0) return fail_msg(R2X_ERR_INVALID, "r2x_adam_step: negative numel");
        if (groups[i].numel > 0 && (!groups[i].param || !groups[i].grad || !groups[i].exp_avg || !groups[i].exp_avg_sq))
            return fail_msg(R2X_ERR_INVALID, "r2x_adam_step: null pointer");
        if (groups[i].numel > maxn) maxn = groups[i].numel;
    }
    if (maxn == 0) return 0;
    const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
    long long nb = (maxn + 255) / 256;
    int sms;
    R2X_CUDA_OK(sm_count(&sms));
    if (nb > sms * 16) nb = sms * 16;
    // 1 - beta in double, then float: what torch passes to lerp_/addcmul_ (betas are doubles in the ABI: 1.f - 0.999f would be off by 1.3e-5 relative)
    adam_kernel<<<dim3((unsigned)nb, (unsigned)ngroups), 256, 0, st>>>(
        pk, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps, (float)(1.0 / bc1),
        (float)(1.0 / sqrt(bc2)));
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Densification statistics of one iteration (train.py:150-156 + gaussian_model.py:552-556) in one launch:
//   visible = radii > 0;  max_radii2D = max(max_radii2D, radii) | visible;  accum += |dL/dmean2D (x, y)| | visible;
//   denom += 1 | visible.   The guards are the forwards' {count, overflow} words: an overflowed iteration changes nothing.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) densify_stats_kernel(int P, const int* __restrict__ radii,
                                                            const float* __restrict__ grad2d, float* __restrict__ max_radii,
                                                            float* __restrict__ accum, float* __restrict__ denom,
                                                            const uint32_t* guard0, const uint32_t* guard1) {
    if ((guard0 && guard0[1]) || (guard1 && guard1[1])) return;
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= P) return;
    const int r = radii[g];
    if (r <= 0) return;
    max_radii[g] = fmaxf(max_radii[g], (float)r);
    const float gx = grad2d[3 * (size_t)g], gy = grad2d[3 * (size_t)g + 1];
    accum[g] += sqrtf(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)));
    denom[g] += 1.0f;
}

int launch_densify_stats(cudaStream_t st, int P, const int* radii, const float* grad2d, float* max_radii, float* accum,
                         float* denom, const uint32_t* guard0, const uint32_t* guard1) {
    if (P <= 0) return 0;
    densify_stats_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, radii, grad2d, max_radii, accum, denom, guard0, guard1);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

// N views' statistics in one launch: radii[N,P], grad2d[N,P,3]; each Gaussian takes the views in order with the
// single-view kernel's arithmetic on values held in registers (bit for bit N launches of densify_stats_kernel).
__global__ void __launch_bounds__(256) densify_stats_views_kernel(int N, int P, const int* __restrict__ radii,
                                                                  const float* __restrict__ grad2d,
                                                                  float* __restrict__ max_radii, float* __restrict__ accum,
                                                                  float* __restrict__ denom, const uint32_t* guard0,
                                                                  const uint32_t* guard1) {
    if ((guard0 && guard0[1]) || (guard1 && guard1[1])) return;
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= P) return;
    float mr = 0.f, acc = 0.f, den = 0.f;
    bool seen = false;
    for (int v = 0; v < N; ++v) {
        const size_t vg = (size_t)v * P + g;
        const int r = radii[vg];
        if (r <= 0) continue;
        if (!seen) { mr = max_radii[g]; acc = accum[g]; den = denom[g]; seen = true; }
        mr = fmaxf(mr, (float)r);
        const float gx = grad2d[3 * vg], gy = grad2d[3 * vg + 1];
        acc = __fadd_rn(acc, sqrtf(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy))));
        den = __fadd_rn(den, 1.0f);
    }
    if (!seen) return;
    max_radii[g] = mr;
    accum[g] = acc;
    denom[g] = den;
}

int launch_densify_stats_views(cudaStream_t st, int N, int P, const int* radii, const float* grad2d, float* max_radii,
                               float* accum, float* denom, const uint32_t* guard0, const uint32_t* guard1) {
    if (P <= 0) return 0;
    densify_stats_views_kernel<<<(P + 255) / 256, 256, 0, st>>>(N, P, radii, grad2d, max_radii, accum, denom, guard0,
                                                                guard1);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace r2x
