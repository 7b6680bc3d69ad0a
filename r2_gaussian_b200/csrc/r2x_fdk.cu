// r2x_fdk.cu -- FDK (Feldkamp-Davis-Kress) reconstruction of a density volume from cone- or parallel-beam projections.
//
// The reference initialises its Gaussians from TIGRE's `algs.fdk` (r2_gaussian/utils/ct_utils.py::recon_volume called
// by initialize_pcd.py).  FDK is a weighted ramp filter along the detector rows followed by one voxel-driven
// backprojection; both are small data-parallel kernels, and the geometry they need is the rasterizer's own:
//
//   fdk_filter_kernel       one CTA per detector row: cosine weight (cone beam) at each pixel's ndc, moved by the
//                           detector offset (t_u, t_v) pixels when there is one, times the redundancy weight of the
//                           weighting (R2X_FDK_PLAIN none, R2X_FDK_PARKER Parker's for a short scan, R2X_FDK_HALF_FAN
//                           Wang's for an offset detector on a full circle); stage the row in shared memory between two
//                           rows of zeros, then the band-limited Ram-Lak filter as a linear convolution over the whole
//                           row, using the symmetric odd-only taps:
//                             Q_j = (r_j / 4 - sum_{k odd} (r_{j-k} + r_{j+k}) / (pi^2 k^2)) / D
//                           (D = isocentre pitch), summed from the largest odd k < W down to k = 1.
//   fdk_window_kernel       the same weights, then a windowed ramp filter (Shepp-Logan, cosine, Hamming, Hann): taps
//                           h[k] = (1 / 2 pi^2) int_0^pi w Wn(w) cos(w k) dw, closed forms in fdk_window_tap, non-zero at
//                           every k.  Shared memory holds the row and the W taps h[0 .. W-1] (2 W floats, 128 KB at
//                           W = 16384) and no zero pads: a pixel j sums the one-sided taps beyond its nearer edge first,
//                           then the two-sided ones, each from the largest k down to k = 1:
//                             Q_j = (h[0] r_j + sum_{k=1}^{W-1} h[k] (r_{j-k} + r_{j+k})) / D   (r = 0 outside the row)
//   fdk_backproject_kernel  a thread owns one (x, y) voxel column and a run of FDK_ZR voxels along z.  Every view's
//                           homogeneous coordinates are affine in z, so the per-view setup (4 matrix rows, staged per
//                           chunk of views in shared memory) is paid once per run.  Each voxel centre goes through the
//                           same projmatrix, homogeneous divide and ndc -> pixel mapping as the rasterizer, the
//                           filtered view is sampled bilinearly through L1/L2 (__ldg; 0 outside the detector) and
//                           weighted by U^2, U = DSO / z_view (cone; 1 for parallel beam).  The views are summed in
//                           index order in registers and each voxel is stored once: no atomics, so the volume is
//                           bitwise reproducible.  An offset detector needs nothing here: the caller passes the offset
//                           projmatrices.  The scale is pi / N, or 1 for Parker weights (they hold each view's
//                           interval).
//
// The float64 NumPy statements of the same definitions are oracle/fdk_oracle.py (plain),
// tests/fdk_short_scan_oracle.py (short scan, Parker weights) and tests/offset_detector_oracle.py (offset detector,
// half-fan weights).
#include <cmath>
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_common.cuh"

namespace r2x {

constexpr int FDK_MAX_W = 16384;     // filter row staging: (3 W + W / 2) floats of shared memory (<= 227 KB);
                                     // windowed filters 2 W floats
constexpr int FDK_BX = 32, FDK_BY = 4; // backprojection CTA: 32 y-columns x 4 x-columns
constexpr int FDK_ZR = 8;            // voxels per thread along z
constexpr int FDK_VCHUNK = 32;       // views staged in shared memory at a time

static size_t fdk_al256(size_t x) { return (x + 255) & ~(size_t)255; }

size_t fdk_scratch_bytes(int N, int H, int W) {
    if (N < 1 || H < 1 || W < 1) return 256;
    return fdk_al256((size_t)N * H * W * sizeof(float)) + 256;
}

static size_t fdk_filter_smem(int W) { return (size_t)(3 * W + (W + 1) / 2) * sizeof(float); }
static size_t fdk_window_smem(int W) { return (size_t)(2 * W) * sizeof(float); }

template <bool CONE>
__global__ void __launch_bounds__(FDK_BX * FDK_BY) fdk_backproject_kernel(
    int N, int H, int W, const float* __restrict__ q, const float* __restrict__ viewm, const float* __restrict__ projm,
    float dso, int nx, int ny, int nz, float ox, float oy, float oz, float dx, float dy, float dz, float scale,
    float* __restrict__ vol) {
    // per view: projmatrix rows 0, 1, 3 and viewmatrix row 2 as (m[r], m[4+r], m[8+r], m[12+r])
    __shared__ float4 mat[FDK_VCHUNK][4];
    const int y = blockIdx.x * FDK_BX + threadIdx.x;
    const int x = blockIdx.y * FDK_BY + threadIdx.y;
    const int z0 = blockIdx.z * FDK_ZR;
    const int tid = threadIdx.y * FDK_BX + threadIdx.x;
    const bool live = x < nx && y < ny;
    const float X = fmaf((float)x, dx, ox), Y = fmaf((float)y, dy, oy), Z0 = fmaf((float)z0, dz, oz);
    const float half_w = 0.5f * (float)W, half_h = 0.5f * (float)H;
    const float cen_w = 0.5f * (float)(W - 1), cen_h = 0.5f * (float)(H - 1);
    const size_t view_stride = (size_t)H * W;
    float acc[FDK_ZR];
#pragma unroll
    for (int k = 0; k < FDK_ZR; ++k) acc[k] = 0.0f;

    for (int c0 = 0; c0 < N; c0 += FDK_VCHUNK) {
        const int nc = min(FDK_VCHUNK, N - c0);
        __syncthreads();
        for (int e = tid; e < nc * 4; e += FDK_BX * FDK_BY) {
            const int v = e >> 2, slot = e & 3;
            const float* m = (slot == 3 ? viewm : projm) + (size_t)(c0 + v) * 16;
            const int rr = slot == 3 ? 2 : (slot == 2 ? 3 : slot);
            mat[v][slot] = make_float4(m[rr], m[4 + rr], m[8 + rr], m[12 + rr]);
        }
        __syncthreads();
        if (!live) continue;
        for (int v = 0; v < nc; ++v) {
            const float4 P0 = mat[v][0], P1 = mat[v][1], P3 = mat[v][2], V2 = mat[v][3];
            const float ax = fmaf(P0.z, Z0, fmaf(P0.y, Y, fmaf(P0.x, X, P0.w)));
            const float ay = fmaf(P1.z, Z0, fmaf(P1.y, Y, fmaf(P1.x, X, P1.w)));
            const float aw = fmaf(P3.z, Z0, fmaf(P3.y, Y, fmaf(P3.x, X, P3.w))) + 1e-7f;  // the rasterizer's divide
            const float sx = P0.z * dz, sy = P1.z * dz, sw = P3.z * dz;
            float av = 0.0f, sv = 0.0f;
            if (CONE) {
                av = fmaf(V2.z, Z0, fmaf(V2.y, Y, fmaf(V2.x, X, V2.w)));
                sv = V2.z * dz;
            }
            const float* qv = q + (size_t)(c0 + v) * view_stride;
#pragma unroll
            for (int k = 0; k < FDK_ZR; ++k) {
                const float fk = (float)k;
                float w = 1.0f;
                if (CONE) {
                    const float zv = fmaf(fk, sv, av);
                    if (!(zv > 0.0f)) continue;
                    const float u = dso * __frcp_rn(zv);
                    w = u * u;
                }
                const float pw = __frcp_rn(fmaf(fk, sw, aw));
                const float px = fmaf(fmaf(fk, sx, ax) * pw, half_w, cen_w);
                const float py = fmaf(fmaf(fk, sy, ay) * pw, half_h, cen_h);
                if (!(px > -1.0f && px < (float)W && py > -1.0f && py < (float)H)) continue;
                const float fx0 = floorf(px), fy0 = floorf(py);
                const int ix = (int)fx0, iy = (int)fy0;
                const float fx = px - fx0, fy = py - fy0;
                const long long base = (long long)iy * W + ix;
                float s00 = 0.0f, s01 = 0.0f, s10 = 0.0f, s11 = 0.0f;
                if (iy >= 0) {
                    if (ix >= 0) s00 = __ldg(qv + base);
                    if (ix + 1 < W) s01 = __ldg(qv + base + 1);
                }
                if (iy + 1 < H) {
                    if (ix >= 0) s10 = __ldg(qv + base + W);
                    if (ix + 1 < W) s11 = __ldg(qv + base + W + 1);
                }
                const float top = fmaf(fx, s01 - s00, s00), bot = fmaf(fx, s11 - s10, s10);
                acc[k] = fmaf(w, fmaf(fy, bot - top, top), acc[k]);
            }
        }
    }
    if (!live) return;
    float* out = vol + ((size_t)x * ny + y) * nz;
#pragma unroll
    for (int k = 0; k < FDK_ZR; ++k)
        if (z0 + k < nz) out[z0 + k] = acc[k] * scale;
}

// Parker redundancy weight of the ray at arc position beta (radians from the start of the scan) and fan angle gam
// (signed so that its conjugate ray is (beta + pi + 2 gam, -gam)) on a short scan of arc B = pi + 2 delta.  A region
// whose bounds cross (delta - gam <= 0 or delta + gam <= 0) is empty, so no branch divides by a non-positive value.
__device__ __forceinline__ float fdk_parker_weight(float beta, float gam, float arc, float delta) {
    const float rise = delta - gam;
    if (beta < 2.0f * rise) {
        const float s = sinpif(0.25f * beta / rise);
        return s * s;
    }
    if (beta < 3.14159265358979f - 2.0f * gam) return 1.0f;
    if (beta < arc) {
        const float s = sinpif(0.25f * (arc - beta) / (delta + gam));
        return s * s;
    }
    return 0.0f;
}

// Half-fan redundancy weight (Wang 2002) of the ray at fan coordinate a (tan of the fan angle; ndc for parallel beam)
// on a full circle with the axis off the detector's centre: 2 sin^2(pi/4 (1 + sigma a / delta)) on the overlap
// |a| <= delta, 2 beyond it on the wide side (sigma a > delta), 0 beyond it on the narrow side (no pixel lies there).
// w(a) + w(-a) = 2 on the overlap, so a ray measured twice keeps the plain FDK's total weight.
__device__ __forceinline__ float fdk_half_fan_weight(float a, float inv_delta, float sigma) {
    const float x = sigma * a * inv_delta;
    if (x >= 1.0f) return 2.0f;
    if (x <= -1.0f) return 0.0f;
    const float s = sinpif(0.25f * (1.0f + x));
    return 2.0f * (s * s);
}

// The arguments only one weighting reads.
struct FdkWeights {
    const float2* vw = nullptr;          // PARKER: each view's (beta'_v, dbeta_v)
    float arc = 0.0f, delta = 0.0f;      // PARKER: the arc B and delta = (B - pi) / 2
    float fan = 1.0f, hf_inv_delta = 1.0f, hf_sigma = 1.0f;   // HALF_FAN: a = ndc_x * fan, 1 / delta, sign(t_u)
};

// Step 1 of FDK on detector row r (view * H + row) of a detector offset by (t_u, t_v) pixels (zero when centred): each
// pixel's cosine weight (cone beam) at its ndc moved by (su, sv) = (2 t_u / W, -2 t_v / H), then WEIGHT's redundancy
// weight: PARKER its Parker weight at fan angle -atan(a) (cone; 0 for parallel beam) times its view's angular interval,
// HALF_FAN fdk_half_fan_weight of its fan coordinate a = ndc_x * fan.  The weight is computed per pixel, which costs
// little next to the convolution of each pixel.  put(j, p) receives weighted pixel j; the CTA's threads stride the row.
template <int WEIGHT, class Put>
__device__ __forceinline__ void fdk_weight_row(size_t r, int H, int W, const float* __restrict__ projs, float tanx,
                                               float tany, int cone, float su, float sv, const FdkWeights& fw,
                                               Put put) {
    const float* src = projs + r * W;
    const float step = 2.0f / (float)W, first = 1.0f / (float)W - 1.0f;
    const float b = cone ? (fmaf((float)(r % H), 2.0f / (float)H, 1.0f / (float)H - 1.0f) + sv) * tany : 0.0f;
    float2 bv = make_float2(0.0f, 0.0f);
    if (WEIGHT == R2X_FDK_PARKER) bv = fw.vw[r / H];
    for (int j = threadIdx.x; j < W; j += blockDim.x) {
        float p = src[j];
        const float nd = fmaf((float)j, step, first) + su;
        float gam = 0.0f;
        if (cone) {
            const float a = nd * tanx;
            p *= rsqrtf(fmaf(a, a, fmaf(b, b, 1.0f)));
            // column u runs along the rotation, so a ray at +u leans back: gamma = -atan(u / DSD)
            if (WEIGHT == R2X_FDK_PARKER) gam = -atanf(a);
        }
        if (WEIGHT == R2X_FDK_PARKER) p *= fdk_parker_weight(bv.x, gam, fw.arc, fw.delta) * bv.y;
        if (WEIGHT == R2X_FDK_HALF_FAN) p *= fdk_half_fan_weight(nd * fw.fan, fw.hf_inv_delta, fw.hf_sigma);
        put(j, p);
    }
}

// Steps 1-2 of FDK with the band-limited Ram-Lak filter, one CTA per detector row: fdk_weight_row, the row staged in
// shared memory between two rows of zeros and filtered with the Ram-Lak taps (shift-invariant, so the same for any
// offset).
template <int WEIGHT>
__global__ void __launch_bounds__(256) fdk_filter_kernel(int H, int W, const float* __restrict__ projs, float tanx,
                                                         float tany, int cone, float inv_delta, float su, float sv,
                                                         FdkWeights fw, float* __restrict__ q) {
    extern __shared__ float sm[];
    float* row = sm;              // [3W]: zeros | weighted row | zeros
    float* g = sm + 3 * W;        // [(W+1)/2]: g[m] = 1 / (pi^2 (2m+1)^2)
    const size_t r = blockIdx.x;  // view * H + detector row
    fdk_weight_row<WEIGHT>(r, H, W, projs, tanx, tany, cone, su, sv, fw, [&](int j, float p) {
        row[j] = 0.0f;
        row[W + j] = p;
        row[2 * W + j] = 0.0f;
    });
    for (int m = threadIdx.x; m < (W + 1) / 2; m += blockDim.x) {
        const float k = (float)(2 * m + 1);
        g[m] = 1.0f / (9.869604401089358f * k * k);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < W; j += blockDim.x) {
        const float* c = row + W + j;
        // smallest taps first: summed from k = 1 up, the accumulator is near r_j / 4 after a few taps and every tap
        // below half its ulp (k beyond ~3700) is lost, which truncated the filter on wide rows
        float acc = 0.0f;
        for (int m = W / 2 - 1; m >= 0; --m) acc = fmaf(g[m], c[-(2 * m + 1)] + c[2 * m + 1], acc);
        q[r * W + j] = fmaf(0.25f, c[0], -acc) * inv_delta;
    }
}

// Band-limited Ram-Lak tap h_RL[k] in units of 1 / D: 1/4 at 0, -1 / (pi^2 k^2) at odd k, 0 at even k != 0.
__device__ __forceinline__ double fdk_ram_lak_tap(int k) {
    k = abs(k);
    return k == 0 ? 0.25 : (k & 1) ? -1.0 / (9.869604401089358 * k * k) : 0.0;
}

// Tap h[k] (k >= 0, units of 1 / D) of the ramp times WINDOW's Wn (TIGRE's windows at frequency scale 1), in float64:
//   SHEPP_LOGAN  Wn = sin(w/2) / (w/2)   h[k] = -2 / (pi^2 (4k^2 - 1))
//   COSINE       Wn = cos(w/2)           h[k] = -(-1)^k / (pi (4k^2 - 1)) - (1/(2k+1)^2 + 1/(2k-1)^2) / pi^2
//   HAMMING      Wn = 0.54 + 0.46 cos w  h[k] = 0.54 h_RL[k] + 0.23 (h_RL[k-1] + h_RL[k+1])
//   HANN         Wn = (1 + cos w) / 2    h[k] = 0.5 h_RL[k] + 0.25 (h_RL[k-1] + h_RL[k+1])
template <int WINDOW>
__device__ __forceinline__ double fdk_window_tap(int k) {
    const double pi = 3.141592653589793, pi2 = 9.869604401089358, kk = (double)k, d = 4.0 * kk * kk - 1.0;
    if (WINDOW == R2X_FDK_SHEPP_LOGAN) return -2.0 / (pi2 * d);
    if (WINDOW == R2X_FDK_COSINE) {
        const double a = 2.0 * kk + 1.0, b = 2.0 * kk - 1.0;
        return -((k & 1) ? -1.0 : 1.0) / (pi * d) - (1.0 / (a * a) + 1.0 / (b * b)) / pi2;
    }
    const double c0 = WINDOW == R2X_FDK_HAMMING ? 0.54 : 0.5, c1 = WINDOW == R2X_FDK_HAMMING ? 0.23 : 0.25;
    return c0 * fdk_ram_lak_tap(k) + c1 * (fdk_ram_lak_tap(k - 1) + fdk_ram_lak_tap(k + 1));
}

// Steps 1-2 of FDK with WINDOW's ramp filter, one CTA per detector row: fdk_weight_row into shared memory, the taps
// h[0 .. W-1] rounded once from float64 next to it, then the linear convolution over the whole row.  Pixel j's partner
// pixels j - k and j + k both lie in the row for k <= near = min(j, W-1-j), one of them up to far = max(j, W-1-j);
// the sum runs from k = far down to 1, smallest taps first (as fdk_filter_kernel's), with no bounds checks in either
// loop.
template <int WEIGHT, int WINDOW>
__global__ void __launch_bounds__(256) fdk_window_kernel(int H, int W, const float* __restrict__ projs, float tanx,
                                                         float tany, int cone, float inv_delta, float su, float sv,
                                                         FdkWeights fw, float* __restrict__ q) {
    extern __shared__ float sm[];
    float* row = sm;              // [W]: weighted row
    float* h = sm + W;            // [W]: h[k]
    const size_t r = blockIdx.x;  // view * H + detector row
    fdk_weight_row<WEIGHT>(r, H, W, projs, tanx, tany, cone, su, sv, fw, [&](int j, float p) { row[j] = p; });
    for (int k = threadIdx.x; k < W; k += blockDim.x) h[k] = (float)fdk_window_tap<WINDOW>(k);
    __syncthreads();
    for (int j = threadIdx.x; j < W; j += blockDim.x) {
        const float* c = row + j;
        const int near = min(j, W - 1 - j), far = max(j, W - 1 - j);
        const int side = j < W - 1 - j ? 1 : -1;   // the partner that stays in the row beyond `near`
        float acc = 0.0f;
        for (int k = far; k > near; --k) acc = fmaf(h[k], c[side * k], acc);
        for (int k = near; k > 0; --k) acc = fmaf(h[k], c[-k] + c[k], acc);
        q[r * W + j] = fmaf(h[0], c[0], acc) * inv_delta;
    }
}

// isocentre pitch: cone dDetector_u * DSO / DSD = 2 tan_fovx DSO / W; parallel 2 / W (ndc [-1,1] = scene [-1,1])
static double fdk_pitch(int W, float tanx, int mode, float dso) {
    return mode == 1 ? 2.0 * (double)tanx * (double)dso / W : 2.0 / W;
}

using FdkFilterKernel = void (*)(int, int, const float*, float, float, int, float, float, float, FdkWeights, float*);

template <int WEIGHT>
static FdkFilterKernel fdk_filter_for(int window) {
    switch (window) {
        case R2X_FDK_SHEPP_LOGAN: return fdk_window_kernel<WEIGHT, R2X_FDK_SHEPP_LOGAN>;
        case R2X_FDK_COSINE: return fdk_window_kernel<WEIGHT, R2X_FDK_COSINE>;
        case R2X_FDK_HAMMING: return fdk_window_kernel<WEIGHT, R2X_FDK_HAMMING>;
        case R2X_FDK_HANN: return fdk_window_kernel<WEIGHT, R2X_FDK_HANN>;
        default: return fdk_filter_kernel<WEIGHT>;
    }
}

// window: R2X_FDK_RAM_LAK or one of the windowed filters (r2x_fdk's filter field)
static int fdk_filter(cudaStream_t st, int weighting, int window, int N, int H, int W, const float* projs, float tanx,
                      float tany, int mode, float dso, float su, float sv, const FdkWeights& fw, float* q) {
    auto kernel = weighting == R2X_FDK_PARKER     ? fdk_filter_for<R2X_FDK_PARKER>(window)
                  : weighting == R2X_FDK_HALF_FAN ? fdk_filter_for<R2X_FDK_HALF_FAN>(window)
                                                  : fdk_filter_for<R2X_FDK_PLAIN>(window);
    const size_t smem = window == R2X_FDK_RAM_LAK ? fdk_filter_smem(W) : fdk_window_smem(W);
    if (smem > 48 * 1024)
        R2X_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<(unsigned)((long long)N * H), 256, smem, st>>>(H, W, projs, tanx, tany, mode,
                                                            (float)(1.0 / fdk_pitch(W, tanx, mode, dso)), su, sv, fw, q);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

static int fdk_backproject(cudaStream_t st, int N, int H, int W, const float* q, const float* viewm, const float* projm,
                           int mode, float dso, int nx, int ny, int nz, float sx, float sy, float sz, float cx, float cy,
                           float cz, float scale, float* vol) {
    const float dx = sx / nx, dy = sy / ny, dz = sz / nz;
    const float ox = cx - 0.5f * sx + 0.5f * dx, oy = cy - 0.5f * sy + 0.5f * dy, oz = cz - 0.5f * sz + 0.5f * dz;
    const dim3 grid((ny + FDK_BX - 1) / FDK_BX, (nx + FDK_BY - 1) / FDK_BY, (nz + FDK_ZR - 1) / FDK_ZR);
    const dim3 block(FDK_BX, FDK_BY);
    if (mode == 1)
        fdk_backproject_kernel<true><<<grid, block, 0, st>>>(N, H, W, q, viewm, projm, dso, nx, ny, nz, ox, oy, oz, dx, dy,
                                                            dz, scale, vol);
    else
        fdk_backproject_kernel<false><<<grid, block, 0, st>>>(N, H, W, q, viewm, projm, dso, nx, ny, nz, ox, oy, oz, dx,
                                                             dy, dz, scale, vol);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

static int fdk_validate(int N, int H, int W, const float* projs, const float* viewm, const float* projm,
                        float tanx, float tany, int mode, float dso, int nx, int ny, int nz, float sx, float sy,
                        float sz, const void* out, const void* scratch, size_t scratch_bytes) {
    if (N < 1 || H < 1 || W < 1) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad N/H/W (each must be >= 1)");
    if (W > FDK_MAX_W) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad W (detector rows wider than 16384 pixels)");
    if ((long long)N * H > 0x7fffffffLL) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad N*H (too many detector rows)");
    if (nx < 1 || ny < 1 || nz < 1) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad grid (each size must be >= 1)");
    if ((nx + FDK_BY - 1) / FDK_BY > 65535 || (nz + FDK_ZR - 1) / FDK_ZR > 65535)
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad grid (too large)");
    if (mode != 0 && mode != 1) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad mode (0 = parallel, 1 = cone)");
    if (mode == 1 && !(dso > 0.0f && std::isfinite(dso)))
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad DSO (cone beam needs DSO > 0)");
    if (mode == 1 && !(tanx > 0.0f && tany > 0.0f && std::isfinite(tanx) && std::isfinite(tany)))
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad tan_fov (cone beam needs tan_fovx, tan_fovy > 0)");
    if (!(sx > 0.0f && sy > 0.0f && sz > 0.0f)) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad sVoxel (must be > 0)");
    if (!projs || !viewm || !projm || !out || !scratch) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad pointer (NULL)");
    if (scratch_bytes < fdk_scratch_bytes(N, H, W)) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad scratch (too small)");
    return 0;
}

}  // namespace r2x

extern "C" {

size_t r2x_fdk_scratch_bytes(int n_views, int H, int W) { return r2x::fdk_scratch_bytes(n_views, H, W); }

int r2x_fdk(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
            const float* projmatrices, float tan_fovx, float tan_fovy, int mode, float shift_u, float shift_v,
            int weighting, const float* view_weights, float arc, float dso, int nx, int ny, int nz, float sx, float sy,
            float sz, float cx, float cy, float cz, float* out_volume, void* scratch, size_t scratch_bytes) {
    using namespace r2x;
    if (int rc = fdk_validate(n_views, H, W, projs, viewmatrices, projmatrices, tan_fovx, tan_fovy, mode, dso, nx, ny,
                              nz, sx, sy, sz, out_volume, scratch, scratch_bytes))
        return rc;
    if (!(std::isfinite(shift_u) && std::isfinite(shift_v)))
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad shift (must be finite)");
    // the low byte is the redundancy weighting, bits 8 and up the filter
    const int window = weighting & ~0xff;
    if (weighting < 0 || window > R2X_FDK_HANN)
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad weighting (filter field 0x000 = Ram-Lak, 0x100 = Shepp-Logan, "
                                         "0x200 = cosine, 0x300 = Hamming, 0x400 = Hann; no other bits)");
    weighting &= 0xff;
    if (weighting != R2X_FDK_PLAIN && weighting != R2X_FDK_PARKER && weighting != R2X_FDK_HALF_FAN)
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad weighting (0 = plain, 1 = Parker, 2 = half fan)");
    const double pi = 3.141592653589793;
    FdkWeights fw;
    if (weighting == R2X_FDK_PARKER) {
        if (n_views < 2) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad N (a short scan needs >= 2 views)");
        if (!view_weights) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad pointer (view_weights NULL)");
        // Parker weights assume each ray's conjugate is on the detector, which a horizontal offset breaks
        if (shift_u != 0.0f)
            return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad shift_u (a short scan needs shift_u = 0)");
        // the arc must hold pi plus the full fan (within float rounding of the arc) and stay short of a full circle
        const double need = pi + (mode == 1 ? 2.0 * std::atan((double)tan_fovx) : 0.0);
        if (!(std::isfinite(arc) && (double)arc >= need - 1e-6 && (double)arc < 2.0 * pi))
            return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad arc (needs pi + 2 atan(tan_fovx) <= arc < 2 pi)");
        fw.vw = (const float2*)view_weights;
        fw.arc = arc;
        fw.delta = (float)(0.5 * ((double)arc - pi));
    }
    if (weighting == R2X_FDK_HALF_FAN) {
        // the rotation axis strictly inside the detector and off its centre, 0 < |t_u| < W / 2
        if (!(shift_u != 0.0f && 2.0 * std::fabs((double)shift_u) < (double)W))
            return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad shift_u for half fan (needs 0 < |shift_u| < W / 2)");
        const double fan = mode == 1 ? (double)tan_fovx : 1.0;
        fw.fan = (float)fan;
        fw.hf_inv_delta = (float)(1.0 / ((1.0 - 2.0 * std::fabs((double)shift_u) / W) * fan));
        fw.hf_sigma = shift_u > 0.0f ? 1.0f : -1.0f;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    float* q = (float*)(((size_t)scratch + 255) & ~(size_t)255);
    const float su = (float)(2.0 * (double)shift_u / W), sv = (float)(-2.0 * (double)shift_v / H);
    if (int rc = fdk_filter(st, weighting, window, n_views, H, W, projs, tan_fovx, tan_fovy, mode, dso, su, sv, fw, q))
        return rc;
    // Parker's dbeta_v already holds each view's share of the arc
    const float scale = weighting == R2X_FDK_PARKER ? 1.0f : (float)(pi / n_views);
    return fdk_backproject(st, n_views, H, W, q, viewmatrices, projmatrices, mode, dso, nx, ny, nz, sx, sy, sz, cx, cy,
                           cz, scale, out_volume);
}

int r2x_fdk_filter(void* stream, int n_views, int H, int W, const float* projs, float tan_fovx, float tan_fovy,
                   int mode, float dso, float* filtered) {
    if (n_views < 1 || H < 1 || W < 1 || W > r2x::FDK_MAX_W || (long long)n_views * H > 0x7fffffffLL)
        return r2x::fail_msg(R2X_ERR_INVALID, "r2x_fdk_filter: bad N/H/W");
    if (mode != 0 && mode != 1) return r2x::fail_msg(R2X_ERR_INVALID, "r2x_fdk_filter: bad mode");
    if (mode == 1 && !(dso > 0.0f && tan_fovx > 0.0f && tan_fovy > 0.0f))
        return r2x::fail_msg(R2X_ERR_INVALID, "r2x_fdk_filter: bad DSO / tan_fov");
    if (!projs || !filtered) return r2x::fail_msg(R2X_ERR_INVALID, "r2x_fdk_filter: bad pointer (NULL)");
    return r2x::fdk_filter((cudaStream_t)stream, R2X_FDK_PLAIN, R2X_FDK_RAM_LAK, n_views, H, W, projs, tan_fovx, tan_fovy, mode, dso,
                           0.0f, 0.0f, r2x::FdkWeights(), filtered);
}

int r2x_fdk_backproject(void* stream, int n_views, int H, int W, const float* filtered, const float* viewmatrices,
                        const float* projmatrices, int mode, float dso, int nx, int ny, int nz, float sx, float sy,
                        float sz, float cx, float cy, float cz, float* out_volume) {
    if (int rc = r2x::fdk_validate(n_views, H, W, filtered, viewmatrices, projmatrices, 1.0f, 1.0f,
                                   mode, dso, nx, ny, nz, sx, sy, sz, out_volume, filtered, (size_t)-1))
        return rc;
    return r2x::fdk_backproject((cudaStream_t)stream, n_views, H, W, filtered, viewmatrices, projmatrices, mode, dso, nx,
                                ny, nz, sx, sy, sz, cx, cy, cz, (float)(3.141592653589793 / n_views), out_volume);
}

}  // extern "C"
