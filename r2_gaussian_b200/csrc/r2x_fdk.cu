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
//   fdk_helical_kernel      r2x_fdk_helical's backprojection of a helical scan (Tang et al. 2006): the same sample
//                           and U^2 weight, times each view's interval dbeta_v and its 3-D redundancy weight
//                           W_Q(nu_0) / sum over the turns and conjugate rays of the voxel's in-plane line of W_Q(nu_k);
//                           each CTA visits only the views within vertical reach of its z-run.
//
// With a per-view geometry table (r2x_fdk_views) the filter kernels take each row's tan_fov, offset and isocentre pitch
// from its view's row (fdk_view_row) and the backprojection each view's DSO; without one, the scalars.
//
// The float64 NumPy statements of the same definitions are oracle/fdk_oracle.py (plain),
// tests/fdk_short_scan_oracle.py (short scan, Parker weights), tests/offset_detector_oracle.py (offset detector,
// half-fan weights) and tests/fdk_helical_oracle.py (helical weights).
#include <cmath>
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_common.cuh"
#include "r2x_project.cuh"

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
// with a pad of L pixels (r2x_fdk_pad): the extended row takes 2 L more samples and the taps reach W - 1 + L
static size_t fdk_filter_pad_smem(int W, int L) { return (size_t)(3 * W + 2 * L + (W + L + 1) / 2) * sizeof(float); }
static size_t fdk_window_pad_smem(int W, int L) { return (size_t)(2 * W + 3 * L) * sizeof(float); }
constexpr size_t FDK_SMEM_OPTIN = 227 * 1024;   // an sm_90 CTA's largest dynamic shared memory

// TABLE: each view's DSO from its row of the per-view geometry table `vg`; without it `dso` for every view.
template <bool CONE, bool TABLE>
__global__ void __launch_bounds__(FDK_BX * FDK_BY) fdk_backproject_kernel(
    int N, int H, int W, const float* __restrict__ q, const float* __restrict__ viewm, const float* __restrict__ projm,
    float dso, int nx, int ny, int nz, float ox, float oy, float oz, float dx, float dy, float dz, float scale,
    float* __restrict__ vol, const double* __restrict__ vg) {
    // per view: projmatrix rows 0, 1, 3 and viewmatrix row 2 as (m[r], m[4+r], m[8+r], m[12+r]), and its DSO
    __shared__ float4 mat[FDK_VCHUNK][4];
    __shared__ float vdso[TABLE ? FDK_VCHUNK : 1];
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
        if (CONE && TABLE && tid < nc) vdso[tid] = (float)vg[(size_t)(c0 + tid) * VG_COLS + VG_DSO];
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
                    const float u = (TABLE ? vdso[v] : dso) * __frcp_rn(zv);
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

// isocentre pitch: cone dDetector_u * DSO / DSD = 2 tan_fovx DSO / W; parallel 2 / W (ndc [-1,1] = scene [-1,1])
__host__ __device__ inline double fdk_pitch(int W, float tanx, int mode, float dso) {
    return mode == 1 ? 2.0 * (double)tanx * (double)dso / W : 2.0 / W;
}

// A per-view table row's filter arguments, rounded and derived exactly as r2x_fdk derives the scalar ones on the host
// (float32 arguments, su / sv and 1 / pitch in float64 rounded once), so a view filters bit for bit as a scalar call
// with its values.
__device__ __forceinline__ void fdk_view_row(const double* __restrict__ row, int H, int W, int cone, float& tanx,
                                             float& tany, float& inv_delta, float& su, float& sv) {
    tanx = (float)row[VG_TANX];
    tany = (float)row[VG_TANY];
    su = (float)(2.0 * (double)(float)row[VG_SHIFT_U] / W);
    sv = (float)(-2.0 * (double)(float)row[VG_SHIFT_V] / H);
    inv_delta = (float)(1.0 / fdk_pitch(W, tanx, cone, (float)row[VG_DSO]));
}

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

// The truncation pad of r2x_fdk_pad (model in include/r2x.h): weighted pixel j of a row e[0 .. W-1] is also mirrored
// into the extension, e[-k] = t_k r[k-1] and e[W-1+k] = t_k r[W-k] for k = 1 .. L, with the roll-off
// t_k = (1 + cos(pi k / (L + 1))) / 2 rounded once from float64.  Each pixel has at most one image on each side, so
// the weighting pass writes the whole extended row with no extra barrier.
__device__ __forceinline__ float fdk_pad_taper(int k, int L) {
    return (float)(0.5 * (1.0 + cospi((double)k / (double)(L + 1))));
}
__device__ __forceinline__ void fdk_pad_mirror(float* __restrict__ e, int W, int L, int j, float p) {
    if (j < L) e[-(j + 1)] = fdk_pad_taper(j + 1, L) * p;
    if (W - j <= L) e[2 * W - 1 - j] = fdk_pad_taper(W - j, L) * p;
}

// Steps 1-2 of FDK with the band-limited Ram-Lak filter, one CTA per detector row: fdk_weight_row, the row staged in
// shared memory between two rows of zeros and filtered with the Ram-Lak taps (shift-invariant, so the same for any
// offset).  PAD (r2x_fdk_pad): the row is extended by `pad` mirrored, rolled-off pixels on each side
// (fdk_pad_mirror) before the zeros, and the taps reach W - 1 + pad; only the W measured pixels are written.
template <int WEIGHT, bool TABLE, bool PAD = false>
__global__ void __launch_bounds__(256) fdk_filter_kernel(int H, int W, const float* __restrict__ projs, float tanx,
                                                         float tany, int cone, float inv_delta, float su, float sv,
                                                         FdkWeights fw, const double* __restrict__ vg,
                                                         float* __restrict__ q, int pad) {
    extern __shared__ float sm[];
    const int L = PAD ? pad : 0;
    float* row = sm;                  // [3W + 2L]: zeros | e[-L .. W-1+L] | zeros
    float* g = sm + 3 * W + 2 * L;    // [(W+L+1)/2]: g[m] = 1 / (pi^2 (2m+1)^2)
    const size_t r = blockIdx.x;      // view * H + detector row
    if (TABLE) fdk_view_row(vg + (r / H) * VG_COLS, H, W, cone, tanx, tany, inv_delta, su, sv);
    fdk_weight_row<WEIGHT>(r, H, W, projs, tanx, tany, cone, su, sv, fw, [&](int j, float p) {
        row[j] = 0.0f;
        row[W + L + j] = p;
        row[2 * W + 2 * L + j] = 0.0f;
        if (PAD) fdk_pad_mirror(row + W + L, W, L, j, p);
    });
    for (int m = threadIdx.x; m < (W + L + 1) / 2; m += blockDim.x) {
        const float k = (float)(2 * m + 1);
        g[m] = 1.0f / (9.869604401089358f * k * k);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < W; j += blockDim.x) {
        const float* c = row + W + L + j;
        // smallest taps first: summed from k = 1 up, the accumulator is near r_j / 4 after a few taps and every tap
        // below half its ulp (k beyond ~3700) is lost, which truncated the filter on wide rows
        float acc = 0.0f;
        for (int m = (W + L) / 2 - 1; m >= 0; --m) acc = fmaf(g[m], c[-(2 * m + 1)] + c[2 * m + 1], acc);
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
// loop.  PAD (r2x_fdk_pad): the staged row is the extended row e[-pad .. W-1+pad] (fdk_pad_mirror), the taps run to
// h[W-1+pad], and pixel j's partners reach j + pad to its left and W - 1 + pad - j to its right.
template <int WEIGHT, int WINDOW, bool TABLE, bool PAD = false>
__global__ void __launch_bounds__(256) fdk_window_kernel(int H, int W, const float* __restrict__ projs, float tanx,
                                                         float tany, int cone, float inv_delta, float su, float sv,
                                                         FdkWeights fw, const double* __restrict__ vg,
                                                         float* __restrict__ q, int pad) {
    extern __shared__ float sm[];
    const int L = PAD ? pad : 0;
    float* row = sm;                  // [W + 2L]: e[-L .. W-1+L]
    float* h = sm + W + 2 * L;        // [W + L]: h[k]
    const size_t r = blockIdx.x;      // view * H + detector row
    if (TABLE) fdk_view_row(vg + (r / H) * VG_COLS, H, W, cone, tanx, tany, inv_delta, su, sv);
    fdk_weight_row<WEIGHT>(r, H, W, projs, tanx, tany, cone, su, sv, fw, [&](int j, float p) {
        row[L + j] = p;
        if (PAD) fdk_pad_mirror(row + L, W, L, j, p);
    });
    for (int k = threadIdx.x; k < W + L; k += blockDim.x) h[k] = (float)fdk_window_tap<WINDOW>(k);
    __syncthreads();
    for (int j = threadIdx.x; j < W; j += blockDim.x) {
        const float* c = row + L + j;
        const int near = min(j + L, W - 1 + L - j), far = max(j + L, W - 1 + L - j);
        const int side = j + L < W - 1 + L - j ? 1 : -1;   // the partner that stays in the row beyond `near`
        float acc = 0.0f;
        for (int k = far; k > near; --k) acc = fmaf(h[k], c[side * k], acc);
        for (int k = near; k > 0; --k) acc = fmaf(h[k], c[-k] + c[k], acc);
        q[r * W + j] = fmaf(h[0], c[0], acc) * inv_delta;
    }
}

using FdkFilterKernel = void (*)(int, int, const float*, float, float, int, float, float, float, FdkWeights,
                                 const double*, float*, int);

template <int WEIGHT, bool TABLE, bool PAD = false>
static FdkFilterKernel fdk_filter_for(int window) {
    switch (window) {
        case R2X_FDK_SHEPP_LOGAN: return fdk_window_kernel<WEIGHT, R2X_FDK_SHEPP_LOGAN, TABLE, PAD>;
        case R2X_FDK_COSINE: return fdk_window_kernel<WEIGHT, R2X_FDK_COSINE, TABLE, PAD>;
        case R2X_FDK_HAMMING: return fdk_window_kernel<WEIGHT, R2X_FDK_HAMMING, TABLE, PAD>;
        case R2X_FDK_HANN: return fdk_window_kernel<WEIGHT, R2X_FDK_HANN, TABLE, PAD>;
        default: return fdk_filter_kernel<WEIGHT, TABLE, PAD>;
    }
}

// the filter stage's dynamic shared memory with a pad of L pixels (the unpadded layouts at L = 0)
static size_t fdk_filter_stage_smem(int window, int W, int L) {
    if (L == 0) return window == R2X_FDK_RAM_LAK ? fdk_filter_smem(W) : fdk_window_smem(W);
    return window == R2X_FDK_RAM_LAK ? fdk_filter_pad_smem(W, L) : fdk_window_pad_smem(W, L);
}

// window: R2X_FDK_RAM_LAK or one of the windowed filters (r2x_fdk's filter field); pad: r2x_fdk_pad's L (0 runs the
// unpadded kernels; a pad comes without a table and without R2X_FDK_HALF_FAN)
static int fdk_filter(cudaStream_t st, int weighting, int window, int N, int H, int W, const float* projs, float tanx,
                      float tany, int mode, float dso, float su, float sv, const FdkWeights& fw, const double* vg,
                      float* q, int pad = 0) {
    // a table comes with R2X_FDK_PLAIN only (r2x_fdk_views)
    auto kernel = pad > 0 ? (weighting == R2X_FDK_PARKER ? fdk_filter_for<R2X_FDK_PARKER, false, true>(window)
                                                         : fdk_filter_for<R2X_FDK_PLAIN, false, true>(window))
                  : vg                            ? fdk_filter_for<R2X_FDK_PLAIN, true>(window)
                  : weighting == R2X_FDK_PARKER   ? fdk_filter_for<R2X_FDK_PARKER, false>(window)
                  : weighting == R2X_FDK_HALF_FAN ? fdk_filter_for<R2X_FDK_HALF_FAN, false>(window)
                                                  : fdk_filter_for<R2X_FDK_PLAIN, false>(window);
    const size_t smem = fdk_filter_stage_smem(window, W, pad);
    if (smem > 48 * 1024)
        R2X_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<(unsigned)((long long)N * H), 256, smem, st>>>(H, W, projs, tanx, tany, mode,
                                                            (float)(1.0 / fdk_pitch(W, tanx, mode, dso)), su, sv, fw, vg,
                                                            q, pad);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

static int fdk_backproject(cudaStream_t st, int N, int H, int W, const float* q, const float* viewm, const float* projm,
                           int mode, float dso, const double* vg, int nx, int ny, int nz, float sx, float sy,
                           float sz, float cx, float cy, float cz, float scale, float* vol) {
    const float dx = sx / nx, dy = sy / ny, dz = sz / nz;
    const float ox = cx - 0.5f * sx + 0.5f * dx, oy = cy - 0.5f * sy + 0.5f * dy, oz = cz - 0.5f * sz + 0.5f * dz;
    const dim3 grid((ny + FDK_BX - 1) / FDK_BX, (nx + FDK_BY - 1) / FDK_BY, (nz + FDK_ZR - 1) / FDK_ZR);
    const dim3 block(FDK_BX, FDK_BY);
    // parallel beam reads no DSO
    auto kernel = mode == 1 ? (vg ? fdk_backproject_kernel<true, true> : fdk_backproject_kernel<true, false>)
                            : fdk_backproject_kernel<false, false>;
    kernel<<<grid, block, 0, st>>>(N, H, W, q, viewm, projm, dso, nx, ny, nz, ox, oy, oz, dx, dy, dz, scale, vol, vg);
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

// r2x_fdk, and r2x_fdk_views with the scalars standing in for its table (vg) in the checks
static int fdk_run(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
                   const float* projmatrices, float tan_fovx, float tan_fovy, int mode, float shift_u, float shift_v,
                   int weighting, const float* view_weights, float arc, float dso, int nx, int ny, int nz, float sx,
                   float sy, float sz, float cx, float cy, float cz, float* out_volume, void* scratch,
                   size_t scratch_bytes, const double* vg, int pad = 0) {
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
    if (int rc = fdk_filter(st, weighting, window, n_views, H, W, projs, tan_fovx, tan_fovy, mode, dso, su, sv, fw, vg,
                            q, pad))
        return rc;
    // Parker's dbeta_v already holds each view's share of the arc
    const float scale = weighting == R2X_FDK_PARKER ? 1.0f : (float)(pi / n_views);
    return fdk_backproject(st, n_views, H, W, q, viewmatrices, projmatrices, mode, dso, vg, nx, ny, nz, sx, sy, sz, cx,
                           cy, cz, scale, out_volume);
}

// ---- helical FDK (r2x_fdk_helical): Tang et al. 2006's 3-D redundancy weight in the backprojection ----------------

// The scalars of a helical backprojection: the helix z_s(beta) = z0 + h beta (z0 in float64, the kernel forms each
// view's z_s in float64 and rounds it once), the arc [beta_lo, beta_lo + arc), the rotation centre (c_x, c_y), and the
// weight W_Q's Q with band = 1 / (2 (1 - Q)) (0 for Q = 1).  reach bounds |Z - z_s(beta_v)| below which a view can
// reach a voxel: (DSO + the grid's largest in-plane radius about the centre) * tan_fovy, widened by 1e-3.
struct FdkHelix {
    double z0 = 0.0, h = 0.0, beta_lo = 0.0, c_x = 0.0, c_y = 0.0;
    float arc = 0.0f, dso = 0.0f, tany = 0.0f, q = 1.0f, band = 0.0f, reach = 0.0f;
};

// W_Q(nu): 1 for |nu| <= Q, cos^2(pi/2 (|nu| - Q) / (1 - Q)) up to 1, 0 from |nu| = 1 on.
__device__ __forceinline__ float fdk_helix_wq(float nu, float q, float band) {
    const float a = fabsf(nu);
    if (a >= 1.0f) return 0.0f;
    if (a <= q) return 1.0f;
    const float c = cospif((a - q) * band);
    return c * c;
}

// view v's source height z_s(beta_v), rounded once; the window search and the staging both read it from here, so
// both see the same value.
__device__ __forceinline__ float fdk_helix_zs(const double* __restrict__ beta, int v, const FdkHelix& hx) {
    return (float)fma(hx.h, beta[v], hx.z0);
}

// First view index in [0, N) whose key sgn * z_s(beta_v) is > lo (strict) or >= lo; the keys do not decrease with v.
__device__ __forceinline__ int fdk_helix_search(const double* __restrict__ beta, int N, const FdkHelix& hx, float sgn,
                                                float lo, bool strict) {
    int a = 0, b = N;
    while (a < b) {
        const int m = (a + b) >> 1;
        const float key = sgn * fdk_helix_zs(beta, m, hx);
        if (strict ? key > lo : key >= lo) b = m;
        else a = m + 1;
    }
    return a;
}

// Helical FDK backprojection, one thread per (x, y) column and FDK_ZR voxels along z as fdk_backproject_kernel, each
// view sampled as there and weighted by dbeta_v * w(beta_v, x) * U^2.  The CTA loops over the contiguous views whose
// source height lies within `reach` of its z-run (found by binary search; a view outside it has W_Q(nu_0) = 0 at every
// voxel of the CTA, so the skip drops exact zeros).  Per (column, view) it sets up gamma, L and the candidates' m
// ranges once (only the turns whose source lies within vertical reach of the run), then per voxel sums W_Q over them.
__global__ void __launch_bounds__(FDK_BX * FDK_BY) fdk_helical_kernel(
    int N, int H, int W, const float* __restrict__ q, const float* __restrict__ viewm, const float* __restrict__ projm,
    const double* __restrict__ beta, const double* __restrict__ dbeta, FdkHelix hx, int nx, int ny, int nz, float ox,
    float oy, float oz, float dx, float dy, float dz, float* __restrict__ vol) {
    // per view: projmatrix rows 0, 1, 3 and viewmatrix row 2 as fdk_backproject_kernel's; the source (S_x, S_y) and
    // (cos beta, sin beta); z_s, beta - beta_lo and dbeta
    __shared__ float4 mat[FDK_VCHUNK][4];
    __shared__ float4 src[FDK_VCHUNK];
    __shared__ float4 hel[FDK_VCHUNK];
    const int y = blockIdx.x * FDK_BX + threadIdx.x;
    const int x = blockIdx.y * FDK_BY + threadIdx.y;
    const int z0 = blockIdx.z * FDK_ZR;
    const int tid = threadIdx.y * FDK_BX + threadIdx.x;
    const bool live = x < nx && y < ny;
    const float X = fmaf((float)x, dx, ox), Y = fmaf((float)y, dy, oy), Z0 = fmaf((float)z0, dz, oz);
    const float Z1 = fmaf((float)(FDK_ZR - 1), dz, Z0);   // the run's last voxel (past nz too: only widens the bounds)
    const float half_w = 0.5f * (float)W, half_h = 0.5f * (float)H;
    const float cen_w = 0.5f * (float)(W - 1), cen_h = 0.5f * (float)(H - 1);
    const size_t view_stride = (size_t)H * W;
    const float two_pi = 6.28318530717958648f, pi = 3.14159265358979324f;
    const float turn = (float)(6.283185307179586 * hx.h);   // z_s gained per turn
    float acc[FDK_ZR];
#pragma unroll
    for (int k = 0; k < FDK_ZR; ++k) acc[k] = 0.0f;

    // the view window: z_s(beta_v) within reach of [Z0, Z1]; z_s is monotone in v (sign sgn), constant for h = 0
    int vb = 0, ve = N;
    if (hx.h != 0.0) {
        const float sgn = hx.h > 0.0 ? 1.0f : -1.0f;
        const float lo = sgn > 0.0f ? Z0 - hx.reach : -(Z1 + hx.reach);
        const float hi = sgn > 0.0f ? Z1 + hx.reach : -(Z0 - hx.reach);
        vb = fdk_helix_search(beta, N, hx, sgn, lo, true);
        ve = fdk_helix_search(beta, N, hx, sgn, hi, false);
    }

    for (int c0 = vb; c0 < ve; c0 += FDK_VCHUNK) {
        const int nc = min(FDK_VCHUNK, ve - c0);
        __syncthreads();
        for (int e = tid; e < nc * 4; e += FDK_BX * FDK_BY) {
            const int v = e >> 2, slot = e & 3;
            const float* m = (slot == 3 ? viewm : projm) + (size_t)(c0 + v) * 16;
            const int rr = slot == 3 ? 2 : (slot == 2 ? 3 : slot);
            mat[v][slot] = make_float4(m[rr], m[4 + rr], m[8 + rr], m[12 + rr]);
        }
        if (tid < nc) {
            const double b = beta[c0 + tid];
            double sb, cb;
            sincos(b, &sb, &cb);
            src[tid] = make_float4((float)fma((double)hx.dso, cb, hx.c_x), (float)fma((double)hx.dso, sb, hx.c_y),
                                   (float)cb, (float)sb);
            hel[tid] = make_float4(fdk_helix_zs(beta, c0 + tid, hx), (float)(b - hx.beta_lo), (float)dbeta[c0 + tid],
                                   0.0f);
        }
        __syncthreads();
        if (!live) continue;
        for (int v = 0; v < nc; ++v) {
            const float4 S = src[v], G = hel[v];
            const float zs = G.x, brel = G.y;
            // in-plane: d = x - source; zin = L cos(gamma) along the central ray -(cos beta, sin beta), sg = L sin(gamma)
            const float ddx = X - S.x, ddy = Y - S.y;
            const float zin = -fmaf(S.z, ddx, S.w * ddy);
            if (!(zin > 0.0f)) continue;
            const float inv0 = __frcp_rn(zin * hx.tany);
            // nu_0 is affine in z: all of the run off the detector on one side gives W_Q(nu_0) = 0 at every voxel
            const float nu_a = (Z0 - zs) * inv0, nu_b = (Z1 - zs) * inv0;
            if ((nu_a >= 1.0f && nu_b >= 1.0f) || (nu_a <= -1.0f && nu_b <= -1.0f)) continue;
            const float sg = fmaf(S.w, ddx, -S.z * ddy);
            const float gam = atan2f(sg, zin);
            const float l2 = fmaf(zin, zin, sg * sg);
            // the conjugate's L_c cos(gamma) = 2 DSO cos^2(gamma) - L cos(gamma); none when the voxel is off the circle
            const float zc = 2.0f * hx.dso * zin * (zin / l2) - zin;
            const float invc = zc > 0.0f ? __frcp_rn(zc * hx.tany) : 0.0f;
            const float cbase = fmaf(2.0f, gam, pi);   // conjugate at beta + pi + 2 gamma + 2 pi m
            // m ranges: beta_k in [beta_lo, beta_lo + arc), and (h != 0) source within reach of the run
            float dlo = ceilf(-brel / two_pi), dhi = ceilf((hx.arc - brel) / two_pi) - 1.0f;
            float clo = ceilf(-(brel + cbase) / two_pi), chi = ceilf((hx.arc - brel - cbase) / two_pi) - 1.0f;
            if (turn != 0.0f) {
                const float r0 = zin * hx.tany, rc = zc * hx.tany;
                const float a0 = (Z0 - zs - r0) / turn, b0 = (Z1 - zs + r0) / turn;
                dlo = fmaxf(dlo, floorf(fminf(a0, b0)));
                dhi = fminf(dhi, ceilf(fmaxf(a0, b0)));
                const float ac = (Z0 - zs - rc) / turn - cbase / two_pi, bc = (Z1 - zs + rc) / turn - cbase / two_pi;
                clo = fmaxf(clo, floorf(fminf(ac, bc)));
                chi = fminf(chi, ceilf(fmaxf(ac, bc)));
            }
            if (!(invc > 0.0f)) chi = clo - 1.0f;
            const int mdl = (int)dlo, mdh = (int)dhi, mcl = (int)clo, mch = (int)chi;
            float wsum[FDK_ZR];
#pragma unroll
            for (int k = 0; k < FDK_ZR; ++k) wsum[k] = 0.0f;
            for (int m = mdl; m <= mdh; ++m) {
                const float zk = fmaf((float)m, turn, zs);
#pragma unroll
                for (int k = 0; k < FDK_ZR; ++k)
                    wsum[k] += fdk_helix_wq((fmaf((float)k, dz, Z0) - zk) * inv0, hx.q, hx.band);
            }
            for (int m = mcl; m <= mch; ++m) {
                const float zk = fmaf(fmaf((float)m, two_pi, cbase), (float)hx.h, zs);
#pragma unroll
                for (int k = 0; k < FDK_ZR; ++k)
                    wsum[k] += fdk_helix_wq((fmaf((float)k, dz, Z0) - zk) * invc, hx.q, hx.band);
            }
            const float4 P0 = mat[v][0], P1 = mat[v][1], P3 = mat[v][2], V2 = mat[v][3];
            const float ax = fmaf(P0.z, Z0, fmaf(P0.y, Y, fmaf(P0.x, X, P0.w)));
            const float ay = fmaf(P1.z, Z0, fmaf(P1.y, Y, fmaf(P1.x, X, P1.w)));
            const float aw = fmaf(P3.z, Z0, fmaf(P3.y, Y, fmaf(P3.x, X, P3.w))) + 1e-7f;  // the rasterizer's divide
            const float sx = P0.z * dz, sy = P1.z * dz, sw = P3.z * dz;
            const float av = fmaf(V2.z, Z0, fmaf(V2.y, Y, fmaf(V2.x, X, V2.w))), sv = V2.z * dz;
            const float* qv = q + (size_t)(c0 + v) * view_stride;
#pragma unroll
            for (int k = 0; k < FDK_ZR; ++k) {
                const float fk = (float)k;
                const float w0 = fdk_helix_wq((fmaf(fk, dz, Z0) - zs) * inv0, hx.q, hx.band);
                if (!(w0 > 0.0f)) continue;        // wsum >= w0 > 0 from here on
                const float zv = fmaf(fk, sv, av);
                if (!(zv > 0.0f)) continue;
                const float u = hx.dso * __frcp_rn(zv);
                const float w = u * u * (G.z * (w0 / wsum[k]));
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
        if (z0 + k < nz) out[z0 + k] = acc[k];
}

// r2x_fdk_helical: the checks (all before any CUDA work), then the plain filter and the helical backprojection.
static int fdk_helical_run(void* stream, int N, int H, int W, const float* projs, const float* viewm, const float* projm,
                           float tanx, float tany, int mode, int weighting, float dso, const double* beta,
                           const double* dbeta, const double* beta_host, double z0, double pitch, double beta_lo,
                           double beta_hi, double c_x, double c_y, float q_param, int nx, int ny, int nz, float sx,
                           float sy, float sz, float cx, float cy, float cz, float* out, void* scratch,
                           size_t scratch_bytes) {
    if (mode != 1)
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk_helical: bad mode (cone beam only; parallel-beam helices are not "
                                         "supported)");
    if (int rc = fdk_validate(N, H, W, projs, viewm, projm, tanx, tany, mode, dso, nx, ny, nz, sx, sy, sz, out, scratch,
                              scratch_bytes))
        return rc;
    if (!beta || !dbeta || !beta_host) return fail_msg(R2X_ERR_INVALID, "r2x_fdk_helical: bad pointer (beta, dbeta or "
                                                                        "beta_host NULL)");
    if (weighting < 0 || (weighting & 0xff) != R2X_FDK_PLAIN || (weighting & ~0xff) > R2X_FDK_HANN)
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk_helical: bad weighting (the filter field only: 0x000 = Ram-Lak, "
                                         "0x100 = Shepp-Logan, 0x200 = cosine, 0x300 = Hamming, 0x400 = Hann)");
    const double h[6] = {z0, pitch, beta_lo, beta_hi, c_x, c_y};
    for (double v : h)
        if (!std::isfinite(v))
            return fail_msg(R2X_ERR_INVALID, "r2x_fdk_helical: bad helix (z0, pitch, beta_lo, beta_hi, c_x, c_y must "
                                             "be finite)");
    if (!(q_param >= 0.0f && q_param <= 1.0f)) return fail_msg(R2X_ERR_INVALID, "r2x_fdk_helical: bad Q (needs 0 <= Q "
                                                                                 "<= 1)");
    for (int v = 0; v < N; ++v)
        if (!std::isfinite(beta_host[v]) || (v > 0 && !(beta_host[v] > beta_host[v - 1])))
            return fail_msg(R2X_ERR_INVALID, "r2x_fdk_helical: bad beta (must be finite and strictly increasing)");
    if (!(beta_lo <= beta_host[0] && beta_host[N - 1] < beta_hi))
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk_helical: bad arc (needs beta_lo <= beta[0] and beta[N-1] < beta_hi)");
    const double two_pi = 6.283185307179586;
    if (!(beta_hi - beta_lo >= two_pi - 1e-6))
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk_helical: bad arc (beta_hi - beta_lo must be at least 2 pi; a circular "
                                         "short scan takes R2X_FDK_PARKER)");
    const float dx = sx / nx, dy = sy / ny, dz = sz / nz;
    const float ox = cx - 0.5f * sx + 0.5f * dx, oy = cy - 0.5f * sy + 0.5f * dy, oz = cz - 0.5f * sz + 0.5f * dz;
    // the grid's largest in-plane radius about the rotation centre: the farthest corner voxel centre
    double rmax = 0.0;
    for (int i = 0; i < 4; ++i) {
        const double gx = (double)ox + (i & 1 ? (double)(nx - 1) * dx : 0.0) - c_x;
        const double gy = (double)oy + (i & 2 ? (double)(ny - 1) * dy : 0.0) - c_y;
        rmax = std::fmax(rmax, std::sqrt(gx * gx + gy * gy));
    }
    FdkHelix hx;
    hx.z0 = z0;
    hx.h = pitch;
    hx.beta_lo = beta_lo;
    hx.c_x = c_x;
    hx.c_y = c_y;
    hx.arc = (float)(beta_hi - beta_lo);
    hx.dso = dso;
    hx.tany = tany;
    hx.q = q_param;
    hx.band = q_param < 1.0f ? (float)(0.5 / (1.0 - (double)q_param)) : 0.0f;
    hx.reach = (float)(((double)dso + rmax) * (double)tany * (1.0 + 1e-3));
    const cudaStream_t st = (cudaStream_t)stream;
    float* qf = (float*)(((size_t)scratch + 255) & ~(size_t)255);
    if (int rc = fdk_filter(st, R2X_FDK_PLAIN, weighting & ~0xff, N, H, W, projs, tanx, tany, mode, dso, 0.0f, 0.0f,
                            FdkWeights(), nullptr, qf))
        return rc;
    const dim3 grid((ny + FDK_BX - 1) / FDK_BX, (nx + FDK_BY - 1) / FDK_BY, (nz + FDK_ZR - 1) / FDK_ZR);
    fdk_helical_kernel<<<grid, dim3(FDK_BX, FDK_BY), 0, st>>>(N, H, W, qf, viewm, projm, beta, dbeta, hx, nx, ny, nz,
                                                              ox, oy, oz, dx, dy, dz, out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace r2x

extern "C" {

size_t r2x_fdk_scratch_bytes(int n_views, int H, int W) { return r2x::fdk_scratch_bytes(n_views, H, W); }

int r2x_fdk(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
            const float* projmatrices, float tan_fovx, float tan_fovy, int mode, float shift_u, float shift_v,
            int weighting, const float* view_weights, float arc, float dso, int nx, int ny, int nz, float sx, float sy,
            float sz, float cx, float cy, float cz, float* out_volume, void* scratch, size_t scratch_bytes) {
    return r2x::fdk_run(stream, n_views, H, W, projs, viewmatrices, projmatrices, tan_fovx, tan_fovy, mode, shift_u,
                        shift_v, weighting, view_weights, arc, dso, nx, ny, nz, sx, sy, sz, cx, cy, cz, out_volume,
                        scratch, scratch_bytes, nullptr);
}

int r2x_fdk_pad(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
                const float* projmatrices, float tan_fovx, float tan_fovy, int mode, float shift_u, float shift_v,
                int weighting, const float* view_weights, float arc, float dso, int nx, int ny, int nz, float sx,
                float sy, float sz, float cx, float cy, float cz, float* out_volume, void* scratch, size_t scratch_bytes,
                int pad) {
    using namespace r2x;
    if (pad < 0 || pad > W) return fail_msg(R2X_ERR_INVALID, "r2x_fdk_pad: bad pad (needs 0 <= pad <= W)");
    if (weighting >= 0 && (weighting & 0xff) == R2X_FDK_HALF_FAN)
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk_pad: bad weighting (no pad with R2X_FDK_HALF_FAN: an offset "
                                         "detector's truncation is deliberate and its weights already handle it)");
    if (W <= FDK_MAX_W && fdk_filter_stage_smem(weighting & ~0xff, W, pad) > FDK_SMEM_OPTIN)
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk_pad: bad pad (the padded row and its taps exceed 227 KB of shared "
                                         "memory)");
    return fdk_run(stream, n_views, H, W, projs, viewmatrices, projmatrices, tan_fovx, tan_fovy, mode, shift_u,
                   shift_v, weighting, view_weights, arc, dso, nx, ny, nz, sx, sy, sz, cx, cy, cz, out_volume, scratch,
                   scratch_bytes, nullptr, pad);
}

int r2x_fdk_views(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
                  const float* projmatrices, int mode, int weighting, int nx, int ny, int nz, float sx, float sy,
                  float sz, float cx, float cy, float cz, const double* view_geometry,
                  const double* view_geometry_host, float* out_volume, void* scratch, size_t scratch_bytes) {
    using namespace r2x;
    if (mode != 0 && mode != 1) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad mode (0 = parallel, 1 = cone)");
    if (n_views < 1) return fail_msg(R2X_ERR_INVALID, "r2x_fdk: bad N/H/W (each must be >= 1)");
    if ((weighting & 0xff) == R2X_FDK_PARKER || (weighting & 0xff) == R2X_FDK_HALF_FAN)
        return fail_msg(R2X_ERR_INVALID, "r2x_fdk_views: bad weighting (Parker and half-fan weights assume one fixed "
                                         "circle; a per-view table takes R2X_FDK_PLAIN only)");
    if (int rc = view_geometry_check("r2x_fdk_views", n_views, mode, view_geometry, view_geometry_host, false))
        return rc;
    const double* row0 = view_geometry_host;
    return fdk_run(stream, n_views, H, W, projs, viewmatrices, projmatrices, (float)row0[VG_TANX],
                   (float)row0[VG_TANY], mode, (float)row0[VG_SHIFT_U], (float)row0[VG_SHIFT_V], weighting, nullptr,
                   0.0f, (float)row0[VG_DSO], nx, ny, nz, sx, sy, sz, cx, cy, cz, out_volume, scratch, scratch_bytes,
                   view_geometry);
}

int r2x_fdk_helical(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
                    const float* projmatrices, float tan_fovx, float tan_fovy, int mode, int weighting, float dso,
                    const double* beta, const double* dbeta, const double* beta_host, double z0, double pitch,
                    double beta_lo, double beta_hi, double c_x, double c_y, float q, int nx, int ny, int nz, float sx,
                    float sy, float sz, float cx, float cy, float cz, float* out_volume, void* scratch,
                    size_t scratch_bytes) {
    return r2x::fdk_helical_run(stream, n_views, H, W, projs, viewmatrices, projmatrices, tan_fovx, tan_fovy, mode,
                                weighting, dso, beta, dbeta, beta_host, z0, pitch, beta_lo, beta_hi, c_x, c_y, q, nx,
                                ny, nz, sx, sy, sz, cx, cy, cz, out_volume, scratch, scratch_bytes);
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
                           0.0f, 0.0f, r2x::FdkWeights(), nullptr, filtered);
}

int r2x_fdk_backproject(void* stream, int n_views, int H, int W, const float* filtered, const float* viewmatrices,
                        const float* projmatrices, int mode, float dso, int nx, int ny, int nz, float sx, float sy,
                        float sz, float cx, float cy, float cz, float* out_volume) {
    if (int rc = r2x::fdk_validate(n_views, H, W, filtered, viewmatrices, projmatrices, 1.0f, 1.0f,
                                   mode, dso, nx, ny, nz, sx, sy, sz, out_volume, filtered, (size_t)-1))
        return rc;
    return r2x::fdk_backproject((cudaStream_t)stream, n_views, H, W, filtered, viewmatrices, projmatrices, mode, dso,
                                nullptr, nx, ny, nz, sx, sy, sz, cx, cy, cz, (float)(3.141592653589793 / n_views),
                                out_volume);
}

}  // extern "C"
