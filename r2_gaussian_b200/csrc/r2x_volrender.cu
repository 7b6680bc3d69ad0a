// r2x_volrender.cu -- ray casting of a float32 volume: emission-absorption compositing and maximum intensity
// projection.  include/r2x.h states the model.
//
// One thread per pixel, R2X_VR_TILE x R2X_VR_TILE pixels per CTA (neighbouring rays fetch neighbouring voxels, so the
// eight corner loads of a sample mostly hit lines a neighbour already brought into L1), frames on gridDim.z so that an
// orbit is one launch.  The LUT is staged in shared memory once per CTA.  The ray set-up (direction, slab interval,
// sample count) and each sample point are float64 with explicit round-to-nearest operations, so no FMA contraction
// can move a sample count or a cell choice away from a plain float64 statement of the model; the interpolation
// weights, the blend and the compositing are float32.  Pixels are independent and nothing is accumulated across
// threads: no atomics, bitwise reproducible.
#include <cmath>
#include <cstdint>
#include <cstdio>

#include "../../include/r2x.h"
#include "r2x_common.cuh"

namespace r2x {
namespace {

constexpr int VR_TILE = R2X_VR_TILE;
constexpr int VR_THREADS = VR_TILE * VR_TILE;
constexpr int VR_MAX_LUT = 4096;                 // 48 KiB of shared memory: the LUT of one CTA at the default limit
constexpr int VR_MAX_GRID = 65535;
constexpr float VR_T_STOP = 1.0f / 65536.0f;     // the ray stops after the first sample that leaves T < 2^-16

struct VrParams {
    int nx, ny, nz, H, W, parallel, mode, K;
    float c0, inv_range;   // t = clamp((v - c0) * inv_range, 0, 1)
    float expo;            // step / unit
    double step;
    float bg[3];
};

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }

// narrow [s0, s1] to the slab 0 <= o + s d <= hi; false when the ray misses it
__device__ __forceinline__ bool slab(double o, double d, double hi, double& s0, double& s1) {
    if (d == 0.0) return o >= 0.0 && o <= hi;
    const double ta = __ddiv_rn(-o, d), tb = __ddiv_rn(dsub(hi, o), d);
    s0 = fmax(s0, fmin(ta, tb));
    s1 = fmin(s1, fmax(ta, tb));
    return true;
}

// sample point along one axis, clamped into [0, hi]: the cell's lower index and the float32 weight
__device__ __forceinline__ int cell(double o, double d, double s, double hi, float& w) {
    const double p = fmin(fmax(dadd(o, dmul(s, d)), 0.0), hi);
    const double i0 = fmin(floor(p), hi - 1.0);
    w = (float)(p - i0);   // exact in float64: p - floor(p), or 1 at the upper face
    return (int)i0;
}

__device__ __forceinline__ float blend(float a, float b, float w) { return (1.0f - w) * a + w * b; }

__device__ __forceinline__ float transfer(const VrParams& q, float v) {
    return fminf(fmaxf((v - q.c0) * q.inv_range, 0.0f), 1.0f);
}

__device__ __forceinline__ float3 lut_colour(const float* __restrict__ lut, int K, float t) {
    if (K == 1) return make_float3(lut[0], lut[1], lut[2]);
    const float pos = t * (float)(K - 1);
    const int j = min((int)floorf(pos), K - 2);
    const float w = pos - (float)j;
    const float* a = lut + 3 * j;
    return make_float3(blend(a[0], a[3], w), blend(a[1], a[4], w), blend(a[2], a[5], w));
}

__global__ void __launch_bounds__(VR_THREADS) volume_render_kernel(VrParams q, const float* __restrict__ vol,
                                                                   const float* __restrict__ cameras,
                                                                   const float* __restrict__ lut,
                                                                   float* __restrict__ out) {
    extern __shared__ float s_lut[];
    const int tid = threadIdx.y * VR_TILE + threadIdx.x;
    for (int i = tid; i < 3 * q.K; i += VR_THREADS) s_lut[i] = __ldg(lut + i);
    __syncthreads();
    const int x = blockIdx.x * VR_TILE + threadIdx.x, y = blockIdx.y * VR_TILE + threadIdx.y;
    if (x >= q.W || y >= q.H) return;
    const float* cam = cameras + (size_t)blockIdx.z * R2X_VR_CAMERA_FLOATS;

    // ---- the ray: a = ((x + 1/2) - W/2) p, b = ((H/2 - y) - 1/2) p
    const double p = __ldg(cam + 12);
    const double a = dmul(((double)x + 0.5) - 0.5 * q.W, p), b = dmul((0.5 * q.H - (double)y) - 0.5, p);
    double o[3], d[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double P = __ldg(cam + c), f = __ldg(cam + 3 + c), r = __ldg(cam + 6 + c), u = __ldg(cam + 9 + c);
        if (q.parallel) {
            o[c] = dadd(dadd(P, dmul(a, r)), dmul(b, u));
            d[c] = f;
        } else {
            o[c] = P;
            d[c] = dadd(dadd(f, dmul(a, r)), dmul(b, u));
        }
    }
    if (!q.parallel) {
        const double n = __dsqrt_rn(dadd(dadd(dmul(d[0], d[0]), dmul(d[1], d[1])), dmul(d[2], d[2])));
#pragma unroll
        for (int c = 0; c < 3; ++c) d[c] = __ddiv_rn(d[c], n);
    }
    const double hx = q.nx - 1, hy = q.ny - 1, hz = q.nz - 1;
    double s0 = 0.0, s1 = INFINITY;
    const bool meets = slab(o[0], d[0], hx, s0, s1) & slab(o[1], d[1], hy, s0, s1) & slab(o[2], d[2], hz, s0, s1) &&
                       s1 >= s0 && s1 < INFINITY;   // s1 is finite for any unit d

    float rgb[3] = {q.bg[0], q.bg[1], q.bg[2]}, alpha = 0.0f;
    if (meets) {
        const long long n = (long long)floor(__ddiv_rn(dsub(s1, s0), q.step)) + 1;
        const long long sz = q.nz, syz = (long long)q.ny * q.nz;
        float C[3] = {0.0f, 0.0f, 0.0f}, T = 1.0f, m = -INFINITY;
        for (long long k = 0; k < n; ++k) {
            const double s = dadd(s0, dmul((double)k, q.step));
            float wx, wy, wz;
            const int ix = cell(o[0], d[0], s, hx, wx), iy = cell(o[1], d[1], s, hy, wy), iz = cell(o[2], d[2], s, hz, wz);
            const float* v = vol + ((long long)ix * q.ny + iy) * sz + iz;
            const float c00 = blend(__ldg(v), __ldg(v + 1), wz), c01 = blend(__ldg(v + sz), __ldg(v + sz + 1), wz);
            const float c10 = blend(__ldg(v + syz), __ldg(v + syz + 1), wz);
            const float c11 = blend(__ldg(v + syz + sz), __ldg(v + syz + sz + 1), wz);
            const float val = blend(blend(c00, c01, wy), blend(c10, c11, wy), wx);
            if (q.mode == R2X_VR_MIP) {
                m = fmaxf(m, val);
                continue;
            }
            const float t = transfer(q, val);
            if (t == 0.0f) continue;   // alpha = 0: C and T are unchanged
            const float al = 1.0f - exp2f(q.expo * log2f(1.0f - t));
            const float3 col = lut_colour(s_lut, q.K, t);
            const float ta = T * al;
            C[0] += ta * col.x;
            C[1] += ta * col.y;
            C[2] += ta * col.z;
            T *= 1.0f - al;
            if (T < VR_T_STOP) break;
        }
        if (q.mode == R2X_VR_MIP) {
            const float3 col = lut_colour(s_lut, q.K, transfer(q, m));
            rgb[0] = col.x;
            rgb[1] = col.y;
            rgb[2] = col.z;
            alpha = 1.0f;
        } else {
#pragma unroll
            for (int c = 0; c < 3; ++c) rgb[c] = C[c] + T * q.bg[c];
            alpha = 1.0f - T;
        }
    }
    const long long px = ((long long)blockIdx.z * q.H + y) * q.W + x;
    reinterpret_cast<float4*>(out)[px] = make_float4(rgb[0], rgb[1], rgb[2], alpha);
}

int bad(const char* what) {
    char msg[200];
    snprintf(msg, sizeof msg, "r2x_volume_render: bad %s", what);
    return fail_msg(R2X_ERR_INVALID, msg);
}

}  // namespace
}  // namespace r2x

extern "C" {

int r2x_volume_render(void* stream, int nx, int ny, int nz, const float* vol, int n_frames, int H, int W,
                      const float* cameras_dev, int parallel, int mode, float c0, float c1, const float* lut_dev, int K,
                      float step, float unit, const float* background, float* out) {
    using namespace r2x;
    if (!vol || !cameras_dev || !lut_dev || !background || !out) return bad("pointer (NULL)");
    if ((uintptr_t)out % 16) return bad("pointer (out is not 16-byte aligned)");
    if (nx < 2 || ny < 2 || nz < 2) return bad("grid (each axis needs >= 2 samples)");
    if (n_frames < 1 || H < 1 || W < 1) return bad("image (n_frames, H and W must be >= 1)");
    // pixel tiles in 64 bits: H + VR_TILE - 1 is past INT_MAX for H within a tile of it
    const long long tiles_y = ((long long)H + VR_TILE - 1) / VR_TILE, tiles_x = ((long long)W + VR_TILE - 1) / VR_TILE;
    if (n_frames > VR_MAX_GRID || tiles_y > VR_MAX_GRID || tiles_x > VR_MAX_GRID)
        return bad("image (frames and pixel tiles per grid dimension must be <= 65535)");
    if (parallel != 0 && parallel != 1) return bad("parallel (0 or 1)");
    if (mode != R2X_VR_COMPOSITE && mode != R2X_VR_MIP) return bad("mode (0 composite, 1 mip)");
    if (K < 1 || K > VR_MAX_LUT) return bad("K (1 to 4096 LUT entries)");
    if (!std::isfinite(c0) || !std::isfinite(c1) || !(c0 < c1)) return bad("clim (finite c0 < c1)");
    const double range = (double)c1 - (double)c0;
    if (!(range <= 3.4028234663852886e38)) return bad("clim (c1 - c0 must be a finite float)");
    const float inv_range = (float)(1.0 / range);
    if (!std::isfinite(step) || !(step > 0.0f)) return bad("step (finite, > 0)");
    const double diag = std::sqrt((double)(nx - 1) * (nx - 1) + (double)(ny - 1) * (ny - 1) + (double)(nz - 1) * (nz - 1));
    if (diag / step > 2147483647.0) return bad("step (more than 2^31 - 1 samples along the box diagonal)");
    if (!std::isfinite(unit) || !(unit > 0.0f)) return bad("unit (finite, > 0)");
    const float expo = (float)((double)step / unit);
    if (!std::isfinite(expo) || !(expo > 0.0f)) return bad("unit (step / unit must be a finite float > 0)");
    for (int c = 0; c < 3; ++c)
        if (!std::isfinite(background[c])) return bad("background (finite)");

    VrParams q;
    q.nx = nx; q.ny = ny; q.nz = nz; q.H = H; q.W = W; q.parallel = parallel; q.mode = mode; q.K = K;
    q.c0 = c0; q.inv_range = inv_range; q.expo = expo; q.step = step;
    for (int c = 0; c < 3; ++c) q.bg[c] = background[c];
    const dim3 grid((unsigned)tiles_x, (unsigned)tiles_y, (unsigned)n_frames);
    volume_render_kernel<<<grid, dim3(VR_TILE, VR_TILE), 3 * K * sizeof(float), (cudaStream_t)stream>>>(
        q, vol, cameras_dev, lut_dev, out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
