// r2x_prepare.cu -- raw processed cone-beam projections -> the detector stack a real-scan scene stores
// (r2x_projection_prepare, include/r2x.h; r2_gaussian_b200/generate_real_data.py streams a scan through it).
//
// One thread per output pixel (view, row, column), column fastest.  The pixel's value is the reference's per-view chain
// (data_generator/real_dataset/generate_data.py:91-109) evaluated at the source pixels it needs, in the same arithmetic:
//   P(r, c) = r + 5 < H0 ? max0(float32(img[r + 5, c] / rescale * object_scale)) : 0     (float64, one rounding;
//             max0 sets negatives to 0 and keeps -0 and NaN, as p[p < 0] = 0 does)
//   subsample 1: out = P.  Else the float32 INTER_LINEAR resize of P to int(H0 / s) x int(W0 / s) that cv2.resize runs
//   (its IPP path, tests/real_data_oracle.py): per axis x = (d + 0.5) (src / dst) - 0.5 in float64, i = floor(x),
//   t = float32(x - i), neighbours i and min(i + 1, src - 1); columns first, h = fma(tx, P(., j1) - P(., j0), P(., j0)),
//   then rows, out = fma(ty, h(i1) - h(i0), h(i0)); the resized image is read at (row0 + r, col0 + c) (the crop).
// Each output reads its 2 x 2 source pixels straight from the float64 input; nothing is staged.  No atomics, 64-bit
// indexing, bitwise reproducible and independent of how the views are split into calls.
#include <cmath>
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_common.cuh"

namespace r2x {
namespace {

constexpr int PREP_THREADS = 256;
constexpr int PREP_SHIFT_ROWS = 5;          // the FIPS data description: the image sits 5 rows low
constexpr int PREP_BLOCKS_PER_SM = 16;      // grid-stride beyond this: a 721-view full-resolution chunk is ~10^9 pixels

struct PrepGeom {
    int H0, W0;          // raw image
    int Hr, Wr;          // resized (H0, W0 when subsample == 1)
    int row0, col0;      // crop offset into the resized image
    int H, W;            // output
    int resize;
    double sy, sx;       // H0 / Hr, W0 / Wr
    double rescale, object_scale;
};

// P(r, c) of one view: scaled, clamped, moved up 5 rows
__device__ __forceinline__ float prep_pixel(const double* __restrict__ img, const PrepGeom& g, int r, int c) {
    const int rs = r + PREP_SHIFT_ROWS;
    if (rs >= g.H0) return 0.0f;
    const float p = __double2float_rn(__dmul_rn(__ddiv_rn(img[(size_t)rs * g.W0 + c], g.rescale), g.object_scale));
    return p < 0.0f ? 0.0f : p;
}

// i0, i1 and t of destination index d on an axis of n_src source samples (scale = n_src / n_dst)
__device__ __forceinline__ void prep_taps(int d, double scale, int n_src, int& i0, int& i1, float& t) {
    double x = __dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);
    x = x < 0.0 ? 0.0 : x;
    const double f = floor(x);
    i0 = (int)f;
    i1 = i0 + 1 < n_src ? i0 + 1 : n_src - 1;
    t = __double2float_rn(__dsub_rn(x, f));
}

__global__ void __launch_bounds__(PREP_THREADS) projection_prepare_kernel(long long n_out, PrepGeom g,
                                                                          const double* __restrict__ img,
                                                                          float* __restrict__ out) {
    const long long per_view = (long long)g.H * g.W;
    for (long long o = (long long)blockIdx.x * PREP_THREADS + threadIdx.x; o < n_out;
         o += (long long)gridDim.x * PREP_THREADS) {
        const long long v = o / per_view;
        const int rem = (int)(o - v * per_view);
        const int r = rem / g.W, c = rem - r * g.W;
        const double* src = img + (size_t)v * g.H0 * g.W0;
        float val;
        if (!g.resize) {
            val = prep_pixel(src, g, r, c);
        } else {
            int i0, i1, j0, j1;
            float ty, tx;
            prep_taps(g.row0 + r, g.sy, g.H0, i0, i1, ty);
            prep_taps(g.col0 + c, g.sx, g.W0, j0, j1, tx);
            const float a0 = prep_pixel(src, g, i0, j0), b0 = prep_pixel(src, g, i0, j1);
            const float a1 = prep_pixel(src, g, i1, j0), b1 = prep_pixel(src, g, i1, j1);
            const float h0 = __fmaf_rn(tx, __fsub_rn(b0, a0), a0);
            const float h1 = __fmaf_rn(tx, __fsub_rn(b1, a1), a1);
            val = __fmaf_rn(ty, __fsub_rn(h1, h0), h0);
        }
        out[o] = val;
    }
}

// the output geometry of (H0, W0, subsample), or a message naming what is wrong
const char* prep_geometry(int H0, int W0, int subsample, PrepGeom& g) {
    if (H0 < 1 || W0 < 1) return "r2x_projection_prepare: bad image size (H0, W0 >= 1)";
    if (subsample < 1) return "r2x_projection_prepare: bad subsample (must be >= 1)";
    g.H0 = H0;
    g.W0 = W0;
    g.resize = subsample != 1;
    if (!g.resize) {
        g.Hr = g.H = H0;
        g.Wr = g.W = W0;
        g.row0 = g.col0 = 0;
    } else {
        g.Hr = (int)((double)H0 / (double)subsample);
        g.Wr = (int)((double)W0 / (double)subsample);
        if (g.Hr < 1 || g.Wr < 1)
            return "r2x_projection_prepare: bad subsample (int(H0 / subsample) and int(W0 / subsample) must be >= 1)";
        const int off = (g.Hr > g.Wr ? g.Hr - g.Wr : g.Wr - g.Hr) / 2;
        g.row0 = g.Hr > g.Wr ? off : 0;
        g.col0 = g.Wr > g.Hr ? off : 0;
        g.H = g.Hr - 2 * g.row0;
        g.W = g.Wr - 2 * g.col0;
    }
    if ((long long)g.H * g.W >= (1LL << 31)) return "r2x_projection_prepare: bad image size (H * W must be < 2^31)";
    g.sy = (double)H0 / (double)g.Hr;
    g.sx = (double)W0 / (double)g.Wr;
    return nullptr;
}

}  // namespace
}  // namespace r2x

extern "C" {

int r2x_projection_prepare_shape(int H0, int W0, int subsample, int* out_hw) {
    using namespace r2x;
    PrepGeom g;
    if (const char* msg = prep_geometry(H0, W0, subsample, g)) return fail_msg(R2X_ERR_INVALID, msg);
    if (!out_hw) return fail_msg(R2X_ERR_INVALID, "r2x_projection_prepare_shape: bad pointer (NULL)");
    out_hw[0] = g.H;
    out_hw[1] = g.W;
    return 0;
}

int r2x_projection_prepare(void* stream, int n_views, int H0, int W0, int subsample, const double* img,
                           double proj_rescale, double object_scale, float* out) {
    using namespace r2x;
    PrepGeom g;
    if (n_views < 1) return fail_msg(R2X_ERR_INVALID, "r2x_projection_prepare: bad n_views (must be >= 1)");
    if (const char* msg = prep_geometry(H0, W0, subsample, g)) return fail_msg(R2X_ERR_INVALID, msg);
    if (!img || !out) return fail_msg(R2X_ERR_INVALID, "r2x_projection_prepare: bad pointer (NULL)");
    if (!(std::isfinite(proj_rescale) && proj_rescale != 0.0))
        return fail_msg(R2X_ERR_INVALID, "r2x_projection_prepare: bad proj_rescale (must be finite and non-zero)");
    if (!std::isfinite(object_scale))
        return fail_msg(R2X_ERR_INVALID, "r2x_projection_prepare: bad object_scale (must be finite)");
    g.rescale = proj_rescale;
    g.object_scale = object_scale;
    int sms = 0;
    R2X_CUDA_OK(sm_count(&sms));
    const long long n_out = (long long)n_views * g.H * g.W;
    const long long want = (n_out + PREP_THREADS - 1) / PREP_THREADS;
    const long long cap = (long long)sms * PREP_BLOCKS_PER_SM;
    const unsigned nblk = (unsigned)(want < cap ? want : cap);
    projection_prepare_kernel<<<nblk, PREP_THREADS, 0, (cudaStream_t)stream>>>(n_out, g, img, out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
