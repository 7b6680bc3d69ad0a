// r2x_zoom.cu -- cubic B-spline zoom of a 3-D float64 volume, scipy.ndimage.zoom(x, zoom, order=3, mode="nearest")
// (r2x_volume_place / r2x_zoom_cubic, include/r2x.h; r2_gaussian_b200/resample.py and process_raw_data.py call them).
//
// The input is a *placed* volume: a source of uint8, uint16 or float64 voxels with any non-negative strides, set at an
// offset in a volume of its own shape (zero where the source does not reach: expand_to_cube; a negative offset crops:
// crop_to_cube) and normalised, value = (source - lo) / (hi - lo) in float64.  Placement is folded into the fill of the
// padded buffer, so neither the normalised nor the cubed volume is ever materialised.  The zoom is then scipy's:
//   1. pad by 12 voxels on every side with the edge voxel (np.pad(..., 12, mode="edge"));
//   2. prefilter along axis 0, 1, 2 in turn, in place: gain 6, pole z = sqrt(3) - 2, causal start value
//      sum_{k<30} z^k c[m(k)] with m the mirror index of period 2n - 2, c+[i] = c[i] + z c+[i-1],
//      c-[n-1] = z / (z^2 - 1) (c+[n-1] + z c+[n-2]), c-[i] = z (c-[i+1] - c+[i]);
//   3. output index o on an axis maps to x = o (n - 1) / (out - 1) + 12 (factor 1 when out = 1), f = floor(x),
//      t = x - f, and the 4 x 4 x 4 coefficients f-1 .. f+2 are summed with the cubic B-spline weights.
// One thread per line in the prefilter; along the two outer axes adjacent threads take adjacent lines (coalesced
// loads), along the contiguous axis a warp stages 32 lines x 32 voxels through shared memory.  No atomics: every
// output is written by one thread in a fixed order, so results are bitwise reproducible.  64-bit indexing throughout
// (a padded 1094^3 cube has 1.40e9 voxels).
#include <cmath>
#include <cstdint>
#include <cstdio>

#include "../../include/r2x.h"
#include "r2x_common.cuh"

namespace r2x {
namespace {

constexpr int ZOOM_PAD = 12;              // scipy's pre-padding for the spline prefilter
constexpr int ZOOM_MAX_DIM = 32768;       // placed and output sizes; keeps every row count below 2^31
constexpr int CAUSAL_TERMS = 30;          // z^30 = 1.4e-17: the truncated start value is exact in float64
constexpr int ROW_THREADS = 128;          // fill and gather: one block per row, threads along the contiguous axis
constexpr int ROW_BLOCKS_PER_SM = 16;
constexpr int LINE_THREADS = 128;         // prefilter along an outer axis: one thread per line
constexpr int LINE_BATCH = 8;             // voxels loaded before they are used, per thread
constexpr int TILE = 32;                  // prefilter along the contiguous axis: 32 lines x 32 voxels per warp
constexpr int TILE_WARPS = 4;

struct Place {
    const void* src;
    int s0, s1, s2;
    long long st0, st1, st2;
    int m0, m1, m2;
    int off0, off1, off2;
    double lo, hi;
};

template <typename T>
__device__ __forceinline__ double load_voxel(const void* src, long long i) {
    return (double)static_cast<const T*>(src)[i];
}

// dst[A, B, C] = placed volume at (i - pad, j - pad, k - pad), indices clamped to the placed volume (edge padding)
template <typename T>
__global__ void __launch_bounds__(ROW_THREADS) place_fill_kernel(Place p, int pad, double* __restrict__ dst) {
    const int A = p.m0 + 2 * pad, B = p.m1 + 2 * pad, C = p.m2 + 2 * pad;
    const long long rows = (long long)A * B;
    const double span = __dsub_rn(p.hi, p.lo);
    for (long long row = blockIdx.x; row < rows; row += gridDim.x) {
        const int i = (int)(row / B), j = (int)(row - (long long)i * B);
        const int q0 = min(max(i - pad, 0), p.m0 - 1) - p.off0;
        const int q1 = min(max(j - pad, 0), p.m1 - 1) - p.off1;
        const bool in_row = q0 >= 0 && q0 < p.s0 && q1 >= 0 && q1 < p.s1;
        const long long base = (long long)q0 * p.st0 + (long long)q1 * p.st1;
        double* out = dst + row * C;
        for (int k = threadIdx.x; k < C; k += ROW_THREADS) {
            const int q2 = min(max(k - pad, 0), p.m2 - 1) - p.off2;
            double v = 0.0;
            if (in_row && q2 >= 0 && q2 < p.s2)
                v = __ddiv_rn(__dsub_rn(load_voxel<T>(p.src, base + (long long)q2 * p.st2), p.lo), span);
            out[k] = v;
        }
    }
}

__device__ __forceinline__ int mirror_index(int k, int n) {
    const int r = k % (2 * n - 2);
    return r < n ? r : 2 * n - 2 - r;
}

// prefilter of the lines along an outer axis: line l = (o, k) starts at o * ostride + k and steps by `stride`
__global__ void __launch_bounds__(LINE_THREADS) prefilter_outer_kernel(double* __restrict__ v, long long nlines, int c,
                                                                       long long ostride, long long stride, int n,
                                                                       double z) {
    const long long l = (long long)blockIdx.x * LINE_THREADS + threadIdx.x;
    if (l >= nlines) return;
    const long long o = l / c;
    double* p = v + o * ostride + (l - o * c);
    double acc = 0.0, zk = 1.0;
    for (int t = 0; t < CAUSAL_TERMS; ++t) {
        acc += zk * (6.0 * p[mirror_index(t, n) * stride]);
        zk *= z;
    }
    double prev = acc, pprev = 0.0;
    p[0] = prev;
    for (int e0 = 1; e0 < n; e0 += LINE_BATCH) {
        double x[LINE_BATCH];
#pragma unroll
        for (int u = 0; u < LINE_BATCH; ++u)
            if (e0 + u < n) x[u] = p[(long long)(e0 + u) * stride];
#pragma unroll
        for (int u = 0; u < LINE_BATCH; ++u)
            if (e0 + u < n) {
                pprev = prev;
                prev = 6.0 * x[u] + z * prev;
                p[(long long)(e0 + u) * stride] = prev;
            }
    }
    double cur = z / (z * z - 1.0) * (prev + z * pprev);
    p[(long long)(n - 1) * stride] = cur;
    for (int e0 = n - 2; e0 >= 0; e0 -= LINE_BATCH) {
        double x[LINE_BATCH];
#pragma unroll
        for (int u = 0; u < LINE_BATCH; ++u)
            if (e0 - u >= 0) x[u] = p[(long long)(e0 - u) * stride];
#pragma unroll
        for (int u = 0; u < LINE_BATCH; ++u)
            if (e0 - u >= 0) {
                cur = z * (cur - x[u]);
                p[(long long)(e0 - u) * stride] = cur;
            }
    }
}

// prefilter of the contiguous lines (rows of n voxels): each warp takes 32 adjacent rows and walks them 32 voxels at a
// time through a shared tile, loading and storing whole row segments and recursing one row per lane
__global__ void __launch_bounds__(TILE * TILE_WARPS) prefilter_inner_kernel(double* __restrict__ v, long long nrows,
                                                                           int n, double z) {
    __shared__ double tiles[TILE_WARPS][TILE][TILE + 1];
    const int lane = threadIdx.x & (TILE - 1), w = threadIdx.x / TILE;
    double(*tile)[TILE + 1] = tiles[w];
    const long long row0 = ((long long)blockIdx.x * TILE_WARPS + w) * TILE;
    if (row0 >= nrows) return;
    const int nr = (int)min((long long)TILE, nrows - row0);
    double* base = v + row0 * n;
    auto load = [&](int k0) {
        const int k = k0 + lane;
        if (k < n)
            for (int r = 0; r < nr; ++r) tile[r][lane] = base[(long long)r * n + k];
        __syncwarp();
    };
    auto store = [&](int k0) {
        __syncwarp();
        const int k = k0 + lane;
        if (k < n)
            for (int r = 0; r < nr; ++r) base[(long long)r * n + k] = tile[r][lane];
        __syncwarp();
    };
    const int last = (n - 1) / TILE * TILE;
    const bool mine = lane < nr;     // lanes past the last row only help with the loads and stores
    double prev = 0.0, pprev = 0.0;
    for (int k0 = 0; k0 <= last; k0 += TILE) {
        load(k0);
        const int len = min(TILE, n - k0);
        int kk = mine ? 0 : len;
        if (k0 == 0 && mine) {      // n >= 25, so every mirror index of the start value lies in the first tile
            double acc = 0.0, zk = 1.0;
            for (int t = 0; t < CAUSAL_TERMS; ++t) {
                acc += zk * (6.0 * tile[lane][mirror_index(t, n)]);
                zk *= z;
            }
            prev = acc;
            tile[lane][0] = prev;
            kk = 1;
        }
        for (; kk < len; ++kk) {
            pprev = prev;
            prev = 6.0 * tile[lane][kk] + z * prev;
            tile[lane][kk] = prev;
        }
        if (k0 != last) store(k0);   // the last segment stays in the tile for the anticausal pass
    }
    double cur = 0.0;
    for (int k0 = last; k0 >= 0; k0 -= TILE) {
        if (k0 != last) load(k0);
        int kk = mine ? min(TILE, n - k0) - 1 : -1;
        if (k0 == last && mine) {
            cur = z / (z * z - 1.0) * (prev + z * pprev);
            tile[lane][kk] = cur;
            --kk;
        }
        for (; kk >= 0; --kk) {
            cur = z * (cur - tile[lane][kk]);
            tile[lane][kk] = cur;
        }
        store(k0);
    }
}

// first tap and the 4 cubic B-spline weights of output index o on an axis with coordinate factor f
__device__ __forceinline__ int spline_taps(int o, double f, double w[4]) {
    const double x = __dadd_rn(__dmul_rn((double)o, f), (double)ZOOM_PAD);
    const double fl = floor(x);
    const double t = x - fl, s = 1.0 - t;
    w[0] = s * s * s / 6.0;
    w[1] = (t * t * (t - 2.0) * 3.0 + 4.0) / 6.0;
    w[2] = (s * s * (s - 2.0) * 3.0 + 4.0) / 6.0;
    w[3] = t * t * t / 6.0;
    return (int)fl - 1;
}

// out[O0, O1, O2] from the prefiltered coefficients c[A, B, C]: one block per output row, 64 taps per voxel
__global__ void __launch_bounds__(ROW_THREADS) zoom_gather_kernel(const double* __restrict__ c, int B, int C, int O0,
                                                                  int O1, int O2, double f0, double f1, double f2,
                                                                  double* __restrict__ out) {
    const long long rows = (long long)O0 * O1;
    for (long long row = blockIdx.x; row < rows; row += gridDim.x) {
        const int o0 = (int)(row / O1), o1 = (int)(row - (long long)o0 * O1);
        double wx[4], wy[4];
        const int i0 = spline_taps(o0, f0, wx), j0 = spline_taps(o1, f1, wy);
        for (int o2 = threadIdx.x; o2 < O2; o2 += ROW_THREADS) {
            double wz[4];
            const int k0 = spline_taps(o2, f2, wz);
            double acc = 0.0;
#pragma unroll
            for (int a = 0; a < 4; ++a) {
                double ra = 0.0;
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    const double* q = c + ((long long)(i0 + a) * B + (j0 + b)) * C + k0;
                    ra += wy[b] * (wz[0] * q[0] + wz[1] * q[1] + wz[2] * q[2] + wz[3] * q[3]);
                }
                acc += wx[a] * ra;
            }
            out[row * O2 + o2] = acc;
        }
    }
}

bool bad_dim(int n) { return n < 1 || n > ZOOM_MAX_DIM; }

// the placement of `d`, or a message naming what is wrong
const char* check_place(const char* fn, const r2x_place_desc* d, Place& p) {
    static thread_local char msg[160];
    auto say = [&](const char* what) {
        snprintf(msg, sizeof msg, "%s: %s", fn, what);
        return msg;
    };
    if (!d || !d->src) return say("bad pointer (NULL)");
    if (d->dtype != R2X_PLACE_U8 && d->dtype != R2X_PLACE_U16 && d->dtype != R2X_PLACE_F64)
        return say("bad dtype (R2X_PLACE_U8, R2X_PLACE_U16 or R2X_PLACE_F64)");
    for (int a = 0; a < 3; ++a) {
        if (d->src_shape[a] < 1) return say("bad source shape (each size >= 1)");
        if (d->src_strides[a] < 0) return say("bad source strides (each >= 0)");
        if (bad_dim(d->shape[a])) return say("bad placed shape (each size in [1, 32768])");
    }
    if (!(std::isfinite(d->lo) && std::isfinite(d->hi) && d->hi > d->lo))
        return say("bad lo / hi (finite, hi > lo)");
    p = {d->src, d->src_shape[0], d->src_shape[1], d->src_shape[2], d->src_strides[0], d->src_strides[1],
         d->src_strides[2], d->shape[0], d->shape[1], d->shape[2], d->offset[0], d->offset[1], d->offset[2], d->lo, d->hi};
    return nullptr;
}

int launch_fill(const Place& p, int dtype, int pad, double* dst, cudaStream_t st) {
    int sms = 0;
    R2X_CUDA_OK(sm_count(&sms));
    const long long rows = (long long)(p.m0 + 2 * pad) * (p.m1 + 2 * pad);
    const unsigned nblk = (unsigned)min(rows, (long long)sms * ROW_BLOCKS_PER_SM);
    if (dtype == R2X_PLACE_U8) place_fill_kernel<uint8_t><<<nblk, ROW_THREADS, 0, st>>>(p, pad, dst);
    else if (dtype == R2X_PLACE_U16) place_fill_kernel<uint16_t><<<nblk, ROW_THREADS, 0, st>>>(p, pad, dst);
    else place_fill_kernel<double><<<nblk, ROW_THREADS, 0, st>>>(p, pad, dst);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

double coordinate_factor(int n, int out) { return out > 1 ? (double)(n - 1) / (double)(out - 1) : 1.0; }

}  // namespace
}  // namespace r2x

extern "C" {

size_t r2x_zoom_workspace_bytes(int n0, int n1, int n2) {
    using namespace r2x;
    if (bad_dim(n0) || bad_dim(n1) || bad_dim(n2)) return 0;
    return (size_t)(n0 + 2 * ZOOM_PAD) * (n1 + 2 * ZOOM_PAD) * (n2 + 2 * ZOOM_PAD) * sizeof(double);
}

int r2x_volume_place(void* stream, const r2x_place_desc* desc, double* out) {
    using namespace r2x;
    Place p;
    if (const char* msg = check_place("r2x_volume_place", desc, p)) return fail_msg(R2X_ERR_INVALID, msg);
    if (!out) return fail_msg(R2X_ERR_INVALID, "r2x_volume_place: bad pointer (NULL)");
    return launch_fill(p, desc->dtype, 0, out, (cudaStream_t)stream);
}

int r2x_zoom_cubic(void* stream, const r2x_place_desc* desc, int out0, int out1, int out2, void* workspace,
                   size_t workspace_bytes, double* out) {
    using namespace r2x;
    Place p;
    if (const char* msg = check_place("r2x_zoom_cubic", desc, p)) return fail_msg(R2X_ERR_INVALID, msg);
    if (bad_dim(out0) || bad_dim(out1) || bad_dim(out2))
        return fail_msg(R2X_ERR_INVALID, "r2x_zoom_cubic: bad output shape (each size in [1, 32768])");
    if (!workspace || !out) return fail_msg(R2X_ERR_INVALID, "r2x_zoom_cubic: bad pointer (NULL)");
    if (workspace_bytes < r2x_zoom_workspace_bytes(p.m0, p.m1, p.m2))
        return fail_msg(R2X_ERR_INVALID, "r2x_zoom_cubic: bad workspace (smaller than r2x_zoom_workspace_bytes)");
    const cudaStream_t st = (cudaStream_t)stream;
    double* c = static_cast<double*>(workspace);
    const int A = p.m0 + 2 * ZOOM_PAD, B = p.m1 + 2 * ZOOM_PAD, C = p.m2 + 2 * ZOOM_PAD;
    if (int rc = launch_fill(p, desc->dtype, ZOOM_PAD, c, st)) return rc;

    const double z = std::sqrt(3.0) - 2.0;
    const long long BC = (long long)B * C;
    long long lines = BC;                                   // axis 0: lines (j, k), step B * C
    prefilter_outer_kernel<<<(unsigned)((lines + LINE_THREADS - 1) / LINE_THREADS), LINE_THREADS, 0, st>>>(
        c, lines, C, C, BC, A, z);
    R2X_CUDA_OK(cudaGetLastError());
    lines = (long long)A * C;                               // axis 1: lines (i, k), step C
    prefilter_outer_kernel<<<(unsigned)((lines + LINE_THREADS - 1) / LINE_THREADS), LINE_THREADS, 0, st>>>(
        c, lines, C, BC, C, B, z);
    R2X_CUDA_OK(cudaGetLastError());
    const long long rows = (long long)A * B;                // axis 2: contiguous rows
    const long long per_block = (long long)TILE * TILE_WARPS;
    prefilter_inner_kernel<<<(unsigned)((rows + per_block - 1) / per_block), TILE * TILE_WARPS, 0, st>>>(c, rows, C, z);
    R2X_CUDA_OK(cudaGetLastError());

    int sms = 0;
    R2X_CUDA_OK(sm_count(&sms));
    const long long orows = (long long)out0 * out1;
    const unsigned nblk = (unsigned)(orows < (long long)sms * ROW_BLOCKS_PER_SM ? orows : (long long)sms * ROW_BLOCKS_PER_SM);
    zoom_gather_kernel<<<nblk, ROW_THREADS, 0, st>>>(c, B, C, out0, out1, out2, coordinate_factor(p.m0, out0),
                                                     coordinate_factor(p.m1, out1), coordinate_factor(p.m2, out2), out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
