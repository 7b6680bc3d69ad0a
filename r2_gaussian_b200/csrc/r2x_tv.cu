// r2x_tv.cu -- isotropic total variation on a volume: the FGP proximal operator (r2x_tv_prox) and TV(x) as a
// float64 reduction (r2x_tv_value), include/r2x.h.  FISTA-TV (r2_gaussian_b200/recon.py) calls the prox once per
// outer iteration.
//
// Volumes are float32 [nx, ny, nz] (z fastest).  grad x = (dx, dy, dz), forward differences, 0 across the last index
// (Neumann); div p = sum_a (p_a[i] (i_a < n_a - 1) - p_a[i - e_a] (i_a > 0)), so <grad x, p> = -<x, div p>.  The prox
//   x = argmin_{x in C} 1/2 |x - v|^2 + w TV(x),   TV(x) = sum_i |grad x|_i,   C = {x >= 0} (nonneg) or everything,
// is Beck-Teboulle's fast gradient projection on the dual field p (|p_i| <= 1), from p_0 = 0, t_1 = 1:
//   r_1 = 0;  p_k = P_1(r_k - (1/(12 w)) grad P_C(v - w div r_k));  t_{k+1} = (1 + sqrt(1 + 4 t_k^2)) / 2;
//   r_{k+1} = p_k + ((t_k - 1) / t_{k+1}) (p_k - p_{k-1});  x = P_C(v - w div p_niter).
// One launch per inner iteration (tv_fgp_kernel): a CTA owns a 4 x 8 x 32 tile, forms r = p_{k-1} + beta (p_{k-1} -
// p_{k-2}) on the tile and its -1 / +1 halo in shared memory, the primal P_C(v - w div r) on the tile and its +1 halo,
// then grad, the dual step, the projection onto |p| <= 1, and writes p_k.  The momentum field r is never stored: the
// three dual fields p_k, p_{k-1}, p_{k-2} rotate through the caller's scratch (36 bytes per voxel).  Bytes per voxel
// and steady inner iteration: p_{k-1} and p_{k-2} read (24), v read (4), p_k written (12) = 40; halo re-reads come
// from L2.  A last launch (tv_primal_kernel) writes x from p_niter.  Weight 0 skips the dual entirely: x = P_C(v),
// bit for bit.  P_C(u) = (u < 0 ? 0 : u).  Everything is elementwise or a fixed stencil: no atomics, bitwise
// reproducible.
//
// r2x_tv_cp_step is the volume part of one Chambolle-Pock iteration of cp_tv (recon.py): from x, xbar, p and
// g = A^T q it writes p+ = P_{1/nu}(p + sigma nu grad xbar), x+ = P_C(x - tau g + tau nu div p+) and xbar+ = 2 x+ - x
// in one launch (tv_cp_kernel) on the same 4 x 8 x 32 tiles: xbar on the tile's [-1, T] box, p+ on its [-1, T - 1]
// box (the -1 layer is a neighbour's p+, recomputed here with the same instructions, so it is the value that neighbour
// writes), then div p+ and the primal on the tile.  Bytes per voxel: x, xbar, g read (12), p read (12), x+, xbar+
// written (8), p+ written (12) = 44; halo re-reads come from L2.
#include <cmath>
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_common.cuh"

namespace r2x {
namespace {

constexpr int TV_TX = 4, TV_TY = 8, TV_TZ = 32;                  // tile (x, y, z); z along the lanes
constexpr int TV_THREADS = 256;
constexpr int TV_RX = TV_TX + 2, TV_RY = TV_TY + 2, TV_RZ = TV_TZ + 2;   // r on the tile's [-1, T] box
constexpr int TV_XX = TV_TX + 1, TV_XY = TV_TY + 1, TV_XZ = TV_TZ + 1;   // the primal on the tile's [0, T] box
constexpr int TV_RBOX = TV_RX * TV_RY * TV_RZ, TV_XBOX = TV_XX * TV_XY * TV_XZ;

__device__ __forceinline__ float proj_c(float u, int nonneg) { return (nonneg && u < 0.0f) ? 0.0f : u; }

// p_k from r_k = 0 (mode 0), p_{k-1} (mode 1) or p_{k-1} + beta (p_{k-1} - p_{k-2}) (mode 2); dual fields are three
// planes of nvox floats (component a at a * nvox + voxel)
__global__ void __launch_bounds__(TV_THREADS) tv_fgp_kernel(int nx, int ny, int nz, const float* __restrict__ v,
                                                            float w, float step, float beta, int mode, int nonneg,
                                                            const float* __restrict__ pk1,
                                                            const float* __restrict__ pk2, float* __restrict__ out) {
    __shared__ float r[3][TV_RBOX];
    __shared__ float xs[TV_XBOX];
    const size_t nvox = (size_t)nx * ny * nz;
    const int X0 = blockIdx.z * TV_TX, Y0 = blockIdx.y * TV_TY, Z0 = blockIdx.x * TV_TZ;
    for (int e = threadIdx.x; e < TV_RBOX; e += TV_THREADS) {
        const int lz = e % TV_RZ, t = e / TV_RZ, ly = t % TV_RY, lx = t / TV_RY;
        const int X = X0 + lx - 1, Y = Y0 + ly - 1, Z = Z0 + lz - 1;
        float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
        if (mode != 0 && X >= 0 && X < nx && Y >= 0 && Y < ny && Z >= 0 && Z < nz) {
            const size_t i = ((size_t)X * ny + Y) * nz + Z;
            a0 = pk1[i];
            a1 = pk1[nvox + i];
            a2 = pk1[2 * nvox + i];
            if (mode == 2) {
                a0 = fmaf(beta, a0 - pk2[i], a0);
                a1 = fmaf(beta, a1 - pk2[nvox + i], a1);
                a2 = fmaf(beta, a2 - pk2[2 * nvox + i], a2);
            }
        }
        r[0][e] = a0;
        r[1][e] = a1;
        r[2][e] = a2;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < TV_XBOX; e += TV_THREADS) {
        const int lz = e % TV_XZ, t = e / TV_XZ, ly = t % TV_XY, lx = t / TV_XY;
        const int X = X0 + lx, Y = Y0 + ly, Z = Z0 + lz;
        float xv = 0.0f;
        if (X < nx && Y < ny && Z < nz) {
            const int c = ((lx + 1) * TV_RY + ly + 1) * TV_RZ + lz + 1;
            float d = (X < nx - 1 ? r[0][c] : 0.0f) - (X > 0 ? r[0][c - TV_RY * TV_RZ] : 0.0f);
            d += (Y < ny - 1 ? r[1][c] : 0.0f) - (Y > 0 ? r[1][c - TV_RZ] : 0.0f);
            d += (Z < nz - 1 ? r[2][c] : 0.0f) - (Z > 0 ? r[2][c - 1] : 0.0f);
            xv = proj_c(fmaf(-w, d, v[((size_t)X * ny + Y) * nz + Z]), nonneg);
        }
        xs[e] = xv;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < TV_TX * TV_TY * TV_TZ; e += TV_THREADS) {
        const int lz = e % TV_TZ, t = e / TV_TZ, ly = t % TV_TY, lx = t / TV_TY;
        const int X = X0 + lx, Y = Y0 + ly, Z = Z0 + lz;
        if (!(X < nx && Y < ny && Z < nz)) continue;
        const int cx = (lx * TV_XY + ly) * TV_XZ + lz;
        const float x0 = xs[cx];
        const float g0 = X < nx - 1 ? xs[cx + TV_XY * TV_XZ] - x0 : 0.0f;
        const float g1 = Y < ny - 1 ? xs[cx + TV_XZ] - x0 : 0.0f;
        const float g2 = Z < nz - 1 ? xs[cx + 1] - x0 : 0.0f;
        const int c = ((lx + 1) * TV_RY + ly + 1) * TV_RZ + lz + 1;
        float q0 = fmaf(-step, g0, r[0][c]), q1 = fmaf(-step, g1, r[1][c]), q2 = fmaf(-step, g2, r[2][c]);
        const float n2 = fmaf(q2, q2, fmaf(q1, q1, q0 * q0));
        if (n2 > 1.0f) {
            const float s = 1.0f / sqrtf(n2);
            q0 *= s;
            q1 *= s;
            q2 *= s;
        }
        const size_t i = ((size_t)X * ny + Y) * nz + Z;
        out[i] = q0;
        out[nvox + i] = q1;
        out[2 * nvox + i] = q2;
    }
}

// x = P_C(v - w div p); p == nullptr: x = P_C(v) (weight 0)
__global__ void __launch_bounds__(TV_THREADS) tv_primal_kernel(int nx, int ny, int nz, const float* __restrict__ v,
                                                               float w, int nonneg, const float* __restrict__ p,
                                                               float* __restrict__ out) {
    const size_t nvox = (size_t)nx * ny * nz;
    const size_t i = (size_t)blockIdx.x * TV_THREADS + threadIdx.x;
    if (i >= nvox) return;
    if (!p) {
        out[i] = proj_c(v[i], nonneg);
        return;
    }
    const int Z = (int)(i % nz), Y = (int)((i / nz) % ny), X = (int)(i / ((size_t)nz * ny));
    const size_t sx = (size_t)ny * nz, sy = nz;
    float d = (X < nx - 1 ? p[i] : 0.0f) - (X > 0 ? p[i - sx] : 0.0f);
    d += (Y < ny - 1 ? p[nvox + i] : 0.0f) - (Y > 0 ? p[nvox + i - sy] : 0.0f);
    d += (Z < nz - 1 ? p[2 * nvox + i] : 0.0f) - (Z > 0 ? p[2 * nvox + i - 1] : 0.0f);
    out[i] = proj_c(fmaf(-w, d, v[i]), nonneg);
}

constexpr int CP_PX = TV_TX + 1, CP_PY = TV_TY + 1, CP_PZ = TV_TZ + 1;   // p+ on the tile's [-1, T - 1] box
constexpr int CP_PBOX = CP_PX * CP_PY * CP_PZ;

// one Chambolle-Pock iteration after the data dual; xbar is staged on the [-1, T] box (the TV_R* box of tv_fgp_kernel)
__global__ void __launch_bounds__(TV_THREADS) tv_cp_kernel(int nx, int ny, int nz, const float* __restrict__ x,
                                                           const float* __restrict__ xbar, const float* __restrict__ p,
                                                           const float* __restrict__ g, float tau, float sn, float tn,
                                                           float pmax, float pmax2, int nonneg,
                                                           float* __restrict__ x_out, float* __restrict__ xbar_out,
                                                           float* __restrict__ p_out) {
    __shared__ float xb[TV_RBOX];
    __shared__ float pp[3][CP_PBOX];
    const size_t nvox = (size_t)nx * ny * nz;
    const int X0 = blockIdx.z * TV_TX, Y0 = blockIdx.y * TV_TY, Z0 = blockIdx.x * TV_TZ;
    for (int e = threadIdx.x; e < TV_RBOX; e += TV_THREADS) {
        const int lz = e % TV_RZ, t = e / TV_RZ, ly = t % TV_RY, lx = t / TV_RY;
        const int X = X0 + lx - 1, Y = Y0 + ly - 1, Z = Z0 + lz - 1;
        const bool in = X >= 0 && X < nx && Y >= 0 && Y < ny && Z >= 0 && Z < nz;
        xb[e] = in ? xbar[((size_t)X * ny + Y) * nz + Z] : 0.0f;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < CP_PBOX; e += TV_THREADS) {
        const int lz = e % CP_PZ, t = e / CP_PZ, ly = t % CP_PY, lx = t / CP_PY;
        const int X = X0 + lx - 1, Y = Y0 + ly - 1, Z = Z0 + lz - 1;
        float u0 = 0.0f, u1 = 0.0f, u2 = 0.0f;
        if (X >= 0 && X < nx && Y >= 0 && Y < ny && Z >= 0 && Z < nz) {
            const int c = (lx * TV_RY + ly) * TV_RZ + lz;                  // the same voxel in the xbar box
            const float x0 = xb[c];
            const float g0 = X < nx - 1 ? xb[c + TV_RY * TV_RZ] - x0 : 0.0f;
            const float g1 = Y < ny - 1 ? xb[c + TV_RZ] - x0 : 0.0f;
            const float g2 = Z < nz - 1 ? xb[c + 1] - x0 : 0.0f;
            const size_t i = ((size_t)X * ny + Y) * nz + Z;
            u0 = fmaf(sn, g0, p[i]);
            u1 = fmaf(sn, g1, p[nvox + i]);
            u2 = fmaf(sn, g2, p[2 * nvox + i]);
            const float n2 = fmaf(u2, u2, fmaf(u1, u1, u0 * u0));
            if (n2 > pmax2) {
                const float s = pmax / sqrtf(n2);
                u0 *= s;
                u1 *= s;
                u2 *= s;
            }
        }
        pp[0][e] = u0;
        pp[1][e] = u1;
        pp[2][e] = u2;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < TV_TX * TV_TY * TV_TZ; e += TV_THREADS) {
        const int lz = e % TV_TZ, t = e / TV_TZ, ly = t % TV_TY, lx = t / TV_TY;
        const int X = X0 + lx, Y = Y0 + ly, Z = Z0 + lz;
        if (!(X < nx && Y < ny && Z < nz)) continue;
        const int c = ((lx + 1) * CP_PY + ly + 1) * CP_PZ + lz + 1;
        float d = (X < nx - 1 ? pp[0][c] : 0.0f) - (X > 0 ? pp[0][c - CP_PY * CP_PZ] : 0.0f);
        d += (Y < ny - 1 ? pp[1][c] : 0.0f) - (Y > 0 ? pp[1][c - CP_PZ] : 0.0f);
        d += (Z < nz - 1 ? pp[2][c] : 0.0f) - (Z > 0 ? pp[2][c - 1] : 0.0f);
        const size_t i = ((size_t)X * ny + Y) * nz + Z;
        const float xv = x[i];
        const float xp = proj_c(fmaf(tn, d, fmaf(-tau, g[i], xv)), nonneg);
        x_out[i] = xp;
        xbar_out[i] = fmaf(2.0f, xp, -xv);
        p_out[i] = pp[0][c];
        p_out[nvox + i] = pp[1][c];
        p_out[2 * nvox + i] = pp[2][c];
    }
}

constexpr int TVV_THREADS = 256;
constexpr int TVV_MAX_BLOCKS = 1024;
constexpr long long TVV_PER_BLOCK = 8 * TVV_THREADS;

inline int value_blocks(long long n) {
    const long long b = (n + TVV_PER_BLOCK - 1) / TVV_PER_BLOCK;
    return (int)(b < 1 ? 1 : (b > TVV_MAX_BLOCKS ? TVV_MAX_BLOCKS : b));
}

// block b sums |grad x| (float64) over voxels [b chunk, (b + 1) chunk)
__global__ void __launch_bounds__(TVV_THREADS) tv_value_partial_kernel(int nx, int ny, int nz, long long chunk,
                                                                       const float* __restrict__ x,
                                                                       double* __restrict__ partial) {
    __shared__ double s[TVV_THREADS];
    const long long nvox = (long long)nx * ny * nz;
    const long long lo = (long long)blockIdx.x * chunk;
    const long long hi = lo + chunk < nvox ? lo + chunk : nvox;
    const long long sx = (long long)ny * nz;
    double acc = 0.0;
    for (long long i = lo + threadIdx.x; i < hi; i += TVV_THREADS) {
        const int Z = (int)(i % nz), Y = (int)((i / nz) % ny), X = (int)(i / sx);
        const double x0 = (double)x[i];
        const double d0 = X < nx - 1 ? (double)x[i + sx] - x0 : 0.0;
        const double d1 = Y < ny - 1 ? (double)x[i + nz] - x0 : 0.0;
        const double d2 = Z < nz - 1 ? (double)x[i + 1] - x0 : 0.0;
        acc += sqrt(d0 * d0 + d1 * d1 + d2 * d2);
    }
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int h = TVV_THREADS / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = s[0];
}

__global__ void __launch_bounds__(TVV_THREADS) tv_value_final_kernel(int nb, const double* __restrict__ partial,
                                                                     double* __restrict__ out) {
    __shared__ double s[TVV_THREADS];
    double acc = 0.0;
    for (int i = threadIdx.x; i < nb; i += TVV_THREADS) acc += partial[i];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int h = TVV_THREADS / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = s[0];
}

// tiles of t voxels along an axis of n voxels, in 64 bits: n + t - 1 is past INT_MAX for n within a tile of it
inline long long tiles(int n, int t) { return ((long long)n + t - 1) / t; }

bool bad_grid(int nx, int ny, int nz) {
    return nx < 1 || ny < 1 || nz < 1 || tiles(nx, TV_TX) > 65535 || tiles(ny, TV_TY) > 65535;
}

// the tv_fgp_kernel / tv_cp_kernel grid of a grid that passed bad_grid: z tiles on x (up to 2^26), y on y, x on z
dim3 tile_grid(int nx, int ny, int nz) {
    return dim3((unsigned)tiles(nz, TV_TZ), (unsigned)tiles(ny, TV_TY), (unsigned)tiles(nx, TV_TX));
}

bool finite_positive(double v) { return v > 0.0 && std::isfinite(v); }

// [a, a + na) and [b, b + nb) (in floats) share an address
bool overlap(const float* a, size_t na, const float* b, size_t nb) {
    const uintptr_t a0 = (uintptr_t)a, b0 = (uintptr_t)b;
    return a0 < b0 + nb * sizeof(float) && b0 < a0 + na * sizeof(float);
}

}  // namespace
}  // namespace r2x

extern "C" {

size_t r2x_tv_prox_scratch_bytes(int nx, int ny, int nz) {
    if (nx < 1 || ny < 1 || nz < 1) return 0;
    return (size_t)9 * nx * ny * nz * sizeof(float);
}

int r2x_tv_prox(void* stream, int nx, int ny, int nz, const float* v, float weight, int niter, int nonneg, float* out,
                void* scratch, size_t scratch_bytes) {
    using namespace r2x;
    if (bad_grid(nx, ny, nz))
        return fail_msg(R2X_ERR_INVALID, "r2x_tv_prox: bad grid (each size >= 1, nx <= 262140, ny <= 524280)");
    if (!v || !out || !scratch) return fail_msg(R2X_ERR_INVALID, "r2x_tv_prox: bad pointer (NULL)");
    if (!(weight >= 0.0f && std::isfinite(weight)))
        return fail_msg(R2X_ERR_INVALID, "r2x_tv_prox: bad weight (must be finite and >= 0)");
    if (niter < 1) return fail_msg(R2X_ERR_INVALID, "r2x_tv_prox: bad niter (must be >= 1)");
    if (nonneg != 0 && nonneg != 1) return fail_msg(R2X_ERR_INVALID, "r2x_tv_prox: bad nonneg (0 or 1)");
    if (scratch_bytes < r2x_tv_prox_scratch_bytes(nx, ny, nz))
        return fail_msg(R2X_ERR_INVALID, "r2x_tv_prox: bad scratch (smaller than r2x_tv_prox_scratch_bytes)");
    const cudaStream_t st = (cudaStream_t)stream;
    const size_t nvox = (size_t)nx * ny * nz;
    const unsigned nblk = (unsigned)((nvox + TV_THREADS - 1) / TV_THREADS);
    if (weight == 0.0f) {
        tv_primal_kernel<<<nblk, TV_THREADS, 0, st>>>(nx, ny, nz, v, 0.0f, nonneg, nullptr, out);
        R2X_CUDA_OK(cudaGetLastError());
        return 0;
    }
    float* buf[3] = {(float*)scratch, (float*)scratch + 3 * nvox, (float*)scratch + 6 * nvox};
    const float step = (float)(1.0 / (12.0 * (double)weight));
    const dim3 grid = tile_grid(nx, ny, nz);
    double t = 1.0, t_prev = 1.0;   // t_k and t_{k-1} of the launch computing p_k
    for (int k = 1; k <= niter; ++k) {
        const int mode = k == 1 ? 0 : (k == 2 ? 1 : 2);
        const float beta = (float)((t_prev - 1.0) / t);   // r_k = p_{k-1} + ((t_{k-1} - 1) / t_k) (p_{k-1} - p_{k-2})
        tv_fgp_kernel<<<grid, TV_THREADS, 0, st>>>(nx, ny, nz, v, weight, step, beta, mode, nonneg, buf[(k + 2) % 3],
                                                   buf[(k + 1) % 3], buf[k % 3]);
        R2X_CUDA_OK(cudaGetLastError());
        t_prev = t;
        t = 0.5 * (1.0 + std::sqrt(1.0 + 4.0 * t * t));
    }
    tv_primal_kernel<<<nblk, TV_THREADS, 0, st>>>(nx, ny, nz, v, weight, nonneg, buf[niter % 3], out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

size_t r2x_tv_value_scratch_bytes(int nx, int ny, int nz) {
    if (nx < 1 || ny < 1 || nz < 1) return 0;
    return (size_t)r2x::value_blocks((long long)nx * ny * nz) * sizeof(double);
}

int r2x_tv_value(void* stream, int nx, int ny, int nz, const float* x, double* out, void* scratch,
                 size_t scratch_bytes) {
    using namespace r2x;
    if (nx < 1 || ny < 1 || nz < 1) return fail_msg(R2X_ERR_INVALID, "r2x_tv_value: bad grid (each size >= 1)");
    if (!x || !out || !scratch) return fail_msg(R2X_ERR_INVALID, "r2x_tv_value: bad pointer (NULL)");
    if (scratch_bytes < r2x_tv_value_scratch_bytes(nx, ny, nz))
        return fail_msg(R2X_ERR_INVALID, "r2x_tv_value: bad scratch (smaller than r2x_tv_value_scratch_bytes)");
    const long long nvox = (long long)nx * ny * nz;
    const int nb = value_blocks(nvox);
    const long long chunk = (nvox + nb - 1) / nb;
    const cudaStream_t st = (cudaStream_t)stream;
    tv_value_partial_kernel<<<nb, TVV_THREADS, 0, st>>>(nx, ny, nz, chunk, x, (double*)scratch);
    R2X_CUDA_OK(cudaGetLastError());
    tv_value_final_kernel<<<1, TVV_THREADS, 0, st>>>(nb, (const double*)scratch, out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

int r2x_tv_cp_step(void* stream, int nx, int ny, int nz, const float* x, const float* xbar, const float* p,
                   const float* g, float tau, float sigma, float nu, int nonneg, float* x_out, float* xbar_out,
                   float* p_out) {
    using namespace r2x;
    if (bad_grid(nx, ny, nz))
        return fail_msg(R2X_ERR_INVALID, "r2x_tv_cp_step: bad grid (each size >= 1, nx <= 262140, ny <= 524280)");
    if (!x || !xbar || !p || !g || !x_out || !xbar_out || !p_out)
        return fail_msg(R2X_ERR_INVALID, "r2x_tv_cp_step: bad pointer (NULL)");
    const double sn = (double)sigma * nu, tn = (double)tau * nu, pmax = 1.0 / (double)nu;
    if (!finite_positive(tau) || !finite_positive(sigma) || !finite_positive(nu) || !finite_positive((float)sn) ||
        !finite_positive((float)tn) || !finite_positive((float)pmax))
        return fail_msg(R2X_ERR_INVALID,
                        "r2x_tv_cp_step: bad step (tau, sigma, nu, sigma nu, tau nu and 1 / nu finite and > 0)");
    if (nonneg != 0 && nonneg != 1) return fail_msg(R2X_ERR_INVALID, "r2x_tv_cp_step: bad nonneg (0 or 1)");
    const size_t nvox = (size_t)nx * ny * nz;
    const float* ins[4] = {x, xbar, g, p};
    const size_t in_n[4] = {nvox, nvox, nvox, 3 * nvox};
    float* outs[3] = {x_out, xbar_out, p_out};
    const size_t out_n[3] = {nvox, nvox, 3 * nvox};
    for (int o = 0; o < 3; ++o) {
        for (int k = 0; k < 4; ++k)
            if (overlap(outs[o], out_n[o], ins[k], in_n[k]))
                return fail_msg(R2X_ERR_INVALID, "r2x_tv_cp_step: bad alias (an output overlaps an input)");
        for (int k = o + 1; k < 3; ++k)
            if (overlap(outs[o], out_n[o], outs[k], out_n[k]))
                return fail_msg(R2X_ERR_INVALID, "r2x_tv_cp_step: bad alias (two outputs overlap)");
    }
    const dim3 grid = tile_grid(nx, ny, nz);
    tv_cp_kernel<<<grid, TV_THREADS, 0, (cudaStream_t)stream>>>(nx, ny, nz, x, xbar, p, g, tau, (float)sn, (float)tn,
                                                                (float)pmax, (float)(pmax * pmax), nonneg, x_out,
                                                                xbar_out, p_out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
