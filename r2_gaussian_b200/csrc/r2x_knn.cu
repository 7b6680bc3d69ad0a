// Exact 3-nearest-neighbour mean squared distance of a point cloud -- the quantity the reference obtains from
// `simple_knn._C.distCUDA2` to initialise the Gaussian scales (r2_gaussian/gaussian/gaussian_model.py:21,
// :144-150).  The upstream extension (gitlab.inria.fr/bkerbl/simple-knn, an un-vendored submodule of the
// reference) Morton-sorts the cloud and prunes 1024-point boxes; its *result* is the exact mean of the three
// smallest squared distances to other points, which is what this file computes, with a uniform hash grid:
//
//   bbox (1 kernel) -> cell histogram -> exclusive scan (single-pass look-back, r2x_binning) -> scatter into
//   cell order -> per point: search the 3x3x3 cells around it, then grow the searched cube shell by shell
//   until the third-best distance is provably final.
//
// The three smallest distances are a property of the input, not of the traversal order, so the output is
// bitwise reproducible and equal to the brute-force oracle (oracle/r2_oracle.c: orc_knn3_mean_dist2), which
// uses the same float expression fma(dz,dz, fma(dy,dy, dx*dx)).
#include <cfloat>
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_binning.cuh"
#include "r2x_common.cuh"

namespace r2x {

constexpr int KNN_MAX_G = 128;   // cells per axis at most

struct KnnScratch {
    uint32_t* bbox;        // [8]   ordered-uint encoded (min xyz, max xyz)
    uint32_t* total;       // [1]
    uint32_t* count;       // [C]   points per cell (consumed by the scatter)
    uint32_t* incl;        // [C]   inclusive scan of count
    void* scan_state;
    float4* sorted;        // [P]   (x, y, z, original index bits), cell-major
    int G;
};

static int knn_grid(int P) {
    int g = 1;
    while ((long long)g * g * g * 2 < (long long)P && g < KNN_MAX_G) ++g;
    return g;
}
static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

size_t knn_scratch_bytes(int P) {
    if (P < 1) P = 1;
    const size_t G = (size_t)knn_grid(P), C = G * G * G;
    return 256 + al256(64) + 2 * al256(C * sizeof(uint32_t)) + al256(scan_state_bytes((int)C)) +
           al256((size_t)P * sizeof(float4));
}

static KnnScratch knn_view(void* buf, int P) {
    KnnScratch s;
    s.G = knn_grid(P);
    const size_t C = (size_t)s.G * s.G * s.G;
    char* p = (char*)al256((size_t)buf);
    s.bbox = (uint32_t*)p; s.total = s.bbox + 8; p += al256(64);
    s.count = (uint32_t*)p; p += al256(C * sizeof(uint32_t));
    s.incl = (uint32_t*)p; p += al256(C * sizeof(uint32_t));
    s.scan_state = p; p += al256(scan_state_bytes((int)C));
    s.sorted = (float4*)p;
    return s;
}

__device__ __forceinline__ uint32_t f2ord(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(uint32_t o) {
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

__global__ void knn_init_kernel(uint32_t* bbox) {
    if (threadIdx.x < 3) bbox[threadIdx.x] = 0xffffffffu;       // min = +max
    else if (threadIdx.x < 6) bbox[threadIdx.x] = 0u;           // max = -max
}

__global__ void __launch_bounds__(256) knn_bbox_kernel(int P, const float* __restrict__ pts, uint32_t* bbox) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = pts[3 * (size_t)i + a];
            lo[a] = fminf(lo[a], v);
            hi[a] = fmaxf(hi[a], v);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMin(&bbox[a], f2ord(lo[a]));
            atomicMax(&bbox[3 + a], f2ord(hi[a]));
        }
    }
}

// Grid derived from the bounding box: cubic cells of edge h = longest extent / G, dims[a] = cells needed along a.
struct KnnGrid {
    float ox, oy, oz, inv_h, h;
    int nx, ny, nz;
};
__device__ __forceinline__ KnnGrid knn_make_grid(const uint32_t* __restrict__ bbox, int G) {
    KnnGrid g;
    g.ox = ord2f(bbox[0]); g.oy = ord2f(bbox[1]); g.oz = ord2f(bbox[2]);
    const float ex = ord2f(bbox[3]) - g.ox, ey = ord2f(bbox[4]) - g.oy, ez = ord2f(bbox[5]) - g.oz;
    float e = fmaxf(ex, fmaxf(ey, ez));
    if (!(e > 0.f)) e = 1.f;
    g.h = e / (float)G;
    g.inv_h = (float)G / e;
    g.nx = min(G, (int)(ex * g.inv_h) + 1);
    g.ny = min(G, (int)(ey * g.inv_h) + 1);
    g.nz = min(G, (int)(ez * g.inv_h) + 1);
    return g;
}
__device__ __forceinline__ int knn_axis_cell(float v, float o, float inv_h, int n) {
    const int c = (int)((v - o) * inv_h);
    return c < 0 ? 0 : (c >= n ? n - 1 : c);
}

__global__ void __launch_bounds__(256) knn_count_kernel(int P, const float* __restrict__ pts,
                                                        const uint32_t* __restrict__ bbox, int G,
                                                        uint32_t* __restrict__ count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const KnnGrid g = knn_make_grid(bbox, G);
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    const int cx = knn_axis_cell(x, g.ox, g.inv_h, g.nx), cy = knn_axis_cell(y, g.oy, g.inv_h, g.ny),
              cz = knn_axis_cell(z, g.oz, g.inv_h, g.nz);
    atomicAdd(&count[((size_t)cz * g.ny + cy) * g.nx + cx], 1u);
}

__global__ void __launch_bounds__(256) knn_scatter_kernel(int P, const float* __restrict__ pts,
                                                          const uint32_t* __restrict__ bbox, int G,
                                                          uint32_t* __restrict__ count,
                                                          const uint32_t* __restrict__ incl,
                                                          float4* __restrict__ sorted) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const KnnGrid g = knn_make_grid(bbox, G);
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    const int cx = knn_axis_cell(x, g.ox, g.inv_h, g.nx), cy = knn_axis_cell(y, g.oy, g.inv_h, g.ny),
              cz = knn_axis_cell(z, g.oz, g.inv_h, g.nz);
    const size_t c = ((size_t)cz * g.ny + cy) * g.nx + cx;
    const uint32_t k = atomicSub(&count[c], 1u);    // k .. 1
    sorted[incl[c] - k] = make_float4(x, y, z, __uint_as_float((uint32_t)i));
}

__device__ __forceinline__ void knn_insert(float (&best)[3], float d) {
    // ascending insertion, the update rule of simple-knn's updateKBest<3>
    if (d < best[2]) {
        if (d < best[1]) {
            best[2] = best[1];
            if (d < best[0]) { best[1] = best[0]; best[0] = d; }
            else best[1] = d;
        } else best[2] = d;
    }
}

__global__ void __launch_bounds__(128) knn_query_kernel(int P, const uint32_t* __restrict__ bbox, int G,
                                                        const uint32_t* __restrict__ incl,
                                                        const float4* __restrict__ sorted,
                                                        float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const KnnGrid g = knn_make_grid(bbox, G);
    const float4 p = sorted[i];
    const int cx = knn_axis_cell(p.x, g.ox, g.inv_h, g.nx), cy = knn_axis_cell(p.y, g.oy, g.inv_h, g.ny),
              cz = knn_axis_cell(p.z, g.oz, g.inv_h, g.nz);
    float best[3] = {FLT_MAX, FLT_MAX, FLT_MAX};
    const int rmax = max(g.nx, max(g.ny, g.nz));
    for (int r = 0; r <= rmax; ++r) {
        // cells at Chebyshev distance exactly r from (cx,cy,cz)
        const int z0 = max(cz - r, 0), z1 = min(cz + r, g.nz - 1);
        const int y0 = max(cy - r, 0), y1 = min(cy + r, g.ny - 1);
        const int x0 = max(cx - r, 0), x1 = min(cx + r, g.nx - 1);
        for (int z = z0; z <= z1; ++z)
            for (int y = y0; y <= y1; ++y) {
                const bool face = (z == cz - r) || (z == cz + r) || (y == cy - r) || (y == cy + r);
                const size_t rowc = ((size_t)z * g.ny + y) * g.nx;
                if (face) {
                    // the whole x-run of this row belongs to the shell: its cells are contiguous in memory
                    const uint32_t b = (rowc + x0) ? incl[rowc + x0 - 1] : 0u, e = incl[rowc + x1];
                    for (uint32_t j = b; j < e; ++j) {
                        if ((int)j == i) continue;
                        const float4 q = sorted[j];
                        const float dx = p.x - q.x, dy = p.y - q.y, dz = p.z - q.z;
                        knn_insert(best, fmaf(dz, dz, fmaf(dy, dy, dx * dx)));
                    }
                } else {
                    for (int s = 0; s < 2; ++s) {
                        const int x = s ? cx + r : cx - r;
                        if (x < 0 || x >= g.nx || (s && r == 0)) continue;
                        const uint32_t b = (rowc + x) ? incl[rowc + x - 1] : 0u, e = incl[rowc + x];
                        for (uint32_t j = b; j < e; ++j) {
                            if ((int)j == i) continue;
                            const float4 q = sorted[j];
                            const float dx = p.x - q.x, dy = p.y - q.y, dz = p.z - q.z;
                            knn_insert(best, fmaf(dz, dz, fmaf(dy, dy, dx * dx)));
                        }
                    }
                }
            }
        // every unvisited point lies outside the cube of cells [c-r, c+r]^3: its distance is at least the
        // distance from p to the nearest face of that cube which is not a face of the grid
        float bound = FLT_MAX;
        if (cx - r > 0) bound = fminf(bound, p.x - (g.ox + (float)(cx - r) * g.h));
        if (cx + r < g.nx - 1) bound = fminf(bound, (g.ox + (float)(cx + r + 1) * g.h) - p.x);
        if (cy - r > 0) bound = fminf(bound, p.y - (g.oy + (float)(cy - r) * g.h));
        if (cy + r < g.ny - 1) bound = fminf(bound, (g.oy + (float)(cy + r + 1) * g.h) - p.y);
        if (cz - r > 0) bound = fminf(bound, p.z - (g.oz + (float)(cz - r) * g.h));
        if (cz + r < g.nz - 1) bound = fminf(bound, (g.oz + (float)(cz + r + 1) * g.h) - p.z);
        if (bound == FLT_MAX) break;                  // the cube covers the whole grid
        // cell assignment rounds (v - o) * inv_h, so a point may sit up to a few ulps outside its cell's
        // nominal slab: shave the bound accordingly before trusting it
        const float tol = 2e-5f * g.h + 1e-6f * (fabsf(g.ox) + fabsf(g.oy) + fabsf(g.oz) + 3.f * (float)G * g.h);
        bound = fmaxf(bound - tol, 0.f);
        if (best[2] <= bound * bound) break;
    }
    out[__float_as_uint(p.w)] = (best[0] + best[1] + best[2]) / 3.0f;
}

int launch_knn3(cudaStream_t st, int P, const float* points, float* out, void* scratch, size_t scratch_bytes) {
    if (P <= 0) return 0;
    if (!points || !out || !scratch) return fail_msg(R2X_ERR_INVALID, "r2x_knn3_mean_dist2: null pointer");
    if (scratch_bytes < knn_scratch_bytes(P)) return fail_msg(R2X_ERR_INVALID, "r2x_knn3_mean_dist2: scratch too small");
    const KnnScratch s = knn_view(scratch, P);
    const size_t C = (size_t)s.G * s.G * s.G;
    knn_init_kernel<<<1, 32, 0, st>>>(s.bbox);
    int sms;
    R2X_CUDA_OK(sm_count(&sms));
    knn_bbox_kernel<<<sms * 4, 256, 0, st>>>(P, points, s.bbox);
    R2X_CUDA_OK(cudaMemsetAsync(s.count, 0, C * sizeof(uint32_t), st));
    const int nb = (P + 255) / 256;
    knn_count_kernel<<<nb, 256, 0, st>>>(P, points, s.bbox, s.G, s.count);
    if (launch_scan(st, (int)C, s.count, s.incl, s.scan_state, s.total)) return R2X_ERR_CUDA;
    knn_scatter_kernel<<<nb, 256, 0, st>>>(P, points, s.bbox, s.G, s.count, s.incl, s.sorted);
    knn_query_kernel<<<(P + 127) / 128, 128, 0, st>>>(P, s.bbox, s.G, s.incl, s.sorted, out);
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace r2x
