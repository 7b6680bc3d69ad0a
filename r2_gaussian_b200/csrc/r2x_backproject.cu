// r2x_backproject.cu -- the matched backprojector: the exact transpose of r2x_volume_project (r2x_project.cu).
//
// Iterative reconstructions (CGLS, SART / OS-SART, r2_gaussian_b200/recon.py) need A^T for the A that
// r2x_volume_project applies.  The FDK backprojector is not that operator (voxel-driven, bilinear on the detector,
// weighted by (DSO/z)^2), so this one is built from the projector's own samples:
//
//   backproject_rays_kernel    one thread per detector pixel of a chunk of views: the projector's per-ray setup
//                              (project_ray_setup, r2x_project.cuh, the same inlined code) written as two float4,
//                              (g_x, g_y, g_z, k0) and (s_x, s_y, s_z, k1), so the gather sees the projector's float32
//                              sample positions p_k = fma(k, s, g) and k range by construction, for a detector offset
//                              by (t_u, t_v) pixels as well; the gather below finds each voxel's footprint through the
//                              caller's offset projmatrices, so it stays the transpose of the offset projector.  With
//                              a per-view geometry table each view's rays take its row (project_ray_setup), and the
//                              caller's per-view projmatrices carry its FoV and offset.
//   volume_backproject_kernel  a thread owns one voxel x; a CTA is 32 voxels along z (the lanes) x 4 along y.  Per view
//                              (index order; projmatrix / viewmatrix rows staged in shared memory per chunk) the 8
//                              corners of x's open support box (x-1, x+1)^3 go through projmatrix and the rasterizer's
//                              ndc -> pixel mapping; the bounding rectangle widened by one pixel (the whole detector if a
//                              corner has z_view <= 0, cone beam) holds every ray that can sample the box.  For each of
//                              its pixels, row-major, the ray's [k0, k1] is cut to the samples inside the box
//                              (conservatively, in float32 with a rounding slack), each sample is evaluated exactly as
//                              the projector evaluates it and its trilinear weight h_x(p_k) summed in k order; the sum
//                              is multiplied by the pixel's value and added in registers.  Each voxel is stored once
//                              per chunk of views: no atomics, so both outputs are bitwise reproducible.
//
// The float64 NumPy statement of the same operator is tests/backproject_oracle.py (np.add.at over the rays and samples
// of oracle/projector_oracle.py).
#include <cmath>
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_common.cuh"
#include "r2x_project.cuh"

namespace r2x {

constexpr int BP_BZ = 32, BP_BY = 4;   // gather CTA: 32 voxels along z (lanes) x 4 along y
constexpr int BP_CHUNK = 32;           // views per ray table (scratch) and per shared-memory staging
constexpr int BP_RAYS_THREADS = 256;
constexpr double BP_KMAX = 16777216.0; // |k| < 2^24: (float)k is exact, and k0, k1 fit the table's int32

static size_t bp_al256(size_t x) { return (x + 255) & ~(size_t)255; }

size_t backproject_scratch_bytes(int N, int H, int W) {
    if (N < 1 || H < 1 || W < 1) return 256;
    return bp_al256((size_t)(N < BP_CHUNK ? N : BP_CHUNK) * H * W * 2 * sizeof(float4)) + 256;
}

template <bool CONE, bool TABLE>
__global__ void __launch_bounds__(BP_RAYS_THREADS) backproject_rays_kernel(
    int H, int W, const float* __restrict__ viewm, int nx, int ny, int nz, float sx, float sy, float sz, float cx,
    float cy, float cz, float tanx, float tany, float step, ProjShift shift, const double* __restrict__ vg,
    float4* __restrict__ rays) {
    const long long p = (long long)blockIdx.x * BP_RAYS_THREADS + threadIdx.x;
    const long long HW = (long long)H * W;
    if (p >= HW) return;
    const int view = blockIdx.y;
    const int v = (int)(p / W), u = (int)(p % W);
    const ProjRay r = project_ray_setup<CONE, TABLE>(viewm, view, u, v, H, W, nx, ny, nz, sx, sy, sz, cx, cy, cz, tanx, tany,
                                              step, shift, vg);
    long long k0 = r.k0, k1 = r.k1;
    if (k0 > k1) {
        k0 = 1; k1 = 0;                                                   // the ray misses the box
    } else {                                                              // no-ops: |k| < 2^24 inside the box
        k0 = max(k0, -(long long)BP_KMAX);
        k1 = min(k1, (long long)BP_KMAX);
    }
    float4* o = rays + 2 * ((size_t)view * HW + p);
    o[0] = make_float4(r.gx, r.gy, r.gz, __int_as_float((int)k0));
    o[1] = make_float4(r.sx, r.sy, r.sz, __int_as_float((int)k1));
}

// Cut [lo, hi] to the k whose sample fma(k, s, g) on this axis can lie in (c - 1, c + 1); false if none can.  The
// slack covers the float32 rounding of the cut and of the projector's fma (|p| <= |c| + 1 there), so no sample inside
// the open interval is dropped; samples it lets through outside get weight 0.
__device__ __forceinline__ bool bp_axis_cut(float g, float s, float c, float& lo, float& hi) {
    if (s != 0.0f) {
        const float r = __frcp_rn(s);
        const float t1 = (c - 1.0f - g) * r, t2 = (c + 1.0f - g) * r;
        const float slack = fmaf(1e-6f, fmaf(fabsf(c) + 2.0f, fabsf(r), fmaxf(fabsf(t1), fabsf(t2))), 1.0f);
        lo = fmaxf(lo, fminf(t1, t2) - slack);
        hi = fminf(hi, fmaxf(t1, t2) + slack);
        return true;
    }
    return g > c - 1.0f && g < c + 1.0f;
}

// The projector's trilinear weight of lattice point c at a sample p: 1 - f at floor(p), f at floor(p) + 1.
__device__ __forceinline__ float bp_hat(float p, float c) {
    const float p0 = floorf(p), f = p - p0;
    return p0 == c ? 1.0f - f : (p0 + 1.0f == c ? f : 0.0f);
}

template <bool CONE, bool WEIGHT>
__global__ void __launch_bounds__(BP_BZ * BP_BY) volume_backproject_kernel(
    int nv, int H, int W, const float4* __restrict__ rays, const float* __restrict__ projs,
    const float* __restrict__ viewm, const float* __restrict__ projm, int nx, int ny, int nz, float ox, float oy,
    float oz, float dx, float dy, float dz, int first, float scale, float* __restrict__ vol, float* __restrict__ wgt) {
    // per view: projmatrix rows 0, 1, 3 and viewmatrix row 2 as (m[r], m[4+r], m[8+r], m[12+r])
    __shared__ float4 mat[BP_CHUNK][4];
    const int z = blockIdx.x * BP_BZ + threadIdx.x;
    const int y = blockIdx.y * BP_BY + threadIdx.y;
    const int x = blockIdx.z;
    const int tid = threadIdx.y * BP_BZ + threadIdx.x;
    for (int e = tid; e < nv * 4; e += BP_BZ * BP_BY) {
        const int v = e >> 2, slot = e & 3;
        const float* m = (slot == 3 ? viewm : projm) + (size_t)v * 16;
        const int rr = slot == 3 ? 2 : (slot == 2 ? 3 : slot);
        mat[v][slot] = make_float4(m[rr], m[4 + rr], m[8 + rr], m[12 + rr]);
    }
    __syncthreads();
    if (!(y < ny && z < nz)) return;
    const size_t idx = ((size_t)x * ny + y) * nz + z;
    float acc = first ? 0.0f : vol[idx];
    float accw = 0.0f;
    if (WEIGHT && !first) accw = wgt[idx];
    const float xf = (float)x, yf = (float)y, zf = (float)z;
    const float X = fmaf(xf, dx, ox), Y = fmaf(yf, dy, oy), Z = fmaf(zf, dz, oz);
    const float half_w = 0.5f * (float)W, half_h = 0.5f * (float)H;
    const float cen_w = 0.5f * (float)(W - 1), cen_h = 0.5f * (float)(H - 1);
    const size_t HW = (size_t)H * W;
    for (int v = 0; v < nv; ++v) {
        const float4 P0 = mat[v][0], P1 = mat[v][1], P3 = mat[v][2], V2 = mat[v][3];
        // the support box's corners X +- dx, Y +- dy, Z +- dz in pixel space; the rectangle of pixel centres they span
        const float ax = fmaf(P0.z, Z, fmaf(P0.y, Y, fmaf(P0.x, X, P0.w)));
        const float ay = fmaf(P1.z, Z, fmaf(P1.y, Y, fmaf(P1.x, X, P1.w)));
        const float aw = fmaf(P3.z, Z, fmaf(P3.y, Y, fmaf(P3.x, X, P3.w)));
        const float az = CONE ? fmaf(V2.z, Z, fmaf(V2.y, Y, fmaf(V2.x, X, V2.w))) : 1.0f;
        float umin = 3.0e38f, umax = -3.0e38f, vmin = 3.0e38f, vmax = -3.0e38f;
        bool behind = false;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float ex = (c & 1) ? dx : -dx, ey = (c & 2) ? dy : -dy, ez = (c & 4) ? dz : -dz;
            const float qx = fmaf(P0.z, ez, fmaf(P0.y, ey, fmaf(P0.x, ex, ax)));
            const float qy = fmaf(P1.z, ez, fmaf(P1.y, ey, fmaf(P1.x, ex, ay)));
            const float qw = fmaf(P3.z, ez, fmaf(P3.y, ey, fmaf(P3.x, ex, aw)));
            if (CONE) behind |= !(fmaf(V2.z, ez, fmaf(V2.y, ey, fmaf(V2.x, ex, az))) > 0.0f) || !(qw > 0.0f);
            const float rw = __frcp_rn(qw);
            const float pu = fmaf(qx * rw, half_w, cen_w), pv = fmaf(qy * rw, half_h, cen_h);
            umin = fminf(umin, pu); umax = fmaxf(umax, pu);
            vmin = fminf(vmin, pv); vmax = fmaxf(vmax, pv);
        }
        int c0 = 0, c1 = W - 1, r0 = 0, r1 = H - 1;
        if (!behind) {
            // clamp in float before converting (a corner near the source's plane projects far off the detector)
            c0 = max(c0, (int)ceilf(fmaxf(umin, -2.0f)) - 1);
            c1 = min(c1, (int)floorf(fminf(umax, (float)W + 1.0f)) + 1);
            r0 = max(r0, (int)ceilf(fmaxf(vmin, -2.0f)) - 1);
            r1 = min(r1, (int)floorf(fminf(vmax, (float)H + 1.0f)) + 1);
        }
        const float4* rv = rays + 2 * (size_t)v * HW;
        const float* yv = projs + (size_t)v * HW;
        for (int i = r0; i <= r1; ++i) {
            for (int j = c0; j <= c1; ++j) {
                const size_t pix = (size_t)i * W + j;
                const float4 A = __ldg(rv + 2 * pix), B = __ldg(rv + 2 * pix + 1);
                float lo = (float)__float_as_int(A.w), hi = (float)__float_as_int(B.w);   // exact: |k| < 2^24
                if (!(lo <= hi)) continue;
                if (!bp_axis_cut(A.x, B.x, xf, lo, hi) || !bp_axis_cut(A.y, B.y, yf, lo, hi) ||
                    !bp_axis_cut(A.z, B.z, zf, lo, hi))
                    continue;
                const int ka = (int)ceilf(lo), kb = (int)floorf(hi);
                float s = 0.0f;
                for (int k = ka; k <= kb; ++k) {
                    const float fk = (float)k;
                    const float px = fmaf(fk, B.x, A.x), py = fmaf(fk, B.y, A.y), pz = fmaf(fk, B.z, A.z);
                    s = fmaf(bp_hat(px, xf) * bp_hat(py, yf), bp_hat(pz, zf), s);
                }
                if (s == 0.0f) continue;
                acc = fmaf(__ldg(yv + pix), s, acc);
                if (WEIGHT) accw += s;
            }
        }
    }
    vol[idx] = acc * scale;
    if (WEIGHT) wgt[idx] = accw * scale;
}

static int backproject_validate(int N, int H, int W, const float* projs, const float* viewm, const float* projm,
                                float tanx, float tany, int mode, int nx, int ny, int nz, float sx, float sy, float sz,
                                float cx, float cy, float cz, float step, const float* out, const void* scratch,
                                size_t scratch_bytes) {
    if (nx < 1 || ny < 1 || nz < 1)
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad grid (each size must be >= 1)");
    if (nx > 65535 || (ny + BP_BY - 1) / BP_BY > 65535)
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad grid (nx <= 65535, ny <= 262140)");
    if (N < 1 || H < 1 || W < 1)
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad N/H/W (each must be >= 1)");
    if (mode != 0 && mode != 1)
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad mode (0 = parallel, 1 = cone)");
    if (!(sx > 0.0f && sy > 0.0f && sz > 0.0f && std::isfinite(sx) && std::isfinite(sy) && std::isfinite(sz)))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad sVoxel (must be finite and > 0)");
    if (!(std::isfinite(cx) && std::isfinite(cy) && std::isfinite(cz)))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad offOrigin (must be finite)");
    if (!(tanx > 0.0f && tany > 0.0f && std::isfinite(tanx) && std::isfinite(tany)))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad tan_fov (must be finite and > 0)");
    if (!(step > 0.0f && std::isfinite(step)))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad step (must be finite and > 0)");
    // every sample inside the box has |k| step <= the box's half-diagonal
    const double hx = 0.5 * sx * (1.0 + 1.0 / nx), hy = 0.5 * sy * (1.0 + 1.0 / ny), hz = 0.5 * sz * (1.0 + 1.0 / nz);
    if (std::sqrt(hx * hx + hy * hy + hz * hz) / step + 2.0 >= BP_KMAX)
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad step (2^24 or more samples per half ray)");
    if (!projs || !viewm || !projm || !out || !scratch)
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad pointer (NULL)");
    if (scratch_bytes < backproject_scratch_bytes(N, H, W))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad scratch (too small)");
    return 0;
}

template <bool CONE>
static int backproject_launch(cudaStream_t st, int N, int H, int W, const float* projs, const float* viewm,
                              const float* projm, float tanx, float tany, int nx, int ny, int nz, float sx, float sy,
                              float sz, float cx, float cy, float cz, float step, ProjShift shift,
                              const double* vg, float* out, float* wgt, float4* rays) {
    const float dx = sx / nx, dy = sy / ny, dz = sz / nz;
    const float ox = cx - 0.5f * sx + 0.5f * dx, oy = cy - 0.5f * sy + 0.5f * dy, oz = cz - 0.5f * sz + 0.5f * dz;
    const long long HW = (long long)H * W;
    const dim3 gblock(BP_BZ, BP_BY), ggrid((nz + BP_BZ - 1) / BP_BZ, (ny + BP_BY - 1) / BP_BY, nx);
    for (int v0 = 0; v0 < N; v0 += BP_CHUNK) {
        const int nc = min(BP_CHUNK, N - v0);
        const float* vm = viewm + (size_t)v0 * 16;
        const double* g = vg ? vg + (size_t)v0 * VG_COLS : nullptr;
        const dim3 rgrid((unsigned)((HW + BP_RAYS_THREADS - 1) / BP_RAYS_THREADS), nc);
        (g ? backproject_rays_kernel<CONE, true> : backproject_rays_kernel<CONE, false>)<<<rgrid, BP_RAYS_THREADS, 0, st>>>(
            H, W, vm, nx, ny, nz, sx, sy, sz, cx, cy, cz, tanx, tany, step, shift, g, rays);
        R2X_CUDA_OK(cudaGetLastError());
        const int first = v0 == 0;
        const float scale = v0 + nc == N ? step : 1.0f;   // partial sums stay unscaled between chunks
        const float* pv = projs + (size_t)v0 * HW;
        const float* pm = projm + (size_t)v0 * 16;
        if (wgt)
            volume_backproject_kernel<CONE, true><<<ggrid, gblock, 0, st>>>(nc, H, W, rays, pv, vm, pm, nx, ny, nz, ox,
                                                                            oy, oz, dx, dy, dz, first, scale, out, wgt);
        else
            volume_backproject_kernel<CONE, false><<<ggrid, gblock, 0, st>>>(nc, H, W, rays, pv, vm, pm, nx, ny, nz, ox,
                                                                             oy, oz, dx, dy, dz, first, scale, out,
                                                                             nullptr);
        R2X_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

static int backproject_run(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
                           const float* projmatrices, float tan_fovx, float tan_fovy, int mode, ProjShift shift,
                           int nx, int ny, int nz, float sx, float sy, float sz, float cx, float cy, float cz,
                           float step, const double* vg, float* out_volume, float* out_weight, void* scratch) {
    const cudaStream_t st = (cudaStream_t)stream;
    float4* rays = (float4*)(((size_t)scratch + 255) & ~(size_t)255);
    if (mode == 1)
        return backproject_launch<true>(st, n_views, H, W, projs, viewmatrices, projmatrices, tan_fovx, tan_fovy, nx, ny,
                                        nz, sx, sy, sz, cx, cy, cz, step, shift, vg, out_volume, out_weight, rays);
    return backproject_launch<false>(st, n_views, H, W, projs, viewmatrices, projmatrices, tan_fovx, tan_fovy, nx, ny,
                                     nz, sx, sy, sz, cx, cy, cz, step, shift, vg, out_volume, out_weight, rays);
}

}  // namespace r2x

extern "C" {

size_t r2x_volume_backproject_scratch_bytes(int n_views, int H, int W) {
    return r2x::backproject_scratch_bytes(n_views, H, W);
}

int r2x_volume_backproject(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
                           const float* projmatrices, float tan_fovx, float tan_fovy, int mode, float shift_u,
                           float shift_v, int nx, int ny, int nz, float sx, float sy, float sz, float cx, float cy,
                           float cz, float step, float* out_volume, float* out_weight, void* scratch,
                           size_t scratch_bytes) {
    using namespace r2x;
    if (int rc = backproject_validate(n_views, H, W, projs, viewmatrices, projmatrices, tan_fovx, tan_fovy, mode, nx,
                                      ny, nz, sx, sy, sz, cx, cy, cz, step, out_volume, scratch, scratch_bytes))
        return rc;
    if (!(std::isfinite(shift_u) && std::isfinite(shift_v)))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad shift (must be finite)");
    return backproject_run(stream, n_views, H, W, projs, viewmatrices, projmatrices, tan_fovx, tan_fovy, mode,
                           proj_shift(shift_u, shift_v, H, W), nx, ny, nz, sx, sy, sz, cx, cy, cz, step, nullptr,
                           out_volume, out_weight, scratch);
}

int r2x_volume_backproject_views(void* stream, int n_views, int H, int W, const float* projs,
                                 const float* viewmatrices, const float* projmatrices, int mode, int nx, int ny,
                                 int nz, float sx, float sy, float sz, float cx, float cy, float cz, float step,
                                 const double* view_geometry, const double* view_geometry_host, float* out_volume,
                                 float* out_weight, void* scratch, size_t scratch_bytes) {
    using namespace r2x;
    if (mode != 0 && mode != 1)
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad mode (0 = parallel, 1 = cone)");
    if (n_views < 1) return fail_msg(R2X_ERR_INVALID, "r2x_volume_backproject: bad N/H/W (each must be >= 1)");
    if (int rc = view_geometry_check("r2x_volume_backproject_views", n_views, mode, view_geometry, view_geometry_host,
                                     true))
        return rc;
    // the scalars stand in for the table in the shared checks; the ray setup reads every view's row
    const float tanx = (float)view_geometry_host[VG_TANX], tany = (float)view_geometry_host[VG_TANY];
    if (int rc = backproject_validate(n_views, H, W, projs, viewmatrices, projmatrices, tanx, tany, mode, nx, ny, nz,
                                      sx, sy, sz, cx, cy, cz, step, out_volume, scratch, scratch_bytes))
        return rc;
    return backproject_run(stream, n_views, H, W, projs, viewmatrices, projmatrices, tanx, tany, mode,
                           ProjShift{0.0, 0.0}, nx, ny, nz, sx, sy, sz, cx, cy, cz, step, view_geometry, out_volume,
                           out_weight, scratch);
}

}  // extern "C"
