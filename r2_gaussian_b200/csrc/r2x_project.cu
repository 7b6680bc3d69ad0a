// r2x_project.cu -- ray-driven forward projection of a voxel volume (line integrals of its trilinear field).
//
// The reference makes its synthetic datasets with TIGRE's `Ax` (data_generator/synthetic_dataset/generate_data.py).
// This is the same operator, defined so that it agrees with render() by construction: the rays are the rasterizer's
// (scene.make_view geometry, ndc of the pixel centres), the field is the trilinear interpolation of the volume between
// voxel centres (0 at every lattice point outside the grid), and the integral is a Riemann sum at a fixed spacing
// whose sample positions are anchored at the ray's closest approach to the volume centre:
//
//   volume_project_kernel  one thread per detector pixel, a CTA is 32 detector rows (v) x 8 columns (u) of one view.
//                          On a circular scan v runs along world z, the volume's contiguous axis, so the 32 lanes of a
//                          warp read neighbouring z and most of each sample's 8 corner loads fall in one or two 128-byte
//                          lines.  Per-thread setup in float64 (rigid inverse of the viewmatrix, ray, closest approach
//                          t_c, index-space position g_c and step, k range from a slab test); samples
//                          g_k = fma(k, step, g_c) in float32, floor, 8 predicated __ldg loads, float32 sum in k order.
//                          The 32 x 8 tile is staged in shared memory so the [N,H,W] rows are stored in whole sectors.
//                          No atomics: the projections are bitwise reproducible.  A detector offset by (t_u, t_v)
//                          pixels (TIGRE's geo.offDetector) only moves the pixel's ndc in the float64 setup.  With a
//                          per-view geometry table the setup takes the view's tan_fov and shift from it.
//
// The float64 NumPy statement of the same definition is oracle/projector_oracle.py.
#include <cmath>
#include <cstdint>

#include "../../include/r2x.h"
#include "r2x_common.cuh"
#include "r2x_project.cuh"

namespace r2x {

constexpr int PRJ_BV = 32, PRJ_BU = 8;   // CTA: 32 detector rows (lanes) x 8 detector columns
constexpr int PRJ_MAX_VIEWS = 65535;     // views per launch (grid.z); more are launched in chunks

template <bool CONE, bool TABLE>
__global__ void __launch_bounds__(PRJ_BV * PRJ_BU) volume_project_kernel(
    const float* __restrict__ vol, int nx, int ny, int nz, float sx, float sy, float sz, float cx, float cy, float cz,
    int H, int W, const float* __restrict__ viewm, float tanx, float tany, float step, ProjShift shift,
    const double* __restrict__ vg, float* __restrict__ out) {
    __shared__ float tile[PRJ_BV][PRJ_BU + 1];
    const int v = blockIdx.y * PRJ_BV + threadIdx.x;   // detector row
    const int u = blockIdx.x * PRJ_BU + threadIdx.y;   // detector column
    const int view = blockIdx.z;
    float acc = 0.0f;
    if (v < H && u < W) {
        const ProjRay ray = project_ray_setup<CONE, TABLE>(viewm, view, u, v, H, W, nx, ny, nz, sx, sy, sz, cx, cy, cz, tanx,
                                                    tany, step, shift, vg);
        const long long sy_ = nz, sx_ = (long long)ny * nz;
        for (long long k = ray.k0; k <= ray.k1; ++k) {
            const float fk = (float)k;
            const float px = fmaf(fk, ray.sx, ray.gx), py = fmaf(fk, ray.sy, ray.gy), pz = fmaf(fk, ray.sz, ray.gz);
            const float fx0 = floorf(px), fy0 = floorf(py), fz0 = floorf(pz);
            const int ix = (int)fx0, iy = (int)fy0, iz = (int)fz0;
            const float fx = px - fx0, fy = py - fy0, fz = pz - fz0;
            const bool x0 = (unsigned)ix < (unsigned)nx, x1 = (unsigned)(ix + 1) < (unsigned)nx;
            const bool y0 = (unsigned)iy < (unsigned)ny, y1 = (unsigned)(iy + 1) < (unsigned)ny;
            const bool z0 = (unsigned)iz < (unsigned)nz, z1 = (unsigned)(iz + 1) < (unsigned)nz;
            const float* p = vol + (long long)ix * sx_ + (long long)iy * sy_ + iz;
            const float v000 = (x0 && y0 && z0) ? __ldg(p) : 0.0f;
            const float v001 = (x0 && y0 && z1) ? __ldg(p + 1) : 0.0f;
            const float v010 = (x0 && y1 && z0) ? __ldg(p + sy_) : 0.0f;
            const float v011 = (x0 && y1 && z1) ? __ldg(p + sy_ + 1) : 0.0f;
            const float v100 = (x1 && y0 && z0) ? __ldg(p + sx_) : 0.0f;
            const float v101 = (x1 && y0 && z1) ? __ldg(p + sx_ + 1) : 0.0f;
            const float v110 = (x1 && y1 && z0) ? __ldg(p + sx_ + sy_) : 0.0f;
            const float v111 = (x1 && y1 && z1) ? __ldg(p + sx_ + sy_ + 1) : 0.0f;
            const float c00 = fmaf(fz, v001 - v000, v000), c01 = fmaf(fz, v011 - v010, v010);
            const float c10 = fmaf(fz, v101 - v100, v100), c11 = fmaf(fz, v111 - v110, v110);
            const float c0 = fmaf(fy, c01 - c00, c00), c1 = fmaf(fy, c11 - c10, c10);
            acc += fmaf(fx, c1 - c0, c0);
        }
        acc *= step;
    }
    tile[threadIdx.x][threadIdx.y] = acc;
    __syncthreads();
    const int t = threadIdx.y * PRJ_BV + threadIdx.x;
    const int ro = blockIdx.y * PRJ_BV + t / PRJ_BU, co = blockIdx.x * PRJ_BU + t % PRJ_BU;
    if (ro < H && co < W) out[((size_t)view * H + ro) * W + co] = tile[t / PRJ_BU][t % PRJ_BU];
}

static int project_validate(int nx, int ny, int nz, const float* volume, float sx, float sy, float sz, float cx,
                            float cy, float cz, int N, int H, int W, const float* viewm, float tanx, float tany,
                            int mode, float step, const float* out) {
    if (nx < 1 || ny < 1 || nz < 1)
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad grid (each size must be >= 1)");
    if (N < 1 || H < 1 || W < 1) return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad N/H/W (each must be >= 1)");
    if ((H + PRJ_BV - 1) / PRJ_BV > 65535)
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad H (more than 2097120 detector rows)");
    if (mode != 0 && mode != 1) return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad mode (0 = parallel, 1 = cone)");
    if (!(sx > 0.0f && sy > 0.0f && sz > 0.0f && std::isfinite(sx) && std::isfinite(sy) && std::isfinite(sz)))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad sVoxel (must be finite and > 0)");
    if (!(std::isfinite(cx) && std::isfinite(cy) && std::isfinite(cz)))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad offOrigin (must be finite)");
    if (!(tanx > 0.0f && tany > 0.0f && std::isfinite(tanx) && std::isfinite(tany)))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad tan_fov (must be finite and > 0)");
    if (!(step > 0.0f && std::isfinite(step)))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad step (must be finite and > 0)");
    if (!volume || !viewm || !out) return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad pointer (NULL)");
    return 0;
}

static int project_launch(cudaStream_t st, int nx, int ny, int nz, const float* volume, float sx, float sy, float sz,
                          float cx, float cy, float cz, int n_views, int H, int W, const float* viewmatrices,
                          float tan_fovx, float tan_fovy, int mode, ProjShift shift, float step, const double* vg,
                          float* out_projs) {
    const dim3 block(PRJ_BV, PRJ_BU);
    for (int v0 = 0; v0 < n_views; v0 += PRJ_MAX_VIEWS) {
        const int nv = min(PRJ_MAX_VIEWS, n_views - v0);
        const dim3 grid((W + PRJ_BU - 1) / PRJ_BU, (H + PRJ_BV - 1) / PRJ_BV, nv);
        const float* vm = viewmatrices + (size_t)v0 * 16;
        const double* g = vg ? vg + (size_t)v0 * VG_COLS : nullptr;
        float* o = out_projs + (size_t)v0 * H * W;
        auto kernel = mode == 1 ? (g ? volume_project_kernel<true, true> : volume_project_kernel<true, false>)
                                : (g ? volume_project_kernel<false, true> : volume_project_kernel<false, false>);
        kernel<<<grid, block, 0, st>>>(volume, nx, ny, nz, sx, sy, sz, cx, cy, cz, H, W, vm, tan_fovx, tan_fovy, step,
                                       shift, g, o);
        R2X_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

}  // namespace r2x

extern "C" {

int r2x_volume_project(void* stream, int nx, int ny, int nz, const float* volume, float sx, float sy, float sz,
                       float cx, float cy, float cz, int n_views, int H, int W, const float* viewmatrices,
                       float tan_fovx, float tan_fovy, int mode, float shift_u, float shift_v, float step,
                       float* out_projs) {
    using namespace r2x;
    if (int rc = project_validate(nx, ny, nz, volume, sx, sy, sz, cx, cy, cz, n_views, H, W, viewmatrices, tan_fovx,
                                  tan_fovy, mode, step, out_projs))
        return rc;
    if (!(std::isfinite(shift_u) && std::isfinite(shift_v)))
        return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad shift (must be finite)");
    return project_launch((cudaStream_t)stream, nx, ny, nz, volume, sx, sy, sz, cx, cy, cz, n_views, H, W,
                          viewmatrices, tan_fovx, tan_fovy, mode, proj_shift(shift_u, shift_v, H, W), step, nullptr,
                          out_projs);
}

int r2x_volume_project_views(void* stream, int nx, int ny, int nz, const float* volume, float sx, float sy, float sz,
                             float cx, float cy, float cz, int n_views, int H, int W, const float* viewmatrices,
                             int mode, float step, const double* view_geometry, const double* view_geometry_host,
                             float* out_projs) {
    using namespace r2x;
    if (mode != 0 && mode != 1) return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad mode (0 = parallel, 1 = cone)");
    if (n_views < 1) return fail_msg(R2X_ERR_INVALID, "r2x_volume_project: bad N/H/W (each must be >= 1)");
    if (int rc = view_geometry_check("r2x_volume_project_views", n_views, mode, view_geometry, view_geometry_host,
                                     true))
        return rc;
    // the scalars stand in for the table in the shared checks; the kernels read every view's row
    const float tanx = (float)view_geometry_host[VG_TANX], tany = (float)view_geometry_host[VG_TANY];
    if (int rc = project_validate(nx, ny, nz, volume, sx, sy, sz, cx, cy, cz, n_views, H, W, viewmatrices, tanx, tany,
                                  mode, step, out_projs))
        return rc;
    return project_launch((cudaStream_t)stream, nx, ny, nz, volume, sx, sy, sz, cx, cy, cz, n_views, H, W,
                          viewmatrices, tanx, tany, mode, ProjShift{0.0, 0.0}, step, view_geometry, out_projs);
}

}  // extern "C"
