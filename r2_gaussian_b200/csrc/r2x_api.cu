// r2x_api.cu -- the C ABI declared in include/r2x.h: buffer carving, stage orchestration, error
// reporting.  Stage order (both pipelines): preprocess -> scan(tiles_touched) -> [sync variant: read R,
// obtain the binning buffer] -> emit instances -> stable tile-id sort + ranges -> render.
#include <atomic>
#include <cstdio>
#include <cstring>
#include <string>
#include "../../include/r2x.h"
#include "r2x_binning.cuh"
#include "r2x_raster.cuh"
#include "r2x_voxel.cuh"

namespace r2x {
int launch_adam(cudaStream_t st, int ngroups, const r2x_adam_group* groups, double beta1, double beta2, double eps,
                long long step, const float* const* grads2, const uint32_t* guard0, const uint32_t* guard1);
int launch_densify_stats(cudaStream_t st, int P, const int* radii, const float* grad2d, float* max_radii, float* accum,
                         float* denom, const uint32_t* guard0, const uint32_t* guard1);

static thread_local std::string g_err;
static thread_local Activation g_act = {0, 0, 0.f, 0.f};
Activation current_activation() { return g_act; }
void set_activation(const Activation* a) { g_act = a ? *a : Activation{0, 0, 0.f, 0.f}; }

int fail(cudaError_t e, const char* what, const char* file, int line) {
    char buf[512];
    snprintf(buf, sizeof(buf), "CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
    g_err = buf;
    return R2X_ERR_CUDA;
}
int fail_msg(int code, const char* msg) {
    g_err = msg;
    return code;
}
cudaError_t sm_count(int* n) {
    // Per-device cache; concurrent first calls store the same value, so relaxed atomics suffice.
    static std::atomic<int> cache[64];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    int v = (dev >= 0 && dev < 64) ? cache[dev].load(std::memory_order_relaxed) : 0;
    if (v <= 0) {
        e = cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        if (e != cudaSuccess) return e;
        if (v <= 0) return cudaErrorInvalidDevice;
        if (dev >= 0 && dev < 64) cache[dev].store(v, std::memory_order_relaxed);
    }
    *n = v;
    return cudaSuccess;
}

namespace {

inline size_t al(size_t v) { return (v + 255) / 256 * 256; }

struct Carver {
    char* p;
    explicit Carver(const void* base) : p((char*)al((size_t)base)) {}
    template <typename T>
    T* take(size_t count) {
        T* r = (T*)p;
        p += al(count * sizeof(T));
        return r;
    }
};

struct RasterState {
    RasterGeom geom;
    void* scan_state;
    uint32_t* status;  // [0] = R, [1] = overflow flag
};

size_t raster_geom_bytes(int P) {
    size_t p = (size_t)(P > 0 ? P : 1);
    return al(p * 32) + al(p * 16) + al(p * 12) + 4 * al(p * 4) + al(scan_state_bytes((int)p)) + al(16) + 512;
}
RasterState carve_raster(const void* buf, int P, int W, int H) {
    size_t p = (size_t)(P > 0 ? P : 1);
    Carver c(buf);
    RasterState s;
    s.geom.rec = c.take<float4>(2 * p);
    s.geom.aux = c.take<float4>(p);
    s.geom.depth = c.take<float>(p);
    s.geom.mu = c.take<float>(p);
    s.geom.cube = c.take<uint16_t>(6 * p);
    s.geom.tiles_touched = c.take<uint32_t>(p);
    s.geom.offsets = c.take<uint32_t>(p);
    s.scan_state = c.take<char>(scan_state_bytes((int)p));
    s.status = c.take<uint32_t>(4);
    s.geom.gx = (W + R2X_TILE - 1) / R2X_TILE;
    s.geom.gy = (H + R2X_TILE - 1) / R2X_TILE;
    return s;
}

struct VoxelState {
    VoxelGeom geom;
    void* scan_state;
    uint32_t* status;
};
size_t voxel_geom_bytes(int P) {
    size_t p = (size_t)(P > 0 ? P : 1);
    return al(p * 64) + al(p * 12) + 2 * al(p * 4) + al(scan_state_bytes((int)p)) + al(16) + 512;
}
VoxelState carve_voxel(const void* buf, int P) {
    size_t p = (size_t)(P > 0 ? P : 1);
    Carver c(buf);
    VoxelState s;
    s.geom.rec = c.take<float4>(4 * p);
    s.geom.cube = c.take<uint16_t>(6 * p);
    s.geom.tiles_touched = c.take<uint32_t>(p);
    s.geom.offsets = c.take<uint32_t>(p);
    s.scan_state = c.take<char>(scan_state_bytes((int)p));
    s.status = c.take<uint32_t>(4);
    return s;
}

// image buffer = ranges[T] | work plan | direct-binning table (when T <= DIRECT_MAX_TILES)
TilePlan carve_plan(const void* image_buf, int tiles, const BinningView& bv) {
    char* p = (char*)al((size_t)image_buf) + al((size_t)tiles * sizeof(uint2));
    return plan_view(p, tiles, bv);
}
// voxelizer: work items may hold up to VOX_CHUNK_CAP instances (walked in segments), see plan_chunk_for
TilePlan carve_voxel_plan(const void* image_buf, int tiles, const BinningView& bv) {
    TilePlan pl = carve_plan(image_buf, tiles, bv);
    pl.chunk_cap = VOX_CHUNK_CAP;
    return pl;
}
DirectBin carve_directbin(const void* image_buf, int P, int tiles) {
    char* p = (char*)al((size_t)image_buf) + al((size_t)tiles * sizeof(uint2)) + plan_bytes(tiles);
    return directbin_view(p, P, tiles);
}

TwoLevel carve_two_level(const void* image_buf, int P, int gx, int gy, int gz, const BinningView& bv) {
    const int tiles = gx * gy * gz;
    char* p = (char*)al((size_t)image_buf) + al((size_t)tiles * sizeof(uint2)) + plan_bytes(tiles);
    return two_level_view(p, P, gx, gy, gz, bv);
}

// sorted position -> tile id through the ranges (direct binning keeps no per-instance tile array)
__global__ void export_keys_ranges_kernel(long long R, const uint32_t* d_total, const uint2* ranges, int T,
                                          const uint32_t* point_list, const float* depth, int depth_stride,
                                          uint64_t* keys, uint32_t* point_list_out) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= R || s >= (long long)*d_total) return;
    const uint32_t g = point_list[s];
    if (keys) {
        int lo = 0, hi = T;   // largest tile with ranges[tile].x <= s among non-empty ones
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if ((long long)ranges[mid].x <= s) lo = mid; else hi = mid;
        }
        while (lo > 0 && ranges[lo].x == ranges[lo].y) --lo;   // skip empty tiles sharing the same start
        const float d = depth[(size_t)depth_stride * g];
        keys[s] = ((uint64_t)(uint32_t)lo << 32) | (uint64_t)__float_as_uint(d);
    }
    if (point_list_out) point_list_out[s] = g;
}

int sort_passes(int num_tiles) {
    int bits = 1;
    while ((1ll << bits) < (long long)num_tiles) ++bits;
    return (bits + 7) / 8;
}

__global__ void status_kernel(uint32_t* status, long long capacity, uint32_t* status_out) {
    const uint32_t R = status[0];
    const uint32_t ov = ((long long)R > capacity) ? 1u : 0u;
    status[1] = ov;
    if (status_out) { status_out[0] = R; status_out[1] = ov; }
}

int debug_sync(cudaStream_t st, int debug, const char* stage) {
    if (!debug) return 0;
    cudaError_t e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(e, stage, __FILE__, __LINE__);
    return 0;
}
#define R2X_TRY(expr)            \
    do {                         \
        int _rc = (expr);        \
        if (_rc != 0) return _rc; \
    } while (0)

// ---- export kernels ---------------------------------------------------------------------------
// tile ranges in the reference's convention: an empty tile reads (0, 0) (the reference zero-fills `ranges` and only
// writes the non-empty ones, RAS/rasterizer_impl.cu:308-321); direct binning keeps (start, start) internally
__global__ void export_ranges_kernel(int T, const uint2* __restrict__ ranges, uint32_t* __restrict__ out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const uint2 r = ranges[t];
    const bool empty = (r.x == r.y);
    out[2 * (size_t)t] = empty ? 0u : r.x;
    out[2 * (size_t)t + 1] = empty ? 0u : r.y;
}

__global__ void raster_export_geom_kernel(int P, RasterGeom geom, float* means2D, float* depths, float* conic_opacity,
                                          float* mus, uint32_t* tiles_touched, uint32_t* point_offsets) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= P) return;
    const float4 r0 = geom.rec[2 * (size_t)g], r1 = geom.rec[2 * (size_t)g + 1], a = geom.aux[g];
    if (means2D) { means2D[2 * (size_t)g] = r0.x; means2D[2 * (size_t)g + 1] = r0.y; }
    if (depths) depths[g] = geom.depth[g];
    if (conic_opacity) {
        conic_opacity[4 * (size_t)g] = a.x; conic_opacity[4 * (size_t)g + 1] = a.y;
        conic_opacity[4 * (size_t)g + 2] = a.z; conic_opacity[4 * (size_t)g + 3] = a.w;
    }
    if (mus) mus[g] = geom.mu[g];
    if (tiles_touched) tiles_touched[g] = geom.tiles_touched[g];
    if (point_offsets) point_offsets[g] = geom.offsets[g];
}
__global__ void voxel_export_geom_kernel(int P, VoxelGeom geom, float* means3D_norm, float* depths,
                                         float* conic_opacity, uint32_t* tiles_touched, uint32_t* point_offsets) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= P) return;
    const float4 r0 = geom.rec[4 * (size_t)g], r1 = geom.rec[4 * (size_t)g + 1], r2 = geom.rec[4 * (size_t)g + 2];
    if (means3D_norm) {
        means3D_norm[3 * (size_t)g] = r0.x; means3D_norm[3 * (size_t)g + 1] = r0.y; means3D_norm[3 * (size_t)g + 2] = r0.z;
    }
    if (depths) depths[g] = geom.rec[4 * (size_t)g + 3].y;
    if (conic_opacity) {
        const float L = 1.4426950408889634f;
        float* co = conic_opacity + 7 * (size_t)g;
        co[0] = r1.x / (0.5f * L); co[1] = r1.y / L; co[2] = r1.z / L; co[3] = r1.w / (0.5f * L);
        co[4] = r2.x / L; co[5] = r2.y / (0.5f * L); co[6] = geom.rec[4 * (size_t)g + 3].x;
    }
    if (tiles_touched) tiles_touched[g] = geom.tiles_touched[g];
    if (point_offsets) point_offsets[g] = geom.offsets[g];
}
// keys[s] = (tile << 32) | float_bits(depth of point_list[s]); depth lives at float index depth_idx of
// the Gaussian's record (record stride rec_stride float4).
__global__ void export_keys_kernel(long long R, const uint32_t* d_total, const uint32_t* sorted_tiles,
                                   const uint32_t* point_list, const float* depth, int depth_stride,
                                   uint64_t* keys, uint32_t* point_list_out) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= R || s >= (long long)*d_total) return;   // R = carve capacity, *d_total = live instances
    const uint32_t g = point_list[s];
    if (keys) {
        const float d = depth[(size_t)depth_stride * g];
        keys[s] = ((uint64_t)sorted_tiles[s] << 32) | (uint64_t)__float_as_uint(d);
    }
    if (point_list_out) point_list_out[s] = g;
}

// ---- shared forward tail: emit -> sort -> ranges ---------------------------------------------
int bin_instances(cudaStream_t st, int P, const uint16_t* cube, const uint32_t* tiles_touched,
                  const uint32_t* offsets, int gx, int gy, int num_tiles, const uint32_t* d_total,
                  const BinningView& bv, long long R_launch, uint2* ranges) {
    if (R_launch > 0) R2X_TRY(launch_emit(st, P, cube, tiles_touched, offsets, gx, gy, d_total, bv));
    R2X_TRY(launch_sort_and_ranges(st, R_launch, num_tiles, d_total, bv, ranges, nullptr));
    return 0;
}

int raster_forward_impl(cudaStream_t st, int P, int W, int H, const float* means3D, const float* opacities,
                        const float* scales, float scale_modifier, const float* rotations,
                        const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                        float tan_fovx, float tan_fovy, int prefiltered, int mode, float* out_color, int* radii,
                        void* geom_buf, void* image_buf, r2x_alloc_fn binning_alloc, void* alloc_user,
                        void* binning_buf, long long capacity, uint32_t* status_dev, int debug, int* num_rendered) {
    if (W <= 0 || H <= 0 || P < 0) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: bad P/W/H");
    if (!out_color || !geom_buf || !image_buf) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: null output/state buffer");
    if (mode != 0 && mode != 1) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: mode must be 0 (parallel) or 1 (cone)");
    if (num_rendered) *num_rendered = 0;
    RasterState s = carve_raster(geom_buf, P, W, H);
    const int tiles = s.geom.gx * s.geom.gy;
    if (s.geom.gx > 65535 || s.geom.gy > 65535) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: detector too large");
    uint2* ranges = (uint2*)al((size_t)image_buf);
    if (P == 0) {
        R2X_CUDA_OK(cudaMemsetAsync(out_color, 0, sizeof(float) * (size_t)W * H, st));
        R2X_CUDA_OK(cudaMemsetAsync(ranges, 0, sizeof(uint2) * tiles, st));
        R2X_CUDA_OK(cudaMemsetAsync(s.status, 0, 16, st));
        if (status_dev) R2X_CUDA_OK(cudaMemsetAsync(status_dev, 0, 8, st));
        return 0;
    }
    if (!means3D || !opacities || !radii || !viewmatrix || !projmatrix)
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: null input");
    if (!cov3D_precomp && (!scales || !rotations))
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: need scales+rotations or cov3D_precomp");
    const bool direct = direct_ok(tiles);
    DirectBin db{};
    if (direct) {
        db = carve_directbin(image_buf, P, tiles);
    }
    R2X_TRY(launch_raster_preprocess(st, P, means3D, scales, scale_modifier, rotations, opacities, cov3D_precomp,
                                     viewmatrix, projmatrix, W, H, tan_fovx, tan_fovy, mode, prefiltered, radii,
                                     s.geom, direct ? &db : nullptr));
    R2X_TRY(debug_sync(st, debug, "raster preprocess"));
    if (direct) {
        // tile ranges, work plan and R come straight from the per-CTA tile histograms
        const long long cap0 = binning_alloc ? (1ll << 62) : capacity;
        R2X_TRY(launch_direct_scan(st, db, s.status, cap0, binning_alloc ? nullptr : status_dev));
    } else {
        R2X_TRY(launch_scan(st, P, s.geom.tiles_touched, s.geom.offsets, s.scan_state, s.status));
    }
    R2X_TRY(debug_sync(st, debug, "raster scan"));
    long long R_launch;
    if (binning_alloc) {  // synchronous variant: learn R, size the binning buffer exactly
        uint32_t R = 0;
        R2X_CUDA_OK(cudaMemcpyAsync(&R, s.status, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        R2X_CUDA_OK(cudaStreamSynchronize(st));
        if (num_rendered) *num_rendered = (int)R;
        binning_buf = binning_alloc(binning_bytes((long long)R), alloc_user);
        if (!binning_buf) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: binning allocator returned NULL");
        capacity = R;
        R_launch = R;
    } else {
        if (!binning_buf || capacity < 0) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward_async: no binning buffer");
        R_launch = capacity;
    }
    BinningView bv = binning_view(binning_buf, capacity);
    const TilePlan plan = carve_plan(image_buf, tiles, bv);
    if (direct) {
        R2X_TRY(launch_direct_fill(st, P, s.geom.cube, s.geom.tiles_touched, s.geom.offsets, db, ranges, plan, bv,
                                   s.geom.gx, s.geom.gy, s.status));
    } else {
        status_kernel<<<1, 1, 0, st>>>(s.status, capacity, status_dev);
        R2X_TRY(bin_instances(st, P, s.geom.cube, s.geom.tiles_touched, s.geom.offsets, s.geom.gx, s.geom.gy, tiles,
                              s.status, bv, R_launch, ranges));
        R2X_TRY(launch_plan(st, ranges, plan));
    }
    R2X_TRY(debug_sync(st, debug, "raster binning"));
    R2X_TRY(launch_raster_render(st, W, H, s.geom, ranges, bv.point_list, plan, R_launch, out_color));
    R2X_TRY(debug_sync(st, debug, "raster render"));
    return 0;
}

int voxel_forward_impl(cudaStream_t st, int P, int nx, int ny, int nz, float sx, float sy, float sz, float cx,
                       float cy, float cz, const float* means3D, const float* opacities, const float* scales,
                       float scale_modifier, const float* rotations, const float* cov3D_precomp, int prefiltered,
                       float* out_volume, int* radii_x, int* radii_y, int* radii_z, void* geom_buf, void* image_buf,
                       r2x_alloc_fn binning_alloc, void* alloc_user, void* binning_buf, long long capacity,
                       uint32_t* status_dev, int debug, int* num_rendered) {
    (void)prefiltered;
    if (nx <= 0 || ny <= 0 || nz <= 0 || P < 0) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward: bad P/grid");
    if (!out_volume || !geom_buf || !image_buf) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward: null output/state buffer");
    if (num_rendered) *num_rendered = 0;
    const VoxelGrid vg = make_voxel_grid(nx, ny, nz, sx, sy, sz, cx, cy, cz);
    if (vg.gx > 65535 || vg.gy > 65535 || vg.gz > 65535) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward: grid too large");
    const long long tiles_ll = (long long)vg.gx * vg.gy * vg.gz;
    if (tiles_ll > (1ll << 30)) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward: too many tiles");
    const int tiles = (int)tiles_ll;
    VoxelState s = carve_voxel(geom_buf, P);
    uint2* ranges = (uint2*)al((size_t)image_buf);
    if (P == 0) {
        R2X_CUDA_OK(cudaMemsetAsync(out_volume, 0, sizeof(float) * (size_t)nx * ny * nz, st));
        R2X_CUDA_OK(cudaMemsetAsync(ranges, 0, sizeof(uint2) * (size_t)tiles, st));
        R2X_CUDA_OK(cudaMemsetAsync(s.status, 0, 16, st));
        if (status_dev) R2X_CUDA_OK(cudaMemsetAsync(status_dev, 0, 8, st));
        return 0;
    }
    if (!means3D || !opacities || !radii_x || !radii_y || !radii_z)
        return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward: null input");
    if (!scales)
        return fail_msg(R2X_ERR_INVALID,
                        "r2x_voxel_forward: scales are required (the bounding radius is 3*max(scale)/dVoxel even "
                        "with cov3D_precomp; the reference dereferences scales unconditionally, VOX/forward.cu:137)");
    if (!cov3D_precomp && !rotations) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward: need rotations or cov3D_precomp");
    const bool direct = direct_ok(tiles);
    const bool two_level = two_level_ok(vg.gx, vg.gy, vg.gz);   // more tiles than the direct table holds
    DirectBin db{};
    if (direct) {
        db = carve_directbin(image_buf, P, tiles);
    }
    R2X_TRY(launch_voxel_preprocess(st, P, means3D, scales, scale_modifier, rotations, opacities, cov3D_precomp, vg,
                                    radii_x, radii_y, radii_z, s.geom, direct ? &db : nullptr));
    R2X_TRY(debug_sync(st, debug, "voxel preprocess"));
    if (direct) {
        const long long cap0 = binning_alloc ? (1ll << 62) : capacity;
        R2X_TRY(launch_direct_scan(st, db, s.status, cap0, binning_alloc ? nullptr : status_dev));
    } else {
        R2X_TRY(launch_scan(st, P, s.geom.tiles_touched, s.geom.offsets, s.scan_state, s.status));
    }
    long long R_launch;
    if (binning_alloc) {
        uint32_t R = 0;
        R2X_CUDA_OK(cudaMemcpyAsync(&R, s.status, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        R2X_CUDA_OK(cudaStreamSynchronize(st));
        if (num_rendered) *num_rendered = (int)R;
        binning_buf = binning_alloc(binning_bytes((long long)R), alloc_user);
        if (!binning_buf) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward: binning allocator returned NULL");
        capacity = R;
        R_launch = R;
    } else {
        if (!binning_buf || capacity < 0) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward_async: no binning buffer");
        R_launch = capacity;
    }
    BinningView bv = binning_view(binning_buf, capacity);
    const TilePlan plan = carve_voxel_plan(image_buf, tiles, bv);
    if (direct) {
        R2X_TRY(launch_direct_fill(st, P, s.geom.cube, s.geom.tiles_touched, s.geom.offsets, db, ranges, plan, bv, vg.gx,
                                   vg.gy, s.status));
    } else if (two_level) {
        status_kernel<<<1, 1, 0, st>>>(s.status, capacity, status_dev);
        const TwoLevel tl = carve_two_level(image_buf, P, vg.gx, vg.gy, vg.gz, bv);
        R2X_TRY(launch_two_level(st, P, s.geom.cube, s.geom.tiles_touched, vg.gx, vg.gy, vg.gz, s.status, tl, bv, ranges,
                                 plan));
    } else {
        status_kernel<<<1, 1, 0, st>>>(s.status, capacity, status_dev);
        R2X_TRY(bin_instances(st, P, s.geom.cube, s.geom.tiles_touched, s.geom.offsets, vg.gx, vg.gy, tiles, s.status,
                              bv, R_launch, ranges));
        R2X_TRY(launch_plan(st, ranges, plan));
    }
    R2X_TRY(debug_sync(st, debug, "voxel binning"));
    R2X_TRY(launch_voxel_render(st, vg, s.geom, ranges, bv.point_list, plan, R_launch, out_volume));
    R2X_TRY(debug_sync(st, debug, "voxel render"));
    return 0;
}

}  // namespace
}  // namespace r2x

using namespace r2x;

extern "C" {

const char* r2x_last_error(void) { return g_err.c_str(); }
int r2x_version(void) { return 100; }

size_t r2x_raster_geom_bytes(int P) { return raster_geom_bytes(P); }
size_t r2x_raster_image_bytes(int P, int W, int H) {
    size_t t = (size_t)((W + R2X_TILE - 1) / R2X_TILE) * ((H + R2X_TILE - 1) / R2X_TILE);
    return al(t * sizeof(uint2)) + plan_bytes((int)t) + (direct_ok((int)t) ? directbin_bytes(P, (int)t) : 0) + 1024;
}
size_t r2x_voxel_geom_bytes(int P) { return voxel_geom_bytes(P); }
size_t r2x_voxel_image_bytes(int P, int nx, int ny, int nz) {
    size_t t = (size_t)((nx + 7) / 8) * ((ny + 7) / 8) * ((nz + 7) / 8);
    return al(t * sizeof(uint2)) + plan_bytes((int)t) + (direct_ok((int)t) ? directbin_bytes(P, (int)t) : 0) +
           two_level_bytes(P, (nx + 7) / 8, (ny + 7) / 8, (nz + 7) / 8) + 1024;
}
size_t r2x_binning_bytes(long long R) { return binning_bytes(R); }
size_t r2x_raster_bwd_scratch_bytes(long long R) { return al((size_t)(R > 0 ? R : 1) * 32) + 256; }
size_t r2x_voxel_bwd_scratch_bytes(long long R) { return al((size_t)(R > 0 ? R : 1) * 48) + 256; }

int r2x_raster_forward(void* stream, int P, int W, int H, const float* means3D, const float* opacities,
                       const float* scales, float scale_modifier, const float* rotations,
                       const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                       const float* campos, float tan_fovx, float tan_fovy, int prefiltered, int mode,
                       float* out_color, int* radii, void* geom_buf, void* image_buf, r2x_alloc_fn binning_alloc,
                       void* alloc_user, int debug, int* num_rendered) {
    (void)campos;
    if (!binning_alloc) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: binning_alloc is NULL");
    return raster_forward_impl((cudaStream_t)stream, P, W, H, means3D, opacities, scales, scale_modifier, rotations,
                               cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, prefiltered, mode,
                               out_color, radii, geom_buf, image_buf, binning_alloc, alloc_user, nullptr, 0, nullptr,
                               debug, num_rendered);
}

int r2x_raster_forward_async(void* stream, int P, int W, int H, const float* means3D, const float* opacities,
                             const float* scales, float scale_modifier, const float* rotations,
                             const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                             const float* campos, float tan_fovx, float tan_fovy, int prefiltered, int mode,
                             float* out_color, int* radii, void* geom_buf, void* image_buf, void* binning_buf,
                             long long capacity, uint32_t* status_dev) {
    (void)campos;
    return raster_forward_impl((cudaStream_t)stream, P, W, H, means3D, opacities, scales, scale_modifier, rotations,
                               cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, prefiltered, mode,
                               out_color, radii, geom_buf, image_buf, nullptr, nullptr, binning_buf, capacity,
                               status_dev, 0, nullptr);
}

int r2x_raster_render_only(void* stream, int P, int W, int H, long long R, const void* geom_buf,
                           const void* binning_buf, const void* image_buf, float* out_color) {
    if (P <= 0 || R < 0 || !geom_buf || !image_buf || !out_color || (R > 0 && !binning_buf))
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_render_only: bad args");
    RasterState s = carve_raster(geom_buf, P, W, H);
    BinningView bv = binning_view((void*)binning_buf, R);
    const uint2* ranges = (const uint2*)al((size_t)image_buf);
    const TilePlan plan = carve_plan(image_buf, s.geom.gx * s.geom.gy, bv);
    // the work plan of the forward is still valid: only the queue head and the arrival counters are rewound
    R2X_CUDA_OK(cudaMemsetAsync(plan.counter, 0, sizeof(uint32_t), (cudaStream_t)stream));
    R2X_CUDA_OK(cudaMemsetAsync(plan.tile_done, 0, sizeof(uint32_t) * PLAN_DONE_SLOTS * (size_t)plan.num_tiles, (cudaStream_t)stream));
    return launch_raster_render((cudaStream_t)stream, W, H, s.geom, ranges, bv.point_list, plan, R, out_color);
}

int r2x_voxel_render_only(void* stream, int P, int nx, int ny, int nz, long long R, const void* geom_buf,
                          const void* binning_buf, const void* image_buf, float* out_volume) {
    if (P <= 0 || R < 0 || !geom_buf || !image_buf || !out_volume || (R > 0 && !binning_buf))
        return fail_msg(R2X_ERR_INVALID, "r2x_voxel_render_only: bad args");
    const VoxelGrid vg = make_voxel_grid(nx, ny, nz, 1.f, 1.f, 1.f, 0.f, 0.f, 0.f);  // render needs the tile grid only
    VoxelState s = carve_voxel(geom_buf, P);
    BinningView bv = binning_view((void*)binning_buf, R);
    const uint2* ranges = (const uint2*)al((size_t)image_buf);
    const TilePlan plan = carve_voxel_plan(image_buf, vg.gx * vg.gy * vg.gz, bv);
    R2X_CUDA_OK(cudaMemsetAsync(plan.counter, 0, sizeof(uint32_t), (cudaStream_t)stream));
    R2X_CUDA_OK(cudaMemsetAsync(plan.tile_done, 0, sizeof(uint32_t) * PLAN_DONE_SLOTS * (size_t)plan.num_tiles, (cudaStream_t)stream));
    return launch_voxel_render((cudaStream_t)stream, vg, s.geom, ranges, bv.point_list, plan, R, out_volume);
}

int r2x_raster_backward(void* stream, int P, long long R, int W, int H, const float* means3D, const float* scales,
                        float scale_modifier, const float* rotations, const float* cov3D_precomp,
                        const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                        float tan_fovy, const int* radii, const void* geom_buf, const void* binning_buf,
                        const void* image_buf, void* scratch, const float* dL_dpix, float* dL_dmean2D,
                        float* dL_dopacity, float* dL_dmu, float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale,
                        float* dL_drot, int mode, int debug) {
    (void)campos;
    cudaStream_t st = (cudaStream_t)stream;
    if (P == 0) return 0;
    if (P < 0 || W <= 0 || H <= 0 || R < 0) return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward: bad sizes");
    if (!geom_buf || !image_buf || !dL_dpix || !dL_dmean2D || !dL_dopacity || !dL_dmean3D || !dL_dcov3D ||
        !dL_dscale || !dL_drot || !radii || !means3D)
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward: null pointer");
    if (R > 0 && (!binning_buf || !scratch)) return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward: null binning/scratch");
    RasterState s = carve_raster(geom_buf, P, W, H);
    const uint2* ranges = (const uint2*)al((size_t)image_buf);
    BinningView bv = binning_view((void*)binning_buf, R);
    float4* inst_grad = (float4*)al((size_t)scratch);
    const TilePlan plan = carve_plan(image_buf, s.geom.gx * s.geom.gy, bv);
    const uint32_t* inst_pos = direct_ok(s.geom.gx * s.geom.gy) ? nullptr : bv.inst_pos;   // direct binning: slots are derived
    if (R > 0) R2X_TRY(launch_raster_render_bwd(st, W, H, s.geom, ranges, bv.point_list, inst_pos, plan, R, dL_dpix, inst_grad));
    R2X_TRY(debug_sync(st, debug, "raster render backward"));
    R2X_TRY(launch_raster_gauss_bwd(st, P, means3D, radii, scales, scale_modifier, rotations, cov3D_precomp, viewmatrix,
                                    projmatrix, W, H, tan_fovx, tan_fovy, mode, s.geom, R, bv.inst_pos, inst_grad,
                                    dL_dmean2D, dL_dopacity, dL_dmu, dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot));
    R2X_TRY(debug_sync(st, debug, "raster per-Gaussian backward"));
    return 0;
}

int r2x_mark_visible(void* stream, int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     unsigned char* present) {
    (void)projmatrix;
    if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !present))) return fail_msg(R2X_ERR_INVALID, "r2x_mark_visible: bad args");
    return launch_mark_visible((cudaStream_t)stream, P, means3D, viewmatrix, present);
}

int r2x_raster_export(void* stream, int P, int W, int H, long long R, const void* geom_buf,
                      const void* binning_buf, const void* image_buf, float* means2D, float* depths,
                      float* conic_opacity, float* mus, uint32_t* tiles_touched, uint32_t* point_offsets,
                      uint64_t* keys, uint32_t* point_list, uint32_t* ranges) {
    cudaStream_t st = (cudaStream_t)stream;
    if (P <= 0) return 0;
    RasterState s = carve_raster(geom_buf, P, W, H);
    raster_export_geom_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, s.geom, means2D, depths, conic_opacity, mus,
                                                                tiles_touched, point_offsets);
    const int tiles = s.geom.gx * s.geom.gy;
    if (ranges) export_ranges_kernel<<<(tiles + 255) / 256, 256, 0, st>>>(tiles, (const uint2*)al((size_t)image_buf), ranges);
    if (R > 0 && (keys || point_list)) {
        BinningView bv = binning_view((void*)binning_buf, R);
        if (direct_ok(tiles)) {
            export_keys_ranges_kernel<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(
                R, s.status, (const uint2*)al((size_t)image_buf), tiles, bv.point_list, s.geom.depth, 1, keys, point_list);
        } else {
            const uint32_t* sorted = bv.keys[sort_passes(tiles) & 1];
            export_keys_kernel<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(R, s.status, sorted, bv.point_list, s.geom.depth, 1, keys, point_list);
        }
    }
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

int r2x_voxel_forward(void* stream, int P, int nx, int ny, int nz, float sx, float sy, float sz, float cx, float cy,
                      float cz, const float* means3D, const float* opacities, const float* scales,
                      float scale_modifier, const float* rotations, const float* cov3D_precomp, int prefiltered,
                      float* out_volume, int* radii_x, int* radii_y, int* radii_z, void* geom_buf, void* image_buf,
                      r2x_alloc_fn binning_alloc, void* alloc_user, int debug, int* num_rendered) {
    if (!binning_alloc) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward: binning_alloc is NULL");
    return voxel_forward_impl((cudaStream_t)stream, P, nx, ny, nz, sx, sy, sz, cx, cy, cz, means3D, opacities, scales,
                              scale_modifier, rotations, cov3D_precomp, prefiltered, out_volume, radii_x, radii_y,
                              radii_z, geom_buf, image_buf, binning_alloc, alloc_user, nullptr, 0, nullptr, debug,
                              num_rendered);
}

int r2x_voxel_forward_async(void* stream, int P, int nx, int ny, int nz, float sx, float sy, float sz, float cx,
                            float cy, float cz, const float* means3D, const float* opacities, const float* scales,
                            float scale_modifier, const float* rotations, const float* cov3D_precomp,
                            int prefiltered, float* out_volume, int* radii_x, int* radii_y, int* radii_z,
                            void* geom_buf, void* image_buf, void* binning_buf, long long capacity,
                            uint32_t* status_dev) {
    return voxel_forward_impl((cudaStream_t)stream, P, nx, ny, nz, sx, sy, sz, cx, cy, cz, means3D, opacities, scales,
                              scale_modifier, rotations, cov3D_precomp, prefiltered, out_volume, radii_x, radii_y,
                              radii_z, geom_buf, image_buf, nullptr, nullptr, binning_buf, capacity, status_dev, 0,
                              nullptr);
}

int r2x_voxel_backward(void* stream, int P, long long R, int nx, int ny, int nz, float sx, float sy, float sz,
                       float cx, float cy, float cz, const float* means3D, const float* scales, float scale_modifier,
                       const float* rotations, const float* cov3D_precomp, const int* radii_x, const int* radii_y,
                       const int* radii_z, const void* geom_buf, const void* binning_buf, const void* image_buf,
                       void* scratch, const float* dL_dvol, float* dL_dopacity, float* dL_dmean3D, float* dL_dcov3D,
                       float* dL_dscale, float* dL_drot, int debug) {
    (void)means3D;
    cudaStream_t st = (cudaStream_t)stream;
    if (P == 0) return 0;
    if (P < 0 || nx <= 0 || ny <= 0 || nz <= 0 || R < 0) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_backward: bad sizes");
    if (!geom_buf || !image_buf || !dL_dvol || !dL_dopacity || !dL_dmean3D || !dL_dcov3D || !dL_dscale || !dL_drot ||
        !radii_x || !radii_y || !radii_z)
        return fail_msg(R2X_ERR_INVALID, "r2x_voxel_backward: null pointer");
    if (R > 0 && (!binning_buf || !scratch)) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_backward: null binning/scratch");
    const VoxelGrid vg = make_voxel_grid(nx, ny, nz, sx, sy, sz, cx, cy, cz);
    VoxelState s = carve_voxel(geom_buf, P);
    const uint2* ranges = (const uint2*)al((size_t)image_buf);
    BinningView bv = binning_view((void*)binning_buf, R);
    float4* inst_grad = (float4*)al((size_t)scratch);
    const TilePlan plan = carve_voxel_plan(image_buf, vg.gx * vg.gy * vg.gz, bv);
    // direct and two-level binning keep no per-instance slot array: the slots are derived (emission_slot())
    const uint32_t* inst_pos = (direct_ok(vg.gx * vg.gy * vg.gz) || two_level_ok(vg.gx, vg.gy, vg.gz)) ? nullptr : bv.inst_pos;
    if (R > 0) R2X_TRY(launch_voxel_render_bwd(st, vg, s.geom, ranges, bv.point_list, inst_pos, plan, R, dL_dvol, inst_grad));
    R2X_TRY(debug_sync(st, debug, "voxel render backward"));
    R2X_TRY(launch_voxel_gauss_bwd(st, P, radii_x, radii_y, radii_z, scales, scale_modifier, rotations, cov3D_precomp, vg,
                                   s.geom, R, bv.inst_pos, inst_grad, dL_dopacity, dL_dmean3D, dL_dcov3D, dL_dscale,
                                   dL_drot));
    R2X_TRY(debug_sync(st, debug, "voxel per-Gaussian backward"));
    return 0;
}

int r2x_voxel_export(void* stream, int P, int nx, int ny, int nz, long long R, const void* geom_buf,
                     const void* binning_buf, const void* image_buf, float* means3D_norm, float* depths,
                     float* conic_opacity, uint32_t* tiles_touched, uint32_t* point_offsets, uint64_t* keys,
                     uint32_t* point_list, uint32_t* ranges) {
    cudaStream_t st = (cudaStream_t)stream;
    if (P <= 0) return 0;
    VoxelState s = carve_voxel(geom_buf, P);
    voxel_export_geom_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, s.geom, means3D_norm, depths, conic_opacity,
                                                               tiles_touched, point_offsets);
    const size_t tiles = (size_t)((nx + 7) / 8) * ((ny + 7) / 8) * ((nz + 7) / 8);
    if (ranges) export_ranges_kernel<<<(unsigned)((tiles + 255) / 256), 256, 0, st>>>((int)tiles, (const uint2*)al((size_t)image_buf), ranges);
    if (R > 0 && (keys || point_list)) {
        BinningView bv = binning_view((void*)binning_buf, R);
        if (direct_ok((int)tiles) || two_level_ok((nx + 7) / 8, (ny + 7) / 8, (nz + 7) / 8)) {
            export_keys_ranges_kernel<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(
                R, s.status, (const uint2*)al((size_t)image_buf), (int)tiles, bv.point_list, reinterpret_cast<const float*>(s.geom.rec) + 13, 16, keys, point_list);
        } else {
            const uint32_t* sorted = bv.keys[sort_passes((int)tiles) & 1];
            export_keys_kernel<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(R, s.status, sorted, bv.point_list, reinterpret_cast<const float*>(s.geom.rec) + 13, 16, keys, point_list);
        }
    }
    R2X_CUDA_OK(cudaGetLastError());
    return 0;
}

// ---- folded activations: the same four calls on RAW density / scale / rotation parameters -----------------------
namespace {
struct ActScope {
    explicit ActScope(const r2x_activation* a) {
        Activation v = {1, a ? a->scale_mode : 0, a ? a->scale_lo : 0.f, a ? a->scale_hi : 0.f};
        set_activation(&v);
    }
    ~ActScope() { set_activation(nullptr); }
};
}  // namespace

int r2x_raster_forward_async_raw(void* stream, int P, int W, int H, const float* means3D, const float* raw_density,
                                 const float* raw_scales, float scale_modifier, const float* raw_rotations,
                                 const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                                 float tan_fovy, int mode, float* out_color, int* radii, void* geom_buf, void* image_buf,
                                 void* binning_buf, long long capacity, uint32_t* status_dev, const r2x_activation* act) {
    if (!act || !raw_scales || !raw_rotations) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward_async_raw: null argument");
    ActScope scope(act);
    return r2x_raster_forward_async(stream, P, W, H, means3D, raw_density, raw_scales, scale_modifier, raw_rotations, nullptr,
                                    viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, 0, mode, out_color, radii, geom_buf,
                                    image_buf, binning_buf, capacity, status_dev);
}

int r2x_raster_backward_raw(void* stream, int P, long long R, int W, int H, const float* means3D, const float* raw_scales,
                            float scale_modifier, const float* raw_rotations, const float* viewmatrix,
                            const float* projmatrix, const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                            const void* geom_buf, const void* binning_buf, const void* image_buf, void* scratch,
                            const float* dL_dpix, float* dL_dmean2D, float* dL_draw_density, float* dL_dmean3D,
                            float* dL_dcov3D, float* dL_draw_scale, float* dL_draw_rot, int mode, const r2x_activation* act) {
    if (!act || !raw_scales || !raw_rotations) return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_raw: null argument");
    ActScope scope(act);
    return r2x_raster_backward(stream, P, R, W, H, means3D, raw_scales, scale_modifier, raw_rotations, nullptr, viewmatrix,
                               projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buf, binning_buf, image_buf, scratch,
                               dL_dpix, dL_dmean2D, dL_draw_density, nullptr, dL_dmean3D, dL_dcov3D, dL_draw_scale,
                               dL_draw_rot, mode, 0);
}

int r2x_voxel_forward_async_raw(void* stream, int P, int nx, int ny, int nz, float sx, float sy, float sz, float cx,
                                float cy, float cz, const float* means3D, const float* raw_density,
                                const float* raw_scales, float scale_modifier, const float* raw_rotations,
                                float* out_volume, int* radii_x, int* radii_y, int* radii_z, void* geom_buf,
                                void* image_buf, void* binning_buf, long long capacity, uint32_t* status_dev,
                                const r2x_activation* act) {
    if (!act || !raw_scales || !raw_rotations) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward_async_raw: null argument");
    ActScope scope(act);
    return r2x_voxel_forward_async(stream, P, nx, ny, nz, sx, sy, sz, cx, cy, cz, means3D, raw_density, raw_scales,
                                   scale_modifier, raw_rotations, nullptr, 0, out_volume, radii_x, radii_y, radii_z, geom_buf,
                                   image_buf, binning_buf, capacity, status_dev);
}

int r2x_voxel_backward_raw(void* stream, int P, long long R, int nx, int ny, int nz, float sx, float sy, float sz, float cx,
                           float cy, float cz, const float* means3D, const float* raw_scales, float scale_modifier,
                           const float* raw_rotations, const int* radii_x, const int* radii_y, const int* radii_z,
                           const void* geom_buf, const void* binning_buf, const void* image_buf, void* scratch,
                           const float* dL_dvol, float* dL_draw_density, float* dL_dmean3D, float* dL_dcov3D,
                           float* dL_draw_scale, float* dL_draw_rot, const r2x_activation* act) {
    if (!act || !raw_scales || !raw_rotations) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_backward_raw: null argument");
    ActScope scope(act);
    return r2x_voxel_backward(stream, P, R, nx, ny, nz, sx, sy, sz, cx, cy, cz, means3D, raw_scales, scale_modifier,
                              raw_rotations, nullptr, radii_x, radii_y, radii_z, geom_buf, binning_buf, image_buf, scratch,
                              dL_dvol, dL_draw_density, dL_dmean3D, dL_dcov3D, dL_draw_scale, dL_draw_rot, 0);
}

size_t r2x_knn_scratch_bytes(int P) { return r2x::knn_scratch_bytes(P); }

int r2x_knn3_mean_dist2(void* stream, int P, const float* points, float* mean_dist2, void* scratch,
                        size_t scratch_bytes) {
    if (P < 0) return fail_msg(R2X_ERR_INVALID, "r2x_knn3_mean_dist2: bad P");
    return r2x::launch_knn3((cudaStream_t)stream, P, points, mean_dist2, scratch, scratch_bytes);
}

size_t r2x_image_loss_scratch_bytes(int H, int W) { return r2x::image_loss_scratch_bytes(H, W); }

int r2x_image_loss(void* stream, int H, int W, const float* image, const float* target, float w_l1, float w_dssim,
                   float* loss_out, float* grad_out, void* scratch, size_t scratch_bytes) {
    return r2x::launch_image_loss((cudaStream_t)stream, H, W, image, target, w_l1, w_dssim, loss_out, grad_out, scratch,
                                  scratch_bytes);
}

size_t r2x_tv3d_scratch_bytes(int nx, int ny, int nz) { return r2x::tv3d_scratch_bytes(nx, ny, nz); }

int r2x_tv3d_loss(void* stream, int nx, int ny, int nz, const float* vol, int reduction_mean, float* loss_out,
                  float* grad_out, void* scratch, size_t scratch_bytes) {
    return r2x::launch_tv3d((cudaStream_t)stream, nx, ny, nz, vol, reduction_mean, loss_out, grad_out, scratch,
                            scratch_bytes);
}

int r2x_adam_step(void* stream, int ngroups, const r2x_adam_group* groups, double beta1, double beta2, double eps,
                  long long step) {
    if (ngroups > 0 && !groups) return fail_msg(R2X_ERR_INVALID, "r2x_adam_step: null groups");
    return r2x::launch_adam((cudaStream_t)stream, ngroups, groups, beta1, beta2, eps, step, nullptr, nullptr, nullptr);
}

int r2x_adam_step_sum(void* stream, int ngroups, const r2x_adam_group* groups, const float* const* grads2, double beta1,
                      double beta2, double eps, long long step, const uint32_t* guard0, const uint32_t* guard1) {
    if (ngroups > 0 && !groups) return fail_msg(R2X_ERR_INVALID, "r2x_adam_step_sum: null groups");
    return r2x::launch_adam((cudaStream_t)stream, ngroups, groups, beta1, beta2, eps, step, grads2, guard0, guard1);
}

int r2x_densify_stats(void* stream, int P, const int* radii, const float* dL_dmean2D, float* max_radii2D,
                      float* xyz_gradient_accum, float* denom, const uint32_t* guard0, const uint32_t* guard1) {
    if (P > 0 && (!radii || !dL_dmean2D || !max_radii2D || !xyz_gradient_accum || !denom))
        return fail_msg(R2X_ERR_INVALID, "r2x_densify_stats: null pointer");
    return r2x::launch_densify_stats((cudaStream_t)stream, P, radii, dL_dmean2D, max_radii2D, xyz_gradient_accum, denom,
                                     guard0, guard1);
}

}  // extern "C"
