// r2x_api.cu -- the C ABI declared in include/r2x.h: buffer carving, stage orchestration, error
// reporting.  Stage order (both pipelines): preprocess -> binning (bin_forward: scan -> [sync variant: read R,
// obtain the binning buffer] -> direct fill | two-level | emit + stable tile-id sort + ranges, and the work plan)
// -> render.
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
int launch_densify_stats_views(cudaStream_t st, int N, int P, const int* radii, const float* grad2d, float* max_radii,
                               float* accum, float* denom, const uint32_t* guard0, const uint32_t* guard1);
size_t image_loss_views_scratch_bytes(int N, int H, int W);
int launch_image_loss_views(cudaStream_t st, int N, int H, int W, const float* images, const float* targets, float w_l1,
                            float w_dssim, float* loss_out, float* grad_out, void* scratch, size_t scratch_bytes);

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

// ---- binning front-end shared by both pipelines --------------------------------------------------
// What the front-end needs to know about a pipeline: its tile grid, whether it has a two-level binning path, and the
// largest work-plan chunk its render kernels take.
struct Pipeline {
    const char* name;   // "raster" | "voxel": error messages, debug stages
    int gx, gy, gz;
    bool two_level;
    int chunk_cap;
    int tiles() const { return gx * gy * gz; }
    BinPath path() const { return bin_path(gx, gy, gz, two_level); }
};
Pipeline raster_pipeline(int W, int H) {
    return {"raster", (W + R2X_TILE - 1) / R2X_TILE, (H + R2X_TILE - 1) / R2X_TILE, 1, false, PLAN_CHUNK};
}
// voxelizer work items may hold up to VOX_CHUNK_CAP instances (walked in segments), see plan_chunk_for
Pipeline voxel_pipeline(int nx, int ny, int nz) {
    return {"voxel", (nx + R2X_VTILE - 1) / R2X_VTILE, (ny + R2X_VTILE - 1) / R2X_VTILE, (nz + R2X_VTILE - 1) / R2X_VTILE,
            true, VOX_CHUNK_CAP};
}

struct ImageViews {
    uint2* ranges;   // [T]
    TilePlan plan;   // its extra-item list and partial sums live in the binning buffer
    DirectBin db;    // direct binning only
    TwoLevel tl;     // two-level binning only
};
// image buffer = ranges[T] | work plan | direct-binning table (T <= DIRECT_MAX_TILES) or two-level scratch (sized by the
// geometry alone, whatever R2X_VOXEL_BINNING says).  Returns the size r2x_*_image_bytes reports; carves *v when given.
// With `vb` (batched views; pp is the stacked grid, P the virtual Gaussian count) the direct table is the banded one.
size_t image_layout(const void* buf, int P, const Pipeline& pp, const BinningView& bv, ImageViews* v,
                    const ViewBands* vb = nullptr) {
    const size_t t = (size_t)pp.gx * pp.gy * pp.gz;
    const int T = (int)t;
    const size_t head = al(t * sizeof(uint2)) + plan_bytes(T);
    const bool direct = pp.path() == BinPath::Direct;
    const size_t tail = direct ? (vb ? directbin_views_bytes(*vb) : directbin_bytes(P, T))
                        : pp.two_level ? two_level_bytes(P, pp.gx, pp.gy, pp.gz) : 0;
    if (v) {
        char* base = (char*)al((size_t)buf);
        v->ranges = (uint2*)base;
        v->plan = plan_view(base + al(t * sizeof(uint2)), T, bv);
        v->plan.chunk_cap = pp.chunk_cap;
        v->db = !direct ? DirectBin{} : vb ? directbin_views_view(base + head, *vb) : directbin_view(base + head, P, T);
        v->tl = (!direct && tail) ? two_level_view(base + head, P, pp.gx, pp.gy, pp.gz, bv) : TwoLevel{};
    }
    return head + tail + 1024;
}
ImageViews image_views(const void* buf, int P, const Pipeline& pp, const BinningView& bv, const ViewBands* vb = nullptr) {
    ImageViews v;
    image_layout(buf, P, pp, bv, &v, vb);
    return v;
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
// keys[s] = (tile << 32) | float_bits(depth of point_list[s]); the depth of Gaussian g is depth[depth_stride * g]
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

// the voxelizer's view-space depth of Gaussian g is rec[4 g + 3].y: float 13 of its 16-float record
const float* voxel_depth(const VoxelGeom& geom) { return reinterpret_cast<const float*>(geom.rec + 3) + 1; }
constexpr int VOX_DEPTH_STRIDE = 4 * sizeof(float4) / sizeof(float);

// ranges (reference convention), keys and point_list of a forward's binning; the depth of Gaussian g is
// depth[depth_stride * g]
void export_binning(cudaStream_t st, int P, const Pipeline& pp, long long R, const void* binning_buf,
                    const void* image_buf, const uint32_t* status, const float* depth, int depth_stride, uint64_t* keys,
                    uint32_t* point_list, uint32_t* ranges) {
    const int T = pp.tiles();
    const ImageViews img = image_views(image_buf, P, pp, BinningView{});
    if (ranges) export_ranges_kernel<<<(unsigned)((T + 255) / 256), 256, 0, st>>>(T, img.ranges, ranges);
    if (R <= 0 || (!keys && !point_list)) return;
    const BinningView bv = binning_view((void*)binning_buf, R);
    const unsigned grid = (unsigned)((R + 255) / 256);
    if (pp.path() == BinPath::Radix)
        export_keys_kernel<<<grid, 256, 0, st>>>(R, status, sorted_tile_ids(bv, T), bv.point_list, depth, depth_stride,
                                                 keys, point_list);
    else
        export_keys_ranges_kernel<<<grid, 256, 0, st>>>(R, status, img.ranges, T, bv.point_list, depth, depth_stride,
                                                        keys, point_list);
}

// P == 0: zero output, empty ranges, R = 0 and no overflow
int forward_empty(cudaStream_t st, const Pipeline& pp, float* out, size_t out_elems, const void* image_buf,
                  uint32_t* status, uint32_t* status_dev) {
    R2X_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float) * out_elems, st));
    R2X_CUDA_OK(cudaMemsetAsync(image_views(image_buf, 0, pp, BinningView{}).ranges, 0, sizeof(uint2) * (size_t)pp.tiles(), st));
    R2X_CUDA_OK(cudaMemsetAsync(status, 0, 16, st));
    if (status_dev) R2X_CUDA_OK(cudaMemsetAsync(status_dev, 0, 8, st));
    return 0;
}

// The binning sequence of both forwards, after their preprocess: scan (direct binning: direct_scan, which also publishes
// the ranges, the work plan and R); [synchronous variant (binning_alloc): read R back, allocate the binning buffer];
// then direct fill, two-level binning, or emit + sort + ranges and the plan.  R and the overflow flag go to status
// (and, asynchronous variant, to status_dev); on overflow the ranges are empty.  The render then reads *bv (its
// capacity sizes the render grid) and *img.
int bin_forward(cudaStream_t st, const Pipeline& pp, BinPath path, int P, const uint16_t* cube,
                const uint32_t* tiles_touched, uint32_t* offsets, void* scan_state, uint32_t* status,
                const void* image_buf, r2x_alloc_fn binning_alloc, void* alloc_user, void* binning_buf,
                long long capacity, uint32_t* status_dev, int debug, int* num_rendered, BinningView* bv,
                ImageViews* img, const ViewBands* vb = nullptr) {
    const std::string fn = std::string("r2x_") + pp.name + "_forward";
    if (path == BinPath::Direct) {
        // tile ranges, work plan and R come straight from the per-CTA tile histograms (the plan's extra-item list,
        // which lives in the binning buffer, is written by direct_fill)
        const ImageViews pre = image_views(image_buf, P, pp, BinningView{}, vb);
        const long long cap0 = binning_alloc ? (1ll << 62) : capacity;
        uint32_t* sd = binning_alloc ? nullptr : status_dev;
        if (vb) R2X_TRY(launch_direct_scan_views(st, pre.db, *vb, pre.ranges, pre.plan, status, cap0, sd));
        else R2X_TRY(launch_direct_scan(st, pre.db, pre.ranges, pre.plan, status, cap0, sd));
    } else {
        R2X_TRY(launch_scan(st, P, tiles_touched, offsets, scan_state, status));
    }
    R2X_TRY(debug_sync(st, debug, (std::string(pp.name) + " scan").c_str()));
    if (binning_alloc) {  // synchronous variant: learn R, size the binning buffer exactly
        uint32_t R = 0;
        R2X_CUDA_OK(cudaMemcpyAsync(&R, status, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        R2X_CUDA_OK(cudaStreamSynchronize(st));
        if (num_rendered) *num_rendered = (int)R;
        binning_buf = binning_alloc(binning_bytes((long long)R), alloc_user);
        if (!binning_buf) return fail_msg(R2X_ERR_INVALID, (fn + ": binning allocator returned NULL").c_str());
        capacity = R;
    } else if (!binning_buf || capacity < 0) {
        return fail_msg(R2X_ERR_INVALID, (fn + "_async: no binning buffer").c_str());
    }
    *bv = binning_view(binning_buf, capacity);
    *img = image_views(image_buf, P, pp, *bv, vb);
    if (path == BinPath::Direct) {
        if (vb)
            R2X_TRY(launch_direct_fill_views(st, P, cube, tiles_touched, offsets, img->db, *vb, img->plan, *bv, pp.gx, pp.gy,
                                             status));
        else
            R2X_TRY(launch_direct_fill(st, P, cube, tiles_touched, offsets, img->db, img->plan, *bv, pp.gx, pp.gy, status));
    } else {
        status_kernel<<<1, 1, 0, st>>>(status, capacity, status_dev);
        if (path == BinPath::TwoLevel) {
            R2X_TRY(launch_two_level(st, P, cube, tiles_touched, pp.gx, pp.gy, pp.gz, status, img->tl, *bv, img->ranges,
                                     img->plan));
        } else {
            if (capacity > 0) R2X_TRY(launch_emit(st, P, cube, tiles_touched, offsets, pp.gx, pp.gy, status, *bv));
            R2X_TRY(launch_sort_and_ranges(st, capacity, pp.tiles(), status, *bv, img->ranges));
            R2X_TRY(launch_plan(st, img->ranges, img->plan));
        }
    }
    return debug_sync(st, debug, (std::string(pp.name) + " binning").c_str());
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
    if (s.geom.gx > 65535 || s.geom.gy > 65535) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: detector too large");
    const Pipeline pp = raster_pipeline(W, H);
    if (P == 0) return forward_empty(st, pp, out_color, (size_t)W * H, image_buf, s.status, status_dev);
    if (!means3D || !opacities || !radii || !viewmatrix || !projmatrix)
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: null input");
    if (!cov3D_precomp && (!scales || !rotations))
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward: need scales+rotations or cov3D_precomp");
    const BinPath path = pp.path();
    ImageViews img = image_views(image_buf, P, pp, BinningView{});
    R2X_TRY(launch_raster_preprocess(st, P, means3D, scales, scale_modifier, rotations, opacities, cov3D_precomp,
                                     viewmatrix, projmatrix, W, H, tan_fovx, tan_fovy, mode, prefiltered, radii,
                                     s.geom, path == BinPath::Direct ? &img.db : nullptr));
    R2X_TRY(debug_sync(st, debug, "raster preprocess"));
    BinningView bv;
    R2X_TRY(bin_forward(st, pp, path, P, s.geom.cube, s.geom.tiles_touched, s.geom.offsets, s.scan_state, s.status,
                        image_buf, binning_alloc, alloc_user, binning_buf, capacity, status_dev, debug, num_rendered, &bv,
                        &img));
    R2X_TRY(launch_raster_render(st, W, H, s.geom, img.ranges, bv.point_list, img.plan, bv.capacity, out_color));
    R2X_TRY(debug_sync(st, debug, "raster render"));
    return 0;
}

// ---- batched views: N views of one cloud as the bands of one stacked tile grid (ViewBands, r2x_binning.cuh) ----------
struct ViewsShape {
    int Pv;         // virtual Gaussians N * Pp
    ViewBands vb;
    Pipeline pp;    // the stacked grid gx x gy x N (z = view)
};
// Checks the sizes (no CUDA call) and derives the layout of a batched forward / backward.
int views_shape(const char* fn, int P, int N, int W, int H, ViewsShape* s) {
    if (N < 1) return fail_msg(R2X_ERR_INVALID, (std::string(fn) + ": bad N (need at least one view)").c_str());
    if (W <= 0 || H <= 0 || P < 0) return fail_msg(R2X_ERR_INVALID, (std::string(fn) + ": bad P/W/H").c_str());
    const long long gx = (W + R2X_TILE - 1) / R2X_TILE, gy = (H + R2X_TILE - 1) / R2X_TILE;
    if (gx > 65535 || (long long)N * gy > 65535)
        return fail_msg(R2X_ERR_INVALID, (std::string(fn) + ": bad N/W/H (too many tile rows: N * ceil(H / 16) and "
                                                             "ceil(W / 16) must be <= 65535)").c_str());
    const long long Pp = ((long long)(P > 0 ? P : 1) + DIRECT_BLOCK - 1) / DIRECT_BLOCK * DIRECT_BLOCK;
    if (Pp * N > (1ll << 31) - 1 || gx * gy * N > (1ll << 30))
        return fail_msg(R2X_ERR_INVALID, (std::string(fn) + ": bad N/P (too many views x Gaussians or tiles)").c_str());
    s->Pv = (int)(Pp * N);
    s->vb = ViewBands{N, (int)(gx * gy), (int)(Pp / DIRECT_BLOCK)};
    s->pp = Pipeline{"raster_views", (int)gx, (int)gy, N, false, PLAN_CHUNK};
    return 0;
}

int raster_views_forward_impl(cudaStream_t st, int P, int N, int W, int H, const float* means3D, const float* opacities,
                              const float* scales, float scale_modifier, const float* rotations, const float* viewmatrices,
                              const float* projmatrices, float tan_fovx, float tan_fovy, int mode, float* out, int* radii,
                              void* geom_buf, void* image_buf, void* binning_buf, long long capacity,
                              uint32_t* status_dev) {
    const char* fn = "r2x_raster_forward_views_async";
    ViewsShape vs;
    R2X_TRY(views_shape(fn, P, N, W, H, &vs));
    if (!out || !geom_buf || !image_buf) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward_views_async: null output/state buffer");
    if (mode != 0 && mode != 1)
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward_views_async: mode must be 0 (parallel) or 1 (cone)");
    if (!binning_buf || capacity < 0) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward_views_async: no binning buffer");
    if (P > 0 && (!means3D || !opacities || !scales || !rotations || !radii || !viewmatrices || !projmatrices))
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward_views_async: null input");
    RasterState s = carve_raster(geom_buf, vs.Pv, W, H);   // the tile grid of one view
    if (P == 0) return forward_empty(st, vs.pp, out, (size_t)N * W * H, image_buf, s.status, status_dev);
    const BinPath path = vs.pp.path();
    ImageViews img = image_views(image_buf, vs.Pv, vs.pp, BinningView{}, &vs.vb);
    R2X_TRY(launch_raster_preprocess_views(st, P, N, means3D, scales, scale_modifier, rotations, opacities, viewmatrices,
                                           projmatrices, W, H, tan_fovx, tan_fovy, mode, radii, s.geom,
                                           path == BinPath::Direct ? &img.db : nullptr, vs.vb));
    BinningView bv;
    R2X_TRY(bin_forward(st, vs.pp, path, vs.Pv, s.geom.cube, s.geom.tiles_touched, s.geom.offsets, s.scan_state, s.status,
                        image_buf, nullptr, nullptr, binning_buf, capacity, status_dev, 0, nullptr, &bv, &img, &vs.vb));
    return launch_raster_render_views(st, W, H, s.geom.gy, s.geom, img.ranges, bv.point_list, img.plan, bv.capacity, out);
}

int raster_views_backward_impl(cudaStream_t st, int P, int N, long long R, int W, int H, const float* means3D,
                               const float* scales, float scale_modifier, const float* rotations,
                               const float* viewmatrices, const float* projmatrices, float tan_fovx, float tan_fovy,
                               const int* radii, const void* geom_buf, const void* binning_buf, const void* image_buf,
                               void* scratch, const float* dL_dpix, float* dL_dmean2D, float* dL_dopacity,
                               float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale, float* dL_drot, int mode,
                               int debug) {
    const char* fn = "r2x_raster_backward_views";
    ViewsShape vs;
    R2X_TRY(views_shape(fn, P, N, W, H, &vs));
    if (R < 0) return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_views: bad R");
    if (mode != 0 && mode != 1) return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_views: mode must be 0 or 1");
    if (P == 0) return 0;
    if (!geom_buf || !image_buf || !dL_dpix || !dL_dmean2D || !dL_dopacity || !dL_dmean3D || !dL_dcov3D || !dL_dscale ||
        !dL_drot || !radii || !means3D || !scales || !rotations || !viewmatrices || !projmatrices)
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_views: null pointer");
    if (R > 0 && (!binning_buf || !scratch))
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_views: null binning/scratch");
    RasterState s = carve_raster(geom_buf, vs.Pv, W, H);
    BinningView bv = binning_view((void*)binning_buf, R);
    const ImageViews img = image_views(image_buf, vs.Pv, vs.pp, bv, &vs.vb);
    float4* inst_grad = (float4*)al((size_t)scratch);
    const uint32_t* inst_pos = vs.pp.path() == BinPath::Radix ? bv.inst_pos : nullptr;   // otherwise slots are derived
    if (R > 0)
        R2X_TRY(launch_raster_render_bwd_views(st, W, H, s.geom.gy, s.geom, img.ranges, bv.point_list, inst_pos, img.plan,
                                               dL_dpix, inst_grad));
    R2X_TRY(debug_sync(st, debug, "raster views render backward"));
    R2X_TRY(launch_raster_gauss_bwd_views(st, P, N, vs.vb.band_ctas * DIRECT_BLOCK, means3D, radii, scales, scale_modifier,
                                          rotations, viewmatrices, projmatrices, W, H, tan_fovx, tan_fovy, mode, s.geom, R,
                                          inst_grad, dL_dmean2D, dL_dopacity, dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot));
    return debug_sync(st, debug, "raster views per-Gaussian backward");
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
    VoxelState s = carve_voxel(geom_buf, P);
    const Pipeline pp = voxel_pipeline(nx, ny, nz);
    if (P == 0) return forward_empty(st, pp, out_volume, (size_t)nx * ny * nz, image_buf, s.status, status_dev);
    if (!means3D || !opacities || !radii_x || !radii_y || !radii_z)
        return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward: null input");
    if (!scales)
        return fail_msg(R2X_ERR_INVALID,
                        "r2x_voxel_forward: scales are required (the bounding radius is 3*max(scale)/dVoxel even "
                        "with cov3D_precomp; the reference dereferences scales unconditionally, VOX/forward.cu:137)");
    if (!cov3D_precomp && !rotations) return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward: need rotations or cov3D_precomp");
    const BinPath path = pp.path();
    ImageViews img = image_views(image_buf, P, pp, BinningView{});
    R2X_TRY(launch_voxel_preprocess(st, P, means3D, scales, scale_modifier, rotations, opacities, cov3D_precomp, vg,
                                    radii_x, radii_y, radii_z, s.geom, path == BinPath::Direct ? &img.db : nullptr));
    R2X_TRY(debug_sync(st, debug, "voxel preprocess"));
    BinningView bv;
    R2X_TRY(bin_forward(st, pp, path, P, s.geom.cube, s.geom.tiles_touched, s.geom.offsets, s.scan_state, s.status,
                        image_buf, binning_alloc, alloc_user, binning_buf, capacity, status_dev, debug, num_rendered, &bv,
                        &img));
    R2X_TRY(launch_voxel_render(st, vg, s.geom, img.ranges, bv.point_list, img.plan, bv.capacity, out_volume));
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
    return image_layout(nullptr, P, raster_pipeline(W, H), BinningView{}, nullptr);
}
size_t r2x_voxel_geom_bytes(int P) { return voxel_geom_bytes(P); }
size_t r2x_voxel_image_bytes(int P, int nx, int ny, int nz) {
    return image_layout(nullptr, P, voxel_pipeline(nx, ny, nz), BinningView{}, nullptr);
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

size_t r2x_raster_views_geom_bytes(int P, int N) {
    ViewsShape vs;
    return views_shape("r2x_raster_views_geom_bytes", P, N, 1, 1, &vs) ? 0 : raster_geom_bytes(vs.Pv);
}
size_t r2x_raster_views_image_bytes(int P, int N, int W, int H) {
    ViewsShape vs;
    if (views_shape("r2x_raster_views_image_bytes", P, N, W, H, &vs)) return 0;
    return image_layout(nullptr, vs.Pv, vs.pp, BinningView{}, nullptr, &vs.vb);
}

int r2x_raster_forward_views_async(void* stream, int P, int N, int W, int H, const float* means3D,
                                   const float* opacities, const float* scales, float scale_modifier,
                                   const float* rotations, const float* viewmatrices, const float* projmatrices,
                                   float tan_fovx, float tan_fovy, int mode, float* out_color, int* radii,
                                   void* geom_buf, void* image_buf, void* binning_buf, long long capacity,
                                   uint32_t* status_dev) {
    return raster_views_forward_impl((cudaStream_t)stream, P, N, W, H, means3D, opacities, scales, scale_modifier,
                                     rotations, viewmatrices, projmatrices, tan_fovx, tan_fovy, mode, out_color, radii,
                                     geom_buf, image_buf, binning_buf, capacity, status_dev);
}

int r2x_raster_backward_views(void* stream, int P, int N, long long R, int W, int H, const float* means3D,
                              const float* scales, float scale_modifier, const float* rotations,
                              const float* viewmatrices, const float* projmatrices, float tan_fovx, float tan_fovy,
                              const int* radii, const void* geom_buf, const void* binning_buf, const void* image_buf,
                              void* scratch, const float* dL_dpix, float* dL_dmean2D, float* dL_dopacity,
                              float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale, float* dL_drot, int mode,
                              int debug) {
    return raster_views_backward_impl((cudaStream_t)stream, P, N, R, W, H, means3D, scales, scale_modifier, rotations,
                                      viewmatrices, projmatrices, tan_fovx, tan_fovy, radii, geom_buf, binning_buf,
                                      image_buf, scratch, dL_dpix, dL_dmean2D, dL_dopacity, dL_dmean3D, dL_dcov3D,
                                      dL_dscale, dL_drot, mode, debug);
}

int r2x_raster_render_only(void* stream, int P, int W, int H, long long R, const void* geom_buf,
                           const void* binning_buf, const void* image_buf, float* out_color) {
    if (P <= 0 || R < 0 || !geom_buf || !image_buf || !out_color || (R > 0 && !binning_buf))
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_render_only: bad args");
    RasterState s = carve_raster(geom_buf, P, W, H);
    BinningView bv = binning_view((void*)binning_buf, R);
    const ImageViews img = image_views(image_buf, P, raster_pipeline(W, H), bv);
    R2X_TRY(rewind_plan((cudaStream_t)stream, img.plan));
    return launch_raster_render((cudaStream_t)stream, W, H, s.geom, img.ranges, bv.point_list, img.plan, R, out_color);
}

int r2x_voxel_render_only(void* stream, int P, int nx, int ny, int nz, long long R, const void* geom_buf,
                          const void* binning_buf, const void* image_buf, float* out_volume) {
    if (P <= 0 || R < 0 || !geom_buf || !image_buf || !out_volume || (R > 0 && !binning_buf))
        return fail_msg(R2X_ERR_INVALID, "r2x_voxel_render_only: bad args");
    const VoxelGrid vg = make_voxel_grid(nx, ny, nz, 1.f, 1.f, 1.f, 0.f, 0.f, 0.f);  // render needs the tile grid only
    VoxelState s = carve_voxel(geom_buf, P);
    BinningView bv = binning_view((void*)binning_buf, R);
    const ImageViews img = image_views(image_buf, P, voxel_pipeline(nx, ny, nz), bv);
    R2X_TRY(rewind_plan((cudaStream_t)stream, img.plan));
    return launch_voxel_render((cudaStream_t)stream, vg, s.geom, img.ranges, bv.point_list, img.plan, R, out_volume);
}

}  // extern "C"

namespace {
// r2x_raster_backward, and with pose_scratch != NULL also dL_dview / dL_dproj (r2x_raster_backward_pose)
int raster_backward_impl(void* stream, int P, long long R, int W, int H, const float* means3D, const float* scales,
                         float scale_modifier, const float* rotations, const float* cov3D_precomp,
                         const float* viewmatrix, const float* projmatrix, float tan_fovx, float tan_fovy,
                         const int* radii, const void* geom_buf, const void* binning_buf, const void* image_buf,
                         void* scratch, const float* dL_dpix, float* dL_dmean2D, float* dL_dopacity, float* dL_dmu,
                         float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale, float* dL_drot, int mode, int debug,
                         void* pose_scratch, float* dL_dview, float* dL_dproj) {
    cudaStream_t st = (cudaStream_t)stream;
    if (P == 0) {   // no Gaussian: the matrix gradients are zero
        if (pose_scratch) {
            R2X_CUDA_OK(cudaMemsetAsync(dL_dview, 0, 16 * sizeof(float), st));
            R2X_CUDA_OK(cudaMemsetAsync(dL_dproj, 0, 16 * sizeof(float), st));
        }
        return 0;
    }
    if (P < 0 || W <= 0 || H <= 0 || R < 0) return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward: bad sizes");
    if (!geom_buf || !image_buf || !dL_dpix || !dL_dmean2D || !dL_dopacity || !dL_dmean3D || !dL_dcov3D ||
        !dL_dscale || !dL_drot || !radii || !means3D)
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward: null pointer");
    if (R > 0 && (!binning_buf || !scratch)) return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward: null binning/scratch");
    RasterState s = carve_raster(geom_buf, P, W, H);
    const Pipeline pp = raster_pipeline(W, H);
    BinningView bv = binning_view((void*)binning_buf, R);
    const ImageViews img = image_views(image_buf, P, pp, bv);
    float4* inst_grad = (float4*)al((size_t)scratch);
    const uint32_t* inst_pos = pp.path() == BinPath::Radix ? bv.inst_pos : nullptr;   // otherwise slots are derived
    if (R > 0)
        R2X_TRY(launch_raster_render_bwd(st, W, H, s.geom, img.ranges, bv.point_list, inst_pos, img.plan, dL_dpix, inst_grad));
    R2X_TRY(debug_sync(st, debug, "raster render backward"));
    R2X_TRY(launch_raster_gauss_bwd(st, P, means3D, radii, scales, scale_modifier, rotations, cov3D_precomp, viewmatrix,
                                    projmatrix, W, H, tan_fovx, tan_fovy, mode, s.geom, R, bv.inst_pos, inst_grad,
                                    dL_dmean2D, dL_dopacity, dL_dmu, dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot,
                                    pose_scratch, dL_dview, dL_dproj));
    R2X_TRY(debug_sync(st, debug, "raster per-Gaussian backward"));
    return 0;
}
}  // namespace

extern "C" {

int r2x_raster_backward(void* stream, int P, long long R, int W, int H, const float* means3D, const float* scales,
                        float scale_modifier, const float* rotations, const float* cov3D_precomp,
                        const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                        float tan_fovy, const int* radii, const void* geom_buf, const void* binning_buf,
                        const void* image_buf, void* scratch, const float* dL_dpix, float* dL_dmean2D,
                        float* dL_dopacity, float* dL_dmu, float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale,
                        float* dL_drot, int mode, int debug) {
    (void)campos;
    return raster_backward_impl(stream, P, R, W, H, means3D, scales, scale_modifier, rotations, cov3D_precomp, viewmatrix,
                                projmatrix, tan_fovx, tan_fovy, radii, geom_buf, binning_buf, image_buf, scratch, dL_dpix,
                                dL_dmean2D, dL_dopacity, dL_dmu, dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot, mode, debug,
                                nullptr, nullptr, nullptr);
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
    export_binning(st, P, raster_pipeline(W, H), R, binning_buf, image_buf, s.status, s.geom.depth, 1, keys, point_list,
                   ranges);
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
    const Pipeline pp = voxel_pipeline(nx, ny, nz);
    BinningView bv = binning_view((void*)binning_buf, R);
    const ImageViews img = image_views(image_buf, P, pp, bv);
    float4* inst_grad = (float4*)al((size_t)scratch);
    const uint32_t* inst_pos = pp.path() == BinPath::Radix ? bv.inst_pos : nullptr;   // otherwise slots are derived
    if (R > 0)
        R2X_TRY(launch_voxel_render_bwd(st, vg, s.geom, img.ranges, bv.point_list, inst_pos, img.plan, R, dL_dvol, inst_grad));
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
    export_binning(st, P, voxel_pipeline(nx, ny, nz), R, binning_buf, image_buf, s.status, voxel_depth(s.geom),
                   VOX_DEPTH_STRIDE, keys, point_list, ranges);
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
    // P == 0 (an empty shard of a Gaussian-sharded run) passes null parameter pointers: the call below zeroes
    // the output and status and reads no parameter
    if (!act || (P > 0 && (!raw_scales || !raw_rotations)))
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward_async_raw: null argument");
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
    if (!act || (P > 0 && (!raw_scales || !raw_rotations)))
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_raw: null argument");
    ActScope scope(act);
    return r2x_raster_backward(stream, P, R, W, H, means3D, raw_scales, scale_modifier, raw_rotations, nullptr, viewmatrix,
                               projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buf, binning_buf, image_buf, scratch,
                               dL_dpix, dL_dmean2D, dL_draw_density, nullptr, dL_dmean3D, dL_dcov3D, dL_draw_scale,
                               dL_draw_rot, mode, 0);
}

int r2x_raster_forward_views_async_raw(void* stream, int P, int N, int W, int H, const float* means3D,
                                       const float* raw_density, const float* raw_scales, float scale_modifier,
                                       const float* raw_rotations, const float* viewmatrices, const float* projmatrices,
                                       float tan_fovx, float tan_fovy, int mode, float* out_color, int* radii,
                                       void* geom_buf, void* image_buf, void* binning_buf, long long capacity,
                                       uint32_t* status_dev, const r2x_activation* act) {
    if (!act) return fail_msg(R2X_ERR_INVALID, "r2x_raster_forward_views_async_raw: null activation");
    ActScope scope(act);
    return raster_views_forward_impl((cudaStream_t)stream, P, N, W, H, means3D, raw_density, raw_scales, scale_modifier,
                                     raw_rotations, viewmatrices, projmatrices, tan_fovx, tan_fovy, mode, out_color, radii,
                                     geom_buf, image_buf, binning_buf, capacity, status_dev);
}

int r2x_raster_backward_views_raw(void* stream, int P, int N, long long R, int W, int H, const float* means3D,
                                  const float* raw_scales, float scale_modifier, const float* raw_rotations,
                                  const float* viewmatrices, const float* projmatrices, float tan_fovx, float tan_fovy,
                                  const int* radii, const void* geom_buf, const void* binning_buf, const void* image_buf,
                                  void* scratch, const float* dL_dpix, float* dL_dmean2D, float* dL_draw_density,
                                  float* dL_dmean3D, float* dL_dcov3D, float* dL_draw_scale, float* dL_draw_rot, int mode,
                                  const r2x_activation* act) {
    if (!act) return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_views_raw: null activation");
    ActScope scope(act);
    return raster_views_backward_impl((cudaStream_t)stream, P, N, R, W, H, means3D, raw_scales, scale_modifier,
                                      raw_rotations, viewmatrices, projmatrices, tan_fovx, tan_fovy, radii, geom_buf,
                                      binning_buf, image_buf, scratch, dL_dpix, dL_dmean2D, dL_draw_density, dL_dmean3D,
                                      dL_dcov3D, dL_draw_scale, dL_draw_rot, mode, 0);
}

size_t r2x_raster_backward_pose_scratch_bytes(int P) { return raster_pose_scratch_bytes(P); }

int r2x_raster_backward_pose(void* stream, int P, long long R, int W, int H, const float* means3D, const float* scales,
                             float scale_modifier, const float* rotations, const float* cov3D_precomp,
                             const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                             float tan_fovy, const int* radii, const void* geom_buf, const void* binning_buf,
                             const void* image_buf, void* scratch, const float* dL_dpix, float* dL_dmean2D,
                             float* dL_dopacity, float* dL_dmu, float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale,
                             float* dL_drot, int mode, int debug, const r2x_activation* act, float* dL_dviewmatrix,
                             float* dL_dprojmatrix, void* pose_scratch, size_t pose_scratch_bytes) {
    (void)campos;
    if (P < 0 || W <= 0 || H <= 0 || R < 0) return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_pose: bad sizes");
    if (!viewmatrix || !projmatrix || !dL_dviewmatrix || !dL_dprojmatrix)
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_pose: null matrix or matrix gradient");
    if (!pose_scratch || pose_scratch_bytes < raster_pose_scratch_bytes(P))
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_pose: pose_scratch is NULL or smaller than "
                                         "r2x_raster_backward_pose_scratch_bytes(P)");
    if (act && (cov3D_precomp || !scales || !rotations))
        return fail_msg(R2X_ERR_INVALID, "r2x_raster_backward_pose: raw parameters need scales and rotations and no "
                                         "cov3D_precomp");
    if (!act)
        return raster_backward_impl(stream, P, R, W, H, means3D, scales, scale_modifier, rotations, cov3D_precomp,
                                    viewmatrix, projmatrix, tan_fovx, tan_fovy, radii, geom_buf, binning_buf, image_buf,
                                    scratch, dL_dpix, dL_dmean2D, dL_dopacity, dL_dmu, dL_dmean3D, dL_dcov3D, dL_dscale,
                                    dL_drot, mode, debug, pose_scratch, dL_dviewmatrix, dL_dprojmatrix);
    ActScope scope(act);
    return raster_backward_impl(stream, P, R, W, H, means3D, scales, scale_modifier, rotations, nullptr, viewmatrix,
                                projmatrix, tan_fovx, tan_fovy, radii, geom_buf, binning_buf, image_buf, scratch, dL_dpix,
                                dL_dmean2D, dL_dopacity, dL_dmu, dL_dmean3D, dL_dcov3D, dL_dscale, dL_drot, mode, debug,
                                pose_scratch, dL_dviewmatrix, dL_dprojmatrix);
}

int r2x_voxel_forward_async_raw(void* stream, int P, int nx, int ny, int nz, float sx, float sy, float sz, float cx,
                                float cy, float cz, const float* means3D, const float* raw_density,
                                const float* raw_scales, float scale_modifier, const float* raw_rotations,
                                float* out_volume, int* radii_x, int* radii_y, int* radii_z, void* geom_buf,
                                void* image_buf, void* binning_buf, long long capacity, uint32_t* status_dev,
                                const r2x_activation* act) {
    if (!act || (P > 0 && (!raw_scales || !raw_rotations)))
        return fail_msg(R2X_ERR_INVALID, "r2x_voxel_forward_async_raw: null argument");
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
    if (!act || (P > 0 && (!raw_scales || !raw_rotations)))
        return fail_msg(R2X_ERR_INVALID, "r2x_voxel_backward_raw: null argument");
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

size_t r2x_image_loss_views_scratch_bytes(int N, int H, int W) { return r2x::image_loss_views_scratch_bytes(N, H, W); }

int r2x_image_loss_views(void* stream, int N, int H, int W, const float* images, const float* targets, float w_l1,
                         float w_dssim, float* loss_out, float* grad_out, void* scratch, size_t scratch_bytes) {
    return r2x::launch_image_loss_views((cudaStream_t)stream, N, H, W, images, targets, w_l1, w_dssim, loss_out, grad_out,
                                        scratch, scratch_bytes);
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

int r2x_densify_stats_views(void* stream, int N, int P, const int* radii, const float* dL_dmean2D, float* max_radii2D,
                            float* xyz_gradient_accum, float* denom, const uint32_t* guard0, const uint32_t* guard1) {
    if (N < 1 || P < 0) return fail_msg(R2X_ERR_INVALID, "r2x_densify_stats_views: bad N/P");
    if (P > 0 && (!radii || !dL_dmean2D || !max_radii2D || !xyz_gradient_accum || !denom))
        return fail_msg(R2X_ERR_INVALID, "r2x_densify_stats_views: null pointer");
    return r2x::launch_densify_stats_views((cudaStream_t)stream, N, P, radii, dL_dmean2D, max_radii2D, xyz_gradient_accum,
                                           denom, guard0, guard1);
}

}  // extern "C"
