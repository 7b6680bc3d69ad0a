// r2x_raster.cuh -- launchers for the detector-image (X-ray projection) kernels.
#pragma once
#include "r2x_common.cuh"
#include "r2x_binning.cuh"

namespace r2x {

// Per-Gaussian projected state ("geometry buffer"), device pointers carved from the caller's buffer.
struct RasterGeom {
    float4* rec;              // [2P] (pix_x, pix_y, log2(w = rho*mu), 0 [fast path] | w [exact path]), (A,B,C scaled by log2e/2, log2e, log2e/2, K = 2^(-2 A2))
    float4* aux;              // [P]  (A, B, C, rho) raw conic + density (backward / parity export)
    float* depth;             // [P]  view-space depth (the low half of the reference's sort key)
    float* mu;                // [P]  integration factor mu (backward / parity export)
    uint16_t* cube;           // [6P] tile rectangle x0,y0,0,x1,y1,1
    uint32_t* tiles_touched;  // [P]
    uint32_t* offsets;        // [P] inclusive scan of tiles_touched
    int gx, gy;               // tile grid
};

int launch_raster_preprocess(cudaStream_t st, int P, const float* means, const float* scales, float scale_modifier,
                             const float* rots, const float* opac, const float* cov3D_precomp, const float* view,
                             const float* proj, int W, int H, float tan_fovx, float tan_fovy, int mode,
                             int prefiltered, int* radii, const RasterGeom& geom, const DirectBin* db);
int launch_raster_render(cudaStream_t st, int W, int H, const RasterGeom& geom, const uint2* ranges,
                         const uint32_t* point_list, const TilePlan& plan, long long R_launch, float* out_color);
int launch_raster_render_bwd(cudaStream_t st, int W, int H, const RasterGeom& geom, const uint2* ranges,
                             const uint32_t* point_list, const uint32_t* inst_pos, const TilePlan& plan,
                             const float* dL_dpix, float4* inst_grad);
int launch_raster_gauss_bwd(cudaStream_t st, int P, const float* means, const int* radii, const float* scales,
                            float scale_modifier, const float* rots, const float* cov3D_precomp, const float* view,
                            const float* proj, int W, int H, float tan_fovx, float tan_fovy, int mode,
                            const RasterGeom& geom, long long capacity, const uint32_t* inst_pos,
                            const float4* inst_grad, float* dL_dmean2D, float* dL_dopacity, float* dL_dmu, float* dL_dmean3D,
                            float* dL_dcov3D, float* dL_dscale, float* dL_drot, void* pose_scratch = nullptr,
                            float* dL_dview = nullptr, float* dL_dproj = nullptr);
// batched views (r2x_raster_forward_views_async / r2x_raster_backward_views): `geom` is carved for vb.views * Pp
// virtual Gaussians (Pp = vb.band_ctas * DIRECT_BLOCK) with the tile grid of ONE view (geom.gx, geom.gy = band rows);
// `db` (direct binning) is the views layout of directbin_views_view; out / dL_dpix are [views][H][W]
int launch_raster_preprocess_views(cudaStream_t st, int P, int views, const float* means, const float* scales,
                                   float scale_modifier, const float* rots, const float* opac, const float* viewmats,
                                   const float* projmats, int W, int H, float tan_fovx, float tan_fovy, int mode,
                                   int* radii, const RasterGeom& geom, const DirectBin* db, const ViewBands& vb);
int launch_raster_render_views(cudaStream_t st, int W, int H, int band_rows, const RasterGeom& geom, const uint2* ranges,
                               const uint32_t* point_list, const TilePlan& plan, long long R_launch, float* out);
int launch_raster_render_bwd_views(cudaStream_t st, int W, int H, int band_rows, const RasterGeom& geom,
                                   const uint2* ranges, const uint32_t* point_list, const uint32_t* inst_pos,
                                   const TilePlan& plan, const float* dL_dpix, float4* inst_grad);
int launch_raster_gauss_bwd_views(cudaStream_t st, int P, int views, int Pp, const float* means, const int* radii,
                                  const float* scales, float scale_modifier, const float* rots, const float* viewmats,
                                  const float* projmats, int W, int H, float tan_fovx, float tan_fovy, int mode,
                                  const RasterGeom& geom, long long capacity, const float4* inst_grad, float* dL_dmean2D,
                                  float* dL_dopacity, float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale,
                                  float* dL_drot);
// pose_scratch of launch_raster_gauss_bwd (the per-CTA rows of the view / projection matrix gradients)
size_t raster_pose_scratch_bytes(int P);
int launch_mark_visible(cudaStream_t st, int P, const float* means, const float* view, unsigned char* present);

}  // namespace r2x
