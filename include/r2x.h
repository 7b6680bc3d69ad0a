/*
 * r2x.h -- C ABI of libr2xray.so, the H100-native X-ray Gaussian rasterizer + voxelizer.
 *
 * Drop-in boundary for the reference's native entry points (plain pointers and sizes, no torch types):
 *
 *   r2x_raster_forward / _async  <->  CudaRasterizer::Rasterizer::forward   (RAS/rasterizer.h:37-58,
 *                                     bound by RasterizeGaussiansCUDA, SUB/rasterize_points.cu:28-97)
 *   r2x_raster_backward          <->  CudaRasterizer::Rasterizer::backward  (RAS/rasterizer.h:60-85,
 *                                     RasterizeGaussiansBackwardCUDA, SUB/rasterize_points.cu:99-164)
 *   r2x_mark_visible             <->  CudaRasterizer::Rasterizer::markVisible (RAS/rasterizer.h:30-35,
 *                                     markVisible, SUB/rasterize_points.cu:166-186)
 *   r2x_voxel_forward / _async   <->  CudaVoxelizer::Voxelizer::forward     (VOX/voxelizer.h:28-49,
 *                                     VoxelizeGaussiansCUDA, SUB/voxelize_points.cu:29-98)
 *   r2x_voxel_backward           <->  CudaVoxelizer::Voxelizer::backward    (VOX/voxelizer.h:51-72,
 *                                     VoxelizeGaussiansBackwardCUDA, SUB/voxelize_points.cu:102-167)
 *   r2x_*_export                 --   stage outputs for parity tests (the reference keeps them inside
 *                                     its opaque geom/binning/img byte buffers, RAS/rasterizer_impl.h:29-63)
 *
 * (RAS/VOX/SUB = r2_gaussian/submodules/xray-gaussian-rasterization-voxelization/{cuda_rasterizer,
 *  cuda_voxelizer,.} in the reference.)
 *
 * Conventions
 *   - every pointer is a DEVICE pointer on the current CUDA device unless marked "host";
 *     float32, contiguous, same layouts as the reference: means3D[P,3], scales[P,3], rotations[P,4]
 *     (r,x,y,z, consumed un-normalised), opacities[P], cov3D_precomp[P,6] or NULL, viewmatrix /
 *     projmatrix 16 floats column-major-flat (the reference passes them transposed), out_color[1,H,W],
 *     out_volume[nx,ny,nz] (index x*ny*nz + y*nz + z), radii int32[P].
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  All work is enqueued
 *     on it; the *_async entry points never synchronise with the host.
 *   - the three state buffers play the role of the reference's geomBuffer / binningBuffer / imgBuffer:
 *     opaque to the caller, sized by the r2x_*_bytes functions, written by forward, read by backward.
 *   - every function returns 0 on success; otherwise a non-zero code with r2x_last_error() describing
 *     it (invalid argument, CUDA error, capacity overflow).  No CPU fallback exists.
 */
#ifndef R2X_H_INCLUDED
#define R2X_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define R2X_OK 0
#define R2X_ERR_INVALID 1
#define R2X_ERR_CUDA 2
#define R2X_ERR_OVERFLOW 3

/* Allocator callback used by the synchronous forward calls for the binning buffer, whose size depends
 * on the instance count R that is only known mid-forward (the reference does the same through
 * std::function<char*(size_t)>, SUB/utility.h:7-13).  Must return a device pointer to >= nbytes. */
typedef void* (*r2x_alloc_fn)(size_t nbytes, void* user);

const char* r2x_last_error(void);
int r2x_version(void);

/* ---- buffer sizes -------------------------------------------------------------------------- */
size_t r2x_raster_geom_bytes(int P);
size_t r2x_raster_image_bytes(int P, int W, int H);
size_t r2x_voxel_geom_bytes(int P);
size_t r2x_voxel_image_bytes(int P, int nx, int ny, int nz);
size_t r2x_binning_bytes(long long R);             /* shared by rasterizer and voxelizer */
size_t r2x_raster_bwd_scratch_bytes(long long R);  /* per-instance moment buffer of the backward pass */
size_t r2x_voxel_bwd_scratch_bytes(long long R);

/* ---- rasterizer (X-ray projection) --------------------------------------------------------- */
/* Synchronous: one host<->device round trip to learn R (as the reference), binning buffer obtained
 * from `binning_alloc(r2x_binning_bytes(R), alloc_user)`.  *num_rendered (host) receives R. */
int r2x_raster_forward(void* stream, int P, int W, int H, const float* means3D, const float* opacities,
                       const float* scales, float scale_modifier, const float* rotations,
                       const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                       const float* campos, float tan_fovx, float tan_fovy, int prefiltered, int mode,
                       float* out_color, int* radii, void* geom_buf, void* image_buf,
                       r2x_alloc_fn binning_alloc, void* alloc_user, int debug, int* num_rendered);

/* Asynchronous: no host synchronisation.  `binning_buf` must hold r2x_binning_bytes(capacity); if the
 * scene needs more than `capacity` instances the extra ones are dropped and the overflow is reported
 * through `status_dev` (device uint32[2]: {R, overflow flag}), which the caller inspects after it
 * synchronises for its own reasons. */
int r2x_raster_forward_async(void* stream, int P, int W, int H, const float* means3D, const float* opacities,
                             const float* scales, float scale_modifier, const float* rotations,
                             const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                             const float* campos, float tan_fovx, float tan_fovy, int prefiltered, int mode,
                             float* out_color, int* radii, void* geom_buf, void* image_buf, void* binning_buf,
                             long long capacity, uint32_t* status_dev);

/* `R` is the instance count the binning buffer was carved for (num_rendered of the synchronous call,
 * `capacity` of the asynchronous one).  `scratch` holds r2x_raster_bwd_scratch_bytes(R).  All eight
 * gradient arrays are fully written (no pre-zeroing needed): dL_dmean2D[P,3], dL_dopacity[P],
 * dL_dmu[P] (may be NULL), dL_dmean3D[P,3], dL_dcov3D[P,6], dL_dscale[P,3], dL_drot[P,4]. */
int r2x_raster_backward(void* stream, int P, long long R, int W, int H, const float* means3D,
                        const float* scales, float scale_modifier, const float* rotations,
                        const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                        const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                        const void* geom_buf, const void* binning_buf, const void* image_buf, void* scratch,
                        const float* dL_dpix, float* dL_dmean2D, float* dL_dopacity, float* dL_dmu,
                        float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale, float* dL_drot, int mode,
                        int debug);

/* ---- batched views: N views of one cloud in one call ---------------------------------------------
 * All views share W, H, tan_fovx / tan_fovy, mode and scale_modifier; view v has its own
 * viewmatrices[16 v .. 16 v + 15] / projmatrices[16 v ..] (column-major as the single-view calls).
 * out_color[N,H,W]; radii[N,P].  Image v and radii[v] are bit for bit what r2x_raster_forward_async
 * computes for view v alone.  The views are the bands of one stacked tile grid (view v owns tile rows
 * [v ceil(H/16), (v+1) ceil(H/16))), binned and rendered together; N * ceil(H/16) must be <= 65535.
 * The instance count R is the sum over the views; capacity / status_dev as r2x_raster_forward_async.
 * Scales and rotations are required (no cov3D_precomp). */
size_t r2x_raster_views_geom_bytes(int P, int N);
size_t r2x_raster_views_image_bytes(int P, int N, int W, int H);
int r2x_raster_forward_views_async(void* stream, int P, int N, int W, int H, const float* means3D,
                                   const float* opacities, const float* scales, float scale_modifier,
                                   const float* rotations, const float* viewmatrices, const float* projmatrices,
                                   float tan_fovx, float tan_fovy, int mode, float* out_color, int* radii,
                                   void* geom_buf, void* image_buf, void* binning_buf, long long capacity,
                                   uint32_t* status_dev);
/* dL_dpix[N,H,W].  Per-Gaussian gradients are summed over the views in view order in float32
 * (acc = g[0]; acc = acc + g[v]), where g[v] is what r2x_raster_backward returns for view v alone:
 * dL_dopacity[P], dL_dmean3D[P,3], dL_dcov3D[P,6], dL_dscale[P,3], dL_drot[P,4].  dL_dmean2D[N,P,3] is
 * kept per view (densification statistics).  R and scratch as r2x_raster_backward. */
int r2x_raster_backward_views(void* stream, int P, int N, long long R, int W, int H, const float* means3D,
                              const float* scales, float scale_modifier, const float* rotations,
                              const float* viewmatrices, const float* projmatrices, float tan_fovx, float tan_fovy,
                              const int* radii, const void* geom_buf, const void* binning_buf, const void* image_buf,
                              void* scratch, const float* dL_dpix, float* dL_dmean2D, float* dL_dopacity,
                              float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale, float* dL_drot, int mode,
                              int debug);

/* Stage entry points for measurement (bench.py roofline, ncu): re-run ONLY the per-tile accumulation
 * kernel (the reference's renderCUDA, RAS/forward.cu:294-395 / VOX/forward.cu:183-315) on the state a
 * previous forward left in the three buffers.  `R` = the count the binning buffer was carved for. */
int r2x_raster_render_only(void* stream, int P, int W, int H, long long R, const void* geom_buf,
                           const void* binning_buf, const void* image_buf, float* out_color);
int r2x_voxel_render_only(void* stream, int P, int nx, int ny, int nz, long long R, const void* geom_buf,
                          const void* binning_buf, const void* image_buf, float* out_volume);

int r2x_mark_visible(void* stream, int P, const float* means3D, const float* viewmatrix,
                     const float* projmatrix, unsigned char* present);

/* Stage outputs in the reference's layouts (any pointer may be NULL): means2D[P,2], depths[P],
 * conic_opacity[P,4], mus[P], tiles_touched[P], point_offsets[P], keys[R] = (tile<<32)|depth_bits for
 * each entry of point_list[R] (our sorted order: tile-major, Gaussian index ascending), ranges[T,2]. */
int r2x_raster_export(void* stream, int P, int W, int H, long long R, const void* geom_buf,
                      const void* binning_buf, const void* image_buf, float* means2D, float* depths,
                      float* conic_opacity, float* mus, uint32_t* tiles_touched, uint32_t* point_offsets,
                      uint64_t* keys, uint32_t* point_list, uint32_t* ranges);

/* ---- voxelizer (density volume) ------------------------------------------------------------ */
int r2x_voxel_forward(void* stream, int P, int nx, int ny, int nz, float sx, float sy, float sz, float cx,
                      float cy, float cz, const float* means3D, const float* opacities, const float* scales,
                      float scale_modifier, const float* rotations, const float* cov3D_precomp,
                      int prefiltered, float* out_volume, int* radii_x, int* radii_y, int* radii_z,
                      void* geom_buf, void* image_buf, r2x_alloc_fn binning_alloc, void* alloc_user, int debug,
                      int* num_rendered);

int r2x_voxel_forward_async(void* stream, int P, int nx, int ny, int nz, float sx, float sy, float sz,
                            float cx, float cy, float cz, const float* means3D, const float* opacities,
                            const float* scales, float scale_modifier, const float* rotations,
                            const float* cov3D_precomp, int prefiltered, float* out_volume, int* radii_x,
                            int* radii_y, int* radii_z, void* geom_buf, void* image_buf, void* binning_buf,
                            long long capacity, uint32_t* status_dev);

/* Gradients fully written: dL_dopacity[P], dL_dmean3D[P,3], dL_dcov3D[P,6], dL_dscale[P,3], dL_drot[P,4]. */
int r2x_voxel_backward(void* stream, int P, long long R, int nx, int ny, int nz, float sx, float sy, float sz,
                       float cx, float cy, float cz, const float* means3D, const float* scales,
                       float scale_modifier, const float* rotations, const float* cov3D_precomp,
                       const int* radii_x, const int* radii_y, const int* radii_z, const void* geom_buf,
                       const void* binning_buf, const void* image_buf, void* scratch, const float* dL_dvol,
                       float* dL_dopacity, float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale,
                       float* dL_drot, int debug);

/* means3D_norm[P,3], depths[P], conic_opacity[P,7] (a,b,c,d,e,f,rho), others as r2x_raster_export. */
int r2x_voxel_export(void* stream, int P, int nx, int ny, int nz, long long R, const void* geom_buf,
                     const void* binning_buf, const void* image_buf, float* means3D_norm, float* depths,
                     float* conic_opacity, uint32_t* tiles_touched, uint32_t* point_offsets, uint64_t* keys,
                     uint32_t* point_list, uint32_t* ranges);

/* ---- point-cloud initialisation helper ------------------------------------------------------ */
/* Replaces `simple_knn._C.distCUDA2` (imported at r2_gaussian/gaussian/gaussian_model.py:21, called at
 * :144-150; upstream gitlab.inria.fr/bkerbl/simple-knn is an un-vendored submodule of the reference):
 * mean_dist2[i] = mean of the squared distances from points[i] to its 3 nearest OTHER points (exact;
 * FLT_MAX placeholders -> inf when fewer than 3 other points exist).  points[P,3] and mean_dist2[P] are
 * device pointers; scratch needs r2x_knn_scratch_bytes(P) bytes.  Asynchronous on `stream`. */
size_t r2x_knn_scratch_bytes(int P);
int r2x_knn3_mean_dist2(void* stream, int P, const float* points, float* mean_dist2, void* scratch,
                        size_t scratch_bytes);

/* ---- training-step helpers around the hot path (SURVEY 8(f) rank 2) ---------------------------- */
/* loss = w_l1 * mean|image - target| + w_dssim * (1 - mean SSIM(image, target)) for one single-channel H x W
 * image: the reference's `l1_loss` + `ssim` (r2_gaussian/utils/loss_utils.py:37-104: 11-tap Gaussian window,
 * sigma 1.5, zero padding, C1 = 0.01^2, C2 = 0.03^2) as combined in train.py:118-127.
 * loss_out[3] (device) = {mean|x-y|, mean SSIM, loss}; grad_out[H*W] (device, may be NULL) = d loss / d image.
 * Deterministic.  scratch: r2x_image_loss_scratch_bytes(H, W).  H <= 1048560 (65535 rows of 16-pixel tiles): a taller
 * image is refused before any launch. */
size_t r2x_image_loss_scratch_bytes(int H, int W);
int r2x_image_loss(void* stream, int H, int W, const float* image, const float* target, float w_l1,
                   float w_dssim, float* loss_out, float* grad_out, void* scratch, size_t scratch_bytes);
/* The same for N images (1 <= N <= 65535) in the same three launches: images / targets / grad_out [N,H,W],
 * loss_out[N,3]; row v is bit for bit r2x_image_loss of image v.  The same H limit.  scratch:
 * r2x_image_loss_views_scratch_bytes. */
size_t r2x_image_loss_views_scratch_bytes(int N, int H, int W);
int r2x_image_loss_views(void* stream, int N, int H, int W, const float* images, const float* targets, float w_l1,
                         float w_dssim, float* loss_out, float* grad_out, void* scratch, size_t scratch_bytes);

/* 3-D total variation of vol[nx][ny][nz] (`tv_3d_loss`, loss_utils.py:19-34): sum of absolute forward
 * differences along the three axes, divided by their number when reduction_mean != 0 (a 1x1x1 volume has none: its
 * mean is NaN, 0 / 0, and its gradient 0, as autograd gives the reference's).  loss_out[1] (device),
 * grad_out[nx*ny*nz] (device, may be NULL).  scratch: r2x_tv3d_scratch_bytes(nx, ny, nz). */
size_t r2x_tv3d_scratch_bytes(int nx, int ny, int nz);
int r2x_tv3d_loss(void* stream, int nx, int ny, int nz, const float* vol, int reduction_mean, float* loss_out,
                  float* grad_out, void* scratch, size_t scratch_bytes);

/* One Adam step over several parameter tensors in a single launch (torch.optim.Adam as configured at
 * r2_gaussian/gaussian/gaussian_model.py:216: amsgrad off, no weight decay; the four groups xyz / density /
 * scaling / rotation each carry their own learning rate).  `step` counts from 1 (bias correction). */
#define R2X_ADAM_MAX_GROUPS 8
typedef struct r2x_adam_group {
    float* param;        /* [numel] updated in place          */
    const float* grad;   /* [numel]                           */
    float* exp_avg;      /* [numel] first moment, in place    */
    float* exp_avg_sq;   /* [numel] second moment, in place   */
    long long numel;
    float lr;
} r2x_adam_group;
int r2x_adam_step(void* stream, int ngroups, const r2x_adam_group* groups, double beta1, double beta2, double eps,
                  long long step);
/* The same step with the gradient of group i taken as groups[i].grad + grads2[i] (grads2 or an entry may be NULL): what
 * autograd's accumulation of the render() and query() backward passes amounts to (train.py:141), without the
 * accumulation kernels.  guard0 / guard1 (either may be NULL) are the {num_rendered, overflow} status words of the
 * asynchronous forwards this step's gradients came from: if any reports an overflow the launch changes NOTHING, so an
 * iteration whose speculative forward ran out of instance capacity can simply be repeated. */
int r2x_adam_step_sum(void* stream, int ngroups, const r2x_adam_group* groups, const float* const* grads2, double beta1,
                      double beta2, double eps, long long step, const uint32_t* guard0, const uint32_t* guard1);
/* Densification statistics of one iteration in one launch (train.py:150-156, gaussian_model.py:552-556): for the visible
 * Gaussians (radii > 0)  max_radii2D = max(max_radii2D, radii),  xyz_gradient_accum += |dL_dmean2D.xy|,  denom += 1.
 * dL_dmean2D is [P,3]; the other arrays [P] float32.  Guards as above. */
int r2x_densify_stats(void* stream, int P, const int* radii, const float* dL_dmean2D, float* max_radii2D,
                      float* xyz_gradient_accum, float* denom, const uint32_t* guard0, const uint32_t* guard1);
/* The statistics of N >= 1 views in one launch: radii[N,P], dL_dmean2D[N,P,3]; bit for bit N r2x_densify_stats calls
 * in view order, with the same guards. */
int r2x_densify_stats_views(void* stream, int N, int P, const int* radii, const float* dL_dmean2D, float* max_radii2D,
                            float* xyz_gradient_accum, float* denom, const uint32_t* guard0, const uint32_t* guard1);

/* ---- folded parameter activations (SURVEY 8(f) rank 2) ------------------------------------------ */
/* The reference applies softplus (density), a bounded sigmoid or exp (scale) and normalize (rotation) as separate torch
 * kernels before every render() / query() and differentiates through them with autograd
 * (r2_gaussian/gaussian/gaussian_model.py:37-64, :112-126).  The *_raw entry points take the RAW parameters, apply the
 * activations inside the preprocess kernels and return the gradients with respect to the raw parameters (the other
 * arguments and buffers are those of the plain calls; cov3D_precomp does not apply).
 *   scale_mode 0: scale = exp(raw);  1: scale = scale_lo + (scale_hi - scale_lo) * sigmoid(raw). */
typedef struct r2x_activation {
    int scale_mode;
    float scale_lo, scale_hi;
} r2x_activation;
int r2x_raster_forward_async_raw(void* stream, int P, int W, int H, const float* means3D, const float* raw_density,
                                 const float* raw_scales, float scale_modifier, const float* raw_rotations,
                                 const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                                 float tan_fovy, int mode, float* out_color, int* radii, void* geom_buf, void* image_buf,
                                 void* binning_buf, long long capacity, uint32_t* status_dev, const r2x_activation* act);
int r2x_raster_backward_raw(void* stream, int P, long long R, int W, int H, const float* means3D, const float* raw_scales,
                            float scale_modifier, const float* raw_rotations, const float* viewmatrix,
                            const float* projmatrix, const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                            const void* geom_buf, const void* binning_buf, const void* image_buf, void* scratch,
                            const float* dL_dpix, float* dL_dmean2D, float* dL_draw_density, float* dL_dmean3D,
                            float* dL_dcov3D, float* dL_draw_scale, float* dL_draw_rot, int mode, const r2x_activation* act);
/* Batched views on raw parameters: the arguments and buffers of r2x_raster_forward_views_async /
 * r2x_raster_backward_views (no debug flag).  image[v] and radii[v] are bit for bit r2x_raster_forward_async_raw of view
 * v; each raw gradient is the view-order float32 sum (acc = g[0]; acc = acc + g[v]) of r2x_raster_backward_raw's per
 * view, and dL_dmean2D[N,P,3] is kept per view. */
int r2x_raster_forward_views_async_raw(void* stream, int P, int N, int W, int H, const float* means3D,
                                       const float* raw_density, const float* raw_scales, float scale_modifier,
                                       const float* raw_rotations, const float* viewmatrices, const float* projmatrices,
                                       float tan_fovx, float tan_fovy, int mode, float* out_color, int* radii,
                                       void* geom_buf, void* image_buf, void* binning_buf, long long capacity,
                                       uint32_t* status_dev, const r2x_activation* act);
int r2x_raster_backward_views_raw(void* stream, int P, int N, long long R, int W, int H, const float* means3D,
                                  const float* raw_scales, float scale_modifier, const float* raw_rotations,
                                  const float* viewmatrices, const float* projmatrices, float tan_fovx, float tan_fovy,
                                  const int* radii, const void* geom_buf, const void* binning_buf, const void* image_buf,
                                  void* scratch, const float* dL_dpix, float* dL_dmean2D, float* dL_draw_density,
                                  float* dL_dmean3D, float* dL_dcov3D, float* dL_draw_scale, float* dL_draw_rot, int mode,
                                  const r2x_activation* act);

/* ---- view- and projection-matrix gradients of the rasterizer backward (per-view pose refinement) -------------- */
/* r2x_raster_backward (act == NULL) or r2x_raster_backward_raw (act != NULL: raw scales / rotations, dL_dopacity is the
 * raw density gradient, cov3D_precomp must be NULL) with the same per-Gaussian outputs, bit for bit, that also writes
 * dL_dviewmatrix[16] / dL_dprojmatrix[16] (device): the gradient with respect to the 16 floats exactly as passed
 * (column-major flat, as the reference stores them).  Every discrete decision of the forward is held fixed (cull,
 * radius, tile rectangles, alpha cut, the clamp of the view-space point, the 1e-7 regularisations), the convention of
 * the per-Gaussian gradients.  Entries the rasterizer never reads get 0: viewmatrix[3, 7, 11, 15] and
 * projmatrix[2, 6, 10, 14].  One row of partial sums per 256 Gaussians goes to `pose_scratch`
 * (>= r2x_raster_backward_pose_scratch_bytes(P) bytes), summed in a fixed order in float64: no atomics, bitwise
 * reproducible.  Arguments are checked before any CUDA work. */
size_t r2x_raster_backward_pose_scratch_bytes(int P);
int r2x_raster_backward_pose(void* stream, int P, long long R, int W, int H, const float* means3D, const float* scales,
                             float scale_modifier, const float* rotations, const float* cov3D_precomp,
                             const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                             float tan_fovy, const int* radii, const void* geom_buf, const void* binning_buf,
                             const void* image_buf, void* scratch, const float* dL_dpix, float* dL_dmean2D,
                             float* dL_dopacity, float* dL_dmu, float* dL_dmean3D, float* dL_dcov3D, float* dL_dscale,
                             float* dL_drot, int mode, int debug, const r2x_activation* act, float* dL_dviewmatrix,
                             float* dL_dprojmatrix, void* pose_scratch, size_t pose_scratch_bytes);

/* ---- per-view pose corrections on the device (pose.PoseCorrection, NativeTrainStep(pose=...)) ------------------ */
/* omega / nu [n_views, 3] (device): per-view twists xi = (omega, nu), a LEFT perturbation in the camera frame,
 * T' = exp(xi) T, with world_view_transform = T^T and full_proj_transform = T^T projection_matrix (all 16 floats,
 * device, row-major as the torch tensors store them).  r2x_pose_apply writes the corrected matrices of view
 * `view_index`:  out_view = view + view D^T,  out_full = full + (view D^T) proj,  D = exp(xi) - I formed in float64
 * with the coefficients and the series switch (theta^2 < 1e-2) of pose._coefficients; each entry is the float64 sum,
 * rounded to float32 once, and a zero increment counts as -0.0, so a zero twist returns both matrices bit for bit.
 * The camera centre is not an output: the raster kernels never read `campos`, callers pass the camera's own.
 * r2x_pose_grad writes dL_domega / dL_dnu [n_views, 3] in full: row `view_index` is the chain rule of dL_dview /
 * dL_dproj (as r2x_raster_backward_pose writes them) through that same float64 expression (exact derivative, forward
 * mode), rounded once; every other row, and row `anchor` (-1: none) always, is 0.  The base full_proj_transform does
 * not enter the derivative.  Arguments are checked before any CUDA work; one small launch each, asynchronous. */
int r2x_pose_apply(void* stream, const float* omega, const float* nu, int n_views, int view_index,
                   const float* world_view_transform, const float* full_proj_transform, const float* projection_matrix,
                   float* out_world_view_transform, float* out_full_proj_transform);
int r2x_pose_grad(void* stream, const float* omega, const float* nu, int n_views, int view_index, int anchor,
                  const float* world_view_transform, const float* projection_matrix, const float* dL_dview,
                  const float* dL_dproj, float* dL_domega, float* dL_dnu);

/* ---- horizontal detector offset on the device (detector.DetectorOffset, NativeTrainStep(detector=...)) ---------- */
/* offset[1] (device): s, the shift of the detector along u in pixels; a view whose content lies s columns towards
 * larger column index than the nominal geometry predicts has s > 0.  The shift moves every projected 2-D mean by s
 * pixels and leaves rays, conics and mu alone, so only the full projection changes.
 * r2x_detector_offset_apply writes, for each of n_views full projections (16 floats each, row-major as the torch
 * tensors store them, i.e. the rasterizer's column-major matrix), the matrix whose x row (entries 0, 4, 8, 12) gains
 * (2 s / W) times its w row (entries 3, 7, 11, 15); every other entry is copied.  Each entry is the float64 sum rounded
 * to float32 once, and a zero increment counts as -0.0, so s = 0 returns the input bit for bit.  The view matrix does
 * not change.  out_full_proj may not alias full_proj.
 * r2x_detector_offset_grad writes dL_doffset[0] = (2 / W) sum over the n_views x P rows of dL_dmean2D[n_views, P, 3]
 * of the x component (dL/dndc as every raster backward writes it), i.e. the sum of dL/dpix_x with cull, radii and tile
 * rectangles held fixed.  Two launches: float64 partial sums of contiguous chunks into `scratch`
 * (>= r2x_detector_offset_grad_scratch_bytes(P, n_views) bytes), then their sum in a fixed order: no atomics, bitwise
 * reproducible; the result is written, not accumulated.  Arguments are checked before any CUDA work; asynchronous. */
int r2x_detector_offset_apply(void* stream, const float* offset, int W, int n_views, const float* full_proj,
                              float* out_full_proj);
size_t r2x_detector_offset_grad_scratch_bytes(int P, int n_views);
int r2x_detector_offset_grad(void* stream, int P, int n_views, int W, const float* dL_dmean2D, float* dL_doffset,
                             void* scratch, size_t scratch_bytes);

int r2x_voxel_forward_async_raw(void* stream, int P, int nx, int ny, int nz, float sx, float sy, float sz, float cx,
                                float cy, float cz, const float* means3D, const float* raw_density,
                                const float* raw_scales, float scale_modifier, const float* raw_rotations,
                                float* out_volume, int* radii_x, int* radii_y, int* radii_z, void* geom_buf,
                                void* image_buf, void* binning_buf, long long capacity, uint32_t* status_dev,
                                const r2x_activation* act);
int r2x_voxel_backward_raw(void* stream, int P, long long R, int nx, int ny, int nz, float sx, float sy, float sz, float cx,
                           float cy, float cz, const float* means3D, const float* raw_scales, float scale_modifier,
                           const float* raw_rotations, const int* radii_x, const int* radii_y, const int* radii_z,
                           const void* geom_buf, const void* binning_buf, const void* image_buf, void* scratch,
                           const float* dL_dvol, float* dL_draw_density, float* dL_dmean3D, float* dL_dcov3D,
                           float* dL_draw_scale, float* dL_draw_rot, const r2x_activation* act);

/* ---- device-side row compaction for densify / clone / split / prune ------------------------------ */
/* Replaces the boolean-mask indexing + torch.cat sequence of the reference's optimizer surgery
 * (r2_gaussian/gaussian/gaussian_model.py:335-403, :503-550).  r2x_mask_select turns a byte mask into the stable
 * list of selected row indices and their count, both on the device (no host round trip).  r2x_gather_rows gathers up
 * to R2X_GATHER_MAX_TENSORS row-major float tensors through one such list in ONE launch: source row s of tensor t is
 * src0[s] for s < n0, else src1[s - n0] (src1 == NULL: zeros -- fresh Adam moments); `select` == NULL: identity. */
#define R2X_GATHER_MAX_TENSORS 16
typedef struct r2x_gather_desc {
    const float* src0;   /* [n0, width]                          */
    const float* src1;   /* [*, width] rows appended after src0, or NULL = zeros */
    float* dst;          /* [nsel, width]                        */
    long long n0;
    int width;
} r2x_gather_desc;
size_t r2x_mask_select_scratch_bytes(int n);
int r2x_mask_select(void* stream, int n, const unsigned char* mask, int* idx_out, uint32_t* count_dev, void* scratch,
                    size_t scratch_bytes);
int r2x_gather_rows(void* stream, int ntensors, const r2x_gather_desc* descs, const int* select, long long nsel);

/* ---- FDK reconstruction (initial volume for the point cloud) ------------------------------------ */
/* Replaces TIGRE's `algs.fdk` (r2_gaussian/utils/ct_utils.py::recon_volume, called by initialize_pcd.py).  Lengths in
 * the scene-scaled units of the dataset readers.  projs[N,H,W] (rows = v, columns = u); viewmatrices / projmatrices
 * [N,16] are the rasterizer's per-view matrices, tan_fovx / tan_fovy the values render() passes (parallel beam: 1).
 *   1. cone beam: cosine weight P * DSD / sqrt(DSD^2 + u^2 + v^2) at the pixel centres;
 *   2. ramp filter along each row, linear convolution over the whole row (0 beyond it), at the isocentre pitch D (cone:
 *      dDetector_u * DSO / DSD = 2 tan_fovx DSO / W; parallel: 2 / W, the rasterizer's detector spans ndc [-1,1]):
 *      Q_j = (1 / D) sum_k h[k] P'_{j-k} with the taps h[k] = (1 / 2 pi^2) int_0^pi w Wn(w) cos(w k) dw of the filter
 *      field of `weighting` (TIGRE's `geo.filter` windows at frequency scale 1; tests/fdk_window_oracle.py):
 *        R2X_FDK_RAM_LAK      Wn = 1, the band-limited Ram-Lak filter: h[0] = 1/4, h[k odd] = -1 / (pi^2 k^2), 0 at
 *                             even k != 0 (oracle/fdk_oracle.py);
 *        R2X_FDK_SHEPP_LOGAN  Wn = sin(w/2) / (w/2): h[k] = -2 / (pi^2 (4k^2 - 1));
 *        R2X_FDK_COSINE       Wn = cos(w/2): h[k] = -(-1)^k / (pi (4k^2 - 1)) - (1/(2k+1)^2 + 1/(2k-1)^2) / pi^2;
 *        R2X_FDK_HAMMING      Wn = 0.54 + 0.46 cos w: h[k] = 0.54 h_RL[k] + 0.23 (h_RL[k-1] + h_RL[k+1]);
 *        R2X_FDK_HANN         Wn = (1 + cos w) / 2: h[k] = 0.5 h_RL[k] + 0.25 (h_RL[k-1] + h_RL[k+1]);
 *      (h_RL = the Ram-Lak taps).  The filter changes the taps only: steps 1 and 3, the pitch, the redundancy weights
 *      and the scale are the same for every filter;
 *   3. voxel-driven backprojection: voxel centres center - s/2 + (i + 1/2) s/n, projected through projmatrix and the
 *      rasterizer's ndc -> pixel mapping, bilinear sample (0 outside the detector), weight U^2 with U = DSO / z_view
 *      (cone; 0 for z_view <= 0) or 1 (parallel); out_volume[nx,ny,nz] = (pi / N) * sum over views in index order.
 * Detector offset: shift_u, shift_v are TIGRE's `geo.offDetector` in pixels, t_u = offDetector[0] / dDetector_u and
 * t_v = offDetector[1] / dDetector_v of the scanner file (r2_gaussian/utils/ct_utils.py::get_geometry_tigre;
 * scene.detector_shift states the convention); 0, 0 for a centred detector.  Image pixel (row i, column j) holds the
 * ray of the centred detector's fractional pixel (i - t_v, j + t_u), so step 1 takes its cosine weight at ndc
 * ((2j+1)/W - 1 + 2 t_u/W, (2i+1)/H - 1 - 2 t_v/H); step 3 goes through the caller's projmatrices, which must be the
 * offset ones (scene.make_view(..., use_offDetector=True)).  A zero offset gives the centred result bit for bit.
 * weighting = one redundancy weight below OR-ed with one filter of step 2 (R2X_FDK_RAM_LAK is 0, so a bare weight is
 * Ram-Lak); any other bit or value is refused.  The redundancy weight step 1 also applies (the plain FDK's is
 * oracle/fdk_oracle.py):
 *   R2X_FDK_PLAIN     none.  It reconstructs a cone-beam short scan as if it were a full one (as TIGRE's default fdk).
 *   R2X_FDK_PARKER    a short scan (Parker 1982, in Silver 2000's overscan form; tests/fdk_short_scan_oracle.py): an arc
 *                     B = arc with pi + 2 gamma_max <= B < 2 pi (gamma_max = atan(tan_fovx) for cone beam, 0 for
 *                     parallel beam) measures some rays once and some twice.  P' = w(beta'_v, gamma_j) * dbeta_v * P,
 *                     with gamma_j = -atan(ndc_x(j) tan_fovx) (cone; the detector's u axis runs along the rotation) or 0
 *                     (parallel), delta = (B - pi) / 2 and the Parker weight w = sin^2(pi/4 beta' / (delta - gamma))
 *                     for beta' < 2 (delta - gamma), 1 up to pi - 2 gamma, sin^2(pi/4 (B - beta') / (delta + gamma)) up
 *                     to B, 0 beyond; step 3 sums with scale 1 instead of pi / N.  view_weights[N,2] (device) holds each
 *                     view's (beta'_v, dbeta_v): its arc position from the start of the scan and its angular interval,
 *                     as fdk.short_scan_views computes them in float64 (they are not read on the host, so their
 *                     finiteness is the caller's).  Refuses N < 2, a NULL view_weights, B outside [pi + 2 gamma_max,
 *                     2 pi) and shift_u != 0 (Parker weights assume each ray's conjugate is on the detector).
 *   R2X_FDK_HALF_FAN  a full circle with the axis off the detector's centre (Wang 2002; tests/offset_detector_oracle.py;
 *                     the caller checks the circle): P' = w(a_j) * P for the fan coordinate a_j = ndc_x(j) * (cone:
 *                     tan_fovx; parallel: 1), with delta = (1 - 2|t_u|/W) * (tan_fovx or 1), sigma = sign(t_u) and
 *                     w = 2 sin^2(pi/4 (1 + sigma a / delta)) for |a| <= delta, 2 for sigma a > delta; the scale stays
 *                     pi / N.  Refuses unless 0 < |shift_u| < W/2.
 * view_weights and arc are read for R2X_FDK_PARKER only.  Deterministic (no atomics).  `scratch` holds
 * r2x_fdk_scratch_bytes(N, H, W) (the filtered views).  Asynchronous on `stream`.  Limits: W <= 16384, N * H < 2^31,
 * nx <= 262140, nz <= 524280. */
#define R2X_FDK_PLAIN 0
#define R2X_FDK_PARKER 1
#define R2X_FDK_HALF_FAN 2
#define R2X_FDK_RAM_LAK 0x000
#define R2X_FDK_SHEPP_LOGAN 0x100
#define R2X_FDK_COSINE 0x200
#define R2X_FDK_HAMMING 0x300
#define R2X_FDK_HANN 0x400
size_t r2x_fdk_scratch_bytes(int n_views, int H, int W);
int r2x_fdk(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
            const float* projmatrices, float tan_fovx, float tan_fovy, int mode, float shift_u, float shift_v,
            int weighting, const float* view_weights, float arc, float dso, int nx, int ny, int nz, float sx, float sy,
            float sz, float cx, float cy, float cz, float* out_volume, void* scratch, size_t scratch_bytes);
/* The two stages of r2x_fdk on their own (measurement; centred, R2X_FDK_PLAIN, Ram-Lak): filtered[N,H,W] = steps 1-2;
 * out_volume = step 3 of it. */
int r2x_fdk_filter(void* stream, int n_views, int H, int W, const float* projs, float tan_fovx, float tan_fovy,
                   int mode, float dso, float* filtered);
int r2x_fdk_backproject(void* stream, int n_views, int H, int W, const float* filtered, const float* viewmatrices,
                        const float* projmatrices, int mode, float dso, int nx, int ny, int nz, float sx, float sy,
                        float sz, float cx, float cy, float cz, float* out_volume);

/* ---- forward projection of a voxel volume (synthetic projection data) --------------------------- */
/* Replaces TIGRE's `Ax` (data_generator/synthetic_dataset/generate_data.py).  Lengths in the scene-scaled units of the
 * dataset readers.  volume[nx,ny,nz] (index x*ny*nz + y*nz + z) with size (sx,sy,sz) centred at (cx,cy,cz);
 * viewmatrices[N,16] are the rasterizer's per-view matrices, tan_fovx / tan_fovy the values render() passes (parallel
 * beam: 1); out_projs[N,H,W] (rows = v, columns = u).  For every detector pixel (row i, column j):
 *   ray    ndc = ((2j+1)/W - 1 + 2 shift_u/W, (2i+1)/H - 1 - 2 shift_v/H) in float64, where (shift_u, shift_v) is the
 *          detector offset in pixels as for r2x_fdk (0, 0 when centred; zero shifts give the centred rays bit for bit;
 *          finite); cone beam: from the camera centre along camera-frame
 *          (ndc_x tan_fovx, ndc_y tan_fovy, 1); parallel beam: from camera-frame (ndc_x, ndc_y, 0) along (0, 0, 1); both
 *          taken to world space by the rigid inverse of the viewmatrix; unit direction d, so t is a length.
 *   field  f = trilinear interpolation between the voxel centres c - s/2 + (i + 1/2) s/n, every lattice point outside
 *          [0,n) having value 0: continuous, nonzero only inside the box c +- (s/2 + s/(2n)).
 *   value  step * sum_k f(o + (t_c + k step) d) over the integers k whose sample lies inside that box (cone beam also
 *          t > 0), with t_c = (c - o).d the ray's closest approach to the volume centre, summed in k order in float32.
 *          A ray that misses the box gives exactly 0.  The callers pass step = accuracy * min(s/n).
 * The sample positions do not depend on where the ray enters or leaves the box, so samples that rounding moves across
 * its boundary sit where the field is ~0.  Deterministic (no atomics).  Asynchronous on `stream`.
 * Limits: H <= 2097120 (grid.y), W and N up to INT_MAX (views are launched 65535 at a time), N*H*W indexed in 64 bits. */
int r2x_volume_project(void* stream, int nx, int ny, int nz, const float* volume, float sx, float sy, float sz,
                       float cx, float cy, float cz, int n_views, int H, int W, const float* viewmatrices,
                       float tan_fovx, float tan_fovy, int mode, float shift_u, float shift_v, float step,
                       float* out_projs);

/* ---- matched backprojection: the transpose of r2x_volume_project (iterative reconstruction) ------------------- */
/* Replaces TIGRE's `Atb` inside `algs.cgls` / `algs.sart` / `algs.ossart` (r2_gaussian/utils/ct_utils.py).  Same
 * geometry arguments and units as r2x_volume_project, plus the per-view projmatrices (the rasterizer's, as for r2x_fdk)
 * for each voxel's detector footprint (with a detector offset the offset ones, scene.make_view(...,
 * use_offDetector=True), so that the footprint covers the offset rays).  projs[N,H,W] (rows = v, columns = u);
 * out_volume / out_weight [nx,ny,nz]:
 *   out_volume[x] = step * sum over views (index order) of sum over pixels of projs[v,i,j] * sum_{k in K} h_x(p_k)
 *   out_weight[x] = the same with projs = 1 (optional: NULL skips it)
 * where p_k = fmaf(k, s, g) is r2x_volume_project's own float32 index-space sample of pixel (i, j), K its own k range
 * (the box test, and t > 0 for cone beam), and h_x(p) the trilinear weight the projector gives lattice point x at p:
 * per axis 1 - f at floor(p) and f at floor(p) + 1, f = p - floor(p).  So out_volume = A^T projs over exactly the
 * (ray, sample, voxel) triples of r2x_volume_project; only the float32 rounding of the sums differs.  Both outputs are
 * written in full (no memset needed).  Deterministic (no atomics).  `scratch` holds
 * r2x_volume_backproject_scratch_bytes(N, H, W) (the projector's ray setup for up to 32 views at a time).
 * Asynchronous on `stream`.  Limits: nx <= 65535, ny <= 262140, fewer than 2^24 samples per half ray. */
size_t r2x_volume_backproject_scratch_bytes(int n_views, int H, int W);
int r2x_volume_backproject(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
                           const float* projmatrices, float tan_fovx, float tan_fovy, int mode, float shift_u,
                           float shift_v, int nx, int ny, int nz, float sx, float sy, float sz, float cx, float cy,
                           float cz, float step, float* out_volume, float* out_weight, void* scratch,
                           size_t scratch_bytes);

/* ---- isotropic total variation on a volume (FISTA-TV, r2_gaussian_b200/recon.py and tv.py) --------------------- */
/* Volumes are float32 [nx,ny,nz] (z fastest).  grad x = forward differences along x, y, z, 0 across the last index;
 *   TV(x) = sum over voxels of sqrt(dx^2 + dy^2 + dz^2)      (isotropic; not the anisotropic r2x_tv3d_loss)
 * r2x_tv_prox writes out = argmin over x in C of 1/2 |x - v|^2 + weight TV(x), C = {x >= 0} when nonneg, else all,
 * by `niter` iterations of Beck-Teboulle's fast gradient projection (FGP) on the dual field p[3,nx,ny,nz]: cold start
 * p = 0, step 1 / (12 weight), projection onto |p_voxel| <= 1, out = P_C(v - weight div p) (the recurrence is stated in
 * csrc/r2x_tv.cu).  niter + 1 launches; the three dual fields it rotates live in `scratch` (>=
 * r2x_tv_prox_scratch_bytes(nx, ny, nz) = 36 bytes per voxel).  weight 0 writes P_C(v) bit for bit (u < 0 ? 0 : u, or
 * v itself).  out may not alias v.
 * r2x_tv_value writes out[0] (device, float64) = TV(x) with each term in float64: float64 partial sums of contiguous
 * chunks into `scratch` (>= r2x_tv_value_scratch_bytes), then their sum in a fixed order.
 * Both: no atomics, bitwise reproducible; arguments are checked before any CUDA work; asynchronous on `stream`.
 * Limits: nx <= 262140, ny <= 524280. */
size_t r2x_tv_prox_scratch_bytes(int nx, int ny, int nz);
int r2x_tv_prox(void* stream, int nx, int ny, int nz, const float* v, float weight, int niter, int nonneg, float* out,
                void* scratch, size_t scratch_bytes);
size_t r2x_tv_value_scratch_bytes(int nx, int ny, int nz);
int r2x_tv_value(void* stream, int nx, int ny, int nz, const float* x, double* out, void* scratch,
                 size_t scratch_bytes);

/* ---- real-scan projection preparation (r2_gaussian_b200/generate_real_data.py) ---------------------------------- */
/* Replaces the reference's per-view numpy + cv2 chain (data_generator/real_dataset/generate_data.py:91-109).
 * img[n_views, H0, W0] (device, float64: the processed scan's `img` arrays) -> out[n_views, H, W] (device, float32):
 *   1. p = float32(img / proj_rescale * object_scale), both operations in float64, one rounding;
 *   2. p < 0 -> 0 (-0 and NaN are kept);
 *   3. the image moves up 5 rows, zero fill (row r takes row r + 5);
 *   4. subsample != 1: resize to int(H0 / subsample) x int(W0 / subsample) as cv2.resize's float32 INTER_LINEAR does
 *      on the x86-64 OpenCV builds (their IPP path; tests/real_data_oracle.py states it): per axis the source position
 *      (d + 0.5) (src / dst) - 0.5 in float64, float32 fraction t, fma(t, b - a, a) along the columns, then along
 *      the rows, the last source sample repeated at the far edge; then the longer axis is centre-cropped by
 *      int(diff / 2) on each side (a difference of 1 crops nothing).  subsample 1 neither resizes nor crops.
 * r2x_projection_prepare_shape writes (H, W) to out_hw[2] without touching the GPU.  Arguments are checked before any
 * CUDA work (n_views >= 1, H0, W0, subsample >= 1, a resized size >= 1, H * W < 2^31, proj_rescale finite and
 * non-zero, object_scale finite).  Deterministic (no atomics; each output depends only on its view, so any split of the
 * views into calls gives the same bits).  Asynchronous on `stream`.  n_views * H0 * W0 is indexed in 64 bits. */
int r2x_projection_prepare_shape(int H0, int W0, int subsample, int* out_hw);
int r2x_projection_prepare(void* stream, int n_views, int H0, int W0, int subsample, const double* img,
                           double proj_rescale, double object_scale, float* out);

/* ---- multi-GPU exchange step: one-shot sum over NVLink peer memory ------------------------------ */
/* The Gaussian-sharded projector (one process per GPU, every rank renders its index shard) needs ONE exchange per
 * projection: the sum of the per-rank partial detector images (BASELINE north_star; the reference itself is
 * single-GPU).  These entry points replace the NCCL all-reduce for that step: buffers are cudaMalloc'ed
 * (r2x_peer_alloc), shared between the processes of one node as CUDA IPC handles (64 bytes, r2x_ipc_export /
 * r2x_ipc_open), and r2x_peer_allreduce_sum signals, waits and adds the `world` partial buffers in rank order
 * (bitwise identical result on every rank).  bufs[p] / flags[p]: rank p's partial buffer (n floats) and flag
 * array (R2X_MAX_PEERS uint32, zero-initialised) as mapped in THIS process; `epoch` increases by one per call;
 * callers double-buffer the partial buffers by epoch parity.  status_dev[0] is set to 1 if a peer never arrived
 * within the time-out (~2 s; r2x_peer_allreduce_sum_t takes it in SM clock cycles) -- the sum is then invalid and
 * the caller must check the status word at its next synchronisation point (sharded.check_peer_exchange). */
#define R2X_MAX_PEERS 16
int r2x_peer_alloc(size_t bytes, void** dev_ptr);
int r2x_peer_free(void* dev_ptr);
int r2x_ipc_export(void* dev_ptr, unsigned char* handle64);
int r2x_ipc_open(const unsigned char* handle64, void** dev_ptr);
int r2x_ipc_close(void* dev_ptr);
int r2x_peer_allreduce_sum(void* stream, int world, int rank, const float* const* bufs, uint32_t* const* flags,
                           uint32_t epoch, float* out, long long n, uint32_t* status_dev);
int r2x_peer_allreduce_sum_t(void* stream, int world, int rank, const float* const* bufs, uint32_t* const* flags,
                             uint32_t epoch, float* out, long long n, uint32_t* status_dev, long long timeout_cycles);

#ifdef __cplusplus
}
#endif
#endif /* R2X_H_INCLUDED */
