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

/* ---- horizontal detector offset from the projections (detector.estimate_offset) ------------------------------------
 * The model.  A circular scan measures most rays twice.  Image column c of a view sees the detector coordinate
 * u = du (c - (W - 1) / 2 - sigma): sigma is the column shift of the rotation axis from the detector centre (the
 * caller's candidate, the DetectorOffset s minus the scanner file's t_u).  Column pitch du = sDetector_u / nDetector_u.
 *   parallel beam (mode 0): P(beta, u) = P(beta + pi, -u) in every row, so for a pair (i, j) with beta_j - beta_i = pi
 *     the sample m (0 <= m < W) of row r compares view i at column m + sigma with view j at column W - 1 - m + sigma,
 *     rows row_lo .. row_lo + n_rows - 1 (both columns carry the same fraction, so both see the same interpolation);
 *   cone beam (mode 1): in the mid-plane, P(beta, gamma) = P(beta + pi - 2 gamma, -gamma) with gamma = atan(u / DSD)
 *     and gamma > 0 towards larger column index, so a pair (i, j) with d = beta_j - beta_i in [0, 2 pi) shares the one
 *     ray at t = DSD tan((pi - d) / 2) / du pixels from the axis: view i at column (W - 1) / 2 + t + sigma against view
 *     j at column (W - 1) / 2 - t + sigma, both in image row (H - 1) / 2 + t_v (n_rows must be 1).
 * Every value is linear in the column and (cone beam) the row, formed in float64 from the float32 projections; a
 * sample counts when both of its columns lie in [0, W - 1] (and its row in [0, H - 1]).  For each of the K candidate
 * shifts sigma[k] (host-free: device float64) the entry point writes
 *   num[k] = sum (a - b)^2,   den[k] = sum (a^2 + b^2),   count[k] = the number of valid samples
 * over the pair table pair_views int32 [n_pairs, 2] (view i, view j; 0 <= i, j < N, the caller's promise) and
 * pair_dbeta float64 [n_pairs] (beta_j - beta_i; read in cone beam only).  projs is float32 [N, H, W].
 * Two launches: per candidate, a fixed grid of contiguous sample chunks summed in a fixed tree into `scratch`
 * (>= r2x_detector_offset_cost_scratch_bytes bytes), then the chunks of each candidate added in order: no atomics,
 * two calls give the same bits.  Limits: 1 <= K <= 65535, n_pairs x n_rows x (W or 1) samples < 2^62; anything else
 * is refused before any CUDA work.  Asynchronous. */
size_t r2x_detector_offset_cost_scratch_bytes(int mode, int W, int n_pairs, int n_rows, int K);
int r2x_detector_offset_cost(void* stream, int mode, int N, int H, int W, const float* projs, int n_pairs,
                             const int* pair_views, const double* pair_dbeta, double DSD, double du, double t_v,
                             int row_lo, int n_rows, int K, const double* sigma, double* num, double* den,
                             long long* count, void* scratch, size_t scratch_bytes);

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
/* r2x_fdk of a laterally truncated scan (the object wider than the detector's field of view): r2x_fdk's arguments and
 * scratch plus a pad of L = `pad` pixels, 0 <= L <= W, that extends each row past its edges before step 2 so that the
 * filter does not see a step there (Ohnesorge et al., Med. Phys. 27(1), 2000; float64 statement in
 * tests/fdk_pad_oracle.py).  Per detector row, after step 1 (cosine and any Parker weight), with r[0 .. W-1] the
 * weighted row:
 *   e[i] = r[i] for 0 <= i < W;  e[-k] = t_k r[k-1] and e[W-1+k] = t_k r[W-k] for k = 1 .. L, where
 *   t_k = (1 + cos(pi k / (L + 1))) / 2: a mirror about each edge, rolled off to zero;
 *   Q_j = (1 / D) sum_{i=-L}^{W-1+L} h[j-i] e[i] for 0 <= j < W, with the taps h of the filter field.
 * Only Q_0 .. Q_{W-1} are written and backprojected (step 3 unchanged).  L = 0 is r2x_fdk bit for bit.  Refuses, before
 * any CUDA work, pad < 0, pad > W, R2X_FDK_HALF_FAN (a shifted detector's truncation is deliberate and its weights
 * handle it) and a padded row whose stage exceeds 227 KB of shared memory ((3 W + 2 L + ceil((W + L) / 2)) floats for
 * Ram-Lak, (2 W + 3 L) for a window: any pad up to W = 9685), then everything r2x_fdk refuses. */
int r2x_fdk_pad(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
                const float* projmatrices, float tan_fovx, float tan_fovy, int mode, float shift_u, float shift_v,
                int weighting, const float* view_weights, float arc, float dso, int nx, int ny, int nz, float sx,
                float sy, float sz, float cx, float cy, float cz, float* out_volume, void* scratch, size_t scratch_bytes,
                int pad);
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

/* Per-view geometry (helical scans, calibrated benches; scene.view_scanner).  r2x_fdk_views, r2x_volume_project_views
 * and r2x_volume_backproject_views are r2x_fdk, r2x_volume_project and r2x_volume_backproject with the scalars
 * tan_fovx, tan_fovy, shift_u, shift_v and dso replaced by one row per view of the table view_geometry, device float64
 * [N, 5] (row-major):
 *   column 0  tan_fovx of view v   (tan of half its horizontal FoV, sDetector_u / 2 / DSD_v; parallel beam: 1)
 *   column 1  tan_fovy of view v   (sDetector_v / 2 / DSD_v; parallel beam: 1)
 *   column 2  shift_u of view v    (its offDetector_u in pixels, t_u of scene.detector_shift)
 *   column 3  shift_v of view v    (its offDetector_v in pixels)
 *   column 4  dso of view v        (its DSO: FDK's isocentre pitch and (DSO / z_view)^2 weight; unread by the projector
 *                                   pair, whose rays need only the view matrix and the FoV)
 * Every value is rounded to float32 where it is read, as the scalar entry points' float arguments are, so view v is
 * bit for bit the scalar call with its values, and a table whose rows all equal the scalars is bit for bit the scalar
 * entry point.  A view's DSO and its volume position offOrigin_v live in its view matrix: the camera of view v is the
 * nominal one at DSO_v translated by offOrigin - offOrigin_v, with the grid kept at (cx, cy, cz) (scene.make_view).
 * view_geometry_host is the same table in host memory: it is checked before any CUDA work (present, every value finite,
 * tan_fov > 0 (always for the projector pair, cone beam for FDK), dso > 0 in cone beam) and the device copy matching it
 * is the caller's promise.  r2x_fdk_views takes R2X_FDK_PLAIN with any filter field; Parker and half-fan weights assume
 * one fixed circle and are refused, as is a NULL table.  Otherwise each behaves, and is limited, as its scalar entry. */
int r2x_fdk_views(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
                  const float* projmatrices, int mode, int weighting, int nx, int ny, int nz, float sx, float sy,
                  float sz, float cx, float cy, float cz, const double* view_geometry,
                  const double* view_geometry_host, float* out_volume, void* scratch, size_t scratch_bytes);
/* Helical FDK (Tang et al. 2006, "A three-dimensional-weighted cone beam filtered backprojection (CB-FBP) algorithm for
 * image reconstruction in volumetric CT -- helical scanning", Phys. Med. Biol. 51:855), in native cone-beam geometry on
 * the flat detector; float64 statement in tests/fdk_helical_oracle.py.  Cone beam only.
 *   Helix.  One DSO, one DSD, a centred detector and one offOrigin x / y; the volume position's z is affine in each
 *     view's unwrapped angle beta, so in the grid frame (scene.camera_pose) the source of view v is at
 *     (DSO cos beta + c_x, DSO sin beta + c_y, z_s(beta)), z_s(beta) = z0 + pitch * beta (pitch signed, per radian;
 *     0 is a circle).  beta[N] (device) and beta_host[N] are the views' angles, strictly increasing; the caller sorts
 *     the views (and their projections and matrices) into that order.  The arc is [beta_lo, beta_hi) with
 *     beta_lo <= beta[0], beta[N-1] < beta_hi and beta_hi - beta_lo >= 2 pi; dbeta[N] (device) is each view's
 *     quadrature interval (fdk.helix_views: between the midpoints of its neighbours, beta_lo and beta_hi at the ends).
 *   Filter.  Steps 1-2 of r2x_fdk with R2X_FDK_PLAIN and the filter field of `weighting` (no other bits).
 *   Conjugates.  For voxel x and view beta: d = the in-plane vector from the source to x, L = |d|, gamma its fan angle
 *     from the central ray, signed so that the source at beta + pi + 2 gamma lies on the same in-plane line (R2X_FDK_PARKER's
 *     convention).  K(beta, x) = {(beta + 2 pi m, L)} u {(beta + pi + 2 gamma + 2 pi m, 2 DSO cos(gamma) - L)} over the
 *     integers m with beta_lo <= beta_k < beta_hi (a conjugate with 2 DSO cos(gamma) - L <= 0 does not exist; a view
 *     with L cos(gamma) <= 0 gets weight 0), each with its detector row nu_k = (Z - z_s(beta_k)) / (L_k cos(gamma)
 *     tan_fovy); nu_0 is minus the ndc row at which the view samples x.
 *   Weight.  W_Q(nu) = 1 for |nu| <= Q, cos^2(pi/2 (|nu| - Q) / (1 - Q)) for Q < |nu| < 1, 0 for |nu| >= 1 (the last
 *     rule first: Q = 1 gives 1 inside the detector, 0 on and beyond its edge); 0 <= Q <= 1.
 *     w(beta, x) = W_Q(nu_0) / sum_{k in K} W_Q(nu_k) (0 when W_Q(nu_0) = 0).
 *   Backprojection.  out_volume(x) = sum over views in index order of dbeta_v * w(beta_v, x) * U^2 * Qf_v(x), with Qf_v
 *     sampled and U = DSO / z_view as in step 3 of r2x_fdk.  With pitch 0, Q = 1 and a full circle, a voxel whose two
 *     conjugate rays both hit the detector gets w = 1/2 and dbeta = 2 pi / N: the plain FDK's pi / N.
 * Each CTA visits only the views whose source height lies within (DSO + the grid's largest in-plane radius about
 * (c_x, c_y)) * tan_fovy of its voxels (widened by 1e-3): the others have W_Q(nu_0) = 0 there, so the skip drops exact
 * zeros.  Refuses, before any CUDA work: parallel beam, NULL pointers, a non-finite helix, Q outside [0, 1], beta_host
 * not finite and strictly increasing, beta outside [beta_lo, beta_hi), an arc shorter than 2 pi (within 1e-6), any
 * weighting bit but the filter field, and what r2x_fdk refuses.  Deterministic (no atomics).  `scratch` holds
 * r2x_fdk_scratch_bytes(N, H, W).  Asynchronous on `stream`.  Limits as r2x_fdk's. */
int r2x_fdk_helical(void* stream, int n_views, int H, int W, const float* projs, const float* viewmatrices,
                    const float* projmatrices, float tan_fovx, float tan_fovy, int mode, int weighting, float dso,
                    const double* beta, const double* dbeta, const double* beta_host, double z0, double pitch,
                    double beta_lo, double beta_hi, double c_x, double c_y, float q, int nx, int ny, int nz, float sx,
                    float sy, float sz, float cx, float cy, float cz, float* out_volume, void* scratch,
                    size_t scratch_bytes);
int r2x_volume_project_views(void* stream, int nx, int ny, int nz, const float* volume, float sx, float sy, float sz,
                             float cx, float cy, float cz, int n_views, int H, int W, const float* viewmatrices,
                             int mode, float step, const double* view_geometry, const double* view_geometry_host,
                             float* out_projs);
int r2x_volume_backproject_views(void* stream, int n_views, int H, int W, const float* projs,
                                 const float* viewmatrices, const float* projmatrices, int mode, int nx, int ny,
                                 int nz, float sx, float sy, float sz, float cx, float cy, float cz, float step,
                                 const double* view_geometry, const double* view_geometry_host, float* out_volume,
                                 float* out_weight, void* scratch, size_t scratch_bytes);

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

/* ---- one Chambolle-Pock iteration for data-constrained TV (cp_tv, r2_gaussian_b200/recon.py and tv.py) ---------- */
/* Chambolle-Pock (primal-dual hybrid gradient) on  minimise TV(x) subject to |A x - b| <= eps, x in C,  with
 * K = [A; nu grad] (the grad / div = -grad^T of r2x_tv_prox).  The data dual q and its prox stay with the caller, in
 * projection space; this call is the rest of the iteration, given g = A^T q (r2x_volume_backproject of the new q):
 *   p_out    = P_{1/nu}(p + sigma nu grad xbar)                   per voxel: u, scaled by (1/nu) / |u| when |u| > 1/nu
 *   x_out    = P_C(x - tau g + tau nu div p_out)                  C = {x >= 0} when nonneg (u < 0 ? 0 : u), else all
 *   xbar_out = 2 x_out - x                                        (one fmaf)
 * x, xbar, g, x_out, xbar_out are float32 [nx,ny,nz] (z fastest); p, p_out are float32 [3,nx,ny,nz] (component a at
 * a * nx*ny*nz + voxel).  One launch (tv_cp_kernel in csrc/r2x_tv.cu): a CTA owns a 4 x 8 x 32 tile, holds xbar on the
 * tile's [-1, T] box and p_out on its [-1, T - 1] box in shared memory, and writes all three outputs of the tile;
 * 44 bytes per voxel.  p and xbar are read across tile edges, so the outputs are the caller's ping-pong buffers: no
 * output may overlap an input or another output (inputs may overlap each other, e.g. x == xbar).  No scratch.
 * tau, sigma, nu finite and > 0, and sigma nu, tau nu, 1 / nu finite (float32, rounded once from double).  No
 * atomics, bitwise reproducible; arguments are checked before any CUDA work; asynchronous on `stream`.
 * Limits: nx <= 262140, ny <= 524280. */
int r2x_tv_cp_step(void* stream, int nx, int ny, int nz, const float* x, const float* xbar, const float* p,
                   const float* g, float tau, float sigma, float nu, int nonneg, float* x_out, float* xbar_out,
                   float* p_out);

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

/* ---- ring-artifact correction: sorting-based stripe removal (r2_gaussian_b200/stripes.py, remove_stripes.py) ------ */
/* Vo, Atwood and Drakopoulos, Optics Express 26 (2018), `remove_stripe_based_sorting` of sarepy / algotom with the 1-D
 * window.  in[n, H, W] (device, float32: views, detector rows, detector columns) -> out[n, H, W]; K = 2h + 1 odd.  Each
 * row r is handled on its own, as the sinogram S[v, c] = in[v, r, c]:
 *   1. key     key(x) maps the float's bits u to a uint32 with the same total order: u ^ 0xFFFFFFFF for negatives (sign
 *              bit set), u | 0x80000000 otherwise.  -0 < +0, NaNs sort by their bits beyond -inf and +inf; every input
 *              has a defined output and none is refused for its value.
 *   2. sort    each column c over the views, ascending by (key, v): ties go to the lower view, the sort is stable.  This
 *              gives rank k = 0 .. n - 1, the sorted value T[k, c] and its view pi(k, c).
 *   3. median  M[k, c] = the element of rank h, by key, of T[k, c - h .. c + h]; a column j outside [0, W - 1] reads
 *              -j - 1 or 2W - 1 - j (scipy.ndimage's mode="reflect"), which needs h <= W.
 *   4. put     out[pi(k, c), r, c] = M[k, c].
 * The output holds only input values: nothing is rounded, and K = 1 is the identity bit for bit.  On finite inputs
 * without +-0 ties this is sarepy's argsort(kind="stable") / median_filter(size=(1, K), mode="reflect") / inverse
 * permutation.  Two passes (csrc/r2x_stripes.cu): one CTA per (row, column tile) sorts (key << 32 | v) words in shared
 * memory and writes the sorted keys (uint32) and views (uint16) rank-major, [H][n][W], into scratch; then one CTA per
 * (row, rank, 256-column tile) takes the windowed median and scatters it into out.  Scratch:
 * r2x_remove_stripes_scratch_bytes(n, H, W) = 6 n H W bytes (no GPU; 0 for a bad shape), 16-byte aligned.
 * out == in (in place) is allowed; no other overlap of in, out and the scratch is.  Arguments are checked before any
 * CUDA work: non-NULL pointers, 1 <= n <= R2X_STRIPES_MAX_VIEWS, H, W >= 1, H W < 2^31, K odd in [1, 255] with
 * h <= W, enough scratch, no overlap.  n H W is indexed in 64 bits.  No atomics, bitwise reproducible; rows are
 * independent, so any split of the rows into calls gives the same bits.  Asynchronous on `stream`. */
#define R2X_STRIPES_MAX_VIEWS 8192
#define R2X_STRIPES_MAX_SIZE 255
size_t r2x_remove_stripes_scratch_bytes(int n, int H, int W);
int r2x_remove_stripes(void* stream, int n, int H, int W, int K, const float* in, float* out, void* scratch,
                       size_t scratch_bytes);

/* ---- metal artifact reduction: metal-trace inpainting (r2_gaussian_b200/mar.py, reduce_metal.py, recon --mar) ------- */
/* Projection-domain MAR: linear interpolation across the metal trace (LI-MAR, Kalender et al. 1987) and, with a prior,
 * normalised interpolation (NMAR, Meyer et al., Med. Phys. 37, 2010).  p[n, H, W] (device, float32: views, detector
 * rows, detector columns), m[n, H, W] the projection of the metal mask (chord length through metal, the caller's units),
 * P[n, H, W] the projection of the NMAR prior or NULL.  Each row (view v, row r) is handled on its own, c = 0 .. W - 1:
 *   raw trace   t0[c] = m[c] > tau                           (a NaN m is not trace)
 *   trace       t[c] = any t0[k] for k in [c - d, c + d] clipped to [0, W - 1]              (d >= 0 columns)
 *   values      q = p without a prior; with one, Pe[c] = P[c] > eps ? P[c] : eps (a NaN P gives eps) and
 *               q[c] = p[c] / Pe[c], rounded to nearest
 *   outside t   out[c] = p[c] bit for bit (never normalised and de-normalised)
 *   inside t    l < c the nearest column outside t on the left, r > c on the right:
 *                 both    s = (float)(c - l) / (float)(r - l),  v = q[l] + s * (q[r] - q[l]), each operation rounded
 *                         to nearest on its own (no FMA contraction)
 *                 one     v = that side's q
 *                 neither (the whole row is trace) v = 1 with a prior; without one out[c] = p[c]
 *               out[c] = v * Pe[c] (rounded to nearest) with a prior, v without one
 *   trace       trace[v, r, c] = t[c] (uint8 0 / 1) when trace is not NULL.
 * A NaN that arithmetic produces (an interpolation, a division or product by Pe) is the canonical 0x7FFFFFFF whatever
 * NaN went in; a copied value (outside the trace, a one-sided value without a prior) keeps its bits.
 * The rules select and interpolate; a numpy float32 restatement gives the same bits.  One CTA of 256 threads per (view,
 * row), the row staged in shared memory: the dilation from an exclusive prefix count of t0, l and r from a block
 * max-scan / reverse min-scan of each thread's run of columns, so a row costs O(W) whatever its trace (csrc/r2x_mar.cu).
 * Shared memory per CTA: 9 W + 4 bytes without a prior, 13 W + 4 with one; R2X_MAR_MAX_W = 16384 keeps it under the
 * 227 KB opt-in of sm_90.  out == p (in place) is allowed; out and trace may not overlap anything else.  Arguments are
 * checked before any CUDA work: non-NULL p, m, out; n, H, W >= 1; n H < 2^31 (the grid); W <= R2X_MAR_MAX_W; finite
 * tau; finite eps > 0 (also without a prior); d >= 0; no overlap.  n H W is indexed in 64 bits.  No atomics, bitwise
 * reproducible; rows are independent, so any split of the stack into calls gives the same bits.  Asynchronous on
 * `stream`. */
#define R2X_MAR_MAX_W 16384
int r2x_mar_inpaint(void* stream, int n, int H, int W, const float* p, const float* m, float tau, int d,
                    const float* P, float eps, float* out, uint8_t* trace);

/* ---- cubic B-spline zoom of a placed volume (r2_gaussian_b200/resample.py, process_raw_data.py) ------------------ */
/* A placed volume V[shape] is a source volume set at `offset` and normalised:
 *   V[p] = (float64(src[p - offset]) - lo) / (hi - lo)   where p - offset lies in src_shape, else 0,
 * both operations in float64, one rounding each.  src is device memory of element type `dtype`, read at
 * sum_a q[a] * src_strides[a] (elements; a transposed host array keeps its strides).  A positive offset pads with zeros
 * (expand_to_cube), a negative one crops (crop_to_cube), lo = 0, hi = 1 passes the values through unchanged.
 * r2x_volume_place writes V (float64, C order) to out.
 * r2x_zoom_cubic writes scipy.ndimage.zoom(V, zoom, order=3, mode="nearest") to out[out0, out1, out2] (float64): V padded
 * by 12 edge voxels per side into `workspace`, the cubic B-spline prefilter along each axis in place (gain 6, pole
 * sqrt(3) - 2, mirror start value), then output index o maps to x = o (n - 1) / (out - 1) + 12 (factor 1 when
 * out = 1) and sums the 4 x 4 x 4 coefficients floor(x) - 1 .. floor(x) + 2 with the cubic B-spline weights.  The
 * caller chooses out = int(round(n * zoom)) per axis and uses r2x_volume_place when every factor is exactly 1 (scipy
 * returns a copy there).  r2x_zoom_workspace_bytes(shape) = (shape + 24)^3 * 8 bytes, 0 for a bad shape; no GPU needed.
 * Arguments are checked before any CUDA work (non-NULL pointers, dtype, src_shape >= 1, strides >= 0, shape and out
 * sizes in [1, 32768], lo and hi finite with hi > lo, workspace large enough).  64-bit indexing, no atomics, bitwise
 * reproducible.  Asynchronous on `stream`. */
#define R2X_PLACE_U8 0
#define R2X_PLACE_U16 1
#define R2X_PLACE_F64 2
typedef struct r2x_place_desc {
    const void* src;            /* device                                        */
    int dtype;                  /* R2X_PLACE_U8, R2X_PLACE_U16 or R2X_PLACE_F64   */
    int src_shape[3];
    long long src_strides[3];   /* in elements, >= 0                             */
    int shape[3];               /* the placed volume                             */
    int offset[3];              /* its index of source voxel (0, 0, 0)           */
    double lo, hi;
} r2x_place_desc;
size_t r2x_zoom_workspace_bytes(int n0, int n1, int n2);
int r2x_volume_place(void* stream, const r2x_place_desc* desc, double* out);
int r2x_zoom_cubic(void* stream, const r2x_place_desc* desc, int out0, int out1, int out2, void* workspace,
                   size_t workspace_bytes, double* out);

/* ---- isosurface of a volume: marching cubes (r2_gaussian_b200/mesh.py, extract_mesh.py) ------------------------- */
/* Replaces skimage.measure.marching_cubes in the reference's create_vol_mesh (r2_gaussian/utils/plot_utils.py).
 * vol[nx,ny,nz] (device, float32, z fastest) is sampled at the integer index points (i, j, k); level is finite.
 *   inside   a sample is inside iff v > level (strict; NaN is outside).
 *   cubes    cube s = (i, j, k) for i < nx-1, j < ny-1, k < nz-1; corner b in 0..7 sits at s + (b&1, b>>1&1, b>>2&1);
 *            the case is the 8-bit mask of its inside corners.  Cube edges are numbered axis-major: 0-3 along x (lower
 *            corners 0, 2, 4, 6), 4-7 along y (0, 1, 4, 5), 8-11 along z (0, 1, 2, 3).  A grid edge is owned by its
 *            lower sample and axis (s, a) and is cut iff exactly one end is inside.
 *   vertex   a = v[p0] (lower end), b = v[p1]; t = (level - a) / (b - a) in float32 (IEEE division); the vertex is p0
 *            except along axis a, where it is float32(p0[a]) + t.  No FMA: a numpy float32 statement gives the same
 *            bits.  Index space.  A vertex may land on a sample that equals level; degenerate triangles are kept.
 *   table    generated on the host by a rule, checked, and copied to __constant__ memory on first use per device:
 *            1. face rule: on each cube face, each maximal run of inside corners along the face's 4-cycle is cut off
 *               by one segment joining the two cut edges that bound it (diagonal inside corners are separated, diagonal
 *               outside corners joined).  Two cubes sharing a face derive the same segments: no cracks.
 *            2. the segments chain into closed loops (each cut edge ends one segment and starts one).
 *            3. every triangle is counter-clockwise seen from the outside region (values <= level): (v1-v0)x(v2-v0)
 *               points from inside to outside; a closed surface around a high-valued blob has positive signed volume.
 *            4. loops in order of their smallest edge; each is a fan from the first vertex, walking the loop in its
 *               direction from its smallest edge, whose fan diagonals join no two edges of a common cube face.
 *            A table without such an apex for some loop, or with more than 5 triangles in a case, is refused.
 *   order    vertices by owning sample (i ny + j) nz + k, then axis x < y < z; triangles by cube (linear index of its
 *            lower sample), then table order.  verts float32 [V,3] (x = i, y = j, z = k), faces int32 [T,3].
 * r2x_marching_cubes_table copies the table out (no GPU): ntri[256], edges[256][15], -1 padded.
 * r2x_marching_cubes_count classifies every sample and writes totals_dev[2] (device) = {V, T} in 64 bits.
 * r2x_marching_cubes_emit, on the scratch the count pass just filled, scans the per-word counts and writes the mesh;
 * every write is bounded by the V and T it is given (wrong totals give a short mesh, never an out-of-bounds write),
 * and V or T >= 2^31 returns R2X_ERR_OVERFLOW before any work.  Vertex ids come from the scans: the mesh is indexed and
 * shared, with no welding pass.  Scratch (r2x_marching_cubes_scratch_bytes, no GPU; 0 for a bad grid): 5 uint32 words
 * per 32 samples, 0.625 bytes per sample, plus 8 bytes per 32768 samples and under 2 KiB; the count pass fills 0.375 bytes
 * per sample of it (inside bits and two per-word counts).  Arguments are checked before any CUDA work (non-NULL
 * pointers, each size >= 1 -- an axis shorter than 2 has no cubes --, nx ny nz <= 2^31 - 1, finite level, enough
 * scratch).  64-bit addressing, no atomics on the output, bitwise reproducible; asynchronous on `stream`. */
int r2x_marching_cubes_table(int* ntri /* 256 */, signed char* edges /* 256 * 15 */);
size_t r2x_marching_cubes_scratch_bytes(int nx, int ny, int nz);
int r2x_marching_cubes_count(void* stream, int nx, int ny, int nz, const float* vol, float level, long long* totals_dev,
                             void* scratch, size_t scratch_bytes);
int r2x_marching_cubes_emit(void* stream, int nx, int ny, int nz, const float* vol, float level, long long V,
                            long long T, float* verts, int* faces, void* scratch, size_t scratch_bytes);

/* ---- volume rendering: emission-absorption and MIP ray casting (r2_gaussian_b200/volume_render.py, render_volume.py) */
/* Replaces the pyvista / VTK volume plot of the reference's scripts/plot_volume.py.  Parity with VTK's pixels is not
 * claimed.  vol[nx,ny,nz] (device, float32, z fastest), every axis >= 2.  Index space: sample vol[i,j,k] sits at the
 * point (i, j, k); the field is the trilinear interpolant of the samples on the box B = [0,nx-1] x [0,ny-1] x [0,nz-1].
 *   camera   cameras_dev (device, float32) holds R2X_VR_CAMERA_FLOATS = 16 floats per frame:
 *            P[3] position, f[3] unit view direction, r[3] unit right, u[3] unit up, p pixel pitch, 3 unused.
 *            The host builds them in float64 from a position P, focal point F and view-up U: f = normalize(F - P),
 *            r = normalize(f x U), u = r x f; p = 2 tan(view_angle / 2) / H (perspective) or 2 S / H (parallel, S the
 *            parallel scale: half the image height in voxels).  Pixel (row y from the top, column x) has offsets
 *            a = ((x + 1/2) - W/2) p and b = ((H/2 - y) - 1/2) p.  Perspective: the ray leaves o = P along
 *            d = normalize((f + a r) + b u); parallel (`parallel` = 1): it leaves o = (P + a r) + b u along d = f.
 *   samples  [s_in, s_out] is the ray's parameter interval inside B (slab method, per axis (0 - o)/d and
 *            ((n-1) - o)/d; an axis with d = 0 constrains nothing if 0 <= o <= n-1 and misses otherwise), with s_in
 *            clamped to >= 0.  s_out < s_in misses.  Otherwise the samples are s_k = s_in + k step for
 *            k = 0 .. floor((s_out - s_in) / step), each formed from k, at the point o + s_k d, clamped into B; the
 *            cell is i0 = min(floor(p), n - 2) per axis, w = p - i0, and the value is the trilinear blend with weights
 *            (1 - w, w) along each axis.  The ray set-up and sample points are float64 without FMA (a numpy float64
 *            statement gives the same sample counts and points); w is rounded to float32 and everything after it is
 *            float32.
 *   transfer t = clamp((v - c0) * (1 / (c1 - c0)), 0, 1) (the reciprocal rounded once to float32); colour from the
 *            K-entry RGB LUT lut_dev (device, float32 [K][3]): pos = t (K - 1), j = min(floor(pos), K - 2),
 *            w = pos - j, colour = (1 - w) L[j] + w L[j+1]; K = 1 is a constant colour.  Opacity alpha_tf = t.
 *   mode 0   composite: alpha = 1 - (1 - alpha_tf)^(step / unit) (unit: the opacity unit distance, in voxels); front
 *            to back from C = 0, T = 1: C += T alpha colour, T *= 1 - alpha; the ray stops after the first sample
 *            that leaves T < 2^-16.  RGB = C + T background, A = 1 - T.
 *   mode 1   MIP: m = the largest sampled value; RGB = colour(t(m)), A = 1 for a ray that meets B.
 *            A ray that misses B gets RGB = background, A = 0 in both modes.
 *   output   out (device, float32) [n_frames, H, W, 4] RGBA.  No shading, no jitter, no texture filtering.
 * One thread per pixel, R2X_VR_TILE x R2X_VR_TILE pixel tiles, frames on the grid's z dimension; no atomics, bitwise
 * reproducible; asynchronous on `stream`.  background[3] is a host pointer.  Arguments are checked before any CUDA
 * work: non-NULL pointers, nx ny nz >= 2, n_frames H W >= 1, parallel 0 or 1, mode 0 or 1, 1 <= K <= 4096, finite
 * c0 < c1 with c1 - c0 a finite float, finite step > 0 with at most 2^31 - 1 samples along the box diagonal, finite unit > 0, a finite background,
 * frames and pixel tiles per grid dimension <= 65535 (so n_frames H W 4 < 2^62 for the 64-bit output index). */
#define R2X_VR_CAMERA_FLOATS 16
#define R2X_VR_TILE 16
#define R2X_VR_COMPOSITE 0
#define R2X_VR_MIP 1
int r2x_volume_render(void* stream, int nx, int ny, int nz, const float* vol, int n_frames, int H, int W,
                      const float* cameras_dev, int parallel, int mode, float c0, float c1, const float* lut_dev, int K,
                      float step, float unit, const float* background, float* out);

/* ---- scene view: depth-tested triangles, line segments and ellipsoids (scene_view.py, visualize_scene.py) ---- */
/* Replaces the open3d window of the reference's scripts/visualize_scene.py with a headless rasterizer.  Pixel parity
 * with open3d is not claimed.  Everything is in scene units.
 *   input    n_prims primitives; primitive i has pos[i] (device, float64 [3][3]: three points, a segment uses the first
 *            two), meta[i] (device, int32 [2]: kind, texture index) and attr[i] (device, float32 [R2X_SV_ATTR = 12]):
 *              R2X_SV_FLAT     0 triangle, colour attr[0:3]
 *              R2X_SV_MESH     1 triangle, base colour attr[0:3], per-vertex normals attr[3:6], [6:9], [9:12] (world)
 *              R2X_SV_TEXTURED 2 triangle, per-vertex texture coordinates (u, v) in attr[3:5], [5:7], [7:9]
 *              R2X_SV_LINE     3 segment pos[i][0] -> pos[i][1], colour attr[0:3], width w = attr[3] pixels (> 0)
 *              R2X_SV_ELLIPSOID 4 solid ellipsoid E = { c + R diag(s) v : |v| <= 1 } (the 1-sigma ellipsoid of
 *                              Sigma = R S^2 R^T): centre c = pos[i][0], semi-axes s = pos[i][1] (all > 0; pos[i][2] is
 *                              ignored), colour attr[0:3], quaternion (w, x, y, z) = attr[3:7] (non-zero)
 *            tex (device, float32 [n_tex][tex_h][tex_w]) and lut (device, float32 [K][3]) serve textured triangles.
 *   camera   cameras (device, float32) holds R2X_SV_CAMERA_FLOATS = 16 floats per frame, the record of the volume
 *            renderer (P, f, r, u, pitch p; `parallel` selects the projection), read as float64.  Camera coordinates of
 *            a point X: d = X - P, (x, y, z) = (d.r, d.u, d.f), each dot product ((d0 a0 + d1 a1) + d2 a2).
 *            Screen: sx = W/2 + x / q, sy = H/2 - y / q with q = z p (perspective) or q = p (parallel); pixel (column x,
 *            row y from the top) has its centre at (x + 1/2, y + 1/2).
 *   clip     in camera coordinates, against 5 planes in order, inside iff the value is >= 0: z - near; and the guard band
 *            G = R2X_SV_GUARD = 2^20 pixels: g - x, g + x, g - y, g + y with g = G p z (perspective) or G p (parallel).
 *            A triangle is clipped Sutherland-Hodgman (vertices in order, each edge a -> b keeps a if inside and adds the
 *            cut if the two sides differ); every cut point is formed from the edge's inside end A to its outside end B:
 *            t = dA / (dA - dB), A + t (B - A), so two triangles that share an edge get the same cut points.  The
 *            polygon (3 to 8 vertices; fewer than 3 is nothing) is the fan (0, k, k+1).  A segment keeps the part
 *            inside every plane, its outside end replaced by the cut.  Anything wholly behind the near plane is dropped.
 *   snap     screen points are snapped to 1/256 pixel: X = rint(256 sx), Y = rint(256 sy) (int64, ties to even).
 *   coverage triangle (fan triangle A, B, C; zero area dropped; negative area: B and C swapped, both windings drawn):
 *            pixel centre p = (256 x + 128, 256 y + 128) is covered iff for each edge a -> b (A->B, B->C, C->A)
 *            e = dx (py - ay) - dy (px - ax) with (dx, dy) = b - a is > 0, or = 0 on an edge with dy < 0 or (dy = 0 and
 *            dx > 0) (top-left rule).  All int64, exact: two triangles sharing an edge never both cover a pixel and
 *            never both miss one.  A polygon covers the union of its fan.
 *            segment (ends a, b = the snapped points / 256, in pixels; c = pixel centre; all float64, round to nearest):
 *            d = b - a, e = c - a, L = d.d, t = clamp((e.d) / L, 0, 1) (0 if L = 0), q = e - t d; covered iff
 *            q.q <= r r with r = w / 2.
 *   depth    triangle: with the camera-space plane n = (V1 - V0) x (V2 - V0), c = n.V0 of the unclipped vertices and the
 *            pixel's a = ((x + 1/2) - W/2) p, b = ((H/2 - y) - 1/2) p: z = c / ((n0 a + n1 b) + n2) (perspective) or
 *            ((c - n0 a) - n1 b) / n2 (parallel) -- perspective-correct.  Segment: 1/z = (1 - t)/za + t/zb
 *            (perspective) or z = za + t (zb - za) (parallel), za, zb the clipped ends' depths.  z below near (or NaN)
 *            becomes near; then rounded once to float32.
 *   visible  each covered pixel does a 64-bit atomicMin of (float bits of z) << 32 | i into keys (device, uint64
 *            [n_frames][H][W], all ones where nothing is drawn).  Positive floats order as their bits: the nearest
 *            primitive wins and ties go to the lower id; the minimum does not depend on the order of the atomics.
 *   shading  one thread per pixel decodes the id.  Flat triangles and segments: their colour.  Mesh and textured
 *            triangles: the point P on the plane (perspective (a z, b z, z), parallel (a, b, z), z as above) has weights
 *            w_v = n.((V_{v+1} - P) x (V_{v+2} - P)) / n.n (1/3 each if n.n = 0).  Mesh: N = sum w_v N_v, D = the
 *            pixel's ray direction in world coordinates ((f + a r) + b u, or f), lambda = min(|N.D| / sqrt(N.N D.D), 1)
 *            (0 if N = 0), colour = base (A + (1 - A) lambda) with A = R2X_SV_AMBIENT = 0.25: a two-sided headlight.
 *            Textured: (u, v) = sum w_v uv_v, texel column min(max(floor(u tex_w), 0), tex_w - 1), row likewise from v
 *            and tex_h, value t clamped to [0, 1] (NaN -> 0), colour from the LUT as the volume renderer maps t
 *            (float32, no FMA).  Float64 until the colour is rounded to float32.  Uncovered: background[3] (host).
 *   ellipsoid (kind 4; float64, every operation rounded to nearest in the order written, dot products as above)
 *            rotation  q = attr[3:7] read as float64, m = sqrt(((w w + x x) + y y) + z z), (w, x, y, z) /= m, and R is
 *                      build_rotation's matrix: R00 = 1 - 2 (y y + z z), R01 = 2 (x y - w z), R02 = 2 (x z + w y),
 *                      R10 = 2 (x y + w z), R11 = 1 - 2 (x x + z z), R12 = 2 (y z - w x), R20 = 2 (x z - w y),
 *                      R21 = 2 (y z + w x), R22 = 1 - 2 (x x + y y); k_j = 1 / s_j.
 *            ray       pixel (x, y) with a, b as below: perspective O = P, D = (f + a r) + b u; parallel
 *                      O = (P + a r) + b u, D = f.  D.f is 1 up to the camera's rounding: the ray parameter is the depth.
 *            hit       w = O - c; e_j = ((R0j w0 + R1j w1) + R2j w2) k_j, g_j likewise from D; A = g.g, B = g.e,
 *                      C = e.e - 1, Delta = B B - A C.  Covered iff Delta >= 0 and the larger root is >= near, with the
 *                      roots t1 = h / A and t2 = C / h (t2 = t1 if h = 0), h = -(B + copysign(sqrt(Delta), B)); z is
 *                      the smaller root if it is >= near, else the larger (a camera inside, or an ellipsoid cut by the
 *                      near plane, sees the inside surface).  The key is written as for the other kinds.
 *            box       c' = the camera coordinates of c; M_ij = ((r_0 R0j + r_1 R1j) + r_2 R2j) s_j with the camera
 *                      rows r, u, f for i = 0, 1, 2; S_kl = (M_k0 M_l0 + M_k1 M_l1) + M_k2 M_l2 (Sigma in camera
 *                      coordinates).  Nothing if c'_z + sqrt(S_zz) < near.  Perspective with c'_z - sqrt(S_zz) < near,
 *                      or with a2 = c'_z c'_z - S_zz not > 0: the whole frame.  Perspective otherwise: in x the tangent
 *                      planes through the camera, b1 = c'_x c'_z - S_xz, c0 = c'_x c'_x - S_xx,
 *                      d = sqrt(max(b1 b1 - a2 c0, 0)), alpha = (b1 -+ d) / a2, sx = W/2 + alpha / p; in y likewise
 *                      from c'_y, S_yz, S_yy, sy = H/2 - beta / p.  Parallel: sx = W/2 + (c'_x -+ sqrt(S_xx)) / p,
 *                      sy = H/2 - (c'_y +- sqrt(S_yy)) / p.  Pixel box: columns min(max(floor(sx_lo) - 1, 0), W) to
 *                      max(min(floor(sx_hi) + 1, W - 1), -1), rows likewise (empty if reversed).
 *            shading   the hit is recomputed from the id: H = O + z D (per component O_i + z D_i), v = H - c,
 *                      m_j = (R0j v0 + R1j v1) + R2j v2, n_i = (R_i0 (m_0 k_0) k_0 + R_i1 (m_1 k_1) k_1) + R_i2 (m_2 k_2) k_2
 *                      (n = R diag(1/s^2) R^T (H - c)), lambda = min(|n.D| / sqrt(n.n D.D), 1) (0 if n = 0), colour =
 *                      base (A + (1 - A) lambda): the mesh's headlight.
 *   output   rgb (device, float32 [n_frames][H][W][3]).
 * Work: a primitive whose clamped pixel box is at most R2X_SV_TILE = 16 pixels on each side is rasterized by one thread;
 * a larger one is split into the 16 x 16 tiles of its box, one CTA (one thread per pixel) per tile.  Frames on the
 * grid's z dimension.  Scratch (r2x_scene_raster_scratch_bytes, no GPU; 0 for bad sizes): 64 bytes plus 40 bytes per
 * (primitive, frame).  Arguments are checked before any CUDA work: non-NULL pointers (tex only with n_tex > 0),
 * 1 <= n_prims with n_prims n_frames <= 2^31 - 1, 1 <= n_frames <= 65535, 1 <= H, W <= R2X_SV_MAX_SIDE = 16384,
 * texture sides 1 to 16384 with n_tex tex_h tex_w <= 2^31 - 1, 1 <= K <= 4096, parallel 0 or 1, finite near > 0, a
 * finite background, enough scratch.  The contents of pos / meta / attr / tex (finite points, widths > 0, kinds,
 * texture indices < n_tex, semi-axes > 0, non-zero quaternions) are the caller's to check.  Asynchronous on `stream`; two calls give the same bits. */
#define R2X_SV_CAMERA_FLOATS 16
#define R2X_SV_ATTR 12
#define R2X_SV_TILE 16
#define R2X_SV_MAX_SIDE 16384
#define R2X_SV_GUARD 1048576.0
#define R2X_SV_AMBIENT 0.25
#define R2X_SV_FLAT 0
#define R2X_SV_MESH 1
#define R2X_SV_TEXTURED 2
#define R2X_SV_LINE 3
#define R2X_SV_ELLIPSOID 4
size_t r2x_scene_raster_scratch_bytes(int n_prims, int n_frames);
int r2x_scene_raster(void* stream, int n_prims, const double* pos, const int* meta, const float* attr, int n_tex,
                     int tex_h, int tex_w, const float* tex, const float* lut, int K, int n_frames, int H, int W,
                     const float* cameras, int parallel, double near, const float* background,
                     unsigned long long* keys, float* rgb, void* scratch, size_t scratch_bytes);

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
