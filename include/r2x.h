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
 * Deterministic.  scratch: r2x_image_loss_scratch_bytes(H, W). */
size_t r2x_image_loss_scratch_bytes(int H, int W);
int r2x_image_loss(void* stream, int H, int W, const float* image, const float* target, float w_l1,
                   float w_dssim, float* loss_out, float* grad_out, void* scratch, size_t scratch_bytes);

/* 3-D total variation of vol[nx][ny][nz] (`tv_3d_loss`, loss_utils.py:19-34): sum of absolute forward
 * differences along the three axes, divided by their number when reduction_mean != 0.  loss_out[1] (device),
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
