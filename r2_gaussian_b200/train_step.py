"""One training iteration as a fixed sequence of libr2xray calls on preallocated buffers.

The reference's iteration (train.py:104-160) is render() -> L1 + D-SSIM -> query() of a random TV crop -> backward ->
densification statistics -> Adam, expressed as ~270 torch kernels behind autograd.  With the fused kernels of this
package the GPU needs ~0.55 ms for it at 100k Gaussians / 512^2, but the autograd path still spends ~1 ms of HOST time
per iteration (about fifty small torch ops, four autograd.Function round trips, thirty allocations).  `NativeTrainStep`
issues the same kernels directly:

    raster forward (raw parameters)      r2x_raster_forward_async_raw        [image summed over ranks when sharded]
    L1 + D-SSIM value and gradient       r2x_image_loss
    TV-crop query forward                r2x_voxel_forward_async_raw         [volume summed over ranks when sharded]
    TV value and gradient                r2x_tv3d_loss
    both backward passes                 r2x_voxel_backward_raw, r2x_raster_backward_raw
    densification statistics             r2x_densify_stats
    Adam on the four parameter tensors   r2x_adam_step_sum  (gradient = raster part + voxel part)

No autograd graph, no per-iteration allocation, no host synchronisation: both forwards are speculative (instance
capacity from `_C._Workspace.provision`, after the previous call of the same shape), and the statistics / Adam launches
are GUARDED by the forwards' overflow flags on the device, so an overflowed iteration changes nothing; the host reads
the flags one iteration late (`check()`, through `_C._Workspace.read`, which raises the hint) and repeats that
iteration.

With `pose=(PoseCorrection, FusedAdam over [omega] and [nu], one group each)` the step also refines the view's pose
(`pose.py`), still without autograd or host synchronisation:

    corrected matrices of view i         r2x_pose_apply                       (before the raster forward)
    raster backward + matrix gradients   r2x_raster_backward_pose             (replaces r2x_raster_backward_raw; the
                                                                               same per-Gaussian gradients bit for bit)
    twist gradient of view i             r2x_pose_grad                        (row `pose_anchor` held at 0)
    Adam on omega and nu                 r2x_adam_step_sum                    (after the Gaussians', same guards)

`__call__` then takes the view index; the pose step count is kept like the Gaussians' (undone when `check()` repeats an
iteration).  Pose refinement with Gaussian sharding is refused at bind time: each rank would hold only a partial sum
of the matrix gradients.  With `pose=None` the launch sequence is the one above.

With `detector=(DetectorOffset, FusedAdam over [offset])` the step also learns the horizontal detector offset
(`detector.py`), for one camera or a batch:

    shifted full projections             r2x_detector_offset_apply            (the B views' matrices, one launch)
    offset gradient                      r2x_detector_offset_grad             (from this step's dL/dmean2D)
    Adam on the offset                   r2x_adam_step_sum                    (after the Gaussians', same guards)

The offset's step count is kept like the pose's.  Not combined with pose refinement or Gaussian sharding.

A LIST of B > 1 cameras (with a [B,H,W] target) makes one iteration of B views: the objective is
sum_v [L1 + lambda_dssim (1 - SSIM)](view v) + B lambda_tv TV(crop), one Adam step, the statistics of every view in view
order.  The raster and loss calls become their batched forms (r2x_raster_forward_views_async_raw, r2x_image_loss_views,
r2x_raster_backward_views_raw, r2x_densify_stats_views), so each view's image and image gradient is bit for bit its
single-view one and the launch count does not grow with B.  The buffers are bound per B; a repeated iteration repeats
the same batch.  Batches take no pose refinement and no Gaussian sharding.  A list of one camera is the single-view
iteration.

The model's tensors are updated in place: `GaussianModel._xyz/_density/_scaling/_rotation`, the `FusedAdam` state of
`gaussians.optimizer` (same `exp_avg`, `exp_avg_sq`, `step`, so checkpoints and the densification surgery are
unchanged) and `max_radii2D / xyz_gradient_accum / denom`.  After densification (new tensors) the step re-binds itself.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import torch

from . import _C, fused, sharded
from ._lib import AdamGroup, check, load


def enabled() -> bool:
    return fused.enabled() and os.environ.get("R2X_NATIVE_STEP", "1") != "0"


class NativeTrainStep:
    def __init__(self, gaussians, lambda_dssim: float, lambda_tv: float = 0.0, tv_vol_nVoxel=None, tv_vol_sVoxel=None,
                 scaling_modifier: float = 1.0, pose=None, pose_anchor: int = 0, detector=None):
        self.gm = gaussians
        self.pose, self.pose_opt = (None, None) if pose is None else pose
        self.det, self.det_opt = (None, None) if detector is None else detector
        if self.pose is not None and self.det is not None:
            raise ValueError("NativeTrainStep: pose refinement and the detector offset cannot be combined")
        self.pose_anchor = int(pose_anchor)
        self.lambda_dssim, self.lambda_tv = float(lambda_dssim), float(lambda_tv)
        self.tv_n = None if tv_vol_nVoxel is None else tuple(int(v) for v in tv_vol_nVoxel)
        self.tv_s = None if tv_vol_sVoxel is None else tuple(float(v) for v in tv_vol_sVoxel)
        self.use_tv = self.lambda_tv > 0 and self.tv_n is not None
        self.scale_modifier = float(scaling_modifier)
        self.lib = load()
        self._bound = None          # identity of the tensors the buffers were made for
        self._pending = None        # (host status words, event, keys, caps, args) of the last enqueued iteration
        self.repeats = 0            # iterations repeated after a capacity overflow

    # ------------------------------------------------------------------ buffers
    def _signature(self, H, W, B):
        gm = self.gm
        sig = (sharded.enabled(), gm._xyz.data_ptr(), gm._density.data_ptr(), gm._scaling.data_ptr(), gm._rotation.data_ptr(),
               int(gm._xyz.shape[0]), H, W, B, gm.max_radii2D.data_ptr(), gm.xyz_gradient_accum.data_ptr())
        if self.pose is not None:
            sig += (self.pose.omega.data_ptr(), self.pose.nu.data_ptr())
        if self.det is not None:
            sig += (self.det.offset.data_ptr(),)
        return sig

    def _bind(self, H, W, B):
        gm, lib = self.gm, self.lib
        dev = gm._xyz.device
        P = int(gm._xyz.shape[0])
        self.P, self.H, self.W, self.B, self.dev = P, H, W, B, dev
        f32 = dict(dtype=torch.float32, device=dev)
        u8 = dict(dtype=torch.uint8, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        self.sharded = sharded.enabled()
        if B > 1 and (self.sharded or self.pose is not None):
            raise RuntimeError("NativeTrainStep: a batch of views takes no Gaussian sharding and no pose refinement")
        with torch.cuda.device(dev):
            # raster.  Gaussian-sharded runs: the image travels through the exchange with one extra word, this rank's
            # overflow flag, so that after the sum EVERY rank knows whether ANY rank's forward overflowed (the summed
            # image is then wrong everywhere) and all ranks skip / repeat the iteration together.  B views: images,
            # radii and dL/dmean2D per view, the stacked camera matrices, and the batched forward's state.
            self.image_ext = torch.zeros(B * H * W + 4, **f32)
            self.image = self.image_ext[:B * H * W].view(B, H, W)
            self.flag_r = self.image_ext[B * H * W:B * H * W + 1]
            self.radii = torch.empty((P,) if B == 1 else (B, P), **i32)
            if B == 1:
                self.geom, self.img = _C.RASTER.state(P, (W, H), dev)
            else:
                self.geom, self.img = _C.views_state(P, B, W, H, dev)
                self.views = torch.empty((B, 4, 4), **f32); self.projs = torch.empty((B, 4, 4), **f32)
            self.status_r = torch.zeros(2, **i32)
            self.key_r = _C.raster_key(dev, P, W, H) if B == 1 else _C.views_key(dev, P, B, W, H)
            self.g2 = torch.empty((P, 3) if B == 1 else (B, P, 3), **f32)
            self.gd = torch.empty((P, 1), **f32); self.g3 = torch.empty((P, 3), **f32)
            self.gcov = torch.empty((P, 6), **f32); self.gs = torch.empty((P, 3), **f32); self.gr = torch.empty((P, 4), **f32)
            # image loss
            self.loss_scratch_bytes = int(lib.r2x_image_loss_scratch_bytes(H, W) if B == 1 else
                                          lib.r2x_image_loss_views_scratch_bytes(B, H, W))
            self.loss_scratch = torch.empty(self.loss_scratch_bytes, **u8)
            # L1, SSIM, lambda_l1 L1 + lambda_dssim (1 - SSIM); one row per view
            self.loss_out = torch.zeros(3 if B == 1 else (B, 3), **f32)
            self.dL_dimage = torch.empty((H, W) if B == 1 else (B, H, W), **f32)
            # TV crop
            if self.use_tv:
                nx, ny, nz = self.tv_n
                self.vol_ext = torch.zeros(nx * ny * nz + 4, **f32)
                self.vol = self.vol_ext[:nx * ny * nz].view(nx, ny, nz)
                self.flag_v = self.vol_ext[nx * ny * nz:nx * ny * nz + 1]
                self.rx = torch.empty((P,), **i32); self.ry = torch.empty((P,), **i32); self.rz = torch.empty((P,), **i32)
                self.geom_v, self.img_v = _C.VOXEL.state(P, self.tv_n, dev)
                self.status_v = torch.zeros(2, **i32)
                self.key_v = _C.voxel_key(dev, P, nx, ny, nz, self.tv_s[0])
                self.tv_scratch_bytes = int(lib.r2x_tv3d_scratch_bytes(nx, ny, nz))
                self.tv_scratch = torch.empty(self.tv_scratch_bytes, **u8)
                self.tv_out = torch.zeros(1, **f32)
                self.dL_dvol = torch.empty((nx, ny, nz), **f32)
                self.gdv = torch.empty((P, 1), **f32); self.g3v = torch.empty((P, 3), **f32); self.gcovv = torch.empty((P, 6), **f32)
                self.gsv = torch.empty((P, 3), **f32); self.grv = torch.empty((P, 4), **f32)
            self.cap_r = self.cap_v = 0
            self.binning_r = self.binning_v = self.scratch_r = self.scratch_v = None
        # Adam: the optimizer's own state tensors, one group per parameter tensor (xyz, density, scaling, rotation)
        opt = gm.optimizer
        self.adam = []
        grads = {id(gm._xyz): (self.g3, self.g3v if self.use_tv else None),
                 id(gm._density): (self.gd, self.gdv if self.use_tv else None),
                 id(gm._scaling): (self.gs, self.gsv if self.use_tv else None),
                 id(gm._rotation): (self.gr, self.grv if self.use_tv else None)}
        for group in opt.param_groups:
            for p in group["params"]:
                if id(p) not in grads:
                    raise RuntimeError("NativeTrainStep: the optimizer holds a parameter that is not one of the model's four")
                st = opt.state[p]
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                self.adam.append((group, p, st, *grads[id(p)]))
        if len(self.adam) != 4:
            raise RuntimeError("NativeTrainStep: expected the four parameter groups of GaussianModel.training_setup")
        n = len(self.adam)
        self.adam_groups = (AdamGroup * n)()
        self.adam_grads2 = (C.c_void_p * n)()
        for k, (group, p, st, g1, g2) in enumerate(self.adam):
            a = self.adam_groups[k]
            a.param, a.grad, a.exp_avg, a.exp_avg_sq = p.data_ptr(), g1.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr()
            a.numel = p.numel()
            self.adam_grads2[k] = g2.data_ptr() if g2 is not None else None
        self.act = fused._act(gm.raw_parameters())
        if self.pose is not None:
            self._bind_pose(P, dev)
        if self.det is not None:
            self._bind_detector(P, B, dev)
        self._bound = self._signature(H, W, B)

    def _bind_pose(self, P, dev):
        """Buffers of the pose path: corrected matrices, their gradients, the pose gradients and the two Adam groups
        (omega, nu) on the pose optimizer's own state tensors."""
        if self.sharded:
            raise RuntimeError("NativeTrainStep: pose refinement is not supported with Gaussian sharding (every rank "
                               "would hold only its shard's part of the matrix gradients)")
        corr, opt = self.pose, self.pose_opt
        for name, p in (("omega", corr.omega), ("nu", corr.nu)):
            if p.device != dev or p.dtype != torch.float32 or not p.is_contiguous():
                raise RuntimeError(f"NativeTrainStep: pose {name} must be contiguous float32 on {dev}")
        groups = [(g, g["params"]) for g in opt.param_groups]
        if len(groups) != 2 or groups[0][1] != [corr.omega] or groups[1][1] != [corr.nu]:
            raise RuntimeError("NativeTrainStep: the pose optimizer must hold two groups, [omega] and [nu]")
        self.n_views = int(corr.omega.shape[0])
        if not -1 <= self.pose_anchor < self.n_views:
            raise ValueError(f"NativeTrainStep: pose anchor {self.pose_anchor} out of range for {self.n_views} views")
        f32 = dict(dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            self.pose_view = torch.empty((4, 4), **f32); self.pose_full = torch.empty((4, 4), **f32)
            self.pose_gview = torch.empty((4, 4), **f32); self.pose_gproj = torch.empty((4, 4), **f32)
            self.pose_scratch_bytes = int(self.lib.r2x_raster_backward_pose_scratch_bytes(P))
            self.pose_scratch = torch.empty(self.pose_scratch_bytes, dtype=torch.uint8, device=dev)
            self.g_omega, self.g_nu = torch.empty_like(corr.omega), torch.empty_like(corr.nu)
        self.pose_adam = []
        for (group, _), p, g in zip(groups, (corr.omega, corr.nu), (self.g_omega, self.g_nu)):
            st = opt.state[p]
            if len(st) == 0:
                st["step"] = torch.tensor(0.0, dtype=torch.float32)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            self.pose_adam.append((group, p, st, g))
        self.pose_groups = (AdamGroup * 2)()
        for k, (group, p, st, g) in enumerate(self.pose_adam):
            a = self.pose_groups[k]
            a.param, a.grad, a.exp_avg, a.exp_avg_sq = p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr()
            a.numel = p.numel()

    def _bind_detector(self, P, B, dev):
        """Buffers of the detector-offset path: the shifted full projections, the offset gradient and its scratch, and
        one Adam group on the detector optimizer's own state tensors."""
        if self.sharded:
            raise RuntimeError("NativeTrainStep: the detector offset is not supported with Gaussian sharding (every rank "
                               "would hold only its shard's part of the gradient sum)")
        det, opt = self.det, self.det_opt
        p = det.offset
        if p.device != dev or p.dtype != torch.float32 or not p.is_contiguous() or tuple(p.shape) != (1,):
            raise RuntimeError(f"NativeTrainStep: the detector offset must be a contiguous float32 [1] on {dev}")
        groups = opt.param_groups
        if len(groups) != 1 or groups[0]["params"] != [p]:
            raise RuntimeError("NativeTrainStep: the detector optimizer must hold one group, [offset]")
        f32 = dict(dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            self.det_full = torch.empty((4, 4) if B == 1 else (B, 4, 4), **f32)
            self.det_grad = torch.empty(1, **f32)
            self.det_scratch_bytes = int(self.lib.r2x_detector_offset_grad_scratch_bytes(P, B))
            self.det_scratch = torch.empty(self.det_scratch_bytes, dtype=torch.uint8, device=dev)
        st = opt.state[p]
        if len(st) == 0:
            st["step"] = torch.tensor(0.0, dtype=torch.float32)
            st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        self.det_adam = (groups[0], p, st)
        self.det_groups = (AdamGroup * 1)()
        a = self.det_groups[0]
        a.param, a.grad, a.exp_avg, a.exp_avg_sq = p.data_ptr(), self.det_grad.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr()
        a.numel = 1

    def _provision(self):
        """Instance capacities for this iteration: both forwards are speculative.  The buffers only ever grow."""
        dev = self.dev
        want_r = _C._Workspace.provision(self.key_r, self.P * self.B, _C.RASTER.seed, speculative=True)
        if want_r > self.cap_r:
            self.cap_r = want_r
            self.binning_r, self.scratch_r = _C.binning_buffer(want_r, dev), _C.RASTER.bwd_scratch(want_r, dev)
        if self.use_tv:
            want_v = _C._Workspace.provision(self.key_v, self.P, _C.VOXEL.seed, speculative=True)
            if want_v > self.cap_v:
                self.cap_v = want_v
                self.binning_v, self.scratch_v = _C.binning_buffer(want_v, dev), _C.VOXEL.bwd_scratch(want_v, dev)

    # ------------------------------------------------------------------ one iteration
    def __call__(self, cam, gt, tv_centre=None, apply_update: bool = True, view: int | None = None,
                 pose_update: bool | None = None, detector_update: bool | None = None):
        """Enqueue one iteration.  `cam`: camera (render_query.render's contract), or a list of B cameras sharing image
        size, field of view and mode; `gt`: [1,H,W] or [H,W] CUDA float32 target ([B,H,W] for B cameras); `tv_centre`:
        3 floats (ignored without TV).  With `pose`: `view` is the camera's row of the PoseCorrection and `pose_update`
        (default: `apply_update`) whether the pose Adam steps; with `detector`, `detector_update` (default: `apply_update`)
        whether the offset's Adam steps.  Returns {"render", "radii", "viewspace_grad", "loss"
        (device [3]: L1, SSIM, image total; [B,3] for B cameras), "tv" (device [1] or None)} -- views of buffers that
        the next call overwrites."""
        self.check()                                            # the previous iteration (one late; no stall)
        if isinstance(cam, (list, tuple)):
            if not cam:
                raise ValueError("NativeTrainStep: empty camera list")
            cam = cam[0] if len(cam) == 1 else list(cam)
        B = len(cam) if isinstance(cam, list) else 1
        c0 = cam[0] if B > 1 else cam
        H, W = int(c0.image_height), int(c0.image_width)
        if B > 1:
            key = lambda c: (int(c.image_height), int(c.image_width), int(c.mode), float(c.FoVx), float(c.FoVy))
            if any(key(c) != key(c0) for c in cam[1:]):
                raise ValueError("NativeTrainStep: the cameras of a batch must share image size, field of view and mode")
        if self._bound != self._signature(H, W, B):
            self._bind(H, W, B)
        if self.P == 0 and not self.sharded:
            raise RuntimeError("NativeTrainStep: empty model")
        # an EMPTY SHARD of a Gaussian-sharded run goes through the same sequence: the library calls are no-ops that
        # produce a zero image / volume (and zero status words), and the rank takes part in both exchanges with the same
        # buffer sizes as its peers
        pose_args = None
        if self.pose is not None:
            if view is None or not 0 <= int(view) < self.n_views:
                raise ValueError(f"NativeTrainStep: pose refinement needs the view index (0..{self.n_views - 1}), got {view}")
            pose_args = (int(view), bool(apply_update if pose_update is None else pose_update))
        det_update = None
        if self.det is not None:
            det_update = bool(apply_update if detector_update is None else detector_update)
        args = (cam, gt, None if tv_centre is None else tuple(float(v) for v in tv_centre), bool(apply_update), pose_args,
                det_update)
        self._enqueue(*args)
        return self.result

    def _enqueue(self, cam, gt, tv_centre, apply_update, pose_args, det_update):
        gm, lib, dev, P, H, W, B = self.gm, self.lib, self.dev, self.P, self.H, self.W, self.B
        self._provision()
        c0 = cam[0] if B > 1 else cam
        mode = int(c0.mode)
        if mode == 0:
            tfx = tfy = 1.0
        elif mode == 1:
            tfx, tfy = math.tan(c0.FoVx * 0.5), math.tan(c0.FoVy * 0.5)
        else:
            raise ValueError("Unsupported mode!")
        gt = gt.reshape(H, W) if B == 1 else gt.reshape(B, H, W)
        if gt.dtype != torch.float32 or not gt.is_contiguous() or gt.device != dev:
            gt = gt.to(device=dev, dtype=torch.float32).contiguous()
        if B > 1:
            torch.stack([c.world_view_transform for c in cam], out=self.views)
            torch.stack([c.full_proj_transform for c in cam], out=self.projs)
            view, proj, campos = self.views, self.projs, None
        else:
            view, proj, campos = cam.world_view_transform, cam.full_proj_transform, cam.camera_center
        act = C.byref(self.act)
        sm = self.scale_modifier
        xyz, dens, scal, rot = gm._xyz, gm._density, gm._scaling, gm._rotation
        with torch.cuda.device(dev):
            st = torch.cuda.current_stream(dev).cuda_stream
            if pose_args is not None:
                # the corrected matrices of this view (the camera centre stays the camera's: the kernels never read it)
                corr = self.pose
                check(lib.r2x_pose_apply(st, corr.omega.data_ptr(), corr.nu.data_ptr(), self.n_views, pose_args[0],
                                         view.data_ptr(), proj.data_ptr(), cam.projection_matrix.data_ptr(),
                                         self.pose_view.data_ptr(), self.pose_full.data_ptr()), "r2x_pose_apply")
                view, proj = self.pose_view, self.pose_full
            if det_update is not None:
                # the shifted full projections of the B views (the view matrices stay the cameras')
                check(lib.r2x_detector_offset_apply(st, self.det.offset.data_ptr(), W, B, proj.data_ptr(),
                                                    self.det_full.data_ptr()), "r2x_detector_offset_apply")
                proj = self.det_full
            if B == 1:
                check(lib.r2x_raster_forward_async_raw(
                    st, P, W, H, xyz.data_ptr(), dens.data_ptr(), scal.data_ptr(), sm, rot.data_ptr(), view.data_ptr(),
                    proj.data_ptr(), campos.data_ptr(), tfx, tfy, mode, self.image.data_ptr(), self.radii.data_ptr(),
                    self.geom.data_ptr(), self.img.data_ptr(), self.binning_r.data_ptr(), self.cap_r,
                    self.status_r.data_ptr(), act), "r2x_raster_forward_async_raw")
            else:
                check(lib.r2x_raster_forward_views_async_raw(
                    st, P, B, W, H, xyz.data_ptr(), dens.data_ptr(), scal.data_ptr(), sm, rot.data_ptr(),
                    view.data_ptr(), proj.data_ptr(), tfx, tfy, mode, self.image.data_ptr(), self.radii.data_ptr(),
                    self.geom.data_ptr(), self.img.data_ptr(), self.binning_r.data_ptr(), self.cap_r,
                    self.status_r.data_ptr(), act), "r2x_raster_forward_views_async_raw")
            image = self.image
            if self.sharded:
                self.flag_r.copy_(self.status_r[1:2])          # my overflow flag rides with the image
                sharded.sharded_sum_(self.image_ext)
                self.status_r[1:2].copy_(self.flag_r)          # ... and comes back as "any rank overflowed"
            if B == 1:
                check(lib.r2x_image_loss(st, H, W, image.data_ptr(), gt.data_ptr(), 1.0, self.lambda_dssim,
                                         self.loss_out.data_ptr(), self.dL_dimage.data_ptr(),
                                         self.loss_scratch.data_ptr(), self.loss_scratch_bytes), "r2x_image_loss")
            else:
                check(lib.r2x_image_loss_views(st, B, H, W, image.data_ptr(), gt.data_ptr(), 1.0, self.lambda_dssim,
                                               self.loss_out.data_ptr(), self.dL_dimage.data_ptr(),
                                               self.loss_scratch.data_ptr(), self.loss_scratch_bytes),
                      "r2x_image_loss_views")
            if self.use_tv:
                nx, ny, nz = self.tv_n
                grid = (nx, ny, nz, self.tv_s[0], self.tv_s[1], self.tv_s[2], tv_centre[0], tv_centre[1], tv_centre[2])
                check(lib.r2x_voxel_forward_async_raw(
                    st, P, *grid, xyz.data_ptr(), dens.data_ptr(), scal.data_ptr(), sm, rot.data_ptr(), self.vol.data_ptr(),
                    self.rx.data_ptr(), self.ry.data_ptr(), self.rz.data_ptr(), self.geom_v.data_ptr(), self.img_v.data_ptr(),
                    self.binning_v.data_ptr(), self.cap_v, self.status_v.data_ptr(), act), "r2x_voxel_forward_async_raw")
                vol = self.vol
                if self.sharded:
                    self.flag_v.copy_(self.status_v[1:2])
                    sharded.sharded_sum_(self.vol_ext)
                    self.status_v[1:2].copy_(self.flag_v)
                check(lib.r2x_tv3d_loss(st, nx, ny, nz, vol.data_ptr(), 1, self.tv_out.data_ptr(), self.dL_dvol.data_ptr(),
                                        self.tv_scratch.data_ptr(), self.tv_scratch_bytes), "r2x_tv3d_loss")
                # B views: the TV term carries weight B lambda_tv (B times the batch mean of the single-view objective)
                self.dL_dvol.mul_(self.lambda_tv if B == 1 else B * self.lambda_tv)
                check(lib.r2x_voxel_backward_raw(
                    st, P, self.cap_v, *grid, xyz.data_ptr(), scal.data_ptr(), sm, rot.data_ptr(), self.rx.data_ptr(),
                    self.ry.data_ptr(), self.rz.data_ptr(), self.geom_v.data_ptr(), self.binning_v.data_ptr(),
                    self.img_v.data_ptr(), self.scratch_v.data_ptr(), self.dL_dvol.data_ptr(), self.gdv.data_ptr(),
                    self.g3v.data_ptr(), self.gcovv.data_ptr(), self.gsv.data_ptr(), self.grv.data_ptr(), act),
                    "r2x_voxel_backward_raw")
            if B > 1:
                check(lib.r2x_raster_backward_views_raw(
                    st, P, B, self.cap_r, W, H, xyz.data_ptr(), scal.data_ptr(), sm, rot.data_ptr(), view.data_ptr(),
                    proj.data_ptr(), tfx, tfy, self.radii.data_ptr(), self.geom.data_ptr(), self.binning_r.data_ptr(),
                    self.img.data_ptr(), self.scratch_r.data_ptr(), self.dL_dimage.data_ptr(), self.g2.data_ptr(),
                    self.gd.data_ptr(), self.g3.data_ptr(), self.gcov.data_ptr(), self.gs.data_ptr(), self.gr.data_ptr(),
                    mode, act), "r2x_raster_backward_views_raw")
            elif pose_args is None:
                check(lib.r2x_raster_backward_raw(
                    st, P, self.cap_r, W, H, xyz.data_ptr(), scal.data_ptr(), sm, rot.data_ptr(), view.data_ptr(),
                    proj.data_ptr(), campos.data_ptr(), tfx, tfy, self.radii.data_ptr(), self.geom.data_ptr(),
                    self.binning_r.data_ptr(), self.img.data_ptr(), self.scratch_r.data_ptr(), self.dL_dimage.data_ptr(),
                    self.g2.data_ptr(), self.gd.data_ptr(), self.g3.data_ptr(), self.gcov.data_ptr(), self.gs.data_ptr(),
                    self.gr.data_ptr(), mode, act), "r2x_raster_backward_raw")
            else:
                # the same per-Gaussian gradients, bit for bit, plus dL/d(view, full), chained to the view's twist
                check(lib.r2x_raster_backward_pose(
                    st, P, self.cap_r, W, H, xyz.data_ptr(), scal.data_ptr(), sm, rot.data_ptr(), None, view.data_ptr(),
                    proj.data_ptr(), campos.data_ptr(), tfx, tfy, self.radii.data_ptr(), self.geom.data_ptr(),
                    self.binning_r.data_ptr(), self.img.data_ptr(), self.scratch_r.data_ptr(), self.dL_dimage.data_ptr(),
                    self.g2.data_ptr(), self.gd.data_ptr(), None, self.g3.data_ptr(), self.gcov.data_ptr(),
                    self.gs.data_ptr(), self.gr.data_ptr(), mode, 0, act, self.pose_gview.data_ptr(),
                    self.pose_gproj.data_ptr(), self.pose_scratch.data_ptr(), self.pose_scratch_bytes),
                    "r2x_raster_backward_pose")
                corr = self.pose
                check(lib.r2x_pose_grad(st, corr.omega.data_ptr(), corr.nu.data_ptr(), self.n_views, pose_args[0],
                                        self.pose_anchor, cam.world_view_transform.data_ptr(),
                                        cam.projection_matrix.data_ptr(), self.pose_gview.data_ptr(),
                                        self.pose_gproj.data_ptr(), self.g_omega.data_ptr(), self.g_nu.data_ptr()),
                      "r2x_pose_grad")
            if det_update is not None:
                check(lib.r2x_detector_offset_grad(st, P, B, W, self.g2.data_ptr(), self.det_grad.data_ptr(),
                                                   self.det_scratch.data_ptr(), self.det_scratch_bytes),
                      "r2x_detector_offset_grad")
            guard_v = self.status_v.data_ptr() if self.use_tv else None
            if B == 1:
                check(lib.r2x_densify_stats(st, P, self.radii.data_ptr(), self.g2.data_ptr(), gm.max_radii2D.data_ptr(),
                                            gm.xyz_gradient_accum.data_ptr(), gm.denom.data_ptr(),
                                            self.status_r.data_ptr(), guard_v), "r2x_densify_stats")
            else:
                check(lib.r2x_densify_stats_views(st, B, P, self.radii.data_ptr(), self.g2.data_ptr(),
                                                  gm.max_radii2D.data_ptr(), gm.xyz_gradient_accum.data_ptr(),
                                                  gm.denom.data_ptr(), self.status_r.data_ptr(), guard_v),
                      "r2x_densify_stats_views")
            if apply_update:
                steps = set()
                for k, (group, p, stt, _g1, _g2) in enumerate(self.adam):
                    stt["step"] += 1
                    steps.add(int(stt["step"].item()))
                    self.adam_groups[k].lr = float(group["lr"])
                if len(steps) != 1:
                    raise RuntimeError("NativeTrainStep: the four parameters' Adam step counts differ")
                b1, b2 = self.adam[0][0]["betas"]
                check(lib.r2x_adam_step_sum(st, len(self.adam), C.cast(self.adam_groups, C.c_void_p),
                                            C.cast(self.adam_grads2, C.c_void_p) if self.use_tv else None, float(b1),
                                            float(b2), float(self.adam[0][0]["eps"]), steps.pop(), self.status_r.data_ptr(),
                                            guard_v), "r2x_adam_step_sum")
            if pose_args is not None and pose_args[1]:
                # the pose optimizer's step, guarded by BOTH forwards' status words like the Gaussians' own
                steps = set()
                for k, (group, _p, stt, _g) in enumerate(self.pose_adam):
                    stt["step"] += 1
                    steps.add(int(stt["step"].item()))
                    self.pose_groups[k].lr = float(group["lr"])
                if len(steps) != 1:
                    raise RuntimeError("NativeTrainStep: the pose parameters' Adam step counts differ")
                pg = self.pose_adam[0][0]
                b1, b2 = pg["betas"]
                if self.pose_adam[1][0]["betas"] != pg["betas"] or self.pose_adam[1][0]["eps"] != pg["eps"]:
                    raise RuntimeError("NativeTrainStep: the two pose groups must share betas and eps")
                check(lib.r2x_adam_step_sum(st, 2, C.cast(self.pose_groups, C.c_void_p), None, float(b1), float(b2),
                                            float(pg["eps"]), steps.pop(), self.status_r.data_ptr(), guard_v),
                      "r2x_adam_step_sum")
            if det_update:
                # the offset's step, guarded by both forwards' status words like the Gaussians' own
                group, _p, stt = self.det_adam
                stt["step"] += 1
                self.det_groups[0].lr = float(group["lr"])
                b1, b2 = group["betas"]
                check(lib.r2x_adam_step_sum(st, 1, C.cast(self.det_groups, C.c_void_p), None, float(b1), float(b2),
                                            float(group["eps"]), int(stt["step"].item()), self.status_r.data_ptr(),
                                            guard_v), "r2x_adam_step_sum")
            # the status words travel to pinned host memory behind an event; read one iteration late
            host = _C._Workspace.to_host(self.status_r), (_C._Workspace.to_host(self.status_v) if self.use_tv else None)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(dev))
        self._pending = (host, ev, (cam, gt, tv_centre, apply_update, pose_args, det_update))
        self.result = {"render": image, "radii": self.radii, "viewspace_grad": self.g2, "loss": self.loss_out,
                       "tv": self.tv_out if self.use_tv else None}

    def total_loss(self) -> float:
        """Host value of the last iteration's loss (synchronises; logging only): for B views the batch mean of the image
        losses plus lambda_tv TV, comparable with a single-view iteration's."""
        t = float(self.loss_out[2]) if self.B == 1 else float(self.loss_out[:, 2].double().mean())
        return t + self.lambda_tv * float(self.tv_out[0]) if self.use_tv else t

    def check(self):
        """Resolve the last enqueued iteration: update the capacity hints; if a forward had overflowed (its launches
        changed nothing on the device), undo the host-side step count and run that iteration again."""
        if self._pending is None:
            return
        host, ev, args = self._pending
        self._pending = None
        ev.synchronize()
        ov_r = _C._Workspace.read(host[0], self.key_r)[1]
        ov_v = _C._Workspace.read(host[1], self.key_v)[1] if self.use_tv else 0
        if ov_r or ov_v:
            self.repeats += 1
            if self.repeats > 8:
                raise _C.CapacityOverflow("NativeTrainStep: the instance capacity keeps overflowing")
            if args[3]:
                for _group, _p, stt, _g1, _g2 in self.adam:
                    stt["step"] -= 1
            if args[4] is not None and args[4][1]:
                for _group, _p, stt, _g in self.pose_adam:
                    stt["step"] -= 1
            if args[5]:
                self.det_adam[2]["step"] -= 1
            self._enqueue(*args)
            self.check()

    flush = check
