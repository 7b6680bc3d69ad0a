"""The horizontal detector offset of a scan (centre-of-rotation offset), learned with the scene.

The most common geometry error of a real cone-beam scan is one constant shift of the detector across the rotation
axis, the same in every view.  Unlike a per-view pose error it is well posed in a full rotation: a scene translation
moves the projections sinusoidally with the angle, so no static scene fakes a shift that is constant over all views.

`DetectorOffset(device)` holds `offset`, a leaf tensor [1] (zero at start): s, the shift in detector pixels.

Convention.  s > 0 when the measured images show their content s columns towards LARGER column index than the
nominal geometry predicts.  In scene units at the detector that is s * sDetector[1] / nDetector[1] (`scene_units`).
Scanner files store nDetector / sDetector / dDetector as [v, u] but offDetector as [u, v] (the reference's
scanner yml comments index 0 "u direction"; its ct_utils hands TIGRE geo.offDetector = [cfg[1], cfg[0]], TIGRE's own
[v, u] order).  TIGRE places detector column j at u = dDetector_u * (j - nDetector_u / 2 + 0.5) + offDetector_u, and
image columns run along u (the reference flips only v), so a detector mounted with a horizontal offset d shows its
content d / dDetector_u columns towards SMALLER index: the learned offset corresponds to the scanner file's
offDetector[0] (u; TIGRE's geo.offDetector[1]) = -s * dDetector[1] = -s * sDetector[1] / nDetector[1]
(`scene.detector_shift`'s t_u = -s).  The learned offset is reported, not written back into the scene: put it into the
scanner file and run the projector, FDK and training with `use_offDetector` (`--use_offDetector`).  With
`trainer --use_offDetector` the learned s acts on top of the file's offset.

The map.  The shift moves the detector, not the source: every ray, conic and mu stays the same, and only each
Gaussian's 2-D mean moves by s pixels along u.  Since the rasterizer maps ndc to pixels by ((x / w + 1) W - 1) / 2,
the shifted full projection is the camera's with its x row plus (2 s / W) times its w row (`r2x_detector_offset_apply`,
float64, rounded once; s = 0 gives the camera's matrix bit for bit).  With cull, radii and tile rectangles held fixed
(the convention of every per-Gaussian gradient),

    dL/ds = sum over views and Gaussians of dL/dpix_x = (2 / W) sum dL_dmean2D.x

(`r2x_detector_offset_grad`: a fixed-order float64 sum, bitwise reproducible).  dL_dmean2D is what every raster
backward already writes -- `viewspace_points.grad` of `render()`, the [B, P, 3] one of a batched render -- so no
matrix gradient is needed and batches of views work.

In a custom loop:

    det = DetectorOffset("cuda")
    det_opt = FusedAdam([det.offset], lr=2e-2, eps=1e-15)
    pkg = render(det.camera(cam), gaussians, pipe)
    loss(pkg["render"], gt).backward()
    det.grad_from(pkg["viewspace_points"].grad, cam.image_width)     # writes det.offset.grad
    det_opt.step(); det_opt.zero_grad()

`NativeTrainStep(detector=(det, det_opt))` and `trainer --detector_offset_refine` do the same on the device.  Not
supported together with pose refinement or Gaussian sharding (each rank would see only its shard's part of the sum).
"""
from __future__ import annotations

import copy

import torch

from ._lib import check, load

SIGN_CONVENTION = ("offset_px > 0: the measured projections show their content offset_px columns towards larger column "
                   "index than the nominal geometry predicts; offset_scene = offset_px * sDetector[1] / nDetector[1] "
                   "(scene units at the detector); a scanner file would carry offDetector[0] (u; TIGRE geo.offDetector[1]) = "
                   "-offset_scene")


class DetectorOffset:
    """One horizontal detector offset in pixels, `offset` (leaf float32 tensor [1] on `device`, zero at start)."""

    def __init__(self, device=None):
        self.offset = torch.nn.Parameter(torch.zeros(1, dtype=torch.float32, device=device))

    def _check(self):
        p = self.offset
        if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous() or p.shape != (1,):
            raise RuntimeError("DetectorOffset: offset must be a contiguous float32 CUDA tensor of shape [1]")
        return p.device

    def apply(self, full: torch.Tensor, W: int) -> torch.Tensor:
        """Full projections [..., 4, 4] (n matrices) with the offset applied, in one launch; not differentiable (the
        gradient comes from `grad_from`)."""
        dev = self._check()
        full = full.detach()
        if full.dtype != torch.float32 or full.device != dev or not full.is_contiguous():
            full = full.to(device=dev, dtype=torch.float32).contiguous()
        if full.numel() == 0 or full.numel() % 16 != 0 or full.shape[-2:] != (4, 4):
            raise ValueError("DetectorOffset: full projections must have shape [..., 4, 4]")
        out = torch.empty_like(full)
        with torch.cuda.device(dev):
            check(load().r2x_detector_offset_apply(torch.cuda.current_stream(dev).cuda_stream, self.offset.data_ptr(),
                                                   int(W), full.numel() // 16, full.data_ptr(), out.data_ptr()),
                  "r2x_detector_offset_apply")
        return out

    def camera(self, cam):
        """A copy of `cam` whose full_proj_transform carries the offset (bit for bit the camera's at zero)."""
        return self.cameras([cam])[0]

    def cameras(self, cams):
        """Copies of `cams` (one image width) with the offset applied, in one launch."""
        cams = list(cams)
        if not cams:
            return []
        W = int(cams[0].image_width)
        if any(int(c.image_width) != W for c in cams):
            raise ValueError("DetectorOffset.cameras: the cameras must share one image width")
        full = self.apply(torch.stack([c.full_proj_transform.detach().reshape(4, 4) for c in cams]), W)
        out = []
        for c, f in zip(cams, full):
            o = copy.copy(c)
            o.full_proj_transform = f
            out.append(o)
        return out

    def grad_from(self, dL_dmean2D: torch.Tensor, W: int) -> torch.Tensor:
        """Write offset.grad = (2 / W) sum of dL_dmean2D[..., 0] over [P, 3] (one view) or [B, P, 3] (B views) and
        return it.  `dL_dmean2D` is `viewspace_points.grad` of the render made with `camera()` / `cameras()`."""
        dev = self._check()
        g = dL_dmean2D
        if g is None:
            raise ValueError("DetectorOffset.grad_from: no screen-space gradient (was backward() called?)")
        if g.dim() == 2:
            g = g.unsqueeze(0)
        if g.dim() != 3 or g.shape[2] != 3:
            raise ValueError("DetectorOffset.grad_from: dL_dmean2D must have shape [P, 3] or [B, P, 3]")
        if g.dtype != torch.float32 or g.device != dev or not g.is_contiguous():
            g = g.to(device=dev, dtype=torch.float32).contiguous()
        n, P = int(g.shape[0]), int(g.shape[1])
        lib = load()
        with torch.cuda.device(dev):
            nbytes = int(lib.r2x_detector_offset_grad_scratch_bytes(P, n))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            grad = torch.empty(1, dtype=torch.float32, device=dev)
            check(lib.r2x_detector_offset_grad(torch.cuda.current_stream(dev).cuda_stream, P, n, int(W),
                                               g.data_ptr() if P else None, grad.data_ptr(), scratch.data_ptr(),
                                               nbytes), "r2x_detector_offset_grad")
        self.offset.grad = grad
        return grad

    def scene_units(self, scanner_cfg: dict) -> float:
        """The offset in scene units at the detector: s * sDetector[1] / nDetector[1] (host read)."""
        return float(self.offset.detach()[0]) * float(scanner_cfg["sDetector"][1]) / float(scanner_cfg["nDetector"][1])
