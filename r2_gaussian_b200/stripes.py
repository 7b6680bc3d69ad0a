"""Ring-artifact correction of projections: the sorting-based stripe removal of Vo, Atwood and Drakopoulos (Optics
Express 26, 2018; sarepy's and algotom's `remove_stripe_based_sorting`) on the GPU, r2x_remove_stripes.

A detector pixel whose gain or offset differs from its neighbours' adds the same error to every view: a vertical stripe
in each sinogram, which every reconstruction turns into a ring.  Each detector column of a sinogram is sorted over the
views, the sorted sinogram is median-filtered across `size` neighbouring columns, and the values go back to the views
they came from.  The output holds only input values, needs no angles or geometry, and `size` 1 returns the input bit
for bit.  include/r2x.h states the model; tests/stripe_oracle.py is its numpy restatement.
"""
from __future__ import annotations

DEFAULT_SIZE = 5            # from the window sweep in DESIGN §8, where sarepy's 21 scored below 5 on every scene
MAX_SIZE = 255
MAX_VIEWS = 8192


def check_size(size: int, W: int | None = None) -> int:
    """`size` as an int, or ValueError unless it is odd, in [1, 255] and (size - 1) / 2 <= W."""
    if isinstance(size, bool) or int(size) != size or size < 1 or size > MAX_SIZE or size % 2 == 0:
        raise ValueError(f"the stripe filter size must be an odd integer in [1, {MAX_SIZE}], got {size}")
    if W is not None and (size - 1) // 2 > W:
        raise ValueError(f"the stripe filter size {size} needs (size - 1) / 2 <= the detector width {W}")
    return int(size)


def scratch_bytes(n: int, H: int, W: int) -> int:
    """r2x_remove_stripes_scratch_bytes: 6 bytes per sample, 0 for a shape the kernel refuses."""
    from ._lib import load

    return int(load().r2x_remove_stripes_scratch_bytes(int(n), int(H), int(W)))


def remove_stripes(projs, size: int = DEFAULT_SIZE, out=None):
    """Stripe removal of a contiguous CUDA float32 [N, H, W] stack (views, detector rows, detector columns) with a
    median window of `size` columns, on the current stream.  `out` is a contiguous float32 [N, H, W] tensor on the
    same device (`projs` itself for in place) or None for a new one; it is returned."""
    import torch

    from ._lib import check, load

    if not isinstance(projs, torch.Tensor) or projs.device.type != "cuda" or projs.dtype != torch.float32 \
            or projs.dim() != 3 or not projs.is_contiguous():
        raise ValueError("remove_stripes: projs must be a contiguous CUDA float32 [N, H, W] tensor")
    n, H, W = (int(s) for s in projs.shape)
    size = check_size(size, W)
    if not 1 <= n <= MAX_VIEWS:
        raise ValueError(f"remove_stripes: {n} views; the kernel takes 1 to {MAX_VIEWS}")
    need = scratch_bytes(n, H, W)
    if need == 0:
        raise ValueError(f"remove_stripes: shape {[n, H, W]} is out of range (H * W must be < 2^31)")
    if out is None:
        out = torch.empty_like(projs)
    if tuple(out.shape) != (n, H, W) or out.dtype != torch.float32 or not out.is_contiguous() \
            or out.device != projs.device:
        raise ValueError(f"remove_stripes: out must be a contiguous float32 {[n, H, W]} tensor on {projs.device}")
    with torch.cuda.device(projs.device):
        scratch = torch.empty(need, dtype=torch.uint8, device=projs.device)
        stream = torch.cuda.current_stream(projs.device).cuda_stream
        rc = load().r2x_remove_stripes(stream, n, H, W, size, projs.data_ptr(), out.data_ptr(), scratch.data_ptr(),
                                       need)
    check(rc, "r2x_remove_stripes")
    return out
