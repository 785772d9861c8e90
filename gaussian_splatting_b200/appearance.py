"""Per-image appearance correction with bilateral grids, on native kernels (csrc/gsr_bilagrid.cu).

Phone and DSLR captures change exposure, white balance and vignetting from image to image.  Without a per-image
photometric model the optimiser bakes those changes into floaters and view-dependent colour.  "Bilateral Guided
Radiance Field Processing" (Wang et al., SIGGRAPH 2024) gives each training image a small bilateral grid of affine
colour transforms, sliced by pixel position and luminance and applied to the rendered image before the loss:

    fx = (j + 0.5) / W (GX - 1),  fy = (i + 0.5) / H (GY - 1),  fz = clamp(0.299 r + 0.587 g + 0.114 b, 0, 1) (L - 1)
    a = trilinear interpolation of grids[id] at (fz, fy, fx),  out = A[:, :3] rgb + A[:, 3],  A = a.reshape(3, 4)

i.e. F.grid_sample(grids[id], (2x - 1, 2y - 1, 2 lum - 1), border padding, align_corners=True), then the affine.
Gradients reach the grids and the image (directly and through the luminance guidance).  The grid gradient is
deterministic: two backward calls give the same bits, and views that share a grid add their gradients in view order.

Grid ids are host values (an int, a sequence or a CPU integer tensor): they are range-checked on the host, so an
out-of-range id never reaches a kernel, and reach the device through a pinned, non-blocking copy, so there is no host
sync.  A CUDA id tensor raises ValueError (checking it would need a sync).  There is no CPU path.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

from . import native

MAX_GUIDANCE = 256  # GSR_BILAGRID_MAX_L
_IDS = {}


def _check_float_cuda(t, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a tensor, got {type(t).__name__}")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")


def _check_grids(grids):
    _check_float_cuda(grids, "grids")
    if grids.dim() != 5 or grids.shape[1] != 12:
        raise ValueError(f"grids must be [N,12,L,GY,GX], got shape {tuple(grids.shape)}")
    if grids.shape[0] < 1 or min(grids.shape[2:]) < 2:
        raise ValueError(f"grids need N >= 1 and L, GY, GX >= 2, got shape {tuple(grids.shape)}")
    if grids.shape[2] > MAX_GUIDANCE:
        raise ValueError(f"at most {MAX_GUIDANCE} guidance levels, got {grids.shape[2]}")


def _host_ids(image_ids, C, N):
    """image_ids as a tuple of C python ints in [0, N)"""
    if isinstance(image_ids, torch.Tensor):
        if image_ids.is_cuda:
            raise ValueError("image_ids must be host values (an int, a sequence or a CPU tensor), not a CUDA tensor: "
                             "an out-of-range id is caught on the host before any launch")
        if image_ids.dtype.is_floating_point or image_ids.dtype.is_complex or image_ids.dtype == torch.bool:
            raise ValueError(f"image_ids must be integers, got {image_ids.dtype}")
        ids = image_ids.reshape(-1).tolist()
    elif isinstance(image_ids, (int, np.integer)):
        ids = [image_ids]
    else:
        ids = list(np.asarray(image_ids).reshape(-1))
        if any(not isinstance(i, (int, np.integer)) or isinstance(i, (bool, np.bool_)) for i in ids):
            raise ValueError(f"image_ids must be integers, got {image_ids!r}")
    ids = tuple(int(i) for i in ids)
    if len(ids) != C:
        raise ValueError(f"expected {C} image id(s), one per view, got {len(ids)}")
    bad = [i for i in ids if not 0 <= i < N]
    if bad:
        raise ValueError(f"image ids {bad} are out of range for {N} grids")
    return ids


def _device_ids(ids, device):
    """int32 [C] on the device, copied from pinned memory without blocking the host and kept per (ids, device)"""
    key = (ids, str(device))
    t = _IDS.get(key)
    if t is None:
        t = torch.tensor(ids, dtype=torch.int32).pin_memory().to(device, non_blocking=True)
        if len(_IDS) >= 1024:
            _IDS.clear()
        _IDS[key] = t
    return t


class _BilateralSlice(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grids, rgb, ids):
        ctx.save_for_backward(grids, rgb)
        ctx.ids = ids
        return native().bilagrid_slice_forward(rgb, grids, ids)

    @staticmethod
    def backward(ctx, grad_out):
        grids, rgb = ctx.saved_tensors
        need_grids, need_rgb = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_grids or need_rgb):
            return None, None, None
        d_rgb, d_grids = native().bilagrid_slice_backward(rgb, grids, ctx.ids, grad_out.float(), need_rgb, need_grids)
        return d_grids, d_rgb, None


class _TotalVariation(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grids):
        ctx.save_for_backward(grids)
        return native().bilagrid_tv_forward(grids)

    @staticmethod
    def backward(ctx, grad_out):
        (grids,) = ctx.saved_tensors
        return native().bilagrid_tv_backward(grids, grad_out.detach().float().reshape(1).contiguous())


def bilateral_slice(grids: torch.Tensor, image: torch.Tensor, image_ids) -> torch.Tensor:
    """Apply each view's bilateral grid to it.

    grids: [N,12,L,GY,GX] float32 on a CUDA device.  image: [H,W,3] (what `rasterize` returns) or [C,H,W,3] (what
    `rasterize_batch` returns), float32 on the grids' device, any strides.  image_ids: the grid of each view as host
    values (an int, a sequence or a CPU integer tensor), C of them.  Returns a contiguous tensor of image's shape,
    differentiable with respect to grids and image."""
    _check_grids(grids)
    _check_float_cuda(image, "image")
    if image.dim() not in (3, 4) or image.shape[-1] != 3:
        raise ValueError(f"image must be [H,W,3] or [C,H,W,3], got shape {tuple(image.shape)}")
    if image.device != grids.device:
        raise ValueError(f"image is on {image.device}, grids on {grids.device}")
    if image.numel() == 0:
        raise ValueError(f"image is empty: shape {tuple(image.shape)}")
    single = image.dim() == 3
    rgb = image.unsqueeze(0) if single else image
    ids = _device_ids(_host_ids(image_ids, rgb.shape[0], grids.shape[0]), grids.device)
    out = _BilateralSlice.apply(grids.contiguous(), rgb, ids)
    return out[0] if single else out


def total_variation(grids: torch.Tensor) -> torch.Tensor:
    """sum over the L, GY and GX axes of mean((G[..., k + 1, ...] - G[..., k, ...])^2), each mean over all N grids,
    as a 0-dim tensor on the device (no host sync); differentiable with respect to grids."""
    _check_grids(grids)
    return _TotalVariation.apply(grids.contiguous())


def identity_grids(num_images: int, grid_x: int = 16, grid_y: int = 16, grid_guidance: int = 8,
                   device=None) -> torch.Tensor:
    """[num_images, 12, grid_guidance, grid_y, grid_x] float32 with A = [I | 0] at every node"""
    ident = torch.tensor([1.0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], dtype=torch.float32, device=device)
    return ident.view(1, 12, 1, 1, 1).repeat(num_images, 1, grid_guidance, grid_y, grid_x)


class BilateralGrid(nn.Module):
    """One bilateral grid per training image, identity-initialised.

    `grids` is an ordinary Parameter: give it its own Adam group (the paper's trainer uses lr 2e-3) and add
    `lambda * tv_loss()` (lambda = 10 there) to the loss."""

    def __init__(self, num_images: int, grid_x: int = 16, grid_y: int = 16, grid_guidance: int = 8, device=None):
        super().__init__()
        if num_images < 1 or min(grid_x, grid_y, grid_guidance) < 2:
            raise ValueError("need num_images >= 1 and grid_x, grid_y, grid_guidance >= 2")
        self.grids = nn.Parameter(identity_grids(num_images, grid_x, grid_y, grid_guidance, device))

    def forward(self, image: torch.Tensor, image_ids) -> torch.Tensor:
        return bilateral_slice(self.grids, image, image_ids)

    def tv_loss(self) -> torch.Tensor:
        return total_variation(self.grids)
