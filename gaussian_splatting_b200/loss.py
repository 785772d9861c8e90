"""The training step's photometric loss on native kernels (csrc/gsr_loss.cu).

The reference trainer's loss (splat_py/trainer.py:363-374)

    loss = (1 - ssim_frac) * L1(image, gt_image) + ssim_frac * (1 - SSIM(image, gt_image))

in one forward kernel and one backward kernel, instead of ~30 torch kernels (the 5-way stack of moment maps, the
depthwise convolutions and their transposes, the elementwise passes, the permutes to and from NCHW).  SSIM is the
11-tap Gaussian window (sigma 1.5) over the windows lying fully inside the image, C1 = (0.01 data_range)^2,
C2 = (0.03 data_range)^2, mean over B*C*(H-10)*(W-10) window origins — the definition the SSIM stand-in of
tools/e2e (torchmetrics' StructuralSimilarityIndexMeasure call signature) implements.

Images are [H,W,C] (the rasterizer's layout) or [B,C,H,W], with any strides: the trainer's
image.unsqueeze(0).permute(0,3,1,2) view is read in place, and the gradient comes back in pred's own layout, so the
rasterizer's backward receives an HWC-contiguous gradient without a copy.  Gradients flow to pred only.  There is no
CPU path: CPU tensors raise RuntimeError.
"""
from __future__ import annotations

import functools

import torch

from . import native

SSIM_TAPS = 11
SSIM_SIGMA = 1.5
SSIM_K1, SSIM_K2 = 0.01, 0.03


@functools.lru_cache(maxsize=None)
def gaussian_window():
    """The 11 window taps, formed in fp32 exactly as the SSIM stand-in forms them (then widened to float)."""
    x = torch.arange(SSIM_TAPS, dtype=torch.float32) - (SSIM_TAPS - 1) / 2
    g = torch.exp(-(x * x) / (2 * SSIM_SIGMA * SSIM_SIGMA))
    g = g / g.sum()
    return tuple(float(v) for v in g)


def _spatial(t: torch.Tensor):
    if t.dim() == 3:
        return t.shape[0], t.shape[1]
    if t.dim() == 4:
        return t.shape[2], t.shape[3]
    raise ValueError(f"expected an [H,W,C] or [B,C,H,W] image, got shape {tuple(t.shape)}")


def _validate(pred: torch.Tensor, target: torch.Tensor):
    if pred.shape != target.shape:
        raise ValueError(f"pred and target shapes differ: {tuple(pred.shape)} vs {tuple(target.shape)}")
    H, W = _spatial(pred)
    if H < SSIM_TAPS or W < SSIM_TAPS:
        raise ValueError(f"SSIM needs H and W of at least {SSIM_TAPS}, got {H}x{W}")
    if target.requires_grad:
        raise ValueError("target must not require grad: the loss has no gradient with respect to the target")


class _PhotometricLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, l1_weight, ssim_weight, data_range, which):
        c1, c2 = (SSIM_K1 * data_range) ** 2, (SSIM_K2 * data_range) ** 2
        out = native().photometric_loss_forward(pred, target, list(gaussian_window()), c1, c2, l1_weight, ssim_weight)
        ctx.save_for_backward(pred, target)
        ctx.params = (c1, c2, l1_weight, ssim_weight)
        return out[which]

    @staticmethod
    def backward(ctx, grad_out):
        if not ctx.needs_input_grad[0]:
            return None, None, None, None, None, None
        pred, target = ctx.saved_tensors
        c1, c2, l1_weight, ssim_weight = ctx.params
        g = grad_out.detach().to(pred.dtype).reshape(1)
        grad = native().photometric_loss_backward(pred, target, list(gaussian_window()), c1, c2, l1_weight,
                                                  ssim_weight, g)
        return grad, None, None, None, None, None


def photometric_loss(image: torch.Tensor, gt_image: torch.Tensor, ssim_frac: float,
                     data_range: float = 1.0) -> torch.Tensor:
    """(1 - ssim_frac) * L1(image, gt_image) + ssim_frac * (1 - SSIM(image, gt_image)) as a 0-dim tensor.

    image / gt_image: [H,W,C] or [B,C,H,W], float32 or float64, on the same CUDA device, any strides.
    Differentiable with respect to `image` only."""
    _validate(image, gt_image)
    frac = float(ssim_frac)
    return _PhotometricLoss.apply(image, gt_image, 1.0 - frac, frac, float(data_range), 0)


def ssim(pred: torch.Tensor, target: torch.Tensor, data_range: float = 1.0) -> torch.Tensor:
    """SSIM (mean over the valid window origins) as a 0-dim tensor, differentiable with respect to `pred`.

    Same kernels as photometric_loss with no L1 term; under torch.no_grad() only the forward kernel runs."""
    _validate(pred, target)
    # loss = -(1 - SSIM) has SSIM's gradient; out[2] is SSIM itself
    return _PhotometricLoss.apply(pred, target, 0.0, -1.0, float(data_range), 2)
