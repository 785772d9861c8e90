"""The fp64 photometric-loss oracle (oracle/loss_oracle.py) against the SSIM stand-in the training tools use
(tools/e2e/shims/torchmetrics/image.py) and the trainer's loss expression (splat_py/trainer.py:363-374): same value
in fp64, and the oracle's closed-form gradient equals torch autograd through the stand-in.  CPU only."""
import sys
from pathlib import Path

import pytest
import torch

from oracle import loss_oracle

SHIMS = Path(__file__).resolve().parents[1] / "tools" / "e2e" / "shims"


def _shim_ssim():
    sys.path.insert(0, str(SHIMS))
    try:
        from torchmetrics.image import StructuralSimilarityIndexMeasure
    finally:
        sys.path.remove(str(SHIMS))
    return StructuralSimilarityIndexMeasure(data_range=1.0)


def _trainer_loss(ssim_mod, image, gt, frac):
    """The trainer's expression on [H,W,C] images through the permuted NCHW views, or on [B,C,H,W] directly."""
    if image.dim() == 3:
        p, t = image.unsqueeze(0).permute(0, 3, 1, 2), gt.unsqueeze(0).permute(0, 3, 1, 2)
    else:
        p, t = image, gt
    l1 = torch.nn.functional.l1_loss(image, gt)
    return (1.0 - frac) * l1 + frac * (1.0 - ssim_mod(p, t))


SHAPES = [(11, 11, 3), (12, 30, 3), (37, 53, 3), (2, 3, 12, 15), (2, 1, 20, 17)]


def _pair(shape, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(shape, generator=g, dtype=torch.float64)
    b = (a + 0.2 * torch.randn(shape, generator=g, dtype=torch.float64)).clamp(0, 1)
    return a, b


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("frac", [0.0, 0.2, 1.0])
def test_oracle_forward_equals_shim(shape, frac):
    ssim_mod = _shim_ssim()
    a, b = _pair(shape, 1)
    want = float(_trainer_loss(ssim_mod, a, b, frac))
    loss, l1, s = loss_oracle.forward(a, b, frac)
    assert abs(loss - want) <= 1e-12, (loss, want)
    assert abs(l1 - float(torch.nn.functional.l1_loss(a, b))) <= 1e-14


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("frac", [0.0, 0.2, 1.0])
def test_oracle_gradient_equals_autograd_through_shim(shape, frac):
    ssim_mod = _shim_ssim()
    a, b = _pair(shape, 2)
    x = a.clone().requires_grad_(True)
    (3.0 * _trainer_loss(ssim_mod, x, b, frac)).backward()
    g = loss_oracle.grad(a, b, frac, grad_loss=3.0)
    assert g.shape == a.shape
    err = float((g - x.grad).abs().max())
    assert err <= 1e-10, err


def test_oracle_single_window_is_exact_ssim():
    """11x11: exactly one window origin per channel; identical images give SSIM 1 and zero SSIM gradient."""
    a, _ = _pair((11, 11, 3), 3)
    loss, l1, s = loss_oracle.forward(a, a, 1.0)
    assert abs(s - 1.0) < 1e-14 and l1 == 0.0 and abs(loss) < 1e-14
    assert float(loss_oracle.grad(a, a, 1.0).abs().max()) < 1e-12
