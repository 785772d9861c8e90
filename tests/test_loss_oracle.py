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


def _shifted_loss(p, t, frac, data_range=1.0):
    """The loss evaluated on p - k, t - k (k the target's mean per channel) with k added back to the moments, so that
    the variances are formed from local deviations; differentiable in p.  The window's taps are fp32 values and do not
    sum to exactly 1 (nor does the 2-D window), so k enters through the window's total weight W:
        mu = mu' + k W,  cov(x, y) = cov' + k (1 - W)(mu_x' + mu_y') + k^2 W (1 - W)."""
    p, t = loss_oracle._nchw(p), loss_oracle._nchw(t)
    C = p.shape[1]
    c1, c2 = (loss_oracle.K1 * data_range) ** 2, (loss_oracle.K2 * data_range) ** 2
    k = t.mean(dim=(0, 2, 3), keepdim=True)
    W = float(loss_oracle.window().sum()) ** 2
    mp_, mt_, epp_, ett_, ept_ = loss_oracle._moments(p - k, t - k)
    mp, mt = mp_ + k * W, mt_ + k * W

    def cov(exy, mx, my):
        return exy - mx * my + k * (1 - W) * (mx + my) + k * k * W * (1 - W)

    s_pp, s_tt, s_pt = cov(epp_, mp_, mp_), cov(ett_, mt_, mt_), cov(ept_, mp_, mt_)
    s = (2 * mp * mt + c1) * (2 * s_pt + c2) / ((mp * mp + mt * mt + c1) * (s_pp + s_tt + c2))
    one_minus_ssim = (1 - s).mean()
    return (1.0 - frac) * (p - t).abs().mean() + frac * one_minus_ssim, one_minus_ssim


def _smooth(shape, seed, mean, amp=0.1):
    """A smooth field around `mean` plus a small texture ([H,W,C], fp64)."""
    g = torch.Generator().manual_seed(seed)
    H, W, C = shape
    y = torch.arange(H, dtype=torch.float64)[:, None, None]
    x = torch.arange(W, dtype=torch.float64)[None, :, None]
    ph = 6.283 * torch.rand(3, C, generator=g, dtype=torch.float64)
    f = mean + amp * (torch.sin(x / 17 + ph[0]) * torch.cos(y / 23 + ph[1]) + 0.5 * torch.sin((x + y) / 41 + ph[2]))
    return f + 0.01 * torch.rand(shape, generator=g, dtype=torch.float64), g


def _regime(name):
    """(pred, target, data_range) in the regimes of tests/test_loss_regimes_gpu.py, as fp32 values widened to fp64."""
    shape = (60, 80, 3)
    dr = 1.0
    if name.startswith("converged"):
        _, mean, sigma = name.split("_")
        p, g = _smooth(shape, 1, float(mean))
        t = p + float(sigma) * torch.randn(shape, generator=g, dtype=torch.float64)
    elif name == "flat_sigma1e-4":
        p = torch.full(shape, 0.95, dtype=torch.float64)
        t = p + 1e-4 * torch.randn(shape, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    elif name in ("flat_0", "flat_1"):
        level = float(name[-1])
        p = torch.full(shape, level, dtype=torch.float64)
        step = torch.rand(shape, generator=torch.Generator().manual_seed(3)) < 0.01
        t = torch.where(step, p + (1 / 255 if level == 0 else -1 / 255), p)
    elif name == "quantised":
        p, _ = _smooth(shape, 4, 0.6, amp=0.25)
        t = torch.round(255 * p) / 255
    elif name == "out_of_range":
        p, g = _smooth(shape, 5, 0.55, amp=0.5)
        t = (p + 0.01 * torch.randn(shape, generator=g, dtype=torch.float64)).clamp(0, 1)
    else:  # data_range_255 / data_range_0.5
        dr = float(name.split("_")[-1])
        p, g = _smooth(shape, 6, 0.85)
        t = p + 0.01 * torch.randn(shape, generator=g, dtype=torch.float64)
        p, t = p * dr, t * dr
    return p.float().double(), t.float().double(), dr


REGIMES = ["converged_0.5_0.03", "converged_0.5_0.003", "converged_0.85_0.01", "converged_0.85_0.003", "flat_sigma1e-4",
           "flat_0", "flat_1", "quantised", "out_of_range", "data_range_255", "data_range_0.5"]


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("frac", [0.0, 0.2, 1.0])
def test_oracle_agrees_with_shifted_evaluation(regime, frac):
    """The oracle keeps 1 - SSIM and the gradient to 1e-9 where the images nearly agree: its own cancellation is not
    what a kernel comparison against it measures."""
    p, t, dr = _regime(regime)
    loss, _, s = loss_oracle.forward(p, t, frac, dr)
    x = p.clone().requires_grad_(True)
    ref_loss, ref_term = _shifted_loss(x, t, frac, dr)
    ref_loss.backward()
    ref_loss, ref_term, term = ref_loss.item(), ref_term.item(), 1.0 - s
    assert ref_term > 1e-7, ref_term
    assert abs(term - ref_term) <= 1e-9 * ref_term, (term, ref_term)
    assert abs(loss - ref_loss) <= 1e-9 * abs(ref_loss), (loss, ref_loss)
    g = loss_oracle.grad(p, t, frac, dr)
    err = float((g - x.grad).abs().max() / x.grad.abs().max())
    assert err <= 1e-9, err


def test_oracle_single_window_is_exact_ssim():
    """11x11: exactly one window origin per channel; identical images give SSIM 1 and zero SSIM gradient."""
    a, _ = _pair((11, 11, 3), 3)
    loss, l1, s = loss_oracle.forward(a, a, 1.0)
    assert abs(s - 1.0) < 1e-14 and l1 == 0.0 and abs(loss) < 1e-14
    assert float(loss_oracle.grad(a, a, 1.0).abs().max()) < 1e-12
