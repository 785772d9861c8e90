"""Photometric loss kernels in the regimes training spends its steps in — needs a GPU.

tests/test_loss_gpu.py checks the kernels on noisy, uncorrelated pairs (SSIM 0.1-0.8).  Late in training the render is
close to the ground truth: SSIM is 0.9-0.999, 1 - SSIM is 1e-2 to 1e-5, and flat backgrounds match to within one
8-bit step.  There the textbook SSIM arithmetic (E[x^2] - mu^2 in fp32, S rounded per window, D_mu + 2p D_pp + t D_pt
in the backward) loses most of its digits, so these cases hold the kernels to the fp64 oracle (oracle/loss_oracle.py,
evaluated on the fp32 inputs widened to fp64) there: converged smooth images, flat saturated regions, an 8-bit
quantised target, out-of-range predictions, data_range other than 1, identical images (exact), shapes at the tile
edges, 4K, and the fp64 instantiation.  Every input is generated on the device from a seed."""
import math

import pytest
import torch

from gaussian_splatting_b200.loss import photometric_loss, ssim
from oracle import loss_oracle

pytestmark = pytest.mark.gpu

FRACS = [0.0, 0.2, 1.0]
LOSS_TOL = 1e-5       # relative error of the total loss
SSIM_TERM_TOL = 1e-4  # relative error of 1 - SSIM, wherever 1 - SSIM >= 1e-6
GRAD_TOL = 1e-4       # max |d| / max |ref| of the gradient
FP64_TOL = 1e-9


def dev():
    return torch.device("cuda:0")


def _gen(seed):
    return torch.Generator(device=dev()).manual_seed(seed)


def smooth_field(shape, seed, mean, amp=0.1, texture=0.01, dtype=torch.float32):
    """A smooth image around `mean` (two low-frequency waves per channel) plus a small uniform texture.
    shape is [H,W,C] or [B,C,H,W]."""
    g = _gen(seed)
    nchw = len(shape) == 4
    H, W = (shape[2], shape[3]) if nchw else (shape[0], shape[1])
    C = shape[1] if nchw else shape[2]
    B = shape[0] if nchw else 1
    y = torch.arange(H, device=dev(), dtype=torch.float64).view(1, 1, H, 1)
    x = torch.arange(W, device=dev(), dtype=torch.float64).view(1, 1, 1, W)
    ph = 2 * math.pi * torch.rand(3, B, C, 1, 1, generator=g, device=dev(), dtype=torch.float64)
    f = mean + amp * (torch.sin(x / 17 + ph[0]) * torch.cos(y / 23 + ph[1]) + 0.5 * torch.sin((x + y) / 41 + ph[2]))
    f = f + texture * torch.rand(B, C, H, W, generator=g, device=dev(), dtype=torch.float64)
    f = f if nchw else f[0].permute(1, 2, 0)
    return f.to(dtype).contiguous()


def converged(shape, seed, mean, sigma, dtype=torch.float32):
    """pred a smooth field, gt = pred + N(0, sigma)."""
    p = smooth_field(shape, seed, mean, dtype=dtype)
    t = p + sigma * torch.randn(p.shape, generator=_gen(seed + 1000), device=dev(), dtype=dtype)
    return p, t


def flat(shape, seed, level):
    """Both images exactly `level` (0 or 1) except one 8-bit step towards the inside of [0, 1] at ~1% of the target's
    elements."""
    p = torch.full(shape, float(level), device=dev())
    step = torch.rand(shape, generator=_gen(seed), device=dev()) < 0.01
    t = torch.where(step, p + (1.0 / 255 if level == 0 else -1.0 / 255), p)
    return p, t


def quantised(shape, seed):
    """gt the 8-bit quantisation of a smooth field, pred the field itself (within half a step of gt)."""
    p = smooth_field(shape, seed, 0.6, amp=0.25)
    return p, torch.round(255 * p) / 255


def out_of_range(shape, seed):
    """pred spans [-0.2, 1.3] (unclamped colours), gt a clamped and perturbed copy."""
    p = smooth_field(shape, seed, 0.55, amp=0.5, texture=0.0)
    t = (p + 0.01 * torch.randn(p.shape, generator=_gen(seed + 1000), device=dev())).clamp(0, 1)
    return p, t


def _rel(x, ref):
    return float((x.double() - ref.double()).abs().max() / ref.double().abs().max().clamp_min(1e-300))


def _run(p, t, frac, data_range=1.0):
    x = p.detach().clone().requires_grad_(True)
    loss = photometric_loss(x, t, frac, data_range)
    loss.backward()
    with torch.no_grad():
        one_minus_ssim = photometric_loss(p, t, 1.0, data_range)  # 1 - SSIM without rounding SSIM near 1
        s = ssim(p, t, data_range)
    return loss.detach(), x.grad, one_minus_ssim, s


def check(p, t, frac, data_range=1.0, tol=None, label=""):
    """Kernels against the fp64 oracle on the same (widened) inputs: total loss, 1 - SSIM, ssim() and the gradient."""
    fp64 = p.dtype == torch.float64
    loss_tol, term_tol, grad_tol = (FP64_TOL,) * 3 if fp64 else (LOSS_TOL, SSIM_TERM_TOL, GRAD_TOL)
    if tol is not None:
        grad_tol = tol
    loss, grad, one_minus, s = _run(p, t, frac, data_range)
    want, _, s_ref = loss_oracle.forward(p.double(), t.double(), frac, data_range)
    g_ref = loss_oracle.grad(p.double(), t.double(), frac, data_range)
    om_ref = 1.0 - s_ref
    loss_err = abs(float(loss) - want) / abs(want)
    term_err = abs(float(one_minus) - om_ref) / om_ref
    # ssim() returns SSIM in the image dtype: one rounding of a value near 1 on top of the term's error
    ssim_err = abs(float(s) - s_ref)
    ssim_bound = term_tol * om_ref + (0.0 if fp64 else 2.0 ** -24)
    grad_err = _rel(grad, g_ref)
    print(f"{label} frac={frac}: 1-SSIM {om_ref:.3e}, loss rel err {loss_err:.2e}, 1-SSIM rel err {term_err:.2e}, "
          f"ssim() abs err {ssim_err:.2e}, grad max|d|/max|ref| {grad_err:.2e}")
    assert loss_err <= loss_tol, ("loss", loss_err)
    if om_ref >= 1e-6:
        assert term_err <= term_tol, ("1 - SSIM", term_err)
        assert ssim_err <= ssim_bound, ("ssim()", ssim_err, ssim_bound)
    assert grad_err <= grad_tol, ("grad", grad_err)


CONVERGED = [(mean, sigma) for mean in (0.5, 0.85) for sigma in (0.03, 0.01, 0.003)]


@pytest.mark.parametrize("mean,sigma", CONVERGED)
@pytest.mark.parametrize("frac", FRACS)
def test_converged_smooth_images(mean, sigma, frac):
    p, t = converged((180, 240, 3), 11, mean, sigma)
    check(p, t, frac, label=f"converged mean={mean} sigma={sigma}")


@pytest.mark.parametrize("mean,sigma", CONVERGED)
@pytest.mark.parametrize("frac", FRACS)
def test_converged_fp64(mean, sigma, frac):
    p, t = converged((61, 83, 3), 12, mean, sigma, torch.float64)
    check(p, t, frac, label=f"fp64 converged mean={mean} sigma={sigma}")


@pytest.mark.parametrize("level", [0.0, 1.0])
@pytest.mark.parametrize("frac", FRACS)
def test_flat_saturated_regions(level, frac):
    p, t = flat((120, 160, 3), 13, level)
    check(p, t, frac, label=f"flat at {level}")


@pytest.mark.parametrize("frac", FRACS)
def test_quantised_target(frac):
    p, t = quantised((150, 200, 3), 14)
    check(p, t, frac, label="8-bit target")


@pytest.mark.parametrize("frac", FRACS)
def test_out_of_range_prediction(frac):
    p, t = out_of_range((150, 200, 3), 15)
    assert float(p.min()) < -0.1 and float(p.max()) > 1.2
    check(p, t, frac, label="pred in [-0.2, 1.3]")


@pytest.mark.parametrize("data_range", [255.0, 0.5])
@pytest.mark.parametrize("frac", FRACS)
def test_data_range(data_range, frac):
    p, t = converged((120, 160, 3), 16, 0.85, 0.01)
    check(p * data_range, t * data_range, frac, data_range, label=f"data_range={data_range}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("same", ["same_tensor", "bitwise_copy"])
@pytest.mark.parametrize("frac", FRACS)
def test_identical_images_are_exact(dtype, same, frac):
    p = smooth_field((75, 131, 3), 17, 0.85, dtype=dtype)
    t = p if same == "same_tensor" else p.clone()
    loss, grad, one_minus, s = _run(p, t, frac)
    assert float(loss) == 0.0 and float(one_minus) == 0.0, (float(loss), float(one_minus))
    assert float(s) == 1.0, float(s)
    assert bool((grad == 0).all()), float(grad.abs().max())
    x = p.detach().clone().requires_grad_(True)
    ssim(x, t).backward()
    assert bool((x.grad == 0).all()), float(x.grad.abs().max())


# window origins are tiled 32 x 16: H = 16k + 10 / 16k + 11 / 16k + 26 and W = 32k + 10 / 32k + 11 / 32k + 42 put the last
# valid origin on, just past and one halo past a tile edge; H = 11 leaves one row of origins
@pytest.mark.parametrize("H", [11, 42, 59, 74])
@pytest.mark.parametrize("W", [42, 75, 138])
@pytest.mark.parametrize("frac", FRACS)
def test_tile_edge_shapes(H, W, frac):
    p, t = converged((H, W, 3), 18, 0.85, 0.003)
    check(p, t, frac, label=f"{H}x{W}")


@pytest.mark.parametrize("shape", [(3, 1, 59, 75), (3, 4, 59, 75), (42, 75, 1), (42, 75, 4)])
@pytest.mark.parametrize("frac", FRACS)
def test_channels_and_batch(shape, frac):
    p, t = converged(shape, 19, 0.85, 0.003)
    check(p, t, frac, label=str(shape))


@pytest.mark.parametrize("frac", FRACS)
def test_converged_4k(frac):
    p, t = converged((2160, 3840, 3), 20, 0.85, 0.003)
    check(p, t, frac, label="2160x3840")
