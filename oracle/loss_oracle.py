"""fp64 CPU restatement of the photometric loss (gaussian_splatting_b200/loss.py, csrc/gsr_loss.cu).  TEST
INFRASTRUCTURE ONLY — imported by tests/ (and nothing in the product path).

Forward: the SSIM stand-in's definition (tools/e2e/shims/torchmetrics/image.py) with the 2-D window as the outer
product of the 1-D taps, valid windows only, and the L1 mean.  Backward in closed form, the way the native backward
computes it: the three partial-derivative maps dS/dmu_p, dS/dE[p^2], dS/dE[pt] at every valid window origin,
blurred back onto the pixels by the transposed (flipped-window) convolution.  Pinned against torch autograd through
the stand-in in tests/test_loss_oracle.py.  Runs on the CPU; the GPU tests also evaluate it in fp64 on the device
(same torch expressions) to keep the 1080p comparisons fast.
"""
import torch
import torch.nn.functional as F

TAPS, SIGMA, K1, K2 = 11, 1.5, 0.01, 0.03


def window():
    """The 11 taps as the stand-in forms them (fp32), widened to fp64."""
    x = torch.arange(TAPS, dtype=torch.float32) - (TAPS - 1) / 2
    g = torch.exp(-(x * x) / (2 * SIGMA * SIGMA))
    return (g / g.sum()).to(torch.float64)


def _nchw(t):
    t = torch.as_tensor(t).to(torch.float64)
    return t.permute(2, 0, 1).unsqueeze(0) if t.dim() == 3 else t


def _window2d(C, device):
    w = window().to(device)
    return (w[:, None] * w[None, :]).expand(C, 1, TAPS, TAPS).contiguous()


def _moments(p, t):
    C = p.shape[1]
    k = _window2d(C, p.device)
    blur = lambda x: F.conv2d(x, k, groups=C)  # noqa: E731
    return blur(p), blur(t), blur(p * p), blur(t * t), blur(p * t)


def forward(pred, target, ssim_frac, data_range=1.0):
    """(loss, L1, SSIM) as python floats; pred / target [H,W,C] or [B,C,H,W].

    1 - S is formed per window from the moments of d = p - t, (mu_d^2 b2 + a1 s_dd) / (b1 b2), since b1 - a1 = mu_d^2
    and b2 - a2 = s_dd: 1 - a1 a2 / (b1 b2) would cancel most digits where the images nearly agree."""
    p, t = _nchw(pred), _nchw(target)
    C = p.shape[1]
    c1, c2 = (K1 * data_range) ** 2, (K2 * data_range) ** 2
    mp, mt, epp, ett, ept = _moments(p, t)
    k = _window2d(C, p.device)
    d = p - t
    mu_d = F.conv2d(d, k, groups=C)
    s_dd = F.conv2d(d * d, k, groups=C) - mu_d * mu_d
    a1 = 2 * mp * mt + c1
    b1 = mp * mp + mt * mt + c1
    b2 = (epp - mp * mp) + (ett - mt * mt) + c2
    one_minus_s = (mu_d * mu_d * b2 + a1 * s_dd) / (b1 * b2)
    l1 = float(d.abs().mean())
    one_minus_ssim = float(one_minus_s.mean())
    return (1.0 - ssim_frac) * l1 + ssim_frac * one_minus_ssim, l1, 1.0 - one_minus_ssim


def grad(pred, target, ssim_frac, data_range=1.0, grad_loss=1.0):
    """d loss / d pred in closed form, in pred's shape ([H,W,C] or [B,C,H,W]), fp64."""
    p, t = _nchw(pred), _nchw(target)
    C = p.shape[1]
    c1, c2 = (K1 * data_range) ** 2, (K2 * data_range) ** 2
    mp, mt, epp, ett, ept = _moments(p, t)
    a1 = 2 * mp * mt + c1
    a2 = 2 * (ept - mp * mt) + c2
    b1 = mp * mp + mt * mt + c1
    b2 = (epp - mp * mp) + (ett - mt * mt) + c2
    den = b1 * b2
    s = a1 * a2 / den
    d_mu = (2 * mt * (a2 - a1) - s * 2 * mp * (b2 - b1)) / den  # dS/dmu_p
    d_pp = -s / b2                                                # dS/dE[p^2]
    d_pt = 2 * a1 / den                                           # dS/dE[pt]
    k = _window2d(C, p.device)
    back = lambda d: F.conv_transpose2d(d, k, groups=C)  # noqa: E731  (flipped-window blur onto the pixels)
    n_valid = s.numel()
    g = grad_loss * ((1.0 - ssim_frac) * torch.sign(p - t) / p.numel()
                     - ssim_frac / n_valid * (back(d_mu) + 2 * p * back(d_pp) + t * back(d_pt)))
    return g[0].permute(1, 2, 0) if torch.as_tensor(pred).dim() == 3 else g
