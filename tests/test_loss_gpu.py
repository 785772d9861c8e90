"""Photometric loss kernels (csrc/gsr_loss.cu through gaussian_splatting_b200.loss) — needs a GPU.

Checked against (1) the fp64 oracle (oracle/loss_oracle.py), (2) the SSIM stand-in of tools/e2e evaluated the way the
trainer evaluates its loss, (3) gradcheck of the fp64 instantiation; plus layout independence (bit for bit), run to
run determinism, argument errors, and rasterize + loss + backward end to end against the stand-in path."""
import sys
from pathlib import Path

import pytest
import torch

from gaussian_splatting_b200 import synth
from gaussian_splatting_b200.loss import photometric_loss, ssim
from gaussian_splatting_b200.rasterize import rasterize
from oracle import loss_oracle

pytestmark = pytest.mark.gpu

SHIMS = Path(__file__).resolve().parents[1] / "tools" / "e2e" / "shims"
FRACS = [0.0, 0.2, 1.0]


def dev():
    return torch.device("cuda:0")


def _shim_ssim():
    sys.path.insert(0, str(SHIMS))
    try:
        from torchmetrics.image import StructuralSimilarityIndexMeasure
    finally:
        sys.path.remove(str(SHIMS))
    return StructuralSimilarityIndexMeasure(data_range=1.0).to(dev())


def _shim_loss(ssim_mod, image, gt, frac):
    """The trainer's loss through the stand-in (tools/e2e/train_view_parallel.py)."""
    if image.dim() == 3:
        p, t = image.unsqueeze(0).permute(0, 3, 1, 2), gt.unsqueeze(0).permute(0, 3, 1, 2)
    else:
        p, t = image, gt
    l1 = torch.nn.functional.l1_loss(image, gt)
    return (1.0 - frac) * l1 + frac * (1.0 - ssim_mod(p, t))


def _pair(shape, seed, dtype=torch.float32):
    g = torch.Generator(device=dev()).manual_seed(seed)
    a = torch.rand(shape, generator=g, device=dev(), dtype=dtype)
    b = (a + 0.2 * torch.randn(shape, generator=g, device=dev(), dtype=dtype)).clamp(0, 1)
    return a, b


def _fused(a, b, frac, grad_loss=1.0):
    x = a.detach().clone().requires_grad_(True) if a.is_contiguous() else a.detach().requires_grad_(True)
    loss = photometric_loss(x, b, frac)
    (grad_loss * loss).backward()
    return loss.detach(), x.grad


def _rel(x, ref):
    return float((x.double() - ref.double()).abs().max() / ref.double().abs().max().clamp_min(1e-300))


@pytest.mark.parametrize("shape", [(11, 11, 3), (37, 53, 3), (96, 128, 3), (1080, 1920, 3), (2, 3, 40, 50)])
@pytest.mark.parametrize("frac", FRACS)
def test_fp32_kernels_against_fp64_oracle(shape, frac):
    a, b = _pair(shape, 1)
    loss, grad = _fused(a, b, frac)
    want, _, _ = loss_oracle.forward(a.double(), b.double(), frac)
    g_ref = loss_oracle.grad(a.double(), b.double(), frac)
    loss_err = abs(float(loss) - want) / abs(want)
    grad_err = _rel(grad, g_ref)
    print(f"{shape} frac={frac}: loss rel err {loss_err:.2e}, grad max|d|/max|ref| {grad_err:.2e}")
    assert loss_err <= 1e-5 and grad_err <= 1e-4, (loss_err, grad_err)


@pytest.mark.parametrize("frac", FRACS)
def test_against_shim_on_gpu_1080p(frac):
    a, b = _pair((1080, 1920, 3), 2)
    loss, grad = _fused(a, b, frac)
    x = a.clone().requires_grad_(True)
    ref = _shim_loss(_shim_ssim(), x, b, frac)
    ref.backward()
    loss_err = abs(float(loss) - float(ref)) / abs(float(ref))
    grad_err = _rel(grad, x.grad)
    print(f"1080p frac={frac}: loss rel err vs shim {loss_err:.2e}, grad {grad_err:.2e}")
    assert loss_err <= 1e-5 and grad_err <= 1e-4, (loss_err, grad_err)


def _permuted_nchw(shape, seed):
    """A [B,C,H,W] leaf whose memory is BHWC (the trainer's permuted view of the rasterizer's image)."""
    B, C, H, W = shape
    g = torch.Generator(device=dev()).manual_seed(seed)
    base = torch.rand(B, H, W, C, generator=g, device=dev(), dtype=torch.float64)
    return base.permute(0, 3, 1, 2)


@pytest.mark.parametrize("case", ["hwc", "permuted"])
def test_gradcheck_fp64(case):
    if case == "hwc":
        a, b = _pair((13, 17, 3), 3, torch.float64)
    else:
        a = _permuted_nchw((2, 3, 12, 15), 4)
        b = (a + 0.2 * torch.randn(a.shape, device=dev(), dtype=torch.float64)).clamp(0, 1)
        assert not a.is_contiguous()
    x = a.detach().requires_grad_(True)
    for frac in (0.2, 1.0):
        assert torch.autograd.gradcheck(lambda p: photometric_loss(p, b, frac), (x,), eps=1e-6, atol=1e-7, rtol=1e-4)
    assert torch.autograd.gradcheck(lambda p: ssim(p, b), (x,), eps=1e-6, atol=1e-7, rtol=1e-4)


def test_layouts_are_bit_identical_and_gradient_stays_hwc():
    H, W = 75, 131
    a, b = _pair((H, W, 3), 5)
    results = {}
    for name in ("hwc", "permuted", "nchw"):
        if name == "hwc":
            x, t = a.clone().requires_grad_(True), b
        elif name == "permuted":
            x = a.clone().requires_grad_(True)
            xx, t = x.unsqueeze(0).permute(0, 3, 1, 2), b.unsqueeze(0).permute(0, 3, 1, 2)
        else:
            x = a.permute(2, 0, 1).unsqueeze(0).contiguous().requires_grad_(True)
            t = b.permute(2, 0, 1).unsqueeze(0).contiguous()
        loss = photometric_loss(xx if name == "permuted" else x, t, 0.2)
        loss.backward()
        g = x.grad if name != "nchw" else x.grad[0].permute(1, 2, 0)
        results[name] = (loss.detach(), g.contiguous(), ssim(xx if name == "permuted" else x, t).detach())
    for name in ("permuted", "nchw"):
        assert torch.equal(results[name][0], results["hwc"][0]), name
        assert torch.equal(results[name][1], results["hwc"][1]), name
        assert torch.equal(results[name][2], results["hwc"][2]), name

    # the gradient reaching the rasterizer's image node is HWC-contiguous (no copy in its backward)
    cam = synth.make_camera("tiny", device=dev())
    gaus = synth.make_gaussians(500, "tiny", sh_degree=0, seed=0, device=dev(), requires_grad=True)
    image, _, _ = rasterize(gaus, synth.make_pose(device=dev()), cam, 0.3, 500.0, 100, 3.0, True,
                            torch.zeros(3, device=dev()))
    seen = []
    image.register_hook(lambda g: seen.append(g))
    gt = torch.rand(image.shape, device=dev())
    photometric_loss(image, gt, 0.2).backward()
    assert seen and seen[0].shape == image.shape and seen[0].is_contiguous()


def test_deterministic_and_scales_with_upstream_gradient():
    a, b = _pair((540, 960, 3), 6)
    l1, g1 = _fused(a, b, 0.2)
    l2, g2 = _fused(a, b, 0.2)
    assert torch.equal(l1, l2) and torch.equal(g1, g2)
    _, g3 = _fused(a, b, 0.2, grad_loss=3.0)
    ref = 3.0 * g1.double()
    ulp = torch.abs(torch.nextafter(g3, torch.full_like(g3, float("inf"))) - g3).double()
    assert bool(((g3.double() - ref).abs() <= ulp).all())


def test_argument_errors():
    a, b = _pair((20, 20, 3), 7)
    with pytest.raises(ValueError):
        photometric_loss(a[:10], b[:10], 0.2)          # H < 11
    with pytest.raises(ValueError):
        ssim(a[:, :10], b[:, :10])                    # W < 11
    with pytest.raises(ValueError):
        photometric_loss(a, b[:19], 0.2)              # shape mismatch
    with pytest.raises(ValueError):
        photometric_loss(a, b.clone().requires_grad_(True), 0.2)
    with pytest.raises(RuntimeError):
        photometric_loss(a.cpu(), b.cpu(), 0.2)
    with pytest.raises(RuntimeError):
        ssim(a, b.double())


def test_end_to_end_rasterize_loss_backward_matches_shim():
    res = "720p"
    cam = synth.make_camera(res, device=dev())
    T = synth.make_pose(0, 3, device=dev())
    bg = torch.zeros(3, device=dev())
    gaus = synth.make_gaussians(100_000, res, sh_degree=3, seed=0, device=dev(), requires_grad=True)
    fields = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")
    gt = torch.rand(cam.height, cam.width, 3, device=dev(), generator=torch.Generator(device=dev()).manual_seed(9))
    ssim_mod = _shim_ssim()
    out = {}
    for arm in ("shim", "fused"):
        for f in fields:
            getattr(gaus, f).grad = None
        image, _, uv = rasterize(gaus, T, cam, 0.3, 500.0, 100, 3.0, True, bg)
        uv.retain_grad()
        loss = _shim_loss(ssim_mod, image, gt, 0.2) if arm == "shim" else photometric_loss(image, gt, 0.2)
        loss.backward()
        out[arm] = {f: getattr(gaus, f).grad.clone() for f in fields}
        out[arm]["uv"] = uv.grad.clone()
    errs = {k: _rel(out["fused"][k], out["shim"][k]) for k in out["shim"]}
    print("rasterize + loss + backward, max|d|/max|ref| vs the stand-in:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert all(v <= 1e-4 for v in errs.values()), errs
