"""Bilateral-grid slice and total variation on the GPU: against the fp64 oracle, determinism, batches against single
views, layouts, recovery of a colour transform by optimisation, and the training step end to end."""
import numpy as np
import pytest
import torch

from oracle import bilagrid_oracle as bo

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0") if torch.cuda.is_available() else None


def _grids(N, L, GY, GX, seed=0, noise=0.1):
    from gaussian_splatting_b200.appearance import identity_grids

    g = torch.Generator(device=DEV).manual_seed(seed)
    return identity_grids(N, GX, GY, L, DEV) + noise * torch.randn(N, 12, L, GY, GX, device=DEV, generator=g)


def _image(C, H, W, seed=1, lo=-0.15, hi=1.15):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return lo + (hi - lo) * torch.rand(C, H, W, 3, device=DEV, generator=g)


def _np(t):
    return t.detach().cpu().numpy()


# (N, L, GY, GX, C, H, W, ids)
ORACLE_CASES = {
    "default_1080p": (2, 8, 16, 16, 1, 1080, 1920, [1]),
    "default_small": (3, 8, 16, 16, 2, 37, 53, [2, 0]),
    "odd_1080p": (2, 3, 4, 6, 1, 1080, 1920, [0]),
    "odd_small": (3, 3, 4, 6, 2, 37, 53, [1, 1]),
    "coarse_many_levels": (1, 19, 2, 3, 1, 61, 47, [0]),
    "fine_grid_tiny_image": (2, 5, 33, 40, 2, 9, 13, [0, 1]),
}


@pytest.mark.parametrize("case", list(ORACLE_CASES))
def test_slice_matches_the_fp64_oracle(case):
    from gaussian_splatting_b200.appearance import bilateral_slice

    N, L, GY, GX, C, H, W, ids = ORACLE_CASES[case]
    grids = _grids(N, L, GY, GX).requires_grad_()
    image = _image(C, H, W).requires_grad_()
    # a unit-scale upstream gradient: the guidance term scales it by (L - 1), and the 1e-5 bound is absolute
    g_out = 2 * torch.rand(C, H, W, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7)) - 1
    out = bilateral_slice(grids, image, ids)
    out.backward(g_out)
    ref = bo.slice_forward(_np(grids), _np(image), ids)
    d_rgb, d_grids = bo.slice_backward(_np(grids), _np(image), ids, _np(g_out))
    assert out.is_contiguous() and out.shape == image.shape
    assert np.abs(_np(out) - ref).max() < 1e-5
    assert np.abs(_np(image.grad) - d_rgb).max() < 1e-5
    assert np.abs(_np(grids.grad) - d_grids).max() < 1e-4 * np.abs(d_grids).max()


def test_single_image_input():
    from gaussian_splatting_b200.appearance import bilateral_slice

    grids = _grids(3, 8, 16, 16).requires_grad_()
    image = _image(1, 45, 70)[0].requires_grad_()
    out = bilateral_slice(grids, image, 2)
    assert out.shape == (45, 70, 3) and out.is_contiguous()
    out.square().sum().backward()
    ref = bo.slice_forward(_np(grids), _np(image)[None], [2])[0]
    assert np.abs(_np(out) - ref).max() < 1e-5
    assert image.grad.shape == image.shape
    assert float(grids.grad[:2].abs().max()) == 0.0 and float(grids.grad[2].abs().max()) > 0.0


def test_identity_grids_return_the_input():
    from gaussian_splatting_b200.appearance import BilateralGrid

    m = BilateralGrid(4, device=DEV)
    image = _image(2, 1080, 1920)
    out = m(image, torch.tensor([3, 0]))
    assert float((out - image).abs().max()) < 1e-6


def _fwd_bwd(grids, image, ids, g_out, need=(True, True)):
    from gaussian_splatting_b200.appearance import bilateral_slice

    grids = grids.detach().clone().requires_grad_(need[0])
    image = image.detach().clone().requires_grad_(need[1])
    out = bilateral_slice(grids, image, ids)
    out.backward(g_out)
    return out.detach(), (image.grad if need[1] else None), (grids.grad if need[0] else None)


def test_backward_is_deterministic():
    grids, image = _grids(3, 8, 16, 16), _image(4, 540, 960)
    g_out = torch.randn_like(image)
    a = _fwd_bwd(grids, image, [0, 2, 2, 1], g_out)
    b = _fwd_bwd(grids, image, [0, 2, 2, 1], g_out)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_batch_equals_single_views_bit_for_bit():
    N, C = 6, 4
    grids, image = _grids(N, 8, 16, 16), _image(C, 180, 320)
    g_out = torch.randn_like(image)
    ids = [4, 0, 5, 2]
    out, d_rgb, d_grids = _fwd_bwd(grids, image, ids, g_out)
    for c, n in enumerate(ids):
        o1, r1, g1 = _fwd_bwd(grids, image[c:c + 1], [n], g_out[c:c + 1])
        assert torch.equal(out[c:c + 1], o1)
        assert torch.equal(d_rgb[c:c + 1], r1)
        assert torch.equal(d_grids[n], g1[n])
    for n in set(range(N)) - set(ids):
        assert torch.equal(d_grids[n], torch.zeros_like(d_grids[n]))


def test_duplicate_ids_sum_in_view_order():
    N = 4
    grids, image = _grids(N, 8, 16, 16), _image(3, 180, 320)
    g_out = torch.randn_like(image)
    ids = [1, 3, 1]
    _, _, d_grids = _fwd_bwd(grids, image, ids, g_out)
    single = [_fwd_bwd(grids, image[c:c + 1], [n], g_out[c:c + 1])[2][n] for c, n in enumerate(ids)]
    assert torch.equal(d_grids[1], single[0] + single[2])
    assert torch.equal(d_grids[3], single[1])
    for n in (0, 2):
        assert torch.equal(d_grids[n], torch.zeros_like(d_grids[n]))


def test_gradients_only_where_required():
    grids, image = _grids(2, 8, 16, 16), _image(1, 64, 96)
    g_out = torch.randn_like(image)
    _, r_both, g_both = _fwd_bwd(grids, image, [1], g_out)
    _, r_only, _ = _fwd_bwd(grids, image, [1], g_out, need=(False, True))
    _, _, g_only = _fwd_bwd(grids, image, [1], g_out, need=(True, False))
    assert torch.equal(r_both, r_only) and torch.equal(g_both, g_only)


def test_permuted_layout_gives_the_same_bits():
    grids = _grids(3, 8, 16, 16)
    chw = _image(2, 3 * 97, 131).reshape(2, 3, 97, 131, 3)[..., 0]  # [C,3,H,W] contiguous
    image = chw.permute(0, 2, 3, 1)                                  # [C,H,W,3] view, channel stride H*W
    assert not image.is_contiguous()
    g_out = torch.randn(2, 97, 131, 3, device=DEV)
    g_perm = g_out.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
    a = _fwd_bwd(grids, image, [2, 0], g_perm)
    b = _fwd_bwd(grids, image.contiguous(), [2, 0], g_out)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("shape", [(1, 12, 8, 16, 16), (300, 12, 8, 16, 16), (3, 12, 3, 4, 6)])
def test_total_variation_matches_fp64_and_is_deterministic(shape):
    from gaussian_splatting_b200.appearance import total_variation

    grids = _grids(shape[0], *shape[2:], noise=0.3).requires_grad_()
    tv = total_variation(grids)
    assert tv.dim() == 0 and tv.is_cuda
    g64 = grids.detach().double().requires_grad_()
    ref = bo.total_variation(g64)
    ref.backward()
    assert abs(float(tv) - float(ref)) <= 1e-6 * abs(float(ref))
    (2.5 * tv).backward()
    assert float((grids.grad.double() - 2.5 * g64.grad).abs().max()) <= 1e-6 * float((2.5 * g64.grad).abs().max())
    grad1 = grids.grad.clone()
    grids.grad = None
    tv2 = total_variation(grids)
    (2.5 * tv2).backward()
    assert torch.equal(tv, tv2) and torch.equal(grids.grad, grad1)


def test_optimisation_recovers_a_colour_transform():
    from gaussian_splatting_b200.appearance import BilateralGrid

    torch.manual_seed(0)
    H, W = 96, 128
    rgb = (torch.rand(H, W, 3) * 0.8 + 0.1).to(DEV)
    M = torch.tensor([[1.15, 0.05, 0.0], [0.0, 0.95, 0.03], [0.02, 0.0, 0.85]], device=DEV)
    b = torch.tensor([0.03, -0.02, 0.05], device=DEV)
    target = rgb @ M.T + b
    m = BilateralGrid(1, 16, 16, 8, device=DEV)
    opt = torch.optim.Adam(m.parameters(), lr=2e-3)
    first = None
    for _ in range(200):
        loss = (m(rgb, 0) - target).abs().mean()
        first = float(loss) if first is None else first
        opt.zero_grad()
        loss.backward()
        opt.step()
    last = float((m(rgb, 0) - target).abs().mean())
    assert last < first / 20, (first, last)


def test_training_step_end_to_end_matches_the_grid_sample_formulation():
    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.appearance import BilateralGrid
    from gaussian_splatting_b200.loss import photometric_loss
    from gaussian_splatting_b200.rasterize import rasterize

    res = "small"
    cam = synth.make_camera(res, device=DEV)
    T = synth.make_pose(0, 3, device=DEV)
    bg = torch.full((3,), 0.5, device=DEV)
    gt = _image(1, cam.height, cam.width, seed=3, lo=0.0, hi=1.0)[0]
    bgrid = BilateralGrid(2, device=DEV)
    with torch.no_grad():
        bgrid.grids.add_(0.1 * torch.randn(bgrid.grids.shape, device=DEV,
                                           generator=torch.Generator(device=DEV).manual_seed(9)))

    grads = []
    for native_slice in (True, False):
        gaus = synth.make_gaussians(20000, res, sh_degree=3, seed=0, device=DEV, requires_grad=True)
        grids = bgrid.grids.detach().clone().requires_grad_()
        image, _, _ = rasterize(gaus, T, cam, 0.3, 500.0, 100, 3.0, True, bg)
        if native_slice:
            from gaussian_splatting_b200.appearance import bilateral_slice

            out = bilateral_slice(grids, image, 1)
        else:
            out = bo.grid_sample_slice(grids, image[None], [1])[0]
        loss = photometric_loss(out, gt, 0.2)
        loss.backward()
        grads.append({k: getattr(gaus, k).grad.detach().clone()
                      for k in ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")} | {"grids": grids.grad})
    for k, ref in grads[1].items():
        err = float((grads[0][k] - ref).abs().max())
        assert err <= 2e-4 * float(ref.abs().max()), (k, err, float(ref.abs().max()))
