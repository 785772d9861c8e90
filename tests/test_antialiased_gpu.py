"""rasterize(antialiased=True) on the GPU: records, image and gradients against the CPU oracle
(tests/antialiased_oracle.py) — needs an H100."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import rasterize as R
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera
from tests import antialiased_oracle as aao
from tests import gradrows, scenes
from tests.gradrows import PARAM_FLOOR, PARAM_RTOL, RENDER_C
from tests.test_gradient_rows_gpu import check_forward, flip_pixels, gaussians_from, np_scene, ragged

pytestmark = pytest.mark.gpu
BG = 0.5
PARAMS = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")
RENDER_C_DA = dict(RENDER_C, z=16384.0)
R_R2, R_OPA = 2, 3   # record slots: culling bound tau', opacity


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def bits(a):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def run(sc, grads=None, masks=True, depth_alpha=False, **kw):
    """Fused forward (+ backward of <G,image> [+ <Gd,depth> + <Ga,alpha>] when grads is given, any of them None).
    Returns outputs (with the state), the gaussians (with .grad) and the render-stage rows the per-gaussian backward
    got."""
    R.USE_CONTRIBUTION_MASKS = masks
    try:
        g = gaussians_from(sc)
        cam = Camera(sc["W"], sc["H"], to_t(sc["K"]))
        out = rasterize(g, to_t(sc["T"]), cam, 0.3, 500.0, 100, 3.0, True, torch.full((3,), BG, device=dev()),
                        return_state=True, render_depth_alpha=depth_alpha, **kw)
        seen = []
        if grads is not None:
            image = out[0]
            proj = next(f for f, i in image.grad_fn.next_functions if f is not None and i == 1)
            proj.register_prehook(lambda grad_outputs: seen.append(grad_outputs[1].detach().clone()))
            maps = out[:1] + (out[3:5] if depth_alpha else ())
            pairs = [(t, to_t(G).view_as(t)) for t, G in zip(maps, grads) if G is not None]
            torch.autograd.backward([t for t, _ in pairs], [G for _, G in pairs])
    finally:
        R.USE_CONTRIBUTION_MASKS = True
    return out, g, (seen[0].view(-1, 12).double().cpu().numpy() if seen else None)


def oracle(sc):
    return aao.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"],
                         sc["K"], sc["H"], sc["W"], 0.3, 500.0, 100.0, 3.0, background=np.full(3, BG, np.float32))


def upstream3(sc, seed=1):
    H, W = sc["H"], sc["W"]
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal((H, W, 3)) / (3.0 * H * W)).astype(np.float32),
            (rng.standard_normal((H, W)) / (H * W)).astype(np.float32),
            (rng.standard_normal((H, W)) / (H * W)).astype(np.float32))


def small(shd):
    """2000 gaussians at 64 x 64, many of them sub-pixel (screen sigma 0.15 - 8 px)."""
    return np_scene(2000, "tiny", shd, sigma_px=(0.8, 0.8, 0.15, 8.0))


# 1. ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("depth_alpha", [False, True])
def test_antialiased_false_is_the_default(depth_alpha):
    """Image, mask, uv (and depth, alpha) bit for bit.  The render backward accumulates its per-gaussian sums with
    atomic reductions, so two identical calls already differ in the last bits of the gradients: those are compared
    against the spread of two default calls."""
    sc = small(3)
    G = upstream3(sc)
    grads = G if depth_alpha else G[:1]
    out0, g0, rows0 = run(sc, grads, depth_alpha=depth_alpha)
    out1, g1, rows1 = run(sc, grads, depth_alpha=depth_alpha, antialiased=False)
    for a, b in zip(out0[:-1], out1[:-1]):
        assert np.array_equal(bits(a), bits(b)) if a.is_floating_point() else torch.equal(a, b)
    _, g2, rows2 = run(sc, grads, depth_alpha=depth_alpha)
    assert gradrows.global_rel(rows1, rows0) <= max(4 * gradrows.global_rel(rows2, rows0), 2e-5)
    for k in PARAMS:
        spread = gradrows.global_rel(getattr(g2, k).grad, getattr(g0, k).grad)
        assert gradrows.global_rel(getattr(g1, k).grad, getattr(g0, k).grad) <= max(4 * spread, 2e-5), k
    # and the mode does change something
    out2, _, _ = run(sc, None, depth_alpha=depth_alpha, antialiased=True)
    assert not np.array_equal(bits(out0[0]), bits(out2[0]))


# 2. ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shd", [0, 1, 2, 3])
def test_records_and_image_match_the_fp32_oracle(shd):
    """The records' opacity slot (sigmoid(o) * rho) against the fp32 oracle's: bit for bit on at least 85 % of the
    records whose dilated covariance (a, b, c) is bit-identical (measured: 90 %; equal a, c can hide an undilated
    covariance a few ulp apart, which det0's cancellation amplifies: the camera-frame positions come from torch.matmul
    here and from the oracle's own transform there), within 1e-5 overall.  The culling bound tau' is formed from it:
    -1 exactly where it is at most 0.998/255, else gsr_record.cuh cull_tau on the record's own fields to fp32
    rounding, and never looser than the default mode's.  The image equals the oracle's wherever the walk does
    (test_gradient_rows_gpu's rules)."""
    sc = small(shd)
    (img, mask, uv, st), _, _ = run(sc, antialiased=True)
    o = oracle(sc)
    assert (o.rho < 0.5).mean() > 0.1 and (o.rho < 1).all()
    rec = st.records.cpu().numpy()[o.keep]
    a32, c32 = o.conic[:, 0] + np.float32(0.25), o.conic[:, 2] + np.float32(0.25)
    same = (rec[:, 4] == a32) & (rec[:, 5] == o.conic[:, 1] * np.float32(0.5) * 2) & (rec[:, 6] == c32)
    print(f"sh{shd}: covariance bit-identical on {int(same.sum())} of {len(same)} records")
    assert same.sum() > 500   # 921 of 2000 measured on one H100
    ulp = np.abs(bits(rec[:, R_OPA]).astype(np.int64) - bits(o.opacity).astype(np.int64))
    print(f"sh{shd}: opacity bit-identical on {float((ulp[same] == 0).mean()):.4f} of those, max {int(ulp.max())} ulp")
    assert (ulp[same] == 0).mean() >= 0.85
    assert gradrows.global_rel(rec[:, R_OPA], o.opacity) < 1e-5
    r64 = rec.astype(np.float64)   # tau' from the record's own fields
    a, c, bh, det = r64[:, 4], r64[:, 6], 0.5 * r64[:, 5], r64[:, 7]
    lam = 0.5 * (a + c) + np.sqrt(0.25 * (a - c) ** 2 + bh * bh)
    opa = r64[:, R_OPA]
    live = opa > np.float32(0.0039137)
    tau = np.maximum(2 * np.log(np.where(live, opa, 1.0) * np.float32(255.6)), 0) * (1.06 + 4e-6 * lam * lam / det)
    assert (rec[~live, R_R2] == -1).all()
    np.testing.assert_allclose(rec[live, R_R2], tau[live], rtol=2e-5, atol=1e-6)
    (_, _, _, st0), _, _ = run(sc)
    tau0 = st0.records.cpu().numpy()[o.keep][:, R_R2]
    assert (rec[:, R_R2] <= tau0).all() and (rec[:, R_R2] < tau0).mean() > 0.5
    bad = check_forward(img, o, mask, uv)
    assert int(bad.sum()) <= 3


# 3. ------------------------------------------------------------------------------------------------------------
def rows_vs_oracle(tag, sc, masks=True, depth_alpha=False):
    o = oracle(sc)
    G, Gd, Ga = upstream3(sc)
    (img, mask, uv, st), _, _ = run(sc, masks=masks, antialiased=True)
    flips = flip_pixels(check_forward(img, o, mask, uv), st.w_per_pixel, o, G)
    G, Gd, Ga = (np.where(flips[..., None] if a.ndim == 3 else flips, 0, a).astype(np.float32) for a in (G, Gd, Ga))
    if not depth_alpha:
        Gd, Ga = np.zeros_like(Gd), np.zeros_like(Ga)
    _, g, slab = run(sc, (G, Gd, Ga) if depth_alpha else (G,), masks=masks, depth_alpha=depth_alpha, antialiased=True)
    d = aao.rasterize_backward(o, G, Gd, Ga)
    mine = dict(rgb=slab[:, 0:3], opacity=slab[:, 3], uv=slab[:, 4:6], conic=slab[:, 6:9], z=slab[:, 9])
    fields = ("rgb", "opacity", "uv", "conic") + (("z",) if depth_alpha else ())
    allowed = gradrows.flips_allowed(int(o.keep.sum()))
    eps = gradrows.EPS[np.dtype(np.float32)]
    res = [gradrows.render_rows(f"{tag} render {k}", mine[k], getattr(d.render, k), getattr(d.mass, k),
                                RENDER_C_DA[k], eps, allowed) for k in fields]
    pr = aao.project_backward(o, mine["rgb"], mine["opacity"], mine["uv"], mine["conic"],
                              mine["z"] if depth_alpha else None)
    res += [gradrows.param_rows(f"{tag} {k}", getattr(g, k).grad, getattr(pr, k), PARAM_RTOL, PARAM_FLOOR, allowed)
            for k in PARAMS if getattr(g, k) is not None]
    gradrows.assert_all(res)
    for k in PARAMS:   # end to end against the oracle's whole chain, globally
        if getattr(g, k) is not None:
            assert gradrows.global_rel(getattr(g, k).grad, getattr(d, k)) < 5e-4, (tag, k)


def rows_cases():
    cases = [(f"sh{s}", True, False, lambda s=s: small(s)) for s in range(4)]
    cases += [("50x37", True, False, lambda: ragged(50, 37, 1)),
              ("720p", True, False, lambda: np_scene(100_000, "720p", 3, seed=0)),
              ("sh3 no masks", False, False, lambda: small(3)),
              ("sh3 depth+alpha", True, True, lambda: small(3)),
              ("sh0 depth+alpha no masks", False, True, lambda: small(0)),
              ("exact huge", True, False, lambda: scenes.flagged_scene("exact huge"))]
    return cases


@pytest.mark.parametrize("tag,masks,depth_alpha,make", rows_cases(), ids=[c[0] for c in rows_cases()])
def test_gradient_rows(tag, masks, depth_alpha, make):
    rows_vs_oracle(tag, make(), masks=masks, depth_alpha=depth_alpha)


# 4. ------------------------------------------------------------------------------------------------------------
def test_degenerate_gaussians_get_finite_exactly_zero_gradients():
    """Gaussians whose scales underflow (e^-40: the product c0 c2 underflows to 0 in fp32, so det0 <= 0 and
    rho == 0): every gradient is finite, theirs are exactly zero, and the others' are not."""
    sc = small(3)
    deg = np.arange(0, 2000, 7)
    sc["scale"][deg] = -40.0
    o = oracle(sc)
    vis_deg = deg[o.keep[deg]]
    assert len(vis_deg) > 100 and (o.rho[np.flatnonzero(o.keep).searchsorted(vis_deg)] == 0).all()
    G = upstream3(sc)
    (_, _, _, _, _, st), g, _ = run(sc, G, depth_alpha=True, antialiased=True)
    rec = st.records.cpu().numpy()
    assert (rec[vis_deg, R_OPA] == 0).all() and (rec[vis_deg, R_R2] == -1).all()
    for k in PARAMS:
        gk = getattr(g, k).grad.cpu().numpy()
        assert np.isfinite(gk).all(), k
        assert not gk[deg].any(), k
        assert np.abs(np.delete(gk, deg, axis=0)).max() > 0, k


# 5. ------------------------------------------------------------------------------------------------------------
def test_alpha_loss_gives_exactly_zero_colour_gradients():
    sc = small(3)
    _, _, Ga = upstream3(sc)
    _, g, slab = run(sc, (None, None, Ga), depth_alpha=True, antialiased=True)
    assert not g.rgb.grad.any() and not g.sh.grad.any()
    assert g.xyz.grad.abs().max() > 0 and g.opacity.grad.abs().max() > 0 and g.scale.grad.abs().max() > 0
