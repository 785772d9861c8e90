"""rasterize(..., features=F) on the GPU: feature maps and their gradients against the colour path and the CPU oracle
(tests/features_oracle.py) — needs an H100."""
from pathlib import Path

import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import rasterize as R
from gaussian_splatting_b200.densify import WeightStats
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera, Gaussians
from oracle import cpu_oracle as orc
from tests import features_oracle as fo
from tests import gradrows, scenes
from tests.gradrows import PARAM_FLOOR, PARAM_RTOL, RENDER_C
from tests.test_gradient_rows_gpu import check_forward, flip_pixels, np_scene

pytestmark = pytest.mark.gpu
SH0 = 0.28209479177387814
REL_TOL = 1e-4


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def bits(a):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# the scenes of tests/golden (tiny, small, deep), without SH: the records' colours are then SH0 * rgb
GOLDEN = {"tiny": ("synth_tiny", 2000, "tiny", (2.0, 0.5, 0.5, 8.0)),
          "small": ("synth_small", 12000, "small", (2.5, 0.5, 0.5, 10.0)),
          "deep": ("synth_deep_nosh", 60000, "small", (2.5, 0.5, 0.5, 10.0))}


def golden_scene(name):
    if name in scenes.FLAGGED:   # SH degree 0 already
        return scenes.flagged_scene(name)
    _, n, res, sig = GOLDEN[name]
    sc = scenes.np_scene(n, res, sh_degree=0, seed=0, view=0, n_views=3, sigma_px=sig)
    sc["sh"] = None
    return sc


def gaussians(sc, requires_grad=True):
    P = {k: to_t(sc[k]).requires_grad_(requires_grad) for k in ("xyz", "rgb", "opacity", "scale", "quaternion")}
    sh = None if sc["sh"] is None else to_t(sc["sh"]).requires_grad_(requires_grad)
    return Gaussians(P["xyz"], P["rgb"], P["opacity"], P["scale"], P["quaternion"], sh)


def render(sc, g, features=None, bg=0.0, masks=True, **kw):
    R.USE_CONTRIBUTION_MASKS = masks
    try:
        return rasterize(g, to_t(sc["T"]), Camera(sc["W"], sc["H"], to_t(sc["K"])), 0.3, 500.0, 100, 3.0, True,
                         torch.full((3,), bg, device=dev()), return_state=True, features=features, **kw)
    finally:
        R.USE_CONTRIBUTION_MASKS = True


def colour_features(g):
    return (g.rgb.detach() * torch.tensor(SH0, dtype=torch.float32, device=dev())).contiguous()


# 1. identity -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masks", [True, False])
@pytest.mark.parametrize("filter3d", [False, True])
@pytest.mark.parametrize("antialiased", [False, True])
@pytest.mark.parametrize("name", list(GOLDEN) + list(scenes.FLAGGED))
def test_colour_features_render_the_image_on_black_bit_for_bit(name, antialiased, filter3d, masks):
    sc = golden_scene(name)
    g = gaussians(sc)
    f3d = torch.full((sc["xyz"].shape[0],), 0.004, device=dev()) if filter3d else None
    img, _, _, fmap, st = render(sc, g, colour_features(g), masks=masks, antialiased=antialiased, filter3d=f3d)
    assert fmap.shape == img.shape
    assert np.array_equal(bits(fmap), bits(img)), int((bits(fmap) != bits(img)).sum())
    assert float(img.detach().abs().max()) > 0
    if name == "deep":  # the weight recurrence's chunk-local index wraps (> 960 splats in the busiest tiles)
        assert int((st.ranges[1:] - st.ranges[:-1]).max()) > 960


@pytest.mark.parametrize("masks", [True, False])
@pytest.mark.parametrize("name", ["tiny"] + list(scenes.FLAGGED))
def test_two_chunk_colour_features_render_the_image_twice(name, masks):
    """F = SH0 * [rgb, rgb], D = 6: channels 3-5 come from the second 4-channel chunk (blockIdx.z = 1, also in the
    exact recompute of flagged pixels) and must equal the image bit for bit, as channels 0-2 do."""
    sc = golden_scene(name)
    g = gaussians(sc)
    F = colour_features(g)
    img, _, _, fmap, _ = render(sc, g, torch.cat([F, F], 1).contiguous(), masks=masks)
    assert fmap.shape == img.shape[:2] + (6,)
    for c0 in (0, 3):
        b = bits(fmap[..., c0:c0 + 3])
        assert np.array_equal(b, bits(img)), (c0, int((b != bits(img)).sum()))
    assert float(img.detach().abs().max()) > 0


# 2. gradient identity ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masks", [True, False])
@pytest.mark.parametrize("name", list(GOLDEN))
def test_feature_loss_gradients_equal_the_image_loss_gradients(name, masks):
    """F = SH0 * rgb, black background: a loss <G, feature_map> gives the geometry the gradients <G, image> does, and
    grad_F is the rgb gradient over SH0, within the atomics noise the golden fixtures record for the reference."""
    sc = golden_scene(name)
    G = to_t(np.random.default_rng(5).standard_normal((sc["H"], sc["W"], 3)).astype(np.float32) / (sc["H"] * sc["W"]))
    g_img = gaussians(sc)
    img, _, uv_i, _ = render(sc, g_img, masks=masks)
    uv_i.retain_grad()
    img.backward(G)
    g_ft = gaussians(sc)
    F = colour_features(g_ft).requires_grad_(True)
    _, _, uv_f, fmap, _ = render(sc, g_ft, F, masks=masks)
    uv_f.retain_grad()
    fmap.backward(G)
    assert not g_ft.rgb.grad.any()
    gd = np.load(Path(__file__).resolve().parent / "golden" / (GOLDEN[name][0] + "_fp32.npz"))
    noise = dict(zip(gd["ref_noise_keys"].tolist(), gd["ref_noise"].tolist()))
    for k in ("xyz", "quaternion", "scale", "opacity"):
        tol = max(REL_TOL, 10 * noise.get("g_" + k, 0.0))
        r = gradrows.global_rel(getattr(g_ft, k).grad, getattr(g_img, k).grad)
        assert r < tol, (k, r, tol)
    assert gradrows.global_rel(uv_f.grad, uv_i.grad) < max(REL_TOL, 10 * noise.get("g_uv", 0.0))
    assert gradrows.global_rel(F.grad * SH0, g_img.rgb.grad) < max(REL_TOL, 10 * noise.get("g_rgb", 0.0))


# 3. oracle parity --------------------------------------------------------------------------------------------------
def feature_run(sc, F, G=None, masks=True):
    """Fused forward, and the backward of <G, feature_map> alone; returns outputs, gaussians, F and the slab rows."""
    g = gaussians(sc)
    Ft = to_t(F).requires_grad_(True)
    out = render(sc, g, Ft, bg=0.5, masks=masks)
    seen = []
    if G is not None:
        proj = next(f for f, i in out[0].grad_fn.next_functions if f is not None and i == 1)
        proj.register_prehook(lambda grad_outputs: seen.append(grad_outputs[1].detach().clone()))
        out[3].backward(to_t(G))
    return out, g, Ft, (seen[0].view(-1, 12).double().cpu().numpy() if seen else None)


@pytest.mark.parametrize("D,scene", [pytest.param(D, None, id=str(D)) for D in (1, 4, 7, 16, 33, 64)]
                         + [pytest.param(D, "exact huge", id=f"exact huge-{D}") for D in (5, 33)])
def test_feature_map_and_gradients_match_the_oracle(D, scene):
    """scene "exact huge": most pixels' feature sums come from feature_pixel_exact_warp, chunks 0 .. (D - 1) / 4."""
    sc = np_scene(2000, "tiny", 3, sigma_px=(2.0, 0.5, 0.5, 8.0)) if scene is None else scenes.flagged_scene(scene)
    N, H, W = sc["xyz"].shape[0], sc["H"], sc["W"]
    rng = np.random.default_rng(D)
    F = rng.standard_normal((N, D)).astype(np.float32)
    o = orc.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], sc["K"],
                      H, W, 0.3, 500.0, 100.0, 3.0, background=np.full(3, 0.5, np.float32))
    (img, mask, uv, fmap, st), _, _, _ = feature_run(sc, F)
    ref = fo.render_forward(o, F[o.keep])
    assert fmap.shape == (H, W, D)
    assert np.abs(fmap.detach().cpu().numpy() - ref).max() <= 1e-4
    G = (rng.standard_normal((H, W, D)) / (H * W)).astype(np.float32)
    Gc = (rng.standard_normal((H, W, 3)) / (H * W)).astype(np.float32)
    flips = flip_pixels(check_forward(img, o, mask, uv), st.w_per_pixel, o, Gc)
    G = np.where(flips[..., None], 0, G).astype(np.float32)
    _, g, Ft, slab = feature_run(sc, F, G)
    d = fo.rasterize_backward(o, F, G)
    allowed = gradrows.flips_allowed(int(o.keep.sum()))
    eps = gradrows.EPS[np.dtype(np.float32)]
    mine = dict(F=Ft.grad.double().cpu().numpy(), opacity=slab[:, 3], uv=slab[:, 4:6], conic=slab[:, 6:9])
    res = [gradrows.render_rows(f"D={D} render {k}", mine[k], getattr(d.render, k), getattr(d.mass, k),
                                RENDER_C["rgb" if k == "F" else k], eps, allowed) for k in ("F", "opacity", "uv", "conic")]
    pr = orc.project_backward(o, np.zeros((N, 3)), mine["opacity"], mine["uv"], mine["conic"])
    res += [gradrows.param_rows(f"D={D} {k}", getattr(g, k).grad, getattr(pr, k), PARAM_RTOL, PARAM_FLOOR, allowed)
            for k in ("xyz", "quaternion", "scale", "opacity")]
    gradrows.assert_all(res)
    assert not g.rgb.grad.any() and (g.sh is None or not g.sh.grad.any())
    assert not Ft.grad[torch.from_numpy(~o.keep).to(dev())].any()


# 4. nothing else moves ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("depth_alpha,antialiased,masks", [(False, False, True), (True, False, True),
                                                          (True, True, False), (False, True, True)])
def test_features_change_no_other_output_or_gradient(depth_alpha, antialiased, masks):
    sc = np_scene(2000, "tiny", 3, sigma_px=(2.0, 0.5, 0.5, 8.0))
    N, H, W = sc["xyz"].shape[0], sc["H"], sc["W"]
    rng = np.random.default_rng(7)
    G = to_t((rng.standard_normal((H, W, 3)) / (H * W)).astype(np.float32))
    Gd = to_t((rng.standard_normal((H, W, 1)) / (H * W)).astype(np.float32))
    outs = []
    for with_f in (False, True):
        g = gaussians(sc)
        ws = WeightStats(N, dev())
        F = to_t(rng.standard_normal((N, 5)).astype(np.float32)).requires_grad_(True) if with_f else None
        out = render(sc, g, F, bg=0.5, masks=masks, render_depth_alpha=depth_alpha, antialiased=antialiased,
                     weight_stats=ws)
        out[2].retain_grad()
        loss = (out[0] * G).sum()
        if depth_alpha:
            loss = loss + (out[3] * Gd).sum() + (out[4] * Gd).sum()
        if with_f:
            loss = loss + (out[-2] * 0.0).sum()
        loss.backward()
        outs.append((out, g, ws))
    (o0, g0, w0), (o1, g1, w1) = outs
    n_maps = 5 if depth_alpha else 3
    for a, b in zip(o0[:n_maps], o1[:n_maps]):
        assert np.array_equal(bits(a.float()), bits(b.float()))
    assert torch.equal(w0.pixel_count, w1.pixel_count) and torch.equal(w0.weight_max, w1.weight_max)
    # the render backward's (and the weight sums') float atomics sum in no fixed order: two identical calls differ in
    # the last bits, so the gradients are compared at that noise; that the feature backward adds nothing for a zero
    # feature loss is checked bit for bit on the slab below
    assert gradrows.global_rel(w1.weight_sum, w0.weight_sum) < 1e-6
    assert gradrows.global_rel(o1[2].grad, o0[2].grad) < 2e-5
    for k in ("xyz", "quaternion", "scale", "opacity", "rgb", "sh"):
        assert gradrows.global_rel(getattr(g1, k).grad, getattr(g0, k).grad) < 2e-5, k
    st = o1[-1]
    slab = torch.randn(N * 12, device=dev())
    before = slab.clone()
    F = to_t(rng.standard_normal((N, 8)).astype(np.float32))
    gF = R.native().fused_render_features_backward(torch.zeros(H, W, 8, device=dev()), slab, st.P, st.records,
                                                   st._ids_sorted, st.ranges, st.n_per_pixel, st.w_per_pixel,
                                                   st.masks, st.keys_sorted, st.id_bits, F)
    assert torch.equal(slab, before) and not gF.any()


# 5. speculation, no_grad, 3 M ---------------------------------------------------------------------------------------
def test_eager_fitting_and_overflowing_speculation_give_the_same_feature_bits():
    sc = np_scene(100_000, "720p", 3, seed=0)
    N = sc["xyz"].shape[0]
    F = to_t(np.random.default_rng(1).standard_normal((N, 6)).astype(np.float32))
    key = (dev().index if dev().index is not None else torch.cuda.current_device(), N, sc["H"], sc["W"])
    R._PAIR_HISTORY.pop(key, None)
    maps = {}
    for name in ("eager", "fitting", "overflow"):
        if name == "overflow":
            R._PAIR_HISTORY[key] = [1000]
        out = render(sc, gaussians(sc), F, bg=0.5)
        assert out[-1].speculation_overflowed == (name == "overflow"), name
        maps[name] = out[3]
    R._PAIR_HISTORY.pop(key, None)
    assert float(maps["eager"].detach().abs().max()) > 0
    for name in ("fitting", "overflow"):
        assert np.array_equal(bits(maps[name]), bits(maps["eager"])), name


@pytest.mark.parametrize("masks", [True, False])
def test_no_grad_call_gives_the_same_feature_map(masks):
    sc = np_scene(2000, "tiny", 3, sigma_px=(2.0, 0.5, 0.5, 8.0))
    F = to_t(np.random.default_rng(2).standard_normal((sc["xyz"].shape[0], 9)).astype(np.float32))
    ref = render(sc, gaussians(sc), F.clone().requires_grad_(True), masks=masks)[3]
    with torch.no_grad():
        out = render(sc, gaussians(sc, requires_grad=False), F, masks=masks)
    assert out[-1].masks.numel() == 0 and not out[3].requires_grad
    assert np.array_equal(bits(out[3]), bits(ref))


def test_headline_scene_with_32_channels():
    g, cam, T, G = scenes.headline_inputs(1080, dev())
    N = g.xyz.shape[0]
    F = torch.randn(N, 32, device=dev(), generator=torch.Generator(device=dev()).manual_seed(3)).requires_grad_(True)
    img, mask, uv, fmap = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, torch.zeros(3, device=dev()), features=F)
    assert fmap.shape == (1080, 1920, 32) and torch.isfinite(fmap).all()
    loss = (img * G).sum() + (fmap * fmap).sum() * 1e-6
    loss.backward()
    assert torch.isfinite(F.grad).all() and F.grad.abs().sum() > 0
    assert not F.grad[mask].any()
    assert torch.isfinite(g.xyz.grad).all()
