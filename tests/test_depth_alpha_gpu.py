"""rasterize(render_depth_alpha=True) on the GPU: depth and alpha maps and their gradients against the CPU oracle
(tests/depth_alpha_oracle.py) — needs an H100."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import rasterize as R
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera, Gaussians
from tests import depth_alpha_oracle as dao
from tests import gradrows, scenes
from tests.gradrows import PARAM_FLOOR, PARAM_RTOL, RENDER_C
from tests.test_gradient_rows_gpu import check_forward, flip_pixels, gaussians_from, np_scene, ragged, stack

pytestmark = pytest.mark.gpu
BG = 0.5
FIELDS = ("rgb", "opacity", "uv", "conic", "z")
PARAMS = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")
# the z row's sums are alpha*weight*dD: products of the same kind as rgb's, bounded the same way
RENDER_C_DA = dict(RENDER_C, z=16384.0)


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def run(sc, grads=None, masks=True, depth_alpha=True, far=500.0):
    """Fused forward (+ backward of <G,image> + <Gd,depth> + <Ga,alpha> when grads = (G, Gd, Ga), any of them None).
    Returns outputs, the state, the gaussians (with .grad) and the render-stage rows the per-gaussian backward got."""
    R.USE_CONTRIBUTION_MASKS = masks
    try:
        g = gaussians_from(sc)
        cam = Camera(sc["W"], sc["H"], to_t(sc["K"]))
        out = rasterize(g, to_t(sc["T"]), cam, 0.3, far, 100, 3.0, True, torch.full((3,), BG, device=dev()),
                        return_state=True, render_depth_alpha=depth_alpha)
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


def gpu_z(st):
    """Camera-frame z of every gaussian as the tile kernels decode it from the depth keys."""
    k = st.zkey.cpu().numpy().view(np.uint32).astype(np.uint64)
    if st.depth_base:
        bits = k + st.depth_base
    else:
        bits = np.where(k & 0x80000000, k & 0x7FFFFFFF, ~k & 0xFFFFFFFF)
    return bits.astype(np.uint32).view(np.float32)


def oracle(sc):
    return dao.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"],
                         sc["K"], sc["H"], sc["W"], 0.3, 500.0, 100.0, 3.0, background=np.full(3, BG, np.float32))


def upstream3(sc, seed=1):
    H, W = sc["H"], sc["W"]
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal((H, W, 3)) / (3.0 * H * W)).astype(np.float32),
            (rng.standard_normal((H, W)) / (H * W)).astype(np.float32),
            (rng.standard_normal((H, W)) / (H * W)).astype(np.float32))


def bits(a):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# 1. ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["sh3", "deep", "exact huge"])
def test_image_mask_uv_and_image_gradients_unchanged(kind):
    """"exact huge": most pixels come from the recompute, render_pixel_exact_warp_depth against render_pixel_exact_warp."""
    sc = {"sh3": lambda: np_scene(2000, "tiny", 3, sigma_px=(2.0, 0.5, 0.5, 8.0)), "deep": lambda: stack(3000, -5.0),
          "exact huge": lambda: scenes.flagged_scene("exact huge")}[kind]()
    G = upstream3(sc)[0]
    (img0, m0, uv0, st0), g0, _ = run(sc, (G,), depth_alpha=False)
    (img1, m1, uv1, d1, a1, st1), g1, _ = run(sc, (G, None, None))
    assert np.array_equal(bits(img0), bits(img1)) and torch.equal(m0, m1) and np.array_equal(bits(uv0), bits(uv1))
    assert d1.shape == (sc["H"], sc["W"], 1) and a1.shape == (sc["H"], sc["W"], 1)
    for k in PARAMS:
        if getattr(g0, k) is not None:
            assert gradrows.global_rel(getattr(g1, k).grad, getattr(g0, k).grad) < 2e-5, k


# 2. ------------------------------------------------------------------------------------------------------------
def bitwise_cases():
    cases = [(f"sh{s}", lambda s=s: np_scene(2000, "tiny", s, sigma_px=(2.0, 0.5, 0.5, 8.0)), 500.0) for s in range(4)]
    cases += [(f"{H}x{W}", lambda H=H, W=W, s=s: ragged(H, W, s), 500.0)
              for H, W, s in [(50, 37, 1), (17, 33, 2), (1, 64, 0), (64, 1, 3)]]
    cases.append(("deep", lambda: stack(3000, -5.0), 500.0))
    # the exact recompute (tests/scenes.py FLAGGED); far = inf: it decodes z from base-0 (full-range) depth keys
    cases += [(n, lambda n=n: scenes.flagged_scene(n), 500.0) for n in scenes.FLAGGED]
    cases.append(("exact huge far=inf", lambda: scenes.flagged_scene("exact huge"), float("inf")))
    return cases


@pytest.mark.parametrize("name,make,far", bitwise_cases(), ids=[c[0] for c in bitwise_cases()])
def test_depth_and_alpha_match_the_oracle_where_the_walk_does(name, make, far):
    """Where the walk matches the fp32 oracle bit for bit — image, final transmittance weight and splat count — alpha
    is bit-identical on at least 90 % of them and within 1e-6 on all, and depth within 1e-5 relative (the oracle's walk
    fed the z the kernels decode from the keys).  Matching outputs do not pin every blend weight: the oracle's exp2f and
    the GPU's ex2.approx can give a splat's alpha an ulp apart, which the image and the final weight can round away but
    the depth sum (z ~ 2-10, hundreds of splats) accumulates (measured on one H100: z bit-identical, alpha bit-identical
    on every such pixel at 64x64, depth up to 13 ulp off; in the deep stack's >960-splat walks alpha too).
    Elsewhere both agree to fp32 rounding.  The kernels' own depth is checked bit for bit across two z sources in the
    4k test below."""
    sc = make()
    (img, _, _, depth, alpha, st), _, _ = run(sc, far=far)
    assert (st.depth_base == 0) == (far == float("inf"))
    o = oracle(sc)
    z = gpu_z(st)[o.keep]
    assert gradrows.global_rel(z, o.z) < 1e-6
    _, _, _, d_ref, a_ref = dao.render_forward(o.uv, o.opacity, o.rgb, o.conic, z, o.ranges, o.sorted_idx,
                                               o.background, sc["H"], sc["W"])
    same = ((bits(img) == bits(o.image)).all(2) & (bits(st.w_per_pixel) == bits(o.wlast))
            & (st.n_per_pixel.cpu().numpy() == o.n))
    a, d = alpha.detach().cpu().numpy()[..., 0], depth.detach().cpu().numpy()[..., 0]
    print(f"{name}: {int(same.sum())} of {same.size} pixels walk alike; {int((same & (a_ref > 0)).sum())} covered")
    assert (same & (a_ref > 0)).sum() > 0
    a_same = float((bits(a)[same] == bits(a_ref)[same]).mean())
    print(f"{name}: alpha bit-identical on {a_same:.4f} of them")
    assert a_same >= 0.9 and np.abs(a[same] - a_ref[same]).max() <= 1e-6, name
    rel = np.abs(d[same].astype(np.float64) - d_ref[same]) / np.maximum(np.abs(d_ref[same]), 1e-30)
    assert rel.max() <= 1e-5, (name, float(rel.max()))
    assert np.abs(a - a_ref).max() < 1e-5 and gradrows.global_rel(d, d_ref) < 1e-5, name
    if name == "deep":
        assert int(o.n.max()) > 960 and (st.masks.view(-1, 4) != 0).any(0).all()


# 3. / 6. -------------------------------------------------------------------------------------------------------
def rows_vs_oracle(tag, sc, masks=True, negate_depth=False, check=True):
    o = oracle(sc)
    G, Gd, Ga = upstream3(sc)
    (img, mask, uv, depth, alpha, st), _, _ = run(sc, masks=masks)
    # pixels where the oracle and the GPU may skip different splats get no upstream gradient (test_gradient_rows_gpu)
    flips = flip_pixels(check_forward(img, o, mask, uv), st.w_per_pixel, o, G)
    G, Gd, Ga = (np.where(flips[..., None] if a.ndim == 3 else flips, 0, a).astype(np.float32) for a in (G, Gd, Ga))
    _, g, slab = run(sc, (G, Gd, Ga), masks=masks)
    d = dao.rasterize_backward(o, G, -Gd if negate_depth else Gd, Ga)
    mine = dict(rgb=slab[:, 0:3], opacity=slab[:, 3], uv=slab[:, 4:6], conic=slab[:, 6:9], z=slab[:, 9])
    allowed = gradrows.flips_allowed(int(o.keep.sum()))
    eps = gradrows.EPS[np.dtype(np.float32)]
    res = [gradrows.render_rows(f"{tag} render {k}", mine[k], getattr(d.render, k), getattr(d.mass, k),
                                RENDER_C_DA[k], eps, allowed) for k in FIELDS]
    pr = dao.project_backward(o, mine["rgb"], mine["opacity"], mine["uv"], mine["conic"], mine["z"])
    res += [gradrows.param_rows(f"{tag} {k}", getattr(g, k).grad, getattr(pr, k), PARAM_RTOL, PARAM_FLOOR, allowed)
            for k in PARAMS if getattr(g, k) is not None]
    if check:
        gradrows.assert_all(res)
        for k in PARAMS:   # end to end against the oracle's whole chain, globally
            if getattr(g, k) is not None:
                assert gradrows.global_rel(getattr(g, k).grad, getattr(d, k)) < 5e-4, (tag, k)
    return res, o


def rows_cases():
    cases = [(f"sh{s}", True, lambda s=s: np_scene(2000, "tiny", s, sigma_px=(2.0, 0.5, 0.5, 8.0))) for s in range(4)]
    cases += [(f"{H}x{W}", True, lambda H=H, W=W, s=s: ragged(H, W, s))
              for H, W, s in [(50, 37, 1), (17, 33, 2), (1, 64, 0), (64, 1, 3)]]
    cases += [("720p", True, lambda: np_scene(100_000, "720p", 3, seed=0)),
              ("saturated", True, lambda: stack(6000, 3.0, spread=0.05, scale=(0.03, 0.07))),
              ("deep masks", True, lambda: stack(3000, -5.0)), ("deep no masks", False, lambda: stack(3000, -5.0)),
              ("sh3 no masks", False, lambda: np_scene(2000, "tiny", 3, sigma_px=(2.0, 0.5, 0.5, 8.0)))]
    cases += [(n, True, lambda n=n: scenes.flagged_scene(n)) for n in scenes.FLAGGED]
    cases.append(("exact huge no masks", False, lambda: scenes.flagged_scene("exact huge")))
    return cases


@pytest.mark.parametrize("tag,masks,make", rows_cases(), ids=[c[0] for c in rows_cases()])
def test_gradient_rows_with_depth_and_alpha_losses(tag, masks, make):
    rows_vs_oracle(tag, make(), masks=masks)


def test_row_check_sees_the_depth_term():
    """Negative control: the GPU rows against an oracle run with the depth gradient negated fail the row check (every
    render-stage field the depth term enters; the parameter rows are fed the GPU's own render rows)."""
    sc = np_scene(2000, "tiny", 0, sigma_px=(2.0, 0.5, 0.5, 8.0))
    res, _ = rows_vs_oracle("negated dD", sc, negate_depth=True, check=False)
    print("\n".join(map(str, res)))
    failed = {r.name.split()[-1] for r in res[:len(FIELDS)] if not r.ok}
    assert {"z", "opacity", "uv", "conic"} <= failed, failed


# 4. ------------------------------------------------------------------------------------------------------------
def test_z_decoded_from_full_range_keys_and_the_id_array_fallback():
    """4k, 200k gaussians (z in [1, 11]).  far = inf: full 32-bit depth keys, and the id does not fit the key, so the
    kernels read z from the per-gaussian depth keys; far = 500: keys relative to bits(near), id in the key.  Same
    splats, same order: depth and alpha bit-identical."""
    big = scenes.np_scene(200_000, "4k", sh_degree=0, seed=9, view=0, n_views=1)
    (img_a, _, _, d_a, a_a, st_a), _, _ = run(big, far=float("inf"))
    (img_b, _, _, d_b, a_b, st_b), _, _ = run(big, far=500.0)
    assert st_a.depth_base == 0 and st_a.depth_bits == 32 and st_a.keys_sorted.numel() == 0
    assert st_b.depth_base != 0 and st_b.keys_sorted.numel() > 0
    z = gpu_z(st_b)[st_b.visible.cpu().numpy().astype(bool)]
    assert z.min() >= 0.9 and z.max() <= 12.0
    assert np.array_equal(gpu_z(st_a)[st_a.visible.cpu().numpy().astype(bool)], z)
    assert np.array_equal(bits(img_a), bits(img_b))
    assert np.array_equal(bits(a_a), bits(a_b)) and np.array_equal(bits(d_a), bits(d_b))
    assert float(a_a.detach().max()) > 0.5 and float(d_a.detach().max()) > 0.5


# 5. ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["depth", "alpha"])
def test_depth_or_alpha_loss_gives_exactly_zero_colour_gradients(which):
    sc = np_scene(2000, "tiny", 3, sigma_px=(2.0, 0.5, 0.5, 8.0))
    _, Gd, Ga = upstream3(sc)
    _, g, slab = run(sc, (None, Gd, None) if which == "depth" else (None, None, Ga))
    assert not g.rgb.grad.any() and not g.sh.grad.any()
    assert g.xyz.grad.abs().max() > 0 and g.opacity.grad.abs().max() > 0
    assert (np.abs(slab[:, 9]).max() > 0) == (which == "depth")


def test_argument_errors():
    sc = np_scene(200, "tiny", 1)
    cam = Camera(64, 64, to_t(sc["K"]))
    bg = torch.full((3,), BG, device=dev())
    g = gaussians_from(sc)
    with pytest.raises(ValueError):
        rasterize(g, to_t(sc["T"]), cam, 0.3, 500.0, 100, 3.0, False, bg, render_depth_alpha=True)
    g64 = Gaussians(*(t.double() if t is not None else None for t in (g.xyz, g.rgb, g.opacity, g.scale,
                                                                       g.quaternion, None)))
    with pytest.raises(TypeError):
        rasterize(g64, to_t(sc["T"]).double(), Camera(64, 64, to_t(sc["K"]).double()), 0.3, 500.0, 100, 3.0, True,
                  bg.double(), render_depth_alpha=True)
