"""rasterize(absgrad=True) on the GPU: the per-pixel absolute screen-space gradients against the CPU oracle
(tests/absgrad_oracle.py), against their definition, and through densification — needs an H100."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import rasterize as R
from gaussian_splatting_b200 import synth
from gaussian_splatting_b200.densify import AdaptiveDensityControl, DensificationStats, DensifyConfig
from gaussian_splatting_b200.flat_adam import FlatAdam
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera
from tests import absgrad_oracle as abo
from tests import antialiased_oracle as aao
from tests import depth_alpha_oracle as dao
from tests import gradrows, scenes
from tests.gradrows import RENDER_C
from tests.test_gradient_rows_gpu import check_forward, flip_pixels, gaussians_from, np_scene, ragged, stack

pytestmark = pytest.mark.gpu
BG = 0.5
PARAMS = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def bits(a):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def run(sc, grads=None, masks=True, depth_alpha=False, antialiased=False, absgrad=True, far=500.0, retain=False):
    """Fused forward (+ backward of <G,image> [+ <Gd,depth> + <Ga,alpha>] when grads is given, any of them None).
    Returns (outputs incl. the state, gaussians with .grad, uv)."""
    R.USE_CONTRIBUTION_MASKS = masks
    try:
        g = gaussians_from(sc)
        cam = Camera(sc["W"], sc["H"], to_t(sc["K"]))
        out = rasterize(g, to_t(sc["T"]), cam, 0.3, far, 100, 3.0, True, torch.full((3,), BG, device=dev()),
                        return_state=True, render_depth_alpha=depth_alpha, antialiased=antialiased, absgrad=absgrad)
        uv = out[2]
        if retain:
            uv.retain_grad()
        if grads is not None:
            maps = out[:1] + (out[3:5] if depth_alpha else ())
            pairs = [(t, to_t(G).view_as(t)) for t, G in zip(maps, grads) if G is not None]
            torch.autograd.backward([t for t, _ in pairs], [G for _, G in pairs])
    finally:
        R.USE_CONTRIBUTION_MASKS = True
    return out, g, uv


def upstream3(sc, seed=1):
    H, W = sc["H"], sc["W"]
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal((H, W, 3)) / (3.0 * H * W)).astype(np.float32),
            (rng.standard_normal((H, W)) / (H * W)).astype(np.float32),
            (rng.standard_normal((H, W)) / (H * W)).astype(np.float32))


def small(s):
    return np_scene(2000, "tiny", s, sigma_px=(2.0, 0.5, 0.5, 8.0))


# 1. ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,depth_alpha", [("sh3", False), ("deep", False), ("sh3", True)])
def test_outputs_and_gradients_unchanged(kind, depth_alpha):
    """absgrad=True leaves image, mask, uv (and depth / alpha) bit-identical; uv.grad and every parameter gradient
    stay within the run-to-run spread of the atomic reductions (the criterion of the depth/alpha and anti-aliased
    tests)."""
    sc = small(3) if kind == "sh3" else stack(3000, -5.0)
    grads = upstream3(sc) if depth_alpha else upstream3(sc)[:1]
    out0, g0, uv0 = run(sc, grads, depth_alpha=depth_alpha, absgrad=False, retain=True)
    out1, g1, uv1 = run(sc, grads, depth_alpha=depth_alpha, absgrad=True, retain=True)
    n = 5 if depth_alpha else 3
    for a, b in zip(out0[:n], out1[:n]):
        assert np.array_equal(bits(a), bits(b))
    assert out0[-1].uv_absgrad is None and not hasattr(uv0, "absgrad")
    assert uv1.absgrad.shape == uv1.shape and float(uv1.absgrad.max()) > 0
    assert gradrows.global_rel(uv1.grad, uv0.grad) < 2e-5
    for k in PARAMS:
        if getattr(g0, k) is not None:
            assert gradrows.global_rel(getattr(g1, k).grad, getattr(g0, k).grad) < 2e-5, k


# 2. ------------------------------------------------------------------------------------------------------------
def oracle(sc, antialiased):
    f = aao.rasterize if antialiased else dao.rasterize
    return f(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], sc["K"], sc["H"],
             sc["W"], 0.3, 500.0, 100.0, 3.0, background=np.full(3, BG, np.float32))


def absgrad_vs_oracle(tag, sc, masks=True, depth_alpha=False, antialiased=False):
    o = oracle(sc, antialiased)
    G, Gd, Ga = upstream3(sc)
    # pixels where the oracle and the GPU may skip different splats get no upstream gradient (test_gradient_rows_gpu)
    out, _, _ = run(sc, masks=masks, antialiased=antialiased, absgrad=False)
    flips = flip_pixels(check_forward(out[0], o, out[1], out[2]), out[-1].w_per_pixel, o, G)
    G, Gd, Ga = (np.where(flips[..., None] if a.ndim == 3 else flips, 0, a).astype(np.float32) for a in (G, Gd, Ga))
    grads = (G, Gd, Ga) if depth_alpha else (G,)
    out, _, uv = run(sc, grads, masks=masks, depth_alpha=depth_alpha, antialiased=antialiased)
    st = out[-1]
    r = abo.uv_backward(o, G, Gd if depth_alpha else None, Ga if depth_alpha else None)
    assert uv.absgrad is st.uv_absgrad and uv.absgrad.shape == (int(o.keep.sum()), 2)
    allowed = gradrows.flips_allowed(int(o.keep.sum()))
    eps = gradrows.EPS[np.dtype(np.float32)]
    res = gradrows.render_rows(f"{tag} absgrad", uv.absgrad, r.absgrad, r.mass, RENDER_C["uv"], eps, allowed)
    gradrows.assert_all([res])
    assert (r.absgrad > 0).sum() > 0.5 * (r.mass > 0).sum()


SCENES = [(f"sh{s}", lambda s=s: small(s)) for s in range(4)]
SCENES += [("50x37", lambda: ragged(50, 37, 1)), ("17x33", lambda: ragged(17, 33, 2)),
           ("720p", lambda: np_scene(100_000, "720p", 3, seed=0)), ("deep", lambda: stack(3000, -5.0)),
           ("saturated", lambda: stack(6000, 3.0, spread=0.05, scale=(0.03, 0.07)))]
SCENES += [(n, lambda n=n: scenes.flagged_scene(n)) for n in scenes.FLAGGED]   # the exact recompute
VARIANTS = [("masks", dict()), ("no masks", dict(masks=False)), ("depth", dict(depth_alpha=True)),
            ("aa", dict(antialiased=True))]
ROW_CASES = [(f"{s} {v}", make, kw) for s, make in SCENES for v, kw in VARIANTS
             if v in ("masks", "no masks") or s in ("sh0", "sh3", "50x37", "720p", "deep", "saturated")]


@pytest.mark.parametrize("tag,make,kw", ROW_CASES, ids=[c[0] for c in ROW_CASES])
def test_absgrad_rows_against_the_fp32_oracle(tag, make, kw):
    absgrad_vs_oracle(tag, make(), **kw)


# 3. ------------------------------------------------------------------------------------------------------------
def test_absgrad_is_the_sum_of_one_hot_uv_gradients():
    """Without the oracle's absgrad: one backward's uv.absgrad against the sum over all H*W pixels of |uv.grad| of
    backward passes whose upstream gradient is that pixel's alone.  The oracle's m_uv only scales the bound."""
    sc = np_scene(400, "tiny", 0, seed=3, sigma_px=(2.5, 0.5, 0.5, 8.0))
    H, W = 24, 32
    sc = dict(sc, H=H, W=W, K=sc["K"].copy())
    sc["K"][0, 2], sc["K"][1, 2] = W / 2.0, H / 2.0
    G = upstream3(sc)[0]
    _, _, uv = run(sc, (G,))
    ab = uv.absgrad.double().cpu().numpy()
    total = np.zeros_like(ab)
    for p in range(H * W):
        G1 = np.zeros_like(G)
        G1.reshape(-1, 3)[p] = G.reshape(-1, 3)[p]
        _, _, uv1 = run(sc, (G1,), retain=True)
        total += np.abs(uv1.grad.double().cpu().numpy())
    o = oracle(sc, False)
    mass = abo.uv_backward(o, G).mass
    assert ab.shape == mass.shape and (ab > 0).sum() >= 50
    res = gradrows.render_rows("one-hot", ab, total, mass, 256.0, gradrows.EPS[np.dtype(np.float32)],
                               gradrows.flips_allowed(len(ab)))
    gradrows.assert_all([res])


# 4. ------------------------------------------------------------------------------------------------------------
def test_opposite_pulls_cancel_in_uv_grad_but_not_in_absgrad():
    """One isotropic splat centred at (32.5, 32.5), between four pixels, under an upstream gradient mirror-symmetric
    about that centre in x and in y: a pixel's pull on the mean is its offset from the mean times the same factor as
    its mirror image's, so mirrored pixels pull in exactly opposite directions.  Pixels 32 and 33 share a lane, 31..34
    span two lane groups and two tiles, so |uv.grad| ~ 0 only if every partial sum cancels, and absgrad stays clearly
    positive only if the absolute value is taken per pixel, before the lane and group sums."""
    sc = scenes.np_scene(1, "tiny", sh_degree=0, seed=0)
    sc["xyz"] = np.array([[0.0, 0.0, 4.0]], np.float32)
    sc["quaternion"] = np.array([[1.0, 0.0, 0.0, 0.0]], np.float32)
    sc["scale"] = np.log(np.full((1, 3), 0.15, np.float32))
    sc["opacity"] = np.full((1, 1), 1.0, np.float32)
    sc["T"] = np.eye(4, dtype=np.float32)
    sc["K"] = np.array([[64, 0, 32.5], [0, 64, 32.5], [0, 0, 1]], np.float32)
    H, W = sc["H"], sc["W"]
    rng = np.random.default_rng(5)
    q = rng.standard_normal((31, 31)).astype(np.float32) / (H * W)   # pixels 2..32 in x and y
    G2 = np.zeros((H, W), np.float32)
    G2[2:33, 2:33], G2[2:33, 33:64] = q, q[:, ::-1]                  # pixel 65 - x mirrors x about 32.5
    G2[33:64, 2:33], G2[33:64, 33:64] = q[::-1, :], q[::-1, ::-1]
    assert np.array_equal(G2[:, 2:], G2[:, :1:-1]) and np.array_equal(G2[2:, :], G2[:1:-1, :])
    G = np.repeat(G2[:, :, None], 3, axis=2)
    _, _, uv = run(sc, (G,), retain=True)
    ab, gr = uv.absgrad.cpu().numpy(), uv.grad.cpu().numpy()
    print("uv.grad", gr, "absgrad", ab)
    assert uv.shape == (1, 2) and float(uv[0, 0]) == 32.5 and float(uv[0, 1]) == 32.5
    assert (ab > 0).all()
    assert (np.abs(gr) <= 1e-4 * ab).all(), (gr, ab)


# 5. ------------------------------------------------------------------------------------------------------------
def test_absgrad_is_set_by_every_backward_without_retain_grad():
    sc = small(1)
    G = upstream3(sc)[0]
    out, g, uv = run(sc)
    image, st = out[0], out[-1]
    image.backward(to_t(G), retain_graph=True)
    assert uv.grad is None and uv.absgrad is st.uv_absgrad and uv.absgrad.shape == (st.M, 2)
    first = uv.absgrad
    image.backward(to_t(G))
    assert uv.absgrad is st.uv_absgrad and uv.absgrad is not first
    assert gradrows.global_rel(uv.absgrad, first) < 2e-5  # replaced, not accumulated


@pytest.mark.parametrize("depth_alpha", [False, True])
def test_everything_culled_on_the_key_value_fallback(depth_alpha):
    """The empty 4k view with far = inf (separate id array, P = 0), first view (eager pair count) and steady state
    (speculative sizing): uv.absgrad and state.uv_absgrad are [0, 2]."""
    n = 200_000
    sc = scenes.np_scene(n, "4k", sh_degree=0, seed=0)
    sc["xyz"] = sc["xyz"].copy()
    sc["xyz"][:, 2] = -5.0
    G = to_t(synth.make_upstream_grad("4k").numpy())
    key = (dev().index if dev().index is not None else torch.cuda.current_device(), n, sc["H"], sc["W"])
    R._PAIR_HISTORY.pop(key, None)
    for view in ("first view", "steady state"):
        out, g, uv = run(sc, depth_alpha=depth_alpha, far=float("inf"))
        loss = (out[0] * G).sum()
        if depth_alpha:
            loss = loss + out[3].sum() + out[4].sum()
        loss.backward()
        assert uv.shape == (0, 2) and uv.absgrad.shape == (0, 2) and out[-1].uv_absgrad.shape == (0, 2), view
        assert float(g.xyz.grad.abs().max()) == 0.0, view
    assert R._PAIR_HISTORY[key] == [0, 0]
    R._PAIR_HISTORY.pop(key, None)


# 6. ------------------------------------------------------------------------------------------------------------
def test_densification_statistics_on_absgrad():
    sc = small(3)
    K = to_t(sc["K"])
    G = upstream3(sc)[0]
    out, g, uv = run(sc, (G,), retain=True)
    st = out[-1]
    N = sc["xyz"].shape[0]
    vis = st.vis_idx.long()
    # with the flag: the torch expression on uv.absgrad
    ab, xg = uv.absgrad.clone(), g.xyz.grad.clone()
    s1 = DensificationStats(N, dev())
    s1.accumulate(st, uv, g.xyz, K, absgrad=True)
    exp = torch.zeros(N, 2, device=dev())
    exp[vis] += torch.abs(ab * torch.stack([K[0, 0], K[1, 1]]))
    assert torch.equal(s1.uv_grad_accum, exp)
    assert torch.equal(s1.xyz_grad_accum, torch.abs(xg)) and int(s1.grad_accum_count.sum()) == st.M
    # without it: |uv.grad| exactly as before (the reference's expression)
    ug = uv.grad.clone()
    s0 = DensificationStats(N, dev())
    s0.accumulate(st, uv, g.xyz, K)
    exp0 = torch.zeros(N, 2, device=dev())
    ug[:, 0] *= K[0, 0]
    ug[:, 1] *= K[1, 1]
    exp0[vis] += torch.abs(ug)
    assert torch.equal(s0.uv_grad_accum, exp0)
    # a view rendered without absgrad is refused
    out2, g2, uv2 = run(sc, (G,), absgrad=False, retain=True)
    with pytest.raises(RuntimeError):
        DensificationStats(N, dev()).accumulate(out2[-1], uv2, g2.xyz, K, absgrad=True)


def test_adaptive_density_control_runs_on_absgrad_statistics():
    gs = synth.make_gaussians(20_000, "small", sh_degree=3, seed=4, device=dev(), requires_grad=True,
                              sigma_px=(2.5, 0.5, 0.5, 10.0))
    opt = FlatAdam.for_gaussians(gs)
    cam = synth.make_camera("small", device=dev())
    stats = DensificationStats(gs.xyz.shape[0], dev())
    adc = AdaptiveDensityControl(gs, opt, stats, DensifyConfig())
    bg = torch.full((3,), BG, device=dev())
    for view in range(3):
        T = synth.make_pose(view, 3, device=dev())
        image, mask, uv, st = rasterize(gs, T, cam, 0.3, 500.0, 100, 3.0, True, bg, return_state=True, absgrad=True)
        image.backward(synth.make_upstream_grad("small", device=dev()))
        stats.accumulate(st, uv, gs.xyz, cam.K, absgrad=True)
        for f in ("xyz", "rgb", "opacity", "scale", "quaternion", "sh"):
            getattr(gs, f).grad = None
    n0 = gs.xyz.shape[0]
    assert float(stats.uv_grad_accum.max()) > 0
    torch.manual_seed(0)
    info = adc.adaptive_density_control(1500)
    print(info)
    assert info["densify"] > 0 and gs.xyz.shape[0] == info["n_out"] and info["n_in"] == n0
    assert stats.grad_accum_count.shape[0] == gs.xyz.shape[0]
    opt.step(torch.zeros_like(opt.p))
