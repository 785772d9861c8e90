"""Mip-Splatting's 3-D filter on the GPU: rasterize(..., filter3d=f) against the CPU oracle (tests/filter3d_oracle.py),
against the baked parameters, and compute_filter3d against the oracle's sampling pass — needs an H100."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import native
from gaussian_splatting_b200 import rasterize as R
from gaussian_splatting_b200 import synth
from gaussian_splatting_b200.densify import AdaptiveDensityControl, DensificationStats, DensifyConfig
from gaussian_splatting_b200.filter3d import bake_filter3d, compute_filter3d
from gaussian_splatting_b200.flat_adam import FlatAdam
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera
from tests import filter3d_oracle as fo
from tests import gradrows, scenes
from tests.gradrows import PARAM_FLOOR, PARAM_RTOL, RENDER_C
from oracle import cpu_oracle as orc
from tests.test_gradient_rows_gpu import gaussians_from, np_scene, ragged
from tests.test_filter3d_oracle import live_filter

pytestmark = pytest.mark.gpu
BG = 0.5
PARAMS = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")
# Row bounds: tests/gradrows.py's constants.  Worst row ratios measured over all cases of test_gradient_rows on one H100
# 80GB HBM3 (400 W power limit): render rgb 0.25, opacity 0.089, uv 0.19, conic 0.17, z 0.0014 (all at 720p, z with
# depth/alpha); parameters xyz 0.0046, quaternion 0.84 (720p), scale 0.25, opacity 0.043, rgb 0.00093, sh 0.012.  No
# row beyond its bound in any case.
RENDER_C_DA = dict(RENDER_C, z=16384.0)
R_R2, R_OPA = 2, 3   # record slots: culling bound tau', opacity


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def bits(a):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def run(sc, grads=None, masks=True, depth_alpha=False, g=None, **kw):
    """Fused forward (+ backward of <G,image> [+ <Gd,depth> + <Ga,alpha>] when grads is given, any of them None).
    Returns outputs (with the state), the gaussians (with .grad) and the render-stage rows the per-gaussian backward
    got."""
    R.USE_CONTRIBUTION_MASKS = masks
    try:
        g = gaussians_from(sc) if g is None else g
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


def device_exp(sc):
    """exp(scale) as the kernels' expf forms it (torch.exp on the device): the host's expf can differ by an ulp, and
    the filter's t_k = v_k / (v_k + f^2) keeps that difference where the unfiltered covariance rounds it away."""
    return torch.exp(to_t(sc["scale"])).cpu().numpy()


def oracle(sc, f, antialiased=False):
    """The fp32 oracle fed the device's exp(s) and sigmoid(o) (torch on the device evaluates them as the kernels do)."""
    sigma = torch.sigmoid(to_t(sc["opacity"]).reshape(-1)).cpu().numpy()
    return fo.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], sc["K"],
                        sc["H"], sc["W"], f, antialiased=antialiased, mh_dist=3.0,
                        background=np.full(3, BG, np.float32), e=device_exp(sc), sigma=sigma)


# Pixels whose colour may differ from the oracle's beyond rounding: threshold flips, where the host's exp2f and the
# device's ex2.approx put an alpha on opposite sides of the 1/255 skip.  The filter lowers most opacities (coef median
# 0.79 on the bench scene), so more splats sit near that threshold than in the default mode: measured 10 such pixels of
# 921 600 at 720p (tests/test_gradient_rows_gpu.py allows 9 there), at most 0 at 64 x 64.  Allowed: max(3, H W / 50 000).
def flips_allowed_px(n_pixels):
    return max(3, n_pixels // 50_000)


def check_forward(image, o, mask=None, uv=None):
    """test_gradient_rows_gpu.check_forward with the allowance above; returns the pixels beyond rounding."""
    if mask is not None:
        assert (mask.cpu().numpy() == o.culling_mask).all(), "culling mask differs from the oracle"
        assert gradrows.global_rel(uv.detach().cpu().numpy(), o.uv) < 1e-6
    diff = np.abs(image.detach().cpu().numpy().astype(np.float64) - o.image).max(2)
    bad = diff > 1e-4 * np.abs(o.image).max()
    print(f"forward: {int(bad.sum())} pixels beyond 1e-4 of {bad.size}")
    assert int(bad.sum()) <= flips_allowed_px(bad.size), f"{int(bad.sum())} pixels beyond 1e-4"
    return bad


def flip_pixels(bad_image, w_gpu, o, G):
    """test_gradient_rows_gpu.flip_pixels with the allowance above: pixels left out of the backward."""
    forward = bad_image | (np.abs(w_gpu.cpu().numpy().astype(np.float64) - o.wlast) > 1e-4)
    near = orc.rasterize_backward(o, G).near
    print(f"pixels left out: {int(forward.sum())} forward, {int(near.sum())} near the threshold, of {near.size}")
    assert int(forward.sum()) <= flips_allowed_px(forward.size), f"{int(forward.sum())} pixels differ in the forward"
    assert int(near.sum()) <= max(3, near.size // 100), f"{int(near.sum())} pixels near the threshold"
    return forward | near


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
@pytest.mark.parametrize("antialiased", [False, True], ids=["plain", "antialiased"])
@pytest.mark.parametrize("depth_alpha", [False, True])
def test_no_filter_and_zero_filter_are_the_default(depth_alpha, antialiased):
    """filter3d=None and filter3d=zeros: image, mask, uv (depth, alpha) and records bit for bit.  The render backward
    accumulates with atomic reductions, so gradients are compared against the spread of two default calls."""
    sc = small(3)
    G = upstream3(sc)
    grads = G if depth_alpha else G[:1]
    kw = dict(depth_alpha=depth_alpha, antialiased=antialiased)
    out0, g0, rows0 = run(sc, grads, **kw)
    out1, g1, rows1 = run(sc, grads, filter3d=None, **kw)
    out2, g2, rows2 = run(sc, grads, filter3d=torch.zeros(2000, device=dev()), **kw)
    out3, g3, rows3 = run(sc, grads, **kw)
    for other in (out1, out2):
        for a, b in zip(out0[:-1], other[:-1]):
            assert np.array_equal(bits(a), bits(b)) if a.is_floating_point() else torch.equal(a, b)
        vis = out0[-1].visible.bool()
        assert torch.equal(out0[-1].records[vis], other[-1].records[vis])
    spread_rows = gradrows.global_rel(rows3, rows0)
    for rows in (rows1, rows2):
        assert gradrows.global_rel(rows, rows0) <= max(4 * spread_rows, 2e-5)
    for k in PARAMS:
        spread = gradrows.global_rel(getattr(g3, k).grad, getattr(g0, k).grad)
        for g in (g1, g2):
            assert gradrows.global_rel(getattr(g, k).grad, getattr(g0, k).grad) <= max(4 * spread, 2e-5), k
    # and a live filter does change something
    out4, _, _ = run(sc, None, filter3d=to_t(live_filter(sc)), **kw)
    assert not np.array_equal(bits(out0[0]), bits(out4[0]))


# 2. ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("antialiased", [False, True], ids=["plain", "antialiased"])
@pytest.mark.parametrize("shd", [0, 1, 2, 3])
def test_records_and_image_match_the_fp32_oracle(shd, antialiased):
    """Records of the in-kernel transform (fused_preprocess_forward without caller positions, which the oracle restates
    exactly) against the fp32 oracle fed the device's exp(s) and sigmoid(o) (torch on the device, the kernels'
    expf): covariance (a, b, c) and opacity slots bit for bit, with and without the filter.  The image through
    rasterize() equals the oracle's wherever the walk does."""
    sc = small(shd)
    f = live_filter(sc)
    ext = native()
    t = {k: to_t(sc[k]) for k in ("xyz", "quaternion", "scale", "opacity", "rgb", "T", "K")}
    sh = None if sc["sh"] is None else to_t(sc["sh"])
    centre = None if sh is None else ext.camera_centre(t["T"])
    mode = ext.MODE_ANTIALIASED if antialiased else 0

    def records(m, filt):
        return ext.fused_preprocess_forward(t["xyz"], None, t["quaternion"], t["scale"], t["opacity"].reshape(-1),
                                            t["rgb"], sh, t["T"], t["K"], centre, sc["H"], sc["W"], 0.3, 500.0, 100.0,
                                            3.0, 0, False, m, filt)[0].cpu().numpy()

    rec0, rec = records(mode, None), records(mode | ext.MODE_FILTER3D, to_t(f))
    pg = fo.orc.project(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], sc["K"],
                        sc["H"], sc["W"], 0.3, 500.0, 100.0)
    vis = np.flatnonzero(pg.visible)
    e = device_exp(sc)
    sigma = torch.sigmoid(t["opacity"].reshape(-1)).cpu().numpy()[vis]

    def oracle_records(filt):
        conic, coef, _ = fo.filtered_conic(pg.xyz_cam, sc["quaternion"], sc["scale"], filt, sc["T"], sc["K"],
                                           pg.visible, e)
        conic, coef = conic[vis], coef[vis]
        opa = (sigma * coef).astype(np.float32)
        if antialiased:
            opa = fo.aao.compensate(conic, opa)[1]
        out = np.zeros((len(vis), 4), np.float32)
        out[:, 0] = conic[:, 0] + np.float32(0.25)
        out[:, 1] = (conic[:, 1] * np.float32(0.5)) * np.float32(2)
        out[:, 2] = conic[:, 2] + np.float32(0.25)
        out[:, 3] = opa
        return out, coef

    cols = [4, 5, 6, R_OPA]
    ref0, _ = oracle_records(np.zeros(2000, np.float32))
    ref, coef = oracle_records(f)
    assert (coef < 0.9).mean() > 0.5
    same0 = (bits(rec0[vis][:, cols]) == bits(ref0)).all(1)
    same = (bits(rec[vis][:, cols]) == bits(ref)).all(1)
    print(f"sh{shd}: records equal to the oracle's: default {int(same0.sum())}, filtered {int(same.sum())} of "
          f"{len(vis)}")
    assert same0.all() and same.all()
    (img, mask, uv, st), _, _ = run(sc, antialiased=antialiased, filter3d=to_t(f))
    bad = check_forward(img, oracle(sc, f, antialiased), mask, uv)
    assert int(bad.sum()) <= 3


# 3. ------------------------------------------------------------------------------------------------------------
def rows_vs_oracle(tag, sc, masks=True, depth_alpha=False, antialiased=False, absgrad=False):
    f = live_filter(sc)
    o = oracle(sc, f, antialiased)
    G, Gd, Ga = upstream3(sc)
    kw = dict(antialiased=antialiased, absgrad=absgrad, filter3d=to_t(f))
    (img, mask, uv, st), _, _ = run(sc, masks=masks, **kw)
    flips = flip_pixels(check_forward(img, o, mask, uv), st.w_per_pixel, o, G)
    G, Gd, Ga = (np.where(flips[..., None] if a.ndim == 3 else flips, 0, a).astype(np.float32) for a in (G, Gd, Ga))
    if not depth_alpha:
        Gd, Ga = np.zeros_like(Gd), np.zeros_like(Ga)
    _, g, slab = run(sc, (G, Gd, Ga) if depth_alpha else (G,), masks=masks, depth_alpha=depth_alpha, **kw)
    d = fo.rasterize_backward(o, G, Gd, Ga)
    mine = dict(rgb=slab[:, 0:3], opacity=slab[:, 3], uv=slab[:, 4:6], conic=slab[:, 6:9], z=slab[:, 9])
    fields = ("rgb", "opacity", "uv", "conic") + (("z",) if depth_alpha else ())
    allowed = gradrows.flips_allowed(int(o.keep.sum()))
    eps = gradrows.EPS[np.dtype(np.float32)]
    res = [gradrows.render_rows(f"{tag} render {k}", mine[k], getattr(d.render, k), getattr(d.mass, k),
                                RENDER_C_DA[k], eps, allowed) for k in fields]
    pr = fo.project_backward(o, mine["rgb"], mine["opacity"], mine["uv"], mine["conic"],
                             mine["z"] if depth_alpha else None)
    res += [gradrows.param_rows(f"{tag} {k}", getattr(g, k).grad, getattr(pr, k), PARAM_RTOL, PARAM_FLOOR, allowed)
            for k in PARAMS if getattr(g, k) is not None]
    gradrows.assert_all(res)
    for k in PARAMS:   # end to end against the oracle's whole chain, globally
        if getattr(g, k) is not None:
            assert gradrows.global_rel(getattr(g, k).grad, getattr(d, k)) < 5e-4, (tag, k)


def rows_cases():
    cases = [(f"sh{s}", dict(), lambda s=s: small(s)) for s in range(4)]
    cases += [("50x37", dict(), lambda: ragged(50, 37, 1)),
              ("720p", dict(), lambda: np_scene(100_000, "720p", 3, seed=0)),
              ("sh3 no masks", dict(masks=False), lambda: small(3)),
              ("sh3 depth+alpha", dict(depth_alpha=True), lambda: small(3)),
              ("sh0 depth+alpha no masks", dict(masks=False, depth_alpha=True), lambda: small(0)),
              ("sh3 antialiased", dict(antialiased=True), lambda: small(3)),
              ("sh2 antialiased depth+alpha", dict(antialiased=True, depth_alpha=True), lambda: small(2)),
              ("720p antialiased", dict(antialiased=True), lambda: np_scene(100_000, "720p", 3, seed=0)),
              ("sh3 absgrad", dict(absgrad=True), lambda: small(3)),
              ("exact huge", dict(), lambda: scenes.flagged_scene("exact huge"))]
    return cases


@pytest.mark.parametrize("tag,kw,make", rows_cases(), ids=[c[0] for c in rows_cases()])
def test_gradient_rows(tag, kw, make):
    rows_vs_oracle(tag, make(), **kw)


# 4. ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("antialiased", [False, True], ids=["plain", "antialiased"])
def test_filter_equals_the_baked_parameters_through_autograd(antialiased):
    """rasterize(filter3d=f) against rasterize(bake_filter3d(g, f)), forward and gradients through autograd.  The two
    round differently (v + f^2 in the kernel, exp(2 s') after the bake's log; sigmoid(o) coef against
    sigmoid(logit(sigmoid(o) coef))), so they agree to fp32 rounding, not bit for bit.  Measured on one H100 (720p, 100k
    gaussians, both modes): image max |diff| 3.0e-7, no pixel beyond 1e-4; per-row gradient error / row max at most
    9.7e-5 (opacity), 99th percentile at most 3.8e-6.  Bounds: no pixel beyond 1e-4 in 10^4, 99th percentile 1e-4, max
    1e-3."""
    sc = np_scene(100_000, "720p", 3, seed=0)
    f = to_t(live_filter(sc))
    G = upstream3(sc)[0]
    (img_f, mask_f, uv_f, _), g_f, _ = run(sc, (G,), antialiased=antialiased, filter3d=f)
    gb = gaussians_from(sc)
    baked = bake_filter3d(gb, f)
    (img_b, mask_b, uv_b, _), _, _ = run(sc, (G,), antialiased=antialiased, g=baked)
    assert torch.equal(mask_f, mask_b) and torch.equal(uv_f, uv_b)
    diff = (img_f - img_b).abs().amax(2)
    off = float((diff > 1e-4).float().mean())
    print(f"image: max |diff| {float(diff.max()):.3g}, median {float(diff.median()):.3g}, beyond 1e-4 on {off:.2e} "
          "of the pixels")
    assert off <= 1e-4
    for k in PARAMS:
        a, b = gradrows.as_rows(getattr(gb, k).grad), gradrows.as_rows(getattr(g_f, k).grad)
        rel = np.abs(a - b).max(1) / (np.abs(b).max(1) + 1e-3 * np.abs(b).max())
        print(f"{k}: row error / row max: median {np.median(rel):.3g}, 99th percentile {np.quantile(rel, 0.99):.3g}, "
              f"max {rel.max():.3g}; global {gradrows.global_rel(a, b):.3g}")
        assert np.quantile(rel, 0.99) <= 1e-4 and rel.max() <= 1e-3, k


# 5. ------------------------------------------------------------------------------------------------------------
def cameras(C, seed=0):
    """C cameras on a ring around the origin, looking in, with mixed focal lengths (fx != fy) and image sizes."""
    rng = np.random.default_rng(seed)
    Ts, Ks, Ws, Hs = [], [], [], []
    for c in range(C):
        a = 2 * np.pi * c / C + rng.uniform(-0.1, 0.1)
        Rm = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]])
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = Rm, [rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), rng.uniform(3.0, 6.0)]
        W, H = int(rng.integers(200, 1200)), int(rng.integers(150, 900))
        fx = rng.uniform(0.6, 1.4) * W
        Ks.append(np.array([[fx, 0, W / 2], [0, fx * rng.uniform(0.9, 1.1), H / 2], [0, 0, 1]], np.float32))
        Ts.append(T.astype(np.float32))
        Ws.append(W)
        Hs.append(H)
    return np.stack(Ts), np.stack(Ks), np.array(Ws, np.int32), np.array(Hs, np.int32)


@pytest.mark.parametrize("C", [1, 7, 129, 300])
@pytest.mark.parametrize("N", [1, 127, 128, 129, 100_003])
def test_compute_filter3d_matches_the_fp32_oracle_bit_for_bit(N, C):
    """Shared-memory chunks of 128 cameras: C = 129 and 300 take two and three."""
    rng = np.random.default_rng(N + C)
    xyz = (rng.standard_normal((N, 3)) * [1.5, 1.0, 1.5]).astype(np.float32)
    if N > 10:
        xyz[: N // 50] = [0.0, 50.0, 0.0]     # above every camera: unseen, take the largest f
    Ts, Ks, Ws, Hs = cameras(C, seed=C)
    f = compute_filter3d(to_t(xyz), to_t(Ts), to_t(Ks), Ws.tolist(), Hs.tolist()).cpu().numpy()
    ref = fo.sample(xyz, Ts, Ks, Ws, Hs)
    assert np.array_equal(bits(f), bits(ref)), int((bits(f) != bits(ref)).sum())
    if N > 10:
        assert (ref[: N // 50] == ref.max()).all() and ref.min() > 0


def test_compute_filter3d_edge_cases():
    xyz = to_t(np.array([[0, 0, -1.0]], np.float32))
    T, K = to_t(np.eye(4, dtype=np.float32)[None]), to_t(np.array([[[100.0, 0, 50], [0, 100.0, 50], [0, 0, 1]]], np.float32))
    assert float(compute_filter3d(xyz, T, K, [100], [100])[0]) == 0.0           # nothing seen: zeros
    assert compute_filter3d(xyz[:0], T, K, [100], [100]).numel() == 0
    with pytest.raises(ValueError):
        compute_filter3d(xyz, T, K, [100, 100], [100])
    with pytest.raises(ValueError):
        compute_filter3d(xyz, T, K, [100], [100], margin=-0.1)
    with pytest.raises(TypeError):
        compute_filter3d(xyz.double(), T, K, [100], [100])


# 6. ------------------------------------------------------------------------------------------------------------
def test_argument_errors_and_a_stale_filter_after_densification():
    sc = small(3)
    g = gaussians_from(sc)
    cam = Camera(64, 64, to_t(sc["K"]))
    bg, T = torch.full((3,), BG, device=dev()), to_t(sc["T"])
    with pytest.raises(ValueError):
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, filter3d=torch.zeros(2000, device=dev(), requires_grad=True))
    with pytest.raises(ValueError):
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, False, bg, filter3d=torch.zeros(2000, device=dev()))
    with pytest.raises(TypeError):
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, filter3d=torch.zeros(2000, device=dev(), dtype=torch.float64))
    # [N, 1] works like [N]
    f = to_t(live_filter(sc))
    a = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, filter3d=f)[0]
    b = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, filter3d=f.view(-1, 1))[0]
    assert torch.equal(a, b)

    # two densification passes: the filter of the old N is refused, a recomputed one works
    gs = synth.make_gaussians(20_000, "small", sh_degree=3, seed=4, device=dev(), requires_grad=True,
                              sigma_px=(2.5, 0.5, 0.5, 10.0))
    opt = FlatAdam.for_gaussians(gs)
    camS = synth.make_camera("small", device=dev())
    poses = [synth.make_pose(v, 3, device=dev()) for v in range(3)]
    train = dict(camera_T_worlds=torch.stack(poses), Ks=camS.K[None].expand(3, 3, 3).contiguous(),
                 widths=[camS.width] * 3, heights=[camS.height] * 3)
    stats = DensificationStats(gs.xyz.shape[0], dev())
    adc = AdaptiveDensityControl(gs, opt, stats, DensifyConfig())
    filt = compute_filter3d(gs.xyz, **train)
    changed = 0
    for step in range(2):
        for T in poses:
            image, mask, uv, st = rasterize(gs, T, camS, 0.3, 500.0, 100, 3.0, True, bg, return_state=True,
                                            filter3d=filt)
            uv.retain_grad()
            image.backward(synth.make_upstream_grad("small", device=dev()))
            stats.accumulate(st, uv, gs.xyz, camS.K)
            for k in PARAMS:
                getattr(gs, k).grad = None
        torch.manual_seed(step)
        info = adc.adaptive_density_control(1500 + 100 * step)
        print(info)
        if info["n_out"] != info["n_in"]:
            changed += 1
            with pytest.raises(ValueError):
                rasterize(gs, poses[0], camS, 0.3, 500.0, 100, 3.0, True, bg, filter3d=filt)
        filt = compute_filter3d(gs.xyz, **train)
        assert filt.shape[0] == gs.xyz.shape[0]
    assert changed >= 1
