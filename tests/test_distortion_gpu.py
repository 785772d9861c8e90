"""Radial-tangential lens distortion on the GPU: rasterize(..., distortion=k) and rasterize_batch against the fp64 CPU
oracle (tests/distortion_oracle.py), the fp32 render oracle, barrel distortion drawing what the pinhole cannot and
culling what folds back, zero coefficients against the pinhole, and the existing invariants in distortion mode — needs
an H100."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import rasterize_batch
from gaussian_splatting_b200.densify import WeightStats
from gaussian_splatting_b200.rasterize import distortion_r2_max, rasterize
from gaussian_splatting_b200.structs import Camera, Gaussians
from oracle import cpu_oracle as orc
from tests import depth_alpha_oracle as dao
from tests import distortion_oracle as dto
from tests import gradrows
from tests.scenes import SH0
from tests.test_filter3d_gpu import flips_allowed_px
from tests.test_filter3d_oracle import live_filter
from tests.test_gradient_rows_gpu import gaussians_from, np_scene

pytestmark = pytest.mark.gpu
BG = 0.5
K0 = (0.0, 0.0, 0.0, 0.0, 0.0)
KR = (-0.6, 0.1, 0.0, 0.0, 0.0)              # barrel, folds back inside the tiny scene's frustum (s = 0.686)
KF = (-0.12, 0.03, 5e-4, -3e-4, 0.01)        # a typical OPENCV calibration
KS = {"zero": K0, "radial": KR, "full": KF}
MODES = {"plain": {}, "depth": dict(render_depth_alpha=True), "antialiased": dict(antialiased=True),
         "filter3d": dict(filter3d=True), "all": dict(render_depth_alpha=True, antialiased=True, filter3d=True)}
PARAMS = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def bits(a):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def scene(shd, n=2000):
    """2000 gaussians at 64 x 64 (screen sigma 0.15 - 8 px), seen through the lens."""
    return np_scene(n, "tiny", shd, sigma_px=(0.8, 0.8, 0.15, 8.0))


def run(sc, k, mode, grads=True, seed=1):
    """Fused forward with distortion=k and the mode's flags, then the backward of <G,image> (+ <Gd,depth> + <Ga,alpha>).
    Returns the outputs (state last), the gaussians (with .grad), the render-stage rows the per-gaussian backward got
    and the filter."""
    flags = dict(MODES[mode])
    f = None
    if flags.pop("filter3d", False):
        f = live_filter(sc)
        flags["filter3d"] = to_t(f)
    g = gaussians_from(sc)
    out = rasterize(g, to_t(sc["T"]), Camera(sc["W"], sc["H"], to_t(sc["K"])), 0.3, 500.0, 100, 3.0, True,
                    torch.full((3,), BG, device=dev()), return_state=True, distortion=k, **flags)
    seen = []
    if grads:
        rng = np.random.default_rng(seed)
        H, W = sc["H"], sc["W"]
        image = out[0]
        proj = next(fn for fn, i in image.grad_fn.next_functions if fn is not None and i == 1)
        proj.register_prehook(lambda grad_outputs: seen.append(grad_outputs[1].detach().clone()))
        maps = [out[0]] + ([out[3], out[4]] if flags.get("render_depth_alpha") else [])
        ups = [to_t((rng.standard_normal(tuple(m.shape)) / m.numel()).astype(np.float32)) for m in maps]
        torch.autograd.backward(maps, ups)
    return out, g, (seen[0].view(-1, 12).double().cpu().numpy() if seen else None), f


def oracle(sc, k, mode, f, smax):
    flags = MODES[mode]
    return dto.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"],
                         sc["K"], sc["H"], sc["W"], k, antialiased=flags.get("antialiased", False), filter3d=f,
                         background=np.full(3, BG), smax=smax)


def boundary(o, sc, smax, eps=1e-5):
    """Gaussians within fp32 rounding of a cull boundary: near / far, the padded image edges, r2_max."""
    pg = o.pg
    z, u, v = pg.xyz_cam[:, 2], pg.uv[:, 0], pg.uv[:, 1]
    W, H, pad = sc["W"], sc["H"], 100.0
    close = lambda a, b: np.abs(a - b) <= eps * np.maximum(1.0, np.abs(b))  # noqa: E731
    return (close(z, 0.3) | close(z, 500.0) | close(u, -pad) | close(u, W + pad) | close(v, -pad) | close(v, H + pad)
            | (close(pg.s, smax) if np.isfinite(smax) else False))


# 1. per-gaussian forward and backward against the fp64 oracle -----------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("shd", [0, 1, 2, 3])
@pytest.mark.parametrize("k", list(KS), ids=list(KS))
def test_per_gaussian_stage_matches_the_fp64_oracle(k, shd, mode):
    sc = scene(shd)
    out, g, rows, f = run(sc, KS[k], mode)
    st = out[-1]
    smax = distortion_r2_max(KS[k])
    o = oracle(sc, KS[k], mode, f, smax)
    mask = out[1].cpu().numpy()
    edge = boundary(o, sc, smax)
    assert int(edge.sum()) == 0, int(edge.sum())
    assert (mask == o.culling_mask).all(), int((mask != o.culling_mask).sum())
    assert o.keep.sum() > 500
    rec = st.records.double().cpu().numpy()[o.keep]
    assert gradrows.global_rel(out[2].detach().cpu().numpy(), o.uv) <= 1e-4
    conic = np.stack([rec[:, 4] - 0.25, rec[:, 5], rec[:, 6] - 0.25], 1)
    assert gradrows.global_rel(conic, o.conic) <= 1e-4
    assert gradrows.global_rel(rec[:, 3], o.opacity) <= 1e-4
    # backward fed the GPU's own rows
    d = dto.project_backward(o, rows[:, 0:3], rows[:, 3], rows[:, 4:6], rows[:, 6:9],
                             rows[:, 9] if MODES[mode].get("render_depth_alpha") else None)
    for name in PARAMS:
        t = getattr(g, name)
        if t is None:
            continue
        got = t.grad.double().cpu().numpy().reshape(getattr(d, name).shape)
        assert np.isfinite(got).all(), name
        assert gradrows.global_rel(got, getattr(d, name)) <= 1e-4, (name, gradrows.global_rel(got, getattr(d, name)))


# 2. image and per-pixel state against the fp32 render oracle fed the GPU's per-gaussian outputs ----------------------------
@pytest.mark.parametrize("k", list(KS), ids=list(KS))
def test_image_and_pixel_state_match_the_render_oracle_fed_the_gpu_records(k):
    sc = scene(3)
    out, _, _, _ = run(sc, KS[k], "depth", grads=False)
    st = out[-1]
    vis = st.vis_idx.long()
    rec = st.records[vis].cpu().numpy()
    uv = rec[:, 0:2].copy()
    conic = np.stack([rec[:, 4] - np.float32(0.25), rec[:, 5], rec[:, 6] - np.float32(0.25)], 1).astype(np.float32)
    opa = rec[:, 3].copy()
    rgb = (rec[:, 9:12] / np.float32(SH0)).astype(np.float32)
    T = sc["T"].astype(np.float32)
    xyz_cam = (sc["xyz"][vis.cpu().numpy()] @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    H, W = sc["H"], sc["W"]
    sorted_idx, ranges = orc.tile_lists(uv, xyz_cam, conic, (W + 15) // 16, (H + 15) // 16, 3.0)
    image, n, w, depth, alpha = dao.render_forward(uv, opa, rgb, conic, np.ascontiguousarray(xyz_cam[:, 2]), ranges,
                                                   sorted_idx, np.full(3, BG, np.float32), H, W)
    diff = np.abs(out[0].detach().cpu().numpy().astype(np.float64) - image).max(2)
    bad = diff > 1e-4 * np.abs(image).max()
    assert int(bad.sum()) <= flips_allowed_px(bad.size), int(bad.sum())
    assert (np.abs(st.n_per_pixel.cpu().numpy() - n) > 0).sum() <= flips_allowed_px(bad.size)
    assert np.abs(out[4].detach().cpu().numpy()[..., 0] - alpha)[~bad].max() <= 1e-4


# 3. barrel distortion: what the pinhole cannot draw, and what folds back -------------------------------------------------
KB = (-0.3, 0.0, 0.0, 0.0, 0.0)  # folds at s = 1 / 0.9
W3, H3, F3 = 640, 480, 450.0


def _one(xyz, scale=-4.0):
    n = len(xyz)
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=dev()).requires_grad_(True)  # noqa: E731
    return Gaussians(t(xyz), t(np.full((n, 3), 2.0)), t(np.full((n, 1), 0.0)), t(np.full((n, 3), scale)),
                     t(np.tile([1.0, 0.0, 0.0, 0.0], (n, 1))), None)


def _k3():
    return torch.tensor([[F3, 0, W3 / 2], [0, F3, H3 / 2], [0, 0, 1]], dtype=torch.float32, device=dev())


def test_barrel_distortion_draws_a_gaussian_the_pinhole_cannot_where_the_model_puts_it():
    """a = x / z = 0.837 (s = 0.7 < r2_max = 1.11): the pinhole puts it at u = 697 > W = 640 and culls it (no padding),
    the barrel lens pulls it in to u = 617.  The drawn splat's centroid is the oracle's (u, v) within 0.1 px."""
    z = 5.0
    p = np.array([[np.sqrt(0.7) * z, 0.0, z]])
    args = (torch.eye(4, device=dev()), Camera(W3, H3, _k3()), 0.3, 500.0, 0.0, 3.0, True, torch.zeros(3, device=dev()))
    g = _one(p, scale=np.log(0.05))
    img_pin, mask_pin, _ = rasterize(g, *args)
    assert bool(mask_pin[0]) and float(img_pin.detach().abs().max()) == 0.0
    img, mask, uv = rasterize(g, *args, distortion=KB)
    assert not bool(mask[0])
    u_ref, _ = dto.project_point(p[0], _k3().double().cpu().numpy(), KB)
    u, v = uv.detach().cpu().numpy()[0]
    assert abs(u - u_ref[0]) <= 1e-3 and abs(v - u_ref[1]) <= 1e-3, (u, v, u_ref)
    assert F3 * np.sqrt(0.7) + W3 / 2 > W3 and u < W3 - 15
    lum = img.sum(2).detach().double().cpu().numpy()
    yy, xx = np.mgrid[0:H3, 0:W3]
    cu, cv = (lum * xx).sum() / lum.sum(), (lum * yy).sum() / lum.sum()
    assert abs(cu - u_ref[0]) <= 0.1 and abs(cv - u_ref[1]) <= 0.1, (cu, cv, u_ref)
    img.sum().backward()
    assert torch.isfinite(g.xyz.grad).all() and bool((g.xyz.grad != 0).any())


def test_a_gaussian_beyond_the_fold_is_culled_and_the_image_there_is_the_background():
    """s = 2 > r2_max: the model maps it back to u = 575, inside the image; it is culled and every pixel is the
    background."""
    z = 5.0
    p = np.array([[np.sqrt(2.0) * z, 0.0, z]])
    uv_ref, s = dto.project_point(p[0], _k3().double().cpu().numpy(), KB)
    assert s >= distortion_r2_max(KB) and 0 < uv_ref[0] < W3 - 30
    bg = torch.tensor([0.2, 0.3, 0.4], device=dev())
    g = _one(p, scale=np.log(0.05))
    img, mask, uv = rasterize(g, torch.eye(4, device=dev()), Camera(W3, H3, _k3()), 0.3, 500.0, 0.0, 3.0, True, bg,
                              distortion=KB)
    assert bool(mask[0])
    assert torch.equal(img, bg.expand(H3, W3, 3))


# 4. zero coefficients against the pinhole ----------------------------------------------------------------------------------
def test_zero_coefficients_are_the_pinhole_up_to_fp32_rounding():
    sc = scene(3)
    out_d, _, _, _ = run(sc, K0, "depth", grads=False)
    g = gaussians_from(sc)
    out_p = rasterize(g, to_t(sc["T"]), Camera(sc["W"], sc["H"], to_t(sc["K"])), 0.3, 500.0, 100, 3.0, True,
                      torch.full((3,), BG, device=dev()), return_state=True, render_depth_alpha=True)
    assert torch.equal(out_d[1], out_p[1])
    a, b = out_d[2].detach().double(), out_p[2].detach().double()
    assert float((a - b).abs().max()) <= 4 * float(b.abs().max()) * 2.0 ** -23
    vis = out_p[-1].vis_idx.long()
    ra, rb = out_d[-1].records[vis].double(), out_p[-1].records[vis].double()
    for col in (4, 5, 6):  # the conic: fp32 rounding of J, amplified by the 2-D covariance's conditioning
        assert float((ra[:, col] - rb[:, col]).abs().max()) <= 1e-4 * float(rb[:, col].abs().max()), col
    diff = (out_d[0] - out_p[0]).abs().amax(2)
    bad = diff > 1e-4
    assert int(bad.sum()) <= flips_allowed_px(bad.numel()), int(bad.sum())


# 5. the existing invariants in distortion mode ---------------------------------------------------------------------------------
def test_features_equal_the_image_on_black_uv_grad_absgrad_and_weight_stats():
    sc = scene(0)
    g = gaussians_from(sc)
    cam = Camera(sc["W"], sc["H"], to_t(sc["K"]))
    T = to_t(sc["T"])
    F = (g.rgb.detach() * SH0).contiguous()
    img, mask, uv, fmap = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, torch.zeros(3, device=dev()),
                                    features=F, distortion=KF)
    assert np.array_equal(bits(fmap), bits(img))
    ws = WeightStats(len(sc["xyz"]), dev())
    img, mask, uv = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, torch.zeros(3, device=dev()), absgrad=True,
                              weight_stats=ws, distortion=KF)
    uv.retain_grad()
    img.sum().backward()
    assert uv.grad is not None and bool((uv.grad != 0).any())
    assert uv.absgrad is not None and bool((uv.absgrad >= uv.grad.abs() - 1e-6).all())
    assert float(ws.weight_sum.sum()) > 0 and int(ws.pixel_count.sum()) > 0


def test_distortion_none_is_the_pinhole_bit_for_bit():
    """distortion=None: image, mask and uv bit for bit, and the gradients within the render backward's atomics noise
    (measured between two calls without the argument)."""
    sc = scene(3)
    outs = []
    for kw in ({}, {}, dict(distortion=None)):
        g = gaussians_from(sc)
        img, mask, uv = rasterize(g, to_t(sc["T"]), Camera(sc["W"], sc["H"], to_t(sc["K"])), 0.3, 500.0, 100, 3.0,
                                  True, torch.full((3,), BG, device=dev()), **kw)
        img.sum().backward()
        outs.append(((img, mask, uv), [getattr(g, p).grad for p in PARAMS]))
    for a, b in zip(outs[0][0], outs[2][0]):
        assert np.array_equal(bits(a), bits(b))
    for a, a2, b in zip(outs[0][1], outs[1][1], outs[2][1]):
        assert _rel(b, a) <= max(1e-6, 10 * _rel(a2, a))


# 6. rasterize_batch ------------------------------------------------------------------------------------------------------
def _batch_inputs(C):
    sc = scene(3)
    from gaussian_splatting_b200 import synth

    T = torch.stack([synth.make_pose(v, 4, device=dev()) for v in range(C)])
    return sc, T


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("mixed", [False, True], ids=["shared", "per-view"])
@pytest.mark.parametrize("mode", ["plain", "all"])
def test_batch_views_are_rasterize_bit_for_bit_and_gradients_match_the_loop(mixed, mode):
    C = 3
    sc, T = _batch_inputs(C)
    ks = [KF, K0, KR] if mixed else [KF] * C
    flags = dict(MODES[mode])
    if flags.pop("filter3d", False):
        flags["filter3d"] = to_t(live_filter(sc))
    cam = Camera(sc["W"], sc["H"], to_t(sc["K"]))
    bg = torch.full((3,), BG, device=dev())
    rng = np.random.default_rng(5)
    G = to_t(rng.standard_normal((C, sc["H"], sc["W"], 3)).astype(np.float32))

    def loop():
        g = gaussians_from(sc)
        outs = [rasterize(g, T[c], cam, 0.3, 500.0, 100, 3.0, True, bg, distortion=ks[c], **flags) for c in range(C)]
        torch.autograd.backward([o[0] for o in outs], [G[c] for c in range(C)])
        return outs, g

    g = gaussians_from(sc)
    b = rasterize_batch(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, distortion=ks if mixed else KF, **flags)
    b[0].backward(G)
    (l1, gl), (_, gl2) = loop(), loop()
    for c in range(C):
        assert np.array_equal(bits(b[0][c]), bits(l1[c][0])), c
        assert torch.equal(b[1][c], l1[c][1]), c
        assert np.array_equal(bits(b[2][c]), bits(l1[c][2])), c
        if flags.get("render_depth_alpha"):
            assert np.array_equal(bits(b[3][c]), bits(l1[c][3])) and np.array_equal(bits(b[4][c]), bits(l1[c][4]))
    for name in PARAMS:
        gb, ga, ga2 = getattr(g, name).grad, getattr(gl, name).grad, getattr(gl2, name).grad
        tol = max(1e-5, 10 * _rel(ga2, ga))
        assert _rel(gb, ga) <= tol, (name, _rel(gb, ga), tol)
