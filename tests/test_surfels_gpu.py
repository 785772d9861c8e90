"""rasterize_surfels on the GPU against the fp64 oracle (tests/surfels_oracle.py), rasterize, and itself — needs an
H100.  Scenes and helpers live in this file."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import native
from gaussian_splatting_b200.densify import DensificationStats
from gaussian_splatting_b200.flat_adam import FlatAdam
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera, Gaussians
from gaussian_splatting_b200.surfels import depth_normals, rasterize_surfels
from tests import gradrows, scenes
from tests import surfels_oracle as so
from tests.gradrows import PARAM_FLOOR, PARAM_RTOL

pytestmark = pytest.mark.gpu
NEAR, FAR, PAD, MH = 0.3, 500.0, 100.0, 3.0
EPS32 = 2.0 ** -24
RENDER_C = 16384.0   # gradrows' render-stage constant
MAPS = (("image", 3), ("depth", 1), ("alpha", 1), ("normal", 3), ("dist", 1))


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def to_np(t):
    return t.detach().cpu().numpy().astype(np.float64)


def bits(t):
    return np.ascontiguousarray(t.detach().cpu().numpy(), np.float32).view(np.uint32)


# (gaussians, resolution, seed, sigma_px): the fp64 oracle visits every surfel at every pixel, so "deep" stacks many
# surfels on the 64 x 64 frame rather than filling a larger one
SCENES = {"tiny": (2000, "tiny", 0, (2.0, 0.5, 0.5, 8.0)), "small": (5000, "small", 0, (2.5, 0.5, 0.5, 10.0)),
          "deep": (12000, "tiny", 1, (2.5, 0.5, 0.5, 10.0))}


def synth_scene(name, sh_degree):
    n, res, seed, sig = SCENES[name]
    sc = scenes.np_scene(n, res, sh_degree=sh_degree, seed=seed, sigma_px=sig)
    if sh_degree == 0:
        sc["sh"] = None
    return sc


def gaussians(sc, requires_grad=True):
    P = {k: to_t(sc[k]).requires_grad_(requires_grad) for k in ("xyz", "rgb", "opacity", "scale", "quaternion")}
    sh = None if sc.get("sh") is None else to_t(sc["sh"]).requires_grad_(requires_grad)
    return Gaussians(P["xyz"], P["rgb"], P["opacity"], P["scale"], P["quaternion"], sh)


def camera(sc):
    return Camera(sc["W"], sc["H"], to_t(sc["K"]))


def render(sc, g, bg=(0.0, 0.0, 0.0), **kw):
    out = rasterize_surfels(g, to_t(sc["T"]), camera(sc), NEAR, FAR, PAD, MH,
                            torch.tensor(bg, dtype=torch.float32, device=dev()), return_state=True, **kw)
    return dict(zip(("image", "mask", "uv", "depth", "alpha", "normal", "dist", "state"), out))


def oracle(sc, bg, out, **kw):
    """The fp64 oracle, blending in the kernels' order: by their fp32 p_z (the sort keys), ties by index."""
    return so.render(sc, np.asarray(bg, float), near=NEAR, far=FAR, pad=PAD, mh=MH,
                     sort_z=to_np(out["state"].surfels)[:, 3], **kw)


def upstream(sc, seed=1):
    rng = np.random.default_rng(seed)
    H, W = sc["H"], sc["W"]
    return {k: rng.normal(size=(H, W, c)) / np.sqrt(H * W) for k, c in MAPS}


def compare_forward(out, o, allowed_frac=0.005, tol=1e-4, near_frac=0.02):
    """Pixels where a map differs from the oracle beyond rounding (tol of the map's largest value; 1e-3 for the
    distortion, a sum of squared depth differences): threshold flips, counted and bounded.  Flips where the oracle's
    walk meets a branch near its threshold (o.near) are bounded by near_frac of the image, the others by
    allowed_frac."""
    flips = np.zeros(o.alpha.shape[:2], bool)
    per = {}
    for k, _ in MAPS:
        ref = getattr(o, k)
        t = (1e-3 if k == "dist" else tol) * max(np.abs(ref).max(), 1e-12)
        assert np.isfinite(to_np(out[k])).all(), k
        d = np.abs(to_np(out[k]) - ref).max(2) > t
        per[k] = int(d.sum())
        flips |= d
    near = o.near > 0
    n_other, n_near = int((flips & ~near).sum()), int((flips & near).sum())
    lim, lim_near = max(3, int(flips.size * allowed_frac)), max(3, int(flips.size * near_frac))
    print(f"forward: {n_other} + {n_near} near a threshold, of {flips.size} pixels, beyond rounding (allowed {lim} + "
          f"{lim_near}); per map {per}")
    assert n_other <= lim and n_near <= lim_near, f"{n_other} + {n_near} pixels differ from the oracle"
    return flips


# ---- outputs -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sh", [0, 3])
@pytest.mark.parametrize("name", list(SCENES))
def test_culling_mask_and_uv_are_rasterize_s(name, sh):
    sc = synth_scene(name, sh)
    g = gaussians(sc, requires_grad=False)
    out = render(sc, g)
    img, mask_r, uv_r = rasterize(g, to_t(sc["T"]), camera(sc), NEAR, FAR, PAD, MH, True, torch.zeros(3, device=dev()))
    # the surfel stage also culls a disk that does not lie in front of the camera (none in these scenes)
    assert bool((out["mask"] == mask_r).all())
    assert (bits(out["uv"]) == bits(uv_r)).all()


@pytest.mark.parametrize("sh", [0, 3])
@pytest.mark.parametrize("name", list(SCENES))
def test_outputs_and_gradients_match_the_oracle(name, sh):
    sc = synth_scene(name, sh)
    bg = np.array([0.2, 0.4, 0.7]) if name != "deep" else np.zeros(3)
    g = gaussians(sc)
    out = render(sc, g, bg=tuple(bg))
    out["uv"].retain_grad()
    st = out["state"]
    G = upstream(sc)
    od = oracle(sc, bg, out, grads=G)
    assert (to_np(out["mask"]) == (od.visible == 0)).all(), "culling mask differs from the oracle"
    flips = compare_forward(out, od)
    # backward: pixels that flipped in the forward, or whose walk meets a branch near its threshold, are left out
    leave = flips | (od.near > 0)
    print(f"backward leaves out {int(leave.sum())} pixels ({int((od.near > 0).sum())} near a threshold)")
    # a deep stack walks dozens of surfels per pixel, each with its own chance of a branch near its threshold
    assert int((od.near > 0).sum()) <= max(3, leave.size // (4 if name == "deep" else 50))
    for k in G:
        G[k][leave] = 0.0
    od = oracle(sc, bg, out, grads=G)
    Gt = {k: to_t(v.astype(np.float32)) for k, v in G.items()}
    loss = sum((out[k] * Gt[k]).sum() for k, _ in MAPS)
    loss.backward()
    ext = native()
    rows = ext.surfel_render_backward(st.N, st.surfels, st.ranges, st.background, st.H, st.W, st.P, st.keys_sorted,
                                      st.ids_sorted, st.id_bits, NEAR, st.m_scale, MH, out["alpha"].detach(), st.last,
                                      st.totals, Gt["image"], Gt["depth"], Gt["alpha"], Gt["normal"], Gt["dist"])
    vis = to_np(~out["mask"]).astype(bool)
    M = int(vis.sum())
    allowed = gradrows.flips_allowed(M)
    res = [gradrows.render_rows("render rows", to_np(rows)[vis][:, :19], od.rows[vis][:, :19], od.mass[vis][:, :19],
                                RENDER_C, EPS32, allowed)]
    # uv.grad: d loss / d footprint translation, bounded by the masses of the row entries it is formed from
    M2 = to_np(st.surfels)[vis][:, 10:13]
    mx = (od.mass[vis][:, 0:3] * np.abs(M2)).sum(1) + od.mass[vis][:, 16]
    my = (od.mass[vis][:, 3:6] * np.abs(M2)).sum(1) + od.mass[vis][:, 17]
    res.append(gradrows.render_rows("uv.grad", out["uv"].grad, od.uv_grad[vis], np.stack([mx, my], 1), RENDER_C,
                                    EPS32, allowed))
    # the per-gaussian backward fed the oracle's rows
    centre = ext.camera_centre(to_t(sc["T"])) if sh else None
    opl = g.opacity.detach().reshape(-1).contiguous()
    pg = ext.surfel_backward(to_t(od.rows.astype(np.float32)), g.xyz.detach(), g.quaternion.detach(),
                             g.scale.detach(), opl, None if g.sh is None else g.sh.detach(), to_t(sc["T"]),
                             to_t(sc["K"]), centre, st.visible, st.surfels, None, None, None, False)
    names = ["xyz", "quaternion", "scale", "opacity", "rgb"] + (["sh"] if sh else [])
    for k, mine in zip(names, pg):
        res.append(gradrows.param_rows(f"param {k}", mine, od.g[k], PARAM_RTOL, PARAM_FLOOR, allowed))
    gradrows.assert_all(res)
    # and end to end: the autograd gradients are those rows' (global criterion)
    for k in names:
        ref = od.g[k]
        err = gradrows.global_rel(getattr(g, k).grad, ref)
        print(f"end to end {k}: {err:.2e}")
        assert err < 2e-3, k
    assert (g.scale.grad[:, 2] == 0).all()


# ---- binning -----------------------------------------------------------------------------------------------------------
def grazing_scene(n=48, seed=3, H=256, W=256):
    """Large surfels seen at grazing angles, some near the camera plane: footprints far wider than 64 tiles (the OBB
    fallback of the pair emission) and disks that just fail or just pass the in-front cull."""
    rng = np.random.default_rng(seed)
    K = np.array([[220.0, 0, 127.3], [0, 230.0, 128.6], [0, 0, 1]])
    z = np.concatenate([rng.uniform(1.5, 6.0, n - 12), rng.uniform(0.35, 0.8, 12)])
    size = np.concatenate([rng.uniform(0.03, 0.2, n - 12), rng.uniform(0.2, 0.45, 12)])
    uv = rng.uniform(-20, W + 20, (n, 2))
    xyz = np.column_stack([(uv[:, 0] - K[0, 2]) * z / K[0, 0], (uv[:, 1] - K[1, 2]) * z / K[1, 1], z])
    # tilt about a random in-plane axis by 60-88 degrees: the surfel's plane nearly contains the ray
    ang = rng.uniform(np.radians(60), np.radians(88), n)
    ax = rng.normal(size=(n, 2))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    q = np.column_stack([np.cos(ang / 2), ax * np.sin(ang / 2)[:, None], np.zeros(n)])
    scale = np.column_stack([np.log(size[:, None] * rng.uniform(0.7, 1.0, (n, 2)) * z[:, None]), np.zeros(n)])
    opa = rng.uniform(-1.0, 2.0, (n, 1))
    rgb = rng.uniform(0, 3, (n, 3))
    return dict(xyz=xyz.astype(np.float32), quaternion=q.astype(np.float32), scale=scale.astype(np.float32),
                opacity=opa.astype(np.float32), rgb=rgb.astype(np.float32), sh=None, T=np.eye(4, dtype=np.float32),
                K=K.astype(np.float32), H=H, W=W)


def test_binning_is_conservative_for_large_grazing_surfels():
    sc = grazing_scene()
    g = gaussians(sc, requires_grad=False)
    ext = native()
    fw = ext.surfel_forward(g.xyz, None, g.quaternion, g.scale, g.opacity.reshape(-1).contiguous(), g.rgb, None,
                            to_t(sc["T"]), to_t(sc["K"]), None, sc["H"], sc["W"], NEAR, FAR, PAD, MH, 0)
    vis, win = fw[3].bool().cpu().numpy(), fw[6].cpu().numpy()
    assert (win[vis] == -1).sum() >= 3, "no window beyond 64 tiles"
    # surfels in the frustum whose disk reaches behind the camera plane are culled, and only those
    out = render(sc, g)
    o = oracle(sc, np.zeros(3), out)
    p = sc["xyz"].astype(np.float64)
    in_frustum = (p[:, 2] >= NEAR) & (np.abs(o.uv - 128) <= 128 + PAD).all(1)
    assert (in_frustum & (o.visible == 0)).sum() >= 1 and (in_frustum & (o.visible == 1) & (p[:, 2] < 0.8)).sum() >= 1
    assert (to_np(out["mask"]) == (o.visible == 0)).all()
    # a tile the binning missed would differ over whole pixel blocks: only isolated rounding flips are allowed
    compare_forward(out, o, allowed_frac=0.0005, tol=2e-4)


# ---- edge cases --------------------------------------------------------------------------------------------------------
def test_every_surfel_culled_gives_the_background_and_zero_gradients():
    sc = synth_scene("tiny", 0)
    sc["xyz"] = sc["xyz"].copy()
    sc["T"] = sc["T"].copy()
    sc["T"][2, 3] -= 1000.0  # everything far behind the camera
    g = gaussians(sc)
    out = render(sc, g, bg=(0.1, 0.2, 0.3))
    assert bool(out["mask"].all()) and out["uv"].shape == (0, 2)
    torch.testing.assert_close(out["image"], torch.tensor([0.1, 0.2, 0.3], device=dev()).expand_as(out["image"]),
                               rtol=0, atol=0)
    for k in ("depth", "alpha", "normal", "dist"):
        assert bool((out[k] == 0).all()), k
    sum(out[k].sum() for k in ("image", "depth", "alpha", "normal", "dist")).backward()
    for t in (g.xyz, g.quaternion, g.scale, g.opacity, g.rgb):
        assert bool((t.grad == 0).all())


def _one(quat, scale, xyz, opacity, H, W, K):
    return dict(xyz=np.array([xyz], np.float32), quaternion=np.array([quat], np.float32),
                scale=np.array([scale], np.float32), opacity=np.array([[np.log(opacity / (1 - opacity))]], np.float32),
                rgb=np.full((1, 3), 1.5, np.float32), sh=None, T=np.eye(4, dtype=np.float32),
                K=np.array(K, np.float32), H=H, W=W)


def test_exactly_edge_on_surfel_is_finite_and_matches_the_oracle():
    q = (np.cos(np.pi / 4), 0.0, np.sin(np.pi / 4), 0.0)  # plane x = 0 through the camera centre
    sc = _one(q, (np.log(0.01), np.log(0.2), 0.0), (0.0, 0.0, 2.0), 0.8, 31, 41, [[60, 0, 20], [0, 50, 15], [0, 0, 1]])
    g = gaussians(sc)
    out = render(sc, g)
    for k, _ in MAPS:
        assert torch.isfinite(out[k]).all(), k
    o = oracle(sc, np.zeros(3), out)
    off = np.arange(sc["W"]) != 20  # the column x = c_x images the plane itself
    np.testing.assert_allclose(to_np(out["alpha"])[:, off], o.alpha[:, off], atol=1e-6)
    np.testing.assert_allclose(to_np(out["depth"])[:, off], o.depth[:, off], atol=1e-5)
    sum(out[k].sum() for k, _ in MAPS).backward()
    for t in (g.xyz, g.quaternion, g.scale, g.opacity, g.rgb):
        assert bool(torch.isfinite(t.grad).all())


def test_one_pixel_wide_image():
    sc = synth_scene("tiny", 0)
    sc["W"] = 1
    sc["K"] = sc["K"].copy()
    sc["K"][0, 2] = 0.0
    g = gaussians(sc)
    out = render(sc, g, bg=(0.5, 0.5, 0.5))
    o = oracle(sc, np.full(3, 0.5), out)
    assert int((o.alpha > 0).sum()) > 10
    compare_forward(out, o, allowed_frac=0.05)
    sum(out[k].sum() for k, _ in MAPS).backward()
    assert bool(torch.isfinite(g.xyz.grad).all())


# ---- training plumbing -------------------------------------------------------------------------------------------------
def test_grad_out_and_state_hold_the_autograd_gradients():
    sc = synth_scene("small", 3)
    g = gaussians(sc)
    n, rest = sc["xyz"].shape[0], sc["sh"].shape[2]
    ends = native().flat_section_ends(n, rest)
    buf = torch.full((ends[-1],), float("nan"), device=dev())
    out = render(sc, g, bg=(0.3, 0.3, 0.3), grad_out=buf)
    G = {k: to_t(v.astype(np.float32)) for k, v in upstream(sc, seed=4).items()}
    sum((out[k] * G[k]).sum() for k, _ in MAPS).backward()
    st = out["state"]
    assert st.grad_flat.data_ptr() == buf.data_ptr()
    starts = [0] + list(ends[:-1])
    for (s0, e0), t in zip(zip(starts, ends), (g.xyz, g.quaternion, g.scale, g.opacity, g.rgb, g.sh)):
        assert (bits(buf[s0:s0 + t.numel()]) == bits(t.grad.reshape(-1))).all()
    assert not torch.isnan(buf).any()


def test_flat_adam_step_and_densification_statistics_on_a_surfel_scene():
    sc = synth_scene("tiny", 3)
    g = gaussians(sc)
    out = render(sc, g)
    out["uv"].retain_grad()
    (out["image"].sum() + out["dist"].sum()).backward()
    st = out["state"]
    stats = DensificationStats(sc["xyz"].shape[0], dev())
    stats.accumulate(st, out["uv"], g.xyz, to_t(sc["K"]))
    vis = st.vis_idx.long()
    assert int(stats.grad_accum_count.sum()) > 0 and bool((stats.grad_accum_count <= 1).all())
    assert float(stats.uv_grad_accum[vis].abs().sum()) > 0
    opt = FlatAdam.for_gaussians(g)
    before = opt.p.clone()
    opt.step(st.grad_flat, visible=st.visible)
    moved = (opt.p != before).view(-1)
    assert bool(moved.any()) and torch.isfinite(opt.p).all()


def test_two_forwards_are_bit_identical():
    sc = synth_scene("small", 3)
    g = gaussians(sc, requires_grad=False)
    a, b = render(sc, g), render(sc, g)
    for k in ("image", "uv", "depth", "alpha", "normal", "dist"):
        assert (bits(a[k]) == bits(b[k])).all(), k
    assert bool((a["mask"] == b["mask"]).all())


# ---- an end-to-end fit -------------------------------------------------------------------------------------------------
def _plane_views(n_views=4, H=64, W=64):
    """A textured plane through (0, 0, 4) with normal n, seen from n_views cameras: target images and poses."""
    n = np.array([0.35, -0.25, -1.0])
    n /= np.linalg.norm(n)
    c0 = np.array([0.0, 0.0, 4.0])
    K = np.array([[60.0, 0, 31.5], [0, 60.0, 31.5], [0, 0, 1]])
    e1 = np.cross(n, [0, 1, 0])
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(n, e1)
    views = []
    for v in range(n_views):
        a = 0.15 * (v - (n_views - 1) / 2)
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        T = np.eye(4)
        T[:3, :3] = R
        T[:3, 3] = -R @ np.array([0.6 * np.sin(a), 0.0, 0.0])
        ys, xs = np.mgrid[0:H, 0:W]
        rays_c = np.stack([(xs - K[0, 2]) / K[0, 0], (ys - K[1, 2]) / K[1, 1], np.ones_like(xs, float)], -1)
        rays_w = rays_c @ R  # R^T r
        origin = -R.T @ T[:3, 3]
        t = ((c0 - origin) @ n) / (rays_w @ n)
        X = origin + t[..., None] * rays_w
        u, w = (X - c0) @ e1, (X - c0) @ e2
        tex = 0.5 + 0.4 * np.stack([np.sin(6 * u), np.cos(5 * w), np.sin(4 * (u + w))], -1)
        views.append((T.astype(np.float32), tex.astype(np.float32)))
    return views, K.astype(np.float32), n, c0, e1, e2


def test_fit_to_a_textured_tilted_plane():
    torch.manual_seed(0)
    views, K, n_w, c0, e1, e2 = _plane_views()
    rng = np.random.default_rng(0)
    N = 2000
    uvw = rng.uniform(-2.2, 2.2, (N, 2))
    xyz = c0 + uvw[:, :1] * e1 + uvw[:, 1:] * e2 + rng.normal(0, 0.15, (N, 1)) * n_w
    q = rng.normal(size=(N, 4))
    sc = dict(xyz=xyz.astype(np.float32), quaternion=q.astype(np.float32),
              scale=np.full((N, 3), np.log(0.08), np.float32), opacity=np.zeros((N, 1), np.float32),
              rgb=np.full((N, 3), 0.5 / 0.28209479177387814, np.float32), sh=None)
    g = gaussians(sc)
    params = [g.xyz, g.quaternion, g.scale, g.opacity, g.rgb]
    opt = torch.optim.Adam([{"params": [g.xyz], "lr": 2e-3}, {"params": [g.quaternion], "lr": 1e-2},
                            {"params": [g.scale], "lr": 5e-3}, {"params": [g.opacity], "lr": 5e-2},
                            {"params": [g.rgb], "lr": 2.5e-2}])
    cam = Camera(64, 64, to_t(K))
    targets = [(to_t(T), to_t(img)) for T, img in views]
    l1s = []
    for step in range(300):
        T, target = targets[step % len(targets)]
        image, mask, uv, depth, alpha, normal, dist = rasterize_surfels(g, T, cam, 0.2, 100.0, 10.0, 3.0,
                                                                        torch.zeros(3, device=dev()))
        l1 = (image - target).abs().mean()
        N_d = depth_normals(depth, alpha, cam)
        normal_loss = (1 - (normal * N_d).sum(-1)).mean()
        loss = l1 + 100.0 * dist.mean() + 0.05 * normal_loss
        opt.zero_grad()
        loss.backward()
        opt.step()
        l1s.append(float(l1))
    with torch.no_grad():
        T, target = targets[1]
        image, mask, uv, depth, alpha, normal, dist = rasterize_surfels(g, T, cam, 0.2, 100.0, 10.0, 3.0,
                                                                        torch.zeros(3, device=dev()))
        n_c = T[:3, :3] @ torch.tensor(n_w, dtype=torch.float32, device=dev())
        cos = (torch.nn.functional.normalize(normal, dim=-1) @ n_c).abs()
        covered = alpha[..., 0] > 0.5
        mean_cos = float(cos[covered].mean())
    first, last = np.mean(l1s[:8]), np.mean(l1s[-8:])
    print(f"fit: L1 {first:.4f} -> {last:.4f}, normals |cos| {mean_cos:.4f} over {int(covered.sum())} pixels")
    # one seeded run on an H100: L1 0.2881 -> 0.0257 (x0.089), |cos| 0.9135 over 4019 pixels; thresholds leave a
    # margin of about 2.8x on the loss ratio and of 0.06 on the alignment
    assert last < 0.25 * first
    assert mean_cos > 0.85
