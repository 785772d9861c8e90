"""rasterize_surfels through fisheye and OPENCV lenses on the GPU, against the fp64 lens oracle
(tests/surfels_lens_oracle.py), rasterize with the same lens, the pinhole surfels and itself — needs an H100.  Scenes,
tolerances and the comparison helpers are those of tests/test_surfels_gpu.py."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import native
from gaussian_splatting_b200.densify import DensificationStats
from gaussian_splatting_b200.flat_adam import FlatAdam
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera
from gaussian_splatting_b200.surfels import _surfel_lens, depth_normals, rasterize_surfels
from tests import gradrows
from tests import surfels_lens_oracle as lo
from tests.gradrows import PARAM_FLOOR, PARAM_RTOL
from tests.test_surfels_gpu import (EPS32, FAR, MAPS, MH, NEAR, PAD, RENDER_C, SCENES, bits, camera, compare_forward,
                                    dev, gaussians, grazing_scene, synth_scene, to_np, to_t, upstream)

pytestmark = pytest.mark.gpu

# a ScanNet++-like fisheye, a typical OPENCV calibration, and barrel distortion that folds inside the tiny scene's
# frustum (s = 0.686)
LENSES = {"fisheye": ("fisheye", (0.03, -0.01, 0.002, -0.0005)),
          "opencv": ("distortion", (-0.12, 0.03, 5e-4, -3e-4, 0.01)),
          "barrel": ("distortion", (-0.6, 0.1, 0.0, 0.0, 0.0))}


def lens_kw(name):
    lens, k = LENSES[name]
    return {lens: k}


def render(sc, g, lens_name, bg=(0.0, 0.0, 0.0), **kw):
    out = rasterize_surfels(g, to_t(sc["T"]), camera(sc), NEAR, FAR, PAD, MH,
                            torch.tensor(bg, dtype=torch.float32, device=dev()), return_state=True,
                            **lens_kw(lens_name), **kw)
    return dict(zip(("image", "mask", "uv", "depth", "alpha", "normal", "dist", "state"), out))


def oracle(sc, bg, out, lens_name, **kw):
    lens, k = LENSES[lens_name]
    return lo.render(sc, np.asarray(bg, float), lens, k, near=NEAR, far=FAR, pad=PAD, mh=MH,
                     sort_z=to_np(out["state"].surfels)[:, 3], **kw)


# ---- centres, mask and rays --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lens_name", list(LENSES))
@pytest.mark.parametrize("name", list(SCENES))
def test_uv_depth_keys_and_mask_are_rasterize_s(name, lens_name):
    sc = synth_scene(name, 3)
    g = gaussians(sc, requires_grad=False)
    out = render(sc, g, lens_name)
    img, mask_r, uv_r = rasterize(g, to_t(sc["T"]), camera(sc), NEAR, FAR, PAD, MH, True, torch.zeros(3, device=dev()),
                                  **lens_kw(lens_name))
    # the surfel stage culls on top only the disks that do not lie in front of the camera (none in these scenes)
    assert bool((out["mask"] == mask_r).all())
    assert (bits(out["uv"]) == bits(uv_r)).all()
    # the depth keys: the record's p_z is rasterize's camera-frame z
    o = oracle(sc, np.zeros(3), out, lens_name)
    vis = to_np(~out["mask"]).astype(bool)
    np.testing.assert_allclose(to_np(out["state"].surfels)[vis, 3], (sc["xyz"] @ sc["T"][:3, :3].T.astype(np.float64)
                                                                     + sc["T"][:3, 3])[vis, 2], rtol=1e-6)
    assert (o.visible == to_np(~out["mask"])).mean() > 0.999


@pytest.mark.parametrize("lens_name", list(LENSES))
def test_ray_map_matches_the_oracle(lens_name):
    sc = synth_scene("small", 0)
    lens, k = LENSES[lens_name]
    code, consts = _surfel_lens(k if lens == "fisheye" else None, k if lens == "distortion" else None, dev())
    rays = to_np(native().surfel_rays(code, consts, to_t(sc["K"]), sc["H"], sc["W"]))
    sc1 = dict(sc, xyz=sc["xyz"][:1], quaternion=sc["quaternion"][:1], scale=sc["scale"][:1],
               opacity=sc["opacity"][:1], rgb=sc["rgb"][:1])
    ref = lo.render(sc1, np.zeros(3), lens, k).rays
    valid_g, valid_o = rays[..., 2] > 0, ref[..., 2] > 0
    # invalid pixels agree except pixels on the limit within rounding
    assert (valid_g != valid_o).sum() <= max(2, valid_o.size // 10000)
    both = valid_g & valid_o
    np.testing.assert_allclose(rays[both], ref[both], rtol=0, atol=4 * 2.0 ** -24)
    assert (rays[~valid_g] == 0).all()


# ---- outputs and gradients against the oracle --------------------------------------------------------------------------
@pytest.mark.parametrize("sh", [0, 3])
@pytest.mark.parametrize("lens_name", list(LENSES))
@pytest.mark.parametrize("name", list(SCENES))
def test_outputs_and_gradients_match_the_oracle(name, lens_name, sh):
    sc = synth_scene(name, sh)
    bg = np.array([0.2, 0.4, 0.7]) if name != "deep" else np.zeros(3)
    g = gaussians(sc)
    out = render(sc, g, lens_name, bg=tuple(bg))
    out["uv"].retain_grad()
    st = out["state"]
    G = upstream(sc)
    od = oracle(sc, bg, out, lens_name, grads=G)
    assert (to_np(out["mask"]) == (od.visible == 0)).all(), "culling mask differs from the oracle"
    flips = compare_forward(out, od)
    leave = flips | (od.near > 0)
    assert int((od.near > 0).sum()) <= max(3, leave.size // (4 if name == "deep" else 50))
    for k in G:
        G[k][leave] = 0.0
    od = oracle(sc, bg, out, lens_name, grads=G)
    Gt = {k: to_t(v.astype(np.float32)) for k, v in G.items()}
    sum((out[k] * Gt[k]).sum() for k, _ in MAPS).backward()
    ext = native()
    rows = ext.surfel_lens_render_backward(st.rays, st.N, st.surfels, st.ranges, st.background, st.H, st.W, st.P,
                                           st.keys_sorted, st.ids_sorted, st.id_bits, NEAR, st.m_scale, MH,
                                           out["alpha"].detach(), st.last, st.totals, Gt["image"], Gt["depth"],
                                           Gt["alpha"], Gt["normal"], Gt["dist"])
    vis = to_np(~out["mask"]).astype(bool)
    M = int(vis.sum())
    allowed = gradrows.flips_allowed(M)
    res = [gradrows.render_rows("render rows", to_np(rows)[vis][:, :19], od.rows[vis][:, :19], od.mass[vis][:, :19],
                                RENDER_C, EPS32, allowed)]
    # uv.grad against the oracle's J_n^-T g_n + g_c, globally (it mixes row entries through the lens Jacobian)
    err = gradrows.global_rel(out["uv"].grad, od.uv_grad[vis])
    print(f"uv.grad: {err:.2e}")
    assert err < 2e-3
    centre = ext.camera_centre(to_t(sc["T"])) if sh else None
    opl = g.opacity.detach().reshape(-1).contiguous()
    pg = ext.surfel_lens_backward(*st.lens, to_t(od.rows.astype(np.float32)), g.xyz.detach(), g.quaternion.detach(),
                                  g.scale.detach(), opl, None if g.sh is None else g.sh.detach(), to_t(sc["T"]),
                                  to_t(sc["K"]), centre, st.visible, st.surfels, None, None, None, False)
    names = ["xyz", "quaternion", "scale", "opacity", "rgb"] + (["sh"] if sh else [])
    for k, mine in zip(names, pg):
        res.append(gradrows.param_rows(f"param {k}", mine, od.g[k], PARAM_RTOL, PARAM_FLOOR, allowed))
    gradrows.assert_all(res)
    for k in names:
        err = gradrows.global_rel(getattr(g, k).grad, od.g[k])
        print(f"end to end {k}: {err:.2e}")
        assert err < 2e-3, k
    assert (g.scale.grad[:, 2] == 0).all()


def test_zero_coefficients_match_the_pinhole_surfels():
    sc = synth_scene("small", 3)
    G = {k: to_t(v.astype(np.float32)) for k, v in upstream(sc, seed=2).items()}
    res = []
    for kw in ({}, dict(distortion=(0.0, 0.0, 0.0, 0.0, 0.0))):
        g = gaussians(sc)
        out = rasterize_surfels(g, to_t(sc["T"]), camera(sc), NEAR, FAR, PAD, MH, torch.full((3,), 0.3, device=dev()),
                                **kw)
        sum((m * G[k]).sum() for m, (k, _) in zip(out[:1] + out[3:], MAPS)).backward()
        res.append((out, [t.grad.clone() for t in (g.xyz, g.quaternion, g.scale, g.opacity, g.rgb, g.sh)]))
    (a, ga), (b, gb) = res
    # the lens projects through 1 / z and its polynomial, the pinhole through f x / z: equal up to rounding, so a few
    # centres on the padding's edge and a few threshold pixels may flip
    assert int((a[1] != b[1]).sum()) <= 2
    keep = ~(a[1] | b[1])
    if a[2].shape == b[2].shape:
        torch.testing.assert_close(a[2], b[2], rtol=0, atol=1e-3)
    for x, y in zip(a[:1] + a[3:], b[:1] + b[3:]):
        off = ((x - y).abs() > 2e-4 * float(y.detach().abs().max())).reshape(x.shape[0], x.shape[1], -1).any(-1)
        assert int(off.sum()) <= max(3, off.numel() // 200), int(off.sum())
    for x, y in zip(ga, gb):
        assert gradrows.global_rel(x[keep], to_np(y[keep])) < 1e-2


# ---- binning -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lens_name", ["fisheye", "opencv"])
def test_binning_is_conservative_for_large_grazing_surfels(lens_name):
    sc = grazing_scene()
    if lens_name == "fisheye":
        # the widest field: the image corners at about 80 degrees
        sc["K"] = np.array([[100.0, 0, 127.3], [0, 100.0, 128.6], [0, 0, 1]], np.float32)
    g = gaussians(sc, requires_grad=False)
    out = render(sc, g, lens_name)
    vis, win = to_np(~out["mask"]).astype(bool), None
    o = oracle(sc, np.zeros(3), out, lens_name)
    assert (to_np(out["mask"]) == (o.visible == 0)).all()
    assert vis.sum() >= 10
    compare_forward(out, o, allowed_frac=0.0005, tol=2e-4)
    del win


def test_fisheye_pixels_beyond_theta_max_show_the_background_and_get_no_gradient():
    # k1 = -0.3 folds at about 49 degrees; a 90 x 90 px frame with f = 30 reaches 56 degrees at its corners
    sc = synth_scene("tiny", 0)
    sc = dict(sc, K=np.array([[30.0, 0, 31.5], [0, 30.0, 31.5], [0, 0, 1]], np.float32))
    g = gaussians(sc)
    bg = (0.1, 0.2, 0.3)
    out = rasterize_surfels(g, to_t(sc["T"]), camera(sc), NEAR, FAR, PAD, MH,
                            torch.tensor(bg, device=dev()), return_state=True, fisheye=(-0.3, 0.0, 0.0, 0.0))
    st = out[-1]
    dead = to_np(st.rays)[..., 2] == 0
    assert dead.sum() > 50
    torch.testing.assert_close(out[0][torch.from_numpy(dead).to(dev())],
                               torch.tensor(bg, device=dev()).expand(int(dead.sum()), 3), rtol=0, atol=0)
    for m in out[3:7]:
        assert bool((m[torch.from_numpy(dead).to(dev())] == 0).all())
    # a gradient only on the dead pixels reaches no gaussian
    Gd = torch.from_numpy(dead).to(dev()).float()[..., None]
    ((out[0] * Gd).sum() + (out[3] * Gd).sum() + (out[4] * Gd).sum() + (out[6] * Gd).sum()).backward()
    for t in (g.xyz, g.quaternion, g.scale, g.opacity, g.rgb):
        assert bool((t.grad == 0).all())


# ---- depth normals -----------------------------------------------------------------------------------------------------
def test_depth_normals_recover_a_tilted_plane_through_a_fisheye():
    H, W = 48, 64
    K = torch.tensor([[25.0, 0, 31.5], [0, 25.0, 23.5], [0, 0, 1]], device=dev())
    k = (0.03, -0.01, 0.002, -0.0005)
    code, consts = _surfel_lens(k, None, dev())
    d = native().surfel_rays(code, consts, K, H, W).double()
    n = torch.tensor([0.3, -0.4, -1.0], dtype=torch.float64, device=dev())
    n = n / n.norm()
    t = -3.0 / (d @ n)          # the ray's distance to the plane n . X = -3
    z = t * d[..., 2]
    alpha = torch.full((H, W, 1), 0.8, dtype=torch.float64, device=dev())
    out = depth_normals((z * 0.8)[..., None], alpha, Camera(W, H, K.double()), fisheye=k)
    facing = n if float(n[2]) < 0 else -n
    torch.testing.assert_close(out[1:-1, 1:-1], facing.expand(H - 2, W - 2, 3), atol=1e-6, rtol=0)
    # through K^-1 (no lens) the same depth gives other, wrong normals
    wrong = depth_normals((z * 0.8)[..., None], alpha, Camera(W, H, K.double()))
    assert float((wrong[1:-1, 1:-1] - facing).abs().max()) > 1e-2


# ---- training plumbing -------------------------------------------------------------------------------------------------
def test_grad_out_flat_adam_and_densification_on_a_lens_scene():
    sc = synth_scene("small", 3)
    g = gaussians(sc)
    n, rest = sc["xyz"].shape[0], sc["sh"].shape[2]
    ends = native().flat_section_ends(n, rest)
    buf = torch.full((ends[-1],), float("nan"), device=dev())
    out = render(sc, g, "fisheye", bg=(0.3, 0.3, 0.3), grad_out=buf)
    out["uv"].retain_grad()
    G = {k: to_t(v.astype(np.float32)) for k, v in upstream(sc, seed=4).items()}
    sum((out[k] * G[k]).sum() for k, _ in MAPS).backward()
    st = out["state"]
    assert st.grad_flat.data_ptr() == buf.data_ptr()
    starts = [0] + list(ends[:-1])
    for (s0, e0), t in zip(zip(starts, ends), (g.xyz, g.quaternion, g.scale, g.opacity, g.rgb, g.sh)):
        assert (bits(buf[s0:s0 + t.numel()]) == bits(t.grad.reshape(-1))).all()
    stats = DensificationStats(n, dev())
    stats.accumulate(st, out["uv"], g.xyz, to_t(sc["K"]))
    assert int(stats.grad_accum_count.sum()) > 0
    assert float(stats.uv_grad_accum[st.vis_idx.long()].abs().sum()) > 0
    opt = FlatAdam.for_gaussians(g)
    before = opt.p.clone()
    opt.step(st.grad_flat, visible=st.visible)
    assert bool((opt.p != before).any()) and torch.isfinite(opt.p).all()


@pytest.mark.parametrize("lens_name", ["fisheye", "opencv"])
def test_two_forwards_are_bit_identical(lens_name):
    sc = synth_scene("small", 3)
    g = gaussians(sc, requires_grad=False)
    a, b = render(sc, g, lens_name), render(sc, g, lens_name)
    for k in ("image", "uv", "depth", "alpha", "normal", "dist"):
        assert (bits(a[k]) == bits(b[k])).all(), k


# ---- an end-to-end fit -------------------------------------------------------------------------------------------------
def test_fit_to_a_textured_tilted_plane_through_a_fisheye():
    """A textured plane through (0, 0, 4), normal n, seen through a wide fisheye from four cameras; the targets are
    ray-traced along the lens's own rays.  300 steps of L1 + distortion + normal consistency."""
    torch.manual_seed(0)
    H = W = 64
    k = (0.03, -0.01, 0.002, -0.0005)
    K = torch.tensor([[30.0, 0, 31.5], [0, 30.0, 31.5], [0, 0, 1]], device=dev())
    code, consts = _surfel_lens(k, None, dev())
    rays = native().surfel_rays(code, consts, K, H, W).double().cpu().numpy()
    n_w = np.array([0.35, -0.25, -1.0])
    n_w /= np.linalg.norm(n_w)
    c0 = np.array([0.0, 0.0, 4.0])
    e1 = np.cross(n_w, [0, 1, 0])
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(n_w, e1)
    views = []
    for v in range(4):
        a = 0.15 * (v - 1.5)
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        T = np.eye(4)
        T[:3, :3] = R
        T[:3, 3] = -R @ np.array([0.6 * np.sin(a), 0.0, 0.0])
        origin = -R.T @ T[:3, 3]
        rw = rays @ R
        t = ((c0 - origin) @ n_w) / np.where(np.abs(rw @ n_w) > 1e-9, rw @ n_w, 1e-9)
        X = origin + t[..., None] * rw
        u, w = (X - c0) @ e1, (X - c0) @ e2
        tex = 0.5 + 0.4 * np.stack([np.sin(6 * u), np.cos(5 * w), np.sin(4 * (u + w))], -1)
        depth = t * rays[..., 2]
        views.append((to_t(T.astype(np.float32)), to_t(tex.astype(np.float32)), depth, (np.abs(u) < 2) & (np.abs(w) < 2)))
    rng = np.random.default_rng(0)
    N = 3000
    uvw = rng.uniform(-2.6, 2.6, (N, 2))
    xyz = c0 + uvw[:, :1] * e1 + uvw[:, 1:] * e2 + rng.normal(0, 0.15, (N, 1)) * n_w
    sc = dict(xyz=xyz.astype(np.float32), quaternion=rng.normal(size=(N, 4)).astype(np.float32),
              scale=np.full((N, 3), np.log(0.08), np.float32), opacity=np.zeros((N, 1), np.float32),
              rgb=np.full((N, 3), 0.5 / 0.28209479177387814, np.float32), sh=None)
    g = gaussians(sc)
    opt = torch.optim.Adam([{"params": [g.xyz], "lr": 2e-3}, {"params": [g.quaternion], "lr": 1e-2},
                            {"params": [g.scale], "lr": 5e-3}, {"params": [g.opacity], "lr": 5e-2},
                            {"params": [g.rgb], "lr": 2.5e-2}])
    cam = Camera(W, H, K)

    def depth_error(T, depth_ref, on):
        with torch.no_grad():
            out = rasterize_surfels(g, T, cam, 0.2, 100.0, 10.0, 3.0, torch.zeros(3, device=dev()), fisheye=k)
        a = to_np(out[4])[..., 0]
        m = on & (a > 0.5)
        return float(np.median(np.abs(to_np(out[3])[..., 0][m] / a[m] - depth_ref[m]))), int(m.sum())

    err0 = depth_error(views[1][0], views[1][2], views[1][3])
    for step in range(300):
        T, target, _, _ = views[step % 4]
        image, mask, uv, depth, alpha, normal, dist = rasterize_surfels(g, T, cam, 0.2, 100.0, 10.0, 3.0,
                                                                        torch.zeros(3, device=dev()), fisheye=k)
        N_d = depth_normals(depth, alpha, cam, fisheye=k)
        loss = ((image - target).abs().mean() + 100.0 * dist.mean()
                + 0.05 * (1 - (normal * N_d).sum(-1)).mean())
        opt.zero_grad()
        loss.backward()
        opt.step()
    err1 = depth_error(views[1][0], views[1][2], views[1][3])
    print(f"fit through a fisheye: median |expected depth - plane| {err0[0]:.4f} -> {err1[0]:.4f} over {err1[1]} px")
    # one seeded run on an H100: 0.1325 -> 0.0430 over 744 pixels
    assert err1[1] > 500
    assert err1[0] < 0.5 * err0[0] and err1[0] < 0.06
