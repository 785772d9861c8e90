"""rasterize_surfels(..., features=F) on the GPU, for the pinhole, a ScanNet++-like fisheye and an OPENCV calibration:
against the surfel colour (bitwise identities), the fp64 chunk composition of the surfel oracles
(tests/surfels_features_oracle.py), a run without features, and itself — needs an H100.  Scenes, tolerances and the
comparison helpers are those of tests/test_surfels_gpu.py and tests/test_surfels_lens_gpu.py."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import native
from gaussian_splatting_b200.flat_adam import FlatAdam
from gaussian_splatting_b200.structs import Camera
from gaussian_splatting_b200.surfels import rasterize_surfels
from tests import gradrows
from tests import surfels_features_oracle as fo
from tests.gradrows import PARAM_FLOOR, PARAM_RTOL
from tests.test_surfels_gpu import (EPS32, FAR, MAPS, MH, NEAR, PAD, RENDER_C, bits, camera, dev, gaussians,
                                    synth_scene, to_np, to_t, upstream)
from tests.test_surfels_lens_gpu import LENSES

pytestmark = pytest.mark.gpu
CAMS = ("pinhole", "fisheye", "opencv")
GEOM = ("xyz", "quaternion", "scale", "opacity")


def cam_kw(cam):
    if cam == "pinhole":
        return {}
    lens, k = LENSES[cam]
    return {lens: k}


def render(sc, g, cam, features=None, bg=(0.0, 0.0, 0.0), **kw):
    out = rasterize_surfels(g, to_t(sc["T"]), camera(sc), NEAR, FAR, PAD, MH,
                            torch.tensor(bg, dtype=torch.float32, device=dev()), return_state=True,
                            features=features, **cam_kw(cam), **kw)
    names = ("image", "mask", "uv", "depth", "alpha", "normal", "dist") + (("fmap",) if features is not None else ())
    assert len(out) == len(names) + 1
    return dict(zip(names + ("state",), out))


def colours(sc, cam):
    """the surfel records' colours (state.surfels[:, 13:16]) of a run without features"""
    g = gaussians(sc, requires_grad=False)
    return render(sc, g, cam)["state"].surfels[:, 13:16].contiguous()


def padded(F):
    D = F.shape[1]
    return torch.nn.functional.pad(F, (0, (D + 3) // 4 * 4 - D)).contiguous()


def feature_backward(st, F, G, rows):
    """the feature backward alone on the given rows (in place) -> d loss / d F [N, D]"""
    gp = native().surfel_features_backward(st.rays, st.surfels, st.ranges, st.H, st.W, st.P, st.keys_sorted,
                                           st.ids_sorted, st.id_bits, MH, st.last, st.totals, padded(F), F.shape[1],
                                           G.contiguous(), rows)
    return gp[:, :F.shape[1]]


def colour_rows(st, alpha, G_image):
    z = lambda k: torch.zeros(st.H, st.W, k, device=dev())  # noqa: E731
    args = (st.N, st.surfels, st.ranges, st.background, st.H, st.W, st.P, st.keys_sorted, st.ids_sorted, st.id_bits,
            NEAR, st.m_scale, MH, alpha.detach(), st.last, st.totals, G_image, z(1), z(1), z(3), z(1))
    ext = native()
    return ext.surfel_render_backward(*args) if st.lens is None else ext.surfel_lens_render_backward(st.rays, *args)


# ---- bitwise identities ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", CAMS)
def test_colours_and_ones_give_the_image_and_alpha_bit_for_bit(cam):
    sc = synth_scene("small", 3)
    col = colours(sc, cam)
    g = gaussians(sc, requires_grad=False)
    N = col.shape[0]
    ones = torch.ones(N, 1, device=dev())
    a = render(sc, g, cam, features=col)
    assert (bits(a["fmap"]) == bits(a["image"])).all()
    b = render(sc, g, cam, features=ones)
    assert (bits(b["fmap"]) == bits(b["alpha"])).all()
    assert float(b["alpha"].max()) > 0.9
    # two chunks: the colours, then ones
    c = render(sc, g, cam, features=torch.cat([col, ones.expand(N, 5)], 1).contiguous())
    assert (bits(c["fmap"][..., :3]) == bits(c["image"])).all()
    for k in range(3, 8):
        assert (bits(c["fmap"][..., k:k + 1]) == bits(c["alpha"])).all(), k


@pytest.mark.parametrize("cam", CAMS)
def test_the_colour_is_the_special_case_of_the_gradient(cam):
    """F = the colours with the upstream G on the feature map: d loss / d F is the colour rows' G_C, and the geometry
    gradients and uv.grad are the image loss's."""
    sc = synth_scene("small", 3)
    col = colours(sc, cam)
    G = to_t(upstream(sc, seed=7)["image"].astype(np.float32))
    g_img = gaussians(sc)
    a = render(sc, g_img, cam)
    a["uv"].retain_grad()
    (a["image"] * G).sum().backward()
    rows = colour_rows(a["state"], a["alpha"], G)
    g_f = gaussians(sc)
    F = col.clone().requires_grad_(True)
    b = render(sc, g_f, cam, features=F)
    b["uv"].retain_grad()
    (b["fmap"] * G).sum().backward()
    vis = to_np(~b["mask"]).astype(bool)
    err = gradrows.global_rel(F.grad[torch.from_numpy(vis).to(dev())], to_np(rows[:, 10:13])[vis])
    print(f"{cam}: d loss / d F against G_C {err:.2e}")
    assert err < 1e-5
    assert bool((F.grad[torch.from_numpy(~vis).to(dev())] == 0).all())
    for k in GEOM:
        err = gradrows.global_rel(getattr(g_f, k).grad, to_np(getattr(g_img, k).grad))
        print(f"{cam}: {k} {err:.2e}")
        assert err < 1e-4, k
    err = gradrows.global_rel(b["uv"].grad, to_np(a["uv"].grad))
    print(f"{cam}: uv.grad {err:.2e}")
    assert err < 1e-4


# ---- against the fp64 oracle -----------------------------------------------------------------------------------------
ORACLE_CASES = [("tiny", 1, 0), ("tiny", 16, 3), ("small", 5, 3), ("small", 3, 0), ("deep", 5, 0), ("deep", 3, 3)]


@pytest.mark.parametrize("cam", CAMS)
@pytest.mark.parametrize("name,D,sh", ORACLE_CASES)
def test_feature_map_and_gradients_match_the_oracle(name, D, sh, cam):
    sc = synth_scene(name, sh)
    rng = np.random.default_rng(D)
    N = sc["xyz"].shape[0]
    Fn = rng.normal(size=(N, D)).astype(np.float32)
    g = gaussians(sc)
    F = to_t(Fn).requires_grad_(True)
    out = render(sc, g, cam, features=F)
    out["uv"].retain_grad()
    st = out["state"]
    lens, kc = (None, None) if cam == "pinhole" else LENSES[cam]
    ref = lambda G=None: fo.render(sc, Fn, grads=G, lens=lens, kc=kc, near=NEAR, far=FAR, pad=PAD, mh=MH,  # noqa: E731
                                   sort_z=to_np(st.surfels)[:, 3])
    o = ref()
    assert (to_np(out["mask"]) == (o.visible == 0)).all(), "culling mask differs from the oracle"
    # forward: threshold flips counted and bounded as in tests/test_surfels_gpu.py
    fm = to_np(out["fmap"])
    assert np.isfinite(fm).all()
    flips = np.abs(fm - o.fmap).max(2) > 1e-4 * max(np.abs(o.fmap).max(), 1e-12)
    near = o.near > 0
    n_other, n_near = int((flips & ~near).sum()), int((flips & near).sum())
    lim, lim_near = max(3, flips.size // 200), max(3, flips.size // 50)
    print(f"forward: {n_other} + {n_near} near a threshold of {flips.size} pixels beyond rounding")
    assert n_other <= lim and n_near <= lim_near
    leave = flips | near
    assert int(near.sum()) <= max(3, leave.size // (4 if name == "deep" else 50))
    G = rng.normal(size=(sc["H"], sc["W"], D)) / np.sqrt(sc["H"] * sc["W"])
    G[leave] = 0.0
    od = ref(G)
    Gt = to_t(G.astype(np.float32))
    (out["fmap"] * Gt).sum().backward()
    rows = torch.zeros(N, 20, device=dev())
    gF = feature_backward(st, F.detach(), Gt, rows)
    vis = to_np(~out["mask"]).astype(bool)
    allowed = gradrows.flips_allowed(int(vis.sum()))
    res = [gradrows.render_rows("render rows", to_np(rows)[vis][:, :19], od.rows[vis][:, :19], od.mass[vis][:, :19],
                                RENDER_C, EPS32, allowed),
           gradrows.render_rows("grad F", to_np(gF)[vis], od.g["F"][vis], od.mass_F[vis], RENDER_C, EPS32, allowed)]
    if cam == "pinhole":
        M2 = to_np(st.surfels)[vis][:, 10:13]
        mx = (od.mass[vis][:, 0:3] * np.abs(M2)).sum(1) + od.mass[vis][:, 16]
        my = (od.mass[vis][:, 3:6] * np.abs(M2)).sum(1) + od.mass[vis][:, 17]
        res.append(gradrows.render_rows("uv.grad", out["uv"].grad, od.uv_grad[vis], np.stack([mx, my], 1), RENDER_C,
                                        EPS32, allowed))
    else:
        err = gradrows.global_rel(out["uv"].grad, od.uv_grad[vis])
        print(f"uv.grad: {err:.2e}")
        assert err < 2e-3
    # the per-gaussian backward fed the oracle's rows
    ext = native()
    centre = ext.camera_centre(to_t(sc["T"])) if sh else None
    args = (to_t(od.rows.astype(np.float32)), g.xyz.detach(), g.quaternion.detach(), g.scale.detach(),
            g.opacity.detach().reshape(-1).contiguous(), None if g.sh is None else g.sh.detach(), to_t(sc["T"]),
            to_t(sc["K"]), centre, st.visible, st.surfels, None, None, None, False)
    pg = ext.surfel_backward(*args) if st.lens is None else ext.surfel_lens_backward(*st.lens, *args)
    for k, mine in zip(GEOM, pg):
        res.append(gradrows.param_rows(f"param {k}", mine, od.g[k], PARAM_RTOL, PARAM_FLOOR, allowed))
    gradrows.assert_all(res)
    # and end to end through autograd
    for k in GEOM:
        err = gradrows.global_rel(getattr(g, k).grad, od.g[k])
        print(f"end to end {k}: {err:.2e}")
        assert err < 2e-3, k
    err = gradrows.global_rel(F.grad, od.g["F"])
    print(f"end to end F: {err:.2e}")
    assert err < 2e-3
    assert (g.rgb.grad == 0).all()


# ---- nothing else moves ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", CAMS)
def test_features_leave_every_other_output_and_gradient_unchanged(cam):
    sc = synth_scene("small", 3)
    g = gaussians(sc, requires_grad=False)
    N = sc["xyz"].shape[0]
    F = torch.randn(N, 6, device=dev(), generator=torch.Generator(dev()).manual_seed(0))
    a, b = render(sc, g, cam), render(sc, g, cam, features=F)
    for k in ("image", "uv", "depth", "alpha", "normal", "dist"):
        assert (bits(a[k]) == bits(b[k])).all(), k
    assert bool((a["mask"] == b["mask"]).all())
    # the feature backward with a zero upstream gradient adds nothing: the colour rows keep their bits
    G = {k: to_t(v.astype(np.float32)) for k, v in upstream(sc, seed=3).items()}
    st = b["state"]
    rows = colour_rows(st, b["alpha"], G["image"])
    before = rows.clone()
    gF = feature_backward(st, F, torch.zeros(st.H, st.W, 6, device=dev()), rows)
    assert (bits(rows) == bits(before)).all()
    assert bool((gF == 0).all())
    # end to end: a feature map without a gradient runs no feature backward (F.grad stays None), and a zero gradient
    # changes no gaussian gradient beyond the atomics' order
    grads = []
    for mode in ("none", "unused", "zero"):
        gg = gaussians(sc)
        Fr = F.clone().requires_grad_(True)
        out = render(sc, gg, cam, features=None if mode == "none" else Fr)
        out["uv"].retain_grad()
        loss = sum((out[k] * G[k]).sum() for k, _ in MAPS)
        if mode == "zero":
            loss = loss + (out["fmap"] * 0.0).sum()
        loss.backward()
        if mode == "unused":
            assert Fr.grad is None
        if mode == "zero":
            assert bool((Fr.grad == 0).all())
        grads.append([t.grad for t in (gg.xyz, gg.quaternion, gg.scale, gg.opacity, gg.rgb, gg.sh, out["uv"])])
    for other in grads[1:]:
        for x, y in zip(grads[0], other):
            assert gradrows.global_rel(y, to_np(x)) < 1e-5


# ---- edge cases ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", CAMS)
def test_odd_widths_and_a_misaligned_f(cam):
    sc = synth_scene("tiny", 0)
    col = colours(sc, cam)
    g = gaussians(sc, requires_grad=False)
    N = col.shape[0]
    ones = torch.ones(N, 1, device=dev())
    # D = 6 (a padded chunk), and a contiguous [N, 4] F whose storage starts 4 bytes past a 16-byte boundary
    out = render(sc, g, cam, features=torch.cat([col, ones.expand(N, 3)], 1).contiguous())
    assert out["fmap"].shape == (sc["H"], sc["W"], 6)
    assert (bits(out["fmap"][..., :3]) == bits(out["image"])).all()
    assert (bits(out["fmap"][..., 5:]) == bits(out["alpha"])).all()
    buf = torch.empty(N * 4 + 1, device=dev())
    Fm = buf[1:].view(N, 4)
    Fm.copy_(torch.cat([col, ones], 1))
    assert Fm.is_contiguous() and Fm.data_ptr() % 16 != 0
    out = render(sc, g, cam, features=Fm)
    assert (bits(out["fmap"][..., :3]) == bits(out["image"])).all()
    assert (bits(out["fmap"][..., 3:]) == bits(out["alpha"])).all()
    # gradients through the padded and the misaligned F
    for F in (torch.cat([col, ones.expand(N, 3)], 1).requires_grad_(True), Fm.detach().requires_grad_(True)):
        gg = gaussians(sc)
        o = render(sc, gg, cam, features=F)
        (o["fmap"] * 1.5).sum().backward()
        assert F.grad.shape == F.shape and bool(torch.isfinite(F.grad).all())
        vis = ~o["mask"]
        assert float(F.grad[vis].abs().sum()) > 0 and bool((F.grad[~vis] == 0).all())


def test_f_without_grad_still_moves_the_geometry_and_no_grad_renders_the_same():
    sc = synth_scene("tiny", 0)
    g = gaussians(sc)
    N = sc["xyz"].shape[0]
    F = torch.rand(N, 2, device=dev(), generator=torch.Generator(dev()).manual_seed(1))
    out = render(sc, g, "pinhole", features=F)
    (out["fmap"] ** 2).sum().backward()
    for k in GEOM:
        assert float(getattr(g, k).grad.abs().sum()) > 0, k
    assert F.grad is None
    with torch.no_grad():
        again = render(sc, g, "pinhole", features=F)
    assert (bits(again["fmap"]) == bits(out["fmap"])).all()


def test_every_surfel_culled_gives_zero_features_and_zero_gradients():
    sc = synth_scene("tiny", 0)
    sc["T"] = sc["T"].copy()
    sc["T"][2, 3] -= 1000.0
    g = gaussians(sc)
    F = torch.ones(sc["xyz"].shape[0], 3, device=dev(), requires_grad=True)
    out = render(sc, g, "pinhole", features=F)
    assert bool(out["mask"].all()) and bool((out["fmap"] == 0).all())
    out["fmap"].sum().backward()
    assert bool((F.grad == 0).all()) and bool((g.xyz.grad == 0).all())


def test_one_pixel_wide_image():
    sc = synth_scene("tiny", 0)
    sc["W"] = 1
    sc["K"] = sc["K"].copy()
    sc["K"][0, 2] = 0.0
    g = gaussians(sc)
    F = torch.ones(sc["xyz"].shape[0], 1, device=dev(), requires_grad=True)
    out = render(sc, g, "pinhole", features=F)
    assert float(out["alpha"].max()) > 0
    assert (bits(out["fmap"]) == bits(out["alpha"])).all()
    out["fmap"].sum().backward()
    assert bool(torch.isfinite(g.xyz.grad).all()) and float(F.grad.abs().sum()) > 0


def test_fisheye_pixels_beyond_theta_max_give_zero_and_no_gradient():
    sc = synth_scene("tiny", 0)
    sc = dict(sc, K=np.array([[30.0, 0, 31.5], [0, 30.0, 31.5], [0, 0, 1]], np.float32))
    g = gaussians(sc)
    F = torch.ones(sc["xyz"].shape[0], 2, device=dev(), requires_grad=True)
    out = rasterize_surfels(g, to_t(sc["T"]), camera(sc), NEAR, FAR, PAD, MH, torch.zeros(3, device=dev()),
                            return_state=True, fisheye=(-0.3, 0.0, 0.0, 0.0), features=F)
    fmap, st = out[7], out[-1]
    dead = torch.from_numpy(to_np(st.rays)[..., 2] == 0).to(dev())
    assert int(dead.sum()) > 50
    assert bool((fmap[dead] == 0).all()) and float(fmap[~dead].max()) > 0
    (fmap * dead[..., None].float()).sum().backward()
    assert bool((F.grad == 0).all())
    for t in (g.xyz, g.quaternion, g.scale, g.opacity):
        assert bool((t.grad == 0).all())


# ---- training plumbing -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", ["pinhole", "fisheye"])
def test_grad_out_and_flat_adam_with_a_feature_loss(cam):
    sc = synth_scene("small", 3)
    g = gaussians(sc)
    n, rest = sc["xyz"].shape[0], sc["sh"].shape[2]
    ends = native().flat_section_ends(n, rest)
    buf = torch.full((ends[-1],), float("nan"), device=dev())
    F = torch.randn(n, 5, device=dev(), generator=torch.Generator(dev()).manual_seed(2)).requires_grad_(True)
    out = render(sc, g, cam, features=F, grad_out=buf)
    target = torch.rand_like(out["fmap"])
    ((out["image"] - 0.5).abs().mean() + ((out["fmap"] - target) ** 2).mean()).backward()
    st = out["state"]
    assert st.grad_flat.data_ptr() == buf.data_ptr()
    starts = [0] + list(ends[:-1])
    for (s0, e0), t in zip(zip(starts, ends), (g.xyz, g.quaternion, g.scale, g.opacity, g.rgb, g.sh)):
        assert (bits(buf[s0:s0 + t.numel()]) == bits(t.grad.reshape(-1))).all()
    assert not torch.isnan(buf).any() and float(F.grad.abs().sum()) > 0
    opt = FlatAdam.for_gaussians(g)
    before = opt.p.clone()
    opt.step(st.grad_flat, visible=st.visible)
    assert bool((opt.p != before).any()) and torch.isfinite(opt.p).all()


@pytest.mark.parametrize("cam", CAMS)
def test_two_forwards_are_bit_identical(cam):
    sc = synth_scene("small", 3)
    g = gaussians(sc, requires_grad=False)
    F = torch.randn(sc["xyz"].shape[0], 7, device=dev(), generator=torch.Generator(dev()).manual_seed(3))
    a, b = render(sc, g, cam, features=F), render(sc, g, cam, features=F)
    assert (bits(a["fmap"]) == bits(b["fmap"])).all()


# ---- a fit -----------------------------------------------------------------------------------------------------------
def test_fit_per_surfel_labels_to_a_label_image():
    """2 000 surfels on a textured tilted plane (fixed geometry) seen from four cameras; each surfel's ground-truth
    label (one of four bands of the texture) rendered as a one-hot feature map is the target.  F alone (D = 4) is
    optimised from zero."""
    torch.manual_seed(0)
    from tests.test_surfels_gpu import _plane_views

    views, K, n_w, c0, e1, e2 = _plane_views()
    rng = np.random.default_rng(0)
    N = 2000
    uvw = rng.uniform(-2.2, 2.2, (N, 2))
    xyz = c0 + uvw[:, :1] * e1 + uvw[:, 1:] * e2
    # the surfel's tangent axes along e1, e2: R = [e1 e2 n] as a quaternion
    R = np.column_stack([e1, e2, np.cross(e1, e2)])
    w = np.sqrt(max(1e-12, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    q = np.array([w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)])
    sc = dict(xyz=xyz.astype(np.float32), quaternion=np.tile(q, (N, 1)).astype(np.float32),
              scale=np.full((N, 3), np.log(0.09), np.float32), opacity=np.full((N, 1), 1.5, np.float32),
              rgb=np.full((N, 3), 1.0, np.float32), sh=None)
    g = gaussians(sc, requires_grad=False)
    labels = (np.floor(np.sin(3 * uvw[:, 0]) + np.cos(2 * uvw[:, 1]) + 2).clip(0, 3)).astype(np.int64)
    F_gt = torch.nn.functional.one_hot(torch.from_numpy(labels), 4).float().to(dev())
    cam = Camera(64, 64, to_t(K))
    targets = []
    with torch.no_grad():
        for T, _ in views:
            out = rasterize_surfels(g, to_t(T), cam, 0.2, 100.0, 10.0, 3.0, torch.zeros(3, device=dev()),
                                    features=F_gt)
            targets.append((to_t(T), out[7], out[4][..., 0] > 0.5))
    F = torch.zeros(N, 4, device=dev(), requires_grad=True)
    opt = torch.optim.Adam([F], lr=0.05)
    losses = []
    for step in range(200):
        T, target, _ = targets[step % len(targets)]
        fmap = rasterize_surfels(g, T, cam, 0.2, 100.0, 10.0, 3.0, torch.zeros(3, device=dev()), features=F)[7]
        loss = ((fmap - target) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    with torch.no_grad():
        T, target, covered = targets[1]
        fmap = rasterize_surfels(g, T, cam, 0.2, 100.0, 10.0, 3.0, torch.zeros(3, device=dev()), features=F)[7]
        match = float((fmap.argmax(-1) == target.argmax(-1))[covered].float().mean())
    first, last = np.mean(losses[:4]), np.mean(losses[-4:])
    print(f"label fit: loss {first:.5f} -> {last:.6f} (x{last / first:.4f}), argmax agrees on {match:.4f} of "
          f"{int(covered.sum())} covered pixels; {len(np.unique(labels))} labels")
    # one seeded run on an H100: loss 0.1404 -> 1.9e-5 (x1.4e-4), argmax agrees on 0.9988 of 3361 covered pixels;
    # the thresholds leave a margin of about 7x on the loss ratio and of 0.03 on the agreement
    assert int(covered.sum()) > 1000
    assert last < 1e-3 * first
    assert match > 0.97
