"""rasterize_surfels(..., median_depth=True) on the GPU, for the pinhole, a ScanNet++-like fisheye and an OPENCV
calibration: exact answers on fronto-parallel stacks, the fp64 oracle (tests/surfels_median_oracle.py), a run without
the median, and itself — needs an H100.  Scenes, tolerances and helpers are those of tests/test_surfels_gpu.py,
tests/test_surfels_lens_gpu.py and tests/test_surfels_features_gpu.py."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import native
from gaussian_splatting_b200.flat_adam import FlatAdam
from gaussian_splatting_b200.structs import Camera
from gaussian_splatting_b200.surfels import depth_normals, rasterize_surfels
from tests import gradrows
from tests import surfels_median_oracle as mo
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


def lens_of(cam):
    return (None, None) if cam == "pinhole" else LENSES[cam]


def render(sc, g, cam, median=True, features=None, bg=(0.0, 0.0, 0.0), **kw):
    out = rasterize_surfels(g, to_t(sc["T"]), camera(sc), NEAR, FAR, PAD, MH,
                            torch.tensor(bg, dtype=torch.float32, device=dev()), return_state=True,
                            features=features, median_depth=median, **cam_kw(cam), **kw)
    names = (("image", "mask", "uv", "depth", "alpha", "normal", "dist") + (("median",) if median else ())
             + (("fmap",) if features is not None else ()))
    assert len(out) == len(names) + 1
    return dict(zip(names + ("state",), out))


def oracle(sc, out, cam, grads=None):
    lens, kc = lens_of(cam)
    return mo.render(sc, grads=grads, lens=lens, kc=kc, near=NEAR, far=FAR, pad=PAD, mh=MH,
                     sort_z=to_np(out["state"].surfels)[:, 3])


def median_backward(st, G, rows):
    """the median backward alone on the given rows (in place)"""
    native().surfel_median_backward(st.rays, st.surfels, st.H, st.W, MH, st.median_ids, G.contiguous(), rows)


def check_exact(out):
    """every pixel without alpha has median 0 and id -1; every id >= 0 is a visible gaussian whose intersection z is
    the median; the median is finite"""
    st = out["state"]
    ids = st.median_ids
    med = out["median"][..., 0]
    assert ids.shape == med.shape == out["alpha"].shape[:2] and ids.dtype == torch.int32
    empty = out["alpha"][..., 0] == 0
    assert bool((ids[empty] == -1).all()) and bool((med[empty] == 0).all())
    assert bool((ids[~empty] >= 0).all())
    assert bool(torch.isfinite(med).all())
    hit = ids >= 0
    assert bool((st.visible[ids[hit].long()] == 1).all())


# ---- exact answers -----------------------------------------------------------------------------------------------------
def fronto_parallel_stack(n=48, seed=0, H=64, W=64):
    """Unrotated surfels (identity pose): every hit's z is its p_z, exactly, in fp32 as in fp64.  Overlapping disks
    at distinct depths with opacities from 0.15 to 0.8, so pixels cross 0.5 on many different layers."""
    rng = np.random.default_rng(seed)
    K = np.array([[60.0, 0, 31.7], [0, 62.0, 32.2], [0, 0, 1]])
    z = rng.permutation(np.linspace(2.0, 6.0, n))
    uv = rng.uniform(-4, W + 4, (n, 2))
    xyz = np.column_stack([(uv[:, 0] - K[0, 2]) * z / K[0, 0], (uv[:, 1] - K[1, 2]) * z / K[1, 1], z])
    scale = np.column_stack([np.log(rng.uniform(5, 14, (n, 2)) * z[:, None] / K[0, 0]), np.zeros(n)])
    opa = rng.uniform(0.15, 0.8, (n, 1))
    return dict(xyz=xyz.astype(np.float32), quaternion=np.tile([1.0, 0, 0, 0], (n, 1)).astype(np.float32),
                scale=scale.astype(np.float32), opacity=np.log(opa / (1 - opa)).astype(np.float32),
                rgb=np.ones((n, 3), np.float32), sh=None, T=np.eye(4, dtype=np.float32), K=K.astype(np.float32),
                H=H, W=W)


@pytest.mark.parametrize("cam", CAMS)
def test_fronto_parallel_stack_gives_the_layer_s_p_z_bit_for_bit(cam):
    sc = fronto_parallel_stack()
    g = gaussians(sc, requires_grad=False)
    out = render(sc, g, cam)
    check_exact(out)
    st = out["state"]
    ids = st.median_ids
    hit = ids >= 0
    assert int(hit.sum()) > 2000
    # the median is the layer's fp32 p_z (the record's p_z slot), bit for bit
    pz = st.surfels[:, 3]
    assert (bits(out["median"][..., 0][hit]) == bits(pz[ids[hit].long()])).all()
    # and the layer is the oracle's wherever the oracle's walk meets no branch near its threshold
    o = oracle(sc, out, cam)
    mine = to_np(ids).astype(np.int64)
    differ = mine != o.id
    flagged = o.flag > 0
    print(f"{cam}: {int(hit.sum())} pixels with a median on {len(np.unique(mine[mine >= 0]))} layers, "
          f"{int(flagged.sum())} flagged, {int((differ & flagged).sum())} of them differ")
    assert len(np.unique(mine[mine >= 0])) > 20
    assert not (differ & ~flagged).any()
    assert int(flagged.sum()) <= differ.size // 20


# ---- against the fp64 oracle -------------------------------------------------------------------------------------------
ORACLE_CASES = [("tiny", 0), ("tiny", 3), ("small", 0), ("small", 3), ("deep", 0), ("deep", 3)]


@pytest.mark.parametrize("cam", CAMS)
@pytest.mark.parametrize("name,sh", ORACLE_CASES)
def test_median_and_gradients_match_the_oracle(name, sh, cam):
    sc = synth_scene(name, sh)
    g = gaussians(sc)
    out = render(sc, g, cam)
    out["uv"].retain_grad()
    st = out["state"]
    check_exact(out)
    o = oracle(sc, out, cam)
    assert (to_np(out["mask"]) == (o.visible == 0)).all(), "culling mask differs from the oracle"
    ids = to_np(st.median_ids).astype(np.int64)
    med = to_np(out["median"])[..., 0]
    scale = max(np.abs(o.median).max(), 1e-12)
    differ = (ids != o.id) | (np.abs(med - o.median) > 1e-5 * scale)
    flagged = o.flag > 0
    n_other, n_flag = int((differ & ~flagged).sum()), int((differ & flagged).sum())
    print(f"forward: {n_other} unflagged + {n_flag} flagged of {differ.size} pixels differ; {int(flagged.sum())} "
          f"flagged")
    assert n_other == 0
    assert n_flag <= max(3, differ.size // 50)
    assert int(flagged.sum()) <= max(3, differ.size // (4 if name == "deep" else 20))
    # backward: flagged pixels and those that differ are left out
    rng = np.random.default_rng(7)
    G = rng.normal(size=(sc["H"], sc["W"])) / np.sqrt(sc["H"] * sc["W"])
    G[differ | flagged] = 0.0
    od = oracle(sc, out, cam, grads=G)
    Gt = to_t(G.astype(np.float32))
    (out["median"][..., 0] * Gt).sum().backward()
    rows = torch.zeros(st.N, 20, device=dev())
    median_backward(st, Gt, rows)
    vis = to_np(~out["mask"]).astype(bool)
    allowed = gradrows.flips_allowed(int(vis.sum()))
    res = [gradrows.render_rows("median rows", to_np(rows)[vis][:, :19], od.rows[vis][:, :19], od.mass[vis][:, :19],
                                RENDER_C, EPS32, allowed)]
    ext = native()
    # uv.grad: the uv.grad kernel fed the oracle's rows
    ref_rows = to_t(od.rows.astype(np.float32))
    ref_uv = (ext.surfel_uv_grad(st.vis_idx, st.surfels, ref_rows) if st.lens is None
              else ext.surfel_lens_uv_grad(*st.lens, st.K, st.vis_idx, st.surfels, ref_rows))
    err = gradrows.global_rel(out["uv"].grad, to_np(ref_uv))
    print(f"uv.grad: {err:.2e}")
    assert err < 2e-3
    # the per-gaussian backward fed the oracle's rows
    centre = ext.camera_centre(to_t(sc["T"])) if sh else None
    args = (ref_rows, g.xyz.detach(), g.quaternion.detach(), g.scale.detach(),
            g.opacity.detach().reshape(-1).contiguous(), None if g.sh is None else g.sh.detach(), to_t(sc["T"]),
            to_t(sc["K"]), centre, st.visible, st.surfels, None, None, None, False)
    pg = ext.surfel_backward(*args) if st.lens is None else ext.surfel_lens_backward(*st.lens, *args)
    for k, mine in zip(("xyz", "quaternion"), pg):
        res.append(gradrows.param_rows(f"param {k}", mine, od.g[k], PARAM_RTOL, PARAM_FLOOR, allowed))
    gradrows.assert_all(res)
    # z does not depend on the scales: their gradient is fp32 cancellation only
    gx = np.abs(od.g["xyz"]).max()
    assert np.abs(to_np(pg[2])).max() <= 1e-4 * gx
    # and end to end through autograd
    for k in ("xyz", "quaternion"):
        err = gradrows.global_rel(getattr(g, k).grad, od.g[k])
        print(f"end to end {k}: {err:.2e}")
        assert err < 2e-3, k
    assert float(g.scale.grad.abs().max()) <= 1e-4 * gx
    assert bool((g.opacity.grad == 0).all()) and bool((g.rgb.grad == 0).all())
    if sh:
        assert bool((g.sh.grad == 0).all())


# ---- nothing else moves ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", CAMS)
def test_median_leaves_every_other_output_and_gradient_unchanged(cam):
    sc = synth_scene("small", 3)
    g = gaussians(sc, requires_grad=False)
    N = sc["xyz"].shape[0]
    F = torch.randn(N, 5, device=dev(), generator=torch.Generator(dev()).manual_seed(0))
    for feats in (None, F):
        a, b = render(sc, g, cam, median=False, features=feats), render(sc, g, cam, features=feats)
        for k in ("image", "uv", "depth", "alpha", "normal", "dist") + (("fmap",) if feats is not None else ()):
            assert (bits(a[k]) == bits(b[k])).all(), k
        assert bool((a["mask"] == b["mask"]).all())
    # the median backward with a zero upstream gradient adds nothing: the rows keep their bits
    st = b["state"]
    rows = torch.randn(N, 20, device=dev(), generator=torch.Generator(dev()).manual_seed(1))
    before = rows.clone()
    median_backward(st, torch.zeros(st.H, st.W, device=dev()), rows)
    assert (bits(rows) == bits(before)).all()
    # a non-zero one writes only dM and d p_z
    median_backward(st, torch.ones(st.H, st.W, device=dev()), rows)
    keep = [k for k in range(20) if k not in range(9) and k != 18]
    assert (bits(rows[:, keep]) == bits(before[:, keep])).all()
    assert bool((rows[:, :9] != before[:, :9]).any())
    # end to end: a median without a gradient runs no median backward, and a zero gradient changes no bit of any
    # gradient (the rows are formed by the same kernels; a zero sum is never added)
    G = {k: to_t(v.astype(np.float32)) for k, v in upstream(sc, seed=3).items()}
    n, rest = N, sc["sh"].shape[2]
    ends = native().flat_section_ends(n, rest)
    grads = []
    for mode in ("none", "unused", "zero"):
        gg = gaussians(sc)
        Fr = F.clone().requires_grad_(True)
        buf = torch.zeros(ends[-1], device=dev())
        out = render(sc, gg, cam, median=mode != "none", features=Fr, grad_out=buf)
        out["uv"].retain_grad()
        loss = sum((out[k] * G[k]).sum() for k, _ in MAPS) + (out["fmap"] ** 2).sum()
        if mode == "zero":
            loss = loss + (out["median"] * 0.0).sum()
        loss.backward()
        grads.append([t.grad for t in (gg.xyz, gg.quaternion, gg.scale, gg.opacity, gg.rgb, gg.sh, out["uv"], Fr)]
                     + [buf])
    for other in grads[1:]:
        for x, y in zip(grads[0], other):
            # the tile backwards' atomics add in any order: compare within their rounding, then the flat buffer with
            # the parameters' own gradients
            assert gradrows.global_rel(y, to_np(x)) < 1e-5


@pytest.mark.parametrize("cam", CAMS)
def test_zero_median_gradient_is_bitwise_nothing(cam):
    """The same rows with and without a zero median backward: every downstream gradient keeps its bits."""
    sc = synth_scene("small", 3)
    g = gaussians(sc, requires_grad=False)
    out = render(sc, g, cam)
    st = out["state"]
    G = {k: to_t(v.astype(np.float32)) for k, v in upstream(sc, seed=5).items()}
    z = lambda k: torch.zeros(st.H, st.W, k, device=dev())  # noqa: E731
    args = (st.N, st.surfels, st.ranges, st.background, st.H, st.W, st.P, st.keys_sorted, st.ids_sorted, st.id_bits,
            NEAR, st.m_scale, MH, out["alpha"].detach(), st.last, st.totals, G["image"], G["depth"], z(1), z(3),
            G["dist"])
    ext = native()
    rows = ext.surfel_render_backward(*args) if st.lens is None else ext.surfel_lens_render_backward(st.rays, *args)
    before = rows.clone()
    median_backward(st, torch.zeros(st.H, st.W, device=dev()), rows)
    assert (bits(rows) == bits(before)).all()


@pytest.mark.parametrize("cam", CAMS)
def test_a_median_only_loss_moves_no_opacity_colour_or_sh(cam):
    sc = synth_scene("small", 3)
    g = gaussians(sc)
    out = render(sc, g, cam)
    ((out["median"] - 3.0) ** 2).mean().backward()
    for t in (g.opacity, g.rgb, g.sh):
        assert bool((t.grad == 0).all())
    assert float(g.xyz.grad.abs().sum()) > 0 and float(g.quaternion.grad.abs().sum()) > 0


# ---- edge cases --------------------------------------------------------------------------------------------------------
def test_every_surfel_culled_gives_zero_median_and_no_id():
    sc = synth_scene("tiny", 0)
    sc["T"] = sc["T"].copy()
    sc["T"][2, 3] -= 1000.0
    g = gaussians(sc)
    out = render(sc, g, "pinhole")
    assert bool(out["mask"].all())
    assert bool((out["median"] == 0).all()) and bool((out["state"].median_ids == -1).all())
    out["median"].sum().backward()
    assert bool((g.xyz.grad == 0).all())


def test_one_pixel_wide_image():
    sc = synth_scene("tiny", 0)
    sc["W"] = 1
    sc["K"] = sc["K"].copy()
    sc["K"][0, 2] = 0.0
    g = gaussians(sc)
    out = render(sc, g, "pinhole")
    check_exact(out)
    assert int((out["state"].median_ids >= 0).sum()) > 10
    o = oracle(sc, out, "pinhole")
    differ = to_np(out["state"].median_ids).astype(np.int64) != o.id
    assert not (differ & (o.flag == 0)).any()
    out["median"].sum().backward()
    assert bool(torch.isfinite(g.xyz.grad).all()) and float(g.xyz.grad.abs().sum()) > 0


def test_fisheye_pixels_beyond_theta_max_have_no_median_and_no_gradient():
    sc = synth_scene("tiny", 0)
    sc = dict(sc, K=np.array([[30.0, 0, 31.5], [0, 30.0, 31.5], [0, 0, 1]], np.float32))
    g = gaussians(sc)
    out = rasterize_surfels(g, to_t(sc["T"]), camera(sc), NEAR, FAR, PAD, MH, torch.zeros(3, device=dev()),
                            return_state=True, fisheye=(-0.3, 0.0, 0.0, 0.0), median_depth=True)
    med, st = out[7], out[-1]
    dead = torch.from_numpy(to_np(st.rays)[..., 2] == 0).to(dev())
    assert int(dead.sum()) > 50
    assert bool((med[dead] == 0).all()) and bool((st.median_ids[dead] == -1).all())
    assert float(med[~dead].max()) > 0
    (med[..., 0] * dead.float()).sum().backward()
    for t in (g.xyz, g.quaternion, g.scale, g.opacity):
        assert bool((t.grad == 0).all())


def test_no_grad_renders_the_same_median():
    sc = synth_scene("tiny", 3)
    g = gaussians(sc)
    out = render(sc, g, "fisheye")
    with torch.no_grad():
        again = render(sc, g, "fisheye")
    assert not again["median"].requires_grad
    assert (bits(again["median"]) == bits(out["median"])).all()
    assert bool((again["state"].median_ids == out["state"].median_ids).all())


# ---- training plumbing -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", ["pinhole", "fisheye"])
def test_grad_out_and_flat_adam_with_a_median_loss(cam):
    sc = synth_scene("small", 3)
    g = gaussians(sc)
    n, rest = sc["xyz"].shape[0], sc["sh"].shape[2]
    ends = native().flat_section_ends(n, rest)
    buf = torch.full((ends[-1],), float("nan"), device=dev())
    F = torch.randn(n, 3, device=dev(), generator=torch.Generator(dev()).manual_seed(2)).requires_grad_(True)
    out = render(sc, g, cam, features=F, grad_out=buf)
    assert out["median"].shape == (sc["H"], sc["W"], 1) and out["fmap"].shape == (sc["H"], sc["W"], 3)
    ((out["image"] - 0.5).abs().mean() + (out["median"] - 4.0).abs().mean() + (out["fmap"] ** 2).mean()).backward()
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
    a, b = render(sc, g, cam), render(sc, g, cam)
    assert (bits(a["median"]) == bits(b["median"])).all()
    assert bool((a["state"].median_ids == b["state"].median_ids).all())


# ---- a fit: 2DGS's bounded-scene recipe --------------------------------------------------------------------------------
def test_fit_with_the_median_depth_of_the_bounded_recipe():
    """2 000 surfels on the textured tilted plane of tests/test_surfels_gpu.py, trained with L1 + distortion + normal
    consistency against depth_normals of the median depth (r = 1).  The median depth's distance to the plane along
    the ray is measured before and after."""
    torch.manual_seed(0)
    from tests.test_surfels_gpu import _plane_views

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
    opt = torch.optim.Adam([{"params": [g.xyz], "lr": 2e-3}, {"params": [g.quaternion], "lr": 1e-2},
                            {"params": [g.scale], "lr": 5e-3}, {"params": [g.opacity], "lr": 5e-2},
                            {"params": [g.rgb], "lr": 2.5e-2}])
    cam = Camera(64, 64, to_t(K))
    targets = [(to_t(T), to_t(img)) for T, img in views]
    Kinv = np.linalg.inv(K.astype(np.float64))
    ys, xs = np.mgrid[0:64, 0:64]
    rays_c = np.stack([xs, ys, np.ones_like(xs)], -1).astype(np.float64) @ Kinv.T

    def plane_error():
        """median over covered pixels of |median - z_plane| (camera z) in view 1"""
        T, _ = views[1]
        with torch.no_grad():
            out = rasterize_surfels(g, to_t(T), cam, 0.2, 100.0, 10.0, 3.0, torch.zeros(3, device=dev()),
                                    median_depth=True)
        med, alpha = to_np(out[7])[..., 0], to_np(out[4])[..., 0]
        R, t = T[:3, :3].astype(np.float64), T[:3, 3].astype(np.float64)
        n_c, p_c = R @ n_w, R @ c0 + t
        z_plane = (p_c @ n_c) / (rays_c @ n_c)
        covered = alpha > 0.5
        return float(np.median(np.abs(med - z_plane)[covered])), int(covered.sum())

    before, _ = plane_error()
    l1s = []
    for step in range(300):
        T, target = targets[step % len(targets)]
        image, mask, uv, depth, alpha, normal, dist, median = rasterize_surfels(
            g, T, cam, 0.2, 100.0, 10.0, 3.0, torch.zeros(3, device=dev()), median_depth=True)
        l1 = (image - target).abs().mean()
        surf_depth = median  # (1 - r) depth / alpha + r median with r = 1
        N_d = depth_normals(surf_depth, torch.ones_like(alpha), cam)
        normal_loss = (1 - (normal * N_d).sum(-1)).mean()
        loss = l1 + 100.0 * dist.mean() + 0.05 * normal_loss
        opt.zero_grad()
        loss.backward()
        opt.step()
        l1s.append(float(l1))
    after, covered = plane_error()
    first, last = np.mean(l1s[:8]), np.mean(l1s[-8:])
    print(f"bounded fit: L1 {first:.4f} -> {last:.4f}; median |median depth - plane| {before:.4f} -> {after:.4f} over "
          f"{covered} pixels")
    # one seeded run on an H100: L1 0.2881 -> 0.0266 (x0.092), median |median depth - plane| 0.0917 -> 0.0461 over 4013
    # pixels; the thresholds leave a margin of about 2.7x on the loss ratio and 1.5x on the depth error
    assert covered > 2000
    assert last < 0.25 * first
    assert after < 0.07 and after < 0.75 * before
