"""rasterize_surfels off the default camera, on the GPU, against the fp64 surfel oracles — needs an H100.

The other surfel test files render synth_scene's camera only: fx = fy, the principal point at the frame's centre,
frames of whole 16 x 16 tiles, a 3 degree yaw, near / far / pad / mh = 0.3 / 500 / 100 / 3 and SH degree 0 or 3.  Each
case here moves several of those parameters at once, so that a kernel that confuses or ignores one of them fails:

    case  frame, K                                    pose               near, far, pad, mh    SH
    A     77 x 53, fx 70, fy 91, c (41.3, 22.8)       general_pose()     0.3, 500, 100, 3      1
    B     77 x 53, as A                               general_pose()     0.8, 12, 0, 2         2   (m_scale 1.07)
    C     61 x 37, fx 55, fy 48, c (20.2, 19.6)       other roll/pitch   0.3, inf, 10, 4       3   (m_scale 1, 32-bit
                                                                                                    depth keys)

Every frame ends in partial tiles.  Each case runs through the pinhole, the fisheye and the OPENCV lens of
tests/test_surfels_lens_gpu.py.  The id-list pair source (sorted gaussian ids instead of (tile | depth | id) keys, taken
when the packed key would need more than 64 bits) is checked against the keys path, kernel by kernel and end to end.
tests/test_surfels_cameras_oracle.py shows on the CPU that the faults each case is chosen for fail its criteria.
Scenes are built here; tolerances and comparison helpers are those of the other surfel test files."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import native, synth
from gaussian_splatting_b200.rasterize import _depth_key_params, rasterize
from gaussian_splatting_b200.structs import Camera
from gaussian_splatting_b200.surfels import rasterize_surfels
from tests import gradrows, scenes
from tests import surfels_features_oracle as fo
from tests import surfels_lens_oracle as lo
from tests import surfels_median_oracle as mo
from tests import surfels_oracle as so
from tests.gradrows import PARAM_FLOOR, PARAM_RTOL
from tests.test_surfels_gpu import (EPS32, MAPS, RENDER_C, bits, camera, compare_forward, dev, gaussians,
                                    grazing_scene, to_np, to_t, upstream)
from tests.test_surfels_lens_gpu import LENSES

pytestmark = pytest.mark.gpu
TILE = 16
CAMS = ("pinhole", "fisheye", "opencv")
GEOM = ("xyz", "quaternion", "scale", "opacity")


def pose(roll, pitch, t):
    """camera_T_world: a roll about z after a pitch about x, then a translation"""
    c, s = np.cos(roll), np.sin(roll)
    cp, sp = np.cos(pitch), np.sin(pitch)
    R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]) @ np.array([[1, 0, 0], [0, cp, -sp], [0, sp, cp]])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T.astype(np.float32)


def intrinsics(fx, fy, cx, cy):
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)


# culls: what the case's scene must lose to the near plane, the far plane and the padding
CASES = {
    "A": SimpleNamespace(W=77, H=53, K=intrinsics(70.0, 91.0, 41.3, 22.8), T=scenes.general_pose(), near=0.3,
                         far=500.0, pad=100.0, mh=3.0, sh=1, culls=("near", "pad")),
    "B": SimpleNamespace(W=77, H=53, K=intrinsics(70.0, 91.0, 41.3, 22.8), T=scenes.general_pose(), near=0.8,
                         far=12.0, pad=0.0, mh=2.0, sh=2, culls=("near", "far", "pad")),
    "C": SimpleNamespace(W=61, H=37, K=intrinsics(55.0, 48.0, 20.2, 19.6), T=pose(-0.55, -0.2, (-0.3, 0.12, 0.25)),
                         near=0.3, far=math.inf, pad=10.0, mh=4.0, sh=3, culls=("near", "pad")),
}


def m_scale(c):
    return c.far / (c.far - c.near) if math.isfinite(c.far) else 1.0


def camera_scene(case, n=None, seed=0, sh_degree=None):
    """n surfels (default 0.45 per pixel, the density of the 64 x 64 scenes: 1836 for A and B, 1015 for C) generated in
    the case's camera frame as synth.make_gaussians does (pixel sigmas of the "tiny" scene), mapped to world coordinates
    through the inverse of its pose.  88% lie at z in [1, 11] with centres in the frame widened by 15% per side; the
    rest sit in front of near = 0.8 (z in [0.1, 0.75]), beyond far = 12 (z in [12.5, 20]) or far outside the frame
    (centres up to two frames away, beyond a padding of 100 px)."""
    c = CASES[case]
    n = int(0.45 * c.W * c.H) if n is None else n
    sh_degree = c.sh if sh_degree is None else sh_degree
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy = c.K[0, 0], c.K[1, 1], c.K[0, 2], c.K[1, 2]
    kind = rng.choice(4, size=n, p=[0.88, 0.04, 0.04, 0.04])
    z = np.where(kind == 1, rng.uniform(0.1, 0.75, n), np.where(kind == 2, rng.uniform(12.5, 20.0, n),
                                                                  rng.uniform(1.0, 11.0, n)))
    lo_, hi_ = np.where(kind == 3, -2.0, -0.15), np.where(kind == 3, 3.0, 1.15)
    u = c.W * rng.uniform(lo_, hi_)
    v = c.H * rng.uniform(lo_, hi_)
    p = np.column_stack([(u - cx) * z / fx, (v - cy) * z / fy, z])
    T = c.T.astype(np.float64)
    xyz = (p - T[:3, 3]) @ T[:3, :3]  # world positions that land at the camera-frame positions above
    sig = np.clip(np.exp(rng.normal(size=(n, 3)) * 0.5 + np.log(2.0)), 0.5, 8.0)
    scale = np.log(z[:, None] * sig / fx)
    sh = rng.normal(0, 0.2, (n, 3, (sh_degree + 1) ** 2 - 1)) if sh_degree else None
    f = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)  # noqa: E731
    return dict(xyz=f(xyz), quaternion=f(rng.normal(size=(n, 4))), scale=f(scale),
                opacity=f(rng.uniform(-2.0, 4.0, (n, 1))), rgb=f(rng.uniform(0, 1, (n, 3)) / scenes.SH0), sh=f(sh),
                T=c.T, K=c.K, H=c.H, W=c.W)


def cam_kw(cam):
    if cam == "pinhole":
        return {}
    lens, k = LENSES[cam]
    return {lens: k}


def lens_of(cam):
    return (None, None) if cam == "pinhole" else LENSES[cam]


def render(sc, g, case, cam, bg=(0.0, 0.0, 0.0), features=None, median=False, **kw):
    c = CASES[case]
    out = rasterize_surfels(g, to_t(sc["T"]), camera(sc), c.near, c.far, c.pad, c.mh,
                            torch.tensor(bg, dtype=torch.float32, device=dev()), return_state=True,
                            features=features, median_depth=median, **cam_kw(cam), **kw)
    names = (("image", "mask", "uv", "depth", "alpha", "normal", "dist") + (("median",) if median else ())
             + (("fmap",) if features is not None else ()))
    assert len(out) == len(names) + 1
    return dict(zip(names + ("state",), out))


def oracle(sc, bg, out, case, cam, **kw):
    """the colour oracle of the lens, blending in the kernels' order (their fp32 p_z)"""
    c = CASES[case]
    args = dict(near=c.near, far=c.far, pad=c.pad, mh=c.mh, sort_z=to_np(out["state"].surfels)[:, 3], **kw)
    if cam == "pinhole":
        return so.render(sc, np.asarray(bg, float), **args)
    lens, k = LENSES[cam]
    return lo.render(sc, np.asarray(bg, float), lens, k, **args)


def check_premises(sc, case, cam, out, o):
    """What the case is chosen for, so that no later edit makes it degenerate: an anisotropic, off-centre K, a pose that
    mixes y with x and z, partial tiles with contributors, every cull of the case taking place, and its m_scale.  o: the
    colour oracle's forward (its alpha, and its projected centres uv through the lens)."""
    c = CASES[case]
    # a fisheye images the whole half-space within about f pi / 2 = 110 px of c: inside A's padding of 100 px
    culls = [k for k in c.culls if not (k == "pad" and case == "A" and cam == "fisheye")]
    K, T = sc["K"], sc["T"]
    assert K[0, 0] != K[1, 1] and K[0, 2] != K[1, 2] and K[0, 2] != c.W / 2 and K[1, 2] != c.H / 2
    assert np.abs(T[1, [0, 2]]).min() > 0.01 and np.abs(T[[0, 2], 1]).min() > 0.01
    assert c.W % TILE and c.H % TILE
    a = to_np(out["alpha"])[..., 0]
    for m in (a, o.alpha[..., 0]):
        assert (m[:, c.W // TILE * TILE:] > 0).sum() >= 10 and (m[c.H // TILE * TILE:, :] > 0).sum() >= 10
    pz = (sc["xyz"].astype(np.float64) @ T[:3, :3].T.astype(np.float64) + T[:3, 3])[:, 2]
    mask = to_np(out["mask"]).astype(bool)
    by = {"near": pz < c.near, "far": pz > c.far}
    in_depth = ~by["near"] & ~by["far"]
    by["pad"] = in_depth & ((o.uv[:, 0] < -c.pad) | (o.uv[:, 0] > c.W + c.pad) | (o.uv[:, 1] < -c.pad) |
                            (o.uv[:, 1] > c.H + c.pad))
    for k in culls:
        assert by[k].any() and mask[by[k]].all(), f"case {case}: nothing culled by {k}"
    assert (~mask).sum() >= c.W * c.H // 5
    st = out["state"]
    assert st.m_scale == m_scale(c)
    if case == "B":
        assert abs(st.m_scale - 1.0) > 0.05
    if case == "C":
        assert st.m_scale == 1.0 and _depth_key_params(c.near, c.far) == (0, 32)
    if c.sh:
        assert sc["sh"].shape[2] == (c.sh + 1) ** 2 - 1


# ---- maps and gradients ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", CAMS)
@pytest.mark.parametrize("case", list(CASES))
def test_maps_and_gradients_match_the_oracle(case, cam):
    c = CASES[case]
    sc = camera_scene(case)
    bg = np.array([0.2, 0.4, 0.7])
    g = gaussians(sc)
    out = render(sc, g, case, cam, bg=tuple(bg))
    out["uv"].retain_grad()
    st = out["state"]
    G = upstream(sc)
    od = oracle(sc, bg, out, case, cam, grads=G)
    check_premises(sc, case, cam, out, od)
    assert (to_np(out["mask"]) == (od.visible == 0)).all(), "culling mask differs from the oracle"
    if cam == "pinhole":
        with torch.no_grad():
            _, mask_r, uv_r = rasterize(g, to_t(sc["T"]), camera(sc), c.near, c.far, c.pad, c.mh, True,
                                        torch.zeros(3, device=dev()))
        assert bool((out["mask"] == mask_r).all())
        assert (bits(out["uv"]) == bits(uv_r)).all()
    flips = compare_forward(out, od)
    # backward: pixels that flipped in the forward, whose walk meets a branch near its threshold, or where a surfel
    # seen nearly edge-on takes its ray-plane intersection with |c2| < |hx| |hy| / 64 (od.ill: that pixel's gradient
    # terms move by about eps32 * 64^2 = 2.4e-4 of themselves when an input is rounded to fp32) are left out.  Case B
    # through the fisheye has one such surfel at 89.6 degrees on the largest gradient: with its pixels, 1-ulp noise on
    # the fp64 oracle's own rays moves its xyz gradient by 6.9e-4 of itself
    leave = flips | (od.near > 0) | (od.ill > 0)
    print(f"backward leaves out {int(leave.sum())} pixels ({int((od.near > 0).sum())} near a threshold, "
          f"{int((od.ill > 0).sum())} ill-conditioned)")
    assert int((od.near > 0).sum()) <= max(3, leave.size // 50)
    assert int((od.ill > 0).sum()) <= max(3, leave.size // 25)
    for k in G:
        G[k][leave] = 0.0
    od = oracle(sc, bg, out, case, cam, grads=G)
    Gt = {k: to_t(v.astype(np.float32)) for k, v in G.items()}
    sum((out[k] * Gt[k]).sum() for k, _ in MAPS).backward()
    ext = native()
    args = (st.N, st.surfels, st.ranges, st.background, st.H, st.W, st.P, st.keys_sorted, st.ids_sorted, st.id_bits,
            c.near, st.m_scale, c.mh, out["alpha"].detach(), st.last, st.totals, Gt["image"], Gt["depth"], Gt["alpha"],
            Gt["normal"], Gt["dist"])
    rows = ext.surfel_render_backward(*args) if st.lens is None else ext.surfel_lens_render_backward(st.rays, *args)
    vis = to_np(~out["mask"]).astype(bool)
    allowed = gradrows.flips_allowed(int(vis.sum()))
    res = [gradrows.render_rows("render rows", to_np(rows)[vis][:, :19], od.rows[vis][:, :19], od.mass[vis][:, :19],
                                RENDER_C, EPS32, allowed)]
    if cam == "pinhole":
        # d loss / d footprint translation, bounded by the masses of the row entries it is formed from
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
    centre = ext.camera_centre(to_t(sc["T"])) if c.sh else None
    pargs = (to_t(od.rows.astype(np.float32)), g.xyz.detach(), g.quaternion.detach(), g.scale.detach(),
             g.opacity.detach().reshape(-1).contiguous(), None if g.sh is None else g.sh.detach(), to_t(sc["T"]),
             to_t(sc["K"]), centre, st.visible, st.surfels, None, None, None, False)
    pg = ext.surfel_backward(*pargs) if st.lens is None else ext.surfel_lens_backward(*st.lens, *pargs)
    names = ["xyz", "quaternion", "scale", "opacity", "rgb"] + (["sh"] if c.sh else [])
    for k, mine in zip(names, pg):
        res.append(gradrows.param_rows(f"param {k}", mine, od.g[k], PARAM_RTOL, PARAM_FLOOR, allowed))
    gradrows.assert_all(res)
    # and end to end through autograd, sh at the case's degree included
    for k in names:
        err = gradrows.global_rel(getattr(g, k).grad, od.g[k])
        print(f"end to end {k}: {err:.2e}")
        assert err < 2e-3, k
    assert (g.scale.grad[:, 2] == 0).all()


# ---- feature channels --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", CAMS)
@pytest.mark.parametrize("case", list(CASES))
def test_feature_map_and_gradients_match_the_oracle(case, cam):
    """D = 5: a full 3-channel chunk of the oracle and a partial one, and a feature stride padded to 8"""
    c = CASES[case]
    D = 5
    sc = camera_scene(case)
    rng = np.random.default_rng(D)
    N = sc["xyz"].shape[0]
    Fn = rng.normal(size=(N, D)).astype(np.float32)
    g = gaussians(sc)
    F = to_t(Fn).requires_grad_(True)
    out = render(sc, g, case, cam, features=F)
    out["uv"].retain_grad()
    st = out["state"]
    lens, kc = lens_of(cam)
    ref = lambda G=None: fo.render(sc, Fn, grads=G, lens=lens, kc=kc, near=c.near, far=c.far, pad=c.pad,  # noqa: E731
                                   mh=c.mh, sort_z=to_np(st.surfels)[:, 3])
    o = ref()
    check_premises(sc, case, cam, out, oracle(sc, np.zeros(3), out, case, cam))
    assert (to_np(out["mask"]) == (o.visible == 0)).all(), "culling mask differs from the oracle"
    fm = to_np(out["fmap"])
    assert fm.shape == (c.H, c.W, D) and np.isfinite(fm).all()
    flips = np.abs(fm - o.fmap).max(2) > 1e-4 * max(np.abs(o.fmap).max(), 1e-12)
    near = o.near > 0
    n_other, n_near = int((flips & ~near).sum()), int((flips & near).sum())
    lim, lim_near = max(3, flips.size // 200), max(3, flips.size // 50)
    print(f"forward: {n_other} + {n_near} near a threshold of {flips.size} pixels beyond rounding")
    assert n_other <= lim and n_near <= lim_near
    leave = flips | near
    assert int(near.sum()) <= max(3, leave.size // 50)
    G = rng.normal(size=(c.H, c.W, D)) / np.sqrt(c.H * c.W)
    G[leave] = 0.0
    od = ref(G)
    Gt = to_t(G.astype(np.float32))
    (out["fmap"] * Gt).sum().backward()
    rows = torch.zeros(N, 20, device=dev())
    fpad = torch.nn.functional.pad(F.detach(), (0, 3)).contiguous()
    gF = native().surfel_features_backward(st.rays, st.surfels, st.ranges, st.H, st.W, st.P, st.keys_sorted,
                                           st.ids_sorted, st.id_bits, c.mh, st.last, st.totals, fpad, D, Gt, rows)
    assert gF.shape == (N, 8) and bool((gF[:, D:] == 0).all())
    vis = to_np(~out["mask"]).astype(bool)
    allowed = gradrows.flips_allowed(int(vis.sum()))
    res = [gradrows.render_rows("render rows", to_np(rows)[vis][:, :19], od.rows[vis][:, :19], od.mass[vis][:, :19],
                                RENDER_C, EPS32, allowed),
           gradrows.render_rows("grad F", to_np(gF[:, :D])[vis], od.g["F"][vis], od.mass_F[vis], RENDER_C, EPS32,
                                allowed)]
    ext = native()
    centre = ext.camera_centre(to_t(sc["T"])) if c.sh else None
    pargs = (to_t(od.rows.astype(np.float32)), g.xyz.detach(), g.quaternion.detach(), g.scale.detach(),
             g.opacity.detach().reshape(-1).contiguous(), None if g.sh is None else g.sh.detach(), to_t(sc["T"]),
             to_t(sc["K"]), centre, st.visible, st.surfels, None, None, None, False)
    pg = ext.surfel_backward(*pargs) if st.lens is None else ext.surfel_lens_backward(*st.lens, *pargs)
    for k, mine in zip(GEOM, pg):
        res.append(gradrows.param_rows(f"param {k}", mine, od.g[k], PARAM_RTOL, PARAM_FLOOR, allowed))
    gradrows.assert_all(res)
    for k in GEOM:
        err = gradrows.global_rel(getattr(g, k).grad, od.g[k])
        print(f"end to end {k}: {err:.2e}")
        assert err < 2e-3, k
    err = gradrows.global_rel(F.grad, od.g["F"])
    print(f"end to end F: {err:.2e}")
    assert err < 2e-3
    assert (g.rgb.grad == 0).all()


# ---- median depth ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", CAMS)
@pytest.mark.parametrize("case", list(CASES))
def test_median_and_gradients_match_the_oracle(case, cam):
    c = CASES[case]
    sc = camera_scene(case)
    g = gaussians(sc)
    out = render(sc, g, case, cam, median=True)
    out["uv"].retain_grad()
    st = out["state"]
    lens, kc = lens_of(cam)
    ref = lambda G=None: mo.render(sc, grads=G, lens=lens, kc=kc, near=c.near, far=c.far, pad=c.pad,  # noqa: E731
                                   mh=c.mh, sort_z=to_np(st.surfels)[:, 3])
    o = ref()
    check_premises(sc, case, cam, out, oracle(sc, np.zeros(3), out, case, cam))
    assert (to_np(out["mask"]) == (o.visible == 0)).all(), "culling mask differs from the oracle"
    ids = to_np(st.median_ids).astype(np.int64)
    med = to_np(out["median"])[..., 0]
    hit = ids >= 0
    # the median surfel's z: partial-tile pixels have one too
    assert hit[:, c.W // TILE * TILE:].sum() >= 10 and hit[c.H // TILE * TILE:, :].sum() >= 10
    scale = max(np.abs(o.median).max(), 1e-12)
    differ = (ids != o.id) | (np.abs(med - o.median) > 1e-5 * scale)
    flagged = o.flag > 0
    n_other, n_flag = int((differ & ~flagged).sum()), int((differ & flagged).sum())
    print(f"forward: {n_other} unflagged + {n_flag} flagged of {differ.size} pixels differ; {int(flagged.sum())} "
          f"flagged")
    assert n_other == 0
    assert n_flag <= max(3, differ.size // 50)
    assert int(flagged.sum()) <= max(3, differ.size // 20)
    rng = np.random.default_rng(7)
    G = rng.normal(size=(c.H, c.W)) / np.sqrt(c.H * c.W)
    G[differ | flagged] = 0.0
    od = ref(G)
    Gt = to_t(G.astype(np.float32))
    (out["median"][..., 0] * Gt).sum().backward()
    rows = torch.zeros(st.N, 20, device=dev())
    native().surfel_median_backward(st.rays, st.surfels, st.H, st.W, c.mh, st.median_ids, Gt, rows)
    vis = to_np(~out["mask"]).astype(bool)
    allowed = gradrows.flips_allowed(int(vis.sum()))
    res = [gradrows.render_rows("median rows", to_np(rows)[vis][:, :19], od.rows[vis][:, :19], od.mass[vis][:, :19],
                                RENDER_C, EPS32, allowed)]
    ext = native()
    ref_rows = to_t(od.rows.astype(np.float32))
    ref_uv = (ext.surfel_uv_grad(st.vis_idx, st.surfels, ref_rows) if st.lens is None
              else ext.surfel_lens_uv_grad(*st.lens, st.K, st.vis_idx, st.surfels, ref_rows))
    err = gradrows.global_rel(out["uv"].grad, to_np(ref_uv))
    print(f"uv.grad: {err:.2e}")
    assert err < 2e-3
    centre = ext.camera_centre(to_t(sc["T"])) if c.sh else None
    pargs = (ref_rows, g.xyz.detach(), g.quaternion.detach(), g.scale.detach(),
             g.opacity.detach().reshape(-1).contiguous(), None if g.sh is None else g.sh.detach(), to_t(sc["T"]),
             to_t(sc["K"]), centre, st.visible, st.surfels, None, None, None, False)
    pg = ext.surfel_backward(*pargs) if st.lens is None else ext.surfel_lens_backward(*st.lens, *pargs)
    for k, mine in zip(("xyz", "quaternion"), pg):
        res.append(gradrows.param_rows(f"param {k}", mine, od.g[k], PARAM_RTOL, PARAM_FLOOR, allowed))
    gradrows.assert_all(res)
    gx = np.abs(od.g["xyz"]).max()
    assert np.abs(to_np(pg[2])).max() <= 1e-4 * gx
    for k in ("xyz", "quaternion"):
        err = gradrows.global_rel(getattr(g, k).grad, od.g[k])
        print(f"end to end {k}: {err:.2e}")
        assert err < 2e-3, k
    assert float(g.scale.grad.abs().max()) <= 1e-4 * gx
    assert bool((g.opacity.grad == 0).all()) and bool((g.rgb.grad == 0).all()) and bool((g.sh.grad == 0).all())


# ---- binning -----------------------------------------------------------------------------------------------------------
def grazing_scene_in(case, n=96, seed=3):
    """grazing_scene's surfels (large, seen at 60-88 degrees, a dozen near the camera plane) placed in the case's frame
    through its K, then mapped to world coordinates through the inverse of its pose, orientations included"""
    c = CASES[case]
    sc = grazing_scene(n=n, seed=seed)
    p = sc["xyz"].astype(np.float64)
    Kg = sc["K"].astype(np.float64)
    # the same spread of centres over the case's frame: [-20, W + 20] px
    u = (p[:, 0] * Kg[0, 0] / p[:, 2] + Kg[0, 2] + 20) / 296.0 * (c.W + 40) - 20
    v = (p[:, 1] * Kg[1, 1] / p[:, 2] + Kg[1, 2] + 20) / 296.0 * (c.H + 40) - 20
    z = p[:, 2]
    p = np.column_stack([(u - c.K[0, 2]) * z / c.K[0, 0], (v - c.K[1, 2]) * z / c.K[1, 1], z])
    T = c.T.astype(np.float64)
    xyz = (p - T[:3, 3]) @ T[:3, :3]
    # world orientation R^T R_q: the quaternion product q(R^T) q
    Rt = T[:3, :3].T
    w = np.sqrt(max(1e-12, 1 + np.trace(Rt))) / 2
    a = np.array([w, (Rt[2, 1] - Rt[1, 2]) / (4 * w), (Rt[0, 2] - Rt[2, 0]) / (4 * w), (Rt[1, 0] - Rt[0, 1]) / (4 * w)])
    b = sc["quaternion"].astype(np.float64)
    q = np.column_stack([a[0] * b[:, 0] - a[1] * b[:, 1] - a[2] * b[:, 2] - a[3] * b[:, 3],
                         a[0] * b[:, 1] + a[1] * b[:, 0] + a[2] * b[:, 3] - a[3] * b[:, 2],
                         a[0] * b[:, 2] - a[1] * b[:, 3] + a[2] * b[:, 0] + a[3] * b[:, 1],
                         a[0] * b[:, 3] + a[1] * b[:, 2] - a[2] * b[:, 1] + a[3] * b[:, 0]])
    return dict(sc, xyz=xyz.astype(np.float32), quaternion=q.astype(np.float32), T=c.T, K=c.K, H=c.H, W=c.W), z


def test_binning_is_conservative_for_large_grazing_surfels_under_case_c():
    c = CASES["C"]
    sc, z = grazing_scene_in("C")
    g = gaussians(sc, requires_grad=False)
    out = render(sc, g, "C", "pinhole")
    o = so.render(sc, np.zeros(3), near=c.near, far=c.far, pad=c.pad, mh=c.mh,
                  sort_z=to_np(out["state"].surfels)[:, 3])
    assert (to_np(out["mask"]) == (o.visible == 0)).all()
    # surfels in the frustum whose disk reaches behind the camera plane are culled, and near ones that do not are drawn
    in_frustum = (z >= c.near) & (o.uv[:, 0] >= -c.pad) & (o.uv[:, 0] <= c.W + c.pad) & (o.uv[:, 1] >= -c.pad) & (
        o.uv[:, 1] <= c.H + c.pad)
    assert (in_frustum & (o.visible == 0)).sum() >= 1 and (in_frustum & (o.visible == 1) & (z < 0.8)).sum() >= 1
    assert (o.alpha[:, c.W // TILE * TILE:] > 0).sum() >= 10 and (o.alpha[c.H // TILE * TILE:] > 0).sum() >= 10
    # a tile the binning missed would differ over whole pixel blocks: only isolated rounding flips are allowed
    compare_forward(out, o, allowed_frac=0.0005, tol=2e-4)


# ---- the id-list pair source -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", CAMS)
def test_id_list_pair_source_gives_the_keys_results(cam):
    """Every surfel tile kernel fed the sorted pairs as (tile | depth | id) keys and as the ids alone: the forwards are
    bit-identical and the backward rows equal up to the order of their atomic adds."""
    c = CASES["A"]
    sc = camera_scene("A")
    N = sc["xyz"].shape[0]
    g = gaussians(sc, requires_grad=False)
    out = render(sc, g, "A", cam, bg=(0.2, 0.4, 0.7))
    st = out["state"]
    assert st.id_bits > 0 and st.keys_sorted.numel() >= st.P > 0
    ids = (st.keys_sorted & ((1 << st.id_bits) - 1)).int().contiguous()
    assert int(ids.min()) >= 0 and int(ids.max()) < N
    D = 5
    F = torch.randn(N, D, device=dev(), generator=torch.Generator(dev()).manual_seed(5))
    fpad = torch.nn.functional.pad(F, (0, 3)).contiguous()
    G = {k: to_t(v.astype(np.float32)) for k, v in upstream(sc, seed=6).items()}
    Gf = torch.randn(c.H, c.W, D, device=dev(), generator=torch.Generator(dev()).manual_seed(7)) / c.W
    ext = native()
    per = {}
    for src, (keys, idl, id_bits) in {"keys": (st.keys_sorted, st.ids_sorted, st.id_bits),
                                      "ids": (None, ids, 0)}.items():
        pairs = (st.surfels, st.ranges, st.background, st.H, st.W, st.P, keys, idl, id_bits, c.near, st.m_scale, c.mh)
        fw = (ext.surfel_render_forward(*pairs) if st.lens is None
              else ext.surfel_lens_render_forward(st.rays, *pairs))
        image, depth, alpha, normal, dist, last, totals = fw
        fpairs = (st.rays, st.surfels, st.ranges, st.H, st.W, st.P, keys, idl, id_bits, c.mh, last)
        fmap = ext.surfel_features_forward(*fpairs, fpad, D)
        median, median_ids = ext.surfel_median_forward(*fpairs)
        bargs = (st.N, st.surfels, st.ranges, st.background, st.H, st.W, st.P, keys, idl, id_bits, c.near,
                 st.m_scale, c.mh, alpha, last, totals, G["image"], G["depth"], G["alpha"], G["normal"], G["dist"])
        rows = (ext.surfel_render_backward(*bargs) if st.lens is None
                else ext.surfel_lens_render_backward(st.rays, *bargs))
        frows = torch.zeros(N, 20, device=dev())
        gF = ext.surfel_features_backward(*fpairs, totals, fpad, D, Gf, frows)
        per[src] = dict(image=image, depth=depth, alpha=alpha, normal=normal, dist=dist, last=last, totals=totals,
                        fmap=fmap, median=median, median_ids=median_ids, rows=rows, frows=frows, gF=gF)
    a, b = per["keys"], per["ids"]
    # the keys path reproduces the render that rasterize_surfels returned
    for k in ("image", "depth", "alpha", "normal", "dist"):
        assert (bits(a[k]) == bits(out[k])).all(), k
    assert float(a["alpha"].max()) > 0.5 and int((a["median_ids"] >= 0).sum()) > c.H * c.W // 2
    for k in ("image", "depth", "alpha", "normal", "dist", "totals", "fmap", "median"):
        assert (bits(a[k]) == bits(b[k])).all(), k
    for k in ("last", "median_ids"):
        assert torch.equal(a[k], b[k]), k
    for k in ("rows", "frows", "gF"):
        err = gradrows.global_rel(b[k], to_np(a[k]))
        print(f"{k}: {err:.2e}")
        assert float(a[k].abs().max()) > 0 and err < 1e-5, k


def test_id_list_path_end_to_end_at_720p():
    """1.2 M gaussians at 720p: far = inf needs 32-bit depth keys and leaves no room for the 21-bit id (the pairs take
    the id list), far = 1000 packs (tile | depth | id) keys.  The depth order is the same, so every map but the
    distortion is bit-identical; the distortion scales with m_scale^2; the gradients (none on the distortion) agree up
    to the order of the atomic adds."""
    H, W, D = 720, 1280, 5
    g0 = synth.make_gaussians(1_200_000, "720p", sh_degree=0, seed=0, device=dev())
    N = g0.xyz.shape[0]
    K, T = synth.make_camera("720p", device=dev()).K, synth.make_pose(0, 3, device=dev())
    F0 = torch.randn(N, D, device=dev(), generator=torch.Generator(dev()).manual_seed(1))
    gen = torch.Generator(dev()).manual_seed(2)
    Gs = {k: torch.randn(H, W, ch, device=dev(), generator=gen) / math.sqrt(H * W)
          for k, ch in (("image", 3), ("depth", 1), ("alpha", 1), ("normal", 3), ("median", 1), ("fmap", D))}
    runs = {}
    for far in (math.inf, 1000.0):
        g = type(g0)(*(None if t is None else t.clone().requires_grad_(True) for t in
                       (g0.xyz, g0.rgb, g0.opacity, g0.scale, g0.quaternion, g0.sh)))
        F = F0.clone().requires_grad_(True)
        out = rasterize_surfels(g, T, Camera(W, H, K), 0.3, far, 100.0, 3.0, torch.full((3,), 0.3, device=dev()),
                                return_state=True, features=F, median_depth=True)
        names = ("image", "mask", "uv", "depth", "alpha", "normal", "dist", "median", "fmap", "state")
        o = dict(zip(names, out))
        sum((o[k] * Gs[k]).sum() for k in Gs).backward()
        o["grads"] = {k: getattr(g, k).grad for k in ("xyz", "quaternion", "scale", "opacity", "rgb")}
        o["grads"]["F"] = F.grad
        runs[far] = o
    a, b = runs[math.inf], runs[1000.0]
    assert a["state"].id_bits == 0 and a["state"].keys_sorted.numel() == 0 and a["state"].ids_sorted.numel() > 0
    assert b["state"].id_bits > 0 and b["state"].ids_sorted.numel() == 0
    assert a["state"].P == b["state"].P and a["state"].M == b["state"].M > 500_000
    assert bool((a["mask"] == b["mask"]).all()) and (bits(a["uv"]) == bits(b["uv"])).all()
    for k in ("image", "depth", "alpha", "normal", "median", "fmap"):
        assert (bits(a[k]) == bits(b[k])).all(), k
    assert torch.equal(a["state"].median_ids, b["state"].median_ids)
    # the kernels take m_scale in fp32; m = m_scale (1 - near / z) then differs by the ratio up to one rounding, and
    # the distortion's three running sums (each at most alpha m^2 <= alpha) cancel: a few fp32 roundings of alpha
    r = float(np.float32(b["state"].m_scale)) / float(np.float32(a["state"].m_scale))
    assert r > 1.0 + 1e-4
    da, db = to_np(a["dist"]), to_np(b["dist"]) / r ** 2
    ratio = np.abs(db - da) / (EPS32 * np.maximum(to_np(a["alpha"]), 1e-30))
    print(f"distortion / m_scale ratio^2: {gradrows.global_rel(db, da):.2e} global, worst |diff| / (eps alpha) "
          f"{ratio.max():.3g}")
    assert da.max() > 0 and ratio.max() <= 64
    for k in a["grads"]:
        err = gradrows.global_rel(b["grads"][k], to_np(a["grads"][k]))
        print(f"{k}: {err:.2e}")
        assert err < 1e-5, k
