"""Anti-aliased mode (rasterize(antialiased=True)): the CPU oracle's semantics and gradients, the compensation's known
answers, the argument errors and the new kernels in the built library.  No GPU needed."""
import re

import numpy as np
import pytest
import torch

from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera, Gaussians
from tests import antialiased_oracle as aao
from tests import depth_alpha_oracle as dao
from tests.scenes import np_scene
from tests.test_sass_evidence import _tool_output, sass_counts

SKIP = 1.0 / 255.0


def _forward(sc, mod=aao, **over):
    s = dict(sc, **over)
    return mod.rasterize(s["xyz"], s["quaternion"], s["scale"], s["opacity"], s["rgb"], s["sh"], s["T"], s["K"],
                         s["H"], s["W"], mh_dist=s.get("mh", 3.0), background=np.full(3, s.get("bg", 0.5), s["xyz"].dtype))


def _upstream(H, W, seed=1):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((H, W, 3)) / (3 * H * W), rng.standard_normal((H, W)) / (H * W),
            rng.standard_normal((H, W)) / (H * W))


# fp64 finite differences ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("sh_degree", [0, 3])
@pytest.mark.parametrize("maps", [False, True], ids=["image", "image+depth+alpha"])
def test_fp64_antialiased_backward_matches_finite_differences(sh_degree, maps):
    """<G,image> (+ <Gd,depth> + <Ga,alpha>) against central differences of the dilated fp64 forward, every parameter,
    on a scene with sub-pixel (sigma 0.15 px) and large (8 px) splats.  The compensation is live: rho differs from 1
    on most gaussians (the oracle's plain fp64 branch has no dilation, where rho would be 1).  With SH, xyz is checked
    on the depth and alpha terms alone (the reference sends no gradient to xyz through the view direction)."""
    sc = np_scene(128, "tiny", sh_degree=sh_degree, dtype=np.float64, sigma_px=(0.6, 1.2, 0.15, 8.0))
    G, Gd, Ga = _upstream(64, 64)
    if not maps:
        Gd, Ga = np.zeros_like(Gd), np.zeros_like(Ga)
    rng = np.random.default_rng(2)
    o = _forward(sc)
    assert o.keep.sum() > 64 and len(o.sorted_idx) > 200 and (o.alpha > 0.5).any()
    assert (np.abs(o.rho - 1) > 1e-3).mean() > 0.8 and o.rho.min() < 0.3 and o.rho.max() > 0.99
    # the render stage saw the dilated covariance: the fp64 walk of the undilated one gives another image
    assert np.abs(o.image - _forward(sc, mod=dao).image).max() > 1e-2

    def check(names, G, Gd, Ga):
        d = aao.rasterize_backward(o, G, Gd, Ga)

        def loss(**over):
            p = _forward(sc, **over)
            return float((p.image * G).sum() + (p.depth * Gd).sum() + (p.alpha * Ga).sum())

        vis = np.flatnonzero(o.keep)
        h = 1e-6
        for name in names:
            grad, base = getattr(d, name), sc[name]
            scale = np.abs(grad).max()
            assert scale > 0, name
            for _ in range(6):
                i = int(rng.choice(vis))
                idx = (i,) + tuple(int(rng.integers(0, s)) for s in base.shape[1:])
                plus, minus = base.copy(), base.copy()
                plus[idx] += h
                minus[idx] -= h
                fd = (loss(**{name: plus}) - loss(**{name: minus})) / (2 * h)
                assert abs(fd - grad[idx]) <= 2e-5 * scale + 1e-12, (name, idx, fd, grad[idx])

    if sh_degree:
        check(["quaternion", "scale", "opacity", "rgb", "sh"], G, Gd, Ga)
        if maps:
            check(["xyz"], np.zeros_like(G), Gd, Ga)
    else:
        check(["xyz", "quaternion", "scale", "opacity", "rgb"], G, Gd, Ga)


# known answers for rho ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_rho_known_answers(dtype):
    rho, out = aao.compensate(np.array([[0.75, 0.0, 0.75]], dtype), np.array([0.5], dtype))
    assert rho[0] == 0.75 and out[0] == 0.375           # sqrt(0.5625 / 1), exact in both dtypes
    s = np.array([0.01, 0.02, 0.1, 0.3, 1.0, 4.0, 30.0], np.float64)
    rho, _ = aao.compensate(np.stack([s, 0 * s, s], 1).astype(dtype), np.ones(len(s), dtype))
    np.testing.assert_allclose(rho, s / (s + 0.25), rtol=4e-7 if dtype == np.float32 else 1e-15)
    rho, _ = aao.compensate(np.array([[1e4, 0.0, 1e4]], dtype), np.ones(1, dtype))   # 1e4 px^2: 1 - 2.5e-5
    assert abs(float(rho[0]) - 1) <= 3e-5, rho


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_rho_is_zero_with_finite_zero_gradients_where_det0_is_not_positive(dtype):
    """det0 <= 0 (a needle seen end-on: c0 c2 == bh^2, or below it by rounding): rho == 0, and the gradient through
    rho is exactly zero, not 0 * inf = NaN, whatever the upstream gradient on the compensated opacity."""
    c = np.array([[4.0, 8.0, 4.0], [1.0, 2.0000002, 1.0], [0.0, 0.0, 3.0]], dtype)
    if dtype == np.float32:
        c = np.concatenate([c, np.array([[1e-30, 0.0, 1e-30]], dtype)])   # c0 c2 underflows to 0
    rho, out = aao.compensate(c, np.full(len(c), 0.9, dtype))
    assert (rho == 0).all() and (out == 0).all()
    g = aao.rho_grad(c, rho)
    assert np.isfinite(g).all() and not g.any()


# mass known answer ----------------------------------------------------------------------------------------------
def isolated_scene(variances, sigma=0.9, spacing=24, dtype=np.float32):
    """One isotropic gaussian per cell of a spacing x spacing px grid, on the optical axis' plane z = 4, screen
    variance variances[k] px^2 (camera f = 256, identity pose)."""
    n = len(variances)
    cols = int(np.ceil(np.sqrt(n)))
    H = W = cols * spacing
    f, z = 256.0, 4.0
    k = np.arange(n)
    u = (k % cols + 0.5) * spacing + 0.3 * np.sin(k)        # off the pixel grid
    v = (k // cols + 0.5) * spacing + 0.3 * np.cos(k)
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], dtype)
    xyz = np.stack([(u - W / 2) * z / f, (v - H / 2) * z / f, np.full(n, z)], 1)
    sw = np.sqrt(np.asarray(variances, np.float64)) * z / f
    logit = np.log(sigma / (1 - sigma))
    return dict(xyz=xyz.astype(dtype), quaternion=np.tile(np.array([1.0, 0, 0, 0], dtype), (n, 1)),
                scale=np.log(np.stack([sw, sw, sw], 1)).astype(dtype), opacity=np.full((n, 1), logit, dtype),
                rgb=np.ones((n, 3), dtype), sh=None, T=np.eye(4, dtype=dtype), K=K, H=H, W=W, mh=6.0, bg=0.0), u, v


def test_mass_of_isolated_splats_known_answer():
    """The pixel sum of one splat's alpha is the integral of alpha above the 1/255 skip, 2 pi sqrt(det) (opa - 1/255),
    det = the dilated determinant, opa the record's opacity — in both modes.  With the compensation that is
    2 pi (sigma(o) sqrt(det0) - sqrt(det) / 255): the mass no longer grows with the dilation."""
    var = np.geomspace(0.02, 4.0, 16)
    sc, u, v = isolated_scene(var)
    for mod in (dao, aao):
        o = _forward(sc, mod=mod)
        assert o.keep.all()
        c0, c1, c2 = (o.conic[:, k].astype(np.float64) for k in range(3))
        det = (c0 + 0.25) * (c2 + 0.25) - 0.25 * c1 * c1
        want = 2 * np.pi * np.sqrt(det) * (o.opacity.astype(np.float64) - SKIP)
        got = np.array([o.alpha[int(y) - 11:int(y) + 12, int(x) - 11:int(x) + 12].sum() for x, y in zip(u, v)])
        assert np.isclose(got.sum(), o.alpha.sum())     # every splat's alpha lies in its own window
        np.testing.assert_allclose(got, want, rtol=0.03)
        if mod is aao:
            det0 = c0 * c2 - 0.25 * c1 * c1
            np.testing.assert_allclose(got, 2 * np.pi * (0.9 * np.sqrt(det0) - np.sqrt(det) / 255), rtol=0.03)
            aa = got
        else:
            default = got
    # the dilation adds mass to the smallest splats only: x 1 + 0.25 / var without the compensation
    assert default[0] > 8 * aa[0] and abs(default[-1] / aa[-1] - 1.0625) < 0.01


# resolution consistency -----------------------------------------------------------------------------------------
def subpixel_scene(H, W, n=3000, seed=5, down=1):
    """n gaussians of 0.05-0.4 px^2 screen variance at H x W, rendered at H/down x W/down with K scaled so that a
    low-resolution pixel centre lies at the centre of its down x down block."""
    rng = np.random.default_rng(seed)
    f, z = float(W), rng.uniform(4.0, 6.0, n)
    u, v = rng.uniform(0, W, n), rng.uniform(0, H, n)
    xyz = np.stack([(u - W / 2) * z / f, (v - H / 2) * z / f, z], 1)
    sw = np.sqrt(rng.uniform(0.05, 0.4, (n, 3))) * z[:, None] / f
    K = np.array([[f / down, 0, (W / 2 - (down - 1) / 2) / down], [0, f / down, (H / 2 - (down - 1) / 2) / down],
                  [0, 0, 1]])
    f32 = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    return dict(xyz=f32(xyz), quaternion=f32(rng.standard_normal((n, 4))), scale=f32(np.log(sw)),
                opacity=f32(rng.uniform(0.5, 3.0, (n, 1))), rgb=f32(rng.uniform(0, 1, (n, 3)) / 0.28209479177387814),
                sh=None, T=np.eye(4, dtype=np.float32), K=f32(K), H=H // down, W=W // down, bg=0.0)


def test_resolution_consistency():
    """Sub-pixel splats rendered at 256 x 256, 4 x 4 average-pooled, against the same scene at 64 x 64.  Without the
    compensation the low resolution's dilation blows every splat up to ~16 times its full-resolution mass; with it the
    two images agree far better (measured with this oracle: mean |error| 0.0095 anti-aliased, 0.26 default)."""
    err = {}
    for mod in (dao, aao):
        full = _forward(subpixel_scene(256, 256), mod=mod).image.astype(np.float64)
        low = _forward(subpixel_scene(256, 256, down=4), mod=mod).image.astype(np.float64)
        pooled = full.reshape(64, 4, 64, 4, 3).mean((1, 3))
        err[mod.__name__] = float(np.abs(pooled - low).mean())
    print(err)
    assert err[aao.__name__] < 0.25 * err[dao.__name__]


# argument errors ------------------------------------------------------------------------------------------------
def test_argument_errors():
    sc = np_scene(50, "tiny", sh_degree=1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    g = Gaussians(t(sc["xyz"]), t(sc["rgb"]), t(sc["opacity"]), t(sc["scale"]), t(sc["quaternion"]), t(sc["sh"]))
    cam, bg = Camera(64, 64, t(sc["K"])), torch.full((3,), 0.5)
    with pytest.raises(ValueError):
        rasterize(g, t(sc["T"]), cam, 0.3, 500.0, 100, 3.0, False, bg, antialiased=True)
    g64 = Gaussians(*(x.double() for x in (g.xyz, g.rgb, g.opacity, g.scale, g.quaternion)), None)
    with pytest.raises(TypeError):
        rasterize(g64, t(sc["T"]).double(), Camera(64, 64, t(sc["K"]).double()), 0.3, 500.0, 100, 3.0, True,
                  bg.double(), antialiased=True)


# the kernels in the built library -------------------------------------------------------------------------------
def _usage():
    usage = {}
    for name, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _tool_output("--dump-resource-usage")):
        usage[name] = {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
    return usage


AA_KERNELS = {"k_preprocess_fwd_aa": "k_preprocess_fwd", "k_preprocess_bwd_aa": "k_preprocess_bwd",
              "k_preprocess_bwd_depth_aa": "k_preprocess_bwd_depth"}


def test_antialiased_kernels_stage_through_tma_and_use_no_local_memory():
    """Every instantiation of the new kernels is in the library and keeps the TMA bulk copies (UBLKCP) of its default
    counterpart.  The backward kernels neither spill nor keep anything in local memory (no STL / LDL); the forward adds
    no local-memory access to the default forward's (whose 32-byte frame holds the pose inversion's vectors)."""
    counts, usage = sass_counts(), _usage()
    for new, old in AA_KERNELS.items():
        for args in ("ILi1ELb0E", "ILi4ELb1E", "ILi9ELb1E", "ILi16ELb1E"):
            frag_new, frag_old = f"{len(new)}{new}{args}", f"{len(old)}{old}{args}"
            c_new = next((c for n, c in counts.items() if frag_new in n), None)
            c_old = next(c for n, c in counts.items() if frag_old in n)
            assert c_new is not None, frag_new
            assert c_new["UBLKCP"] == c_old["UBLKCP"] >= 1, (frag_new, c_new["UBLKCP"], c_old["UBLKCP"])
            local = (c_new["STL"], c_new["LDL"])
            assert local == ((0, 0) if "bwd" in new else (c_old["STL"], c_old["LDL"])), (frag_new, local)
            u_new = next(v for k, v in usage.items() if frag_new in k)
            u_old = next(v for k, v in usage.items() if frag_old in k)
            assert u_new["LOCAL"] == 0 and u_new["STACK"] <= u_old["STACK"], (frag_new, u_new, u_old)
