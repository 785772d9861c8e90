"""The oracle's per-entry gradient masses, its per-pixel SH mode, and the per-row gradient comparison of
tests/gradrows.py: no GPU needed."""
from pathlib import Path

import numpy as np
import pytest
import torch

from gaussian_splatting_b200.structs import Camera
from gaussian_splatting_b200.utils import compute_rays_in_world_frame
from oracle import cpu_oracle as orc
from tests import gradrows, scenes

FIELDS = ("rgb", "opacity", "uv", "conic")


def _oracle(sc, G, **kw):
    o = orc.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], sc["K"],
                      sc["H"], sc["W"], background=np.full(3, 0.5, sc["xyz"].dtype), **kw)
    return o, orc.rasterize_backward(o, G)


def view_dirs(sc):
    return compute_rays_in_world_frame(Camera(sc["W"], sc["H"], torch.from_numpy(sc["K"])),
                                       torch.from_numpy(sc["T"])).numpy()


@pytest.fixture(scope="module")
def tiny_sh3():
    sc = scenes.np_scene(2000, "tiny", sh_degree=3, seed=1, view=2, n_views=3, sigma_px=(2.0, 0.5, 0.5, 8.0))
    G = np.random.default_rng(0).standard_normal((64, 64, 3)).astype(np.float32) / (3 * 64 * 64)
    o, d = _oracle(sc, G)
    return sc, o, d


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n_sh", [1, 4])
def test_mass_of_one_gaussian_on_one_pixel(dtype, n_sh):
    """One term per entry: the rgb mass is |term| exactly, the others the magnitudes of the term's parts, so at
    least |term| (up to the rounding of the term itself)."""
    rng = np.random.default_rng(n_sh)
    uv = np.array([[0.3, -0.2]], dtype)
    conic = np.array([[0.9, 0.3, 1.4]], dtype)
    opacity = np.array([[0.7]], dtype)
    rgb = rng.standard_normal((1, 3, n_sh)).astype(dtype) if n_sh > 1 else rng.uniform(0, 1, (1, 3)).astype(dtype)
    vd = np.array([[[0.2, -0.3, 0.93]]], dtype)
    ranges, idx = np.array([0, 1], np.int32), np.array([0], np.int32)
    bg = np.full(3, 0.5, dtype)
    _, n, w = orc.render_forward(uv, opacity, rgb, conic, vd, ranges, idx, bg, 1, 1)
    assert n[0, 0] == 1
    G = np.array([[[0.4, -1.1, 0.6]]], dtype)
    *g, m = orc.render_backward(uv, opacity, rgb, conic, vd, ranges, idx, bg, n, w, G, mass=True)
    for k, gk in zip(FIELDS, g):
        assert (np.abs(gk) > 0).all(), k
        assert (getattr(m, k) * (1 + 4 * gradrows.EPS[np.dtype(dtype)]) >= np.abs(gk)).all(), k
    np.testing.assert_array_equal(m.rgb, np.abs(g[0]))


def test_mass_bounds_the_sum(tiny_sh3):
    sc, o, d = tiny_sh3
    for k in FIELDS:
        mass, s = getattr(d.mass, k), getattr(d.render, k)
        assert mass.shape == s.shape and (mass * (1 + 2.0 ** -20) >= np.abs(s)).all(), k
        assert (mass[o.keep].reshape(int(o.keep.sum()), -1).max(1) > 0).mean() > 0.5, k       # most visible gaussians reach some pixel
        assert (mass[~o.keep] == 0).all(), k


def test_per_pixel_sh_image_matches_the_reference_fixture():
    """The reference's per-pixel SH case of test/test_rasterize.py, against its image stored by the compiled
    reference (row sample + column sums)."""
    gd = np.load(Path(__file__).resolve().parent / "golden" / "fixture6_fp32.npz")
    fx = scenes.reference_fixture()
    fx = dict(fx, opacity=scenes.inverse_sigmoid(fx["opacity"]), sh=np.full((6, 3, 15), 0.1, np.float32))
    o = orc.rasterize(fx["xyz"], fx["quaternion"], fx["scale"], fx["opacity"], fx["rgb"], fx["sh"], fx["T"], fx["K"],
                      480, 640, 0.3, 100.0, 10.0, 3.0, background=np.zeros(3, np.float32), use_sh_precompute=False,
                      view_dirs=view_dirs(fx))
    assert o.rgb.shape == (3, 3, 16)
    img = o.image.reshape(-1, 3).astype(np.float64)
    ref = gd["image_sh_perpixel_rows"]
    rows = scenes.sample_rows(img.shape[0], ref.shape[0])
    assert np.abs(img[rows] - ref).max() < 1e-5 * float(gd["image_sh_perpixel_absmax"])
    assert np.abs(img.sum(0) - gd["image_sh_perpixel_colsum"]).max() < 1e-5 * float(gd["image_sh_perpixel_colabs"].max())
    # precomputed SH along each gaussian's own view direction gives a different image
    pre = orc.rasterize(fx["xyz"], fx["quaternion"], fx["scale"], fx["opacity"], fx["rgb"], fx["sh"], fx["T"], fx["K"],
                        480, 640, 0.3, 100.0, 10.0, 3.0, background=np.zeros(3, np.float32))
    assert np.abs(pre.image - o.image).max() > 1e-4


@pytest.mark.parametrize("sh_degree", [1, 2])
def test_per_pixel_sh_gradients_split_into_rgb_and_sh(sh_degree):
    sc = scenes.np_scene(300, "tiny", sh_degree=sh_degree, seed=2, dtype=np.float64, sigma_px=(3.0, 0.4, 1.0, 6.0))
    G = np.random.default_rng(1).standard_normal((64, 64, 3)) / (3 * 64 * 64)
    o, d = _oracle(sc, G, use_sh_precompute=False, view_dirs=view_dirs(sc))
    n_sh = (sh_degree + 1) ** 2
    assert o.rgb.shape[1:] == (3, n_sh) and d.render.rgb.shape == (300, 3, n_sh)
    np.testing.assert_array_equal(d.rgb, d.render.rgb[:, :, 0])
    np.testing.assert_array_equal(d.sh, d.render.rgb[:, :, 1:])
    # finite differences of the oracle's own fp64 forward on a few sh and rgb entries of visible gaussians
    rng = np.random.default_rng(3)
    h = 1e-6
    for name in ("sh", "rgb"):
        grad = getattr(d, name)
        for _ in range(4):
            i = int(rng.choice(np.flatnonzero(o.keep)))
            idx = (i,) + tuple(int(rng.integers(0, s)) for s in sc[name].shape[1:])
            vals = []
            for sgn in (1, -1):
                p = sc[name].copy()
                p[idx] += sgn * h
                vals.append(float((_oracle(dict(sc, **{name: p}), G, use_sh_precompute=False,
                                           view_dirs=view_dirs(sc))[0].image * G).sum()))
            fd = (vals[0] - vals[1]) / (2 * h)
            assert abs(fd - grad[idx]) <= 2e-5 * np.abs(grad).max() + 1e-12, (name, idx, fd, grad[idx])


def _faint_rows(ref, keep, frac=0.1):
    vis = np.flatnonzero(keep & (np.abs(ref).reshape(len(ref), -1).max(1) > 0))
    mag = np.abs(ref[vis]).reshape(len(vis), -1).max(1)
    return vis[np.argsort(mag)[:max(2, int(frac * len(vis)))]]


@pytest.fixture(scope="module")
def tiny_sh2_fp64():
    sc = scenes.np_scene(2000, "tiny", sh_degree=2, seed=1, view=2, n_views=3, dtype=np.float64,
                         sigma_px=(2.0, 0.5, 0.5, 8.0))
    G = np.random.default_rng(0).standard_normal((64, 64, 3)) / (3 * 64 * 64)
    o, d = _oracle(sc, G)
    return sc, o, d


@pytest.mark.parametrize("perturb", ["zero_faint", "swap_faint"])
def test_row_check_catches_what_the_global_check_misses(tiny_sh3, tiny_sh2_fp64, perturb):
    """Negative control on oracle data: its sums rounded to the branch's precision pass the row check; zeroing the
    rows of the faintest 10 % of the visible gaussians (fp32 scene) or swapping two faint rows (fp64 scene, where no
    row may miss its bound) passes the old global criterion and fails the row check."""
    sc, o, d = tiny_sh3 if perturb == "zero_faint" else tiny_sh2_fp64
    dt = sc["xyz"].dtype
    allowed = gradrows.flips_allowed(int(o.keep.sum()), dt)
    eps = gradrows.EPS[np.dtype(dt)]

    def perturbed(ref):
        faint = _faint_rows(ref, o.keep)
        bad = ref.astype(dt)
        if perturb == "zero_faint":
            bad[faint] = 0
        else:
            a, b = faint[-1], faint[-2]
            bad[[a, b]] = bad[[b, a]]
            assert not np.array_equal(bad[a], ref[a])
        assert gradrows.global_rel(bad, ref) < gradrows.GLOBAL_TOL
        return bad

    for k in FIELDS:
        ref, mass = getattr(d.render, k), getattr(d.mass, k)
        assert gradrows.render_rows(k, ref.astype(dt), ref, mass, gradrows.RENDER_C[k], eps, allowed).ok, k
        r = gradrows.render_rows(k, perturbed(ref), ref, mass, gradrows.RENDER_C[k], eps, allowed)
        assert not r.ok, (k, str(r))
    for k in ("xyz", "scale", "sh"):
        ref = getattr(d, k)
        assert gradrows.param_rows(k, ref.astype(dt), ref, gradrows.PARAM_RTOL, gradrows.PARAM_FLOOR, allowed).ok, k
        r = gradrows.param_rows(k, perturbed(ref), ref, gradrows.PARAM_RTOL, gradrows.PARAM_FLOOR, allowed)
        assert not r.ok, (k, str(r))
