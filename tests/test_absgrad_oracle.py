"""Absolute screen-space gradients (rasterize(absgrad=True)): the CPU oracle's definition and properties, the absgrad
kernels in the built library, and the argument errors that need no GPU."""
import re

import numpy as np
import pytest

from tests import absgrad_oracle as abo
from tests import antialiased_oracle as aao
from tests import depth_alpha_oracle as dao
from tests.gradrows import EPS
from tests.scenes import np_scene
from tests.test_sass_evidence import _tool_output


def tiny(sh_degree=0, n=300, seed=0, H=20, W=24, dtype=np.float64):
    """A 64x64 synthetic scene seen through an H x W window (same focal length, centred principal point)."""
    sc = np_scene(n, "tiny", sh_degree=sh_degree, seed=seed, dtype=dtype, sigma_px=(3.0, 0.4, 1.0, 6.0))
    K = sc["K"].copy()
    K[0, 2], K[1, 2] = W / 2.0, H / 2.0
    return dict(sc, K=K, H=H, W=W)


def forward(sc, antialiased=False):
    f = aao.rasterize if antialiased else dao.rasterize
    return f(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], sc["K"], sc["H"],
             sc["W"], background=np.full(3, 0.5, sc["xyz"].dtype))


def upstream(H, W, seed=1, depth=False):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((H, W, 3)) / (3 * H * W)
    if not depth:
        return G, None, None
    return G, rng.standard_normal((H, W)) / (H * W), rng.standard_normal((H, W)) / (H * W)


def one_hot_sum(o, G, Gd, Ga):
    """sum over pixels p of |g_uv| of the EXISTING oracle backward (depth_alpha_oracle.render_backward, gradchecked)
    run with the upstream gradients of pixel p alone."""
    H, W = o.n.shape
    oo = o if not hasattr(o, "render_conic") else type(o)(**dict(vars(o), conic=o.render_conic))
    zero = np.zeros((H, W))
    total = np.zeros((o.uv.shape[0], 2))
    for py in range(H):
        for px in range(W):
            G1, Gd1, Ga1 = np.zeros_like(G), zero.copy(), zero.copy()
            G1[py, px] = G[py, px]
            if Gd is not None:
                Gd1[py, px], Ga1[py, px] = Gd[py, px], Ga[py, px]
            g, _, _ = dao.render_backward(oo, G1, Gd1, Ga1)
            total += np.abs(g.uv)
    return total


CASES = [("sh0", 0, False, False), ("sh3", 3, False, False), ("sh0 depth/alpha", 0, True, False),
         ("sh3 antialiased", 3, False, True)]


@pytest.mark.parametrize("name,sh,depth,aa", CASES, ids=[c[0] for c in CASES])
def test_fp64_absgrad_is_the_sum_of_one_hot_uv_gradients(name, sh, depth, aa):
    """The definition: sum_p |d <G_p, out_p> / d uv| equals the sum over H*W one-hot backward passes of the existing
    fp64 oracle of |uv gradient|, to 1e-12 relative (only the summation order differs)."""
    sc = tiny(sh)
    o = forward(sc, aa)
    M = o.uv.shape[0]
    assert M >= 20 and len(o.sorted_idx) >= 20, (M, len(o.sorted_idx))
    G, Gd, Ga = upstream(sc["H"], sc["W"], depth=depth)
    r = abo.uv_backward(o, G, Gd, Ga)
    ref = one_hot_sum(o, G, Gd, Ga)
    assert (ref > 0).sum() >= 20
    np.testing.assert_allclose(r.absgrad, ref, rtol=1e-12, atol=1e-300)
    # the signed sums are the existing oracle's
    full, _, _ = dao.render_backward(o if not aa else type(o)(**dict(vars(o), conic=o.render_conic)), G,
                                     np.zeros((sc["H"], sc["W"])) if Gd is None else Gd,
                                     np.zeros((sc["H"], sc["W"])) if Ga is None else Ga)
    np.testing.assert_allclose(r.uv, full.uv, rtol=1e-12, atol=1e-12 * np.abs(full.uv).max())
    if aa:
        assert (o.rho < 0.999).any()  # the compensation is live


def test_fp32_kernel_order_agrees_with_the_one_hot_sums():
    """The fp32 branch forms the absolute values in the tile kernel's order (eu = 2c*hu - (b+b)*hv, times |rdet| per
    gaussian); the one-hot sums of the fp32 oracle take |d_u| in the reference's order.  Same terms, different
    roundings: within a few ulp of the mass."""
    sc = tiny(3, dtype=np.float32)
    o = forward(sc)
    G = upstream(sc["H"], sc["W"])[0].astype(np.float32)
    r = abo.uv_backward(o, G)
    ref = one_hot_sum(o, G, None, None)
    assert (ref > 0).sum() >= 20
    assert np.all(np.abs(r.absgrad - ref) <= 64 * EPS[np.dtype(np.float32)] * r.mass), \
        float((np.abs(r.absgrad - ref) / np.maximum(r.mass, 1e-300)).max())


@pytest.fixture(scope="module")
def fp64_case():
    sc = tiny(3)
    o = forward(sc)
    G, Gd, Ga = upstream(sc["H"], sc["W"], depth=True)
    return sc, o, G, Gd, Ga, abo.uv_backward(o, G, Gd, Ga)


def test_absgrad_bounds_the_signed_sum_and_is_bounded_by_the_mass(fp64_case):
    _, _, _, _, _, r = fp64_case
    tol = 1e-12 * r.mass
    assert np.all(r.absgrad >= np.abs(r.uv) - tol)
    assert np.all(r.absgrad <= r.mass + tol)
    # on this scene the per-pixel terms do cancel: absgrad is well above |uv.grad| somewhere
    assert (r.absgrad > 2 * np.abs(r.uv) + tol).any()


def test_absgrad_is_even_and_degree_one_homogeneous_in_the_upstream_gradient(fp64_case):
    _, o, G, Gd, Ga, r = fp64_case
    # G -> -G negates every term exactly and 2G doubles it; the pixels' terms are summed with atomics in any order
    for k in (-1.0, 2.0, 0.3):
        s = abo.uv_backward(o, k * G, k * Gd, k * Ga)
        np.testing.assert_allclose(s.absgrad, abs(k) * r.absgrad, rtol=1e-12, atol=1e-300, err_msg=str(k))


def test_absgrad_is_zero_where_a_splat_contributes_nowhere(fp64_case):
    """Visible gaussians no tile lists (the frustum cull keeps a 100-pixel margin around the 24x20 window) have
    exactly zero absgrad, and every gaussian with a non-zero signed sum has a non-zero absgrad."""
    _, o, _, _, _, r = fp64_case
    listed = np.zeros(o.uv.shape[0], bool)
    listed[np.asarray(o.sorted_idx)] = True
    assert (~listed).sum() > 0 and listed.sum() > 0
    assert not r.absgrad[~listed].any()
    assert np.all(r.absgrad[r.uv != 0] > 0)


def test_a_splat_on_a_single_pixel_has_absgrad_equal_to_its_signed_sum():
    """On a 1x1 image every splat contributes to exactly one pixel: nothing can cancel, absgrad == |uv.grad|."""
    sc = tiny(0, n=400, H=1, W=1)
    o = forward(sc)
    assert len(o.sorted_idx) >= 3
    G, Gd, Ga = upstream(1, 1, depth=True)
    r = abo.uv_backward(o, G, Gd, Ga)
    assert np.count_nonzero(r.uv) >= 6
    assert np.array_equal(r.absgrad, np.abs(r.uv))


# ---- the kernels in the built library --------------------------------------------------------------------------------
def _usage():
    text = _tool_output("--dump-resource-usage")
    return {name: {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
            for name, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", text)}


# DESIGN.md 3.12: (masks, depth) -> (registers at most, CTAs per SM)
ABS_KERNELS = {(True, False): (64, 8), (False, False): (80, 6), (True, True): (96, 5), (False, True): (96, 5)}


@pytest.mark.parametrize("masks,depth", list(ABS_KERNELS), ids=[f"masks{int(m)}-depth{int(d)}" for m, d in ABS_KERNELS])
def test_absgrad_kernels_keep_the_occupancy_design_md_states(masks, depth):
    usage = _usage()
    frag = f"k_render_bwd_absILb{int(masks)}ELb{int(depth)}E"
    hits = [v for k, v in usage.items() if frag in k]
    assert hits, f"{frag} not in the library"
    u = hits[0]
    regs, ctas = ABS_KERNELS[(masks, depth)]
    assert u["REG"] <= regs and u["STACK"] == 0 and u["LOCAL"] == 0, u
    assert ctas * u["REG"] * 128 <= 65536 and ctas * (u["SHARED"] + 1024) <= 227 * 1024, u


def test_absgrad_backward_flushes_the_row_tail_with_one_vector_reduction():
    """Three 16-byte vector reductions per (gaussian, tile) pair — the third covers conic2 z|0 |u| |v| — and no scalar
    global atomic in the flush."""
    text = _tool_output("-sass")
    for depth in (0, 1):
        body = text.split(f"Function : _ZN3gsr16k_render_bwd_absILb1ELb{depth}E", 1)[1].split("Function :", 1)[0]
        assert len(re.findall(r"REDG\.E\.ADD\.F32x4", body)) >= 3, depth
        assert not re.search(r"(?:REDG|ATOMG)\.E\.ADD\.F32(?:\.FTZ)?(?:\.RN)?\.STRONG", body), depth


# ---- argument errors ------------------------------------------------------------------------------------------------
def test_argument_errors_without_a_gpu():
    torch = pytest.importorskip("torch")
    from gaussian_splatting_b200.rasterize import rasterize
    from gaussian_splatting_b200.structs import Camera, Gaussians

    sc = np_scene(50, "tiny", 1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    g = Gaussians(t(sc["xyz"]), t(sc["rgb"]), t(sc["opacity"]), t(sc["scale"]), t(sc["quaternion"]), t(sc["sh"]))
    cam = Camera(64, 64, t(sc["K"]))
    bg = torch.full((3,), 0.5)
    with pytest.raises(ValueError, match="absgrad"):
        rasterize(g, t(sc["T"]), cam, 0.3, 500.0, 100, 3.0, False, bg, absgrad=True)
    g64 = Gaussians(*(x.double() for x in (g.xyz, g.rgb, g.opacity, g.scale, g.quaternion)), None)
    with pytest.raises(TypeError, match="absgrad"):
        rasterize(g64, t(sc["T"]).double(), Camera(64, 64, t(sc["K"]).double()), 0.3, 500.0, 100, 3.0, True,
                  bg.double(), absgrad=True)


def test_densification_statistics_refuse_a_view_without_absgrad():
    torch = pytest.importorskip("torch")
    from types import SimpleNamespace

    from gaussian_splatting_b200.densify import DensificationStats

    stats = DensificationStats(4, "cpu")
    st = SimpleNamespace(uv_absgrad=None, vis_idx32=torch.zeros(0, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="absgrad=True"):
        stats.accumulate(st, torch.zeros(0, 2), torch.zeros(4, 3), torch.eye(3), absgrad=True)
