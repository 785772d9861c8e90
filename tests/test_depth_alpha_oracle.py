"""Depth and alpha maps (rasterize(render_depth_alpha=True)): the CPU oracle's semantics and gradients, and the
depth kernels in the built library.  No GPU needed."""
import re

import numpy as np
import pytest

from tests import depth_alpha_oracle as dao
from tests.scenes import np_scene
from tests.test_sass_evidence import _tool_output, sass_counts


def _forward(sc, **over):
    s = dict(sc, **over)
    return dao.rasterize(s["xyz"], s["quaternion"], s["scale"], s["opacity"], s["rgb"], s["sh"], s["T"], s["K"],
                         s["H"], s["W"], background=np.full(3, 0.5, s["xyz"].dtype))


def _upstream(H, W, seed=1):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((H, W, 3)) / (3 * H * W), rng.standard_normal((H, W)) / (H * W),
            rng.standard_normal((H, W)) / (H * W))


@pytest.mark.parametrize("sh_degree", [0, 3])
def test_fp64_depth_alpha_backward_matches_finite_differences(sh_degree):
    """<G,image> + <Gd,depth> + <Ga,alpha> against central differences of the oracle's fp64 forward, every parameter.
    With SH the reference sends no gradient to xyz through the view direction, so xyz is checked on the depth and
    alpha terms alone there (the image's SH colours then do not enter the loss)."""
    sc = np_scene(128, "tiny", sh_degree=sh_degree, dtype=np.float64, sigma_px=(3.0, 0.4, 1.0, 6.0))
    G, Gd, Ga = _upstream(64, 64)
    rng = np.random.default_rng(2)

    def check(names, G):
        o = _forward(sc)
        assert o.keep.sum() > 64 and len(o.sorted_idx) > 200 and (o.alpha > 0.5).any()
        d = dao.rasterize_backward(o, G, Gd, Ga)

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
        check(["quaternion", "scale", "opacity", "rgb", "sh"], G)
        check(["xyz", "quaternion", "scale", "opacity"], np.zeros_like(G))
    else:
        check(["xyz", "quaternion", "scale", "opacity", "rgb"], G)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_one_gaussian_known_answer(dtype):
    """A single splat: every pixel's blend weight is its alpha, so alpha = opacity * exp(-mh/2) and depth = z * alpha
    (one fma on 0: the rounded product in fp32)."""
    sc = np_scene(1, "tiny", sh_degree=0, dtype=dtype)
    sc["xyz"] = np.array([[0.05, -0.03, 3.0]], dtype)
    sc["T"] = np.eye(4, dtype=dtype)
    sc["scale"] = np.log(np.full((1, 3), 0.15, dtype))
    sc["quaternion"] = np.array([[1, 0, 0, 0]], dtype)
    sc["opacity"] = np.array([[0.8]], dtype)
    o = _forward(sc)
    assert o.keep.all()
    u, v = o.uv[0].astype(np.float64)
    a, b2, c = o.conic[0].astype(np.float64)
    if dtype == np.float32:
        a, c = a + 0.25, c + 0.25
    py, px = np.mgrid[0:64, 0:64].astype(np.float64)
    du, dv = px - u, py - v
    mh = (c * du * du - b2 * du * dv + a * dv * dv) / (a * c - 0.25 * b2 * b2)
    ref = o.opacity[0] * np.exp(-0.5 * mh)
    lit = o.alpha > 0   # pixels of the tiles the splat was binned to (fp32: above the 1/255 skip)
    assert lit.sum() > 50 and (o.n[lit] == 1).all()
    if dtype == np.float32:
        assert (ref[~lit] < 1.0001 / 255.0).all()
    np.testing.assert_allclose(o.alpha[lit], ref[lit], rtol=1e-5 if dtype == np.float32 else 1e-12)
    z = o.z[0]
    assert np.array_equal(o.depth, (o.alpha * z).astype(dtype))   # fma(w, z, 0) rounds w*z once
    assert np.array_equal(o.alpha[~lit], np.zeros((~lit).sum(), dtype)) and not o.depth[~lit].any()


def test_mass_bounds_every_render_stage_sum():
    """The masses the per-row check scales its bound by cover the new terms: the z row's mass bounds |z| (and the
    opacity row's its |sum|, now with the depth and alpha parts of d_alpha), and the opacity mass grows by those
    parts.  The z row carries exactly the depth term."""
    sc = np_scene(2000, "tiny", sh_degree=0, seed=1, view=2, n_views=3, sigma_px=(2.0, 0.5, 0.5, 8.0))
    o = _forward(sc)
    G, Gd, Ga = (a.astype(np.float32) for a in _upstream(64, 64))
    d = dao.rasterize_backward(o, G, Gd, Ga)
    for k in ("rgb", "opacity", "z"):
        val, mass = getattr(d.render, k), getattr(d.mass, k)
        assert (mass >= np.abs(val) * (1 - 1e-12)).all(), k
    assert np.abs(d.render.z).max() > 0 and (d.mass.z > 0).sum() > 100
    d_img = dao.rasterize_backward(o, G, np.zeros_like(Gd), np.zeros_like(Ga))
    assert not d_img.render.z.any() and not d_img.mass.z.any()
    assert (d.mass.opacity >= d_img.mass.opacity).all() and (d.mass.opacity > d_img.mass.opacity).any()
    d_z = dao.rasterize_backward(o, np.zeros_like(G), Gd, np.zeros_like(Ga))
    assert np.array_equal(d_z.render.z, d.render.z)


def test_depth_alpha_kernels_exist_flush_with_vector_reductions_and_keep_no_stack():
    """The depth instantiations (gather mode, masks on and off) are in the library; the backward flushes its ten sums
    per pair with vector reductions (two 16-byte, one 8-byte); the masked kernels the fused path uses keep nothing in
    local memory."""
    counts = sass_counts()
    for k in ("k_render_fwd_depth", "k_render_bwd_depth"):
        for masks in (0, 1):
            c = next((c for name, c in counts.items() if f"{len(k)}{k}ILb{masks}E" in name), None)
            assert c is not None, (k, masks)
            assert c["LDGSTS"] >= 3 and c["SYNCS"] >= 1, (k, dict(c))
    assert any("22k_preprocess_bwd_depthILi16ELb1E" in n for n in counts)
    text = _tool_output("-sass")
    for masks in (0, 1):
        body = text.split(f"Function : _ZN3gsr18k_render_bwd_depthILb{masks}E", 1)[1].split("Function :", 1)[0]
        assert len(re.findall(r"REDG\.E\.ADD\.F32x4", body)) >= 2, masks
        assert len(re.findall(r"REDG\.E\.ADD\.F32x2", body)) >= 1, masks
    usage = {}
    for name, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _tool_output("--dump-resource-usage")):
        usage[name] = {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
    for frag in ("k_render_fwd_depthILb1E", "k_render_bwd_depthILb1E", "k_render_bwd_depthILb0E"):
        u = next(v for k, v in usage.items() if frag in k)
        assert u["STACK"] == 0 and u["LOCAL"] == 0, (frag, u)
