"""BASELINE.json configs[0]: 128 Gaussians, 64x64 image, fp64, no GPU.

The oracle's analytic backward (restating src/render_backward.cu + src/projection_backward.cu) is
checked against central finite differences of the oracle's own fp64 forward — the CPU counterpart of
the reference's fp64 `gradcheck` tests (test/test_rasterize_autograd.py, test_cuda_autograd_functions.py).
"""
import numpy as np
import pytest

from oracle import cpu_oracle as orc
from tests.scenes import np_scene


def _loss(sc, G, **over):
    s = dict(sc, **over)
    o = orc.rasterize(s["xyz"], s["quaternion"], s["scale"], s["opacity"], s["rgb"], s["sh"], s["T"], s["K"], s["H"],
                      s["W"], background=np.full(3, 0.5))
    return float((o.image * G).sum()), o


@pytest.mark.parametrize("sh_degree", [0, 1, 2, 3])
def test_fp64_backward_matches_finite_differences(sh_degree):
    sc = np_scene(128, "tiny", sh_degree=sh_degree, dtype=np.float64, sigma_px=(3.0, 0.4, 1.0, 6.0))
    rng = np.random.default_rng(1)
    G = rng.standard_normal((64, 64, 3)) / (3 * 64 * 64)
    _, o = _loss(sc, G)
    assert o.keep.sum() > 64 and len(o.sorted_idx) > 200
    d = orc.rasterize_backward(o, G)
    # with SH the reference sends NO gradient to xyz through the view direction
    # (splat_py/cuda_autograd_functions.py:127 returns None) — its xyz gradient is then not the true
    # derivative, so finite differences can only pin it in the SH-free case
    names = (["quaternion", "scale", "opacity", "rgb", "sh"] if sh_degree else
             ["xyz", "quaternion", "scale", "opacity", "rgb"])
    vis = np.flatnonzero(o.keep)
    h = 1e-6
    for name in names:
        grad = getattr(d, name)
        base = sc[name]
        scale = np.abs(grad).max()
        assert scale > 0
        for _ in range(6):
            i = int(rng.choice(vis))
            idx = (i,) + tuple(int(rng.integers(0, s)) for s in base.shape[1:])
            plus, minus = base.copy(), base.copy()
            plus[idx] += h
            minus[idx] -= h
            fd = (_loss(sc, G, **{name: plus})[0] - _loss(sc, G, **{name: minus})[0]) / (2 * h)
            assert abs(fd - grad[idx]) <= 2e-5 * scale + 1e-12, (name, idx, fd, grad[idx])


def test_fp32_and_fp64_branches_agree_on_geometry():
    """uv / conic / tile lists do not depend on the branch (only the renderer's alpha rule does)."""
    s32 = np_scene(128, "tiny", sh_degree=0, dtype=np.float32)
    s64 = {k: (v.astype(np.float64) if isinstance(v, np.ndarray) else v) for k, v in s32.items()}
    a = orc.project(s32["xyz"], s32["quaternion"], s32["scale"], s32["opacity"], s32["rgb"], None, s32["T"], s32["K"],
                    64, 64, 0.3, 500.0, 100.0)
    b = orc.project(s64["xyz"], s64["quaternion"], s64["scale"], s64["opacity"], s64["rgb"], None, s64["T"], s64["K"],
                    64, 64, 0.3, 500.0, 100.0)
    assert (a.visible == b.visible).all()
    k = a.visible.astype(bool)
    np.testing.assert_allclose(a.uv[k], b.uv[k], rtol=2e-5, atol=1e-3)
    np.testing.assert_allclose(a.conic[k], b.conic[k], rtol=2e-4, atol=1e-4)
