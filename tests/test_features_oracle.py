"""Feature maps (rasterize(..., features=F)): the CPU oracle's semantics and gradients, the argument checks of
rasterize and of the C entry points, and the kernels of libgsr_features.so.  No GPU needed."""
import ctypes as C
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import depth_alpha_oracle as dao
from tests import features_oracle as fo
from tests.scenes import np_scene

ROOT = Path(__file__).resolve().parents[1]
FEATURES_LIB = ROOT / "gaussian_splatting_b200" / "libgsr_features.so"
MAIN_LIB = ROOT / "gaussian_splatting_b200" / "libgsr_b200.so"
BAD_ARG = -1


def _oracle(sc):
    return dao.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"],
                         sc["K"], sc["H"], sc["W"], background=np.full(3, 0.5, sc["xyz"].dtype))


@pytest.mark.parametrize("D,sh_degree", [(1, 0), (3, 1), (5, 2)])
def test_fp64_feature_backward_matches_finite_differences(D, sh_degree):
    """<G, feature_map> against central differences of the oracle's fp64 feature forward, for F, opacity, uv and conic
    of the compact gaussians (the pair list held fixed, as the kernels differentiate it)."""
    sc = np_scene(128, "tiny", sh_degree=sh_degree, dtype=np.float64, sigma_px=(3.0, 0.4, 1.0, 6.0))
    o = _oracle(sc)
    assert o.keep.sum() > 64 and len(o.sorted_idx) > 200 and (o.alpha > 0.5).any()
    rng = np.random.default_rng(D)
    M = int(o.keep.sum())
    F = rng.standard_normal((M, D))
    G = rng.standard_normal((64, 64, D)) / (64 * 64)
    chunk = 960
    g, _ = fo.backward(o.uv, o.opacity, o.conic, F, o.ranges, o.sorted_idx, o.n, o.wlast, G, chunk)
    inputs = dict(uv=o.uv, opacity=np.asarray(o.opacity).reshape(-1), conic=o.conic, F=F)

    def loss(**over):
        a = dict(inputs, **over)
        return float((fo.forward(a["uv"], a["opacity"], a["conic"], a["F"], o.ranges, o.sorted_idx, 64, 64) * G).sum())

    h = 1e-6
    for name in ("F", "opacity", "uv", "conic"):
        grad, base = getattr(g, name), inputs[name]
        scale = np.abs(grad).max()
        assert scale > 0, name
        for _ in range(8):
            idx = tuple(int(rng.integers(0, s)) for s in base.shape)
            plus, minus = base.copy(), base.copy()
            plus[idx] += h
            minus[idx] -= h
            fd = (loss(**{name: plus}) - loss(**{name: minus})) / (2 * h)
            assert abs(fd - grad[idx]) <= 2e-5 * scale + 1e-12, (name, idx, fd, grad[idx])


def test_feature_map_of_the_colours_is_the_image_on_black():
    """F = SH0 * rgb (the records' colours): the fp32 feature walk reproduces the oracle's image on a black background
    bit for bit, and the gradient on F is the colour gradient over SH0."""
    sc = np_scene(2000, "tiny", sh_degree=0, sigma_px=(2.0, 0.5, 0.5, 8.0))
    o = dao.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], None, sc["T"], sc["K"],
                      sc["H"], sc["W"], background=np.zeros(3, np.float32))
    F = (o.rgb * np.float32(0.28209479177387814)).astype(np.float32)
    fmap = fo.render_forward(o, F)
    assert np.array_equal(fmap.view(np.uint32), o.image.view(np.uint32))
    G = np.random.default_rng(0).standard_normal((64, 64, 3)).astype(np.float32)
    d = fo.rasterize_backward(o, _full(o, F), G)
    dc = dao.rasterize_backward(o, G, np.zeros((64, 64), np.float32), np.zeros((64, 64), np.float32))
    for k in ("F", "opacity", "uv", "conic"):
        mine, ref = getattr(d.render, k), getattr(dc.render, "rgb" if k == "F" else k)
        if k == "F":  # the colour row is SH0 * sum(alpha * weight * G), each product rounded in fp32 after the SH0
            mine = mine * 0.28209479177387814
        np.testing.assert_allclose(mine, ref, rtol=1e-5, atol=1e-6 * np.abs(ref).max())


def _full(o, F_compact):
    out = np.zeros((o.keep.shape[0], F_compact.shape[1]), F_compact.dtype)
    out[o.keep] = F_compact
    return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_one_gaussian_known_answer(dtype):
    """A single splat: every pixel's blend weight is its alpha, so feature_map = alpha * F (one fma on 0: the rounded
    product in fp32), and the gradient on F is sum_p alpha_p * G_p."""
    sc = np_scene(1, "tiny", sh_degree=0, dtype=dtype)
    sc["xyz"] = np.array([[0.05, -0.03, 3.0]], dtype)
    sc["T"] = np.eye(4, dtype=dtype)
    sc["scale"] = np.log(np.full((1, 3), 0.15, dtype))
    sc["quaternion"] = np.array([[1, 0, 0, 0]], dtype)
    sc["opacity"] = np.array([[0.8]], dtype)
    o = _oracle(sc)
    assert o.keep.all()
    F = np.array([[0.7, -1.3, 2.5, 0.125, -4.0]], dtype)
    fmap = fo.render_forward(o, F)
    lit = o.alpha > 0
    assert lit.sum() > 50
    assert np.array_equal(fmap, (o.alpha[..., None] * F[0]).astype(dtype))
    assert not fmap[~lit].any()
    G = np.random.default_rng(3).standard_normal((64, 64, 5)).astype(dtype)
    d = fo.rasterize_backward(o, F, G)
    ref = (o.alpha.astype(np.float64)[..., None] * G).sum((0, 1))
    np.testing.assert_allclose(d.F[0], ref, rtol=1e-5 if dtype == np.float32 else 1e-12)


def test_masses_bound_the_feature_rows():
    sc = np_scene(2000, "tiny", sh_degree=0, seed=1, view=2, n_views=3, sigma_px=(2.0, 0.5, 0.5, 8.0))
    o = _oracle(sc)
    rng = np.random.default_rng(4)
    F = rng.standard_normal((sc["xyz"].shape[0], 6)).astype(np.float32)
    G = (rng.standard_normal((64, 64, 6)) / (64 * 64)).astype(np.float32)
    d = fo.rasterize_backward(o, F, G)
    for k in ("F", "opacity"):  # sums of the summands' absolute values (uv / conic: bounds of their factors)
        val, mass = getattr(d.render, k), getattr(d.mass, k)
        assert (mass >= np.abs(val) * (1 - 1e-12)).all(), k
    for k in ("F", "opacity", "uv", "conic"):
        assert np.abs(getattr(d.render, k)).max() > 0 and getattr(d.mass, k).max() > 0, k
    assert not d.F[~o.keep].any()


# ---- argument errors -------------------------------------------------------------------------------------------------
def _gaussians(n=4, dtype=torch.float32, sh=None):
    from gaussian_splatting_b200.structs import Gaussians

    return Gaussians(torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 1, dtype=dtype),
                     torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 4, dtype=dtype), sh)


def _call(g, features, **kw):
    from gaussian_splatting_b200.rasterize import rasterize
    from gaussian_splatting_b200.structs import Camera

    dt = g.xyz.dtype
    return rasterize(g, torch.eye(4, dtype=dt), Camera(64, 64, torch.eye(3, dtype=dt)), 0.3, 500.0, 100, 3.0,
                     kw.pop("use_sh_precompute", True), torch.zeros(3, dtype=dt), features=features, **kw)


def test_rasterize_argument_errors():
    g = _gaussians()
    with pytest.raises(ValueError):
        _call(g, torch.zeros(5, 3))                      # wrong row count
    with pytest.raises(ValueError):
        _call(g, torch.zeros(4))                         # not [N, D]
    with pytest.raises(ValueError):
        _call(g, torch.zeros(4, 0))                      # D < 1
    with pytest.raises(TypeError):
        _call(g, torch.zeros(4, 3, dtype=torch.float64))  # wrong dtype
    with pytest.raises(ValueError):
        _call(g, torch.zeros(4, 3, device="meta"))       # wrong device
    with pytest.raises(ValueError):
        _call(g, torch.zeros(3, 4).t())                  # not contiguous
    with pytest.raises(ValueError):
        _call(g, torch.zeros(4, 3), absgrad=True)        # out of scope
    with pytest.raises(TypeError):
        _call(_gaussians(dtype=torch.float64), torch.zeros(4, 3, dtype=torch.float64))
    with pytest.raises(ValueError):
        _call(_gaussians(sh=torch.zeros(4, 3, 3)), torch.zeros(4, 3), use_sh_precompute=False)
    with pytest.raises(TypeError):
        _call(g, np.zeros((4, 3), np.float32))


def _features_lib():
    if not FEATURES_LIB.exists():
        pytest.skip("libgsr_features.so is not built")
    return C.CDLL(str(FEATURES_LIB))


def test_c_entry_points_reject_bad_arguments_before_any_launch():
    """Pointers are never dereferenced on the host: every call below fails its checks before a launch, so fake
    (16-byte aligned) device addresses are enough."""
    lib = _features_lib()
    P = C.c_void_p
    dev = P(0x10000)
    mis = P(0x10004)
    fwd, bwd = lib.gsr_render_features_forward, lib.gsr_render_features_backward
    fwd.restype = bwd.restype = C.c_int

    def f(rec=dev, keys=dev, ids=None, ranges=dev, H=16, W=16, feat=dev, stride=4, D=3, out=dev):
        return fwd(rec, keys, C.c_int(20), ids, ranges, C.c_int(H), C.c_int(W), feat, C.c_int(stride), C.c_int(D),
                   out, None)

    def b(rec=dev, keys=dev, ids=None, ranges=dev, H=16, W=16, n=dev, w=dev, feat=dev, stride=4, D=3, gmap=dev,
          gfeat=dev, rows=dev, masks=None):
        return bwd(rec, keys, C.c_int(20), ids, ranges, C.c_int(H), C.c_int(W), n, w, feat, C.c_int(stride),
                   C.c_int(D), gmap, gfeat, rows, masks, None)

    for kw in (dict(keys=None), dict(ids=dev), dict(rec=None), dict(ranges=None), dict(H=0), dict(W=-1), dict(D=0),
               dict(stride=5), dict(stride=8), dict(D=5, stride=4), dict(feat=None), dict(feat=mis)):
        assert f(**kw) == BAD_ARG, kw
        assert b(**kw) == BAD_ARG, kw
    assert f(out=None) == BAD_ARG
    for kw in (dict(n=None), dict(w=None), dict(gmap=None), dict(gfeat=None), dict(rows=None), dict(gfeat=mis),
               dict(rows=mis)):
        assert b(**kw) == BAD_ARG, kw


# ---- the library -----------------------------------------------------------------------------------------------------
def _cuobjdump(*args, lib=FEATURES_LIB):
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(exe).exists() or not lib.exists():
        pytest.skip("cuobjdump or the built library is missing")
    return subprocess.run([exe, *args, str(lib)], check=True, capture_output=True, text=True).stdout


def _bodies():
    text = _cuobjdump("-sass")
    return {name.strip(): body for name, body in (f.split("\n", 1) for f in re.split(r"\n\s+Function : ", text)[1:])}


def test_feature_kernels_are_sm90a_and_keep_nothing_in_local_memory():
    elfs = _cuobjdump("--list-elf")
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    bodies = _bodies()
    names = sorted(bodies)
    assert len(names) == 3 and all("k_features_" in n for n in names), names
    assert not any("stats" in n for n in names)
    for name, body in bodies.items():
        assert not re.search(r"\b(?:STL|LDL)\b", body), name
        assert len(re.findall(r"\bLDGSTS\b", body)) >= 4, name   # records + features by cp.async
        assert re.search(r"\bSYNCS\b", body), name                # on the stage mbarrier
    usage = re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage"))
    assert len(usage) == 3
    for name, line in usage:
        u = {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
        assert u["STACK"] == 0 and u["LOCAL"] == 0, (name, u)


def test_feature_backward_flushes_with_vector_reductions():
    for name, body in _bodies().items():
        if "k_features_bwd" in name:
            assert len(re.findall(r"REDG\.E\.ADD\.F32x4", body)) >= 2, name   # grad_F and the uv / conic slots


def test_main_library_does_not_carry_the_feature_kernels():
    assert "k_features" not in _cuobjdump("-sass", lib=MAIN_LIB)
