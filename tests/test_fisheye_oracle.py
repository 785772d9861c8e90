"""Fisheye cameras (rasterize(..., fisheye=k)) without a GPU: the fp64 oracle's VJP against finite differences, its
small-rho branch against an mpmath evaluation, the cull limit theta_max, the argument errors, the new library's surface
and the SASS of every kernel that existed before it."""
import ctypes as C
import json
import re
import shutil
import subprocess
from pathlib import Path

import mpmath as mp
import numpy as np
import pytest
import torch

from tests import fisheye_oracle as feo
from tests.scenes import np_scene

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "gaussian_splatting_b200"
FISHEYE_LIB = PKG / "libgsr_fisheye.so"
K_NONZERO = (0.08, -0.03, 0.01, -0.002)
KS = {"k0": (0.0, 0.0, 0.0, 0.0), "k4": K_NONZERO}


# ---- fp64 finite differences -------------------------------------------------------------------------------------------
def _upstream(H, W, seed=1):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((H, W, 3)) / (3 * H * W), rng.standard_normal((H, W)) / (H * W),
            rng.standard_normal((H, W)) / (H * W))


@pytest.mark.parametrize("k", list(KS), ids=list(KS))
@pytest.mark.parametrize("mode", ["plain", "depth", "antialiased", "filter3d"])
def test_fp64_fisheye_backward_matches_finite_differences(k, mode):
    """<G,image> + <Gd,depth> + <Ga,alpha> against central differences of the fp64 fisheye forward, every parameter
    (SH 0, so that xyz's gradient is complete).  The scene is the tiny synthetic one seen through the fisheye."""
    sc = np_scene(128, "tiny", sh_degree=0, dtype=np.float64, sigma_px=(0.6, 1.2, 0.15, 8.0))
    f3d = None
    if mode == "filter3d":
        f3d = np.exp(sc["scale"].mean(1)) * np.random.default_rng(3).uniform(0.3, 1.5, len(sc["scale"]))
    aa = mode in ("antialiased", "filter3d")
    G, Gd, Ga = _upstream(sc["H"], sc["W"])
    if mode == "plain":
        Gd, Ga = np.zeros_like(Gd), np.zeros_like(Ga)

    def forward(**over):
        s = dict(sc, **over)
        return feo.rasterize(s["xyz"], s["quaternion"], s["scale"], s["opacity"], s["rgb"], s["sh"], s["T"], s["K"],
                             s["H"], s["W"], KS[k], antialiased=aa, filter3d=f3d, background=np.full(3, 0.5))

    o = forward()
    assert o.keep.sum() > 64 and len(o.sorted_idx) > 100
    d = feo.rasterize_backward(o, G, Gd, Ga)

    def loss(**over):
        p = forward(**over)
        return float((p.image * G).sum() + (p.depth * Gd).sum() + (p.alpha * Ga).sum())

    rng = np.random.default_rng(2)
    vis = np.flatnonzero(o.keep)
    h = 1e-6
    for name in ("xyz", "quaternion", "scale", "opacity", "rgb"):
        grad, base = getattr(d, name), sc[name]
        scale = np.abs(grad).max()
        assert np.isfinite(grad).all() and scale > 0, name
        for _ in range(5):
            i = int(rng.choice(vis))
            idx = (i,) + tuple(int(rng.integers(0, s)) for s in base.shape[1:])
            plus, minus = base.copy(), base.copy()
            plus[idx] += h
            minus[idx] -= h
            fd = (loss(**{name: plus}) - loss(**{name: minus})) / (2 * h)
            assert abs(fd - grad[idx]) <= 2e-5 * scale + 1e-12, (name, idx, fd, grad[idx])


# ---- the small-rho branch against mpmath ---------------------------------------------------------------------------------
mp.mp.dps = 40


def _mp_s(x, y, z, k):
    rho = mp.sqrt(x * x + y * y)
    if rho == 0:
        return 1 / z
    th = mp.atan2(rho, z)
    t = th * th
    return th * (1 + t * (k[0] + t * (k[1] + t * (k[2] + t * k[3])))) / rho


def _mp_uv(p, k, fx, fy):
    return [lambda x, y, z: fx * _mp_s(x, y, z, k) * x, lambda x, y, z: fy * _mp_s(x, y, z, k) * y]


def _mp_jacobian(p, k, fx, fy):
    fs = _mp_uv(p, k, fx, fy)
    P = [mp.mpf(v) for v in p]
    return [[mp.diff(f, P, tuple(int(j == c) for j in range(3))) for c in range(3)] for f in fs]


@pytest.mark.parametrize("ratio", [0.0, 1e-8, 1e-5, 1e-3, 1e-1])
@pytest.mark.parametrize("k", list(KS), ids=list(KS))
def test_small_rho_branch_matches_mpmath(ratio, k):
    """s, J and the VJP (J^T g_uv + d<gJ, J>/dp) at rho / z = ratio against a 40-digit evaluation of the model's
    expression and of its derivatives; at rho = 0 J is the pinhole Jacobian [[fx/z, 0, 0], [0, fy/z, 0]]."""
    kk = [mp.mpf(v) for v in KS[k]]
    z = 2.5
    p = np.array([0.6 * ratio * z, -0.8 * ratio * z, z])
    fx, fy = 400.0, 380.0
    s = feo.terms(p, KS[k])[0]
    s_ref = _mp_s(*[mp.mpf(v) for v in p], kk)
    assert abs(s - float(s_ref)) <= 1e-13 * abs(float(s_ref))
    gJ = np.array([0.3, -0.7, 0.2, 0.5, 0.4, -0.6])
    guv = np.array([0.9, -0.2])
    J, g = feo.jacobian_vjp(p, fx, fy, KS[k], gJ, guv)
    Jr = np.array([[float(v) for v in row] for row in _mp_jacobian(p, kk, fx, fy)])
    assert np.abs(J - Jr).max() <= 1e-10 * np.abs(Jr).max(), (J, Jr)
    if ratio == 0.0:
        assert np.array_equal(J, np.array([[fx / z, 0, 0], [0, fy / z, 0]]))
    # d/dp of <gJ, J(p)> + <guv, uv(p)>
    fs = _mp_uv(p, kk, fx, fy)
    P = [mp.mpf(v) for v in p]
    gr = []
    for c in range(3):
        e = tuple(int(j == c) for j in range(3))
        acc = sum(mp.mpf(guv[i]) * mp.diff(fs[i], P, e) for i in range(2))
        for i in range(2):
            for j in range(3):
                e2 = tuple(int(a == c) + int(a == j) for a in range(3))
                acc += mp.mpf(gJ[i * 3 + j]) * mp.diff(fs[i], P, e2)
        gr.append(float(acc))
    gr = np.array(gr)
    assert np.isfinite(g).all() and np.abs(g - gr).max() <= 1e-8 * np.abs(gr).max(), (g, gr)


# ---- theta_max -------------------------------------------------------------------------------------------------------------
THETA_TABLE = [
    (0.0, 0.0, 0.0, 0.0),          # equidistant: monotone, pi/2
    (0.08, -0.03, 0.01, -0.002),   # mild lens: monotone
    (-0.05, 0.01, 0.0, 0.0),       # monotone
    (-0.3, 0.0, 0.0, 0.0),         # folds at theta^2 = 1/0.9
    (-0.1, -0.05, 0.0, 0.0),       # folds
    (0.2, -0.4, 0.05, 0.0),        # folds
    (0.0, 0.0, 0.0, -0.5),         # folds through k4 alone
    (0.5, 0.3, -0.2, 0.01),        # folds
]


def _fe_lib():
    if not FISHEYE_LIB.exists():
        pytest.skip("libgsr_fisheye.so is not built")
    lib = C.CDLL(str(FISHEYE_LIB))
    lib.gsr_fisheye_theta_max.restype = C.c_float
    return lib


@pytest.mark.parametrize("k", THETA_TABLE)
def test_theta_max_is_the_smallest_positive_root_rounded_down(k):
    from gaussian_splatting_b200.rasterize import fisheye_theta_max

    k32 = np.asarray(k, np.float32)
    ref = feo.theta_max(k32.astype(np.float64))
    want = np.float32(ref)
    if float(want) > ref:
        want = np.nextafter(want, np.float32(0))
    c = _fe_lib().gsr_fisheye_theta_max(k32.ctypes.data_as(C.POINTER(C.c_float)))
    py = fisheye_theta_max(k)
    assert abs(np.float32(c) - want) <= np.spacing(want), (k, c, want)
    assert py == float(np.float32(c))
    assert float(np.float32(c)) <= ref
    if all(v == 0 for v in k[1:]) and k[0] >= 0:
        assert ref == np.pi / 2


def test_theta_max_of_non_finite_or_missing_coefficients_is_nan():
    lib = _fe_lib()
    bad = np.array([np.nan, 0, 0, 0], np.float32)
    assert np.isnan(lib.gsr_fisheye_theta_max(bad.ctypes.data_as(C.POINTER(C.c_float))))
    assert np.isnan(lib.gsr_fisheye_theta_max(None))


# ---- argument errors -----------------------------------------------------------------------------------------------------
def _gaussians(n=4, dtype=torch.float32, sh=None):
    from gaussian_splatting_b200.structs import Gaussians

    return Gaussians(torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 1, dtype=dtype),
                     torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 4, dtype=dtype), sh)


def test_rasterize_fisheye_argument_errors():
    from gaussian_splatting_b200.rasterize import rasterize
    from gaussian_splatting_b200.structs import Camera

    def call(g=None, use_sh_precompute=True, **kw):
        g = _gaussians() if g is None else g
        dt = g.xyz.dtype
        return rasterize(g, torch.eye(4, dtype=dt), Camera(64, 64, torch.eye(3, dtype=dt)), 0.3, 500.0, 100, 3.0,
                         use_sh_precompute, torch.zeros(3, dtype=dt), **kw)

    k = (0.1, 0.0, 0.0, 0.0)
    with pytest.raises(TypeError):
        call(_gaussians(dtype=torch.float64), fisheye=k)
    with pytest.raises(ValueError):
        call(_gaussians(sh=torch.zeros(4, 3, 3)), use_sh_precompute=False, fisheye=k)
    for bad in ((0.1, 0.0, 0.0), (0.1, 0.0, 0.0, 0.0, 0.0), [[0.1, 0, 0, 0]], (float("nan"), 0, 0, 0),
                (0, float("inf"), 0, 0), (1e39, 0, 0, 0), torch.zeros(3), torch.zeros(2, 4), "abcd", (0, 0, "x", 0)):
        with pytest.raises(ValueError):
            call(fisheye=bad)
    if torch.cuda.is_available():
        with pytest.raises(ValueError):
            call(fisheye=torch.zeros(4, device="cuda"))
    with pytest.raises(ValueError):
        call(fisheye=torch.zeros(4, device="meta"))


def test_rasterize_batch_fisheye_argument_errors():
    from gaussian_splatting_b200 import rasterize_batch
    from gaussian_splatting_b200.structs import Camera

    def call(g=None, use_sh_precompute=True, **kw):
        g = _gaussians() if g is None else g
        dt = g.xyz.dtype
        return rasterize_batch(g, torch.eye(4, dtype=dt).expand(2, 4, 4), Camera(64, 64, torch.eye(3, dtype=dt)), 0.3,
                               500.0, 100, 3.0, use_sh_precompute, torch.zeros(3, dtype=dt), **kw)

    with pytest.raises(TypeError):
        call(_gaussians(dtype=torch.float64), fisheye=(0, 0, 0, 0))
    with pytest.raises(ValueError):
        call(_gaussians(sh=torch.zeros(4, 3, 3)), use_sh_precompute=False, fisheye=(0, 0, 0, 0))
    for bad in (torch.zeros(3, 4), torch.zeros(2, 3), torch.zeros(2, 2, 4), [(0, 0, 0, 0)] * 3,
                [(0, 0, 0, 0), (0, 0, float("nan"), 0)], torch.zeros(4, device="meta")):
        with pytest.raises(ValueError):
            call(fisheye=bad)


# ---- the library -----------------------------------------------------------------------------------------------------------
def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists():
        pytest.skip(f"{name} is missing")
    return exe


def _cuobjdump(*args, lib=FISHEYE_LIB):
    if not lib.exists():
        pytest.skip("the built library is missing")
    return subprocess.run([_tool("cuobjdump"), *args, str(lib)], check=True, capture_output=True, text=True).stdout


def test_fisheye_header_declares_exactly_the_new_symbols_and_the_library_exports_them():
    header = (ROOT / "include" / "gsr_fisheye.h").read_text()
    declared = set(re.findall(r"^\w[\w\s\*]*?\b(gsr_\w+)\s*\(", header, re.M))
    assert declared == {"gsr_fisheye_theta_max", "gsr_fisheye_preprocess_forward", "gsr_fisheye_preprocess_backward",
                        "gsr_fisheye_batch_preprocess_backward"}, declared
    lib = _fe_lib()
    for name in declared:
        assert hasattr(lib, name), name


def test_fisheye_kernels_are_sm90a_and_keep_their_registers_out_of_local_memory():
    """Every mode combination is there: 16 forward, 32 backward and 32 batched backward kernels.  The backward
    kernels use no local memory; the forward kernels use exactly the stack their pinhole counterparts use (the
    division slow path's saves)."""
    elfs = _cuobjdump("--list-elf")
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage")))
    kinds = {"k_fisheye_preprocess_fwd": 16, "k_fisheye_preprocess_bwd": 32, "k_fisheye_batch_preprocess_bwd": 32}
    for kind, n in kinds.items():
        names = [k for k in usage if re.search(rf"\d{kind}I", k)]
        assert len(names) == n, (kind, len(names))
        for name in names:
            u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[name])}
            assert u["LOCAL"] == 0, (name, u)
            assert u["STACK"] <= (32 if kind.endswith("fwd") else 0), (name, u)


def test_existing_kernels_keep_their_sass():
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_fisheye.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    for lib in ("libgsr_b200.so", "libgsr_batch.so"):
        if not (PKG / lib).exists():
            pytest.skip(f"{lib} is not built")
        now = {k: d for k, (d, n) in sass_digest.per_kernel(PKG / lib).items()}
        assert set(now) == set(rec[lib]), lib
        changed = sorted(k for k, d in rec[lib].items() if now[k] != d)
        assert not changed, (lib, changed)
        assert "fisheye" not in "".join(now)
