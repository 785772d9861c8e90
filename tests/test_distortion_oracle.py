"""Radial-tangential lens distortion (rasterize(..., distortion=k)) without a GPU: the fp64 oracle against a numpy
transcription of COLMAP's OpenCV camera model, its VJP against finite differences, the fold limit r2_max, the argument
errors, camera_from_colmap, the new library's surface and resources, and the SASS of every kernel that existed before
it."""
import ctypes as C
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import distortion_oracle as dto
from tests.scenes import np_scene

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "gaussian_splatting_b200"
DISTORTION_LIB = PKG / "libgsr_distortion.so"
KS = {"zero": (0.0, 0.0, 0.0, 0.0, 0.0), "radial": (-0.3, 0.08, 0.0, 0.0, -0.02),
      "full": (-0.12, 0.03, 5e-4, -3e-4, 0.01)}


# ---- the oracle's projection against COLMAP's OpenCV model -----------------------------------------------------------------
def colmap_full_opencv(a, b, k):
    """COLMAP's FullOpenCVCameraModel::Distortion with k4 = k5 = k6 = 0 (its OpenCVCameraModel when also k3 = 0),
    transcribed: the undistorted normalised point (a, b) plus the distortion offset (du, dv)."""
    k1, k2, p1, p2, k3 = k
    u2, uv, v2 = a * a, a * b, b * b
    r2 = u2 + v2
    r4, r6 = r2 * r2, r2 * r2 * r2
    radial = (1 + k1 * r2 + k2 * r4 + k3 * r6) / 1.0
    du = a * radial + 2 * p1 * uv + p2 * (r2 + 2 * u2) - a
    dv = b * radial + 2 * p2 * uv + p1 * (r2 + 2 * v2) - b
    return a + du, b + dv


def _uv_numpy(p, K, k):
    ad, bd = colmap_full_opencv(p[0] / p[2], p[1] / p[2], k)
    return np.array([K[0, 0] * ad + K[0, 2], K[1, 1] * bd + K[1, 2]])


def _points(n=200, seed=4):
    rng = np.random.default_rng(seed)
    z = rng.uniform(0.5, 8.0, n)
    return np.stack([rng.uniform(-0.9, 0.9, n) * z, rng.uniform(-0.7, 0.7, n) * z, z], 1)


K_TEST = np.array([[410.0, 0.0, 321.5], [0.0, 395.0, 238.25], [0.0, 0.0, 1.0]])


@pytest.mark.parametrize("k", list(KS), ids=list(KS))
def test_oracle_projection_is_colmaps_opencv_model(k):
    for p in _points():
        uv, s = dto.project_point(p, K_TEST, KS[k])
        ref = _uv_numpy(p, K_TEST, KS[k])
        assert np.abs(uv - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max()), (p, uv, ref)
        assert s == pytest.approx((p[0] ** 2 + p[1] ** 2) / p[2] ** 2, rel=1e-14)


@pytest.mark.parametrize("k", list(KS), ids=list(KS))
def test_oracle_jacobian_and_its_derivative_match_central_differences_of_colmaps_model(k):
    """J = d(u, v)/dp and d<gJ, J>/dp + J^T guv of the oracle against central differences of the numpy transcription."""
    rng = np.random.default_rng(7)
    fx, fy = K_TEST[0, 0], K_TEST[1, 1]
    for p in _points(40):
        gJ, guv = rng.standard_normal(6), rng.standard_normal(2)
        J, g = dto.jacobian_vjp(p, fx, fy, KS[k], gJ, guv)
        h = 1e-5 * p[2]
        Jn = np.zeros((2, 3))
        for c in range(3):
            e = np.eye(3)[c] * h
            Jn[:, c] = (_uv_numpy(p + e, K_TEST, KS[k]) - _uv_numpy(p - e, K_TEST, KS[k])) / (2 * h)
        assert np.abs(J - Jn).max() <= 1e-6 * np.abs(Jn).max(), (J, Jn)
        gn = np.zeros(3)
        for c in range(3):
            e = np.eye(3)[c] * h
            Jp, _ = dto.jacobian_vjp(p + e, fx, fy, KS[k], gJ, guv)
            Jm, _ = dto.jacobian_vjp(p - e, fx, fy, KS[k], gJ, guv)
            gn[c] = (gJ * (Jp - Jm).reshape(-1)).sum() / (2 * h) + guv @ Jn[:, c]
        assert np.abs(g - gn).max() <= 1e-6 * np.abs(gn).max(), (g, gn)


# ---- fp64 finite differences through the render oracle ----------------------------------------------------------------------
def _upstream(H, W, seed=1):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((H, W, 3)) / (3 * H * W), rng.standard_normal((H, W)) / (H * W),
            rng.standard_normal((H, W)) / (H * W))


@pytest.mark.parametrize("k", list(KS), ids=list(KS))
@pytest.mark.parametrize("mode", ["plain", "depth", "antialiased", "filter3d"])
def test_fp64_distortion_backward_matches_finite_differences(k, mode):
    """<G,image> + <Gd,depth> + <Ga,alpha> against central differences of the fp64 distorted forward, every parameter
    (SH 0, so that xyz's gradient is complete).  The scene is the tiny synthetic one seen through the lens."""
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
        return dto.rasterize(s["xyz"], s["quaternion"], s["scale"], s["opacity"], s["rgb"], s["sh"], s["T"], s["K"],
                             s["H"], s["W"], KS[k], antialiased=aa, filter3d=f3d, background=np.full(3, 0.5))

    o = forward()
    assert o.keep.sum() > 64 and len(o.sorted_idx) > 100
    d = dto.rasterize_backward(o, G, Gd, Ga)

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


# ---- r2_max --------------------------------------------------------------------------------------------------------------
R2_TABLE = [
    (0.0, 0.0, 0.0, 0.0, 0.0),            # pinhole: +inf
    (-0.12, 0.03, 5e-4, -3e-4, 0.0),      # typical barrel: monotone, +inf
    (0.1, 0.01, 0.0, 0.0, 0.0),           # pincushion: +inf
    (-0.3, 0.0, 0.0, 0.0, 0.0),           # folds at s = 1/0.9
    (-0.3, 0.08, 0.0, 0.0, -0.02),        # folds (cubic)
    (-0.05, 0.0, 1e-3, 1e-3, -0.01),      # folds through k3 alone, tangential terms ignored
    (0.2, -0.4, 0.0, 0.0, 0.05),          # folds
    (-2.0, 1.5, 0.0, 0.0, 0.0),           # folds early
]


def _dt_lib():
    if not DISTORTION_LIB.exists():
        pytest.skip("libgsr_distortion.so is not built")
    lib = C.CDLL(str(DISTORTION_LIB))
    lib.gsr_distortion_r2_max.restype = C.c_float
    return lib


@pytest.mark.parametrize("k", R2_TABLE)
def test_r2_max_is_the_smallest_positive_root_rounded_down(k):
    from gaussian_splatting_b200.rasterize import distortion_r2_max

    k32 = np.asarray(k, np.float32)
    ref = dto.r2_max(k32.astype(np.float64))
    c = _dt_lib().gsr_distortion_r2_max(k32.ctypes.data_as(C.POINTER(C.c_float)))
    py = distortion_r2_max(k)
    assert py == float(np.float32(c))
    if np.isinf(ref):
        assert np.isinf(c) and c > 0, (k, c)
        return
    want = np.float32(ref)
    if float(want) > ref:
        want = np.nextafter(want, np.float32(0))
    assert abs(np.float32(c) - want) <= np.spacing(want), (k, c, want)
    assert float(np.float32(c)) <= ref


def test_r2_max_of_non_finite_or_missing_coefficients_is_nan():
    from gaussian_splatting_b200.rasterize import distortion_r2_max

    lib = _dt_lib()
    for bad in ([np.nan, 0, 0, 0, 0], [0, 0, np.inf, 0, 0], [0, 0, 0, 0, -np.inf]):
        b = np.array(bad, np.float32)
        assert np.isnan(lib.gsr_distortion_r2_max(b.ctypes.data_as(C.POINTER(C.c_float))))
    assert np.isnan(lib.gsr_distortion_r2_max(None))
    with pytest.raises(ValueError):
        distortion_r2_max((np.nan, 0, 0, 0, 0))


# ---- argument errors -----------------------------------------------------------------------------------------------------
def _gaussians(n=4, dtype=torch.float32, sh=None):
    from gaussian_splatting_b200.structs import Gaussians

    return Gaussians(torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 1, dtype=dtype),
                     torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 4, dtype=dtype), sh)


def test_rasterize_distortion_argument_errors():
    from gaussian_splatting_b200.rasterize import rasterize
    from gaussian_splatting_b200.structs import Camera

    def call(g=None, use_sh_precompute=True, **kw):
        g = _gaussians() if g is None else g
        dt = g.xyz.dtype
        return rasterize(g, torch.eye(4, dtype=dt), Camera(64, 64, torch.eye(3, dtype=dt)), 0.3, 500.0, 100, 3.0,
                         use_sh_precompute, torch.zeros(3, dtype=dt), **kw)

    k = (-0.1, 0.01, 0.0, 0.0, 0.0)
    with pytest.raises(TypeError):
        call(_gaussians(dtype=torch.float64), distortion=k)
    with pytest.raises(ValueError):
        call(_gaussians(sh=torch.zeros(4, 3, 3)), use_sh_precompute=False, distortion=k)
    with pytest.raises(ValueError):
        call(distortion=k, fisheye=(0.0, 0.0, 0.0, 0.0))
    for bad in ((0.1, 0.0, 0.0, 0.0), (0.1, 0.0, 0.0, 0.0, 0.0, 0.0), [[0.1, 0, 0, 0, 0]], (float("nan"), 0, 0, 0, 0),
                (0, 0, float("inf"), 0, 0), (0, 0, 0, 0, 1e39), torch.zeros(4), torch.zeros(2, 5), "abcde",
                (0, 0, "x", 0, 0)):
        with pytest.raises(ValueError):
            call(distortion=bad)
    if torch.cuda.is_available():
        with pytest.raises(ValueError):
            call(distortion=torch.zeros(5, device="cuda"))
    with pytest.raises(ValueError):
        call(distortion=torch.zeros(5, device="meta"))


def test_rasterize_batch_distortion_argument_errors():
    from gaussian_splatting_b200 import rasterize_batch
    from gaussian_splatting_b200.structs import Camera

    def call(g=None, use_sh_precompute=True, **kw):
        g = _gaussians() if g is None else g
        dt = g.xyz.dtype
        return rasterize_batch(g, torch.eye(4, dtype=dt).expand(2, 4, 4), Camera(64, 64, torch.eye(3, dtype=dt)), 0.3,
                               500.0, 100, 3.0, use_sh_precompute, torch.zeros(3, dtype=dt), **kw)

    with pytest.raises(TypeError):
        call(_gaussians(dtype=torch.float64), distortion=(0, 0, 0, 0, 0))
    with pytest.raises(ValueError):
        call(_gaussians(sh=torch.zeros(4, 3, 3)), use_sh_precompute=False, distortion=(0, 0, 0, 0, 0))
    with pytest.raises(ValueError):
        call(distortion=(0, 0, 0, 0, 0), fisheye=(0, 0, 0, 0))
    for bad in (torch.zeros(3, 5), torch.zeros(2, 4), torch.zeros(2, 2, 5), [(0, 0, 0, 0, 0)] * 3,
                [(0, 0, 0, 0, 0), (0, 0, float("nan"), 0, 0)], torch.zeros(5, device="meta")):
        with pytest.raises(ValueError):
            call(distortion=bad)


# ---- camera_from_colmap ----------------------------------------------------------------------------------------------------
COLMAP_CASES = [
    ("SIMPLE_PINHOLE", [500.0, 320.0, 240.0], (500, 500, 320, 240), {}),
    ("PINHOLE", [500.0, 510.0, 320.0, 240.0], (500, 510, 320, 240), {}),
    ("SIMPLE_RADIAL", [500.0, 320.0, 240.0, -0.05], (500, 500, 320, 240),
     {"distortion": (-0.05, 0.0, 0.0, 0.0, 0.0)}),
    ("RADIAL", [500.0, 320.0, 240.0, -0.05, 0.01], (500, 500, 320, 240), {"distortion": (-0.05, 0.01, 0.0, 0.0, 0.0)}),
    ("OPENCV", [500.0, 510.0, 320.0, 240.0, -0.1, 0.02, 1e-3, -2e-3], (500, 510, 320, 240),
     {"distortion": (-0.1, 0.02, 1e-3, -2e-3, 0.0)}),
    ("FULL_OPENCV", [500.0, 510.0, 320.0, 240.0, -0.1, 0.02, 1e-3, -2e-3, 0.005, 0.0, 0.0, 0.0], (500, 510, 320, 240),
     {"distortion": (-0.1, 0.02, 1e-3, -2e-3, 0.005)}),
    ("OPENCV_FISHEYE", [500.0, 510.0, 320.0, 240.0, 0.1, -0.02, 0.003, -0.001], (500, 510, 320, 240),
     {"fisheye": (0.1, -0.02, 0.003, -0.001)}),
]


@pytest.mark.parametrize("model,params,fxfycxcy,lens", COLMAP_CASES, ids=[c[0] for c in COLMAP_CASES])
def test_camera_from_colmap(model, params, fxfycxcy, lens):
    from gaussian_splatting_b200.structs import camera_from_colmap

    cam, kw = camera_from_colmap(model, 640, 480, params)
    fx, fy, cx, cy = fxfycxcy
    assert (cam.width, cam.height) == (640, 480)
    assert cam.K.dtype == torch.float32 and cam.K.device.type == "cpu"
    assert torch.equal(cam.K, torch.tensor([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=torch.float32))
    assert kw == lens
    cam2, kw2 = camera_from_colmap(model.lower(), 640, 480, np.asarray(params))
    assert torch.equal(cam2.K, cam.K) and kw2 == kw


def test_camera_from_colmap_refuses_what_it_cannot_project():
    from gaussian_splatting_b200.structs import camera_from_colmap

    for model in ("SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE", "FOV", "THIN_PRISM_FISHEYE", "RAD_TAN_THIN_PRISM_FISHEYE"):
        with pytest.raises(ValueError, match=model):
            camera_from_colmap(model, 640, 480, [500.0, 320.0, 240.0, 0.1, 0.1, 0.1, 0.1, 0.1])
    with pytest.raises(ValueError, match="FULL_OPENCV"):
        camera_from_colmap("FULL_OPENCV", 640, 480, [500, 510, 320, 240, -0.1, 0.02, 0, 0, 0, 0.01, 0, 0])
    with pytest.raises(ValueError, match="OPENCV"):
        camera_from_colmap("OPENCV", 640, 480, [500, 510, 320, 240, -0.1])


# ---- the library -----------------------------------------------------------------------------------------------------------
def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists():
        pytest.skip(f"{name} is missing")
    return exe


def _cuobjdump(*args, lib=DISTORTION_LIB):
    if not lib.exists():
        pytest.skip("the built library is missing")
    return subprocess.run([_tool("cuobjdump"), *args, str(lib)], check=True, capture_output=True, text=True).stdout


def test_distortion_header_declares_exactly_the_new_symbols_and_the_library_exports_them():
    header = (ROOT / "include" / "gsr_distortion.h").read_text()
    declared = set(re.findall(r"^\w[\w\s\*]*?\b(gsr_\w+)\s*\(", header, re.M))
    assert declared == {"gsr_distortion_r2_max", "gsr_distortion_preprocess_forward",
                        "gsr_distortion_preprocess_backward", "gsr_distortion_batch_preprocess_backward"}, declared
    assert re.search(r"#define GSR_DISTORTION_CONSTS 6\b", header)
    lib = _dt_lib()
    for name in declared:
        assert hasattr(lib, name), name


KINDS = {"k_distortion_preprocess_fwd": (16, 6), "k_distortion_preprocess_bwd": (32, 4),
         "k_distortion_batch_preprocess_bwd": (32, 3)}


def test_distortion_kernels_are_sm90a_and_keep_their_registers_out_of_local_memory():
    """Every mode combination is there: 16 forward, 32 backward and 32 batched backward kernels.  The backward
    kernels use no local memory; the forward kernels no more stack than their pinhole counterparts (the division slow
    path's saves, 32 bytes)."""
    elfs = _cuobjdump("--list-elf")
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage")))
    for kind, (n, _) in KINDS.items():
        names = [k for k in usage if re.search(rf"\d{kind}I", k)]
        assert len(names) == n, (kind, len(names))
        for name in names:
            u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[name])}
            assert u["LOCAL"] == 0, (name, u)
            assert u["STACK"] <= (32 if kind.endswith("fwd") else 0), (name, u)


def test_distortion_launch_bounds_are_the_fisheyes():
    """6 / 4 / 3 CTAs of 128 threads per SM: ptxas's register cap of every kernel is the one those bounds give."""
    elf = _cuobjdump("-elf")
    caps = {}
    for name, body in re.findall(r"^\.nv\.info\.(\S+)\n(.*?)(?=^\.|\Z)", elf, re.M | re.S):
        m = re.search(r"EIATTR_MAXREG_COUNT\s*\n\s*Format:\s*\S+\s*\n\s*Value:\s*(0x[0-9a-f]+)", body)
        if m:
            caps[name] = int(m.group(1), 16)
    for kind, (n, ctas) in KINDS.items():
        got = {v for k, v in caps.items() if re.search(rf"\d{kind}I", k)}
        assert sum(1 for k in caps if re.search(rf"\d{kind}I", k)) == n, kind
        assert got == {65536 // (ctas * 128) // 8 * 8}, (kind, got)


def test_existing_kernels_keep_their_sass():
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_distortion.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    for lib in ("libgsr_b200.so", "libgsr_batch.so", "libgsr_fisheye.so"):
        if not (PKG / lib).exists():
            pytest.skip(f"{lib} is not built")
        now = {k: d for k, (d, n) in sass_digest.per_kernel(PKG / lib).items()}
        assert set(now) == set(rec[lib]), lib
        changed = sorted(k for k, d in rec[lib].items() if now[k] != d)
        assert not changed, (lib, changed)
        assert "distortion" not in "".join(now)
