"""Camera self-calibration (rasterize(..., camera.K or the lens coefficients requiring grad)) without a GPU: the fp64
intrinsics and lens-coefficient VJP against central differences of the fp64 forward for every lens and mode,
IntrinsicsDelta, the library's surface and resources, the SASS of every kernel that existed before, and the host
errors."""
import ctypes as C
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import calib_oracle as co
from tests.scenes import np_scene

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "gaussian_splatting_b200"
CALIB_LIB = PKG / "libgsr_calib.so"
LENSES = ("pinhole", "fisheye", "distortion")
LENS_K = {"pinhole": None, "fisheye": (0.08, -0.03, 0.01, -0.002), "distortion": (-0.12, 0.03, 5e-4, -3e-4, 0.01)}


def _upstream(H, W, seed=1):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((H, W, 3)) / (3 * H * W), rng.standard_normal((H, W)) / (H * W),
            rng.standard_normal((H, W)) / (H * W))


@pytest.mark.parametrize("lens", LENSES)
@pytest.mark.parametrize("mode", ["plain", "depth", "antialiased", "filter3d"])
def test_fp64_camera_gradient_matches_central_differences(lens, mode):
    """<G,image> + <Gd,depth> + <Ga,alpha> (plain: the image only) against central differences of the fp64 forward in
    fx, fy, cx, cy and every lens coefficient, the cull limit held at its nominal value (cull decisions get no
    gradient).  The rows are the oracle's own render backward's."""
    from tests import distortion_oracle as dto

    sc = np_scene(128, "tiny", sh_degree=0, dtype=np.float64, sigma_px=(0.6, 1.2, 0.15, 8.0))
    f3d = None
    if mode == "filter3d":
        f3d = np.exp(sc["scale"].mean(1)) * np.random.default_rng(3).uniform(0.3, 1.5, len(sc["scale"]))
    aa = mode in ("antialiased", "filter3d")
    G, Gd, Ga = _upstream(sc["H"], sc["W"])
    if mode == "plain":
        Gd, Ga = np.zeros_like(Gd), np.zeros_like(Ga)
    K0 = np.asarray(sc["K"], np.float64)
    k0 = np.zeros(5) if LENS_K[lens] is None else np.asarray(LENS_K[lens], np.float64)
    o = co.rasterize(lens, sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], K0,
                     sc["H"], sc["W"], None if lens == "pinhole" else k0, antialiased=aa, filter3d=f3d,
                     background=np.full(3, 0.5))
    limit = {} if lens == "pinhole" else ({"tmax": o.kc[-1]} if lens == "fisheye" else {"smax": o.kc[-1]})

    def forward(K, k):
        return co.rasterize(lens, sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"],
                            sc["T"], K, sc["H"], sc["W"], None if lens == "pinhole" else k, antialiased=aa,
                            filter3d=f3d, background=np.full(3, 0.5), **limit)

    assert o.keep.sum() > 64 and len(o.sorted_idx) > 100
    d = dto.rasterize_backward(o, G, Gd, Ga)
    gK, gk, mass = co.camera_grad(o, lens, d.render)
    assert np.isfinite(gK).all() and np.isfinite(gk).all() and len(gk) == co.N_COEFFS[lens]

    def loss(K, k):
        p = forward(K, k)
        return float((p.image * G).sum() + (p.depth * Gd).sum() + (p.alpha * Ga).sum())

    for j, (r, c) in enumerate([(0, 0), (1, 1), (0, 2), (1, 2)]):
        h = 1e-6 * abs(K0[r, c])
        plus, minus = K0.copy(), K0.copy()
        plus[r, c] += h
        minus[r, c] -= h
        fd = (loss(plus, k0) - loss(minus, k0)) / (2 * h)
        assert abs(fd - gK[j]) <= 2e-5 * max(abs(gK[j]), mass[j]) + 1e-12, (lens, mode, r, c, fd, gK[j])
    for j in range(co.N_COEFFS[lens]):
        h = 1e-6
        plus, minus = k0.copy(), k0.copy()
        plus[j] += h
        minus[j] -= h
        fd = (loss(K0, plus) - loss(K0, minus)) / (2 * h)
        assert abs(fd - gk[j]) <= 2e-5 * max(abs(gk[j]), mass[4 + j]) + 1e-12, (lens, mode, j, fd, gk[j])


def test_intrinsics_delta_is_bit_identical_at_zero_and_differentiable():
    from gaussian_splatting_b200.calib import IntrinsicsDelta

    K = torch.tensor([[912.3457, 0.0, 640.1235], [0.0, 901.0001, 359.875], [0.0, 0.0, 1.0]])
    for shared in (False, True):
        d = IntrinsicsDelta(5, shared_focal=shared)
        assert d.log_focal.shape == (5, 1 if shared else 2) and d.principal.shape == (5, 2)
        assert torch.equal(d(K, 3), K)
        Kc = torch.stack([K, K * 1.5, K + 0.25])
        assert torch.equal(d(Kc, [0, 4, 2]), Kc)
        assert torch.equal(d(K, torch.tensor([1, 2])), K.expand(2, 3, 3))
        (d(Kc, [0, 4, 2]) * torch.randn(3, 3, 3)).sum().backward()
        for p in (d.log_focal, d.principal):
            assert torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0
    d = IntrinsicsDelta(2)
    with torch.no_grad():
        d.log_focal[1] = torch.tensor([0.01, -0.02])
        d.principal[1] = torch.tensor([3.0, -4.0])
    out = d(K, 1)
    assert torch.allclose(out, torch.tensor([[K[0, 0] * np.exp(0.01), 0, K[0, 2] + 3],
                                             [0, K[1, 1] * np.exp(-0.02), K[1, 2] - 4], [0, 0, 1]]))
    d = IntrinsicsDelta(2, shared_focal=True, dtype=torch.float64)
    lf = torch.tensor([[0.05], [0.0]], dtype=torch.float64, requires_grad=True)
    pp = torch.tensor([[1.0, 2.0], [0.0, 0.0]], dtype=torch.float64, requires_grad=True)
    torch.autograd.gradcheck(lambda a, b: torch.func.functional_call(d, {"log_focal": a, "principal": b},
                                                                     (K.double(), 0)), (lf, pp))


# ---- host errors ---------------------------------------------------------------------------------------------------------
def test_lens_coefficient_tensor_errors_are_raised_before_any_launch():
    from gaussian_splatting_b200.rasterize import _lens_arg, _lens_input

    k = torch.zeros(4, requires_grad=True)
    assert _lens_input(k, None) is k and _lens_input(None, k) is k
    assert _lens_input([0.1, 0.0, 0.0, 0.0], None) is None
    assert _lens_input(torch.zeros(4), None) is None
    if torch.cuda.is_available():
        with pytest.raises(ValueError, match="CPU tensor"):
            _lens_arg(torch.zeros(4, device="cuda", requires_grad=True), None)
    with pytest.raises(ValueError, match="shape"):
        _lens_arg(torch.zeros(5, requires_grad=True), None)
    with pytest.raises(ValueError, match="shape"):
        _lens_arg(None, torch.zeros(3, 5, requires_grad=True), 4)
    with pytest.raises(ValueError, match="shape"):
        _lens_arg(None, torch.zeros(4, 5, requires_grad=True))
    assert _lens_arg(None, torch.zeros(4, 5, requires_grad=True), 4)[1].shape == (4, 5)


def test_lens_coefficient_gradient_comes_back_in_the_tensors_shape_and_dtype():
    from gaussian_splatting_b200.rasterize import _intrinsics_grad, _lens_grad

    g = torch.arange(10, dtype=torch.float32).view(2, 5)
    k = torch.zeros(5, dtype=torch.float64, requires_grad=True)
    out = _lens_grad(g, k)
    assert out.dtype == torch.float64 and out.shape == (5,) and torch.equal(out, g.double().sum(0))
    k2 = torch.zeros(2, 5, requires_grad=True)
    assert torch.equal(_lens_grad(g, k2), g)
    gK = _intrinsics_grad(torch.tensor([[1.0, 2.0, 3.0, 4.0], [5.0, 6.0, 7.0, 8.0]]))
    assert gK.shape == (2, 3, 3)
    assert torch.equal(gK[1], torch.tensor([[5.0, 0, 7.0], [0, 6.0, 8.0], [0, 0, 0]]))


# ---- the library --------------------------------------------------------------------------------------------------------
def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists():
        pytest.skip(f"{name} is not available")
    return exe


def _cuobjdump(*args, lib=CALIB_LIB):
    if not lib.exists():
        pytest.skip("the built library is missing")
    return subprocess.run([_tool("cuobjdump"), *args, str(lib)], check=True, capture_output=True, text=True).stdout


CAMERA_SYMBOLS = {"gsr_camera_temp_bytes", "gsr_camera_preprocess_backward", "gsr_camera_batch_preprocess_backward"}


def test_calib_header_declares_exactly_the_new_symbols_and_the_library_exports_them():
    header = (ROOT / "include" / "gsr_calib.h").read_text()
    declared = set(re.findall(r"^\w[\w\s\*]*?\b(gsr_\w+)\s*\(", header, re.M))
    assert declared == CAMERA_SYMBOLS, declared
    if not CALIB_LIB.exists():
        pytest.skip("libgsr_calib.so is not built")
    lib = C.CDLL(str(CALIB_LIB))
    for name in declared:
        assert hasattr(lib, name), name
    nm = subprocess.run(["nm", "-D", "--defined-only", str(CALIB_LIB)], capture_output=True, text=True).stdout
    exported = set(re.findall(r"\bT (gsr_\w+)", nm))
    assert exported == declared, exported
    lib.gsr_camera_temp_bytes.restype = C.c_size_t
    for lens, values in ((0, 16), (1, 20), (2, 24)):
        assert lib.gsr_camera_temp_bytes(lens, 3, 1000) == (3 * 8 * values * 4 + 255) // 256 * 256
        assert lib.gsr_camera_temp_bytes(lens, 1, 0) == 0


# the camera-gradient kernels of every lens: 8 modes x 4 SH degrees, single-view and batched; their CTAs per SM
CAMERA_KINDS = {"camera_pinhole": {"k_camera_preprocess_bwd": 4, "k_camera_batch_preprocess_bwd": 3},
                "camera_fisheye": {"k_camera_preprocess_bwd": 4, "k_camera_batch_preprocess_bwd": 3},
                "camera_distortion": {"k_camera_preprocess_bwd": 4, "k_camera_batch_preprocess_bwd": 3}}


def test_camera_kernels_are_sm90a_and_keep_their_registers_out_of_local_memory():
    elfs = _cuobjdump("--list-elf")
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage")))
    for ns, kinds in CAMERA_KINDS.items():
        for kind in kinds:
            names = [k for k in usage if f"{len(ns)}{ns}" in k and re.search(rf"\d{kind}I", k)]
            assert len(names) == 32, (ns, kind, len(names))
            for name in names:
                u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[name])}
                assert u["LOCAL"] == 0 and u["STACK"] == 0, (name, u)
    finish = [k for k in usage if "k_camera_finish" in k]
    assert len(finish) == 3 and len(usage) == 2 * 3 * 32 + 3, sorted(usage)[:4]
    for name in finish:
        u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[name])}
        assert u["LOCAL"] == 0 and u["STACK"] == 0, (name, u)


def test_camera_launch_bounds():
    elf = _cuobjdump("-elf")
    caps = {}
    for name, body in re.findall(r"^\.nv\.info\.(\S+)\n(.*?)(?=^\.|\Z)", elf, re.M | re.S):
        m = re.search(r"EIATTR_MAXREG_COUNT\s*\n\s*Format:\s*\S+\s*\n\s*Value:\s*(0x[0-9a-f]+)", body)
        if m:
            caps[name] = int(m.group(1), 16)
    for ns, kinds in CAMERA_KINDS.items():
        for kind, ctas in kinds.items():
            got = {v for k, v in caps.items() if f"{len(ns)}{ns}" in k and re.search(rf"\d{kind}I", k)}
            assert got == {65536 // (ctas * 128) // 8 * 8}, (ns, kind, got)


def test_existing_kernels_keep_their_sass():
    """Every kernel of every library that existed before the camera gradients, the pose kernels and k_pose_finish
    included, keeps its instructions, and no library gains a kernel: the camera kernels are libgsr_calib.so's."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_calib.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    libs = ("libgsr_b200.so", "libgsr_selective_adam.so", "libgsr_features.so", "libgsr_batch.so",
            "libgsr_fisheye.so", "libgsr_distortion.so", "libgsr_pose.so", "libgsr_bilagrid.so")
    assert set(rec) - {"nvcc"} == set(libs)
    for lib in libs:
        if not (PKG / lib).exists():
            pytest.skip(f"{lib} is not built")
        now = {k: d for k, (d, n) in sass_digest.per_kernel(PKG / lib).items()}
        assert set(now) == set(rec[lib]), (lib, sorted(set(now) ^ set(rec[lib]))[:4])
        changed = sorted(k for k, d in rec[lib].items() if now[k] != d)
        assert not changed, (lib, changed)
