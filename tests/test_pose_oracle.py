"""Camera pose gradients (rasterize(..., camera_T_world requiring grad)) without a GPU: the fp64 pose VJP against
central differences of the fp64 forward for every lens and mode, se3_exp against the matrix exponential, the new
library's surface and resources, and the SASS of every kernel that existed before it."""
import ctypes as C
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import scipy.linalg
import torch

from tests import pose_oracle as po
from tests.scenes import np_scene

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "gaussian_splatting_b200"
POSE_LIB = PKG / "libgsr_pose.so"
LENS_K = {"pinhole": None, "fisheye": (0.08, -0.03, 0.01, -0.002), "distortion": (-0.12, 0.03, 5e-4, -3e-4, 0.01)}


def _upstream(H, W, seed=1):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((H, W, 3)) / (3 * H * W), rng.standard_normal((H, W)) / (H * W),
            rng.standard_normal((H, W)) / (H * W))


@pytest.mark.parametrize("lens", po.LENSES)
@pytest.mark.parametrize("mode", ["plain", "depth", "antialiased", "filter3d"])
def test_fp64_pose_gradient_matches_central_differences(lens, mode):
    """<G,image> + <Gd,depth> + <Ga,alpha> (plain: the image only) against central differences of the fp64 forward
    in all 12 entries of T[:3, :], SH 0 (the view direction does not enter).  The rows are the oracle's own render
    backward's."""
    from tests import distortion_oracle as dto

    sc = np_scene(128, "tiny", sh_degree=0, dtype=np.float64, sigma_px=(0.6, 1.2, 0.15, 8.0))
    f3d = None
    if mode == "filter3d":
        f3d = np.exp(sc["scale"].mean(1)) * np.random.default_rng(3).uniform(0.3, 1.5, len(sc["scale"]))
    aa = mode in ("antialiased", "filter3d")
    G, Gd, Ga = _upstream(sc["H"], sc["W"])
    if mode == "plain":
        Gd, Ga = np.zeros_like(Gd), np.zeros_like(Ga)

    def forward(T):
        return po.rasterize(lens, sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], T,
                            sc["K"], sc["H"], sc["W"], LENS_K[lens], antialiased=aa, filter3d=f3d,
                            background=np.full(3, 0.5))

    T0 = np.asarray(sc["T"], np.float64)
    o = forward(T0)
    assert o.keep.sum() > 64 and len(o.sorted_idx) > 100
    d = dto.rasterize_backward(o, G, Gd, Ga)
    grad, mass = po.pose_grad(o, lens, d.render)
    assert np.isfinite(grad).all() and (grad[3] == 0).all()

    def loss(T):
        p = forward(T)
        return float((p.image * G).sum() + (p.depth * Gd).sum() + (p.alpha * Ga).sum())

    h = 1e-6
    scale = np.abs(grad[:3]).max()
    assert scale > 0
    for r in range(3):
        for c in range(4):
            plus, minus = T0.copy(), T0.copy()
            plus[r, c] += h
            minus[r, c] -= h
            fd = (loss(plus) - loss(minus)) / (2 * h)
            assert abs(fd - grad[r, c]) <= 2e-5 * scale + 1e-12, (lens, mode, r, c, fd, grad[r, c])


def _twist(xi):
    A = np.zeros((4, 4))
    w = xi[3:]
    A[:3, :3] = [[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]
    A[:3, 3] = xi[:3]
    return A


@pytest.mark.parametrize("scale", [2.0, 0.5, 3e-2, 9e-3, 1e-4, 1e-7, 3e-9, 0.0])
def test_se3_exp_is_the_matrix_exponential(scale):
    from gaussian_splatting_b200.pose import se3_exp

    rng = np.random.default_rng(11)
    xis = rng.standard_normal((16, 6)) * scale
    got = se3_exp(torch.from_numpy(xis)).numpy()
    for xi, g in zip(xis, got):
        ref = scipy.linalg.expm(_twist(xi))
        assert np.abs(g - ref).max() <= 1e-13 * max(1.0, np.abs(ref).max()), (xi, g, ref)
        assert np.abs(g[:3, :3] @ g[:3, :3].T - np.eye(3)).max() <= 1e-13


def test_se3_exp_gradient_is_finite_at_zero_and_pose_delta_starts_at_identity():
    from gaussian_splatting_b200.pose import PoseDelta, se3_exp

    xi = torch.zeros(3, 6, dtype=torch.float64, requires_grad=True)
    torch.autograd.gradcheck(se3_exp, (xi,))
    torch.autograd.gradcheck(se3_exp, (torch.randn(3, 6, dtype=torch.float64, requires_grad=True),))
    T = torch.from_numpy(np.asarray(np_scene(128, "tiny", sh_degree=0, dtype=np.float64)["T"])).float()
    d = PoseDelta(4)
    assert torch.equal(d(T, 2), T)
    assert torch.equal(d(T.expand(3, 4, 4), [0, 3, 1]), T.expand(3, 4, 4))
    d.xi.data[1] = torch.tensor([0.1, -0.2, 0.3, 0.01, 0.02, -0.03])
    out = d(T, 1)
    assert torch.allclose(out, se3_exp(d.xi[1].detach()) @ T)


# ---- the library --------------------------------------------------------------------------------------------------------
def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists():
        pytest.skip(f"{name} is not available")
    return exe


def _cuobjdump(*args, lib=POSE_LIB):
    if not lib.exists():
        pytest.skip("the built library is missing")
    return subprocess.run([_tool("cuobjdump"), *args, str(lib)], check=True, capture_output=True, text=True).stdout


def test_pose_header_declares_exactly_the_new_symbols_and_the_library_exports_them():
    header = (ROOT / "include" / "gsr_pose.h").read_text()
    declared = set(re.findall(r"^\w[\w\s\*]*?\b(gsr_\w+)\s*\(", header, re.M))
    assert declared == {"gsr_pose_temp_bytes", "gsr_pose_preprocess_backward",
                        "gsr_pose_batch_preprocess_backward"}, declared
    if not POSE_LIB.exists():
        pytest.skip("libgsr_pose.so is not built")
    lib = C.CDLL(str(POSE_LIB))
    for name in declared:
        assert hasattr(lib, name), name
    nm = subprocess.run(["nm", "-D", "--defined-only", str(POSE_LIB)], capture_output=True, text=True).stdout
    exported = set(re.findall(r"\bT (gsr_\w+)", nm))
    assert exported == declared, exported
    lib.gsr_pose_temp_bytes.restype = C.c_size_t
    assert lib.gsr_pose_temp_bytes(3, 1000) == (3 * 8 * 12 * 4 + 255) // 256 * 256
    assert lib.gsr_pose_temp_bytes(1, 0) == 0


# every lens: 8 modes x 4 SH degrees, single-view and batched; the CTAs per SM of each (DESIGN.md 3.21)
KINDS = {"pose_pinhole": {"k_pose_preprocess_bwd": 4, "k_pose_batch_preprocess_bwd": 3},
         "pose_fisheye": {"k_pose_preprocess_bwd": 4, "k_pose_batch_preprocess_bwd": 3},
         "pose_distortion": {"k_pose_preprocess_bwd": 4, "k_pose_batch_preprocess_bwd": 3}}


def test_pose_kernels_are_sm90a_and_keep_their_registers_out_of_local_memory():
    elfs = _cuobjdump("--list-elf")
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage")))
    for ns, kinds in KINDS.items():
        for kind in kinds:
            names = [k for k in usage if f"{len(ns)}{ns}" in k and re.search(rf"\d{kind}I", k)]
            assert len(names) == 32, (ns, kind, len(names))
            for name in names:
                u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[name])}
                assert u["LOCAL"] == 0 and u["STACK"] == 0, (name, u)
    finish = [k for k in usage if "k_pose_finish" in k]
    assert len(finish) == 1


def test_pose_launch_bounds():
    elf = _cuobjdump("-elf")
    caps = {}
    for name, body in re.findall(r"^\.nv\.info\.(\S+)\n(.*?)(?=^\.|\Z)", elf, re.M | re.S):
        m = re.search(r"EIATTR_MAXREG_COUNT\s*\n\s*Format:\s*\S+\s*\n\s*Value:\s*(0x[0-9a-f]+)", body)
        if m:
            caps[name] = int(m.group(1), 16)
    for ns, kinds in KINDS.items():
        for kind, ctas in kinds.items():
            got = {v for k, v in caps.items() if f"{len(ns)}{ns}" in k and re.search(rf"\d{kind}I", k)}
            assert got == {65536 // (ctas * 128) // 8 * 8}, (ns, kind, got)


def test_existing_kernels_keep_their_sass():
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_pose.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    libs = ("libgsr_b200.so", "libgsr_batch.so", "libgsr_fisheye.so", "libgsr_distortion.so", "libgsr_features.so")
    assert set(rec) - {"nvcc"} == set(libs)
    for lib in libs:
        if not (PKG / lib).exists():
            pytest.skip(f"{lib} is not built")
        now = {k: d for k, (d, n) in sass_digest.per_kernel(PKG / lib).items()}
        assert set(now) == set(rec[lib]), lib
        changed = sorted(k for k, d in rec[lib].items() if now[k] != d)
        assert not changed, (lib, changed)
        assert "k_pose_" not in "".join(now)
