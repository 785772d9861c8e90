"""Rolling-shutter cameras without a GPU: the fp64 oracle (tests/shutter_oracle.py) against central differences, the
fixed-step Newton solve's residual in fp32, an independent per-line check of the shear, se3_log and
shutter_from_endpoints, argument errors, and the library (symbols, resources, launch bounds, untouched SASS)."""
import ctypes as C
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import pose
from gaussian_splatting_b200.rasterize import rasterize, rasterize_batch
from gaussian_splatting_b200.structs import Camera, Gaussians
from tests import shutter_oracle as so

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "gaussian_splatting_b200"
SHUTTER_LIB = PKG / "libgsr_shutter.so"
LENS_K = {"pinhole": None, "fisheye": [0.05, -0.01, 0.002, -0.0005], "distortion": [-0.1, 0.02, 0.001, -0.002, 0.003]}
H, W = 60, 80


# ---- the fp64 oracle -------------------------------------------------------------------------------------------------
def _scene():
    """Gaussians inside the image, beyond each of its four sides (tau* clamped at 0 and at 1 for every readout) and
    one close to the camera, where the readout motion is fast (lambda near its limit)."""
    rng = np.random.default_rng(4)
    K = torch.tensor([[70.0, 0, 39.5], [0, 75.0, 29.5], [0, 0, 1]], dtype=torch.float64)
    uvz = [(20, 15, 4.0), (60, 40, 5.0), (40, 30, 3.5), (-12, 30, 4.0), (95, 25, 4.5), (40, -12, 4.0), (45, 75, 5.0),
           (30, 35, 0.9)]
    xyz = torch.tensor([((u - 39.5) * z / 70.0, (v - 29.5) * z / 75.0, z) for u, v, z in uvz], dtype=torch.float64)
    n = len(uvz)
    quat = torch.from_numpy(rng.standard_normal((n, 4)))
    scale = torch.from_numpy(rng.uniform(-3.5, -2.0, (n, 3)))
    opa = torch.from_numpy(rng.standard_normal(n))
    rows = torch.from_numpy(rng.standard_normal((n, 12)))
    f3d = torch.from_numpy(rng.uniform(0, 0.03, n))
    return xyz, quat, scale, opa, K, rows, f3d


def _xi(readout):
    """a readout motion whose translation moves the near gaussian along the lines at about half the readout's speed"""
    sign = -1.0 if readout in ("bottom_to_top", "right_to_left") else 1.0
    rho = [0.05, 0.4 * sign, 0.05] if readout in so.READOUTS[:2] else [0.46 * sign, 0.05, 0.05]
    return torch.tensor(rho + [0.06, 0.08, -0.04], dtype=torch.float64)
FLAGS = {"plain": {}, "depth": {}, "antialiased": dict(antialiased=True), "filter3d": dict(filter3d=True)}


def _loss(lens, mode, readout, rows, K, f3d):
    """(sum, per-gaussian terms, outputs) of <rows, outputs>: each gaussian's term depends on its own parameters only"""
    def L(xyz, quat, scale, opa, T, xi):
        kw = dict(FLAGS[mode])
        if kw.pop("filter3d", False):
            kw["filter3d"] = f3d
        o = so.forward(lens, xyz, quat, scale, opa, T, K, LENS_K[lens], xi, readout, H, W, **kw)
        per = (rows[:, 3] * o["opacity"] + (rows[:, 4:6] * o["uv"]).sum(1) + (rows[:, 6:9] * o["conic"]).sum(1)
               + (rows[:, 9] * o["z"] if mode == "depth" else 0))
        return per.sum(), per, o
    return L


@pytest.mark.parametrize("readout", so.READOUTS)
@pytest.mark.parametrize("mode", list(FLAGS))
@pytest.mark.parametrize("lens", list(LENS_K))
def test_fp64_oracle_matches_central_differences(lens, mode, readout):
    """Every gaussian parameter, all 12 pose entries and all 6 twist entries, with gaussians clamped at both ends of
    the readout and one near lambda_max.  A gaussian parameter component is stepped in every gaussian at once (each
    gaussian's term depends on its own parameters only)."""
    xyz, quat, scale, opa, K, rows, f3d = _scene()
    T = pose.se3_exp(torch.tensor([0.05, -0.03, 0.02, 0.01, -0.02, 0.015], dtype=torch.float64))
    L = _loss(lens, mode, readout, rows, K, f3d)
    ins = [t.clone().requires_grad_(True) for t in (xyz, quat, scale, opa, T, _xi(readout))]
    val, _, o = L(*ins)
    assert bool(o["clamped"].any()) and float(o["lam"].max()) > 0.3, (o["clamped"], o["lam"])
    assert float(o["lam"].max()) < so.LAMBDA_MAX
    g = torch.autograd.grad(val, ins)
    h = 1e-6

    def diff(i, step):
        a = [x.detach().clone() for x in ins]
        b = [x.detach().clone() for x in ins]
        step(a[i], h)
        step(b[i], -h)
        return L(*a), L(*b)

    for i in range(4):
        t = ins[i]
        fd = torch.zeros_like(t).view(t.shape[0], -1)
        for j in range(fd.shape[1]):
            (_, pa, _), (_, pb, _) = diff(i, lambda x, d: x.view(x.shape[0], -1)[:, j].add_(d))
            fd[:, j] = (pa - pb) / (2 * h)
        err = (g[i].view(fd.shape) - fd).abs().max() / fd.abs().max()
        assert err < 1e-6, (lens, mode, readout, i, float(err))
    for i, n in ((4, 12), (5, 6)):
        fd = torch.zeros(n, dtype=torch.float64)
        for j in range(n):
            (sa, _, _), (sb, _, _) = diff(i, lambda x, d: x.view(-1)[j].add_(d))
            fd[j] = (sa - sb) / (2 * h)
        err = (g[i].reshape(-1)[:n] - fd).abs().max() / fd.abs().max()
        assert err < 1e-6, (lens, mode, readout, i, float(err))


@pytest.mark.parametrize("readout", so.READOUTS)
def test_fp64_oracle_at_zero_twist_is_the_global_shutter_and_its_twist_gradient_is_finite(readout):
    xyz, quat, scale, opa, K, rows, f3d = _scene()
    T = pose.se3_exp(torch.tensor([0.05, -0.03, 0.02, 0.01, -0.02, 0.015], dtype=torch.float64))
    xi = torch.zeros(6, dtype=torch.float64, requires_grad=True)
    L = _loss("pinhole", "plain", readout, rows, K, f3d)
    val, _, o = L(xyz, quat, scale, opa, T, xi)
    p = xyz @ T[:3, :3].T + T[:3, 3]
    assert torch.allclose(o["uv"], so.project("pinhole", p, K, None), atol=1e-12)
    (g,) = torch.autograd.grad(val, [xi])
    fd = torch.zeros(6, dtype=torch.float64)
    for j in range(6):
        e = torch.zeros(6, dtype=torch.float64)
        e[j] = 1e-6
        fd[j] = (L(xyz, quat, scale, opa, T, e)[0] - L(xyz, quat, scale, opa, T, -e)[0]) / 2e-6
    assert torch.isfinite(g).all() and ((g - fd).abs().max() / fd.abs().max()) < 1e-6


# ---- the kernel's fixed Newton iteration in fp32 ---------------------------------------------------------------------
NEWTON_STEPS = 4  # SHUTTER_NEWTON_STEPS of gsr_shutter.cuh
TOL = 2.0 ** -20


def _f32_solve(p0, xi, fx, cx, e1):
    """gsr_shutter.cuh shutter_solve for the pinhole and a top-to-bottom readout, in numpy float32 (series branch of
    the rotation, as every motion below half a radian between the middle line and a gaussian's line takes)"""
    f = np.float32
    rho, w = xi[:3].astype(f), xi[3:].astype(f)

    def point(s):
        ph = (s[:, None] * w).astype(f)
        t = (ph * ph).sum(1).astype(f)
        a = f(1) + t * (f(-1 / 6) + t * (f(1 / 120) + t * (f(-1 / 5040) + t * f(1 / 362880))))
        b = f(0.5) + t * (f(-1 / 24) + t * (f(1 / 720) + t * (f(-1 / 40320) + t * f(1 / 3628800))))
        c = f(1 / 6) + t * (f(-1 / 120) + t * (f(1 / 5040) + t * (f(-1 / 362880) + t * f(1 / 39916800))))
        sr = (s[:, None] * rho).astype(f)
        c1 = np.cross(ph, p0).astype(f)
        c2 = np.cross(ph, c1).astype(f)
        d1 = np.cross(ph, sr).astype(f)
        d2 = np.cross(ph, d1).astype(f)
        return (p0 + (a[:, None] * c1 + b[:, None] * c2 + (sr + b[:, None] * d1 + c[:, None] * d2))).astype(f)

    def evaluate(tau):
        p = point((tau - f(0.5)).astype(f))
        v = (fx * p[:, 1] / p[:, 2] + cx).astype(f)
        pd = (np.cross(w, p) + rho).astype(f)
        Jv = np.stack([np.zeros_like(v), fx / p[:, 2], -fx * p[:, 1] / (p[:, 2] * p[:, 2])], 1).astype(f)
        lam = (e1 * (Jv * pd).sum(1)).astype(f)
        return (e1 * v).astype(f), lam

    r, lam = evaluate(np.full(len(p0), 0.5, f))
    tau = np.clip(r, 0, 1).astype(f)
    for _ in range(NEWTON_STEPS):
        r, lam = evaluate(tau)
        nt = np.clip(tau - (tau - r) / (f(1) - lam), 0, 1).astype(f)
        tau = np.where((lam < so.LAMBDA_MAX) & (nt == nt), nt, tau).astype(f)
    r, lam = evaluate(tau)
    return np.abs(tau - np.clip(r, 0, 1)), lam


def test_fixed_newton_steps_reach_the_tolerance_over_the_admitted_slopes():
    """Points across a 1080-line image, motions along the readout from lambda = -1 to lambda_max (pitch and
    translation along y, plus yaw and roll): after the fixed steps the residual is within 2^-20 wherever lambda is
    below its limit."""
    rng = np.random.default_rng(0)
    Hh, fx = 1080, 1000.0
    e1 = np.float32(1.0 / (Hh - 1))
    n = 20000
    z = rng.uniform(1.0, 20.0, n)
    v = rng.uniform(-50, Hh + 50, n)
    p0 = np.stack([rng.uniform(-1, 1, n) * z, (v - 539.5) * z / fx, z], 1).astype(np.float32)
    worst, covered = 0.0, []
    for lam_target in np.linspace(-1.0, 0.74, 30):
        # lambda ~ -fy * (omega_x + rho_y / z) / (H - 1) at the image centre
        wx = -lam_target * (Hh - 1) / fx  # a positive pitch moves the image up the lines: lambda < 0
        xi = np.array([0.0, 0.02 * wx, 0.0, wx, 0.3 * wx, 0.1 * wx])
        res, lam = _f32_solve(p0, xi, np.float32(fx), np.float32(539.5), e1)
        ok = lam < so.LAMBDA_MAX
        covered.append(lam[ok])
        worst = max(worst, float(res[ok].max()))
    lam_all = np.concatenate(covered)
    assert lam_all.min() < -0.9 and lam_all.max() > 0.7
    assert worst <= TOL, worst


# ---- an independent check of the shear ------------------------------------------------------------------------------
def _splat(img_shape, mean, cov, rows=None):
    """the unnormalised gaussian exp(-d^T cov^-1 d / 2) at integer pixel centres (numpy)"""
    Hh, Ww = img_shape
    ys, xs = np.mgrid[0:Hh, 0:Ww].astype(np.float64)
    d = np.stack([xs - mean[0], ys - mean[1]], -1)
    P = np.linalg.inv(cov)
    return np.exp(-0.5 * np.einsum("...i,ij,...j->...", d, P, d))


def _exp_np(xi):
    rho, w = xi[:3], xi[3:]
    th = np.linalg.norm(w)
    Wx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th < 1e-8:
        R, V = np.eye(3) + Wx, np.eye(3) + Wx / 2
    else:
        R = np.eye(3) + np.sin(th) / th * Wx + (1 - np.cos(th)) / th ** 2 * Wx @ Wx
        V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * Wx + (th - np.sin(th)) / th ** 3 * Wx @ Wx
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, V @ rho
    return T


def _per_line_image(x, Sigma, xi, K, Hh, Ww):
    """What a rolling-shutter sensor records of one gaussian: line k is the frozen-time EWA splat seen from
    T(k / (H - 1)) (numpy only, no part of the model's derivation)"""
    img = np.zeros((Hh, Ww))
    for k in range(Hh):
        T = _exp_np((k / (Hh - 1) - 0.5) * xi)
        p = T[:3, :3] @ x + T[:3, 3]
        u = np.array([K[0, 0] * p[0] / p[2] + K[0, 2], K[1, 1] * p[1] / p[2] + K[1, 2]])
        J = np.array([[K[0, 0] / p[2], 0, -K[0, 0] * p[0] / p[2] ** 2], [0, K[1, 1] / p[2], -K[1, 1] * p[1] / p[2] ** 2]])
        M = J @ T[:3, :3]
        img[k] = _splat((Hh, Ww), u, M @ Sigma @ M.T)[k]
    return img


@pytest.mark.parametrize("motion", ["pan", "vertical"])
def test_sheared_splat_converges_to_the_per_line_image(motion):
    """One gaussian; the model's single sheared splat against the per-line image as the splat shrinks: the relative
    L2 error falls roughly in proportion to its size, and at the smallest size it is at most 1/5 of the error of the
    same splat without the shear (A = I)."""
    Hh, Ww = 120, 120
    K = np.array([[150.0, 0, 59.5], [0, 150.0, 59.5], [0, 0, 1]])
    # >= 5 % of the image over the readout: 0.1 rad of yaw is 15 px across the lines, 0.08 rad of pitch 12 px along
    xi = np.array([0, 0, 0, 0, 0.1, 0.0]) if motion == "pan" else np.array([0, 0.05, 0, 0.08, 0, 0.0])
    x = np.array([0.1, -0.05, 3.0])
    errs, errs_id = [], []
    for sig in (0.08, 0.04, 0.02):
        Sigma = np.diag([sig ** 2, (0.7 * sig) ** 2, (0.5 * sig) ** 2])
        truth = _per_line_image(x, Sigma, xi, K, Hh, Ww)
        t = lambda a: torch.from_numpy(np.asarray(a, np.float64))  # noqa: E731
        q = t([[1.0, 0, 0, 0]])
        o = so.forward("pinhole", t(x[None]), q, t(np.log(np.sqrt(np.diag(Sigma)))[None]), t([0.0]),
                       t(np.eye(4)), t(K), None, t(xi), "top_to_bottom", Hh, Ww)
        mean = o["uv"][0].detach().numpy()
        model = _splat((Hh, Ww), mean, o["cov"][0].detach().numpy())
        # the same splat at the same time without A
        tau = float(o["tau"][0])
        Tt = _exp_np((tau - 0.5) * xi)
        p = Tt[:3, :3] @ x + Tt[:3, 3]
        J = np.array([[K[0, 0] / p[2], 0, -K[0, 0] * p[0] / p[2] ** 2], [0, K[1, 1] / p[2], -K[1, 1] * p[1] / p[2] ** 2]])
        M = J @ Tt[:3, :3]
        plain = _splat((Hh, Ww), mean, M @ Sigma @ M.T)
        nrm = np.linalg.norm(truth)
        errs.append(np.linalg.norm(model - truth) / nrm)
        errs_id.append(np.linalg.norm(plain - truth) / nrm)
    # halving the size roughly halves the error (allow 0.35 .. 0.65 per halving)
    for a, b in zip(errs, errs[1:]):
        assert 0.3 * a <= b <= 0.7 * a, (motion, errs)
    assert errs[-1] * 5 <= errs_id[-1], (motion, errs, errs_id)


# ---- pose helpers --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [0.0, 1e-6, 1e-3, 0.1, 1.0, 3.0])
def test_se3_log_inverts_se3_exp_and_matches_logm(scale):
    from scipy.linalg import logm

    gen = torch.Generator().manual_seed(1)
    xi = torch.randn(8, 6, generator=gen, dtype=torch.float64)
    w = xi[:, 3:]
    xi[:, 3:] = w / w.norm(dim=-1, keepdim=True) * scale
    T = pose.se3_exp(xi)
    back = pose.se3_log(T)
    assert (back - xi).abs().max() < 1e-12
    for Tk, bk in zip(T, back):
        Lm = logm(Tk.numpy()).real
        ref = np.concatenate([Lm[:3, 3], [Lm[2, 1], Lm[0, 2], Lm[1, 0]]])
        assert np.abs(bk.numpy() - ref).max() < 1e-10
    g = torch.autograd.functional.jacobian(pose.se3_log, pose.se3_exp(torch.zeros(6, dtype=torch.float64)))
    assert torch.isfinite(g).all()


def test_shutter_from_endpoints_reproduces_the_first_and_last_line_poses():
    gen = torch.Generator().manual_seed(2)
    Ts = pose.se3_exp(torch.randn(4, 6, generator=gen, dtype=torch.float64))
    Te = pose.se3_exp(0.05 * torch.randn(4, 6, generator=gen, dtype=torch.float64)) @ Ts
    Tm, xi = pose.shutter_from_endpoints(Ts, Te)
    assert (pose.se3_exp(-0.5 * xi) @ Tm - Ts).abs().max() < 1e-12
    assert (pose.se3_exp(0.5 * xi) @ Tm - Te).abs().max() < 1e-12
    Tm0, xi0 = pose.shutter_from_endpoints(Ts, Ts)
    assert xi0.abs().max() < 1e-12 and (Tm0 - Ts).abs().max() < 1e-12


# ---- argument errors before any launch -------------------------------------------------------------------------------
def _cpu_gaussians(n=4, dtype=torch.float32, sh=False):
    return Gaussians(torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 1, dtype=dtype),
                     torch.zeros(n, 3, dtype=dtype), torch.ones(n, 4, dtype=dtype),
                     torch.zeros(n, 3, 15, dtype=dtype) if sh else None)


def _call(xi, readout="top_to_bottom", K=None, dtype=torch.float32, sh=False, precompute=True, h=48, **kw):
    K = torch.eye(3) if K is None else K
    return rasterize(_cpu_gaussians(dtype=dtype, sh=sh), torch.eye(4, dtype=dtype), Camera(64, h, K.to(dtype)), 0.3,
                     100.0, 10, 3.0, precompute, torch.zeros(3, dtype=dtype), rolling_shutter=xi, readout=readout, **kw)


@pytest.mark.parametrize("case, exc", [
    (dict(xi=torch.zeros(5)), ValueError),
    (dict(xi=torch.zeros(2, 6)), ValueError),
    (dict(xi=torch.zeros(6, dtype=torch.float64)), TypeError),
    (dict(xi=[0.0] * 6), TypeError),
    (dict(xi=torch.zeros(6, device="meta")), ValueError),
    (dict(xi=torch.zeros(6), readout="diagonal"), ValueError),
    (dict(xi=None, readout="diagonal"), ValueError),
    (dict(xi=torch.zeros(6), h=1), ValueError),
    (dict(xi=torch.zeros(6), K=torch.eye(3).requires_grad_(True)), ValueError),
    (dict(xi=torch.zeros(6), fisheye=torch.zeros(4, requires_grad=True)), ValueError),
    (dict(xi=torch.zeros(6), dtype=torch.float64), TypeError),
    (dict(xi=torch.zeros(6), sh=True, precompute=False), ValueError),
])
def test_bad_arguments_raise_before_any_launch(case, exc):
    with pytest.raises(exc):
        _call(**case)


def test_bad_batch_twists_raise_before_any_launch():
    g = _cpu_gaussians()
    T = torch.eye(4).expand(2, 4, 4).contiguous()
    with pytest.raises(ValueError):
        rasterize_batch(g, T, Camera(64, 48, torch.eye(3)), 0.3, 100.0, 10, 3.0, True, torch.zeros(3),
                        rolling_shutter=torch.zeros(3, 6))


# ---- the library -----------------------------------------------------------------------------------------------------
def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists():
        pytest.skip(f"{name} is not available")
    return exe


def _cuobjdump(*args, lib=SHUTTER_LIB):
    if not lib.exists():
        pytest.skip("the built library is missing")
    return subprocess.run([_tool("cuobjdump"), *args, str(lib)], check=True, capture_output=True, text=True).stdout


SHUTTER_SYMBOLS = {"gsr_shutter_temp_bytes", "gsr_shutter_preprocess_forward", "gsr_shutter_preprocess_backward",
                   "gsr_shutter_batch_preprocess_backward"}


def test_shutter_header_declares_exactly_the_new_symbols_and_the_library_exports_them():
    header = (ROOT / "include" / "gsr_shutter.h").read_text()
    declared = set(re.findall(r"^\w[\w\s\*]*?\b(gsr_\w+)\s*\(", header, re.M))
    assert declared == SHUTTER_SYMBOLS, declared
    if not SHUTTER_LIB.exists():
        pytest.skip("libgsr_shutter.so is not built")
    lib = C.CDLL(str(SHUTTER_LIB))
    nm = subprocess.run(["nm", "-D", "--defined-only", str(SHUTTER_LIB)], capture_output=True, text=True).stdout
    assert set(re.findall(r"\bT (gsr_\w+)", nm)) == declared
    lib.gsr_shutter_temp_bytes.restype = C.c_size_t
    assert lib.gsr_shutter_temp_bytes(3, 1000) == (3 * 8 * 20 * 4 + 255) // 256 * 256
    assert lib.gsr_shutter_temp_bytes(1, 0) == 0


# the kernels of every lens: 4 SH degrees x (4 forward modes | 8 backward modes); their CTAs per SM
SHUTTER_KINDS = {"k_shutter_preprocess_fwd": (16, 6), "k_shutter_preprocess_bwd": (32, 3),
                 "k_shutter_batch_preprocess_bwd": (32, 2)}
LENS_NS = ("shutter_pinhole", "shutter_fisheye", "shutter_distortion")


def test_shutter_kernels_are_sm90a_and_keep_their_registers_out_of_local_memory():
    """No local memory anywhere and no stack in the backward kernels; the forward keeps the 32-byte stack frame
    every per-gaussian forward of the other libraries has (the camera centre's pivoting)."""
    elfs = _cuobjdump("--list-elf")
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage")))
    for ns in LENS_NS:
        for kind, (count, _) in SHUTTER_KINDS.items():
            names = [k for k in usage if f"{len(ns)}{ns}" in k and re.search(rf"\d{kind}I", k)]
            assert len(names) == count, (ns, kind, len(names))
            for name in names:
                u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[name])}
                assert u["LOCAL"] == 0 and u["STACK"] <= (32 if kind.endswith("fwd") else 0), (name, u)


def test_shutter_launch_bounds():
    elf = _cuobjdump("-elf")
    caps = {}
    for name, body in re.findall(r"^\.nv\.info\.(\S+)\n(.*?)(?=^\.|\Z)", elf, re.M | re.S):
        m = re.search(r"EIATTR_MAXREG_COUNT\s*\n\s*Format:\s*\S+\s*\n\s*Value:\s*(0x[0-9a-f]+)", body)
        if m:
            caps[name] = int(m.group(1), 16)
    for ns in LENS_NS:
        for kind, (_, ctas) in SHUTTER_KINDS.items():
            got = {v for k, v in caps.items() if f"{len(ns)}{ns}" in k and re.search(rf"\d{kind}I", k)}
            assert got == {min(255, 65536 // (ctas * 128) // 8 * 8)}, (ns, kind, got)


def test_existing_kernels_keep_their_sass():
    """Every kernel of every library that existed before the rolling shutter keeps its instructions, and no library
    gains a kernel: the shutter kernels are libgsr_shutter.so's."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_shutter.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    libs = ("libgsr_b200.so", "libgsr_selective_adam.so", "libgsr_features.so", "libgsr_batch.so",
            "libgsr_fisheye.so", "libgsr_distortion.so", "libgsr_pose.so", "libgsr_calib.so", "libgsr_bilagrid.so")
    assert set(rec) - {"nvcc"} == set(libs)
    for lib in libs:
        if not (PKG / lib).exists():
            pytest.skip(f"{lib} is not built")
        now = {k: d for k, (d, n) in sass_digest.per_kernel(PKG / lib).items()}
        assert set(now) == set(rec[lib]), (lib, sorted(set(now) ^ set(rec[lib]))[:4])
        changed = sorted(k for k, d in rec[lib].items() if now[k] != d)
        assert not changed, (lib, changed)
