"""2-D Gaussian surfels through lenses without a GPU: the fp64 lens oracle (tests/surfels_lens_oracle.c) on its rays,
known answers and against central differences; the binning bound of gsr_surfels_lens.cuh compiled for the host;
argument errors; and libgsr_surfels_lens.so (symbols, resources, untouched SASS of every other library)."""
import ctypes as C
import json
import re
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import surfels_lens_oracle as lo
from tests import surfels_oracle as so
from tests.test_surfels_oracle import CASES, _cuobjdump, _stack, _tool, _torch_scene, _upstream

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "gaussian_splatting_b200"
LENS_LIB = PKG / "libgsr_surfels_lens.so"
FISHEYE = (0.03, -0.01, 0.002, -0.0005)
STRONG_FISHEYE = (-0.05, 0.004, 0.0, 0.0)
OPENCV = (-0.12, 0.03, 5e-4, -3e-4, 0.01)
BARREL = (-0.6, 0.1, 0.0, 0.0, 0.0)


def _project(lens, kc, limit, K, d):
    """pixel of the unit ray d [...,3] through the lens (fp64), and whether the ray lies on the monotone branch"""
    k = np.asarray(kc, np.float32).astype(np.float64)
    if lens == "fisheye":
        rho = np.hypot(d[..., 0], d[..., 1])
        th = np.arctan2(rho, d[..., 2])
        t = th * th
        td = th * (1 + t * (k[0] + t * (k[1] + t * (k[2] + t * k[3]))))
        s = np.where(rho > 0, td / np.where(rho > 0, rho, 1), 1 / d[..., 2])
        xd, yd, ok = s * d[..., 0], s * d[..., 1], th < limit
    else:
        a, b = d[..., 0] / d[..., 2], d[..., 1] / d[..., 2]
        s = a * a + b * b
        R = 1 + s * (k[0] + s * (k[1] + s * k[4]))
        xd = a * R + 2 * k[2] * a * b + k[3] * (s + 2 * a * a)
        yd = b * R + k[2] * (s + 2 * b * b) + 2 * k[3] * a * b
        ok = (s < limit) & (d[..., 2] > 0)
    return np.stack([K[0, 0] * xd + K[0, 2], K[1, 1] * yd + K[1, 2]], -1), ok


def _limit(lens, kc):
    return lo.lens_constants(lens, kc)[-1]


# ---- rays ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lens,kc", [("fisheye", FISHEYE), ("fisheye", STRONG_FISHEYE), ("distortion", OPENCV),
                                     ("distortion", BARREL)])
def test_rays_project_back_to_their_pixel(lens, kc):
    sc = _stack(n=1, H=60, W=80)
    sc["K"] = np.array([[18.0, 0, 39.5], [0, 19.0, 29.5], [0, 0, 1]])  # a wide field: the limits lie inside
    o = lo.render(sc, np.zeros(3), lens, kc)
    ys, xs = np.mgrid[0:60, 0:80]
    valid = o.rays[..., 2] > 0
    assert valid.sum() > 200
    if kc != OPENCV:  # the field reaches beyond the lens's monotone branch (OPENCV's has no fold)
        assert (~valid).sum() > 0
    np.testing.assert_allclose(np.linalg.norm(o.rays[valid], axis=-1), 1.0, atol=1e-14)
    pix, ok = _project(lens, kc, _limit(lens, kc), sc["K"], o.rays[valid])
    assert ok.all()
    np.testing.assert_allclose(pix, np.stack([xs[valid], ys[valid]], -1), rtol=0, atol=1e-12)
    assert (o.rays[~valid] == 0).all()


def test_zero_opencv_coefficients_give_the_pinhole_oracle():
    sc = _stack(n=5)
    G = _upstream(sc)
    a = lo.render(sc, np.full(3, 0.2), "distortion", (0.0,) * 5, grads=G)
    b = so.render(sc, np.full(3, 0.2), grads=G)
    for k in ("image", "depth", "alpha", "normal", "dist", "uv", "uv_grad"):
        np.testing.assert_allclose(getattr(a, k), getattr(b, k), rtol=1e-12, atol=1e-13, err_msg=k)
    for k in ("xyz", "quaternion", "scale", "opacity", "rgb"):
        np.testing.assert_allclose(a.g[k], b.g[k], rtol=1e-9, atol=1e-12, err_msg=k)


def test_fronto_parallel_surfel_through_a_strong_fisheye_is_the_closed_form():
    """A surfel on the optical axis facing the camera: the pixel at angle theta meets the plane z = p_z at radius
    p_z tan(theta), beyond 60 degrees too."""
    kc = (-0.02, 0.0, 0.0, 0.0)
    su, pz, opa = 3.0, 1.0, 0.9
    H = W = 61
    f = 12.0
    sc = dict(xyz=np.array([[0.0, 0.0, pz]]), quaternion=np.array([[1.0, 0, 0, 0]]),
              scale=np.array([[np.log(su), np.log(su), 0.0]]), opacity=np.array([[np.log(opa / (1 - opa))]]),
              rgb=np.full((1, 3), 1.0), sh=None, T=np.eye(4), K=np.array([[f, 0, 30.0], [0, f, 30.0], [0, 0, 1]]),
              H=H, W=W)
    o = lo.render(sc, np.zeros(3), "fisheye", kc, mh=3.0)
    ys, xs = np.mgrid[0:H, 0:W]
    td = np.hypot(xs - 30.0, ys - 30.0) / f
    th = td.copy()
    k1 = float(np.float32(kc[0]))  # the coefficients as the kernels see them
    for _ in range(100):  # Newton on theta (1 + k1 theta^2) = theta_d
        th -= (th * (1 + k1 * th * th) - td) / (1 + 3 * k1 * th * th)
    rho3 = (pz * np.tan(th) / su) ** 2
    rho2 = 2 * ((xs - 30.0) ** 2 + (ys - 30.0) ** 2)
    rho = np.minimum(rho3, rho2)
    want = np.minimum(opa * np.exp(-0.5 * rho), 0.99)
    thmax = lo.lens_constants("fisheye", kc)[-1]
    want[(rho > 9.0) | (want < 1 / 255) | (td >= thmax * (1 + k1 * thmax ** 2))] = 0  # no ray beyond theta_max
    a = o.alpha[..., 0]
    wide = (th > np.radians(60)) & (want > 0)
    assert wide.sum() > 20
    np.testing.assert_allclose(a, want, rtol=1e-9, atol=1e-12)
    hit = a > 0
    np.testing.assert_allclose(o.depth[..., 0][hit] / a[hit], pz, rtol=1e-9)


# ---- gradients against central differences ---------------------------------------------------------------------------
@pytest.mark.parametrize("lens,kc", [("fisheye", FISHEYE), ("distortion", OPENCV)])
@pytest.mark.parametrize("case", list(CASES))
def test_gradients_match_central_differences(case, lens, kc):
    cfg = dict(CASES[case])
    bg = np.array(cfg.pop("bg", (0.0, 0.0, 0.0)))
    sc = _stack(**cfg)
    G = _upstream(sc)
    dirs = so.view_dirs(sc)
    o = lo.render(sc, bg, lens, kc, grads=G, dirs=dirs)
    assert o.M == sc["xyz"].shape[0]
    h = 1e-6
    names = ["xyz", "quaternion", "scale", "opacity", "rgb"] + (["sh"] if sc["sh"] is not None else [])
    for name in names:
        num = np.zeros_like(sc[name], dtype=float)
        for idx in np.ndindex(sc[name].shape):
            vals = []
            for sgn in (1, -1):
                s2 = dict(sc)
                s2[name] = sc[name].astype(float).copy()
                s2[name][idx] += sgn * h
                vals.append(so.loss(lo.render(s2, bg, lens, kc, dirs=dirs), G))
            num[idx] = (vals[0] - vals[1]) / (2 * h)
        scale = np.abs(num).max()
        assert scale > 0, name
        np.testing.assert_allclose(o.g[name], num, rtol=0, atol=2e-6 * scale + 1e-9, err_msg=f"{case}: {name}")
    assert (o.g["scale"][:, 2] == 0).all()


# ---- the binning bound -----------------------------------------------------------------------------------------------
_BOUND_SRC = r'''
#include "gsr_surfels_lens.cuh"
extern "C" int surfel_lens_box_host(int lens, const double* Mp, double r2, const double* K4, const float* kc,
                                    double* box) {
    return gsr::surfel::surfel_lens_box(lens, Mp, r2, K4[0], K4[1], K4[2], K4[3], kc, box[0], box[1], box[2], box[3]);
}
'''


@pytest.fixture(scope="module")
def bound_lib():
    nvcc = _tool("nvcc")
    d = Path(tempfile.mkdtemp(prefix="gsr_surfel_bound_"))
    (d / "bound.cu").write_text(_BOUND_SRC)
    subprocess.run([nvcc, "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-shared", f"-I{PKG / 'csrc'}",
                    str(d / "bound.cu"), "-o", str(d / "bound.so")], check=True, capture_output=True)
    lib = C.CDLL(str(d / "bound.so"))
    lib.surfel_lens_box_host.restype = C.c_int
    return lib


def _random_surfels(rng, n, K, grazing):
    out = []
    for _ in range(n):
        # directions across the whole field, some at and beyond the lens limits, and disks near the camera plane
        th = rng.uniform(0, np.radians(89))
        ph = rng.uniform(0, 2 * np.pi)
        dist = rng.choice([rng.uniform(0.3, 8.0), rng.uniform(0.05, 0.4)])
        p = dist * np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        w, x, y, z = q
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        if grazing:  # the plane nearly contains the ray to its centre
            v = p / np.linalg.norm(p)
            t1 = np.cross(v, rng.normal(size=3))
            t1 /= np.linalg.norm(t1)
            t2 = np.cross(t1, v) * np.cos(rng.uniform(0, 0.2)) + v * np.sin(rng.uniform(0, 0.2))
            R = np.column_stack([t1, t2 / np.linalg.norm(t2), np.cross(t1, t2 / np.linalg.norm(t2))])
        su, sv = np.exp(rng.uniform(-4, 0, 2)) * dist
        M = np.column_stack([su * R[:, 0], sv * R[:, 1], p])
        out.append(M.astype(np.float32).astype(np.float64))
    return out


@pytest.mark.parametrize("lens,kc", [("fisheye", FISHEYE), ("fisheye", STRONG_FISHEYE), ("distortion", OPENCV),
                                     ("distortion", BARREL)])
def test_binning_bound_contains_every_valid_point_of_the_disk(bound_lib, lens, kc):
    rng = np.random.default_rng(7)
    K = np.array([[300.0, 0, 320.0], [0, 310.0, 240.0], [0, 0, 1]])
    K4 = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    lim = _limit(lens, kc)
    kcf = np.append(np.asarray(kc, np.float32), np.float32(lim)).astype(np.float32)
    r, r2 = 3.0, 9.0
    t = np.linspace(0, 2 * np.pi, 720, endpoint=False)
    rad = np.concatenate([np.ones_like(t), 0.5 * np.ones_like(t)])
    tt = np.concatenate([t, t])
    checked = empty = 0
    for grazing in (False, True):
        for M in _random_surfels(rng, 1500, K, grazing):
            if not (M[2, 2] > 0 and r2 * (M[2, 0] ** 2 + M[2, 1] ** 2) < M[2, 2] ** 2):
                continue  # culled: the disk reaches behind the camera plane
            box = np.zeros(4)
            any_ = bound_lib.surfel_lens_box_host(C.c_int(lo.LENS_ID[lens]), M.ctypes.data_as(C.c_void_p),
                                                  C.c_double(r2), K4.ctypes.data_as(C.c_void_p),
                                                  kcf.ctypes.data_as(C.c_void_p), box.ctypes.data_as(C.c_void_p))
            ab = np.stack([r * rad * np.cos(tt), r * rad * np.sin(tt), np.ones_like(tt)], 0)
            X = (M @ ab).T
            d = X / np.linalg.norm(X, axis=1, keepdims=True)
            pix, ok = _project(lens, kc, lim, K, d)
            if not any_:
                assert not ok.any()
                empty += 1
                continue
            checked += int(ok.sum())
            inside = ((pix[ok, 0] >= box[0] - 1e-9 * (1 + abs(box[0]))) & (pix[ok, 0] <= box[1] + 1e-9 * (1 + abs(box[1])))
                      & (pix[ok, 1] >= box[2] - 1e-9 * (1 + abs(box[2])))
                      & (pix[ok, 1] <= box[3] + 1e-9 * (1 + abs(box[3]))))
            assert inside.all(), (M, box, pix[ok][~inside][:3])
    assert checked > 100000
    print(f"{lens} {kc}: {checked} boundary points inside their bounds, {empty} disks with no valid ray")


# ---- arguments -------------------------------------------------------------------------------------------------------
def test_lens_arguments_are_checked_before_any_launch():
    from gaussian_splatting_b200.surfels import rasterize_surfels

    g, cam, T, bg = _torch_scene()
    with pytest.raises(ValueError, match="either fisheye or distortion"):
        rasterize_surfels(g, T, cam, 0.3, 100.0, 10.0, 3.0, bg, fisheye=FISHEYE, distortion=OPENCV)
    with pytest.raises(ValueError, match="shape"):
        rasterize_surfels(g, T, cam, 0.3, 100.0, 10.0, 3.0, bg, fisheye=(0.1, 0.2))
    with pytest.raises(ValueError, match="finite"):
        rasterize_surfels(g, T, cam, 0.3, 100.0, 10.0, 3.0, bg, distortion=(np.nan, 0, 0, 0, 0))
    with pytest.raises(ValueError, match="no camera gradient"):
        rasterize_surfels(g, T, cam, 0.3, 100.0, 10.0, 3.0, bg,
                          fisheye=torch.tensor(FISHEYE, requires_grad=True))
    g64, cam64, T64, bg64 = _torch_scene(torch.float64)
    with pytest.raises(TypeError):
        rasterize_surfels(g64, T64, cam64, 0.3, 100.0, 10.0, 3.0, bg64, fisheye=FISHEYE)


# ---- the library -----------------------------------------------------------------------------------------------------
def test_c_abi_exports_exactly_the_declared_symbols():
    header = (ROOT / "include" / "gsr_surfels_lens.h").read_text()
    declared = set(re.findall(r"^(?:int|size_t) (gsr_\w+)\(", header, re.M))
    assert len(declared) == 6
    if not LENS_LIB.exists():
        pytest.skip("libgsr_surfels_lens.so is not built")
    nm = subprocess.run(["nm", "-D", "--defined-only", str(LENS_LIB)], capture_output=True, text=True).stdout
    assert set(re.findall(r"\bT (gsr_\w+)", nm)) == declared


def test_lens_kernels_are_sm90a_and_use_no_local_memory():
    elfs = _cuobjdump("--list-elf", lib=LENS_LIB)
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage", lib=LENS_LIB)))
    names = [k for k in usage if "k_surfel" in k]
    # forward and backward per SH degree and lens, uv.grad and rays per lens, tile forward / backward
    assert len(names) == 22, names
    for name in names:
        u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[name])}
        assert u["LOCAL"] == 0 and u["STACK"] == 0, (name, u)


def test_existing_kernels_keep_their_sass():
    """Every kernel of the eleven libraries that existed before the lens surfels keeps its instructions, the pinhole
    surfel kernels included, and no library gains a kernel."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_surfels_lens.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    libs = ("libgsr_b200.so", "libgsr_selective_adam.so", "libgsr_features.so", "libgsr_batch.so",
            "libgsr_fisheye.so", "libgsr_distortion.so", "libgsr_pose.so", "libgsr_calib.so", "libgsr_shutter.so",
            "libgsr_bilagrid.so", "libgsr_surfels.so")
    assert set(rec) - {"nvcc"} == set(libs)
    for lib in libs:
        if not (PKG / lib).exists():
            pytest.skip(f"{lib} is not built")
        now = {k: d for k, (d, n) in sass_digest.per_kernel(PKG / lib).items()}
        assert set(now) == set(rec[lib]), (lib, sorted(set(now) ^ set(rec[lib]))[:4])
        changed = sorted(k for k, d in rec[lib].items() if now[k] != d)
        assert not changed, (lib, changed)
