"""2-D Gaussian surfels without a GPU: the fp64 oracle (tests/surfels_oracle.c) on known answers and against central
differences, depth_normals, argument errors, and the library (symbols, resources, untouched SASS of every other
library)."""
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from gaussian_splatting_b200.structs import Camera, Gaussians
from tests import surfels_oracle as so

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "gaussian_splatting_b200"
SURFEL_LIB = PKG / "libgsr_surfels.so"
SH0 = so.SH_C["c0"]


def _single(quat, scale, xyz=(0.0, 0.0, 2.0), opacity=0.5, H=31, W=41, K=((60.0, 0, 20.0), (0, 50.0, 15.0), (0, 0, 1))):
    logit = float(np.log(opacity / (1 - opacity)))
    return dict(xyz=np.array([xyz], float), quaternion=np.array([quat], float), scale=np.array([scale], float),
                opacity=np.array([[logit]]), rgb=np.full((1, 3), 0.5 / SH0), sh=None, T=np.eye(4), K=np.array(K),
                H=H, W=W)


# ---- known answers ---------------------------------------------------------------------------------------------------
def test_fronto_parallel_surfel_has_its_depth_normal_and_ellipse():
    su, sv, pz = 0.08, 0.05, 2.0
    sc = _single((1, 0, 0, 0), (np.log(su), np.log(sv), 0.3), xyz=(0.0, 0.0, pz))
    o = so.render(sc, np.zeros(3))
    K = sc["K"]
    ys, xs = np.mgrid[0:sc["H"], 0:sc["W"]]
    dx, dy = xs - K[0, 2], ys - K[1, 2]
    rho3 = dx ** 2 / (K[0, 0] * su / pz) ** 2 + dy ** 2 / (K[1, 1] * sv / pz) ** 2
    rho2 = 2 * (dx ** 2 + dy ** 2)
    want = 0.5 * np.exp(-0.5 * rho3)
    inside = (rho3 <= rho2) & (rho3 <= 9.0) & (want >= 1 / 255)
    a = o.alpha[..., 0]
    assert inside.sum() > 20
    np.testing.assert_allclose(a[inside], want[inside], rtol=1e-12)
    assert (a[a > 0] <= 0.5).all()
    hit = a > 0
    np.testing.assert_allclose(o.depth[..., 0][hit] / a[hit], pz, rtol=1e-12)
    np.testing.assert_allclose(o.normal[hit] / a[hit, None], np.tile([0.0, 0.0, -1.0], (hit.sum(), 1)), atol=1e-12)
    np.testing.assert_allclose(o.image[hit], 0.5 * a[hit, None] * np.ones(3), rtol=1e-12)


def test_edge_on_surfel_renders_through_the_fallback_disk_only():
    # rotation by 90 degrees about y: the surfel's plane x = 0 contains the camera centre
    q = (np.cos(np.pi / 4), 0.0, np.sin(np.pi / 4), 0.0)
    sc = _single(q, (np.log(0.01), np.log(0.2), 0.0), xyz=(0.0, 0.0, 2.0), opacity=0.8)
    o = so.render(sc, np.zeros(3))
    assert o.visible[0] == 1
    K = sc["K"]
    ys, xs = np.mgrid[0:sc["H"], 0:sc["W"]]
    dx, dy = xs - K[0, 2], ys - K[1, 2]
    rho2 = 2 * (dx ** 2 + dy ** 2)
    want = np.where(rho2 <= 9.0, 0.8 * np.exp(-0.5 * rho2), 0.0)
    want[want < 1 / 255] = 0.0
    # the column x = c_x images the plane itself (rays inside it): degenerate, only required to stay finite
    off = dx != 0
    np.testing.assert_allclose(o.alpha[..., 0][off], want[off], rtol=1e-12, atol=0)
    assert np.isfinite(o.alpha).all() and np.isfinite(o.depth).all()
    hit = off & (want > 0)
    np.testing.assert_allclose(o.depth[..., 0][hit] / want[hit], 2.0, rtol=1e-12)


@pytest.mark.parametrize("quat", [(1.0, 0.0, 0.0, 0.0), (0.0, 1.0, 0.0, 0.0)])
def test_normal_faces_the_camera(quat):
    """R = I has n = (0,0,1), facing away: flipped; R = rotation by pi about x has n = (0,0,-1) already."""
    sc = _single(quat, (np.log(0.08), np.log(0.05), 0.0))
    o = so.render(sc, np.zeros(3))
    hit = o.alpha[..., 0] > 0
    np.testing.assert_allclose(o.normal[hit] / o.alpha[hit], np.tile([0.0, 0.0, -1.0], (hit.sum(), 1)), atol=1e-12)


def _stack(n=4, opacity=0.7, sh_degree=0, H=23, W=29, seed=0, offsets=True):
    """Tilted surfels stacked in depth in front of a small camera (overlapping footprints)."""
    rng = np.random.default_rng(seed)
    K = np.array([[40.0, 0, 14.3], [0, 42.0, 11.2], [0, 0, 1]])
    z = 1.5 + 0.35 * np.arange(n)
    off = rng.uniform(-0.08, 0.08, (n, 2)) if offsets else np.zeros((n, 2))
    xyz = np.column_stack([off * z[:, None], z])
    q = np.column_stack([np.ones(n), rng.uniform(-0.35, 0.35, (n, 3))])
    scale = np.column_stack([np.log(rng.uniform(0.06, 0.12, (n, 2)) * z[:, None]), rng.uniform(-2, 0, n)])
    logit = np.full((n, 1), np.log(opacity / (1 - opacity))) + rng.uniform(-0.2, 0.2, (n, 1))
    rgb = rng.uniform(0, 2, (n, 3))
    sh = rng.normal(0, 0.3, (n, 3, (sh_degree + 1) ** 2 - 1)) if sh_degree else None
    c, s = np.cos(0.1), np.sin(0.1)
    T = np.eye(4)
    T[:3, :3] = [[c, 0, s], [0, 1, 0], [-s, 0, c]]
    T[:3, 3] = [0.05, -0.03, 0.1]
    xyz = (xyz - T[:3, 3]) @ T[:3, :3]  # world positions that land at the camera-frame positions above
    return dict(xyz=xyz, quaternion=q, scale=scale, opacity=logit, rgb=rgb, sh=sh, T=T, K=K, H=H, W=W)


def test_distortion_is_the_brute_force_double_sum():
    sc = _stack(n=5)
    o = so.render(sc, np.zeros(3))
    # replay every pixel's blend from the oracle's own per-surfel alphas: render each surfel alone (its alpha map) and
    # composite in depth order
    z_order = np.argsort([(sc["T"][:3, :3] @ x + sc["T"][:3, 3])[2] for x in sc["xyz"]])
    alphas, depths = [], []
    for i in z_order:
        one = {k: (v[i:i + 1] if isinstance(v, np.ndarray) and v.shape[:1] == (5,) else v) for k, v in sc.items()}
        oi = so.render(one, np.zeros(3))
        alphas.append(oi.alpha[..., 0])
        depths.append(np.divide(oi.depth[..., 0], oi.alpha[..., 0], out=np.zeros_like(oi.depth[..., 0]),
                                where=oi.alpha[..., 0] > 0))
    n, f = 0.3, 500.0
    T = np.ones((sc["H"], sc["W"]))
    w, m = [], []
    for a, z in zip(alphas, depths):
        w.append(T * a)
        m.append(np.where(a > 0, f / (f - n) * (1 - n / np.where(a > 0, z, 1.0)), 0.0))
        T = T * (1 - a)
    D = sum(w[i] * w[j] * (m[i] - m[j]) ** 2 for i in range(5) for j in range(i))
    assert D.max() > 1e-6
    np.testing.assert_allclose(o.dist[..., 0], D, rtol=1e-9, atol=1e-15)
    np.testing.assert_allclose(o.alpha[..., 0], sum(w), rtol=1e-12, atol=1e-15)


# ---- gradients against central differences ---------------------------------------------------------------------------
def _upstream(sc, seed=3):
    rng = np.random.default_rng(seed)
    H, W = sc["H"], sc["W"]
    return dict(image=rng.normal(size=(H, W, 3)), depth=rng.normal(size=(H, W, 1)), alpha=rng.normal(size=(H, W, 1)),
                normal=rng.normal(size=(H, W, 3)), dist=rng.normal(size=(H, W, 1)) * 50)


CASES = {"sh0": dict(sh_degree=0), "sh3": dict(sh_degree=3), "background": dict(sh_degree=0, bg=(0.2, 0.5, 0.9)),
         "saturated": dict(sh_degree=0, n=7, opacity=0.97, offsets=False, bg=(0.3, 0.3, 0.3))}


@pytest.mark.parametrize("case", list(CASES))
def test_gradients_match_central_differences(case):
    cfg = dict(CASES[case])
    bg = np.array(cfg.pop("bg", (0.0, 0.0, 0.0)))
    sc = _stack(**cfg)
    G = _upstream(sc)
    dirs = so.view_dirs(sc)  # the colour's view direction is held constant, as in the kernels
    o = so.render(sc, bg, grads=G, dirs=dirs)
    assert o.M == sc["xyz"].shape[0]
    if case == "saturated":
        assert (o.alpha > 0.9999).sum() > 10
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
                vals.append(so.loss(so.render(s2, bg, dirs=dirs), G))
            num[idx] = (vals[0] - vals[1]) / (2 * h)
        ana = o.g[name]
        scale = np.abs(num).max()
        assert scale > 0, name
        np.testing.assert_allclose(ana, num, rtol=0, atol=2e-6 * scale + 1e-9, err_msg=f"{case}: {name}")
    assert (o.g["scale"][:, 2] == 0).all()


def test_uv_grad_sums_to_the_principal_point_gradient():
    sc = _stack(n=5, seed=2)
    G = _upstream(sc, seed=5)
    o = so.render(sc, np.full(3, 0.4), grads=G)
    h = 1e-6
    for k, (r, c) in enumerate(((0, 2), (1, 2))):
        vals = []
        for sgn in (1, -1):
            s2 = dict(sc)
            s2["K"] = sc["K"].copy()
            s2["K"][r, c] += sgn * h
            vals.append(so.loss(so.render(s2, np.full(3, 0.4)), G))
        d = (vals[0] - vals[1]) / (2 * h)
        np.testing.assert_allclose(o.uv_grad[:, k].sum(), d, rtol=1e-6, atol=1e-9)


# ---- depth_normals ---------------------------------------------------------------------------------------------------
def test_depth_normals_recover_a_tilted_plane():
    from gaussian_splatting_b200.surfels import depth_normals

    H, W = 30, 40
    K = torch.tensor([[50.0, 0, 19.5], [0, 55.0, 14.5], [0, 0, 1]], dtype=torch.float64)
    n = torch.tensor([0.3, -0.4, -1.0], dtype=torch.float64)
    n = n / n.norm()
    d = -3.0  # plane n . X = d, in front of the camera
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    rays = torch.stack((xs, ys, torch.ones_like(xs)), -1) @ torch.linalg.inv(K).T
    z = d / (rays @ n)
    alpha = torch.full((H, W, 1), 0.8, dtype=torch.float64)
    out = depth_normals((z * 0.8)[..., None], alpha, Camera(W, H, K))
    assert (out[0] == 0).all() and (out[-1] == 0).all() and (out[:, 0] == 0).all() and (out[:, -1] == 0).all()
    facing = n if float(n[2]) < 0 else -n
    torch.testing.assert_close(out[1:-1, 1:-1], facing.expand(H - 2, W - 2, 3), atol=1e-9, rtol=0)


# ---- arguments -------------------------------------------------------------------------------------------------------
def _torch_scene(dtype=torch.float32):
    n = 4
    g = Gaussians(torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 1, dtype=dtype),
                  torch.zeros(n, 3, dtype=dtype), torch.tensor([[1.0, 0, 0, 0]] * n, dtype=dtype))
    return g, Camera(8, 8, torch.eye(3, dtype=dtype)), torch.eye(4, dtype=dtype), torch.zeros(3, dtype=dtype)


def test_fp64_inputs_raise_type_error():
    from gaussian_splatting_b200.surfels import rasterize_surfels

    g, cam, T, bg = _torch_scene(torch.float64)
    with pytest.raises(TypeError):
        rasterize_surfels(g, T, cam, 0.3, 100.0, 10.0, 3.0, bg)


@pytest.mark.parametrize("which", ["pose", "K"])
def test_camera_that_requires_grad_raises_value_error(which):
    from gaussian_splatting_b200.surfels import rasterize_surfels

    g, cam, T, bg = _torch_scene()
    if which == "pose":
        T.requires_grad_(True)
    else:
        cam.K.requires_grad_(True)
    with pytest.raises(ValueError, match="no camera gradient"):
        rasterize_surfels(g, T, cam, 0.3, 100.0, 10.0, 3.0, bg)


# ---- the library -----------------------------------------------------------------------------------------------------
def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists():
        pytest.skip(f"{name} is not available")
    return exe


def _cuobjdump(*args, lib=SURFEL_LIB):
    if not lib.exists():
        pytest.skip("the built library is missing")
    return subprocess.run([_tool("cuobjdump"), *args, str(lib)], check=True, capture_output=True, text=True).stdout


def test_c_abi_exports_exactly_the_declared_symbols():
    header = (ROOT / "include" / "gsr_surfels.h").read_text()
    declared = set(re.findall(r"^(?:int|size_t) (gsr_\w+)\(", header, re.M))
    assert len(declared) == 6
    if not SURFEL_LIB.exists():
        pytest.skip("libgsr_surfels.so is not built")
    nm = subprocess.run(["nm", "-D", "--defined-only", str(SURFEL_LIB)], capture_output=True, text=True).stdout
    assert set(re.findall(r"\bT (gsr_\w+)", nm)) == declared


def test_surfel_kernels_are_sm90a_and_use_no_local_memory():
    elfs = _cuobjdump("--list-elf")
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage")))
    names = [k for k in usage if "k_surfel" in k]
    assert len(names) == 11, names  # forward and backward per SH degree, tile forward / backward, uv.grad
    for name in names:
        u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[name])}
        assert u["LOCAL"] == 0 and u["STACK"] == 0, (name, u)


def test_existing_kernels_keep_their_sass():
    """Every kernel of the ten libraries that existed before the surfels keeps its instructions, and no library gains
    a kernel: the surfel kernels are libgsr_surfels.so's."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_surfels.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    libs = ("libgsr_b200.so", "libgsr_selective_adam.so", "libgsr_features.so", "libgsr_batch.so",
            "libgsr_fisheye.so", "libgsr_distortion.so", "libgsr_pose.so", "libgsr_calib.so", "libgsr_shutter.so",
            "libgsr_bilagrid.so")
    assert set(rec) - {"nvcc"} == set(libs)
    for lib in libs:
        if not (PKG / lib).exists():
            pytest.skip(f"{lib} is not built")
        now = {k: d for k, (d, n) in sass_digest.per_kernel(PKG / lib).items()}
        assert set(now) == set(rec[lib]), (lib, sorted(set(now) ^ set(rec[lib]))[:4])
        changed = sorted(k for k, d in rec[lib].items() if now[k] != d)
        assert not changed, (lib, changed)
