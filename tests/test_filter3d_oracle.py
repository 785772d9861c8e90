"""Mip-Splatting's 3-D filter (rasterize(..., filter3d=f), compute_filter3d, bake_filter3d): the CPU oracle's semantics
and gradients, known answers, the sampling pass, the argument errors and the new kernels in the built library.  No GPU
needed."""
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from gaussian_splatting_b200.filter3d import bake_filter3d
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera, Gaussians
from oracle import cpu_oracle as orc
from tests import antialiased_oracle as aao
from tests import depth_alpha_oracle as dao
from tests import filter3d_oracle as fo
from tests.scenes import np_scene
from tests.test_sass_evidence import LIB, _tool_output, sass_counts

PARAMS = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")


def live_filter(sc, seed=3, lo=0.3, hi=1.5):
    """A filter comparable to the gaussians' own world sizes (coef far from 1 on most of them), zero on every 9th."""
    rng = np.random.default_rng(seed)
    f = np.exp(np.asarray(sc["scale"], np.float64).mean(1)) * rng.uniform(lo, hi, len(sc["scale"]))
    f[::9] = 0.0
    return f.astype(sc["xyz"].dtype)


def _forward(sc, f, antialiased=False, **over):
    s = dict(sc, **over)
    return fo.rasterize(s["xyz"], s["quaternion"], s["scale"], s["opacity"], s["rgb"], s["sh"], s["T"], s["K"], s["H"],
                        s["W"], f, antialiased=antialiased, mh_dist=3.0,
                        background=np.full(3, 0.5, s["xyz"].dtype))


def _upstream(H, W, seed=1):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((H, W, 3)) / (3 * H * W), rng.standard_normal((H, W)) / (H * W),
            rng.standard_normal((H, W)) / (H * W))


# fp64 finite differences ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("antialiased", [False, True], ids=["plain", "antialiased"])
@pytest.mark.parametrize("sh_degree", [0, 3])
@pytest.mark.parametrize("maps", [False, True], ids=["image", "image+depth+alpha"])
def test_fp64_filter3d_backward_matches_finite_differences(sh_degree, maps, antialiased):
    """<G,image> (+ <Gd,depth> + <Ga,alpha>) against central differences of the filtered fp64 forward, every
    parameter.  The filter is live: coef is below 0.9 on most gaussians.  With SH, xyz is checked on the depth and alpha
    terms alone (no gradient goes to xyz through the view direction)."""
    sc = np_scene(128, "tiny", sh_degree=sh_degree, dtype=np.float64, sigma_px=(0.6, 1.2, 0.15, 8.0))
    f = live_filter(sc)
    G, Gd, Ga = _upstream(64, 64)
    if not maps:
        Gd, Ga = np.zeros_like(Gd), np.zeros_like(Ga)
    rng = np.random.default_rng(2)
    o = _forward(sc, f, antialiased)
    assert o.keep.sum() > 64 and len(o.sorted_idx) > 200 and (o.alpha > 0.3).any()
    assert (o.coef < 0.9).mean() > 0.5 and (o.coef == 1).sum() >= 5
    d = fo.rasterize_backward(o, G, Gd, Ga)

    def check(names, G, Gd, Ga):
        dd = fo.rasterize_backward(o, G, Gd, Ga)

        def loss(**over):
            p = _forward(sc, f, antialiased, **over)
            return float((p.image * G).sum() + (p.depth * Gd).sum() + (p.alpha * Ga).sum())

        vis = np.flatnonzero(o.keep)
        h = 1e-6
        for name in names:
            grad, base = getattr(dd, name), sc[name]
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

    assert np.isfinite(d.scale).all()
    if sh_degree:
        check(["quaternion", "scale", "opacity", "rgb", "sh"], G, Gd, Ga)
        if maps:
            check(["xyz"], np.zeros_like(G), Gd, Ga)
    else:
        check(["xyz", "quaternion", "scale", "opacity", "rgb"], G, Gd, Ga)


# baked parameters -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("antialiased", [False, True], ids=["plain", "antialiased"])
def test_fp64_baked_parameters_render_the_same_and_chain_the_same_gradients(antialiased):
    """bake_filter3d folds the filter into scale and opacity: the plain fp64 render of the baked parameters equals the
    filtered render to 1e-12, and the plain backward chained through bake_filter3d (torch autograd) equals the
    filtered backward."""
    sc = np_scene(128, "tiny", sh_degree=3, dtype=np.float64, sigma_px=(0.6, 1.2, 0.15, 8.0))
    f = live_filter(sc, seed=5)
    G, Gd, Ga = _upstream(64, 64, seed=4)
    o = _forward(sc, f, antialiased)
    t = {k: torch.tensor(sc[k], requires_grad=True) for k in PARAMS}
    baked = bake_filter3d(Gaussians(t["xyz"], t["rgb"], t["opacity"], t["scale"], t["quaternion"], t["sh"]),
                          torch.tensor(f))
    bs = dict(sc, scale=baked.scale.detach().numpy(), opacity=baked.opacity.detach().numpy())
    plain = aao if antialiased else dao
    ob = plain.rasterize(bs["xyz"], bs["quaternion"], bs["scale"], bs["opacity"], bs["rgb"], bs["sh"], bs["T"], bs["K"],
                         bs["H"], bs["W"], mh_dist=3.0, background=np.full(3, 0.5))
    assert np.array_equal(ob.keep, o.keep) and np.array_equal(ob.sorted_idx, o.sorted_idx)
    for k in ("image", "depth", "alpha"):
        assert np.abs(getattr(ob, k) - getattr(o, k)).max() <= 1e-12, k
    d = fo.rasterize_backward(o, G, Gd, Ga)
    db = plain.rasterize_backward(ob, G, Gd, Ga)
    torch.autograd.backward([baked.scale, baked.opacity], [torch.tensor(db.scale), torch.tensor(db.opacity)])
    chained = dict(xyz=db.xyz, quaternion=db.quaternion, rgb=db.rgb, sh=db.sh, scale=t["scale"].grad.numpy(),
                   opacity=t["opacity"].grad.numpy())
    for k in PARAMS:
        ref = getattr(d, k)
        assert np.abs(chained[k] - ref).max() <= 1e-9 * np.abs(ref).max(), k


# known answers ------------------------------------------------------------------------------------------------------
def _one_camera(n, dtype):
    return (np.tile(np.array([0.1, -0.2, 3.0], dtype), (n, 1)), np.eye(4, dtype=dtype),
            np.array([[200, 0, 32], [0, 200, 32], [0, 0, 1]], dtype), np.ones(n, np.uint8))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_isotropic_coef_and_mass_conservation(dtype):
    """Isotropic gaussians: coef = (e^2 / (e^2 + f^2))^(3/2).  Any gaussian: coef sqrt(prod(v + F)) = sqrt(prod v),
    the 3-D mass sigma(o) sqrt(det Sigma) is kept."""
    e = np.geomspace(1e-3, 10.0, 9)
    f = np.geomspace(1e-3, 10.0, 7)
    E, Fm = (a.reshape(-1) for a in np.meshgrid(e, f))
    n = len(E)
    xyz_cam, T, K, vis = _one_camera(n, dtype)
    q = np.tile(np.array([0.9, 0.1, -0.3, 0.2], dtype), (n, 1))
    _, coef, _ = fo.filtered_conic(xyz_cam, q, np.log(np.stack([E, E, E], 1)).astype(dtype), Fm.astype(dtype), T, K, vis)
    want = (E ** 2 / (E ** 2 + Fm ** 2)) ** 1.5
    np.testing.assert_allclose(coef, want, rtol=2e-6 if dtype == np.float32 else 1e-13)
    rng = np.random.default_rng(0)
    s = rng.uniform(-4, 1, (n, 3))
    _, coef, t = fo.filtered_conic(xyz_cam, q, s.astype(dtype), Fm.astype(dtype), T, K, vis)
    v = np.exp(2 * s.astype(dtype).astype(np.float64))
    np.testing.assert_allclose(coef * np.sqrt(np.prod(v + Fm[:, None] ** 2, 1)), np.sqrt(np.prod(v, 1)),
                               rtol=4e-6 if dtype == np.float32 else 1e-13)


def test_zero_filter_reproduces_the_default_records_bit_for_bit():
    """f == 0: v' = v + 0 and coef = 1 exactly, so the conic, opacity and the whole fp32 render are the default ones,
    bit for bit (in the anti-aliased mode too)."""
    sc = np_scene(2000, "tiny", sh_degree=3, sigma_px=(0.8, 0.8, 0.15, 8.0))
    zero = np.zeros(2000, np.float32)
    o = _forward(sc, zero)
    ref = dao.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], sc["K"],
                        sc["H"], sc["W"], mh_dist=3.0, background=np.full(3, 0.5, np.float32))
    assert (o.coef == 1).all()
    for k in ("conic", "opacity", "image", "depth", "alpha", "wlast", "n", "sorted_idx"):
        assert np.array_equal(getattr(o, k), getattr(ref, k)), k
    oa = _forward(sc, zero, antialiased=True)
    ra = aao.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], sc["K"],
                       sc["H"], sc["W"], mh_dist=3.0, background=np.full(3, 0.5, np.float32))
    for k in ("conic", "opacity", "image", "depth", "alpha"):
        assert np.array_equal(getattr(oa, k), getattr(ra, k)), k


def test_underflowing_scale_gives_zero_coef_and_finite_zero_gradients():
    """exp(-60)^2 underflows to 0 in fp32: t = 0, coef = 0, the splat never contributes, and its gradients come out
    exactly zero and finite (1 - t = F / v' has no 0/0)."""
    sc = np_scene(2000, "tiny", sh_degree=3, sigma_px=(0.8, 0.8, 0.15, 8.0))
    deg = np.arange(0, 2000, 7)
    sc["scale"][deg] = -60.0
    f = live_filter(sc)
    f[deg] = np.float32(0.01)
    for aa in (False, True):
        o = _forward(sc, f, antialiased=aa)
        rows = np.flatnonzero(o.keep).searchsorted(deg[o.keep[deg]])
        assert len(rows) > 100 and (o.coef[rows] == 0).all() and (o.opacity[rows] == 0).all()
        G, Gd, Ga = _upstream(sc["H"], sc["W"])
        d = fo.rasterize_backward(o, G, Gd, Ga)
        for k in PARAMS:
            gk = getattr(d, k)
            assert np.isfinite(gk).all(), k
            assert not gk[deg].any(), k
            assert np.abs(np.delete(gk, deg, axis=0)).max() > 0, k


# the sampling pass ------------------------------------------------------------------------------------------------
K100 = np.array([[100.0, 0, 0], [0, 100.0, 0], [0, 0, 1]], np.float32)


def test_sampling_near_plane_is_strict_and_margins_are_inclusive():
    """Identity pose, f = 100, c = 0, W = H = 100, margin 0.25, near 0.5: every quantity below is exact in fp32.  p_z ==
    near is not seen, the next float is; u or v exactly on -m W or (1 + m) W is seen, one ulp beyond is not."""
    nx = lambda a, b: np.nextafter(np.float32(a), np.float32(b))  # noqa: E731
    pts = [  # (x, y, z, seen)
        (0.1, 0.1, 0.5, False), (0.1, 0.1, nx(0.5, 1), True),
        (-0.25, 0.1, 1.0, True), (nx(-0.25, -1), 0.1, 1.0, False),
        (1.25, 0.1, 1.0, True), (nx(1.25, 2), 0.1, 1.0, False),
        (0.1, -0.25, 1.0, True), (0.1, nx(-0.25, -1), 1.0, False),
        (0.1, 1.25, 1.0, True), (0.1, nx(1.25, 2), 1.0, False),
    ]
    xyz = np.array([p[:3] for p in pts], np.float32)
    f = fo.sample(xyz, [np.eye(4)], [K100], [100], [100], near=0.5, margin=0.25, variance=0.25)
    seen = np.array([p[3] for p in pts])
    want = np.where(seen, 0.5 * xyz[:, 2].astype(np.float64) / 100, 0.5 * 1.0 / 100)  # unseen: the largest seen
    np.testing.assert_allclose(f, want, rtol=1e-7)
    # unseen ones take the largest r of the seen ones (here z = 1): distinguishable by moving the seen maximum
    xyz2 = np.concatenate([xyz, [[0.0, 0.0, 4.0]]]).astype(np.float32)
    f2 = fo.sample(xyz2, [np.eye(4)], [K100], [100], [100], near=0.5, margin=0.25, variance=0.25)
    assert np.array_equal(f2[:-1][~seen], np.full((~seen).sum(), np.float32(0.5) * np.float32(4.0 / 100)))


def test_sampling_takes_the_finest_rate_over_cameras_per_camera():
    """r_i = min over the cameras that see i of p_z / max(fx, fy): mixed focal lengths and fx != fy.  Camera 2 (f = 400)
    sees the points at depth 4 (r = 0.01), camera 1 (f = 50 / 80) at depth 2 (r = 0.025); a point camera 2 cannot see
    keeps camera 1's rate."""
    T1 = np.eye(4)
    T2 = np.eye(4)
    T2[2, 3] = 2.0                                          # camera 2 stands 2 units behind camera 1
    K1 = np.array([[50.0, 0, 32], [0, 80.0, 32], [0, 0, 1]])
    K2 = np.array([[400.0, 0, 32], [0, 300.0, 32], [0, 0, 1]])
    xyz = np.array([[0.0, 0.0, 2.0], [0.9, 0.0, 2.0]], np.float32)   # the second is outside camera 2's image
    f = fo.sample(xyz, [T1, T2], [K1, K2], [64, 64], [64, 64], variance=1.0)
    np.testing.assert_allclose(f, [4.0 / 400, 2.0 / 80], rtol=1e-7)


def test_sampling_all_unseen_gives_zeros():
    xyz = np.array([[0, 0, -1.0], [0, 0, 0.1], [100.0, 0, 1]], np.float32)
    assert not fo.sample(xyz, [np.eye(4)], [K100], [100], [100]).any()


def test_sampling_matches_mip_splattings_loop_with_a_shared_focal_length():
    """With one focal length for every camera (and cx = W/2) the per-camera ratio equals Mip-Splatting's separate
    min-depth / max-focal computation."""
    rng = np.random.default_rng(3)
    xyz = (rng.standard_normal((20_000, 3)) * [2.0, 1.5, 2.0]).astype(np.float32)
    Ts, Ks = [], []
    for c in range(12):
        a = 2 * np.pi * c / 12
        R = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]])
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, [0, 0, 4.0]
        Ts.append(T.astype(np.float32))
        Ks.append(np.array([[300.0, 0, 160], [0, 300.0, 120], [0, 0, 1]], np.float32))
    xyz[:50] = [0, 30.0, 0]                                   # above every camera: unseen
    f = fo.sample(xyz, Ts, Ks, [320] * 12, [240] * 12)
    ref = fo.mip_splatting_loop(xyz, Ts, Ks, [320] * 12, [240] * 12)
    assert (f[:50] == f.max()).all()
    np.testing.assert_allclose(f, ref, rtol=2e-6)


# argument errors --------------------------------------------------------------------------------------------------
def test_argument_errors():
    sc = np_scene(50, "tiny", sh_degree=1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    g = Gaussians(t(sc["xyz"]), t(sc["rgb"]), t(sc["opacity"]), t(sc["scale"]), t(sc["quaternion"]), t(sc["sh"]))
    cam, bg, T = Camera(64, 64, t(sc["K"])), torch.full((3,), 0.5), t(sc["T"])
    f = torch.zeros(50)
    with pytest.raises(ValueError):   # per-pixel SH
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, False, bg, filter3d=f)
    with pytest.raises(ValueError):   # a stale filter
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, filter3d=torch.zeros(49))
    with pytest.raises(ValueError):
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, filter3d=torch.zeros(50, 3))
    with pytest.raises(ValueError):   # the filter is a constant
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, filter3d=torch.zeros(50, requires_grad=True))
    g64 = Gaussians(*(x.double() for x in (g.xyz, g.rgb, g.opacity, g.scale, g.quaternion)), None)
    with pytest.raises(TypeError):
        rasterize(g64, T.double(), Camera(64, 64, t(sc["K"]).double()), 0.3, 500.0, 100, 3.0, True, bg.double(),
                  filter3d=f.double())


# the kernels in the built library ---------------------------------------------------------------------------------
def _usage():
    usage = {}
    for name, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _tool_output("--dump-resource-usage")):
        usage[name] = {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
    return usage


F3D_KERNELS = {"k_preprocess_fwd_f3d": "k_preprocess_fwd", "k_preprocess_fwd_aa_f3d": "k_preprocess_fwd_aa",
               "k_preprocess_bwd_f3d": "k_preprocess_bwd", "k_preprocess_bwd_depth_f3d": "k_preprocess_bwd_depth",
               "k_preprocess_bwd_aa_f3d": "k_preprocess_bwd_aa",
               "k_preprocess_bwd_depth_aa_f3d": "k_preprocess_bwd_depth_aa"}


def test_filter3d_kernels_stage_through_tma_and_use_no_local_memory():
    """Every instantiation of the new per-gaussian kernels is in the library and keeps the TMA bulk copies (UBLKCP) of
    its unfiltered counterpart.  The backward kernels keep nothing in local memory (no STL / LDL); the forward kernels
    keep the default forward's 32-byte frame (the pose inversion's vectors) and add no local-memory access to it
    (DESIGN.md 3.13).  The sampling kernels use no local memory."""
    counts, usage = sass_counts(), _usage()
    for new, old in F3D_KERNELS.items():
        for args in ("ILi1ELb0E", "ILi4ELb1E", "ILi9ELb1E", "ILi16ELb1E"):
            frag_new, frag_old = f"{len(new)}{new}{args}", f"{len(old)}{old}{args}"
            c_new = next((c for n, c in counts.items() if frag_new in n), None)
            c_old = next(c for n, c in counts.items() if frag_old in n)
            assert c_new is not None, frag_new
            assert c_new["UBLKCP"] == c_old["UBLKCP"] >= 1, (frag_new, c_new["UBLKCP"], c_old["UBLKCP"])
            local = (c_new["STL"], c_new["LDL"])
            assert local == ((0, 0) if "bwd" in new else (c_old["STL"], c_old["LDL"])), (frag_new, local)
            u_new = next(v for k, v in usage.items() if frag_new in k)
            u_old = next(v for k, v in usage.items() if frag_old in k)
            assert u_new["LOCAL"] == 0 and u_new["STACK"] <= u_old["STACK"], (frag_new, u_new, u_old)
    for k in ("14k_filter3d_min", "15k_filter3d_fill"):
        c = next(c for n, c in counts.items() if k in n)
        u = next(v for n, v in usage.items() if k in n)
        assert c["STL"] == c["LDL"] == 0 and u["LOCAL"] == 0 and u["STACK"] == 0, (k, u)


def test_kernels_that_existed_before_the_filter_compile_to_the_same_sass():
    """Per-kernel digests of the SASS instruction listing (encodings included; tools/dev/sass_digest.py) of every
    kernel the library had before the 3-D filter was added, against the digests recorded then.  Only meaningful with
    the nvcc release that recorded them (skipped otherwise); a change that means to alter one of these kernels records
    the digests again (sass_digest.py --json)."""
    rec = json.loads((Path(__file__).parent / "golden" / "sass_digests_before_filter3d.json").read_text())
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(exe).exists() or not LIB.exists():
        pytest.skip("nvcc or the built library is missing")
    ver = subprocess.run([exe, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if ver != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {ver}")
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", LIB.parents[1] / "tools" / "dev" / "sass_digest.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    now = mod.per_kernel(LIB)
    missing = [k for k in rec["kernels"] if k not in now]
    changed = [k for k, d in rec["kernels"].items() if k in now and now[k][0] != d]
    assert not missing and not changed, (missing, changed)
