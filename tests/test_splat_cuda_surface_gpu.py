"""The drop-in `splat_cuda` operator surface, operator by operator — needs an H100.

  * render_depth_cuda on hand-built tile lists against the depth-walk oracle (tests/depth_oracle.py), at thresholds
    chosen where an fp32-FMA accumulation and the reference's double-precision weight report different surfaces;
  * gaussian_splatting_b200.depth.render_depth against the reference's own render_depth on the compiled reference
    (oracle/_ref), bit for bit, on large, ragged, deep and far scenes;
  * each per-Gaussian backward kernel, row by row, against torch fp64 autograd of a plain restatement of the
    operator's forward (nothing from gsr_math*.cuh or oracle/cpu_oracle.py), in fp32 and fp64;
  * each per-Gaussian forward kernel and the tile binning, bit for bit against the compiled reference, on the same
    edge inputs (N around the 256-thread blocks, z from 1e-3 to 1e3, z <= 0, quaternion norms 1e-3 .. 1e3 of both
    signs, log-scales -8 .. 4, a general pose).
"""
import math
import sys

import numpy as np
import pytest
import torch

import gaussian_splatting_b200 as gsb
from gaussian_splatting_b200 import synth
from gaussian_splatting_b200.depth import render_depth
from gaussian_splatting_b200.structs import Camera, Gaussians
from oracle import ref_loader
from tests import depth_oracle as dor
from tests import gradrows, scenes

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ref_loader.reference_available(),
                               reason="oracle/_ref (the compiled reference) not present")
F32 = np.float32


def dev():
    return torch.device("cuda:0")


def to_t(a, dtype=None):
    x = torch.from_numpy(np.ascontiguousarray(a)).to(dev())
    return x if dtype is None else x.to(dtype)


def assert_bits_equal(a, b, what):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    b = b.detach().cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    ia = a.view(np.uint8).reshape(a.size, -1) if a.size else a
    ib = b.view(np.uint8).reshape(b.size, -1) if b.size else b
    bad = int((ia != ib).any(axis=-1).sum()) if a.size else 0
    assert bad == 0, f"{what}: {bad}/{a.size} values differ bitwise"


def ref_ext():
    return ref_loader.load_reference()[0]


# ------------------------------------------------------------------------------------------------
# 3a. render_depth_cuda on hand-built tile lists, against the depth-walk oracle
# ------------------------------------------------------------------------------------------------
def unit_colour():
    """The float r for which the renderer's colour SH0 * r rounds to exactly 1.0f."""
    sh0 = F32(scenes.SH0)
    r = F32(1.0 / scenes.SH0)
    for step in (0, 1, -1, 2, -2, 3, -3):
        c = F32(r + step * np.spacing(r))
        if sh0 * c == F32(1.0):
            return c
    raise AssertionError("no float r with SH0 * r == 1")


def pythagorean_positions(n):
    """n camera-frame positions with integer coordinates and distinct integer range: every rounding order of
    sqrt(x^2 + y^2 + z^2) gives the same float, and the range differs from z."""
    out, seen = [], set()
    for c in range(2, 60):
        for b in range(1, c + 1):
            for a in range(1, b + 1):
                d = math.isqrt(a * a + b * b + c * c)
                if d * d == a * a + b * b + c * c and d not in seen:
                    seen.add(d)
                    out.append((a, b, c))
    assert len(out) >= n
    return np.array(out[:n], F32)


def test_render_depth_weight_is_rounded_like_the_reference():
    """Each pixel walks a different sequence of wide splats.  The exact fp32 alpha of every (pixel, splat) pair is
    read back from the colour renderer (one splat alone, colour 1, background 0: the image holds the first blend
    weight (float)(1.0 * alpha) = alpha).  At thresholds that separate the reference's accumulation order from an
    fp32 FMA, the depth image must equal the oracle's reference-order answer bit for bit."""
    ext = gsb.native()
    rng = np.random.default_rng(11)
    H, W, N = 32, 48, 32
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    uv = rng.uniform([3.0, 3.0], [W - 3.0, H - 3.0], (N, 2)).astype(F32)
    var = rng.uniform(400.0, 1600.0, (N, 2))
    cov = rng.uniform(-0.5, 0.5, N) * np.sqrt(var[:, 0] * var[:, 1])
    conic = np.stack([var[:, 0], 2.0 * cov, var[:, 1]], 1).astype(F32)
    opacity = rng.uniform(0.3, 0.9, (N, 1)).astype(F32)
    xyz = pythagorean_positions(N)[rng.permutation(N)]
    counts = [6, 7, 8, 9, 10, 12][:tiles]
    lists = [rng.choice(N, k, replace=False).astype(np.int32) for k in counts]
    ranges = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    idx = np.concatenate(lists)
    uv_t, conic_t, opa_t, xyz_t = to_t(uv), to_t(conic), to_t(opacity), to_t(xyz)
    ranges_t, idx_t = to_t(ranges), to_t(idx)

    # alpha of every splat at every pixel, as the GPU computes it
    one = to_t(np.full((N, 3), unit_colour(), F32))
    alpha = np.empty((N, H, W), F32)
    for g in range(N):
        img = torch.zeros(H, W, 3, device=dev())
        npp = torch.zeros(H, W, dtype=torch.int32, device=dev())
        wl = torch.zeros(H, W, device=dev())
        ext.render_tiles_cuda(uv_t, opa_t, one, conic_t, torch.zeros(1, 1, 1, device=dev()),
                              torch.arange(tiles + 1, dtype=torch.int32, device=dev()),
                              torch.full((tiles,), g, dtype=torch.int32, device=dev()),
                              torch.zeros(3, device=dev()), npp, wl, img)
        img = img.cpu().numpy()
        assert (img[..., 0] == img[..., 1]).all() and (img[..., 0] == img[..., 2]).all()
        alpha[g] = img[..., 0]
    # the renderer skips alpha < 1/255 (the depth walk does not) and never clamps: every alpha here is above it
    assert alpha.min() >= 1.0 / 255 and alpha.max() <= opacity.max()

    # per-pixel sequences, grouped by tile (every pixel of a tile walks the same list)
    ty, tx = np.divmod(np.arange(H * W), W)
    tile_of = (ty // 16) * ((W + 15) // 16) + tx // 16
    seqs = []
    for t, lst in enumerate(lists):
        pix = np.flatnonzero(tile_of == t)
        seqs.append((pix, alpha[lst][:, pix // W, pix % W].T.copy(), np.broadcast_to(xyz[lst], (len(pix), len(lst), 3))))

    def oracle(threshold, order):
        out = np.empty(H * W, F32)
        for pix, a, p in seqs:
            out[pix] = dor.first_surface(a, p, threshold, order)
        return out.reshape(H, W, 1)

    thresholds = [t for _, a, _ in seqs for t, _, _ in dor.separating_thresholds(a, limit=2)]
    assert len(thresholds) >= 8
    differ_from_fma, bad = [], {}
    for t in thresholds + [F32(0.05), F32(0.5), F32(0.9), F32(0.999)]:
        depth = torch.full((H, W, 1), -1.0, device=dev())
        ext.render_depth_cuda(xyz_t, uv_t, opa_t, conic_t, ranges_t, idx_t, float(t), depth)
        want = oracle(t, "reference")
        differ_from_fma.append(int((oracle(t, "fma") != want).sum()))
        got = depth.cpu().numpy()
        n_bad = int((got.view(np.int32) != want.view(np.int32)).sum())
        if n_bad:
            bad[float(t)] = n_bad
        if ref_loader.reference_available():
            ref_depth = torch.full((H, W, 1), -1.0, device=dev())
            ref_ext().render_depth_cuda(xyz_t, uv_t, opa_t, conic_t, ranges_t, idx_t, float(t), ref_depth)
            assert_bits_equal(ref_depth, torch.from_numpy(want), f"compiled reference vs the oracle, threshold {float(t)!r}")
    print("pixels where an fp32-FMA accumulation gives another answer, per threshold:", differ_from_fma)
    assert all(d > 0 for d in differ_from_fma[:len(thresholds)])
    assert not bad, f"pixels (of {H * W}) that differ from the reference order, per threshold: {bad}"


# ------------------------------------------------------------------------------------------------
# 3b. render_depth against the reference's render_depth on its own CUDA
# ------------------------------------------------------------------------------------------------
DEPTH_THRESHOLDS = (0.05, 0.2, 0.5, 0.9, 0.99)


def tiny_camera(W, H, f=60.0):
    return Camera(W, H, to_t(np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]], F32)))


def gaussians_np(xyz, quaternion, scale, opacity, rgb):
    return Gaussians(to_t(xyz), to_t(rgb), to_t(opacity), to_t(scale), to_t(quaternion))


def depth_scene(case):
    """(gaussians, camera_T_world, camera) of one 3b case."""
    if case.startswith("3M"):
        g, cam, T, _ = scenes.headline_inputs(1080, dev())
        g = Gaussians(*(t.detach() for t in (g.xyz, g.rgb, g.opacity, g.scale, g.quaternion)))
        return g, (to_t(scenes.general_pose()) if case.endswith("general") else T), cam
    if case.startswith("100k"):
        sc = scenes.np_scene(100_000, "720p", sh_degree=0, seed=0, view=0, n_views=3)
        T = scenes.general_pose() if case.endswith("general") else sc["T"]
        return gaussians_np(*(sc[k] for k in ("xyz", "quaternion", "scale", "opacity", "rgb"))), to_t(T), \
            Camera(sc["W"], sc["H"], to_t(sc["K"]))
    if case in ("17x33", "1x64"):
        H, W = map(int, case.split("x"))
        sc = scenes.np_scene(3000, "tiny", sh_degree=0, seed=4, sigma_px=(2.0, 0.5, 0.5, 8.0))
        return gaussians_np(*(sc[k] for k in ("xyz", "quaternion", "scale", "opacity", "rgb"))), to_t(sc["T"]), \
            tiny_camera(W, H)
    rng = np.random.default_rng(5)
    if case == "deep_stack":
        # 8000 faint splats over one tile; opacity 0.00055 means 960 splats reach at most A = 0.41, so every pixel
        # that passes 0.5 does so in the reference's second 960-splat chunk or later
        n = 8000
        z = rng.uniform(2.0, 6.0, n)
        u, v = rng.uniform(16.0, 32.0, n), rng.uniform(16.0, 32.0, n)
        xyz = np.stack([(u - 32.0) / 60.0 * z, (v - 32.0) / 60.0 * z, z], 1)
        scale = np.log(z[:, None] * rng.uniform(3.0, 6.0, (n, 3)) / 60.0)
        opacity = np.full((n, 1), -7.5)
    else:  # far: the splats right of the image centre pushed 100 .. 800 times further out along their ray,
        # footprint kept, so the right half of the image sees only splats beyond any far plane
        sc = scenes.np_scene(3000, "tiny", sh_degree=0, seed=6, sigma_px=(2.0, 0.5, 0.5, 8.0))
        n = 3000
        k = np.where(sc["xyz"][:, 0] > 0, rng.uniform(100.0, 800.0, n), 1.0)
        xyz, scale = sc["xyz"] * k[:, None], sc["scale"] + np.log(k)[:, None]
        opacity = sc["opacity"]
    q = rng.normal(size=(n, 4))
    g = gaussians_np(xyz.astype(F32), q.astype(F32), scale.astype(F32), opacity.astype(F32),
                     rng.uniform(0, 1, (n, 3)).astype(F32))
    return g, to_t(np.eye(4, dtype=F32)), tiny_camera(64, 64)


@needs_ref
@pytest.mark.parametrize("case", ["100k_720p_yaw", "100k_720p_general", "3M_1080p_yaw", "3M_1080p_general",
                                  "17x33", "1x64", "deep_stack", "far"])
def test_render_depth_matches_the_reference(case):
    ref_loader.load_reference()
    ref_depth = sys.modules["splat_py_ref.depth"]
    ref_structs = sys.modules["splat_py_ref.structs"]
    g, T, cam = depth_scene(case)
    gr = ref_structs.Gaussians(g.xyz, g.rgb, g.opacity, g.scale, g.quaternion)
    cr = ref_structs.Camera(cam.width, cam.height, cam.K)
    near, pad, mh = 0.3, 100, 3.0
    found = {}
    for t in DEPTH_THRESHOLDS:
        mine = render_depth(g, t, T, cam, near, pad, mh)
        ref = ref_depth.render_depth(gr, t, T, cr, near, pad, mh)
        assert_bits_equal(mine, ref, f"{case}: depth at threshold {t}")
        found[t] = mine
    assert bool((found[0.05] > 0).any()), "no pixel reached the lowest threshold"
    if case == "deep_stack":
        from gaussian_splatting_b200.rasterize import project_and_bin

        s = project_and_bin(g, T, cam, near, float("inf"), pad, mh)
        assert int((s.tile_ranges[1:] - s.tile_ranges[:-1]).max()) > 960
        assert bool((found[0.5] > 0).any()), "no pixel crossed 0.5 beyond the first 960 splats"
    if case == "far":
        assert float(found[0.05].max()) > 500.0, "no splat beyond a far plane of 500 was reported"


# ------------------------------------------------------------------------------------------------
# edge inputs shared by 3c and 3d
# ------------------------------------------------------------------------------------------------
NS = [1, 255, 256, 257, 100_003]
K_NP = np.array([[1200.0, 0.0, 960.5], [0.0, 1100.0, 540.25], [0.0, 0.0, 1.0]])
Z_NONPOS = {3: 0.0, 7: -1e-3, 11: -5.0, 12: 0.0}  # rows with z <= 0 (when N is large enough)


def edge_inputs(n, seed=0):
    """float64 numpy arrays of every per-Gaussian operator's inputs."""
    rng = np.random.default_rng(seed + n)
    z = 10.0 ** rng.uniform(-3, 3, n)
    xyz = np.stack([z * rng.uniform(-1.5, 1.5, n), z * rng.uniform(-1.5, 1.5, n), z], 1)
    for r, v in Z_NONPOS.items():
        if r < n:
            xyz[r, 2] = v
    q = rng.normal(size=(n, 4))
    q *= (10.0 ** rng.uniform(-3, 3, n) * rng.choice([-1.0, 1.0], n) / np.linalg.norm(q, axis=1))[:, None]
    s = rng.uniform(-8.0, 4.0, (n, 3))
    T = scenes.general_pose().astype(np.float64)
    d = rng.normal(size=(n, 3))
    world = T[:3, 3] + d / np.linalg.norm(d, axis=1, keepdims=True) * 10.0 ** rng.uniform(-3, 3, n)[:, None]
    return dict(xyz=xyz, q=q, s=s, T=T, K=K_NP, world=world, rng=rng)


# plain restatements of each operator's forward, in torch (used on the CPU in float64)
def f_projection(xyz, K):
    return torch.stack([K[0, 0] * xyz[:, 0] / xyz[:, 2] + K[0, 2], K[1, 1] * xyz[:, 1] / xyz[:, 2] + K[1, 2]], 1)


def f_sigma_world(q, s):
    w, x, y, z = (q / q.norm(dim=1, keepdim=True)).unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    return R @ torch.diag_embed(torch.exp(2 * s)) @ R.transpose(1, 2)


def f_jacobian(xyz, K):
    x, y, z = xyz.unbind(1)
    zero = torch.zeros_like(z)
    return torch.stack([K[0, 0] / z, zero, -K[0, 0] * x / (z * z), zero, K[1, 1] / z, -K[1, 1] * y / (z * z)],
                       1).view(-1, 2, 3)


def f_conic(S, J, T):
    M = J @ T[:3, :3]
    S2 = M @ S @ M.transpose(1, 2)
    return torch.stack([S2[:, 0, 0], S2[:, 0, 1] + S2[:, 1, 0], S2[:, 1, 1]], 1)


# real SH basis up to degree 3 with the operator's signs; the operator keeps its constants in float32 in both
# precisions, so they are rounded to float32 here too
_SHC = {k: float(F32(v)) for k, v in dict(
    c0=0.5 / math.sqrt(math.pi), c1=math.sqrt(3 / (4 * math.pi)), c20=0.5 * math.sqrt(15 / math.pi),
    c22=0.25 * math.sqrt(5 / math.pi), c24=0.25 * math.sqrt(15 / math.pi), c30=0.25 * math.sqrt(35 / (2 * math.pi)),
    c31=0.5 * math.sqrt(105 / math.pi), c32=0.25 * math.sqrt(21 / (2 * math.pi)),
    c33=0.25 * math.sqrt(7 / (2 * math.pi)), c35=0.25 * math.sqrt(105 / math.pi),
    r0=2.0 * math.sqrt(math.pi)).items()}  # r0 = 1 / c0, the factor the operator multiplies by


def sh_basis(d, n_sh):
    x, y, z = d.unbind(1)
    c = _SHC
    Y = [torch.full_like(x, c["c0"]), -c["c1"] * y, c["c1"] * z, -c["c1"] * x,
         c["c20"] * x * y, -c["c20"] * y * z, c["c22"] * (3 * z * z - 1), -c["c20"] * x * z, c["c24"] * (x * x - y * y),
         -c["c30"] * y * (3 * x * x - y * y), c["c31"] * x * y * z, -c["c32"] * y * (5 * z * z - 1),
         c["c33"] * z * (5 * z * z - 3), -c["c32"] * x * (5 * z * z - 1), c["c35"] * z * (x * x - y * y),
         -c["c30"] * x * (x * x - 3 * y * y)]
    return torch.stack(Y[:n_sh], 1)


def f_sh_rgb(sh, world, T):
    """rgb [N,3] from sh [N,3,n_sh]: the basis at the direction from T[:3,3] to the point, over SH0; n_sh = 1 passes
    the coefficients through."""
    if sh.shape[2] == 1:
        return sh[:, :, 0]
    d = world - T[:3, 3]
    Y = sh_basis(d / d.norm(dim=1, keepdim=True), sh.shape[2])
    return (sh * Y[:, None, :]).sum(2) * _SHC["r0"]


# ------------------------------------------------------------------------------------------------
# 3c. backward kernels, row by row, against fp64 autograd
# ------------------------------------------------------------------------------------------------
# Row bound |mine - ref| <= RTOL * max|mass row| (gradrows.compare_rows), allowing no row beyond it.  mass is the
# gradient's sum of magnitudes, sum_j |d out_j / d in_i| * |grad_out_j|: a gradient entry that cancels (the scale
# gradient 2 e_k^2 r_k^T G r_k of a row whose dominant axis has r_k^T G r_k ~ 1e-4 |G|) is judged by the size of the
# terms it cancelled, which is what fp32 arithmetic can resolve.  max|ref row| alone needed 1.1e-3 for such rows in
# fp32, above the 1e-3 error the negative control must catch.  There is no floor: the rows span more than 20 orders
# of magnitude (z from 1e-3 to 1e3, log-scales -8 .. 4), and every row is held to its own scale.
# Worst |mine - ref| / max|mass row| over N in {1, 255, 256, 257, 100003}, one H100 80GB HBM3 (400 W power limit):
#                                      fp32      fp64
#   camera_projection   xyz           2.3e-7    4.4e-16
#   sigma_world         quaternion    2.5e-6    6.0e-15
#                       scale         1.6e-6    4.8e-15
#   projection_jacobian xyz           2.0e-7    5.3e-16
#   conic               sigma_world   2.3e-7    4.8e-16
#                       J             8.3e-6    7.0e-15
#   rgb_from_sh 1/4/9/16 sh           0 / 2.9e-7 / 6.0e-7 / 8.4e-7    0 / 5.4e-16 / 1.3e-15 / 1.7e-15
RTOL = {torch.float32: 3e-5, torch.float64: 1e-13}
PERTURB = 1e-3


def vjp_and_mass(fn, inputs, grad_out):
    """fn maps rows to rows.  Returns, per input, the gradient of <fn(*inputs), grad_out> and its mass
    sum_j |d out_j / d in_i| * |grad_out_j|, from each row's Jacobian (torch fp64 on the CPU)."""
    xs = [torch.from_numpy(np.asarray(a, np.float64)) for a in inputs]
    G = torch.from_numpy(np.asarray(grad_out, np.float64)).reshape(len(xs[0]), -1)

    def one_row(*r):
        return fn(*(t.unsqueeze(0) for t in r)).squeeze(0)

    jac = torch.func.vmap(torch.func.jacrev(one_row, argnums=tuple(range(len(xs)))))(*xs)
    out = []
    for x, J in zip(xs, jac):
        J = J.reshape(len(x), G.shape[1], -1)
        out.append((torch.einsum("no,noi->ni", G, J).reshape(x.shape).numpy(),
                    torch.einsum("no,noi->ni", G.abs(), J.abs()).reshape(x.shape).numpy()))
    return out


def backward_case(op, n, dtype):
    """[(name, gpu result [N, ...] as numpy, (fp64 reference, its mass))] for one backward operator."""
    ext = gsb.native()
    e = edge_inputs(n)
    rng = e["rng"]
    npdt = np.float32 if dtype == torch.float32 else np.float64
    cast = lambda a: np.asarray(a, npdt)  # noqa: E731  (the GPU's inputs; the reference starts from the same values)
    K, T = cast(e["K"]), cast(e["T"])
    Kt, Tt = to_t(K), to_t(T)
    if op == "camera_projection":
        xyz, g = cast(e["xyz"]), cast(rng.normal(size=(n, 2)))
        out = torch.full((n, 3), 12345.0, dtype=dtype, device=dev())
        ext.camera_projection_backward_cuda(to_t(xyz), Kt, to_t(g), out)
        out = out.cpu().numpy()
        pos = xyz[:, 2] > 0
        assert (out[~pos] == 12345.0).all(), "rows with z <= 0 were written"
        ref = vjp_and_mass(lambda x: f_projection(x, torch.from_numpy(K.astype(np.float64))), [xyz[pos]], g[pos])[0]
        return [("xyz", out[pos], ref)]
    if op == "sigma_world":
        q, s, G = cast(e["q"]), cast(e["s"]), cast(rng.normal(size=(n, 3, 3)))
        gq = torch.zeros(n, 4, dtype=dtype, device=dev())
        gs = torch.zeros(n, 3, dtype=dtype, device=dev())
        ext.compute_sigma_world_backward_cuda(to_t(q), to_t(s), to_t(G), gq, gs)
        rq, rs = vjp_and_mass(f_sigma_world, [q, s], G)
        return [("quaternion", gq.cpu().numpy(), rq), ("scale", gs.cpu().numpy(), rs)]
    if op == "jacobian":
        xyz, G = cast(e["xyz"]), cast(rng.normal(size=(n, 2, 3)))
        ok = xyz[:, 2] != 0
        out = torch.zeros(n, 3, dtype=dtype, device=dev())
        ext.compute_projection_jacobian_backward_cuda(to_t(xyz), Kt, to_t(G), out)
        ref = vjp_and_mass(lambda x: f_jacobian(x, torch.from_numpy(K.astype(np.float64))), [xyz[ok]], G[ok])[0]
        return [("xyz", out.cpu().numpy()[ok], ref)]
    if op == "conic":
        xyz = e["xyz"].copy()
        xyz[:, 2] = np.abs(xyz[:, 2]) + (xyz[:, 2] == 0)
        with torch.no_grad():
            S = cast(f_sigma_world(torch.from_numpy(e["q"]), torch.from_numpy(e["s"])).numpy())
            J = cast(f_jacobian(torch.from_numpy(xyz), torch.from_numpy(e["K"])).numpy())
        G = cast(rng.normal(size=(n, 3)))
        gS = torch.zeros(n, 3, 3, dtype=dtype, device=dev())
        gJ = torch.zeros(n, 2, 3, dtype=dtype, device=dev())
        ext.compute_conic_backward_cuda(to_t(S), to_t(J), Tt, to_t(G), gS, gJ)
        rS, rJ = vjp_and_mass(lambda s_, j_: f_conic(s_, j_, torch.from_numpy(T.astype(np.float64))), [S, J], G)
        return [("sigma_world", gS.cpu().numpy(), rS), ("J", gJ.cpu().numpy(), rJ)]
    n_sh = int(op[2:])  # "sh1", "sh4", ...
    world, G = cast(e["world"]), cast(rng.normal(size=(n, 3)))
    Tr = torch.from_numpy(T.astype(np.float64))
    ref = vjp_and_mass(lambda sh, w: f_sh_rgb(sh, w, Tr), [np.zeros((n, 3, n_sh)), world], G)[0]
    res = []
    for shape in ([(n, 3, n_sh)] + ([(n, 3)] if n_sh == 1 else [])):
        out = torch.zeros(shape, dtype=dtype, device=dev())
        ext.precompute_rgb_from_sh_backward_cuda(to_t(world), Tt, to_t(G), out)
        res.append((f"sh {list(shape)}", out.cpu().numpy().reshape(n, 3, n_sh), ref))
    return res


BWD_OPS = ["camera_projection", "sigma_world", "jacobian", "conic", "sh1", "sh4", "sh9", "sh16"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("op", BWD_OPS)
def test_backward_rows_against_fp64_autograd(op, n, dtype):
    def judge(label, mine, ref, mass):
        bound = RTOL[dtype] * np.broadcast_to(gradrows.as_rows(mass).max(1, keepdims=True), gradrows.as_rows(ref).shape)
        return gradrows.compare_rows(label, mine, ref, bound, 0)

    cases = backward_case(op, n, dtype)
    results = []
    for name, mine, (ref, mass) in cases:
        r = judge(f"{op}_backward {name} {str(dtype)[6:]} N={n}", mine, ref, mass)
        err = np.abs(gradrows.as_rows(mine) - gradrows.as_rows(ref))
        print(f"{r}; worst |mine - ref| / max|mass row| = "
              f"{float((err / gradrows.as_rows(mass).max(1, keepdims=True)).max()):.3g}")
        results.append(r)
    gradrows.assert_all(results)
    # negative control: the best-conditioned row, off by a relative 1e-3, is flagged, and no other row
    name, mine, (ref, mass) = cases[0]
    ref_rows, mass_rows = gradrows.as_rows(ref), gradrows.as_rows(mass)
    row = int(np.argmax(np.abs(ref_rows).max(1) / mass_rows.max(1)))
    bent = np.array(mine, np.float64)
    bent[row] *= 1.0 + PERTURB
    r = judge(f"{op} {name} perturbed", bent, ref, mass)
    assert r.bad.tolist() == [row], str(r)


# ------------------------------------------------------------------------------------------------
# 3d. forward kernels and tile binning, bit for bit against the compiled reference
# ------------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("n", NS)
def test_forward_operators_bitwise_against_the_reference(n):
    mine_ext, ref = gsb.native(), ref_ext()
    e = edge_inputs(n)
    xyz, q, s, world = (to_t(e[k].astype(F32)) for k in ("xyz", "q", "s", "world"))
    K, T = to_t(e["K"].astype(F32)), to_t(e["T"].astype(F32))
    sh = to_t(e["rng"].normal(size=(n, 3, 16)).astype(F32))

    def both(fn_name, shape, *args):
        outs = []
        for ext in (mine_ext, ref):
            out = torch.zeros(shape, device=dev())
            getattr(ext, fn_name)(*args, out)
            outs.append(out)
        assert_bits_equal(outs[0], outs[1], f"{fn_name} N={n}")
        return outs[0]

    both("camera_projection_cuda", (n, 2), xyz, K)
    S = both("compute_sigma_world_cuda", (n, 3, 3), q, s)
    J = both("compute_projection_jacobian_cuda", (n, 2, 3), xyz, K)
    pos = xyz[:, 2] > 0  # the conic of a point behind the camera is never formed
    both("compute_conic_cuda", (int(pos.sum()), 3), S[pos].contiguous(), J[pos].contiguous(), T)
    for n_sh in (4, 9, 16):
        both("precompute_rgb_from_sh_cuda", (n, 3), world, sh[:, :, :n_sh].contiguous(), T)
    both("precompute_rgb_from_sh_cuda", (n, 3), world, sh[:, :, :1].contiguous(), T)
    both("precompute_rgb_from_sh_cuda", (n, 3), world, sh[:, :, 0].contiguous(), T)


@needs_ref
@pytest.mark.parametrize("n", NS)
def test_tile_binning_bitwise_against_the_reference(n):
    """get_sorted_gaussian_list: sorted gaussian index and tile ranges of N visible splats of a 720p scene."""
    from gaussian_splatting_b200.rasterize import project_and_bin

    sc = scenes.np_scene(n * 3 // 2 + 1000, "720p", sh_degree=0, seed=n, view=1, n_views=3)
    g = gaussians_np(*(sc[k] for k in ("xyz", "quaternion", "scale", "opacity", "rgb")))
    cam = Camera(sc["W"], sc["H"], to_t(sc["K"]))
    with torch.no_grad():
        st = project_and_bin(g, to_t(sc["T"]), cam, 0.3, 500.0, 100, 3.0)
    uv, xyz_cam, conic = (t.detach()[:n].contiguous() for t in (st.uv, st.xyz_cam, st.conic))
    assert uv.shape[0] == n
    outs = [ext.get_sorted_gaussian_list(1024, uv, xyz_cam, conic, 80, 45, 3.0) for ext in (gsb.native(), ref_ext())]
    assert_bits_equal(outs[0][1], outs[1][1], f"tile ranges N={n}")
    assert_bits_equal(outs[0][0], outs[1][0], f"sorted gaussian index N={n}")
    assert outs[0][0].numel() > 0
