"""Camera self-calibration on the GPU: d loss / d K and d loss / d lens coefficients from rasterize and
rasterize_batch, for every lens, against the fp64 oracle (tests/calib_oracle.py) on the GPU's own rows, the pinhole
gauge identities at the headline size, bitwise invariance of everything else, determinism, batching, edge cases, and
recovery of perturbed intrinsics with IntrinsicsDelta — needs an H100."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import native, rasterize_batch
from gaussian_splatting_b200.calib import IntrinsicsDelta
from gaussian_splatting_b200.densify import WeightStats
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera, Gaussians
from tests import calib_oracle as co
from tests import scenes
from tests.scenes import headline_inputs
from tests.test_gradient_rows_gpu import gaussians_from, np_scene
from tests.test_pose_gpu import BG, LENS_K, MODES, _backward, _capture_rows, _flags, bits, dev, scene, to_t

pytestmark = pytest.mark.gpu
LENSES = ("pinhole", "fisheye", "distortion")
# the bound of the pose gradient (test_pose_gpu.POSE_RTOL): each contribution is the fp32 chain of the per-gaussian
# backward plus a few roundings of the lens's k-derivatives; 2^-13 of sum_i |c_i| per value
RTOL = 2.0 ** -13


def lens_kw(lens, k, C=None):
    """the lens keyword with coefficients k (a CPU tensor that may require grad), [n] or [C,n]"""
    return {} if lens == "pinhole" else {lens: k}


def lens_tensor(lens, C=None, requires_grad=True):
    if lens == "pinhole":
        return None
    k = torch.tensor(LENS_K[lens], dtype=torch.float32)
    if C is not None:
        k = k.expand(C, -1).clone()
    return k.requires_grad_(requires_grad)


def run_single(sc, lens, mode, seed=1, pose_grad=False, K_grad=True, k_grad=True, **extra):
    flags, f = _flags(sc, mode)
    g = gaussians_from(sc)
    T = to_t(sc["T"]).requires_grad_(pose_grad)
    K = to_t(sc["K"]).requires_grad_(K_grad)
    k = lens_tensor(lens, requires_grad=k_grad)
    out = rasterize(g, T, Camera(sc["W"], sc["H"], K), 0.3, 500.0, 100, 3.0, True,
                    torch.full((3,), BG, device=dev()), return_state=True, **lens_kw(lens, k), **flags, **extra)
    seen = _capture_rows(out)
    _backward(out, flags.get("render_depth_alpha", False), seed)
    return out, g, T, K, k, seen[0], f


def _oracle(sc, lens, mode, f, rows, visible):
    flags = MODES[mode]
    o = co.rasterize(lens, sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"],
                     sc["K"], sc["H"], sc["W"], LENS_K[lens], antialiased=flags.get("antialiased", False),
                     filter3d=f, background=np.full(3, BG))
    assert np.array_equal(o.keep, visible), "the oracle culls other gaussians than the GPU"
    return co.camera_grad(o, lens, co.rows_from_slab(rows.cpu().numpy(), flags.get("render_depth_alpha", False)),
                          visible)


def _check(got_K, got_k, want, lens, tag):
    gK, gk, mass = want
    got4 = np.array([got_K[0, 0], got_K[1, 1], got_K[0, 2], got_K[1, 2]], np.float64)
    assert mass[:4].max() > 0
    rest = got_K.copy()
    rest[0, 0] = rest[1, 1] = rest[0, 2] = rest[1, 2] = 0
    assert (rest == 0).all(), (tag, got_K)
    err = np.abs(got4 - gK)
    assert (err <= RTOL * mass[:4] + 1e-12).all(), (tag, (err / np.maximum(mass[:4], 1e-30)).max())
    if lens != "pinhole":
        err = np.abs(np.asarray(got_k, np.float64) - gk)
        assert (err <= RTOL * mass[4:] + 1e-12).all(), (tag, (err / np.maximum(mass[4:], 1e-30)).max())


# ---- 1. the fp64 oracle on the GPU's own rows ---------------------------------------------------------------------
@pytest.mark.parametrize("shd", [0, 1, 2, 3])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("lens", LENSES)
def test_camera_gradient_matches_the_fp64_oracle(lens, mode, shd):
    sc = scene(shd)
    out, g, T, K, k, rows, f = run_single(sc, lens, mode)
    want = _oracle(sc, lens, mode, f, rows, out[-1].visible.cpu().numpy().astype(bool))
    assert K.grad.shape == (3, 3)
    if k is not None:
        assert k.grad.shape == k.shape and k.grad.dtype == k.dtype and k.grad.device.type == "cpu"
    _check(K.grad.double().cpu().numpy(), None if k is None else k.grad.numpy(), want, lens, (lens, mode, shd))


@pytest.mark.parametrize("per_view", [False, True])
@pytest.mark.parametrize("mode", ["plain", "all"])
@pytest.mark.parametrize("lens", LENSES)
def test_batched_camera_gradient_matches_the_fp64_oracle(lens, mode, per_view):
    """Three views of the SH 3 scene, K and the coefficients shared ([3,3], [n]) or per view ([C,3,3], [C,n]): view
    c's values against the oracle on view c's rows; a shared K or k gets the sum over the views."""
    C = 3
    scs = [scenes.np_scene(2000, "tiny", 3, view=c, sigma_px=(0.8, 0.8, 0.15, 8.0)) for c in range(C)]
    sc = scs[0]
    flags, f = _flags(sc, mode)
    g = gaussians_from(sc)
    T = torch.stack([to_t(s["T"]) for s in scs])
    K = (to_t(sc["K"]).expand(C, 3, 3).clone() if per_view else to_t(sc["K"])).requires_grad_(True)
    k = lens_tensor(lens, C if per_view else None)
    out = rasterize_batch(g, T, Camera(sc["W"], sc["H"], K), 0.3, 500.0, 100, 3.0, True,
                          torch.full((3,), BG, device=dev()), return_state=True, **lens_kw(lens, k), **flags)
    seen = _capture_rows(out)
    _backward(out, flags.get("render_depth_alpha", False))
    rows = seen[0].view(C, -1)
    vis = out[-1].visible.cpu().numpy().astype(bool)
    wants = [_oracle(scs[c], lens, mode, f, rows[c], vis[c]) for c in range(C)]
    gotK = K.grad.double().cpu().numpy()
    gotk = None if k is None else k.grad.double().numpy()
    if per_view:
        for c in range(C):
            _check(gotK[c], None if k is None else gotk[c], wants[c], lens, (lens, mode, c))
    else:
        want = tuple(sum(w[i] for w in wants) for i in range(3))
        _check(gotK, gotk, want, lens, (lens, mode, "shared"))


# ---- 2. pinhole gauge identities at the headline size -----------------------------------------------------------------
def test_pinhole_gauge_identities_at_the_headline_size():
    """3M gaussians, 1080p, SH 3, depth/alpha + antialiased + filter3d; T and K require grad in one backward, so both
    use the same rows.  Scaling fx scales the camera frame's x row, and shifting cx shears x by z / fx:
      fx dL/dfx = sum_j T[0,j] dL/dT[0,j],  fy dL/dfy = sum_j T[1,j] dL/dT[1,j],
      fx dL/dcx = sum_j T[2,j] dL/dT[0,j],  fy dL/dcy = sum_j T[2,j] dL/dT[1,j]."""
    H = 1080
    g, cam, T0, G = headline_inputs(H, dev())
    T = T0.clone().requires_grad_(True)
    K = cam.K.clone().requires_grad_(True)
    f = (torch.exp(g.scale.detach().mean(1)) * 0.5).contiguous()
    out = rasterize(g, T, Camera(cam.width, cam.height, K), 0.3, 500.0, 100, 3.0, True,
                    torch.full((3,), BG, device=dev()), render_depth_alpha=True, antialiased=True, filter3d=f)
    out[2].retain_grad()
    gen = torch.Generator().manual_seed(2)
    Gd = (torch.randn(H, 1920, 1, generator=gen, dtype=torch.float64) / (H * 1920)).float().to(dev())
    torch.autograd.backward([out[0], out[3], out[4]], [G, Gd, Gd])
    gT, gK, T64, K64 = T.grad.double(), K.grad.double(), T0.double(), cam.K.double()
    uv, guv = out[2].detach().double(), out[2].grad.double()
    # the uv part of each identity, per gaussian: a cancellation-free scale for the fp32 sums
    uv_mass = [(guv[:, 0] * (uv[:, 0] - K64[0, 2])).abs().sum(), (guv[:, 1] * (uv[:, 1] - K64[1, 2])).abs().sum(),
               K64[0, 0] * guv[:, 0].abs().sum(), K64[1, 1] * guv[:, 1].abs().sum()]
    for (lhs, rhs_terms), m in zip(
            [(K64[0, 0] * gK[0, 0], T64[0] * gT[0]), (K64[1, 1] * gK[1, 1], T64[1] * gT[1]),
             (K64[0, 0] * gK[0, 2], T64[2] * gT[0]), (K64[1, 1] * gK[1, 2], T64[2] * gT[1])], uv_mass):
        mass = float(lhs.abs() + rhs_terms.abs().sum() + m)
        assert abs(float(lhs - rhs_terms.sum())) <= 1e-4 * mass, (float(lhs), float(rhs_terms.sum()), mass)
    assert gK[2].abs().sum() == 0 and gK[0, 1] == 0 and gK[1, 0] == 0


# ---- 3. nothing else changes -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("lens", LENSES)
@pytest.mark.parametrize("opts", ["maps", "features"])
def test_everything_else_is_bit_identical(lens, opts):
    """The forward's outputs (image, mask, uv, depth / alpha, feature map, weight maxima and pixel counts; the weight
    sums, fp32 atomics, to 1e-5) with K and k requiring grad or not.  The gradients are compared on the same rows in
    test_camera_grads_2_repeat_match_camera_grads_1_and_the_batch_matches_single_views."""
    sc = scene(3)
    outs, sums = [], []
    for want in (False, True):
        if opts == "maps":
            mode = "all"
            extra = dict(absgrad=True, weight_stats=WeightStats(len(sc["xyz"]), dev()))
        else:
            mode = "depth"
            extra = dict(features=to_t(np.random.default_rng(5).standard_normal((len(sc["xyz"]), 5)).astype(np.float32))
                         .requires_grad_(True))
        flags, f = _flags(sc, mode)
        g = gaussians_from(sc)
        K = to_t(sc["K"]).requires_grad_(want)
        k = lens_tensor(lens, requires_grad=want)
        out = rasterize(g, to_t(sc["T"]), Camera(sc["W"], sc["H"], K), 0.3, 500.0, 100, 3.0, True,
                        torch.full((3,), BG, device=dev()), return_state=True, **lens_kw(lens, k), **flags, **extra)
        maps = [m for m in out[:-1] if m.dtype == torch.float32 and m.requires_grad and m is not out[2]]
        rng = np.random.default_rng(9)
        torch.autograd.backward(maps, [to_t((rng.standard_normal(tuple(m.shape)) / m.numel()).astype(np.float32))
                                       for m in maps])
        assert (K.grad is not None) == want
        if k is not None:
            assert (k.grad is not None) == want
        rec = list(out[:-1])
        if opts == "maps":
            ws = extra["weight_stats"]
            rec += [ws.weight_max, ws.pixel_count]
            sums.append(ws.weight_sum.double())
        outs.append(rec)
    for a, b in zip(*outs):
        assert np.array_equal(bits(a), bits(b))
    if sums:
        assert torch.allclose(sums[0], sums[1], rtol=1e-5, atol=0)


# ---- 4. determinism, batching and edge cases ---------------------------------------------------------------------------
def _lens_args(st, c=None):
    """The lens keyword arguments of the per-gaussian bindings for a state's lens, view c's constants alone for c"""
    if st.lens is None:
        return dict(lens=native().LENS_PINHOLE, lens_consts=None)
    enum, consts = st.lens
    return dict(lens=enum, lens_consts=consts if c is None else consts[c:c + 1].contiguous())


@pytest.mark.parametrize("lens", LENSES)
def test_camera_grads_2_repeat_match_camera_grads_1_and_the_batch_matches_single_views(lens):
    """On the same rows: two calls give the same bits; the gaussian gradients and the pose gradient equal the pose
    kernels' bit for bit; batched view c equals the single-view call on view c's rows; the rasterize_batch gradients
    are the binding's (a shared K: the sum over the views)."""
    ext = native()
    C = 3
    scs = [scenes.np_scene(5000, "tiny", 3, view=c, sigma_px=(0.8, 0.8, 0.15, 8.0)) for c in range(C)]
    flags, f = _flags(scs[0], "all")
    g = gaussians_from(scs[0])
    T = torch.stack([to_t(s["T"]) for s in scs]).requires_grad_(True)
    K = to_t(scs[0]["K"]).requires_grad_(True)
    k = lens_tensor(lens)
    out = rasterize_batch(g, T, Camera(scs[0]["W"], scs[0]["H"], K), 0.3, 500.0, 100, 3.0, True,
                          torch.full((3,), BG, device=dev()), return_state=True, **lens_kw(lens, k), **flags)
    seen = _capture_rows(out)
    _backward(out, True)
    st = out[-1]
    slab = seen[0].contiguous()
    xyz, q, s, o, sh = (getattr(g, p).detach().contiguous() for p in ("xyz", "quaternion", "scale", "opacity", "sh"))
    Td = T.detach().contiguous()
    Kd = K.detach()
    Ks = Kd.expand(C, 3, 3).contiguous()
    centre = torch.stack([ext.camera_centre(Td[c]) for c in range(C)])
    lk = _lens_args(st)
    args = (slab, xyz, q, s, o.reshape(-1), sh, Td, Ks, centre, st.visible, None, None, None, True, st.mode,
            flags.get("filter3d"))
    a = ext.batch_preprocess_backward(*args, **lk, camera_grads=2)
    b = ext.batch_preprocess_backward(*args, **lk, camera_grads=2)
    for x, y in zip(a, b):
        assert np.array_equal(bits(x), bits(y))
    pose = ext.batch_preprocess_backward(*args, **lk, camera_grads=1)
    assert len(a) == len(pose) + 2
    for x, y in zip(a[:len(pose)], pose):  # gaussian gradients, the flat allocation and g_pose
        assert np.array_equal(bits(x), bits(y))
    g_pose, g_intr, g_lens = a[-3:]
    assert tuple(g_intr.shape) == (C, 4) and tuple(g_lens.shape) == (C, co.N_COEFFS[lens])
    assert np.array_equal(bits(g_pose), bits(T.grad))
    assert torch.allclose(K.grad[[0, 1, 0, 1], [0, 1, 2, 2]], g_intr.sum(0), rtol=1e-6, atol=0)
    if k is not None:
        assert torch.equal(k.grad, g_lens.cpu().double().sum(0).float())
    for c in range(C):
        one = (slab.view(C, -1)[c].contiguous(), xyz, q, s, o.reshape(-1), sh, Td[c].contiguous(), Kd,
               centre[c].contiguous(), st.visible[c].contiguous(), None, None, None, True, st.mode,
               flags.get("filter3d"))
        single = ext.fused_preprocess_backward(*one, **_lens_args(st, c), camera_grads=2)
        assert np.array_equal(bits(single[-3]), bits(g_pose[c])), c
        assert np.array_equal(bits(single[-2]), bits(g_intr[c])), c
        assert np.array_equal(bits(single[-1]), bits(g_lens[c])), c
        pose1 = ext.fused_preprocess_backward(*one, **_lens_args(st, c), camera_grads=1)
        for x, y in zip(single[:len(pose1)], pose1):
            assert np.array_equal(bits(x), bits(y)), c


@pytest.mark.parametrize("lens", LENSES)
def test_camera_grads_of_empty_and_all_culled_scenes_are_zero(lens):
    sc = scene(0)
    K = to_t(sc["K"])
    ext = native()
    z = lambda *shape: torch.zeros(shape, device=dev())  # noqa: E731
    enum = getattr(ext, "LENS_" + lens.upper())
    lc = None
    if lens != "pinhole":
        lim = (ext.fisheye_theta_max if lens == "fisheye" else ext.distortion_r2_max)(list(LENS_K[lens]))
        lc = to_t(np.array(list(LENS_K[lens]) + [lim], np.float32))
    args = (z(0), z(0, 3), z(0, 4), z(0, 3), z(0), None, to_t(sc["T"]), K, None,
            torch.zeros(0, dtype=torch.uint8, device=dev()), None, None, None, True, 0, None)
    for t in ext.fused_preprocess_backward(*args, lens=enum, lens_consts=lc, camera_grads=2)[-3:]:
        assert (t == 0).all()
    T2 = to_t(np.stack([sc["T"], sc["T"]]))
    args = (z(0),) + args[1:6] + (T2, K.expand(2, 3, 3).contiguous(), None,
                                  torch.zeros(2, 0, dtype=torch.uint8, device=dev())) + args[10:]
    outs = ext.batch_preprocess_backward(*args, lens=enum, lens_consts=None if lc is None else torch.cat([lc, lc]),
                                         camera_grads=2)[-3:]
    assert tuple(outs[1].shape) == (2, 4)
    for t in outs:
        assert (t == 0).all()
    # every gaussian behind the camera
    Tb = np.array(sc["T"], np.float32)
    Tb[2, 3] -= 1000.0
    Kg = K.clone().requires_grad_(True)
    k = lens_tensor(lens)
    out = rasterize(gaussians_from(sc), to_t(Tb), Camera(sc["W"], sc["H"], Kg), 0.3, 500.0, 100, 3.0, True,
                    torch.full((3,), BG, device=dev()), **lens_kw(lens, k))
    assert bool(out[1].all())
    out[0].sum().backward()
    assert (Kg.grad == 0).all() and (k is None or (k.grad == 0).all())


def test_lens_and_camera_grads_arguments_reject_bad_values():
    """The per-gaussian bindings raise for an unknown lens, a lens without its constants (or the pinhole with some) and
    camera_grads outside 0..2, one view and a batch, forward and backward."""
    sc = scene(0)
    ext = native()
    z = lambda *shape: torch.zeros(shape, device=dev())  # noqa: E731
    T, K = to_t(sc["T"]), to_t(sc["K"])
    T2, K2 = T.expand(2, 4, 4).contiguous(), K.expand(2, 3, 3).contiguous()
    lc = to_t(np.array(list(LENS_K["fisheye"]) + [ext.fisheye_theta_max(list(LENS_K["fisheye"]))], np.float32))
    gauss = (z(0, 3), None, z(0, 4), z(0, 3), z(0), z(0, 3), None)
    cfg = (None, sc["H"], sc["W"], 0.3, 500.0, 100.0, 3.0, 0)
    fwds = (lambda **kw: ext.fused_preprocess_forward(*gauss, T, K, *cfg, True, 0, None, **kw),
            lambda **kw: ext.batch_preprocess_forward(*gauss, T2, K2, *cfg, 0, None, **kw))
    tail = (None, None, None, True, 0, None)
    bwds = (lambda **kw: ext.fused_preprocess_backward(z(0), z(0, 3), z(0, 4), z(0, 3), z(0), None, T, K, None,
                                                       torch.zeros(0, dtype=torch.uint8, device=dev()), *tail, **kw),
            lambda **kw: ext.batch_preprocess_backward(z(0), z(0, 3), z(0, 4), z(0, 3), z(0), None, T2, K2, None,
                                                       torch.zeros(2, 0, dtype=torch.uint8, device=dev()), *tail,
                                                       **kw))
    for fn in fwds + bwds:
        for lens in (-1, 3):
            with pytest.raises(RuntimeError, match="lens must be 0"):
                fn(lens=lens)
        with pytest.raises(RuntimeError, match="a lens needs its constants"):
            fn(lens=ext.LENS_FISHEYE)
        with pytest.raises(RuntimeError, match="the pinhole takes no lens constants"):
            fn(lens=ext.LENS_PINHOLE, lens_consts=lc)
    for fn in bwds:
        for camera_grads in (-1, 3):
            with pytest.raises(RuntimeError, match="camera_grads must be 0"):
                fn(camera_grads=camera_grads)
        assert len(fn(camera_grads=2)) == 6 + 3  # the valid values still run: flat and the camera gradients


@pytest.mark.parametrize("lens", LENSES)
def test_intrinsics_only_graph_records_masks(lens):
    sc = scene(0)
    g = Gaussians(*(to_t(sc[k]) for k in ("xyz", "rgb", "opacity", "scale", "quaternion")), None)
    delta = IntrinsicsDelta(1, device=dev())
    K = delta(to_t(sc["K"]), 0)
    out = rasterize(g, to_t(sc["T"]), Camera(sc["W"], sc["H"], K), 0.3, 500.0, 100, 3.0, True,
                    torch.full((3,), BG, device=dev()), return_state=True,
                    **lens_kw(lens, None if lens == "pinhole" else LENS_K[lens]))
    assert out[-1].masks.numel() > 0
    (out[0] * to_t(np.random.default_rng(0).standard_normal(tuple(out[0].shape)).astype(np.float32))).sum().backward()
    for p in (delta.log_focal, delta.principal):
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0


# ---- 5. recovery -------------------------------------------------------------------------------------------------------
TRUE_K = {"pinhole": None, "fisheye": (0.10, -0.04, 0.01, -0.002), "distortion": (-0.09, 0.02, 1e-3, -8e-4, 0.01)}


@pytest.mark.parametrize("lens", LENSES)
def test_intrinsics_recovery(lens):
    """4000 gaussians at 128 x 128 (the tiny scene, twice the focal length), frozen; the target is rendered with the true
    camera fx x 1.03, cx + 4 px and, per lens, coefficients off the nominal ones; IntrinsicsDelta and a CPU coefficient
    parameter start at the nominal camera; Adam on the L1 image loss, learning rates decayed by 0.99 per step for 300
    steps.  The intrinsics error max(|fx / fx_true - 1| / 0.03, |cx - cx_true| / 4 px) must fall below 1/10 of the
    start (1)."""
    sc = np_scene(4000, "tiny", 0, sigma_px=(1.0, 0.5, 0.3, 6.0))
    g = Gaussians(*(to_t(sc[k]) for k in ("xyz", "rgb", "opacity", "scale", "quaternion")), None)
    K0 = np.array(sc["K"], np.float32)
    K0[:2] *= 2.0
    Kt = K0.copy()
    Kt[0, 0] *= 1.03
    Kt[0, 2] += 4.0
    bg = torch.full((3,), BG, device=dev())
    with torch.no_grad():
        target = rasterize(g, to_t(sc["T"]), Camera(128, 128, to_t(Kt)), 0.3, 500.0, 100, 3.0, True, bg,
                           **lens_kw(lens, None if lens == "pinhole" else TRUE_K[lens]))[0]
    delta = IntrinsicsDelta(1, device=dev())
    groups = [{"params": [delta.log_focal], "lr": 2e-3}, {"params": [delta.principal], "lr": 0.1}]
    k = None
    if lens != "pinhole":
        k = torch.nn.Parameter(torch.tensor([LENS_K[lens]], dtype=torch.float32))
        groups.append({"params": [k], "lr": 2e-3})
    opt = torch.optim.Adam(groups)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.99)
    K0t = to_t(K0)

    def error():
        with torch.no_grad():
            K = delta(K0t, 0)
            return max(abs(float(K[0, 0]) / Kt[0, 0] - 1) / 0.03, abs(float(K[0, 2]) - Kt[0, 2]) / 4.0)

    e0 = error()
    for _ in range(300):
        opt.zero_grad(set_to_none=True)
        img = rasterize(g, to_t(sc["T"]), Camera(128, 128, delta(K0t, 0)), 0.3, 500.0, 100, 3.0, True, bg,
                        **lens_kw(lens, None if k is None else k[0]))[0]
        (img - target).abs().mean().backward()
        opt.step()
        sched.step()
    e = error()
    print(f"intrinsics recovery {lens}: error {e:.4f} (start {e0:.2f}), K {delta(K0t, 0).detach().cpu().numpy()[:2]}, "
          f"k {None if k is None else k.detach().numpy()}")
    assert e0 == pytest.approx(1.0) and e < 0.1 * e0, e
