"""Rolling-shutter cameras on the GPU: rasterize(..., rolling_shutter=xi) and rasterize_batch against the fp64 oracle
(tests/shutter_oracle.py) on the GPU's own rows, the global-shutter limit at the headline size, per-line ground truth,
invariance, determinism, recovery of a known readout motion, and edge cases — needs an H100."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import native, rasterize_batch
from gaussian_splatting_b200.densify import WeightStats
from gaussian_splatting_b200.pose import se3_exp
from gaussian_splatting_b200.rasterize import _depth_key_params, _lens_state, rasterize
from gaussian_splatting_b200.structs import Camera, Gaussians
from tests import scenes
from tests import shutter_oracle as so
from tests.scenes import headline_inputs
from tests.test_filter3d_oracle import live_filter
from tests.test_gradient_rows_gpu import gaussians_from

pytestmark = pytest.mark.gpu
BG = 0.5
LENSES = ("pinhole", "fisheye", "distortion")
LENS_K = {"pinhole": None, "fisheye": (0.08, -0.03, 0.01, -0.002), "distortion": (-0.12, 0.03, 5e-4, -3e-4, 0.01)}
MODES = {"plain": {}, "depth": dict(render_depth_alpha=True), "antialiased": dict(antialiased=True),
         "filter3d": dict(filter3d=True), "all": dict(render_depth_alpha=True, antialiased=True, filter3d=True)}
# |GPU - fp64 oracle| per gaussian parameter <= RTOL * (the largest |oracle| entry of its row); per camera entry
# <= RTOL * sum_i |contribution_i|.  The fp32 chain is that of the pose kernels (2^-13 there) plus the Newton solve,
# the shear and its VJP (some 10^2 more roundings), so 2^-11.
RTOL = 2.0 ** -11


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def bits(a):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return np.ascontiguousarray(a).view(np.uint8)


def lens_kw(lens, C=None):
    if lens == "pinhole":
        return {}
    k = LENS_K[lens]
    return {lens: k if C is None else [k] * C}


def scene(shd, n=600, view=2):
    return scenes.np_scene(n, "tiny", sh_degree=shd, seed=3, view=view, n_views=3, sigma_px=(0.8, 0.8, 0.15, 8.0))


def twist(sc, scale=1.0):
    """A readout motion that moves the image by about a tenth of its size: a pitch (along the lines), a yaw (across
    them), some roll and a translation of a few percent of the scene depth."""
    K, H, W = sc["K"], sc["H"], sc["W"]
    p = sc["xyz"] @ sc["T"][:3, :3].T + sc["T"][:3, 3]
    depth = float(np.median(p[:, 2]))
    w = np.array([0.1 * H / K[1, 1], 0.08 * W / K[0, 0], 0.03])
    r = 0.03 * depth * np.array([1.0, -0.7, 0.4])
    return torch.tensor(np.concatenate([r, w]) * scale, dtype=torch.float32, device=dev())


def _mode_bits(mode):
    ext = native()
    f = MODES[mode]
    return ((ext.MODE_DEPTH_ALPHA if f.get("render_depth_alpha") else 0)
            | (ext.MODE_ANTIALIASED if f.get("antialiased") else 0) | (ext.MODE_FILTER3D if f.get("filter3d") else 0))


def _native(sc, lens, mode, xi, readout, rows_seed=1, C=None, rows=None):
    """The shutter kernels through the bindings: forward, then the backward on seeded rows with the camera row.
    Single view (C None): xi [6]; batched: sc a list of C scenes sharing the gaussians, xi [C,6]."""
    ext = native()
    scs = [sc] if C is None else sc
    s0 = scs[0]
    xyz, q, s, o, rgb = (to_t(s0[k]) for k in ("xyz", "quaternion", "scale", "opacity", "rgb"))
    sh = None if s0["sh"] is None else to_t(s0["sh"])
    f3d = to_t(live_filter(s0)) if MODES[mode].get("filter3d") else None
    T = torch.stack([to_t(x["T"]) for x in scs]) if C is not None else to_t(s0["T"])
    K = torch.stack([to_t(x["K"]) for x in scs]) if C is not None else to_t(s0["K"])
    ro = None if xi is None else getattr(ext, "READOUT_" + readout.upper())
    return _run(xyz, q, s, o, rgb, sh, T, K, s0["H"], s0["W"], lens, _mode_bits(mode), f3d, xi, ro, rows_seed, C,
                rows)


def _run(xyz, q, s, o, rgb, sh, T, K, H, W, lens, md, f3d, xi, ro, rows_seed=1, C=None, rows=None):
    """forward + backward (camera_grads=1) through the bindings; xi None: the global-shutter (pose) kernels"""
    ext = native()
    N = xyz.shape[0]
    o = o.reshape(-1)
    cen = None
    if sh is not None:
        cen = torch.stack([ext.camera_centre(t) for t in T]) if C is not None else ext.camera_centre(T)
    lstate = _lens_state(None if lens == "pinhole" else (lens, LENS_K[lens] if C is None else [LENS_K[lens]] * C),
                         dev())
    lk = dict(lens=ext.LENS_PINHOLE, lens_consts=None) if lstate is None else dict(lens=lstate[0], lens_consts=lstate[1])
    sk = {} if xi is None else dict(rolling_shutter=xi, readout=ro)
    base, _ = _depth_key_params(0.3, 500.0)
    if C is None:
        fwd = ext.fused_preprocess_forward(xyz, None, q, s, o, rgb, sh, T, K, cen, H, W, 0.3, 500.0, 100.0, 3.0, base,
                                           True, md, f3d, **lk, **sk)
    else:
        fwd = ext.batch_preprocess_forward(xyz, None, q, s, o, rgb, sh, T, K, cen, H, W, 0.3, 500.0, 100.0, 3.0, base,
                                           md, f3d, **lk, **sk)
    records, visible = fwd[0], fwd[2]
    if rows is None:
        gen = torch.Generator().manual_seed(rows_seed)
        rows = (torch.randn(*((C,) if C else ()), N, 12, generator=gen) * 1e-2).to(dev())
    bwd = ext.batch_preprocess_backward if C else ext.fused_preprocess_backward
    if xi is not None:
        sk.update(height=H, width=W)
    out = bwd(rows.reshape(-1) if C is None else rows.reshape(C, -1), xyz, q, s, o, sh, T, K, cen, visible, None,
              None, None, True, md, f3d, **lk, camera_grads=1, **sk)
    n = 6 + (sh is not None)
    return dict(records=records, visible=visible, rows=rows, grads=out[:n - 1], g_pose=out[n],
                g_xi=out[n + 1] if xi is not None else None, f3d=f3d, all=out)


def _oracle(sc, lens, mode, xi, readout, rows, visible, f3d):
    idx = np.nonzero(visible.cpu().numpy())[0]
    d = lambda a: torch.from_numpy(np.asarray(a, np.float64)[idx]).clone().requires_grad_(True)  # noqa: E731
    xyz, q, s = d(sc["xyz"]), d(sc["quaternion"]), d(sc["scale"])
    o = torch.from_numpy(np.asarray(sc["opacity"], np.float64).reshape(-1)[idx]).clone().requires_grad_(True)
    n = len(idx)
    T = torch.from_numpy(np.asarray(sc["T"], np.float64)).expand(n, 4, 4).clone().requires_grad_(True)
    xi64 = xi.double().cpu().expand(n, 6).clone().requires_grad_(True)
    K = torch.from_numpy(np.asarray(sc["K"], np.float64))
    f = None if f3d is None else f3d.double().cpu()[idx]
    out = so.forward(lens, xyz, q, s, o, T, K, LENS_K[lens], xi64, readout, sc["H"], sc["W"],
                     antialiased=MODES[mode].get("antialiased", False), filter3d=f)
    r = rows.double().cpu()[idx]
    L = so.loss_from_rows(out, r, MODES[mode].get("render_depth_alpha", False))
    g = torch.autograd.grad(L, [xyz, q, s, o, T, xi64])
    return idx, out, g


def _check_param(got, want, name):
    got = got.double().cpu().reshape(want.shape[0], -1)
    want = want.reshape(want.shape[0], -1)
    scale = want.abs().max(1, keepdim=True).values + 1e-12 * want.abs().max()
    err = ((got - want).abs() / scale).max().item()
    assert err <= RTOL, (name, err)


def _check_camera(got, contrib, name):
    want, mass = contrib.sum(0), contrib.abs().sum(0)
    err = (got.double().cpu() - want).abs()
    assert (err <= RTOL * mass + 1e-12).all(), (name, (err / mass.clamp_min(1e-30)).max().item())


# ---- 1. the fp64 oracle on the GPU's own rows ---------------------------------------------------------------------
@pytest.mark.parametrize("readout", so.READOUTS)
@pytest.mark.parametrize("mode", ["plain", "depth", "antialiased", "filter3d"])
@pytest.mark.parametrize("shd", [0, 3])
@pytest.mark.parametrize("lens", LENSES)
def test_shutter_matches_the_fp64_oracle(lens, shd, mode, readout):
    sc = scene(shd)
    xi = twist(sc)
    r = _native(sc, lens, mode, xi, readout)
    idx, out, g = _oracle(sc, lens, mode, xi, readout, r["rows"], r["visible"], r["f3d"])
    assert len(idx) > 100 and int(out["clamped"].sum()) > 0, (len(idx), int(out["clamped"].sum()))
    rec = r["records"].double().cpu()[idx]
    uv_err = (rec[:, :2] - out["uv"].detach()).abs().max().item()
    assert uv_err < 2e-3, uv_err
    cov = torch.stack([rec[:, 4] - 0.25, rec[:, 5], rec[:, 6] - 0.25], 1)
    c_err = ((cov - out["conic"].detach()).abs() / out["conic"].detach().abs().max(1, keepdim=True).values).max()
    assert c_err.item() < 1e-3, c_err.item()
    assert out["residual"].max().item() < 1e-9
    for got, want, name in zip(r["grads"][:4], g[:4], ("xyz", "quaternion", "scale", "opacity")):
        _check_param(got[idx], want, name)
    _check_camera(r["g_pose"][:3].reshape(-1), g[4][:, :3].reshape(len(idx), -1), "pose")
    assert (r["g_pose"][3] == 0).all()
    _check_camera(r["g_xi"], g[5], "xi")


@pytest.mark.parametrize("lens", LENSES)
def test_batched_shutter_matches_the_oracle_and_the_single_views(lens):
    """Three views with per-view twists: view c's camera row against the oracle on view c's rows, and every output
    of view c bit-identical to the single-view kernels on the same rows."""
    C = 3
    scs = [scene(3, view=c) for c in range(C)]
    xi = torch.stack([twist(scs[c], 1.0 - 0.3 * c) for c in range(C)])
    r = _native(scs, lens, "all", xi, "top_to_bottom", C=C)
    for c in range(C):
        one = _native(scs[c], lens, "all", xi[c].contiguous(), "top_to_bottom", rows=r["rows"][c].contiguous())
        assert np.array_equal(bits(one["records"]), bits(r["records"][c]))
        assert torch.equal(one["visible"], r["visible"][c])
        assert np.array_equal(bits(one["g_pose"]), bits(r["g_pose"][c]))
        assert np.array_equal(bits(one["g_xi"]), bits(r["g_xi"][c]))
        idx, out, g = _oracle(scs[c], lens, "all", xi[c], "top_to_bottom", r["rows"][c], r["visible"][c], r["f3d"])
        _check_camera(r["g_pose"][c][:3].reshape(-1), g[4][:, :3].reshape(len(idx), -1), ("pose", c))
        _check_camera(r["g_xi"][c], g[5], ("xi", c))


# ---- 2. the global-shutter limit at the headline size --------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("lens", LENSES)
def test_zero_twist_is_the_global_shutter(lens, mode):
    """xi = 0 at 3M gaussians, 1080p, SH 3: image, mask, uv, depth / alpha and weight statistics bit-identical to the
    call without rolling_shutter; gaussian and pose gradients within 1e-6 of their largest entry."""
    H = 1080
    g0, cam, T0, G = headline_inputs(H, dev())
    flags = dict(MODES[mode])
    if flags.pop("filter3d", False):
        flags["filter3d"] = (torch.exp(g0.scale.detach().mean(1)) * 0.5).contiguous()
    res = []
    for xi in (None, torch.zeros(6, device=dev(), requires_grad=True)):
        for p in (g0.xyz, g0.quaternion, g0.scale, g0.opacity, g0.rgb, g0.sh):
            p.grad = None
        T = T0.clone().requires_grad_(True)
        ws = WeightStats(g0.xyz.shape[0], dev())
        out = rasterize(g0, T, cam, 0.3, 500.0, 100, 3.0, True, torch.full((3,), BG, device=dev()),
                        weight_stats=ws, rolling_shutter=xi, **lens_kw(lens), **flags)
        outs = [out[0], out[1], out[2]] + ([out[3], out[4]] if flags.get("render_depth_alpha") else [])
        ups = [G] + ([torch.full_like(out[3], 1e-7), torch.full_like(out[4], 1e-7)]
                     if flags.get("render_depth_alpha") else [])
        torch.autograd.backward([outs[0]] + outs[3:], ups)
        res.append(([o.detach().clone() for o in outs], [ws.weight_sum.clone(), ws.weight_max.clone(),
                                                         ws.pixel_count.clone()],
                    [p.grad.clone() for p in (g0.xyz, g0.quaternion, g0.scale, g0.opacity, g0.rgb, g0.sh)],
                    T.grad.clone(), None if xi is None else xi.grad.clone()))
    (o0, w0, g_0, t0, _), (o1, w1, g_1, t1, gx1) = res
    for a, b in zip(o0, o1):
        assert np.array_equal(bits(a), bits(b))
    assert np.array_equal(bits(w0[1]), bits(w1[1])) and torch.equal(w0[2], w1[2])
    assert torch.allclose(w0[0], w1[0], rtol=1e-5, atol=0)
    assert torch.isfinite(gx1).all()
    # the gradients on the same rows (two render backwards need not repeat bit for bit: fp32 atomics): the pose
    # kernels against the shutter kernels at xi = 0
    gd = g0.xyz.detach(), g0.quaternion.detach(), g0.scale.detach(), g0.opacity.detach(), g0.rgb.detach()
    args = (*gd, g0.sh.detach(), T0, cam.K, H, 1920, lens, _mode_bits(mode), flags.get("filter3d"))
    ref = _run(*args, None, None)
    sht = _run(*args, torch.zeros(6, device=dev()), native().READOUT_TOP_TO_BOTTOM)
    assert np.array_equal(bits(ref["records"]), bits(sht["records"]))
    for a, b in zip(list(ref["grads"]) + [ref["g_pose"]], list(sht["grads"]) + [sht["g_pose"]]):
        assert (a - b).abs().max() <= 1e-6 * a.abs().max(), ((a - b).abs().max().item(), a.abs().max().item())


# ---- 3. per-line ground truth --------------------------------------------------------------------------------------
def _small_scene(n=300, seed=5):
    rng = np.random.default_rng(seed)
    H, W = 64, 96
    K = np.array([[90.0, 0, 47.5], [0, 90.0, 31.5], [0, 0, 1]], np.float32)
    z = rng.uniform(3.0, 6.0, n)
    u, v = rng.uniform(-10, W + 10, n), rng.uniform(-10, H + 10, n)
    xyz = np.stack([(u - K[0, 2]) * z / K[0, 0], (v - K[1, 2]) * z / K[1, 1], z], 1).astype(np.float32)
    q = rng.standard_normal((n, 4)).astype(np.float32)
    s = np.log(rng.uniform(0.006, 0.012, (n, 3))).astype(np.float32)
    o = np.full((n, 1), 3.0, np.float32)
    rgb = rng.uniform(0, 2, (n, 3)).astype(np.float32)
    return dict(xyz=xyz, quaternion=q, scale=s, opacity=o, rgb=rgb, sh=None, T=np.eye(4, dtype=np.float32), K=K,
                H=H, W=W)


@pytest.mark.parametrize("motion", ["pan", "tilt"])
def test_rolling_shutter_matches_per_line_global_renders(motion):
    """Line k of the rolling-shutter image against line k of a global-shutter render at T(k / (H - 1)) (one batch of
    H views): at least 5x closer than the global render at the middle pose."""
    sc = _small_scene()
    H, W = sc["H"], sc["W"]
    w = [0.0, 0.12, 0.0] if motion == "pan" else [0.08, 0.0, 0.0]  # ~12 / 8 % of the image over the readout
    xi = torch.tensor([0.0, 0.0, 0.0] + w, device=dev())
    g = gaussians_from(sc)
    cam = Camera(W, H, to_t(sc["K"]))
    T = to_t(sc["T"])
    bg = torch.full((3,), BG, device=dev())
    with torch.no_grad():
        rs = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, rolling_shutter=xi)[0]
        gs = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg)[0]
        taus = torch.arange(H, device=dev(), dtype=torch.float32) / (H - 1)
        Ts = se3_exp((taus - 0.5)[:, None] * xi[None]) @ T
        per = rasterize_batch(g, Ts.contiguous(), cam, 0.3, 500.0, 100, 3.0, True, bg)[0]
        truth = per[torch.arange(H), torch.arange(H)]
    e_rs = (rs - truth).norm().item()
    e_gs = (gs - truth).norm().item()
    assert e_rs * 5 <= e_gs, (motion, e_rs, e_gs)


# ---- 4. invariance and determinism -----------------------------------------------------------------------------------
@pytest.mark.parametrize("lens", LENSES)
def test_outputs_do_not_depend_on_which_camera_inputs_require_grad_and_rows_repeat(lens):
    sc = scene(3)
    xi = twist(sc)
    a = _native(sc, lens, "all", xi, "left_to_right")
    b = _native(sc, lens, "all", xi, "left_to_right")
    for k in ("records", "visible", "g_pose", "g_xi"):
        assert np.array_equal(bits(a[k]), bits(b[k])), k
    for x, y in zip(a["grads"], b["grads"]):
        assert np.array_equal(bits(x), bits(y))
    outs = []
    for xg, pg in ((False, False), (True, False), (False, True), (True, True)):
        g = gaussians_from(sc)
        T = to_t(sc["T"]).requires_grad_(pg)
        x = xi.clone().requires_grad_(xg)
        out = rasterize(g, T, Camera(sc["W"], sc["H"], to_t(sc["K"])), 0.3, 500.0, 100, 3.0, True,
                        torch.full((3,), BG, device=dev()), render_depth_alpha=True, rolling_shutter=x,
                        **lens_kw(lens))
        outs.append([o.detach().clone() for o in out])
    for o in outs[1:]:
        for p, q in zip(outs[0], o):
            assert np.array_equal(bits(p), bits(q))


# ---- 5. recovery of a known readout motion -------------------------------------------------------------------------
RECOVERY_STEPS = 300


def test_adam_recovers_a_known_readout_motion():
    """Targets rendered with xi* (about 1 degree of pan plus a small translation over the readout); xi alone is
    optimised from 0 with the gaussians fixed."""
    sc = _small_scene(600, seed=7)
    g = Gaussians(*(to_t(sc[k]) for k in ("xyz", "rgb", "opacity", "scale", "quaternion")), None)
    cam = Camera(sc["W"], sc["H"], to_t(sc["K"]))
    T = to_t(sc["T"])
    bg = torch.full((3,), BG, device=dev())
    star = torch.tensor([0.02, -0.01, 0.0, 0.004, 0.0175, 0.002], device=dev())
    with torch.no_grad():
        target = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, rolling_shutter=star)[0]
    xi = torch.zeros(6, device=dev(), requires_grad=True)
    opt = torch.optim.Adam([xi], lr=2e-3)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, RECOVERY_STEPS)
    losses = []
    for _ in range(RECOVERY_STEPS):
        opt.zero_grad()
        img = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, rolling_shutter=xi)[0]
        loss = ((img - target) ** 2).mean()
        loss.backward()
        opt.step()
        sched.step()
        losses.append(loss.item())
    w_err = (xi[3:] - star[3:]).norm().item() / star[3:].norm().item()
    assert w_err < 0.1, (w_err, xi.tolist(), losses[0], losses[-1])
    assert losses[-1] < 1e-2 * losses[0], (losses[0], losses[-1])


# ---- 6. edge cases --------------------------------------------------------------------------------------------------
def test_empty_off_image_and_lambda_max_scenes():
    sc = scene(0)
    xi = twist(sc)
    # N = 0
    empty = {k: (v[:0] if isinstance(v, np.ndarray) and k != "T" and k != "K" else v) for k, v in sc.items()}
    r = _native(empty, "pinhole", "plain", xi, "top_to_bottom")
    assert r["visible"].numel() == 0 and (r["g_xi"] == 0).all() and (r["g_pose"] == 0).all()
    # every gaussian off the image (tau* clamped): nothing visible, zero camera gradients
    far = dict(sc)
    far["xyz"] = sc["xyz"] + np.array([1e3, 0, 0], np.float32)
    r = _native(far, "pinhole", "plain", xi, "top_to_bottom")
    assert int(r["visible"].sum()) == 0 and (r["g_xi"] == 0).all() and (r["g_pose"] == 0).all()
    # a readout motion faster than the readout along the lines (a negative pitch moves the image down the lines,
    # with the readout): lambda >= 3/4 culls
    fast = torch.tensor([0.0, 0.0, 0.0, -3.0 * sc["H"] / sc["K"][1, 1], 0.0, 0.0], device=dev())
    r0 = _native(sc, "pinhole", "plain", xi, "top_to_bottom")
    r1 = _native(sc, "pinhole", "plain", fast, "top_to_bottom")
    assert int(r1["visible"].sum()) < int(r0["visible"].sum()) // 4


def test_absgrad_and_features_with_rolling_shutter():
    sc = scene(0)
    xi = twist(sc).requires_grad_(True)
    g = gaussians_from(sc)
    cam = Camera(sc["W"], sc["H"], to_t(sc["K"]))
    bg = torch.full((3,), BG, device=dev())
    out = rasterize(g, to_t(sc["T"]), cam, 0.3, 500.0, 100, 3.0, True, bg, absgrad=True, rolling_shutter=xi)
    out[0].square().sum().backward()
    assert out[2].absgrad.shape == out[2].shape and (out[2].absgrad >= 0).all()
    assert torch.isfinite(xi.grad).all() and xi.grad.abs().sum() > 0
    F = torch.randn(sc["xyz"].shape[0], 5, device=dev(), requires_grad=True)
    x2 = twist(sc).requires_grad_(True)
    out = rasterize(g, to_t(sc["T"]), cam, 0.3, 500.0, 100, 3.0, True, bg, features=F, rolling_shutter=x2)
    (out[0].sum() + out[3].square().sum()).backward()
    assert F.grad.abs().sum() > 0 and x2.grad.abs().sum() > 0
