"""rasterize_batch on the GPU: every view bit-identical to rasterize, the batched per-gaussian backward bit-identical
to the view-order sum of single-view backwards, and end-to-end gradients equal to a loop of rasterize calls within
the atomics noise — needs an H100."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import rasterize as R
from gaussian_splatting_b200 import native, synth
from gaussian_splatting_b200.densify import DensificationStats
from gaussian_splatting_b200.rasterize import rasterize, rasterize_batch
from gaussian_splatting_b200.structs import Camera, Gaussians
from tests import scenes

pytestmark = pytest.mark.gpu

# the scenes of test_features_gpu.py's GOLDEN (tiny, small, deep) and a 720p one
SCENES = {"tiny": (2000, "tiny", (2.0, 0.5, 0.5, 8.0)), "small": (12000, "small", (2.5, 0.5, 0.5, 10.0)),
          "deep": (60000, "small", (2.5, 0.5, 0.5, 10.0)), "720p": (200_000, "720p", (1.2, 0.6, 0.3, 12.0))}
SH_DEGREE = {"tiny": 3, "small": 1, "deep": 0, "720p": 2}


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy()


def scene(name, sh_degree=None):
    if name == "exact":   # most warps recomputed with the exact arithmetic (tests/scenes.py FLAGGED)
        return scenes.flagged_scene("exact huge")
    n, res, sig = SCENES[name]
    sc = scenes.np_scene(n, res, sh_degree=SH_DEGREE[name] if sh_degree is None else sh_degree, seed=0, view=0,
                         n_views=3, sigma_px=sig)
    if (SH_DEGREE[name] if sh_degree is None else sh_degree) == 0:
        sc["sh"] = None
    return sc


def gaussians(sc):
    P = {k: to_t(sc[k]).requires_grad_(True) for k in ("xyz", "rgb", "opacity", "scale", "quaternion")}
    sh = None if sc["sh"] is None else to_t(sc["sh"]).requires_grad_(True)
    return Gaussians(P["xyz"], P["rgb"], P["opacity"], P["scale"], P["quaternion"], sh)


def poses(C, away=()):
    T = torch.stack([synth.make_pose(c, max(C, 2), device=dev()) for c in range(C)])
    for c in away:  # looks the other way: sees nothing
        T[c, 2, :3] *= -1.0
        T[c, 0, :3] *= -1.0
        T[c, 2, 3] = -T[c, 2, 3] - 50.0
    return T.contiguous()


def exact_views(sc, C):
    """C views of the "exact" scene that keep its exact centres on pixel centres: the identity pose, the principal
    point moved by whole pixels per view."""
    T = torch.eye(4, device=dev()).expand(C, 4, 4).contiguous()
    K = to_t(sc["K"]).expand(C, 3, 3).clone()
    for c in range(C):
        K[c, 0, 2] += c
        K[c, 1, 2] -= 2 * c
    return T, K


def intrinsics(sc, C, distinct):
    K = to_t(sc["K"])
    if not distinct:
        return K
    Ks = K.expand(C, 3, 3).clone()
    for c in range(C):
        Ks[c, 0, 0] *= 1.0 + 0.03 * c
        Ks[c, 1, 2] += 0.5 * c
    return Ks


def backgrounds(C, per_view):
    if not per_view:
        return torch.full((3,), 0.25, device=dev())
    return torch.rand(C, 3, generator=torch.Generator().manual_seed(C)).to(dev())


def grads_of(g):
    return {k: getattr(g, k).grad.clone() for k in ("xyz", "rgb", "opacity", "scale", "quaternion", "sh")
            if getattr(g, k) is not None}


def run_loop(sc, T, K, bg, H, W, G=None, **kw):
    g = gaussians(sc)
    C = T.shape[0]
    outs = []
    for c in range(C):
        Kc = K if K.dim() == 2 else K[c]
        bgc = bg if bg.dim() == 1 else bg[c]
        o = rasterize(g, T[c].contiguous(), Camera(W, H, Kc.contiguous()), 0.3, 500.0, 100, 3.0, True,
                      bgc.contiguous(), return_state=True, **kw)
        o[2].retain_grad()
        outs.append(o)
    if G is not None:
        loss = sum((o[0] * G[c]).sum() + sum((m * G[c][..., :1]).sum() for m in o[3:-1]) for c, o in enumerate(outs))
        loss.backward()
    return g, outs


def run_batch(sc, T, K, bg, H, W, G=None, **kw):
    g = gaussians(sc)
    o = rasterize_batch(g, T, Camera(W, H, K), 0.3, 500.0, 100, 3.0, True, bg, return_state=True, **kw)
    for u in o[2]:
        u.retain_grad()
    if G is not None:
        loss = (o[0] * G).sum() + sum((m * G[..., :1]).sum() for m in o[3:-1])
        loss.backward()
    return g, o


def upstream(C, H, W, seed=3):
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(C, H, W, 3, generator=gen) / (H * W)).to(dev())


def check_forward_equal(loop, batch, depth_alpha):
    _, l_outs = loop
    _, b = batch
    images, mask, uvs = b[:3]
    st = b[-1]
    for c, o in enumerate(l_outs):
        assert np.array_equal(bits(images[c]), bits(o[0])), c
        assert torch.equal(mask[c], o[1]), c
        assert uvs[c].shape == o[2].shape and np.array_equal(bits(uvs[c]), bits(o[2])), c
        v, s = st.views[c], o[-1]
        assert torch.equal(v.n_per_pixel, s.n_per_pixel) and np.array_equal(bits(v.w_per_pixel), bits(s.w_per_pixel))
        assert torch.equal(v.vis_idx32, s.vis_idx32) and torch.equal(v.ranges, s.ranges)
        if depth_alpha:
            assert np.array_equal(bits(b[3][c]), bits(o[3])) and np.array_equal(bits(b[4][c]), bits(o[4])), c


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


# 1. per-view forward parity ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("name", ["tiny", "small", "deep", "exact"])
def test_every_view_is_bit_identical_to_rasterize(name, C):
    sc = scene(name)
    H, W = sc["H"], sc["W"]
    T, K = exact_views(sc, C) if name == "exact" else (poses(C), intrinsics(sc, C, C > 1))
    bg = backgrounds(C, C > 2)
    check_forward_equal(run_loop(sc, T, K, bg, H, W), run_batch(sc, T, K, bg, H, W), False)


@pytest.mark.parametrize("size", [(50, 37), (17, 33), (1080, 1920), (720, 1280)])
def test_odd_and_large_image_sizes(size):
    H, W = size
    sc = scene("720p" if H >= 720 else "tiny")
    K = to_t(sc["K"]).clone()
    K[0, 2], K[1, 2] = W / 2.0, H / 2.0
    T, bg = poses(3), backgrounds(3, True)
    check_forward_equal(run_loop(sc, T, K, bg, H, W), run_batch(sc, T, K, bg, H, W), False)


@pytest.mark.parametrize("masks", [True, False])
@pytest.mark.parametrize("absgrad", [False, True])
@pytest.mark.parametrize("filter3d", [False, True])
@pytest.mark.parametrize("antialiased", [False, True])
@pytest.mark.parametrize("depth_alpha", [False, True])
def test_modes_forward_and_gradients(depth_alpha, antialiased, filter3d, absgrad, masks):
    sc = scene("small")
    H, W, C = sc["H"], sc["W"], 3
    T, K, bg = poses(C, away=(1,)), intrinsics(sc, C, True), backgrounds(C, True)
    f3d = torch.full((sc["xyz"].shape[0],), 0.004, device=dev()) if filter3d else None
    kw = dict(render_depth_alpha=depth_alpha, antialiased=antialiased, filter3d=f3d, absgrad=absgrad)
    G = upstream(C, H, W)
    R.USE_CONTRIBUTION_MASKS = masks
    try:
        loop = run_loop(sc, T, K, bg, H, W, G, **kw)
        loop2 = run_loop(sc, T, K, bg, H, W, G, **kw)
        batch = run_batch(sc, T, K, bg, H, W, G, **kw)
    finally:
        R.USE_CONTRIBUTION_MASKS = True
    check_forward_equal(loop, batch, depth_alpha)
    assert batch[1][2][1].shape[0] == 0 and bool(batch[1][1][1].all())  # the view that sees nothing
    compare_gradients(loop, loop2, batch, absgrad)


def compare_gradients(loop, loop2, batch, absgrad=False):
    """Within 10x the spread of two runs of the single-view path (and never looser than 1e-5 of the largest value:
    the render backward's atomics order is the only difference)."""
    gl, gl2, gb = grads_of(loop[0]), grads_of(loop2[0]), grads_of(batch[0])
    for k in gl:
        tol = max(1e-5, 10 * rel(gl2[k], gl[k]))
        assert rel(gb[k], gl[k]) <= tol, (k, rel(gb[k], gl[k]), tol)
    for c, o in enumerate(loop[1]):
        u_b, u_l, u_l2 = batch[1][2][c], o[2], loop2[1][c][2]
        if u_l.shape[0] == 0:
            continue
        assert rel(u_b.grad, u_l.grad) <= max(1e-5, 10 * rel(u_l2.grad, u_l.grad)), c
        if absgrad:
            assert rel(u_b.absgrad, u_l.absgrad) <= max(1e-5, 10 * rel(u_l2.absgrad, u_l.absgrad)), c


# 3. the batched per-gaussian backward, bitwise ---------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["plain", "depth", "aa", "f3d", "depth_aa_f3d"])
@pytest.mark.parametrize("sh_degree", [0, 1, 2, 3])
def test_batched_per_gaussian_backward_is_the_view_order_sum(sh_degree, mode):
    ext = native()
    sc = scene("small", sh_degree=sh_degree)
    g = gaussians(sc)
    N, C = sc["xyz"].shape[0], 4
    T, K = poses(C), intrinsics(sc, C, True)
    bits_ = {"plain": 0, "depth": ext.MODE_DEPTH_ALPHA, "aa": ext.MODE_ANTIALIASED, "f3d": ext.MODE_FILTER3D,
             "depth_aa_f3d": ext.MODE_DEPTH_ALPHA | ext.MODE_ANTIALIASED | ext.MODE_FILTER3D}[mode]
    f3d = torch.rand(N, generator=torch.Generator().manual_seed(2)).to(dev()) * 0.01 if bits_ & ext.MODE_FILTER3D \
        else None
    sh = None if g.sh is None else g.sh.detach()
    centre = None if sh is None else torch.stack([ext.camera_centre(T[c]) for c in range(C)])
    with torch.no_grad():
        fw = ext.batch_preprocess_forward(g.xyz, None, g.quaternion, g.scale, g.opacity.reshape(-1), g.rgb, sh, T, K,
                                          centre, sc["H"], sc["W"], 0.3, 500.0, 100.0, 3.0, 0, bits_, f3d)
    visible, scan = fw[2], fw[3]
    rows = torch.randn(C, N * 12, generator=torch.Generator().manual_seed(7)).to(dev())
    M_tot = int((scan[:, -1] >> 32).sum())
    guv = torch.randn(M_tot, 2, generator=torch.Generator().manual_seed(8)).to(dev())
    Ms = (scan[:, -1] >> 32).tolist()
    for use_uv in (False, True):
        args = (g.xyz.detach(), g.quaternion.detach(), g.scale.detach(), g.opacity.detach().reshape(-1), sh)
        got = ext.batch_preprocess_backward(rows, *args, T, K, centre, visible, None, guv if use_uv else None,
                                            scan if use_uv else None, not use_uv, bits_, f3d)[-1]
        want, off = None, 0
        for c in range(C):
            gc = guv[off:off + Ms[c]].contiguous() if use_uv else None
            one = ext.fused_preprocess_backward(rows[c].contiguous(), *args, T[c].contiguous(), K[c].contiguous(),
                                                None if centre is None else centre[c].contiguous(),
                                                visible[c].contiguous(), None, gc, scan[c].contiguous() if use_uv
                                                else None, not use_uv, bits_, f3d)[-1]
            off += Ms[c]
            want = one.clone() if want is None else want + one
        # equal up to the sign of zero
        assert torch.equal(got, want), int((got != want).sum())
        assert float(got.abs().max()) > 0


# 4-6. gradients, speculation, densification statistics -------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 2, 4])
@pytest.mark.parametrize("name", ["tiny", "small", "exact"])
def test_gradients_equal_the_loop_within_the_atomics_noise(name, C):
    sc = scene(name)
    H, W = sc["H"], sc["W"]
    T, K = exact_views(sc, C) if name == "exact" else (poses(C), intrinsics(sc, C, True))
    bg = backgrounds(C, True)
    G = upstream(C, H, W)
    loop, loop2, batch = (run_loop(sc, T, K, bg, H, W, G), run_loop(sc, T, K, bg, H, W, G),
                          run_batch(sc, T, K, bg, H, W, G))
    compare_gradients(loop, loop2, batch)
    st = batch[1][-1]
    assert st.grad_flat is not None and st.grad_flat.data_ptr() == batch[0].xyz.grad.data_ptr()


def test_speculation_paths_no_grad_and_grad_out_give_the_same_bits(monkeypatch):
    sc = scene("small")
    H, W, C = sc["H"], sc["W"], 4
    T, K, bg = poses(C), intrinsics(sc, C, True), backgrounds(C, True)
    N = sc["xyz"].shape[0]
    key = (0, N, H, W, C)
    R._PAIR_HISTORY.pop(key, None)
    eager = run_batch(sc, T, K, bg, H, W)                      # first call: eager counts
    fitting = run_batch(sc, T, K, bg, H, W)                    # sized from the history
    assert not fitting[1][-1].speculation_overflowed
    monkeypatch.setattr(R, "_pair_capacity", lambda key: 128)  # far too small a guess: overflow and rerun
    over = run_batch(sc, T, K, bg, H, W)
    monkeypatch.undo()
    assert over[1][-1].speculation_overflowed
    for other in (fitting, over):
        assert np.array_equal(bits(other[1][0]), bits(eager[1][0]))
        for c in range(C):
            assert np.array_equal(bits(other[1][2][c]), bits(eager[1][2][c]))
    with torch.no_grad():
        g = gaussians(sc)
        img = rasterize_batch(g, T, Camera(W, H, K), 0.3, 500.0, 100, 3.0, True, bg)[0]
    assert np.array_equal(bits(img), bits(eager[1][0]))
    G = upstream(C, H, W)
    g = gaussians(sc)
    n_rest = 0 if g.sh is None else g.sh.shape[2]
    out = torch.full((native().flat_section_ends(N, n_rest)[-1],), float("nan"), device=dev())
    img = rasterize_batch(g, T, Camera(W, H, K), 0.3, 500.0, 100, 3.0, True, bg, grad_out=out)[0]
    (img * G).sum().backward()
    assert g.xyz.grad.data_ptr() == out.data_ptr() and torch.isfinite(out).all()


def test_densification_statistics_per_view_equal_the_loop():
    sc = scene("small")
    H, W, C = sc["H"], sc["W"], 3
    T, K, bg = poses(C), intrinsics(sc, C, True), backgrounds(C, False)
    G = upstream(C, H, W)
    N = sc["xyz"].shape[0]
    loop = run_loop(sc, T, K, bg, H, W, G, absgrad=True)
    batch = run_batch(sc, T, K, bg, H, W, G, absgrad=True)
    for absgrad in (False, True):
        s_l, s_b = DensificationStats(N, dev()), DensificationStats(N, dev())
        for c in range(C):
            o = loop[1][c]
            s_l.accumulate(o[-1], o[2], loop[0].xyz, K[c], absgrad=absgrad)
            s_b.accumulate(batch[1][-1].views[c], batch[1][2][c], batch[0].xyz, K[c], absgrad=absgrad)
        assert torch.equal(s_l.grad_accum_count, s_b.grad_accum_count)
        assert rel(s_b.uv_grad_accum, s_l.uv_grad_accum) < 1e-4


def test_empty_scene():
    sc = scene("tiny")
    for k in ("xyz", "rgb", "opacity", "scale", "quaternion", "sh"):
        sc[k] = sc[k][:0]
    H, W, C = sc["H"], sc["W"], 2
    T, K, bg = poses(C), intrinsics(sc, C, False), backgrounds(C, True)
    batch = run_batch(sc, T, K, bg, H, W, upstream(C, H, W))
    check_forward_equal(run_loop(sc, T, K, bg, H, W), batch, False)
    g, o = batch
    assert o[1].shape == (C, 0) and all(u.shape == (0, 2) for u in o[2]) and g.xyz.grad.shape == (0, 3)


# 2 and 7. sorted pairs on both key paths; the headline scene ---------------------------------------------------------
@pytest.mark.parametrize("far", [500.0, float("inf")])
def test_pair_lists_equal_the_single_view_ones(far):
    """far = 500: packed (tile | depth | id) keys; far = inf at 1.2 M gaussians: 32-bit depth keys leave no room for
    the id, and the pairs take the key/value sort."""
    H, W, C = 720, 1280, 8
    g = synth.make_gaussians(200_000 if far == 500.0 else 1_200_000, "720p", sh_degree=0, seed=0, device=dev())
    K, T, bg = synth.make_camera("720p", device=dev()).K, poses(C), backgrounds(C, False)
    with torch.no_grad():
        b = rasterize_batch(g, T, Camera(W, H, K), 0.3, far, 100, 3.0, True, bg, return_state=True)
        for c in range(C):
            s = rasterize(g, T[c].contiguous(), Camera(W, H, K), 0.3, far, 100, 3.0, True, bg, return_state=True)
            v = b[-1].views[c]
            assert v.P == s[-1].P and v.id_bits == s[-1].id_bits
            assert torch.equal(v.ids_sorted, s[-1].ids_sorted) and torch.equal(v.ranges, s[-1].ranges)
            assert np.array_equal(bits(b[0][c]), bits(s[0]))
    assert (b[-1].views[0].id_bits == 0) == (far == float("inf"))


def test_headline_scene_four_views():
    g, cam, _, _ = scenes.headline_inputs(1080, dev())
    T = torch.stack([synth.make_pose(v, 8, device=dev()) for v in range(4)])
    bg = torch.zeros(3, device=dev())
    imgs = rasterize_batch(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg)[0]
    imgs.sum().backward()
    torch.cuda.synchronize()
    with torch.no_grad():
        for c in range(4):
            img = rasterize(g, T[c].contiguous(), cam, 0.3, 500.0, 100, 3.0, True, bg)[0]
            assert np.array_equal(bits(imgs[c]), bits(img)), c
    assert torch.isfinite(g.xyz.grad).all()
