"""Every gaussian's gradient against the fp64 CPU oracle, row by row (tests/gradrows.py) — needs an H100.

The fused path is checked in two stages.  The render-stage slab the tile renderer's backward hands to the
per-gaussian backward (rgb, opacity, uv, conic sums per gaussian) is captured on its way through autograd and held
to c * eps * mass per entry.  That same slab, in double, is fed to the oracle's per-gaussian VJP, and the result is
compared with the parameter gradients the per-gaussian backward made from it.  rasterize_unfused is checked the same
way through the gradients its RenderImage node hands back, and the per-pixel SH (generic) kernels are fed the
oracle's own per-gaussian inputs and tile lists.

A pixel where the oracle and the GPU can skip different splats (an alpha within rounding of the 1/255 threshold:
exp2f against ex2.approx) would spread that difference into the gradient of every gaussian in its walk.  Such
pixels get no upstream gradient in either backward pass: those whose forward colour or final transmittance differs,
and those the oracle's backward reports as meeting an alpha near the threshold (at most 1 % of the image).
"""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import cuda_autograd_functions as af
from gaussian_splatting_b200 import rasterize as R
from gaussian_splatting_b200.rasterize import rasterize, rasterize_unfused
from gaussian_splatting_b200.structs import Camera, Gaussians
from oracle import cpu_oracle as orc
from tests import gradrows, scenes
from tests.gradrows import PARAM_FLOOR, PARAM_RTOL, RENDER_C

pytestmark = pytest.mark.gpu
BG = 0.5
FIELDS = ("rgb", "opacity", "uv", "conic")
PARAMS = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def to_np(t):
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def gaussians_from(sc):
    P = {k: to_t(sc[k]).requires_grad_(True) for k in ("xyz", "rgb", "opacity", "scale", "quaternion")}
    sh = None if sc["sh"] is None else to_t(sc["sh"]).requires_grad_(True)
    return Gaussians(P["xyz"], P["rgb"], P["opacity"], P["scale"], P["quaternion"], sh)


def view_dirs(sc):
    from gaussian_splatting_b200.utils import compute_rays_in_world_frame

    return compute_rays_in_world_frame(Camera(sc["W"], sc["H"], torch.from_numpy(sc["K"])),
                                       torch.from_numpy(sc["T"])).numpy()


def oracle_forward(sc, per_pixel=False):
    return orc.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], sc["K"],
                         sc["H"], sc["W"], 0.3, 500.0, 100.0, 3.0, background=np.full(3, BG, sc["xyz"].dtype),
                         use_sh_precompute=not per_pixel, view_dirs=view_dirs(sc) if per_pixel else None)


def upstream(sc, seed=1):
    H, W = sc["H"], sc["W"]
    G = np.random.default_rng(seed).standard_normal((H, W, 3)) / (3.0 * H * W)
    return G.astype(sc["xyz"].dtype)


def check_forward(image, o, mask=None, uv=None):
    """The forward criterion of test_against_cpu_oracle.  Returns the pixels to leave out of the backward: those whose
    colour or final transmittance differs beyond rounding (a threshold flip)."""
    if mask is not None:
        assert (to_np(mask) == o.culling_mask).all(), "culling mask differs from the oracle"
        assert gradrows.global_rel(to_np(uv), o.uv) < 1e-6
    img = to_np(image).astype(np.float64)
    diff = np.abs(img - o.image).max(2)
    bad = diff > 1e-4 * np.abs(o.image).max()
    assert int(bad.sum()) <= max(3, bad.size // 100_000), f"{int(bad.sum())} pixels beyond 1e-4"
    return bad


def flip_pixels(bad_image, w_gpu, o, G):
    """Pixels left out of the backward: forward colour or (when the GPU's is at hand) final transmittance beyond
    rounding, at most max(3, H*W / 10^5) like the forward criterion, and pixels whose walk in the oracle's backward
    meets an alpha near the 1/255 threshold, at most 1 % of the image."""
    forward = bad_image.copy()
    if w_gpu is not None:
        forward |= np.abs(to_np(w_gpu).astype(np.float64) - o.wlast) > 1e-4
    near = orc.rasterize_backward(o, G).near
    print(f"pixels left out: {int(forward.sum())} forward, {int(near.sum())} near the threshold, of {near.size}")
    assert int(forward.sum()) <= max(3, forward.size // 100_000), f"{int(forward.sum())} pixels differ in the forward"
    assert int(near.sum()) <= max(3, near.size // 100), f"{int(near.sum())} pixels near the threshold"
    return forward | near


def split_slab(slab, N):
    v = slab.view(N, 12)   # interleaved rows: rgb3 opa | uv2 conic0 conic1 | conic2 pad3
    return dict(rgb=v[:, 0:3], opacity=v[:, 3], uv=v[:, 4:6], conic=v[:, 6:9])


def render_results(tag, mine, d, keep, eps, allowed):
    return [gradrows.render_rows(f"{tag} render {k}", mine[k], getattr(d.render, k)[keep], getattr(d.mass, k)[keep],
                                 RENDER_C[k], eps, allowed) for k in FIELDS]


def param_results(tag, g, pr, allowed):
    return [gradrows.param_rows(f"{tag} {k}", getattr(g, k).grad, getattr(pr, k), PARAM_RTOL, PARAM_FLOOR, allowed)
            for k in PARAMS if getattr(g, k) is not None]


def fused_vs_oracle(tag, sc, G=None, masks=True, check=True, zero_block=None):
    """Fused forward + backward; returns (results, oracle forward, state).  zero_block: (rows, cols) slices where
    the GPU's upstream gradient is zeroed but the oracle's is not (a negative control)."""
    o = oracle_forward(sc)
    G = upstream(sc) if G is None else G
    R.USE_CONTRIBUTION_MASKS = masks
    try:
        g = gaussians_from(sc)
        cam = Camera(sc["W"], sc["H"], to_t(sc["K"]))
        image, mask, uv, st = rasterize(g, to_t(sc["T"]), cam, 0.3, 500.0, 100, 3.0, True,
                                        torch.full((3,), BG, device=dev()), return_state=True)
        flips = flip_pixels(check_forward(image, o, mask, uv), st.w_per_pixel, o, G)
        G = np.where(flips[:, :, None], 0, G).astype(np.float32)
        G_gpu = G.copy()
        if zero_block is not None:
            G_gpu[zero_block] = 0
        proj = next(f for f, i in image.grad_fn.next_functions if f is not None and i == 1)
        seen = []
        proj.register_prehook(lambda grad_outputs: seen.append(grad_outputs[1].detach().clone()))
        image.backward(to_t(G_gpu))
    finally:
        R.USE_CONTRIBUTION_MASKS = True
    assert len(seen) == 1 and (st.masks.numel() > 0) == masks
    slab = {k: v.double().cpu().numpy() for k, v in split_slab(seen[0], st.N).items()}
    d = orc.rasterize_backward(o, G)
    M = int(o.keep.sum())
    allowed = gradrows.flips_allowed(M)
    eps = gradrows.EPS[np.dtype(np.float32)]
    res = render_results(tag, slab, d, slice(None), eps, allowed)
    pr = orc.project_backward(o, slab["rgb"], slab["opacity"], slab["uv"], slab["conic"])
    res += param_results(tag, g, pr, allowed)
    for k in PARAMS:   # and the end-to-end gradient against the oracle's whole chain, globally
        if getattr(g, k) is not None and zero_block is None:
            assert gradrows.global_rel(getattr(g, k).grad, getattr(d, k)) < 5e-4, (tag, k)
    if check:
        gradrows.assert_all(res)
    return res, o, st


def np_scene(n, res, shd, seed=1, **kw):
    return scenes.np_scene(n, res, sh_degree=shd, seed=seed, view=2, n_views=3, **kw)


def ragged(H, W, shd):
    sc = np_scene(3000, "tiny", shd, seed=2, sigma_px=(2.0, 0.5, 0.5, 8.0))
    sc["H"], sc["W"] = H, W
    sc["K"] = sc["K"].copy()
    sc["K"][0, 2], sc["K"][1, 2] = W / 2.0, H / 2.0
    return sc


def stack(n, opacity_logit, shd=0, dtype=np.float32, seed=0, spread=0.3, scale=(0.1, 0.3)):
    """n splats stacked on the image centre, all at the same opacity."""
    rng = np.random.default_rng(seed)
    sc = scenes.np_scene(n, "tiny", sh_degree=shd, seed=seed, dtype=dtype)
    sc["xyz"] = np.stack([rng.uniform(-spread, spread, n), rng.uniform(-spread, spread, n), rng.uniform(2, 9, n)],
                         1).astype(dtype)
    sc["scale"] = np.log(rng.uniform(*scale, (n, 3))).astype(dtype)
    sc["opacity"] = np.full((n, 1), opacity_logit, dtype)
    return sc


# ------------------------------------------------------------------------------------------------
# fused path
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shd", [0, 1, 2, 3])
def test_fused_sh_degrees(shd):
    sc = np_scene(2000, "tiny", shd, sigma_px=(2.0, 0.5, 0.5, 8.0))
    assert (sc["sh"] is None) == (shd == 0) and (shd == 0 or sc["sh"].shape[2] == (shd + 1) ** 2 - 1)
    fused_vs_oracle(f"sh{shd}", sc)


@pytest.mark.parametrize("H,W,shd", [(50, 37, 1), (17, 33, 2), (1, 64, 0), (64, 1, 3)])
def test_fused_ragged_sizes(H, W, shd):
    """Odd widths (the second pixel of a lane's pair lies outside the image), partial 4x4 lane blocks, 1-pixel
    strips."""
    sc = ragged(H, W, shd)
    assert W % 2 == 1 or min(H, W) == 1
    assert H % 4 or W % 4
    _, o, _ = fused_vs_oracle(f"{H}x{W}", sc)
    assert int(o.keep.sum()) > 100 and (o.n > 0).any()


def test_fused_720p_100k():
    sc = np_scene(100_000, "720p", 3, seed=0)
    _, o, _ = fused_vs_oracle("720p", sc)
    assert int(o.keep.sum()) > 50_000


@pytest.mark.parametrize("masks", [True, False])
@pytest.mark.parametrize("shd", [0, 3])
def test_fused_deep_tile_variants(masks, shd):
    """Walks of more than 960 splats over several 128-record batches, with contribution-mask bits in all four
    words of a batch; both backward variants (masks on / off) against the oracle, with plain and SH colours."""
    sc = stack(3000, -5.0, shd=shd)
    _, o, st = fused_vs_oracle(f"deep masks={masks} sh{shd}", sc, masks=masks)
    assert int(o.n.max()) > 960 and int(np.diff(o.ranges).max()) > 4 * 128
    if masks:
        words = st.masks.view(-1, 4)
        assert bool((words != 0).any(0).all()), "some word of the 128-bit masks is never used"


@pytest.mark.parametrize("masks", [True, False])
@pytest.mark.parametrize("name", list(scenes.FLAGGED))
def test_fused_flagged_pixels(name, masks):
    """Scenes whose pixels the forward recomputes with the exact arithmetic (tests/scenes.py FLAGGED): every warp
    ("all") or single pixels among walked ones ("scattered").  The image and the final weights come from the
    recompute, the contribution masks the masked backward walks from the walk itself."""
    fused_vs_oracle(f"{name} masks={masks}", scenes.flagged_scene(name), masks=masks)


def test_fused_saturating_stack():
    """Opaque splats stacked in one tile: every pixel saturates and the backward starts at the saturation depth."""
    sc = stack(6000, 3.0, spread=0.05, scale=(0.03, 0.07))
    _, o, _ = fused_vs_oracle("saturated", sc)
    assert int(o.n[30:34, 30:34].min()) < 1000 and np.diff(o.ranges).max() > 2000   # saturated early near the centre


def test_row_check_flags_a_zeroed_block_on_the_gpu():
    """Negative control.  The upstream gradient is faint (x 1e-3) on tile (2, 1), so the gaussians seen mostly there
    have gradients far below the largest ones.  The GPU gradient from it passes the row check.  The GPU gradient from
    the same upstream gradient zeroed on one 4x4 block of that tile, against the oracle's from the unzeroed one, still
    passes the global criterion; the row check flags rows, and only rows of gaussians whose walk covers the block."""
    sc = np_scene(2000, "tiny", 0, sigma_px=(2.0, 0.5, 0.5, 8.0))
    G = upstream(sc)
    G[32:48, 16:32] *= 1e-3
    block = (slice(40, 44), slice(24, 28))
    fused_vs_oracle("faint tile", sc, G=G)
    res, o, _ = fused_vs_oracle("faint tile, block zeroed", sc, G=G, check=False, zero_block=block)
    G_block = np.zeros_like(G)
    G_block[block] = G[block]
    d_block = orc.rasterize_backward(o, G_block)
    covered = np.zeros(len(o.keep), bool)
    for k in FIELDS:
        covered |= (getattr(d_block.mass, k).reshape(len(covered), -1) > 0).any(1)
    assert covered.sum() > 0
    for r in res:
        print(r)
        assert r.global_err < gradrows.GLOBAL_TOL, str(r)
        assert set(r.bad.tolist()) <= set(np.flatnonzero(covered).tolist()), str(r)
    for r in res[:len(FIELDS)]:   # every render-stage field flags more rows than threshold flips may explain
        assert not r.ok and len(r.bad) > r.allowed, str(r)


# ------------------------------------------------------------------------------------------------
# operator-by-operator path
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shd", [1, 2])
def test_unfused_sh_degrees(shd):
    sc = np_scene(2000, "tiny", shd, sigma_px=(2.0, 0.5, 0.5, 8.0))
    o = oracle_forward(sc)
    g = gaussians_from(sc)
    image, mask, uv = rasterize_unfused(g, to_t(sc["T"]), Camera(64, 64, to_t(sc["K"])), 0.3, 500.0, 100, 3.0, True,
                                        torch.full((3,), BG, device=dev()))
    G = upstream(sc)
    G = np.where(flip_pixels(check_forward(image, o, mask, uv), None, o, G)[:, :, None], 0, G).astype(np.float32)
    seen = []
    image.grad_fn.register_hook(lambda grad_inputs, grad_outputs: seen.append([t.detach().clone() for t in grad_inputs[:4]]))
    image.backward(to_t(G))
    keep = o.keep
    M = int(keep.sum())
    rgb, opa, guv, conic = (t.double().cpu().numpy() for t in seen[0])
    assert rgb.shape == (M, 3) and opa.shape == (M, 1) and guv.shape == (M, 2) and conic.shape == (M, 3)
    d = orc.rasterize_backward(o, G)
    allowed = gradrows.flips_allowed(M)
    mine = dict(rgb=rgb, opacity=opa.reshape(-1), uv=guv, conic=conic)
    res = render_results(f"unfused sh{shd}", mine, d, keep, gradrows.EPS[np.dtype(np.float32)], allowed)

    def full(a):
        out = np.zeros((len(keep),) + a.shape[1:])
        out[keep] = a
        return out

    pr = orc.project_backward(o, full(rgb), full(opa.reshape(-1)), full(guv), full(conic))
    res += param_results(f"unfused sh{shd}", g, pr, allowed)
    gradrows.assert_all(res)


# ------------------------------------------------------------------------------------------------
# per-pixel SH: the generic kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shd", [1, 2])
def test_per_pixel_sh_generic_kernels(shd, dtype):
    """RenderImage with [M,3,N_SH] colours along per-pixel view directions, fed the oracle's per-gaussian inputs and
    tile lists.  A low-opacity stack makes some pixel's walk longer than the reference's chunk for this (dtype,
    N_SH), so the chunk-local index of the weight recurrence is exercised."""
    n_sh = (shd + 1) ** 2
    sc = stack(2500, -5.0, shd=shd, dtype=dtype)
    o = oracle_forward(sc, per_pixel=True)
    chunk = orc.REF_CHUNK[(np.dtype(dtype).type, n_sh)]
    assert int(o.n.max()) > chunk, (int(o.n.max()), chunk)
    leaves = [to_t(a).requires_grad_(True) for a in (o.rgb, o.opacity.reshape(-1, 1), o.uv, o.conic)]
    rays = to_t(o.view_dirs)
    image = af.RenderImage.apply(*leaves, rays, to_t(o.ranges), to_t(o.sorted_idx), (sc["H"], sc["W"]),
                                 torch.full((3,), BG, dtype=leaves[0].dtype, device=dev()))
    bad = check_forward(image, o)
    G = upstream(sc)
    if dtype == np.float32:
        G = np.where(flip_pixels(bad, None, o, G)[:, :, None], 0, G).astype(dtype)
    else:
        assert not bad.any()
    image.backward(to_t(G))
    d = orc.render_backward(o.uv, o.opacity, o.rgb, o.conic, o.view_dirs, o.ranges, o.sorted_idx, o.background, o.n,
                            o.wlast, G, mass=True)
    ref = dict(zip(FIELDS, d[:4]))
    mass = d[4]
    M = int(o.keep.sum())
    allowed = gradrows.flips_allowed(M, dtype)
    res = [gradrows.render_rows(f"per-pixel sh{shd} {np.dtype(dtype).name} {k}", leaf.grad, ref[k], getattr(mass, k),
                                (RENDER_C if dtype == np.float32 else gradrows.RENDER_C_FP64)[k],
                                gradrows.EPS[np.dtype(dtype)], allowed)
           for k, leaf in zip(FIELDS, leaves)]
    gradrows.assert_all(res)
