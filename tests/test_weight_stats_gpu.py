"""rasterize(weight_stats=...) on the GPU: the per-gaussian blend-weight statistics against the CPU oracle
(tests/weight_stats_oracle.py), their effect on everything else (none), accumulation, the speculative pair buffers, the
headline size, pruning on the flat buffers, and the kernels in the built library — needs an H100."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import rasterize as R
from gaussian_splatting_b200 import synth
from gaussian_splatting_b200.densify import AdaptiveDensityControl, DensificationStats, DensifyConfig, WeightStats, \
    plan_prune
from gaussian_splatting_b200.flat_adam import FlatAdam
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera
from tests import antialiased_oracle as aao
from tests import depth_alpha_oracle as dao
from tests import filter3d_oracle as fo
from tests import gradrows, scenes
from tests import weight_stats_oracle as wso
from tests.test_gradient_rows_gpu import gaussians_from, np_scene, ragged, stack

pytestmark = pytest.mark.gpu
BG = 0.5
PARAMS = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")


def dev():
    return torch.device("cuda:0")


def to_t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def bits(a):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else a.dtype)


def run(sc, ws=None, grads=None, masks=True, depth_alpha=False, g=None, grad=True, **kw):
    """Fused forward (+ backward of <G,image> [+ <Gd,depth> + <Ga,alpha>] when grads is given).  grad=False: under
    torch.no_grad() (the kernels without contribution masks)."""
    R.USE_CONTRIBUTION_MASKS = masks
    try:
        g = gaussians_from(sc) if g is None else g
        cam = Camera(sc["W"], sc["H"], to_t(sc["K"]))
        with torch.set_grad_enabled(grad):
            out = rasterize(g, to_t(sc["T"]), cam, 0.3, 500.0, 100, 3.0, True, torch.full((3,), BG, device=dev()),
                            return_state=True, render_depth_alpha=depth_alpha, weight_stats=ws, **kw)
        if grads is not None:
            maps = out[:1] + (out[3:5] if depth_alpha else ())
            pairs = [(t, to_t(G).view_as(t)) for t, G in zip(maps, grads) if G is not None]
            torch.autograd.backward([t for t, _ in pairs], [G for _, G in pairs])
    finally:
        R.USE_CONTRIBUTION_MASKS = True
    return out, g


def small(s):
    return np_scene(2000, "tiny", s, sigma_px=(2.0, 0.5, 0.5, 8.0))


def live_filter(sc):
    """A 3-D filter of the scene's order of size (a few hundredths of the world scale), seeded."""
    return (np.random.default_rng(9).uniform(0.0, 0.05, sc["xyz"].shape[0])).astype(np.float32)


def oracle(sc, antialiased=False, f3d=None):
    kw = dict(background=np.full(3, BG, np.float32))
    if f3d is not None:
        sigma = torch.sigmoid(to_t(sc["opacity"]).reshape(-1)).cpu().numpy()
        return fo.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"],
                            sc["K"], sc["H"], sc["W"], f3d, antialiased=antialiased, mh_dist=3.0,
                            e=torch.exp(to_t(sc["scale"])).cpu().numpy(), sigma=sigma, **kw)
    f = aao.rasterize if antialiased else dao.rasterize
    return f(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"], sc["K"], sc["H"],
             sc["W"], 0.3, 500.0, 100.0, 3.0, **kw)


def ulps(a, b):
    """Distance in units in the last place of non-negative fp32 arrays."""
    return np.abs(np.ascontiguousarray(a, np.float32).view(np.int32).astype(np.int64)
                  - np.ascontiguousarray(b, np.float32).view(np.int32).astype(np.int64))


def check_against_oracle(tag, ws, r):
    """pixel_count exactly, weight_max and weight_sum within 1e-5 relative (+ a 1e-6 floor) for every gaussian the
    oracle is certain about.  The weights themselves are not compared to the ulp: the host's exp2f and the device's
    ex2.approx differ by an ulp or two in alpha, and w = alpha (1 - A) magnifies a difference in the accumulated A by
    A / (1 - A) (measured: up to 177 ulps in a saturating tile); counts do not depend on it.  A gaussian some pixel reaches after an alpha within 3e-5 of the 1/255 skip
    (r.uncertain: the host's exp2f and the device's ex2.approx may decide that skip differently, and every later
    splat of the pixel sees another accumulated alpha) may differ by at most that many pixels in its count."""
    cnt, mx, sm = (ws.pixel_count.cpu().numpy().astype(np.int64), ws.weight_max.cpu().numpy(),
                   ws.weight_sum.cpu().numpy().astype(np.float64))
    sure = r.uncertain == 0
    print(f"{tag}: {int((r.count > 0).sum())} gaussians contribute, {int((~sure).sum())} uncertain, "
          f"{int(r.count.sum())} blends")
    assert (r.count > 0).sum() > 0
    bad = np.nonzero(sure & (cnt != r.count))[0]
    assert bad.size == 0, (tag, "count", bad[:10], cnt[bad[:10]], r.count[bad[:10]])
    assert (np.abs(cnt - r.count) <= r.uncertain).all(), (tag, "uncertain count")
    u = ulps(mx, r.max)
    print(f"{tag}: weight_max within {int(u[sure].max())} ulps")
    errm = np.abs(mx.astype(np.float64) - r.max)
    limm = 1e-5 * r.max.astype(np.float64) + 1e-6
    assert (errm[sure] <= limm[sure]).all(), (tag, "max", float((errm[sure] / limm[sure]).max()))
    err = np.abs(sm - r.sum)
    lim = 1e-5 * np.abs(r.sum) + 1e-6
    assert (err[sure] <= lim[sure]).all(), (tag, "sum", float((err[sure] / lim[sure]).max()))


SCENES = [("sh0", lambda: small(0)), ("sh3", lambda: small(3)), ("50x37", lambda: ragged(50, 37, 1)),
          ("720p", lambda: np_scene(100_000, "720p", 3, seed=0)), ("deep", lambda: stack(3000, -5.0)),
          ("saturated", lambda: stack(6000, 3.0, spread=0.05, scale=(0.03, 0.07)))]
# the exact recompute (tests/scenes.py FLAGGED): the statistics of flagged pixels come from the walk, the image from the
# recompute
SCENES += [(n, lambda n=n: scenes.flagged_scene(n)) for n in scenes.FLAGGED]
VARIANTS = [("masks", dict()), ("no masks", dict(masks=False)), ("no_grad", dict(grad=False)),
            ("depth", dict(depth_alpha=True)), ("aa", dict(antialiased=True)), ("f3d", dict(f3d=True)),
            ("f3d aa depth", dict(f3d=True, antialiased=True, depth_alpha=True))]
CASES = [(f"{s} {v}", make, kw) for s, make in SCENES for v, kw in VARIANTS
         if v in ("masks", "no masks") or s in ("sh3", "720p", "saturated")
         or (s in scenes.FLAGGED and v in ("depth", "aa"))]


@pytest.mark.parametrize("tag,make,kw", CASES, ids=[c[0] for c in CASES])
def test_weight_stats_against_the_fp32_oracle(tag, make, kw):
    sc = make()
    kw = dict(kw)
    f3d = live_filter(sc) if kw.pop("f3d", False) else None
    o = oracle(sc, kw.get("antialiased", False), f3d)
    if "saturated" in tag:
        assert int(np.diff(o.ranges).max()) > 2000   # one tile holds more than 2000 splats
    ws = WeightStats(sc["xyz"].shape[0], dev())
    out, _ = run(sc, ws, filter3d=None if f3d is None else to_t(f3d), **kw)
    st = out[-1]
    # the walk over the fused path's own records and pair list: exact counts, max to an ulp, sums to 1e-5
    r = wso.weight_stats_of_records(st.records.cpu().numpy(), st.ranges.cpu().numpy(),
                                    st.ids_sorted.cpu().numpy(), sc["H"], sc["W"])
    check_against_oracle(tag, ws, r)
    # against the host oracle of the whole chain (its own projection): the same gaussians contribute, and the totals
    # agree to the projection's rounding
    ro = wso.weight_stats(o)
    assert np.array_equal(ro.count > 0, r.count > 0) or int(((ro.count > 0) != (r.count > 0)).sum()) <= 3
    assert abs(ro.sum.sum() - r.sum.sum()) <= 1e-4 * r.sum.sum() and abs(int(ro.count.sum()) - int(r.count.sum())) \
        <= 1e-4 * r.count.sum() + 3


@pytest.mark.parametrize("kind,depth_alpha,extra", [("sh3", False, {}), ("deep", False, {}), ("sh3", True, {}),
                                                    ("sh3", True, dict(antialiased=True, absgrad=True))])
def test_outputs_and_gradients_unchanged(kind, depth_alpha, extra):
    """image, mask, uv, n_per_pixel, w_per_pixel, contribution masks (and depth / alpha) bit-identical with and
    without weight_stats; gradients (and uv.absgrad) within the run-to-run spread of the atomic reductions."""
    sc = small(3) if kind == "sh3" else stack(3000, -5.0)
    rng = np.random.default_rng(1)
    H, W = sc["H"], sc["W"]
    grads = ((rng.standard_normal((H, W, 3)) / (3.0 * H * W)).astype(np.float32),
             (rng.standard_normal((H, W)) / (H * W)).astype(np.float32),
             (rng.standard_normal((H, W)) / (H * W)).astype(np.float32))[:3 if depth_alpha else 1]
    out0, g0 = run(sc, None, grads, depth_alpha=depth_alpha, **extra)
    ws = WeightStats(sc["xyz"].shape[0], dev())
    out1, g1 = run(sc, ws, grads, depth_alpha=depth_alpha, **extra)
    n = 5 if depth_alpha else 3
    for a, b in zip(out0[:n], out1[:n]):
        assert np.array_equal(bits(a), bits(b))
    s0, s1 = out0[-1], out1[-1]
    for k in ("n_per_pixel", "w_per_pixel", "masks"):
        assert torch.equal(getattr(s0, k), getattr(s1, k)), k
    assert int(ws.pixel_count.sum()) > 0 and not ws.weight_sum.requires_grad
    for k in PARAMS:
        if getattr(g0, k) is not None:
            assert gradrows.global_rel(getattr(g1, k).grad, getattr(g0, k).grad) < 2e-5, k
    if extra.get("absgrad"):
        assert gradrows.global_rel(s1.uv_absgrad, s0.uv_absgrad) < 2e-5


def test_two_views_accumulate_as_sum_max_sum():
    sc = small(3)
    sc2 = dict(sc, T=scenes.np_scene(2000, "tiny", sh_degree=3, view=1, n_views=3)["T"])
    N = sc["xyz"].shape[0]
    both, a, b = WeightStats(N, dev()), WeightStats(N, dev()), WeightStats(N, dev())
    run(sc, both, grad=False)
    run(sc2, both, grad=False)
    run(sc, a, grad=False)
    run(sc2, b, grad=False)
    assert torch.equal(both.pixel_count, a.pixel_count + b.pixel_count)
    assert torch.equal(both.weight_max, torch.maximum(a.weight_max, b.weight_max))
    assert gradrows.global_rel(both.weight_sum, a.weight_sum + b.weight_sum) < 1e-6
    assert int((a.pixel_count > 0).sum()) > 0 and not torch.equal(a.pixel_count, b.pixel_count)
    both.reset()
    assert int(both.pixel_count.abs().sum()) == 0 and float(both.weight_sum.abs().sum()) == 0.0


@pytest.mark.parametrize("depth_alpha", [False, True])
def test_eager_fitting_and_overflowing_speculation_agree(depth_alpha):
    """The first view of an (N, H, W) reads the pair count eagerly, later ones size the pair buffers from history;
    a too-small guess (history [1000]) renders twice, and the discarded first run must add nothing."""
    sc = np_scene(100_000, "720p", 3, seed=0)
    N = sc["xyz"].shape[0]
    key = (dev().index if dev().index is not None else torch.cuda.current_device(), N, sc["H"], sc["W"])
    R._PAIR_HISTORY.pop(key, None)
    res, masks = {}, {}
    for name in ("eager", "fitting", "overflow"):
        if name == "overflow":
            R._PAIR_HISTORY[key] = [1000]
        ws = WeightStats(N, dev())
        out, _ = run(sc, ws, depth_alpha=depth_alpha)
        assert out[-1].speculation_overflowed == (name == "overflow"), name
        res[name] = ws
        masks[name] = out[-1].masks
    R._PAIR_HISTORY.pop(key, None)
    e = res["eager"]
    for name in ("fitting", "overflow"):
        # the state's contribution masks hold the words of the binned pairs, whatever capacity the run was sized for
        assert torch.equal(masks[name], masks["eager"]), name
        assert torch.equal(res[name].pixel_count, e.pixel_count), name
        assert torch.equal(res[name].weight_max, e.weight_max), name
        assert gradrows.global_rel(res[name].weight_sum, e.weight_sum) < 1e-6, name


def test_headline_size_sum_is_the_alpha_map():
    """3M gaussians, 1080p: sum_i weight_sum_i against the sum of the alpha map (the same weights, summed per pixel)."""
    g, cam, T, _ = scenes.headline_inputs(1080, dev())
    ws = WeightStats(g.xyz.shape[0], dev())
    with torch.no_grad():
        out = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, torch.full((3,), BG, device=dev()),
                        render_depth_alpha=True, weight_stats=ws)
    alpha = out[4].double().sum()
    total = ws.weight_sum.double().sum()
    print("sum of weight_sum", float(total), "sum of alpha", float(alpha), "pixels counted", int(ws.pixel_count.sum()))
    assert float(alpha) > 1e5
    assert abs(float(total - alpha)) <= 1e-5 * float(alpha)


def test_prune_on_flat_adam_keeps_the_planned_rows():
    gs = synth.make_gaussians(20_000, "small", sh_degree=3, seed=4, device=dev(), requires_grad=True,
                              sigma_px=(2.5, 0.5, 0.5, 10.0))
    opt = FlatAdam.for_gaussians(gs)
    cam = synth.make_camera("small", device=dev())
    bg = torch.full((3,), BG, device=dev())
    for view in range(2):   # moments that differ per row
        T = synth.make_pose(view, 3, device=dev())
        image, _, _, st = rasterize(gs, T, cam, 0.3, 500.0, 100, 3.0, True, bg, return_state=True)
        image.backward(synth.make_upstream_grad("small", device=dev()))
        opt.step(st.grad_flat)
        for f in ("xyz", "rgb", "opacity", "scale", "quaternion", "sh"):
            getattr(gs, f).grad = None
    N = gs.xyz.shape[0]
    ws = WeightStats(N, dev())
    with torch.no_grad():
        for view in range(3):
            rasterize(gs, synth.make_pose(view, 3, device=dev()), cam, 0.3, 500.0, 100, 3.0, True, bg, weight_stats=ws)
    before = {f: getattr(gs, f).detach().clone() for f in ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")}
    m_rows = {f: v.clone() for f, v in zip(before, _sections(opt.m, opt.ends, N, gs))}
    v_rows = {f: v.clone() for f, v in zip(before, _sections(opt.v, opt.ends, N, gs))}
    stats = DensificationStats(N, dev())
    adc = AdaptiveDensityControl(gs, opt, stats, DensifyConfig())
    keep = plan_prune(ws.weight_sum, 0.4).src.long()
    info = adc.prune(ws.weight_sum, 0.4)
    assert info == dict(n_in=N, n_out=8000, deleted=12_000) and gs.xyz.shape[0] == 8000
    assert stats.grad_accum_count.shape[0] == 8000
    for f, old in before.items():
        assert torch.equal(getattr(gs, f).detach(), old[keep]), f
    for f, new in zip(before, _sections(opt.m, opt.ends, 8000, gs)):
        assert torch.equal(new, m_rows[f][keep]), f
    for f, new in zip(before, _sections(opt.v, opt.ends, 8000, gs)):
        assert torch.equal(new, v_rows[f][keep]), f
    image, _, _ = rasterize(gs, synth.make_pose(0, 3, device=dev()), cam, 0.3, 500.0, 100, 3.0, True, bg)
    assert image.shape == (cam.height, cam.width, 3) and bool(torch.isfinite(image).all())
    with pytest.raises(ValueError):   # the old statistics are stale now
        rasterize(gs, synth.make_pose(0, 3, device=dev()), cam, 0.3, 500.0, 100, 3.0, True, bg, weight_stats=ws)


def _sections(buf, ends, n, gs):
    widths = dict(xyz=(3,), quaternion=(4,), scale=(3,), opacity=(1,), rgb=(3,), sh=tuple(gs.sh.shape[1:]))
    start, out = 0, []
    for f, end in zip(widths, ends):
        out.append(buf[start:end].view((n,) + widths[f]))
        start = end
    return out


def test_wrong_device_raises():
    sc = small(0)
    ws = WeightStats(sc["xyz"].shape[0], "cpu")
    with pytest.raises(ValueError):
        run(sc, ws)
