"""The blend-weight statistics oracle (tests/weight_stats_oracle.py) against an independent numpy restatement and its
own identities, the semantics of plan_prune, and rasterize(weight_stats=...)'s argument errors.  CPU only."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200.densify import DensificationPlan, WeightStats, plan_prune
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera, Gaussians
from oracle import cpu_oracle as orc
from tests import weight_stats_oracle as wso
from tests.scenes import np_scene


def tiny(n=300, seed=0, H=40, W=48, **kw):
    sc = np_scene(n, "tiny", sh_degree=0, seed=seed, sigma_px=(2.0, 0.5, 0.5, 8.0), **kw)
    sc = dict(sc, H=H, W=W, K=sc["K"].copy())
    sc["K"][0, 2], sc["K"][1, 2] = W / 2.0, H / 2.0
    return sc


def oracle_forward(sc):
    return orc.rasterize(sc["xyz"], sc["quaternion"], sc["scale"], sc["opacity"], sc["rgb"], sc["sh"], sc["T"],
                         sc["K"], sc["H"], sc["W"], 0.3, 500.0, 100.0, 3.0, background=np.full(3, 0.5, np.float32))


def fmaf(a, b, c):
    """fp32 fused multiply-add through fp64 (the fp32 product is exact there; one more rounding to fp32)."""
    return (a.astype(np.float64) * b + c).astype(np.float32)


def numpy_stats(o):
    """Per tile, all 256 pixels at once, the splats of the tile in depth order: the reference forward's skip and
    saturation rules with w = (float)((1 - (double)A) * (double)alpha)."""
    H, W = o.n.shape
    M = o.uv.shape[0]
    s, m, n = np.zeros(M), np.zeros(M, np.float32), np.zeros(M, np.int64)
    A_img = np.zeros((H, W), np.float32)
    f32 = np.float32
    for ty in range((H + 15) // 16):
        for tx in range((W + 15) // 16):
            ys, xs = np.meshgrid(np.arange(ty * 16, min(H, ty * 16 + 16)), np.arange(tx * 16, min(W, tx * 16 + 16)),
                                 indexing="ij")
            px, py = xs.astype(f32).ravel(), ys.astype(f32).ravel()
            A = np.zeros(px.shape, f32)
            tile = ty * ((W + 15) // 16) + tx
            for p in range(o.ranges[tile], o.ranges[tile + 1]):
                g = o.sorted_idx[p]
                live = A.astype(np.float64) <= 0.9999
                du, dv = px - f32(o.uv[g, 0]), py - f32(o.uv[g, 1])
                b = f32(o.conic[g, 1]) * f32(0.5)
                a, c = f32(o.conic[g, 0]) + f32(0.25), f32(o.conic[g, 2]) + f32(0.25)
                det = fmaf(np.array([a]), np.array([c]), -(b * b))[0]
                t3 = dv * (du * (b + b))
                t4 = fmaf(du, du * c, -t3)
                num = fmaf(dv, dv * a, t4)
                mh = num / det
                e = np.exp2((f32(-0.5) * mh) * f32(1.4426950216293334961))
                alpha = np.where(mh > 0, e * f32(np.ravel(o.opacity)[g]), f32(0.0)).astype(f32)
                use = live & (alpha.astype(np.float64) >= 0.00392156862)
                w = (alpha.astype(np.float64) * (1.0 - A.astype(np.float64))).astype(f32)
                if use.any():
                    s[g] += w[use].astype(np.float64).sum()
                    m[g] = max(m[g], w[use].max())
                    n[g] += int(use.sum())
                A = np.where(use, A + w, A).astype(f32)
            A_img[ys.ravel(), xs.ravel()] = A
    return s, m, n, A_img


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_matches_an_independent_numpy_loop(seed):
    o = oracle_forward(tiny(seed=seed))
    r = wso.weight_stats(o)
    s, m, n, A = numpy_stats(o)
    assert (n > 0).sum() > 20
    assert np.array_equal(r.compact_count, n)
    # numpy's exp2 and the C library's exp2f may differ in the last place: weights agree to a few ulps
    np.testing.assert_allclose(r.compact_max, m, rtol=1e-6, atol=0)
    np.testing.assert_allclose(r.compact_sum, s, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(r.alpha, A, rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("seed", [0, 3])
def test_identities_sum_is_alpha_and_count_is_blends(seed):
    """sum_i weight_sum_i = sum_p A_p (A the accumulated alpha: A is the fp32 running sum of the same w), and
    sum_i pixel_count_i = the number of blends; rows of culled gaussians stay zero; max <= sum."""
    o = oracle_forward(tiny(n=2000, seed=seed, H=64, W=64))
    r = wso.weight_stats(o)
    assert np.isclose(r.sum.sum(), r.alpha.astype(np.float64).sum(), rtol=1e-5, atol=0)
    assert int(r.count.sum()) == int(r.nblend.sum()) > 0
    assert (r.sum[~o.keep] == 0).all() and (r.max[~o.keep] == 0).all() and (r.count[~o.keep] == 0).all()
    assert (r.max <= r.sum * (1 + 1e-6) + 1e-12).all() and (r.max <= 1.0).all()
    assert ((r.count > 0) == (r.sum > 0)).all()
    # the blend count is bounded by the oracle forward's per-pixel splat count (which also counts skipped splats)
    assert (r.nblend <= o.n).all()


# plan_prune ---------------------------------------------------------------------------------------------------
def test_plan_prune_keeps_the_rounded_up_fraction_in_ascending_order():
    score = torch.tensor([0.5, 3.0, 1.0, 2.0, 0.0, 4.0, 1.5])
    plan = plan_prune(score, 0.5)          # ceil(3.5) = 4 rows: 5 (4.0), 1 (3.0), 3 (2.0), 6 (1.5)
    assert isinstance(plan, DensificationPlan) and plan.n_in == 7 and plan.n_out == 4
    assert plan.src.dtype == torch.int32 and plan.src.tolist() == [1, 3, 5, 6]
    assert plan.clone_row is None and plan.split_row is None and plan.xyz_add is None
    assert plan.info == dict(n_in=7, n_out=4, deleted=3)
    assert plan_prune(score, 0.01).src.tolist() == [5]   # ceil(0.07) = 1
    assert plan_prune(score, 1 / 7).src.tolist() == [5]  # ceil(1.0) = 1, not 2


def test_plan_prune_breaks_ties_by_the_lower_row():
    score = torch.tensor([1.0, 2.0, 1.0, 1.0, 2.0, 1.0])
    assert plan_prune(score, 0.5).src.tolist() == [0, 1, 4]
    assert plan_prune(score, 4 / 6).src.tolist() == [0, 1, 2, 4]
    ints = torch.tensor([7, 7, 7, 7], dtype=torch.int32)
    assert plan_prune(ints, 0.5).src.tolist() == [0, 1]
    big = torch.zeros(10_000)
    big[::3] = 1.0
    assert plan_prune(big, 0.5).src.tolist() == sorted(list(range(0, 10_000, 3)) + [i for i in range(10_000) if i % 3][:1666])


def test_plan_prune_ranks_nan_scores_last():
    score = torch.tensor([float("nan"), 1.0, float("nan"), 0.0, 2.0])
    assert plan_prune(score, 0.6).src.tolist() == [1, 3, 4]
    assert plan_prune(score, 0.8).src.tolist() == [0, 1, 3, 4]   # NaN rows among themselves: lower row first


def test_plan_prune_identity_and_sizes():
    score = torch.rand(100, generator=torch.Generator().manual_seed(0))
    plan = plan_prune(score, 1.0)
    assert plan.is_identity() and plan.n_out == 100 and plan.info["deleted"] == 0
    assert plan_prune(score, 0.999).is_identity()        # ceil(99.9) = 100
    assert plan_prune(torch.zeros(0), 0.5).is_identity()
    src = plan_prune(score, 0.3).src
    assert src.numel() == 30 and bool((src[1:] > src[:-1]).all())
    assert set(src.tolist()) == set(torch.topk(score, 30).indices.tolist())


def test_plan_prune_argument_errors():
    with pytest.raises(ValueError):
        plan_prune(torch.rand(4), 0.0)
    with pytest.raises(ValueError):
        plan_prune(torch.rand(4), 1.5)
    with pytest.raises(ValueError):
        plan_prune(torch.rand(4, 2), 0.5)
    with pytest.raises(TypeError):
        plan_prune(torch.ones(4, dtype=torch.bool), 0.5)


# WeightStats and rasterize's argument checks ----------------------------------------------------------------------
def test_weight_stats_fields_and_reset():
    ws = WeightStats(5, "cpu")
    assert len(ws) == 5
    assert ws.weight_sum.dtype == ws.weight_max.dtype == torch.float32 and ws.pixel_count.dtype == torch.int32
    ws.weight_sum += 1.0
    ws.weight_max += 2.0
    ws.pixel_count += 3
    ws.reset()
    assert float(ws.weight_sum.abs().sum() + ws.weight_max.abs().sum()) == 0.0 and int(ws.pixel_count.sum()) == 0


def test_argument_errors():
    sc = np_scene(50, "tiny", sh_degree=1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    g = Gaussians(t(sc["xyz"]), t(sc["rgb"]), t(sc["opacity"]), t(sc["scale"]), t(sc["quaternion"]), t(sc["sh"]))
    cam, bg, T = Camera(64, 64, t(sc["K"])), torch.full((3,), 0.5), t(sc["T"])
    ws = WeightStats(50, "cpu")
    with pytest.raises(ValueError):   # per-pixel SH
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, False, bg, weight_stats=ws)
    with pytest.raises(ValueError):   # stale after densification
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, weight_stats=WeightStats(49, "cpu"))
    bad = WeightStats(50, "cpu")
    bad.pixel_count = bad.pixel_count.float()
    with pytest.raises(TypeError):    # wrong dtype
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, weight_stats=bad)
    bad = WeightStats(50, "cpu")
    bad.weight_sum = bad.weight_sum.double()
    with pytest.raises(TypeError):
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, weight_stats=bad)
    bad = WeightStats(50, "cpu")
    bad.weight_max = torch.zeros(50, 2)[:, 0]
    with pytest.raises(ValueError):   # not contiguous
        rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, weight_stats=bad)
    g64 = Gaussians(*(x.double() for x in (g.xyz, g.rgb, g.opacity, g.scale, g.quaternion)), None)
    with pytest.raises(TypeError):    # fp64
        rasterize(g64, T.double(), Camera(64, 64, t(sc["K"]).double()), 0.3, 500.0, 100, 3.0, True, bg.double(),
                  weight_stats=ws)
