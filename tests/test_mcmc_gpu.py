"""3DGS-MCMC kernels on the GPU (csrc/gsr_mcmc.cu through the binding): the relocation against the fp64 oracle, the
apply pass on FlatAdam state against torch indexing, the position noise against the fp64 oracle and its Philox draws,
and a short training run with every MCMC piece in the loop."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import native, synth
from gaussian_splatting_b200.flat_adam import FIELDS, FlatAdam, section_ends
from gaussian_splatting_b200.loss import photometric_loss
from gaussian_splatting_b200.mcmc import (MCMCConfig, MCMCDensityControl, apply_mcmc_plan, plan_grow, plan_relocate,
                                          relocation)
from gaussian_splatting_b200.rasterize import rasterize
from tests import mcmc_oracle as mo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def ulps(a, b):
    a = torch.as_tensor(a).float().cpu().view(torch.int32).long()
    b = torch.as_tensor(b).float().cpu().view(torch.int32).long()
    return (a - b).abs()


# relocation ---------------------------------------------------------------------------------------------------------
def _check_relocation(o, s, ratio, min_opacity=0.005):
    new_o, new_s = native().mcmc_relocation(o.to(DEV), s.to(DEV), ratio.to(DEV), 51, min_opacity)
    _, want_o, want_s = mo.relocation_f64(o.numpy(), s.numpy(), ratio.numpy(), 51, min_opacity)
    rel = np.abs(new_s.cpu().double().numpy() / want_s - 1)
    assert rel.max() <= 1e-6, (rel.max(), int(rel.argmax()))
    assert int(ulps(new_o, torch.from_numpy(want_o)).max()) <= 1
    return rel


def test_relocation_on_the_grid():
    o = torch.tensor([1e-3, 0.005, 0.5, 0.99, 1 - 2.0 ** -23], dtype=torch.float32)
    ratios = torch.tensor(list(range(1, 52)) + [52, 80, 10_000], dtype=torch.int32)
    O = o.repeat_interleave(len(ratios)).contiguous()
    R = ratios.repeat(len(o)).contiguous()
    s = torch.tensor([[0.01, 0.2, 3.0]]).repeat(O.numel(), 1)
    _check_relocation(O, s, R)


def test_relocation_on_a_million_random_rows():
    g = torch.Generator().manual_seed(0)
    n = 1_000_000
    o = torch.cat([torch.rand(n // 2, generator=g),                                 # uniform in (0, 1)
                   torch.exp(torch.rand(n // 4, generator=g) * -16),              # down to 1e-7
                   1 - torch.exp(torch.rand(n - 3 * n // 4, generator=g) * -15)])  # up to 1 - 3e-7
    o = o.clamp(1e-7, 1 - 2.0 ** -23).float()
    s = torch.exp(torch.randn(n, 3, generator=g) * 2 - 4)
    ratio = torch.randint(1, 60, (n,), generator=g, dtype=torch.int32)
    rel = _check_relocation(o, s, ratio)
    print("max relative scale error", rel.max())


def test_relocation_wrapper_and_binding_errors():
    lo = torch.tensor([[-1.0], [0.5]], device=DEV)
    ls = torch.zeros(2, 3, device=DEV)
    o, s = relocation(lo, ls, torch.tensor([1, 3], device=DEV))
    assert torch.equal(o[0], torch.sigmoid(lo[0, 0])) and torch.equal(s[0], torch.ones(3, device=DEV))
    r = torch.ones(2, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError):
        native().mcmc_relocation(torch.sigmoid(lo).double().reshape(-1), ls, r, 51, 0.005)            # dtype
    with pytest.raises(RuntimeError):
        native().mcmc_relocation(torch.sigmoid(lo).reshape(-1), torch.zeros(3, 2, device=DEV).t(), r, 51, 0.005)
    with pytest.raises(RuntimeError):
        native().mcmc_relocation(torch.sigmoid(lo).reshape(-1), ls, r.long(), 51, 0.005)
    with pytest.raises(RuntimeError):
        native().mcmc_relocation(torch.sigmoid(lo).reshape(-1), ls, r, 0, 0.005)


# apply --------------------------------------------------------------------------------------------------------------
def _state(n, sh_degree, seed=0):
    g = synth.make_gaussians(n, "1080p", sh_degree=sh_degree, seed=seed, device=DEV)
    with torch.no_grad():
        g.opacity[::5] = -8.0                                        # a fifth of the rows dead
    for f in FIELDS:
        if getattr(g, f) is not None:
            getattr(g, f).requires_grad_(True)
    opt = FlatAdam.for_gaussians(g)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    opt.m.copy_(torch.randn(opt.m.shape, device=DEV, generator=gen))
    opt.v.copy_(torch.rand(opt.v.shape, device=DEV, generator=gen))
    return g, opt


def _sections(buf, n, n_rest):
    ends = [0] + section_ends(n, n_rest)
    widths = [3, 4, 3, 1, 3, 3 * n_rest][:len(ends) - 1]   # no sh section without SH
    return [(buf[a:a + n * w].view(n, w), buf[a + n * w:b]) for a, b, w in zip(ends, ends[1:], widths)]


@pytest.mark.parametrize("n", [100_000, 3_000_000])
@pytest.mark.parametrize("sh_degree", [0, 3])
@pytest.mark.parametrize("kind", ["relocate", "grow"])
def test_apply_on_flat_adam_state(n, sh_degree, kind):
    g, opt = _state(n, sh_degree)
    n_rest = 0 if g.sh is None else int(g.sh.shape[2])
    cfg = MCMCConfig(cap_max=10 ** 8)
    planner = plan_relocate if kind == "relocate" else plan_grow
    plan = planner(g, cfg, torch.Generator(device=DEV).manual_seed(1))
    assert not plan.is_identity()
    p0, m0, v0 = opt.p.clone(), opt.m.clone(), opt.v.clone()
    new_o, new_s = relocation(g.opacity[plan.sources], g.scale[plan.sources], plan.ratio, cfg.n_max, cfg.min_opacity)
    apply_mcmc_plan(plan, g, opt)
    torch.cuda.synchronize()
    n_out = plan.n_out
    assert g.xyz.shape[0] == n_out and opt.p.numel() == section_ends(n_out, n_rest)[-1]
    src, set_row = plan.src.long(), plan.set_row.long()
    fresh = set_row >= 0
    old = [_sections(b, n, n_rest) for b in (p0, m0, v0)]
    new = [_sections(b, n_out, n_rest) for b in (opt.p, opt.m, opt.v)]
    for k in range(len(new[0])):
        for j in range(3):
            assert not new[j][k][1].any(), ("padding", k, j)                       # section padding is zero
        p_new, p_want = new[0][k][0], old[0][k][0][src]
        if k == 2:   # scale: the kernel's log of the relocation
            p_want = p_want.clone()
            p_want[fresh] = torch.log(new_s[set_row[fresh]])
        elif k == 3:  # opacity: the kernel's logit of the relocation
            p_want = p_want.clone()
            q = new_o[set_row[fresh]]
            p_want[fresh] = torch.log(q / (1 - q)).unsqueeze(1)
        if k in (2, 3):
            assert int(ulps(p_new, p_want).max()) <= 1, k
            assert torch.equal(p_new[~fresh], p_want[~fresh]), k                  # untouched: bit-identical
        else:
            assert torch.equal(p_new, p_want), k                                  # copied fields: bit-equal
        for j in (1, 2):
            mv = new[j][k][0]
            assert not mv[fresh].any(), ("moments of changed rows", k, j)
            assert torch.equal(mv[~fresh], old[j][k][0][src][~fresh]), ("moments kept", k, j)
    # a live source's opacity drops (ratio >= 2); growth may also draw a dead row, which the clamp lifts to min_opacity
    o_old = torch.sigmoid(old[0][3][0][plan.sources, 0])
    o_new = torch.sigmoid(g.opacity.detach()[plan.sources, 0])
    live = o_old > cfg.min_opacity
    assert (o_new[live] < o_old[live]).all()
    assert (o_new >= cfg.min_opacity * (1 - 1e-6)).all()
    opt.step(torch.zeros_like(opt.p))


def test_apply_binding_errors():
    g, opt = _state(1000, 0)
    plan = plan_relocate(g, MCMCConfig(), torch.Generator(device=DEV).manual_seed(1))
    o, s = relocation(g.opacity[plan.sources], g.scale[plan.sources], plan.ratio)
    ok = dict(p_in=opt.p, m_in=opt.m, v_in=opt.v, n_in=1000, n_sh_rest=0, src=plan.src, set_row=plan.set_row,
              new_opacity=o, new_scale=s)
    native().mcmc_apply(**ok)
    for bad in (dict(src=plan.src.long()), dict(src=plan.src[:999]), dict(set_row=None), dict(v_in=None),
                dict(p_in=opt.p.double()), dict(new_scale=s.t()), dict(p_out=opt.p), dict(m_in=opt.m[:-4])):
        with pytest.raises(RuntimeError):
            native().mcmc_apply(**dict(ok, **bad))


# noise --------------------------------------------------------------------------------------------------------------
def _noise_state(n, sh_degree=3, seed=0):
    g = synth.make_gaussians(n, "1080p", sh_degree=sh_degree, seed=seed, device=DEV)
    with torch.no_grad():
        gen = torch.Generator(device=DEV).manual_seed(seed + 1)
        g.opacity.copy_(torch.rand(g.opacity.shape, device=DEV, generator=gen) * 12 - 9)  # w from ~0.6 down to 0
        g.opacity[::3] = -12.0 + torch.rand(g.opacity[::3].shape, device=DEV, generator=gen) * 6  # w ~ 0.6
    opt = FlatAdam.for_gaussians(g)
    return g, opt, 0 if g.sh is None else int(g.sh.shape[2])


def test_noise_matches_the_fp64_oracle_given_eps():
    """Bound: |x - x64| <= 2^-23 |x64| + 3e-5 * scaler * w * |R| v |R|^T |eps|.  The 3e-5 covers the fp32 weight:
    (1 - o) - x0 is formed from an fp32 sigmoid (absolute error ~1e-7), times k = 100 that moves w by up to ~1e-5 of
    itself; the rotation and the products add a few 2^-24."""
    n = 200_000
    g, opt, n_rest = _noise_state(n)
    eps = torch.randn(n, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))
    before = [t.detach().cpu().double().numpy() for t in (g.xyz, g.quaternion, g.scale, g.opacity)]
    scaler = 2e4    # moves the low-opacity rows by about a tenth of a unit
    native().mcmc_noise(opt.p, n, n_rest, scaler, 100.0, 0.995, 0, 0, eps, None)
    want, mag = mo.noise_f64(*before, eps.cpu().double().numpy(), scaler)
    got = g.xyz.detach().cpu().double().numpy()
    err = np.abs(got - want)
    bound = 2.0 ** -23 * np.abs(want) + 3e-5 * mag
    assert (err <= bound).all(), float((err / bound).max())
    moved = np.abs(want - before[0]).max(1)
    assert (moved > 1e-4 * np.abs(before[0]).max(1)).mean() > 0.2                  # the noise is not negligible


def test_noise_draws_are_keyed_and_reproducible():
    n = 100_000
    g, opt, n_rest = _noise_state(n)
    p0 = opt.p.clone()
    out_a, out_b = torch.empty(n, 3, device=DEV), torch.empty(n, 3, device=DEV)
    native().mcmc_noise(opt.p, n, n_rest, 0.5, 100.0, 0.995, 11, 5, None, out_a)
    pa = opt.p.clone()
    opt.p.copy_(p0)
    native().mcmc_noise(opt.p, n, n_rest, 0.5, 100.0, 0.995, 11, 5, out_a, out_b)   # the recorded draws fed back
    assert torch.equal(opt.p, pa) and torch.equal(out_b, out_a)
    opt.p.copy_(p0)
    native().mcmc_noise(opt.p, n, n_rest, 0.5, 100.0, 0.995, 11, 5, None, out_b)    # same (seed, offset)
    assert torch.equal(opt.p, pa) and torch.equal(out_b, out_a)
    for seed, offset in ((11, 6), (12, 5)):
        native().mcmc_noise(p0.clone(), n, n_rest, 0.5, 100.0, 0.995, seed, offset, None, out_b)
        assert (out_b != out_a).float().mean() > 0.999
        assert abs(float(torch.corrcoef(torch.stack([out_a.reshape(-1), out_b.reshape(-1)]))[0, 1])) < 0.02
    # a row's draws do not depend on how many rows there are
    small = torch.empty(1000, 3, device=DEV)
    native().mcmc_noise(torch.zeros(section_ends(1000, 0)[-1], device=DEV), 1000, 0, 0.5, 100.0, 0.995, 11, 5, None,
                        small)
    assert torch.equal(small, out_a[:1000])


def test_noise_draws_are_standard_normal():
    """3 M x 3 draws at one fixed (seed, offset), so the figures are deterministic: mean within 2e-3 (6 sd), variance
    within 3e-3 of 1 (6 sd), Kolmogorov-Smirnov distance below 1.5e-3 (3.3 x the 5 % critical value), components
    uncorrelated within 3e-3."""
    from scipy import stats

    n = 3_000_000
    p = torch.zeros(section_ends(n, 0)[-1], device=DEV)
    eps = torch.empty(n, 3, device=DEV)
    native().mcmc_noise(p, n, 0, 1.0, 100.0, 0.995, 1234, 77, None, eps)
    e = eps.cpu().double().numpy()
    assert np.isfinite(e).all()
    flat = e.reshape(-1)
    ks = stats.kstest(flat, "norm").statistic
    c = np.corrcoef(e.T)
    print("mean", flat.mean(), "var", flat.var(), "ks", ks, "corr", c[0, 1], c[0, 2], c[1, 2])
    assert abs(flat.mean()) < 2e-3 and abs(flat.var() - 1) < 3e-3 and ks < 1.5e-3
    assert max(abs(c[0, 1]), abs(c[0, 2]), abs(c[1, 2])) < 3e-3


def test_noise_leaves_every_other_section_alone():
    n = 3_000_000
    g, opt, n_rest = _noise_state(n, seed=2)
    p0 = opt.p.clone()
    native().mcmc_noise(opt.p, n, n_rest, 0.5, 100.0, 0.995, 3, 9, None, None)
    xyz_end = section_ends(n, n_rest)[0]
    assert torch.equal(opt.p[xyz_end:].view(torch.int32), p0[xyz_end:].view(torch.int32))
    assert not torch.equal(opt.p[:xyz_end], p0[:xyz_end])
    assert torch.isfinite(opt.p[:xyz_end]).all()


def test_noise_binding_errors():
    g, opt, n_rest = _noise_state(1000)
    with pytest.raises(RuntimeError):
        native().mcmc_noise(opt.p, 999, n_rest, 1.0, 100.0, 0.995, 0, 0)               # layout mismatch
    with pytest.raises(RuntimeError):
        native().mcmc_noise(opt.p, 1000, n_rest, 1.0, 100.0, 0.995, 0, 0, torch.zeros(1000, 3, device=DEV).double())
    with pytest.raises(RuntimeError):
        native().mcmc_noise(opt.p, 1000, n_rest, 1.0, 100.0, 0.995, 0, 0, None, torch.zeros(3, 1000, device=DEV).t())
    with pytest.raises(RuntimeError):
        native().mcmc_noise(opt.p, 1000, n_rest, 1.0, 100.0, 0.995, 0, -1)


# end to end ---------------------------------------------------------------------------------------------------------
def test_training_with_mcmc_end_to_end():
    """A small synthetic scene learnt from 4 views of a target set of Gaussians: rasterize, photometric_loss,
    regularize, FlatAdam, inject_noise and refine for 300 steps.  N never exceeds cap_max, nothing becomes non-finite,
    the loss falls, and after every refinement no Gaussian is left below min_opacity: relocated rows sit at or above
    the clamp floor min_opacity (to the logit / sigmoid round trip, 1e-6 relative), which itself still counts as dead
    at the next refinement."""
    res = "small"
    cam = synth.make_camera(res, device=DEV)
    poses = [synth.make_pose(v, 4, device=DEV) for v in range(4)]
    bg = torch.zeros(3, device=DEV)
    target = synth.make_gaussians(3000, res, sh_degree=0, seed=5, device=DEV)
    with torch.no_grad():
        gts = [rasterize(target, T, cam, 0.3, 500.0, 100, 3.0, True, bg)[0] for T in poses]
    g = synth.make_gaussians(1500, res, sh_degree=0, seed=6, device=DEV, requires_grad=True)
    with torch.no_grad():
        g.opacity[::4] = -7.0                                      # some dead from the start
    opt = FlatAdam.for_gaussians(g)
    cfg = MCMCConfig(cap_max=2000, refine_start=20, refine_stop=290, refine_every=40)
    mcmc = MCMCDensityControl(g, opt, cfg, generator=torch.Generator(device=DEV).manual_seed(0))
    xyz_lr = opt.lrs[0]
    losses, infos = [], []
    for step in range(300):
        T = poses[step % 4]
        image, _, _, state = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, return_state=True)
        loss = photometric_loss(image, gts[step % 4], 0.2)
        loss.backward()
        mcmc.regularize(state.grad_flat)
        opt.step(state.grad_flat)
        mcmc.inject_noise(step, xyz_lr, seed=3)
        info = mcmc.refine(step)
        if info is not None:
            infos.append(info)
            o = torch.sigmoid(g.opacity.detach())
            assert g.xyz.shape[0] <= cfg.cap_max
            assert float(o.min()) >= cfg.min_opacity * (1 - 1e-6), info
            assert torch.isfinite(opt.p).all() and torch.isfinite(opt.m).all() and torch.isfinite(opt.v).all()
        for f in FIELDS:
            t = getattr(g, f)
            if t is not None:
                t.grad = None
        losses.append(float(loss))
    print(infos)
    assert len(infos) == 7 and infos[0]["relocated"] > 0 and infos[0]["added"] > 0
    assert g.xyz.shape[0] == cfg.cap_max and infos[-1]["added"] == 0
    assert torch.isfinite(opt.p).all() and np.isfinite(losses).all()
    assert np.mean(losses[-20:]) < 0.9 * np.mean(losses[:20])
