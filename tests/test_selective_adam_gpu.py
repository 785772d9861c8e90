"""Visibility-masked Adam on the flat buffers (csrc/gsr_adam_selective.cu) — needs a GPU.

  1. an all-visible mask is FlatAdam's dense step, bit for bit;
  2. random masks: rows not visible keep p, m, v bit-unchanged, visible rows equal a dense step of a copy bit for
     bit, and everything agrees with the CPU oracle;
  3. end to end: rasterize -> L1 -> backward -> step(state.grad_flat, visible=state.visible) against torch.optim.Adam
     per field with the masked rows restored;
  4. after densification and a new SH band, the step follows the new layout and an old mask is refused;
  5. the sharded kernel with emulated ranks on one GPU, and ShardedFlatAdam over real symmetric memory on 2 GPUs."""
import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import native, synth
from gaussian_splatting_b200.flat_adam import (FIELDS, REFERENCE_LR_MULTIPLIERS, FlatAdam, flatten_gaussians,
                                               section_ends, sh_rest_of_layout)
from gaussian_splatting_b200.rasterize import rasterize
from oracle import adam_oracle

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def element_rows(ends, n):
    """int64 [len]: the row of every element of the flat layout, -1 in the section padding."""
    n_rest = sh_rest_of_layout(ends, n)
    widths = [3, 4, 3, 1, 3, 3 * n_rest][:len(ends)]
    rows = torch.full((ends[-1],), -1, dtype=torch.int64, device=dev())
    start = 0
    for w, end in zip(widths, ends):
        rows[start:start + n * w] = torch.arange(n * w, device=dev()) // w
        start = end
    return rows


def element_mask(ends, n, visible):
    rows = element_rows(ends, n)
    return (rows >= 0) & (visible != 0)[rows.clamp(min=0)]


def lrs_for(ends):
    return [0.002 * REFERENCE_LR_MULTIPLIERS[f] for f in FIELDS[:len(ends)]]


def copy_of(opt):
    c = FlatAdam(opt.p.clone(), opt.ends, opt.lrs, opt.betas, opt.eps)
    c.m.copy_(opt.m)
    c.v.copy_(opt.v)
    c.t = opt.t
    return c


def selective_step_checked(opt, grad, visible):
    """opt.step(grad, visible) must equal: a dense step of a copy where visible, the old values elsewhere (bitwise)."""
    n = visible.numel()
    ref = copy_of(opt)
    ref.step(grad)
    before = [opt.p.clone(), opt.m.clone(), opt.v.clone()]
    opt.step(grad, visible=visible)
    on = element_mask(opt.ends, n, visible)
    for got, dense, old in zip((opt.p, opt.m, opt.v), (ref.p, ref.m, ref.v), before):
        assert torch.equal(got[~on].view(torch.int32), old[~on].view(torch.int32))
        assert torch.equal(got[on].view(torch.int32), dense[on].view(torch.int32))
    assert opt.t == ref.t


@pytest.mark.parametrize("n", [1001, 40000])
@pytest.mark.parametrize("n_rest", [0, 3, 8, 15])
def test_all_visible_is_the_dense_step_bitwise(n, n_rest):
    ends = section_ends(n, n_rest)
    assert len(ends) == (5 if n_rest == 0 else 6)
    gen = torch.Generator(device=dev()).manual_seed(n + n_rest)
    pad = element_rows(ends, n) < 0  # section padding holds zeros, as in every flat buffer of the library
    p0 = torch.randn(ends[-1], device=dev(), generator=gen).masked_fill_(pad, 0.0)
    dense, sel = FlatAdam(p0.clone(), ends, lrs_for(ends)), FlatAdam(p0.clone(), ends, lrs_for(ends))
    vis_u8 = torch.full((n,), 7, dtype=torch.uint8, device=dev())
    vis_b = torch.ones(n, dtype=torch.bool, device=dev())
    for step in range(5):
        g = torch.randn(ends[-1], device=dev(), generator=gen) * 10.0 ** (-4 * torch.rand(ends[-1], device=dev(),
                                                                                            generator=gen))
        g.masked_fill_(pad, 0.0)
        dense.step(g)
        sel.step(g, visible=vis_u8 if step % 2 else vis_b)
    for a, b in ((dense.p, sel.p), (dense.m, sel.m), (dense.v, sel.v)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("density", [0.0, 0.01, 0.3, 0.7])
@pytest.mark.parametrize("n_rest", [3, 15])
def test_random_masks(density, n_rest):
    n = 40001  # not a multiple of 4: every section has padding
    ends = section_ends(n, n_rest)
    lrs = lrs_for(ends)
    rng = np.random.default_rng(int(density * 100) + n_rest)
    p0 = rng.standard_normal(ends[-1]).astype(np.float32)
    opt = FlatAdam(torch.tensor(p0, device=dev()), ends, lrs)
    starts = [0] + ends[:-1]
    lr_el = np.zeros(ends[-1])
    for s, e, lr in zip(starts, ends, lrs):
        lr_el[s:e] = lr
    p, m, v = p0.copy(), np.zeros_like(p0), np.zeros_like(p0)
    for step in range(1, 6):
        g = (rng.standard_normal(ends[-1]) * 10.0 ** rng.uniform(-7, 0, ends[-1])).astype(np.float32)
        g[rng.random(ends[-1]) < 0.25] = 0.0
        vis = torch.tensor(rng.random(n) < density, device=dev())
        gt = torch.tensor(g, device=dev())
        selective_step_checked(opt, gt, vis)
        on = element_mask(ends, n, vis).cpu().numpy()
        pn, mn, vn = adam_oracle.adam_step(p, g, m, v, lr_el, step)
        p, m, v = np.where(on, pn, p), np.where(on, mn, m), np.where(on, vn, v)
    mine = opt.p.cpu().numpy()
    assert np.abs(mine - p).max() <= 1e-6 * np.abs(p).max()
    np.testing.assert_allclose(opt.m.cpu().numpy(), m, rtol=2e-7, atol=1e-35)
    np.testing.assert_allclose(opt.v.cpu().numpy(), v, rtol=2e-7, atol=1e-35)
    if density == 0.0:
        assert np.array_equal(mine.view(np.int32), p0.view(np.int32)) and not opt.m.any() and not opt.v.any()


def test_training_steps_match_torch_optimizer_with_masked_rows_restored():
    """rasterize -> L1 -> backward -> FlatAdam.step(state.grad_flat, visible=state.visible), five steps from poses
    that cull part of the scene, against torch.optim.Adam per field whose masked rows are restored after each step."""
    res, n = "tiny", 3000

    def make():
        return synth.make_gaussians(n, res, sh_degree=3, seed=0, device=dev(), requires_grad=True,
                                    sigma_px=(2.0, 0.5, 0.5, 8.0))

    cam = synth.make_camera(res, device=dev())
    bg = torch.full((3,), 0.5, device=dev())
    target = torch.rand(cam.height, cam.width, 3, device=dev(), generator=torch.Generator(device=dev()).manual_seed(3))
    ga, gb = make(), make()
    flat, ends, names = flatten_gaussians(ga)
    lrs = [0.002 * REFERENCE_LR_MULTIPLIERS[f] for f in names]
    fa = FlatAdam(flat, ends, lrs)
    params_b = [getattr(gb, f) for f in names]
    tb = torch.optim.Adam([dict(params=[t], lr=lr) for t, lr in zip(params_b, lrs)])
    init = {f: getattr(ga, f).detach().clone() for f in names}
    seen = torch.zeros(n, dtype=torch.bool, device=dev())
    for it, view in enumerate((0, 5, -5, 5, 0)):  # yaw 0, +-15 degrees; no culling padding
        T = synth.make_pose(view, 1, device=dev())
        for g in (ga, gb):
            for f in names:
                getattr(g, f).grad = None
        img, _, _, st = rasterize(ga, T, cam, 0.3, 500.0, 0, 3.0, True, bg, return_state=True)
        (img - target).abs().mean().backward()
        vis = st.visible != 0
        assert 0 < int(vis.sum()) < n, "the pose should cull part of the scene"
        seen |= vis
        fa.step(st.grad_flat, visible=st.visible)
        img2, _, _ = rasterize(gb, T, cam, 0.3, 500.0, 0, 3.0, True, bg)
        (img2 - target).abs().mean().backward()
        hidden = ~vis
        old = []
        for t in params_b:
            s = tb.state.get(t, {})
            old.append((t.detach()[hidden].clone(), s["exp_avg"][hidden].clone() if s else None,
                        s["exp_avg_sq"][hidden].clone() if s else None))
        tb.step()
        with torch.no_grad():
            for t, (p_old, m_old, v_old) in zip(params_b, old):
                s = tb.state[t]
                t[hidden] = p_old
                s["exp_avg"][hidden] = m_old if m_old is not None else 0.0
                s["exp_avg_sq"][hidden] = v_old if v_old is not None else 0.0
    never = ~seen
    assert int(never.sum()) > 0
    for f in names:
        assert torch.equal(getattr(ga, f).detach()[never], init[f][never]), f
    on = element_mask(ends, n, seen)
    assert not fa.m[~on].any() and not fa.v[~on].any()
    for f in names:
        a, b = getattr(ga, f).detach(), getattr(gb, f).detach()
        lr = lrs[names.index(f)]
        frac = float(((a - b).abs() > 1e-6 + 1e-5 * b.abs()).float().mean())
        assert float((a - b).abs().max()) <= 2 * 5 * lr + 1e-6 and frac < 0.01, (f, float((a - b).abs().max()), frac)


def test_step_follows_densification_and_a_new_sh_band():
    from gaussian_splatting_b200.densify import AdaptiveDensityControl, DensificationStats, DensifyConfig
    from tests.test_densify_gpu import flat_setup
    from tests.test_densify_plan import make_case

    P, M, V, uv_acc, xyz_acc, cnt = make_case(1001, seed=4, device=dev(), n_rest=3)
    g, opt = flat_setup(P, M, V)
    stats = DensificationStats(1001, dev())
    stats.uv_grad_accum, stats.xyz_grad_accum, stats.grad_accum_count = uv_acc, xyz_acc, cnt
    adc = AdaptiveDensityControl(g, opt, stats, DensifyConfig())
    gen = torch.Generator(device=dev()).manual_seed(2)
    old_mask = torch.rand(1001, device=dev(), generator=gen) < 0.5
    selective_step_checked(opt, torch.randn(opt.p.numel(), device=dev(), generator=gen) * 1e-3, old_mask)
    torch.manual_seed(100)
    adc.adaptive_density_control(800)
    n = g.xyz.shape[0]
    assert n != 1001
    t = opt.t
    with pytest.raises(ValueError, match="stale mask"):
        opt.step(torch.zeros_like(opt.p), visible=old_mask)
    assert opt.t == t
    mask = torch.rand(n, device=dev(), generator=gen) < 0.5
    selective_step_checked(opt, torch.randn(opt.p.numel(), device=dev(), generator=gen) * 1e-3, mask)
    assert adc.add_sh_band() and g.sh.shape[2] == 8
    assert sh_rest_of_layout(opt.ends, n) == 8
    selective_step_checked(opt, torch.randn(opt.p.numel(), device=dev(), generator=gen) * 1e-3, mask)


def _sharded_split(n, world):
    per = ((n // 4 + world - 1) // world) * 4
    return [(min(n, r * per), min(n, (r + 1) * per)) for r in range(world)]


@pytest.mark.parametrize("world", [2, 3])
def test_selective_sharded_kernel_emulated_ranks_on_one_gpu(world):
    """gsr_adam_step_selective_sharded with `world` emulated ranks on one device, each rank with its own parameter,
    gradient and mask buffer: equals a selective FlatAdam step on the rank-ordered mean gradient with the OR of the
    masks, and every replica stays bit-identical."""
    n_g, n_rest = 5001, 15
    ends = section_ends(n_g, n_rest)
    lrs = lrs_for(ends)
    total = ends[-1]
    gen = torch.Generator(device=dev()).manual_seed(11)
    p0 = torch.randn(total, device=dev(), generator=gen)
    params = [p0.clone() for _ in range(world)]
    grads = [torch.empty(total, device=dev()) for _ in range(world)]
    masks = [torch.empty(n_g, dtype=torch.uint8, device=dev()) for _ in range(world)]
    split = _sharded_split(total, world)
    ms = [torch.zeros(hi - lo, device=dev()) for lo, hi in split]
    vs = [torch.zeros(hi - lo, device=dev()) for lo, hi in split]
    ref = FlatAdam(p0.clone(), ends, lrs)
    seen = torch.zeros(n_g, dtype=torch.bool, device=dev())
    for step in range(1, 5):
        for r in range(world):
            grads[r].copy_(torch.randn(total, device=dev(), generator=gen) *
                           10.0 ** (-3.0 * torch.rand(total, device=dev(), generator=gen)))
            masks[r].copy_((torch.rand(n_g, device=dev(), generator=gen) < 0.2).to(torch.uint8) * (r + 1))
        mean = grads[0].clone()
        for r in range(1, world):
            mean += grads[r]          # rank order, like the kernel
        mean *= 1.0 / world
        union = torch.stack(masks).amax(0)
        seen |= union != 0
        ref.step(mean, visible=union)
        gp, pp, vp = ([int(t.data_ptr()) for t in ts] for ts in (grads, params, masks))
        for r, (lo, hi) in enumerate(split):
            native().adam_step_selective_sharded(lo, hi, gp, pp, vp, r, ms[r], vs[r], n_g, n_rest, ends, lrs, 0.9,
                                                 0.999, 1e-8, step)
        torch.cuda.synchronize()
        for r in range(1, world):
            assert torch.equal(params[r].view(torch.int32), params[0].view(torch.int32)), (r, step)
        err = float((params[0] - ref.p).abs().max())
        assert err <= 1e-6 * float(ref.p.abs().max()), (step, err)
    on = element_mask(ends, n_g, seen)
    assert torch.equal(params[0][~on].view(torch.int32), p0[~on].view(torch.int32))
    m_all, v_all = torch.cat(ms), torch.cat(vs)
    assert not m_all[~on].any() and not v_all[~on].any()
    assert float((m_all - ref.m).abs().max()) <= 1e-6 * float(ref.m.abs().max())
    assert float((v_all - ref.v).abs().max()) <= 1e-6 * float(ref.v.abs().max())


def _sharded_worker(rank, world, port, q):
    import os

    import torch.distributed as dist
    import torch.distributed._symmetric_memory as symm_mem

    from gaussian_splatting_b200.flat_adam import ShardedFlatAdam
    from gaussian_splatting_b200.view_parallel import all_reduce_visibility

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    d = torch.device(f"cuda:{rank}")
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=d)
    try:
        n_g, n_rest = 20001, 15
        ends = section_ends(n_g, n_rest)
        lrs = lrs_for(ends)
        total = ends[-1]
        p_sym = symm_mem.empty(total, dtype=torch.float32, device=d)
        g_sym = symm_mem.empty(total, dtype=torch.float32, device=d)
        vis_sym = symm_mem.empty(n_g, dtype=torch.uint8, device=d)
        gen = torch.Generator(device=d).manual_seed(5)       # same parameters on every rank
        p_sym.copy_(torch.randn(total, device=d, generator=gen))
        opt = ShardedFlatAdam(p_sym, g_sym, ends, lrs, visible_sym=vis_sym)
        ref = FlatAdam(p_sym.clone(), ends, lrs)
        worst = 0.0
        for step in range(4):
            grank = torch.Generator(device=d).manual_seed(100 + 10 * step + rank)  # a different "view" per rank
            g_sym.copy_(torch.randn(total, device=d, generator=grank) * 1e-2)
            vis_sym.copy_((torch.rand(n_g, device=d, generator=grank) < 0.3).to(torch.uint8))
            mean = g_sym.clone()
            dist.all_reduce(mean, op=dist.ReduceOp.SUM)
            mean /= world
            ref.step(mean, visible=all_reduce_visibility(vis_sym.clone()))  # NCCL path: OR of the masks
            opt.step()
            torch.cuda.synchronize()
            worst = max(worst, float((p_sym - ref.p).abs().max()) / float(ref.p.abs().max()))
        gathered = [torch.empty_like(p_sym) for _ in range(world)]
        dist.all_gather(gathered, p_sym.clone())
        same = all(torch.equal(gathered[0], t) for t in gathered)
        if rank == 0:
            q.put((worst, same))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs (NVLink peer memory)")
def test_selective_sharded_adam_matches_allreduce_plus_flat():
    import socket

    import torch.multiprocessing as mp

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    worst, same = q.get(timeout=300)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert same, "parameter replicas differ"
    assert worst < 1e-6, worst
