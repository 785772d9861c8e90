"""Per-step densification statistics of the reference's trainer, on device in one kernel.

The reference accumulates, after every optimizer step (splat_py/trainer.py:376-385),
    uv_grad = uv.grad.detach(); uv_grad[:, 0] *= K[0, 0]; uv_grad[:, 1] *= K[1, 1]
    self.uv_grad_accum[~culling_mask] += torch.abs(uv_grad)
    self.xyz_grad_accum += torch.abs(self.gaussians.xyz.grad.detach())
    self.grad_accum_count += (~culling_mask).int()
(two boolean-mask scatters — each a nonzero() with a host sync — and four elementwise kernels over [N]-sized
tensors); `adaptive_density_control` (:208-295) later turns them into the clone / split / delete masks.  Here the
fused rasterizer already knows the indices of the visible Gaussians (`state.vis_idx`, ascending — the order of
the compact uv), so the whole update is `gsr_densify_accumulate`, with no sync.
"""
from __future__ import annotations

import torch

from . import native


class DensificationStats:
    """The three accumulators of splat_py/trainer.py:51-66 (`reset_grad_accum`), same names and shapes."""

    def __init__(self, n_gaussians: int, device, dtype=torch.float32):
        self.uv_grad_accum = torch.zeros(n_gaussians, 2, dtype=dtype, device=device)
        self.xyz_grad_accum = torch.zeros(n_gaussians, 3, dtype=dtype, device=device)
        self.grad_accum_count = torch.zeros(n_gaussians, dtype=torch.int32, device=device)

    def accumulate(self, state, uv: torch.Tensor, xyz: torch.Tensor, K: torch.Tensor, absgrad: bool = False) -> None:
        """state: the `_ViewState` rasterize(..., return_state=True) returned; uv: the compact uv it returned (with
        `.grad` retained); xyz: the position parameter (with `.grad`); K: the camera's 3x3 intrinsic matrix.
        Like the reference, scales `uv.grad` by the focal lengths in place.

        absgrad=True (the view rendered with rasterize(..., absgrad=True)): accumulates `uv.absgrad`, the per-pixel
        absolute screen-space gradients summed (AbsGS), instead of |uv.grad|, scaled in place the same way; uv.grad
        need not be retained.  Consequences for `plan_adaptive_density_control`, which reads the accumulator as
        before:
          * the default percentile selection (use_fractional_densification) works as is; a fixed uv_grad_threshold is
            on a different scale (absgrad >= |uv.grad|, often several times larger) and must be retuned;
          * the "zero gradient" delete rule deletes fewer splats: a splat whose per-pixel pulls cancelled exactly has
            a zero uv.grad but a non-zero absgrad, and is kept."""
        if absgrad:
            g = state.uv_absgrad  # the tensor uv.absgrad also refers to
            if g is None:
                raise RuntimeError("accumulate(absgrad=True) needs a view rendered with rasterize(..., absgrad=True) "
                                   "and its backward")
        else:
            assert uv.grad is not None, "call uv.retain_grad() before backward()"
            g = uv.grad
        native().densify_accumulate(state.vis_idx32, g, xyz.grad.contiguous(), K.contiguous(),
                                    self.uv_grad_accum, self.xyz_grad_accum, self.grad_accum_count)


class WeightStats:
    """Blend-weight importance of every Gaussian, accumulated by the render forward: pass it as
    rasterize(..., weight_stats=ws) and every view adds, over the pixels p where Gaussian i takes part in the colour
    blend (the pixel is in the image and not yet saturated, alpha > 1/255), with w_ip = T_ip * alpha_ip the blend
    weight the image uses:

        weight_sum  f32 [N]  sum_p w_ip          (Mini-Splatting; float atomics: determined up to summation order)
        weight_max  f32 [N]  max_p w_ip          (RadSplat; deterministic)
        pixel_count i32 [N]  number of such p    (deterministic; wraps past 2^31 - 1)

    Indexed by Gaussian row.  Nothing is ever zeroed by the renderer: a loop over the training views (under
    torch.no_grad() or during training) leaves the totals here; `reset()` starts again.  A Gaussian that no view
    reached keeps zeros.  Stale after densification changes N (rasterize raises ValueError): make a new one."""

    def __init__(self, n_gaussians: int, device):
        self.weight_sum = torch.zeros(n_gaussians, dtype=torch.float32, device=device)
        self.weight_max = torch.zeros(n_gaussians, dtype=torch.float32, device=device)
        self.pixel_count = torch.zeros(n_gaussians, dtype=torch.int32, device=device)

    def __len__(self):
        return int(self.weight_sum.shape[0])

    def reset(self) -> None:
        self.weight_sum.zero_()
        self.weight_max.zero_()
        self.pixel_count.zero_()

    def all_reduce(self, group=None) -> None:
        """Combine the ranks' statistics in place (SUM, MAX, SUM), so that view-parallel ranks that rendered different
        views hold the same totals and take the same pruning decision."""
        import torch.distributed as dist

        dist.all_reduce(self.weight_sum, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(self.weight_max, op=dist.ReduceOp.MAX, group=group)
        dist.all_reduce(self.pixel_count, op=dist.ReduceOp.SUM, group=group)


# ---------------------------------------------------------------------------------------------------------
# Adaptive density control on the flat buffers (SURVEY.md §8(f) rank 2)
# ---------------------------------------------------------------------------------------------------------
def _inverse_sigmoid(x: float) -> float:
    """splat_py/utils.py:6-11 (numpy, float64)."""
    import math

    c = min(max(x, 1e-4), 1.0 - 1e-4)
    return math.log(c / (1.0 - c))


class DensifyConfig:
    """The fields of splat_py/config.py `SplatConfig` that adaptive density control reads, same names and
    defaults (config.py:109-158); any object with these attributes (e.g. the reference's SplatConfig) works."""

    def __init__(self, **kw):
        self.use_split = self.use_clone = self.use_delete = True
        self.adaptive_control_start, self.adaptive_control_end, self.adaptive_control_interval = 750, 6500, 100
        self.max_gaussians = 4250000
        self.delete_opacity_threshold = 0.1
        self.clone_scale_threshold = 0.01
        self.use_fractional_densification = True
        self.use_adaptive_fractional_densification = True
        self.uv_grad_percentile = 0.96
        self.scale_norm_percentile = 0.99
        self.uv_grad_threshold = 0.0002
        self.split_scale_factor = 1.6
        self.num_split_samples = 2
        self.reset_opacity_value = 0.20
        self.max_sh_band = 3
        for k, v in kw.items():
            if not hasattr(self, k):
                raise TypeError(f"unknown field {k}")
            setattr(self, k, v)


class DensificationPlan:
    """Which old row every new row comes from and what happens to it (see csrc/gsr_densify.cu)."""

    __slots__ = ("n_in", "src", "clone_row", "split_row", "xyz_sub", "xyz_add", "q_set", "scale_set", "info")

    def __init__(self, n_in):
        self.n_in = n_in
        self.src = self.clone_row = self.split_row = None
        self.xyz_sub = self.xyz_add = self.q_set = self.scale_set = None
        self.info = {}

    @property
    def n_out(self):
        return self.n_in if self.src is None else int(self.src.numel())

    def is_identity(self):
        return self.src is None


def plan_adaptive_density_control(gaussians, stats: DensificationStats, config, iteration: int) -> DensificationPlan:
    """splat_py/trainer.py:208-295 (`adaptive_density_control`) evaluated on per-row scalars only.

    Every mask is computed with the reference's own torch expressions on the same values, so the rows chosen are
    the reference's rows; instead of physically filtering / concatenating 21 tensors after each of the three
    steps (delete, clone, split), the steps compose index arrays, and ONE native pass applies the result
    (`apply_plan`).  Like the reference, reads a few scalars back (counts, quantiles): this runs every
    `adaptive_control_interval` iterations, not every step.  Consumes torch's default CUDA generator exactly like
    the reference (`torch.rand(S * samples, 3)`, trainer.py:174)."""
    from .utils import quaternion_to_rotation_torch

    xyz, quaternion, scale, opacity = gaussians.xyz.detach(), gaussians.quaternion.detach(), gaussians.scale.detach(), \
        gaussians.opacity.detach()
    n = xyz.shape[0]
    dev = xyz.device
    plan = DensificationPlan(n)
    info = plan.info
    if not (config.use_delete or config.use_clone or config.use_split):
        return plan
    # Step 1. delete: low opacity, never seen, zero gradient (trainer.py:213-229)
    keep_mask = opacity > _inverse_sigmoid(config.delete_opacity_threshold)
    keep_mask = keep_mask.squeeze(1)
    zero_view_mask = stats.grad_accum_count == 0
    zero_grad_mask = torch.norm(stats.uv_grad_accum, dim=1) == 0.0
    keep_mask &= ~zero_view_mask
    keep_mask &= ~zero_grad_mask
    delete_count = int(torch.sum(~keep_mask).item())
    info["deleted"] = delete_count if config.use_delete else 0
    uv_acc, xyz_acc, cnt = stats.uv_grad_accum, stats.xyz_grad_accum, stats.grad_accum_count
    src = None  # None = identity
    if delete_count > 0 and config.use_delete:
        src = torch.nonzero(keep_mask).squeeze(1)
        uv_acc, xyz_acc, cnt = uv_acc[keep_mask, :], xyz_acc[keep_mask, :], cnt[keep_mask]
        scale, quaternion = scale[keep_mask, :], quaternion[keep_mask, :]
    n1 = n if src is None else int(src.numel())

    def finish(src_rows, clone_row=None, split_row=None):
        if src_rows is not None:
            plan.src = src_rows.to(torch.int32).contiguous()
            plan.clone_row = None if clone_row is None else clone_row.to(torch.int32).contiguous()
            plan.split_row = None if split_row is None else split_row.to(torch.int32).contiguous()
        info["n_in"], info["n_out"] = n, plan.n_out
        return plan

    if n1 > config.max_gaussians:  # trainer.py:231-234
        info["skipped"] = "max gaussians exceeded"
        return finish(src)

    # Step 2. densify (trainer.py:236-258)
    uv_grad_avg = uv_acc / cnt.unsqueeze(1).float()
    xyz_grad_avg = xyz_acc / cnt.unsqueeze(1).float()
    uv_grad_avg_norm = torch.norm(uv_grad_avg, dim=1)
    if config.use_adaptive_fractional_densification:
        scale_factor = (float(config.adaptive_control_end - iteration)
                        / float(config.adaptive_control_end - config.adaptive_control_start) * 2.0)
    else:
        scale_factor = 1.0
    if config.use_fractional_densification:
        uv_percentile = 1.0 - (1.0 - config.uv_grad_percentile) * (scale_factor if config.use_adaptive_fractional_densification else 1.0)
        uv_split_val = torch.quantile(uv_grad_avg_norm, uv_percentile).item()
    else:
        uv_split_val = config.uv_grad_threshold
    densify_mask = uv_grad_avg_norm > uv_split_val
    scale_max = scale.exp().max(dim=-1).values
    clone_mask = densify_mask & (scale_max <= config.clone_scale_threshold)
    info["densify"], info["uv_split_val"] = int(densify_mask.sum().item()), float(uv_split_val)

    # Step 2.1 clone (trainer.py:260-268, 122-164): rows appended after the n1 survivors
    rows = torch.arange(n1, device=dev) if src is None else src  # old row of every current row
    clone_row = None
    n_clones = int(clone_mask.sum().item()) if config.use_clone else 0
    info["cloned"] = n_clones
    if n_clones > 0:
        plan.xyz_sub = (xyz_grad_avg[clone_mask, :] * 0.01).contiguous()
        clone_row = torch.cat([torch.full((n1,), -1, dtype=torch.int64, device=dev), torch.arange(n_clones, device=dev)])
        rows = torch.cat([rows, rows[clone_mask]])
        scale = torch.cat([scale, scale[clone_mask, :]])
        quaternion = torch.cat([quaternion, quaternion[clone_mask, :]])
        densify_mask = torch.cat([densify_mask, densify_mask[clone_mask]], dim=0)
        scale_max = torch.cat([scale_max, scale_max[clone_mask]], dim=0)

    # Step 2.2 split (trainer.py:270-292, 166-206): parents removed, `samples` new rows each appended at the end
    split_mask = densify_mask & (scale_max > config.clone_scale_threshold)
    scale_percentile = 1.0 - (1.0 - config.scale_norm_percentile) * scale_factor
    scale_split = torch.quantile(scale_max, scale_percentile).item()
    split_mask = split_mask | (scale_max > scale_split)
    n_split = int(split_mask.sum().item()) if config.use_split else 0
    info["split"], info["scale_split"] = n_split, float(scale_split)
    if n_split == 0:
        if src is None and n_clones == 0:
            info["n_in"] = info["n_out"] = n
            return plan  # nothing changes
        return finish(rows, clone_row)
    samples = int(config.num_split_samples)
    split_quaternion = quaternion[split_mask, :].clone().repeat(samples, 1)
    split_scale = scale[split_mask, :].clone().repeat(samples, 1)
    random_samples = torch.rand(n_split * samples, 3, device=dev)
    scale_factors = torch.exp(split_scale)
    random_samples = random_samples * scale_factors
    split_quaternion = split_quaternion / torch.norm(split_quaternion, dim=1, keepdim=True)
    split_rotations = quaternion_to_rotation_torch(split_quaternion)
    random_samples = torch.bmm(split_rotations, random_samples.unsqueeze(-1)).squeeze(-1)
    plan.xyz_add = random_samples.contiguous()
    plan.q_set = split_quaternion.contiguous()
    plan.scale_set = torch.log(torch.exp(split_scale) / config.split_scale_factor).contiguous()
    keep2 = ~split_mask
    parents = rows[split_mask]
    n_keep2 = int(rows.numel()) - n_split
    final_rows = torch.cat([rows[keep2], parents.repeat(samples)])
    if clone_row is not None:
        clone_row = torch.cat([clone_row[keep2], clone_row[split_mask].repeat(samples)])
    split_row = torch.cat([torch.full((n_keep2,), -1, dtype=torch.int64, device=dev),
                           torch.arange(n_split * samples, device=dev)])
    return finish(final_rows, clone_row, split_row)


def plan_prune(score: torch.Tensor, keep_fraction: float) -> DensificationPlan:
    """Delete-only plan keeping the ceil(keep_fraction * N) rows of largest `score` ([N], any real dtype, e.g.
    WeightStats.weight_sum).  Ties are broken by the lower row index; the kept rows stay in ascending original
    order.  keep_fraction = 1 gives the identity plan.  A NaN score ranks below every other score (it is no evidence
    that the row matters).  Reads nothing back to the host."""
    import math

    if score.dim() != 1:
        raise ValueError(f"score must have shape [N], got {tuple(score.shape)}")
    if score.is_complex() or score.dtype == torch.bool:
        raise TypeError(f"score must be real, got {score.dtype}")
    keep_fraction = float(keep_fraction)
    if not (0.0 < keep_fraction <= 1.0):
        raise ValueError(f"keep_fraction must be in (0, 1], got {keep_fraction}")
    n = int(score.shape[0])
    plan = DensificationPlan(n)
    k = min(n, math.ceil(keep_fraction * n))
    plan.info.update(n_in=n, n_out=k, deleted=n - k)
    if k == n:
        return plan
    # stable sort on the descending score: equal scores keep ascending row order, so the lower row wins a tie
    if score.is_floating_point():
        score = torch.nan_to_num(score, nan=float("-inf"))
    order = torch.sort(score, descending=True, stable=True).indices[:k]
    plan.src = torch.sort(order).values.to(torch.int32).contiguous()
    return plan


def apply_plan(plan: DensificationPlan, gaussians, optimizer=None, stats: DensificationStats = None, flat=None,
               out_flat=None):
    """Apply a plan with ONE native pass over the flat parameter buffer and (when `optimizer` is a FlatAdam) both of
    its moment buffers, then re-point the Gaussians' fields (and the optimizer) at the new buffers and reset the
    statistics to the new size (trainer.py:294 `reset_grad_accum`).  `flat`: the flat parameter buffer the fields
    are views of (default: optimizer.p).  Returns the new flat buffer."""
    n_rest = 0 if gaussians.sh is None else int(gaussians.sh.shape[2])
    if flat is None:
        assert optimizer is not None, "need the flat parameter buffer"
        flat = optimizer.p
    n_out = plan.n_out
    if not plan.is_identity():
        m = v = None
        if optimizer is not None:
            m, v = optimizer.m, optimizer.v
        out = native().densify_apply(flat, m, v, plan.n_in, n_rest, plan.src, plan.clone_row, plan.split_row,
                                     plan.xyz_sub, plan.xyz_add, plan.q_set, plan.scale_set, out_flat)
        flat = adopt_flat(gaussians, optimizer, out, n_out)
    if stats is not None:
        stats.__init__(n_out, flat.device)
    return flat


def adopt_flat(gaussians, optimizer, out, n_out: int):
    """Re-point the Gaussians' fields at views of the new flat parameter buffer out[0] (n_out rows, the Gaussians' SH
    width) and, when `optimizer` is given, its p / m / v at out[0] / out[1] / out[2] and its section ends.  Returns
    out[0]."""
    from .flat_adam import FIELDS, section_ends

    n_rest = 0 if gaussians.sh is None else int(gaussians.sh.shape[2])
    new_flat = out[0]
    ends = section_ends(n_out, n_rest)
    names = [f for f in FIELDS if getattr(gaussians, f, None) is not None]
    widths = dict(xyz=(3,), quaternion=(4,), scale=(3,), opacity=(1,), rgb=(3,), sh=(3, n_rest))
    start = 0
    for name, end in zip(names, ends):
        shape = (n_out,) + widths[name]
        numel = n_out
        for d in widths[name]:
            numel *= d
        view = new_flat[start:start + numel].view(shape)
        old = getattr(gaussians, name)
        new = torch.nn.Parameter(view) if isinstance(old, torch.nn.Parameter) else view.requires_grad_(True)
        setattr(gaussians, name, new)
        start = end
    if optimizer is not None:
        optimizer.p, optimizer.m, optimizer.v = new_flat, out[1], out[2]
        optimizer.ends = [int(e) for e in ends]
    return new_flat


class AdaptiveDensityControl:
    """`adaptive_density_control`, `reset_opacity` and `add_sh_band` of the reference's trainer
    (splat_py/trainer.py:68-112, 208-295) for Gaussians whose parameters live in ONE flat buffer driven by FlatAdam.

        adc = AdaptiveDensityControl(gaussians, optimizer, stats, config)
        ... every step: stats.accumulate(state, uv, gaussians.xyz, K)
        ... on the reference's schedule: adc.adaptive_density_control(i); adc.reset_opacity(); adc.add_sh_band()
    """

    def __init__(self, gaussians, optimizer, stats: DensificationStats, config, alloc_flat=None):
        """alloc_flat(n_floats) -> fp32 buffer: where a re-laid-out parameter buffer is to live (e.g. symmetric
        memory for the sharded optimizer); default: an ordinary allocation."""
        self.gaussians, self.optimizer, self.stats, self.config = gaussians, optimizer, stats, config
        self.alloc_flat = alloc_flat

    def adaptive_density_control(self, iteration: int):
        from .flat_adam import section_ends

        plan = plan_adaptive_density_control(self.gaussians, self.stats, self.config, iteration)
        out_flat = None
        if self.alloc_flat is not None and not plan.is_identity():
            n_rest = 0 if self.gaussians.sh is None else int(self.gaussians.sh.shape[2])
            out_flat = self.alloc_flat(section_ends(plan.n_out, n_rest)[-1])
        apply_plan(plan, self.gaussians, self.optimizer, self.stats, out_flat=out_flat)
        return plan.info

    def prune(self, score: torch.Tensor, keep_fraction: float):
        """Keep the ceil(keep_fraction * N) Gaussians of largest `score` (plan_prune; e.g. a WeightStats field) with
        their Adam moments, in one native pass (apply_plan); resets the densification statistics.  Returns the plan's
        info (n_in, n_out, deleted)."""
        from .flat_adam import section_ends

        n = self.gaussians.xyz.shape[0]
        if score.shape != (n,):
            raise ValueError(f"score has shape {tuple(score.shape)} but there are {n} gaussians")
        plan = plan_prune(score, keep_fraction)
        out_flat = None
        if self.alloc_flat is not None and not plan.is_identity():
            n_rest = 0 if self.gaussians.sh is None else int(self.gaussians.sh.shape[2])
            out_flat = self.alloc_flat(section_ends(plan.n_out, n_rest)[-1])
        apply_plan(plan, self.gaussians, self.optimizer, self.stats, out_flat=out_flat)
        return plan.info

    def reset_opacity(self):
        """trainer.py:68-75 + optimizer_manager.py:46-59: opacity <- logit(reset value), its moments <- 0."""
        from .flat_adam import FIELDS

        val = _inverse_sigmoid(self.config.reset_opacity_value)
        with torch.no_grad():
            self.gaussians.opacity.fill_(val)
        names = [f for f in FIELDS if getattr(self.gaussians, f, None) is not None]
        k = names.index("opacity")
        lo = 0 if k == 0 else self.optimizer.ends[k - 1]
        self.optimizer.m[lo:self.optimizer.ends[k]].zero_()
        self.optimizer.v[lo:self.optimizer.ends[k]].zero_()
        self.stats.__init__(self.gaussians.xyz.shape[0], self.gaussians.xyz.device)

    def add_sh_band(self, base_lr: float = 0.002, sh_lr_multiplier: float = 0.1):
        """trainer.py:77-112 + optimizer_manager.py:61-72: SH coefficients per channel 0 -> 3 -> 8 -> 15, new
        coefficients zero, the moments of the WHOLE sh tensor restart from zero (as the reference does)."""
        return add_sh_band(self.gaussians, self.optimizer, self.config.max_sh_band, self.alloc_flat, base_lr,
                           sh_lr_multiplier)


def add_sh_band(gaussians, optimizer, max_sh_band: int, alloc_flat=None, base_lr: float = 0.002,
                sh_lr_multiplier: float = 0.1):
    """One more SH band on the flat buffers (AdaptiveDensityControl.add_sh_band, MCMCDensityControl.add_sh_band):
    SH coefficients per channel 0 -> 3 -> 8 -> 15 up to `max_sh_band`, new coefficients zero, the moments of the
    WHOLE sh tensor restart from zero.  Returns whether a band was added."""
    from .flat_adam import FIELDS, section_ends

    g, opt = gaussians, optimizer
    if max_sh_band == 0:
        return False
    old = 0 if g.sh is None else int(g.sh.shape[2])
    if old == 0:
        new = 3
    elif old == 3 and max_sh_band > 1:
        new = 8
    elif old == 8 and max_sh_band > 2:
        new = 15
    else:
        return False
    n = g.xyz.shape[0]
    ends_new = section_ends(n, new)
    if alloc_flat is not None:
        flat_new = alloc_flat(ends_new[-1])
        flat_new.zero_()
    else:
        flat_new = torch.zeros(ends_new[-1], dtype=torch.float32, device=g.xyz.device)
    m_new = torch.zeros(ends_new[-1], dtype=torch.float32, device=g.xyz.device)
    v_new = torch.zeros_like(m_new)
    keep = opt.ends[4]  # xyz .. rgb sections are laid out identically (their ends do not depend on the sh width)
    flat_new[:keep].copy_(opt.p[:keep])
    m_new[:keep].copy_(opt.m[:keep])
    v_new[:keep].copy_(opt.v[:keep])
    sh_view = flat_new[keep:keep + n * 3 * new].view(n, 3, new)
    if old:
        sh_view[:, :, :old].copy_(g.sh.detach())
    widths = dict(xyz=(3,), quaternion=(4,), scale=(3,), opacity=(1,), rgb=(3,))
    start = 0
    for name, end in zip(FIELDS[:5], ends_new[:5]):
        o = getattr(g, name)
        view = flat_new[start:start + n * widths[name][0]].view((n,) + widths[name])
        setattr(g, name, torch.nn.Parameter(view) if isinstance(o, torch.nn.Parameter) else view.requires_grad_(True))
        start = end
    was_param = isinstance(g.xyz, torch.nn.Parameter)
    g.sh = torch.nn.Parameter(sh_view) if was_param else sh_view.requires_grad_(True)
    opt.p, opt.m, opt.v, opt.ends = flat_new, m_new, v_new, [int(e) for e in ends_new]
    if len(opt.lrs) == 5:
        opt.lrs.append(float(base_lr * sh_lr_multiplier))
    return True
