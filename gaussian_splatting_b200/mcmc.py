"""3DGS-MCMC densification (Kheradmand et al. 2024, "3D Gaussian Splatting as Markov Chain Monte Carlo") for
Gaussians whose parameters live in ONE flat buffer driven by FlatAdam / ShardedFlatAdam.

The Gaussian count has a fixed budget (`cap_max`), there are no opacity resets and no gradient thresholds:

  * refine (every `refine_every` steps in (refine_start, refine_stop)): "dead" Gaussians (sigmoid opacity <=
    min_opacity) are moved onto live ones sampled in proportion to opacity, then N grows by `growth` up to cap_max;
    every sampled source and its copies get the opacity and scale of `relocation`, which keeps the rendered result.
    Both steps are a plan of row indices applied by ONE native pass over the parameter buffer and both Adam moment
    buffers (gsr_mcmc_apply; moments are zero in every row the pass changes).
  * after every optimizer step: SGLD noise on the positions, xyz += lr_xyz * noise_lr * w(o) * Sigma eps
    (gsr_mcmc_noise, in place, counter-based Philox keyed by (seed, row, step): identical on every rank).
  * every step, before the optimizer: L1 regularisers on opacity and scale, added straight into the flat gradient
    buffer (`add_regularizer_grads`).

    mcmc = MCMCDensityControl(gaussians, optimizer, MCMCConfig(cap_max=...))
    ... loss.backward(); mcmc.regularize(state.grad_flat); optimizer.step(state.grad_flat)
    ... mcmc.inject_noise(step, xyz_lr, seed); mcmc.refine(step)
"""
from __future__ import annotations

import torch

from . import native
from .densify import add_sh_band, adopt_flat


class MCMCConfig:
    """3DGS-MCMC hyper-parameters (gsplat's MCMCStrategy defaults); any keyword overrides a field."""

    def __init__(self, **kw):
        self.cap_max = 1_000_000
        self.growth = 0.05          # N grows by this fraction per refinement, up to cap_max
        self.min_opacity = 0.005    # sigmoid opacity at or below this is dead
        self.n_max = 51             # copies per source the relocation formula is evaluated for (more are clamped)
        self.noise_lr = 5e5         # noise scale = xyz learning rate * noise_lr
        self.opacity_reg = 0.01     # opacity_reg * mean(sigmoid(opacity))
        self.scale_reg = 0.01       # scale_reg * mean(exp(scale))
        self.refine_start, self.refine_stop, self.refine_every = 500, 25_000, 100
        self.noise_k, self.noise_x0 = 100.0, 0.995
        self.max_sh_band = 3
        for k, v in kw.items():
            if not hasattr(self, k):
                raise TypeError(f"unknown field {k}")
            setattr(self, k, v)


class MCMCPlan:
    """Row indices only: which old row every new row comes from (src, int32 [n_out]; None = identity) and which rows
    take a relocated opacity / scale (set_row, int32 [n_out], -1 elsewhere, indexing the M drawn copies).  Copy j is
    of old row sources[j] with ratio[j] (int32 [M]) copies in all; apply_mcmc_plan evaluates their opacity and scale
    (gsr_mcmc_relocation with n_max and min_opacity) and applies the plan."""

    __slots__ = ("n_in", "src", "set_row", "sources", "ratio", "n_max", "min_opacity", "info")

    def __init__(self, n_in, config):
        self.n_in = n_in
        self.src = self.set_row = self.sources = self.ratio = None
        self.n_max, self.min_opacity = int(config.n_max), float(config.min_opacity)
        self.info = dict(n_in=n_in, n_out=n_in)

    @property
    def n_out(self):
        return self.n_in if self.src is None else int(self.src.numel())

    def is_identity(self):
        return self.src is None


def _opacity(gaussians):
    return torch.sigmoid(gaussians.opacity.detach().reshape(-1).float())


def relocation(opacity_logit: torch.Tensor, scale_log: torch.Tensor, ratio: torch.Tensor, n_max: int = 51,
               min_opacity: float = 0.005):
    """The opacity and scale of each of `ratio` copies of a Gaussian (logit opacity [n] or [n,1], log scale [n,3]):
    (new_opacity [n], sigmoid space, clamped to [min_opacity, 1 - 2^-23]; new_scale [n,3], exp space).  ratio is
    clamped to [1, n_max].  gsr_mcmc_relocation, evaluated in fp64."""
    o = torch.sigmoid(opacity_logit.detach().reshape(-1).float()).contiguous()
    s = torch.exp(scale_log.detach().float()).contiguous()
    return tuple(native().mcmc_relocation(o, s, ratio.to(torch.int32).contiguous(), int(n_max), float(min_opacity)))


def _set_copies(plan, sampled, n):
    """The drawn rows and their ratio = (times drawn) + 1."""
    plan.sources = sampled
    plan.ratio = (torch.bincount(sampled, minlength=n)[sampled] + 1).to(torch.int32).contiguous()


def _mark_sources(n_out, sampled):
    """set_row [n_out] with set_row[sampled[j]] = j (the largest j for a row sampled more than once: every such j
    holds the same relocation, and the choice is deterministic), -1 elsewhere."""
    set_row = torch.full((n_out,), -1, dtype=torch.int64, device=sampled.device)
    return set_row.scatter_reduce_(0, sampled, torch.arange(sampled.numel(), device=sampled.device), reduce="amax")


def plan_relocate(gaussians, config, generator=None) -> MCMCPlan:
    """Dead rows (sigmoid opacity <= min_opacity) each take a copy of a live row drawn with replacement in proportion
    to opacity (torch.multinomial on `generator`).  Every drawn source and its copies get the relocation of ratio =
    (times drawn) + 1.  No dead row gives the identity; every row dead leaves nothing to copy from: the identity,
    with info["skipped"].  Reads the dead count back to the host."""
    opacity = _opacity(gaussians)
    n = int(opacity.numel())
    plan = MCMCPlan(n, config)
    dead = opacity <= config.min_opacity
    n_dead = int(dead.sum().item())
    plan.info["relocated"] = 0
    if n_dead == 0:
        return plan
    if n_dead == n:
        plan.info["skipped"] = "every gaussian is dead"
        return plan
    dead_idx = torch.nonzero(dead).squeeze(1)
    alive_idx = torch.nonzero(~dead).squeeze(1)
    pick = torch.multinomial(opacity[alive_idx], n_dead, replacement=True, generator=generator)
    sampled = alive_idx[pick]
    _set_copies(plan, sampled, n)
    src = torch.arange(n, device=opacity.device)
    src[dead_idx] = sampled
    set_row = _mark_sources(n, sampled)
    set_row[dead_idx] = torch.arange(n_dead, device=opacity.device)
    plan.src, plan.set_row = src.to(torch.int32).contiguous(), set_row.to(torch.int32).contiguous()
    plan.info["relocated"] = n_dead
    return plan


def grow_count(n: int, config) -> int:
    """n_add = max(0, min(cap_max, floor((1 + growth) * n)) - n)."""
    return max(0, min(int(config.cap_max), int((1.0 + float(config.growth)) * n)) - n)


def plan_grow(gaussians, config, generator=None) -> MCMCPlan:
    """grow_count(N) rows drawn among all rows with replacement in proportion to opacity; each drawn source and its
    copies get the relocation of ratio = (times drawn) + 1, and the copies are appended after row N - 1 in draw
    order."""
    opacity = _opacity(gaussians)
    n = int(opacity.numel())
    plan = MCMCPlan(n, config)
    n_add = grow_count(n, config)
    plan.info["added"] = 0
    if n_add == 0:
        return plan
    if not float(opacity.sum().item()) > 0.0:
        plan.info["skipped"] = "no gaussian has a positive opacity"
        return plan
    sampled = torch.multinomial(opacity, n_add, replacement=True, generator=generator)
    _set_copies(plan, sampled, n)
    plan.src = torch.cat([torch.arange(n, device=opacity.device), sampled]).to(torch.int32).contiguous()
    set_row = _mark_sources(n + n_add, sampled)
    set_row[n:] = torch.arange(n_add, device=opacity.device)
    plan.set_row = set_row.to(torch.int32).contiguous()
    plan.info.update(added=n_add, n_out=n + n_add)
    return plan


def apply_mcmc_plan(plan: MCMCPlan, gaussians, optimizer=None, flat=None, out_flat=None):
    """Evaluate the plan's relocation (gsr_mcmc_relocation) and apply it with ONE native pass (gsr_mcmc_apply) over
    the flat parameter buffer (default optimizer.p) and, with an optimizer, both moment buffers; re-point the fields
    and the optimizer like densify.apply_plan.  Returns the flat buffer."""
    if flat is None:
        flat = optimizer.p
    if plan.is_identity():
        return flat
    assert gaussians.xyz.shape[0] == plan.n_in, "the plan was made for another set of gaussians"
    new_opacity, new_scale = relocation(gaussians.opacity[plan.sources], gaussians.scale[plan.sources], plan.ratio,
                                        plan.n_max, plan.min_opacity)
    n_rest = 0 if gaussians.sh is None else int(gaussians.sh.shape[2])
    m = v = None
    if optimizer is not None:
        m, v = optimizer.m, optimizer.v
    out = native().mcmc_apply(flat, m, v, plan.n_in, n_rest, plan.src, plan.set_row, new_opacity, new_scale, out_flat)
    return adopt_flat(gaussians, optimizer, out, plan.n_out)


def add_regularizer_grads(grad_flat: torch.Tensor, gaussians, config) -> None:
    """Add the gradients of opacity_reg * mean(sigmoid(opacity)) and scale_reg * mean(exp(scale)) (means over all N
    resp. 3N entries) to the opacity and scale sections of the flat gradient buffer, in place.

    Use this instead of adding the two terms to the loss: autograd would sum their gradients with the rasterizer's
    into a new `.grad` tensor of each field, which is not a view of `state.grad_flat`, so FlatAdam.step(grad_flat)
    would silently leave the regularisers out.  No host read."""
    from .flat_adam import section_ends

    n = int(gaussians.xyz.shape[0])
    if n == 0:
        return
    n_rest = 0 if gaussians.sh is None else int(gaussians.sh.shape[2])
    ends = section_ends(n, n_rest)
    assert grad_flat.numel() == ends[-1], "gradient buffer does not match the parameter layout"
    with torch.no_grad():
        if config.opacity_reg:
            o = torch.sigmoid(gaussians.opacity.detach().reshape(-1))
            grad_flat[ends[2]:ends[2] + n].add_(o * (1.0 - o), alpha=float(config.opacity_reg) / n)
        if config.scale_reg:
            grad_flat[ends[1]:ends[1] + 3 * n].add_(torch.exp(gaussians.scale.detach()).reshape(-1),
                                                    alpha=float(config.scale_reg) / (3 * n))


class MCMCDensityControl:
    """3DGS-MCMC on the flat buffers (see the module docstring).

    alloc_flat(n_floats) -> fp32 buffer: where a re-laid-out parameter buffer is to live (e.g. symmetric memory for
    the sharded optimizer); default: an ordinary allocation.  generator: the torch.Generator the refinement draws
    from (give every rank one with the same seed and state); default: torch's default generator of the device."""

    def __init__(self, gaussians, optimizer, config: MCMCConfig, alloc_flat=None, generator=None):
        self.gaussians, self.optimizer, self.config = gaussians, optimizer, config
        self.alloc_flat, self.generator = alloc_flat, generator

    def is_refine_step(self, iteration: int) -> bool:
        c = self.config
        return c.refine_start < iteration < c.refine_stop and iteration % c.refine_every == 0

    def _apply(self, plan):
        from .flat_adam import section_ends

        out_flat = None
        if self.alloc_flat is not None and not plan.is_identity():
            n_rest = 0 if self.gaussians.sh is None else int(self.gaussians.sh.shape[2])
            out_flat = self.alloc_flat(section_ends(plan.n_out, n_rest)[-1])
        apply_mcmc_plan(plan, self.gaussians, self.optimizer, out_flat=out_flat)

    def refine(self, iteration: int):
        """On a refinement step (is_refine_step): relocate the dead Gaussians, then grow.  Returns the info of both
        plans (n_in, relocated, added, n_out, and "skipped" when a step had nothing to work with), or None on any
        other step.  Reads a few counts back to the host."""
        if not self.is_refine_step(iteration):
            return None
        n_in = int(self.gaussians.xyz.shape[0])
        reloc = plan_relocate(self.gaussians, self.config, self.generator)
        self._apply(reloc)
        grow = plan_grow(self.gaussians, self.config, self.generator)
        self._apply(grow)
        info = dict(iter=iteration, n_in=n_in, relocated=reloc.info["relocated"], added=grow.info["added"],
                    n_out=int(self.gaussians.xyz.shape[0]))
        for p in (reloc, grow):
            if "skipped" in p.info:
                info.setdefault("skipped", []).append(p.info["skipped"])
        return info

    def inject_noise(self, step: int, xyz_lr: float, seed: int = 0) -> None:
        """xyz += xyz_lr * noise_lr * w(o) * Sigma eps in place (gsr_mcmc_noise), draws keyed by (seed, row, step).
        Run after the optimizer step.  No host read."""
        g = self.gaussians
        n_rest = 0 if g.sh is None else int(g.sh.shape[2])
        c = self.config
        native().mcmc_noise(self.optimizer.p, int(g.xyz.shape[0]), n_rest, float(xyz_lr) * float(c.noise_lr),
                            float(c.noise_k), float(c.noise_x0), int(seed), int(step))

    def regularize(self, grad_flat) -> None:
        """add_regularizer_grads into the flat gradient buffer (a tensor or a native-layout GradientBucket)."""
        if hasattr(grad_flat, "flat") and hasattr(grad_flat, "layout"):
            if grad_flat.layout != "native":
                raise ValueError("regularize needs a bucket in the native flat layout")
            grad_flat = grad_flat.flat
        add_regularizer_grads(grad_flat, self.gaussians, self.config)

    def add_sh_band(self, base_lr: float = 0.002, sh_lr_multiplier: float = 0.1):
        """densify.add_sh_band: the same band schedule as AdaptiveDensityControl.add_sh_band."""
        return add_sh_band(self.gaussians, self.optimizer, self.config.max_sh_band, self.alloc_flat, base_lr,
                           sh_lr_multiplier)
