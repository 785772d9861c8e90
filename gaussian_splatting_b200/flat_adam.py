"""Adam on the flat Gaussian-parameter buffer (SURVEY.md §8(f) rank 2), the optimizer step that follows the
rasterizer's backward in the reference's training loop (splat_py/trainer.py:374 `optimizer.step()` on the
parameter groups of splat_py/optimizer_manager.py:13-44).

All parameters live in ONE flat fp32 buffer laid out exactly like the gradients the fused backward produces
(`state.grad_flat`: [xyz | quaternion | scale | opacity | rgb | sh], sections 16-byte aligned), so the whole step
is one streaming kernel (`gsr_adam_step`, csrc/gsr_adam.cu) instead of a multi-tensor sweep per operation, with
torch.optim.Adam's values (same per-element operation order as torch's CUDA kernels).

`ShardedFlatAdam` is the view-parallel form: parameters and gradients sit in symmetric memory, rank r owns 1/world
of the elements and of the optimizer state, and ONE kernel per rank does reduce-scatter (peer loads of the
gradient shard over NVLink) + Adam + all-gather (peer stores of the updated parameters).

Both take a visibility mask (`FlatAdam.step(grad, visible=state.visible)`, `ShardedFlatAdam(..., visible_sym=...)`):
the step then updates only the rows the view saw, in one native kernel (`gsr_adam_step_selective`,
csrc/gsr_adam_selective.cu) that reads and writes nothing of the other rows — the sparse Adam of Taming 3DGS and
gsplat's SelectiveAdam, with torch.optim.Adam's values on the rows it updates.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch

from . import native

FIELDS = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")  # section order of the flat layout
REFERENCE_LR_MULTIPLIERS = dict(xyz=0.1, quaternion=2.0, scale=5.0, opacity=10.0, rgb=2.0, sh=0.1)  # config.py:77-88


def section_ends(n_gaussians: int, n_sh_rest: int):
    """Exclusive end (in elements) of each section of the flat layout; the last one is the buffer length."""
    return list(native().flat_section_ends(int(n_gaussians), int(n_sh_rest)))


def sh_rest_of_layout(ends: Sequence[int], n_gaussians: int) -> int:
    """n_sh_rest of the flat layout `ends` of n_gaussians rows.  Raises ValueError when no SH width gives that
    layout for that many rows (a visibility mask from before densification changed the number of gaussians)."""
    n, ends = int(n_gaussians), [int(e) for e in ends]
    if len(ends) == 5:
        cands = [0]
    elif len(ends) == 6 and n > 0:
        k = (ends[5] - ends[4]) // (3 * n)
        # the 16-byte padding adds at most 3 floats; with n == 1 that can hold a whole coefficient, and both widths
        # give the same layout.  Take the wider: it covers every real coefficient, and a zero padding tail stays zero
        # under the step (as it does under the dense step)
        cands = [k, k - 1]
    else:
        cands = []
    for c in cands:
        if c >= 0 and section_ends(n, c) == ends:
            return c
    raise ValueError(f"the visibility mask has {n} rows but the optimizer's parameter buffer has a different number of "
                     "gaussians (a stale mask: densification, pruning or relocation changed N since it was made)")


def check_visible(visible: torch.Tensor, device: torch.device) -> None:
    if not isinstance(visible, torch.Tensor):
        raise TypeError("visible must be a tensor (the rasterizer's state.visible)")
    if visible.dtype not in (torch.bool, torch.uint8):
        raise TypeError(f"visible must be a bool or uint8 tensor, not {visible.dtype}")
    if visible.device != device:
        raise ValueError(f"visible is on {visible.device}, the parameters on {device}")


def flatten_gaussians(gaussians, flat: Optional[torch.Tensor] = None):
    """Move the parameters of `gaussians` into one flat buffer and re-point its fields to views of it.

    Returns (flat, ends, names).  `flat` may be a caller-provided buffer of the right length (e.g. symmetric
    memory).  The fields stay leaf tensors with requires_grad=True, so autograd and the rasterizer see no change.
    """
    n = gaussians.xyz.shape[0]
    n_rest = 0 if gaussians.sh is None else gaussians.sh.shape[2]
    ends = section_ends(n, n_rest)
    names = [f for f in FIELDS if getattr(gaussians, f, None) is not None]
    assert len(names) == len(ends)
    dev = gaussians.xyz.device
    if flat is None:
        flat = torch.zeros(ends[-1], dtype=torch.float32, device=dev)
    else:
        assert flat.numel() == ends[-1] and flat.dtype == torch.float32 and flat.is_contiguous()
        flat.zero_()
    start = 0
    for name, end in zip(names, ends):
        old = getattr(gaussians, name)
        view = flat[start:start + old.numel()].view(old.shape)
        view.copy_(old.detach())
        # the reference's trainer holds nn.Parameters on an nn.Module (colmap_splat.py:58-63): keep the kind
        new = torch.nn.Parameter(view) if isinstance(old, torch.nn.Parameter) else view.requires_grad_(True)
        setattr(gaussians, name, new)
        start = end
    return flat, ends, names


class FlatAdam:
    """torch.optim.Adam(betas, eps, no weight decay, no amsgrad) over the flat buffer, one learning rate per section."""

    def __init__(self, flat_params: torch.Tensor, ends: Sequence[int], lrs: Sequence[float], betas=(0.9, 0.999),
                 eps: float = 1e-8):
        assert flat_params.numel() == ends[-1] and len(lrs) == len(ends)
        self.p, self.ends, self.lrs = flat_params, [int(e) for e in ends], [float(x) for x in lrs]
        self.betas, self.eps, self.t = (float(betas[0]), float(betas[1])), float(eps), 0
        self.m = torch.zeros_like(flat_params)
        self.v = torch.zeros_like(flat_params)

    @classmethod
    def for_gaussians(cls, gaussians, base_lr: float = 0.002, multipliers: Dict[str, float] = REFERENCE_LR_MULTIPLIERS,
                      **kw):
        flat, ends, names = flatten_gaussians(gaussians)
        return cls(flat, ends, [base_lr * multipliers[n] for n in names], **kw)

    def step(self, grad_flat, visible: Optional[torch.Tensor] = None) -> None:
        """`grad_flat`: the flat gradient buffer in the native layout (`state.grad_flat`), or a
        view_parallel.GradientBucket — which must be in the native layout (a "packed" bucket would apply the
        gradients to the wrong sections with the wrong learning rates, so it is rejected).

        `visible` (CUDA bool / uint8 [N], nonzero = seen; the rasterizer's `state.visible`): update only those rows.
        Every element of a visible row gets exactly the dense step's arithmetic, bit for bit; every other row keeps
        p, m and v bit-unchanged and its gradient is ignored, whatever it holds.  The step count still goes up by one
        and drives every row's bias correction (as in Taming 3DGS's sparse Adam and gsplat's SelectiveAdam), so an
        all-nonzero mask is exactly the dense step.  What follows from ignoring those gradients:
          * gradients added to rows the view did not see are dropped — MCMC's `regularize()` terms reach only the
            visible rows;
          * accumulating several views into one gradient buffer before one step needs the OR of their masks
            (`visible_a | visible_b`; `view_parallel.all_reduce_visibility` across ranks);
          * a mask is valid for one layout: after densification, pruning, relocation or a new SH band changed N, an
            old mask raises ValueError.
        No host synchronisation."""
        if hasattr(grad_flat, "flat") and hasattr(grad_flat, "layout"):
            if grad_flat.layout != "native":
                raise ValueError("FlatAdam.step needs a bucket in the native flat layout "
                                 "(GradientBucket.adopt(flat, gaussians) or GradientBucket.native_layout)")
            grad_flat = grad_flat.flat
        assert grad_flat.numel() == self.p.numel(), "gradient buffer does not match the parameter layout"
        if visible is None:
            self.t += 1
            native().adam_step_flat(self.p, grad_flat, self.m, self.v, self.ends, self.lrs, self.betas[0],
                                    self.betas[1], self.eps, self.t)
            return
        check_visible(visible, self.p.device)
        n_rest = sh_rest_of_layout(self.ends, visible.numel())
        native().adam_step_selective(self.p, grad_flat, self.m, self.v, visible.contiguous(), n_rest, self.ends,
                                     self.lrs, self.betas[0], self.betas[1], self.eps, self.t + 1)
        self.t += 1


class ShardedFlatAdam:
    """View-parallel optimizer step over NVLink peer memory (one process per GPU).

    params_flat and grads_flat must have been allocated with torch.distributed._symmetric_memory.empty() and are
    rendezvoused here; rank r owns elements [lo, hi) (16-byte aligned split) and keeps Adam's m, v for that range
    only.  step(): barrier (every rank's backward has written its gradients) -> fused kernel -> barrier (every
    rank's parameter buffer holds the new values).  The gradient average over ranks is part of the kernel.

    visible_sym (optional): a symmetric-memory uint8 [N] buffer (torch.distributed._symmetric_memory.empty) that the
    caller fills with its view's mask (`visible_sym.copy_(state.visible)`) before every step().  The step then
    updates only the rows ANY rank's view saw — the OR of the masks, read over peer memory — with the rank-averaged
    gradient, and leaves every other row bit-unchanged on every replica (FlatAdam.step(visible=...) explains what
    follows from that).  N is fixed by the buffer: a re-layout that changes N needs a new buffer and a new optimizer.
    Without it, step() is the dense step.
    """

    def __init__(self, params_flat: torch.Tensor, grads_flat: torch.Tensor, ends: Sequence[int], lrs: Sequence[float],
                 group=None, betas=(0.9, 0.999), eps: float = 1e-8, visible_sym: Optional[torch.Tensor] = None):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem

        group = group if group is not None else dist.group.WORLD
        self.group = group
        self.hp = symm_mem.rendezvous(params_flat, group)
        self.hg = symm_mem.rendezvous(grads_flat, group)
        self.rank, self.world = self.hp.rank, self.hp.world_size
        n = params_flat.numel()
        assert n == ends[-1] == grads_flat.numel() and n % 4 == 0
        per = ((n // 4 + self.world - 1) // self.world) * 4
        self.lo, self.hi = min(n, self.rank * per), min(n, (self.rank + 1) * per)
        self.p, self.g = params_flat, grads_flat
        self.ends, self.lrs = [int(e) for e in ends], [float(x) for x in lrs]
        self.betas, self.eps, self.t = (float(betas[0]), float(betas[1])), float(eps), 0
        self.m = torch.zeros(self.hi - self.lo, dtype=torch.float32, device=params_flat.device)
        self.v = torch.zeros_like(self.m)
        self.param_ptrs = [int(x) for x in self.hp.buffer_ptrs]
        self.grad_ptrs = [int(x) for x in self.hg.buffer_ptrs]
        self.visible = visible_sym
        if visible_sym is not None:
            if visible_sym.dtype != torch.uint8 or visible_sym.device != params_flat.device:
                raise TypeError("visible_sym must be a uint8 symmetric-memory buffer on the parameters' device")
            self.n_rest = sh_rest_of_layout(self.ends, visible_sym.numel())
            self.hvis = symm_mem.rendezvous(visible_sym, group)
            self.visible_ptrs = [int(x) for x in self.hvis.buffer_ptrs]

    def full_state(self):
        """(m, v) of the WHOLE flat buffer on every rank (all-gather of the shards): what a re-layout of the
        parameter buffer (densification, a new SH band) needs before the state is sharded again."""
        import torch.distributed as dist

        n = self.p.numel()
        per = ((n // 4 + self.world - 1) // self.world) * 4
        out = []
        for shard in (self.m, self.v):
            padded = torch.zeros(per, dtype=torch.float32, device=shard.device)
            padded[:shard.numel()].copy_(shard)
            full = torch.empty(per * self.world, dtype=torch.float32, device=shard.device)
            dist.all_gather_into_tensor(full, padded, group=self.group)
            out.append(full[:n].contiguous())
        return out[0], out[1]

    def load_full_state(self, m_full: torch.Tensor, v_full: torch.Tensor, t: int) -> None:
        """Keep this rank's range of a full (m, v) pair (after a re-layout) and the step count."""
        assert m_full.numel() == self.p.numel() == v_full.numel()
        self.m.copy_(m_full[self.lo:self.hi])
        self.v.copy_(v_full[self.lo:self.hi])
        self.t = int(t)

    def step(self) -> None:
        self.t += 1
        self.hg.barrier(channel=0)  # all gradients (and masks) written (stream-ordered, device-side)
        if self.visible is None:
            native().adam_step_sharded(self.lo, self.hi, self.grad_ptrs, self.param_ptrs, self.rank, self.m, self.v,
                                       self.ends, self.lrs, self.betas[0], self.betas[1], self.eps, self.t)
        else:
            native().adam_step_selective_sharded(self.lo, self.hi, self.grad_ptrs, self.param_ptrs, self.visible_ptrs,
                                                 self.rank, self.m, self.v, self.visible.numel(), self.n_rest,
                                                 self.ends, self.lrs, self.betas[0], self.betas[1], self.eps, self.t)
        self.hp.barrier(channel=1)  # all parameter replicas updated
