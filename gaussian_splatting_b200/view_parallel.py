"""View-parallel use of the rasterizer: one process per GPU, Gaussians replicated, rank r renders its own
view, and the parameter gradients are summed over ranks with ONE collective on a flat bucket.

This is the outer-loop exchange of SURVEY.md §8(e)/(f): the raster path itself has no collective (views are
independent); a trainer that feeds `world_size` views per optimizer step needs exactly one all-reduce of
  d{xyz 3, rgb 3, opacity 1, scale 3, quaternion 4, sh 3K} = 59 floats (K = 15) = 236 B per Gaussian,
plus — every densification interval, not every step — the reference's per-view statistics
(`uv_grad_accum`, `xyz_grad_accum`, `grad_accum_count`; splat_py/trainer.py:51-66, 379-385).

The gradients are contiguous without a flatten copy, in one of two ways:
  * `GradientBucket.adopt(state.grad_flat, params)` — the fused backward already writes all parameter gradients
    of a view into ONE allocation (`rasterize(..., return_state=True)` exposes it as `state.grad_flat`) and
    autograd installs views of it as `.grad`; the bucket is that allocation (one view per rank per step);
  * `GradientBucket(params).attach()` — `.grad` of every parameter is made a view into a flat buffer BEFORE the
    backward pass and autograd accumulates into it in place (several views per rank per step).
Either way `all_reduce()` hands one buffer to NCCL: one launch, `async_op=True` to overlap it with other work.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence

import torch
import torch.distributed as dist

PARAM_FIELDS = ("xyz", "rgb", "opacity", "scale", "quaternion", "sh")


def views_of_rank(step: int, rank: int, world_size: int, n_views: int) -> int:
    """The view rank `rank` renders at optimizer step `step`: consecutive views, one per rank, wrapping
    around the training set (same schedule as bench.py)."""
    return (step * world_size + rank) % n_views


class GradientBucket:
    """Flat gradient storage for a set of parameters.

    bucket = GradientBucket([g.xyz, g.rgb, ...]); bucket.attach() once (and again whenever the parameter set
    changes, e.g. after densification); then per step: bucket.zero(); loss.backward(); bucket.all_reduce().
    """

    # `layout` says how `flat` is arranged, because consumers of the flat buffer depend on it:
    #   "native"  the rasterizer's / FlatAdam's layout: sections in flat_adam.FIELDS order
    #             [xyz | quaternion | scale | opacity | rgb | sh], every section end 16-byte aligned
    #             (native().flat_section_ends); what the fused backward writes and gsr_adam_step reads
    #   "packed"  the caller's parameter order, no padding: good for the collective only
    # FlatAdam.step() refuses a bucket that is not "native".

    def __init__(self, params: Sequence[torch.Tensor]):
        self.params: List[torch.Tensor] = [p for p in params if p is not None]
        assert self.params, "no parameters"
        dev, dt = self.params[0].device, self.params[0].dtype
        assert all(p.device == dev and p.dtype == dt for p in self.params), "one device / dtype per bucket"
        self.numel = sum(p.numel() for p in self.params)
        self.flat = torch.zeros(self.numel, dtype=dt, device=dev)
        self.views: List[torch.Tensor] = []
        self.layout, self.zero_copy = "packed", False
        off = 0
        for p in self.params:
            self.views.append(self.flat[off:off + p.numel()].view(p.shape))
            off += p.numel()

    @classmethod
    def native_layout(cls, named: Dict[str, Optional[torch.Tensor]]) -> "GradientBucket":
        """Bucket in the rasterizer's own flat layout (see `layout` above) for the parameters given by field
        name.  `params` / `views` are in flat_adam.FIELDS order."""
        from .flat_adam import FIELDS, section_ends

        names = [f for f in FIELDS if named.get(f) is not None]
        assert "xyz" in names, "native layout needs at least xyz"
        params = [named[f] for f in names]
        n = named["xyz"].shape[0]
        n_rest = 0 if named.get("sh") is None else named["sh"].shape[2]
        ends = section_ends(n, n_rest)
        assert len(ends) == len(names), "parameter set does not match the native flat layout"
        b = cls.__new__(cls)
        b.params = list(params)
        dev, dt = params[0].device, params[0].dtype
        b.numel = int(ends[-1])
        b.flat = torch.zeros(b.numel, dtype=dt, device=dev)
        b.views, start = [], 0
        for p_, end in zip(params, ends):
            assert start + p_.numel() <= end
            b.views.append(b.flat[start:start + p_.numel()].view(p_.shape))
            start = int(end)
        b.layout, b.zero_copy = "native", False
        return b

    @classmethod
    def for_gaussians(cls, gaussians, native: bool = True) -> "GradientBucket":
        named = {f: getattr(gaussians, f, None) for f in PARAM_FIELDS}
        if native:
            return cls.native_layout(named)
        return cls([named[f] for f in PARAM_FIELDS])

    @classmethod
    def adopt(cls, flat: torch.Tensor, params, names: Optional[Sequence[str]] = None) -> "GradientBucket":
        """Zero-copy bucket over the buffer the fused backward already produced: `rasterize(...,
        return_state=True)` leaves all parameter gradients of the view as views of `state.grad_flat`, and
        autograd installs those views as `.grad` when the parameters had no gradient yet (`p.grad = None`
        before `backward()`).  Falls back to a flatten copy when a gradient lives elsewhere (accumulated
        over several views, or produced by the unfused operator chain).

        `params` is a Gaussians-like object, a {field name: tensor} dict, or a sequence of tensors with `names`
        giving their field names: then the fallback copy is built in the NATIVE layout, so the bucket can feed
        FlatAdam either way.  A bare sequence without names falls back to a "packed" bucket (collective only)."""
        named = None
        if isinstance(params, dict):
            named = params
        elif hasattr(params, "xyz"):
            named = {f: getattr(params, f, None) for f in PARAM_FIELDS}
        elif names is not None:
            named = dict(zip(names, params))
        plist = [p for p in (named.values() if named is not None else params) if p is not None]
        lo = flat.data_ptr()
        hi = lo + flat.numel() * flat.element_size()
        if all(p.grad is not None and lo <= p.grad.data_ptr() < hi for p in plist):
            b = cls.__new__(cls)
            b.params, b.flat, b.numel = list(plist), flat, flat.numel()
            b.views = [p.grad for p in plist]
            b.zero_copy, b.layout = True, "native"
            return b
        b = cls.native_layout(named) if named is not None else cls(plist)
        for p, v in zip(b.params, b.views):
            if p.grad is not None:
                v.copy_(p.grad)
        return b.attach()

    def attach(self) -> "GradientBucket":
        for p, v in zip(self.params, self.views):
            p.grad = v
        return self

    def zero(self) -> None:
        self.flat.zero_()

    def nbytes(self) -> int:
        return self.flat.numel() * self.flat.element_size()

    def all_reduce(self, group=None, average: bool = True, async_op: bool = False):
        """Sum (or average) the bucket over the ranks of `group`.  No-op without an initialised process group
        or with a single rank.  Returns the work handle when async_op=True (call .wait() before the optimizer)."""
        if not dist.is_available() or not dist.is_initialized():
            return None
        world = dist.get_world_size(group)
        if world == 1:
            return None
        for p, v in zip(self.params, self.views):  # autograd must not have replaced a view by a new tensor
            assert p.grad is not None and p.grad.data_ptr() == v.data_ptr(), "call attach() before backward()"
        op = dist.ReduceOp.SUM
        if average:
            if dist.get_backend(group) == "nccl":
                op = dist.ReduceOp.AVG       # averaged inside the collective, no extra pass over the bucket
            else:
                self.flat.div_(world)        # pre-divide: the sum of the pre-divided parts is the mean
        work = dist.all_reduce(self.flat, op=op, group=group, async_op=async_op)
        return work if async_op else None


def all_reduce_statistics(tensors: Iterable[torch.Tensor], group=None) -> None:
    """Sum the densification statistics (dense [N,...] accumulators) over ranks, in place."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    for t in tensors:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)


def all_reduce_visibility(visible: torch.Tensor, group=None) -> torch.Tensor:
    """OR of the ranks' visibility masks (bool or uint8 [N], `state.visible`), in place, as a MAX all-reduce: what
    FlatAdam.step(bucket, visible=...) needs after the gradient all-reduce, so that every replica updates the same rows
    (a row is updated when any rank's view saw it).  A bool mask is reduced through its uint8 view.  No-op without an
    initialised process group or with a single rank.  Returns `visible`."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return visible
    assert visible.dtype in (torch.bool, torch.uint8) and visible.is_contiguous(), "a contiguous bool / uint8 mask"
    buf = visible.view(torch.uint8) if visible.dtype == torch.bool else visible
    dist.all_reduce(buf, op=dist.ReduceOp.MAX, group=group)
    return visible


def broadcast_parameters(gaussians, src: int = 0, group=None) -> None:
    """Make every rank start from rank `src`'s Gaussians (after initialisation or densification on `src`)."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    for f in PARAM_FIELDS:
        t: Optional[torch.Tensor] = getattr(gaussians, f, None)
        if t is not None:
            dist.broadcast(t.data, src=src, group=group)
