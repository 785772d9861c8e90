"""Mip-Splatting's 3-D smoothing filter (Yu et al., CVPR 2024; DESIGN.md 3.13).

A gaussian cannot be resolved finer than the finest rate at which any training camera samples it.  The filter gives
every gaussian a world-space floor f on its standard deviation: rasterize(..., filter3d=f) renders it with the
covariance R diag(exp(2 s) + f^2) R^T and the opacity sigmoid(o) * coef, coef = sqrt(prod_k exp(2 s_k) / (exp(2 s_k)
+ f^2)), which keeps its 3-D mass.  The filter is a constant of the scene: it gets no gradient, and it is recomputed
from the training cameras whenever the gaussians change (after densification) and, once densification has ended,
every few hundred steps.

    f = compute_filter3d(gaussians.xyz, train_T, train_K, widths, heights)      # one native kernel
    image, mask, uv = rasterize(gaussians, T, camera, ..., filter3d=f)
    baked = bake_filter3d(gaussians, f)                                          # export: plain 3DGS parameters
"""
from __future__ import annotations

import torch

from . import native
from .structs import Gaussians


def _stack(x, shape, dtype, device):
    if torch.is_tensor(x):
        t = x
    elif len(x) and torch.is_tensor(x[0]):
        t = torch.stack([torch.as_tensor(a).reshape(shape) for a in x])
    else:
        t = torch.as_tensor(x)
    return t.to(device=device, dtype=dtype).reshape((-1,) + shape).contiguous()


def compute_filter3d(xyz, camera_T_worlds, Ks, widths, heights, near=0.2, margin=0.15, variance=0.2):
    """Filter size [N] (fp32, world units) of every gaussian from C cameras: camera_T_worlds [C,4,4], Ks [C,3,3] (tensors
    or sequences of per-camera tensors), widths / heights (C ints or a tensor), one native launch (gsr_filter3d).

    Camera c sees gaussian i when its camera-frame depth p_z > near and its projection lies within the image widened by
    `margin` of its size on every side; it then samples it at r_c = p_z / max(fx_c, fy_c) world units per pixel.  With
    r_i the smallest r_c over the cameras that see i, f_i = sqrt(variance) * r_i (variance in px^2).  Gaussians that no
    camera sees get the largest f of the others (0 when none is seen).  The defaults are Mip-Splatting's.

    Mip-Splatting's own code takes the minimum depth and the maximum focal length over the cameras separately; the
    ratio per camera used here is the paper's definition, and the two agree when every camera has the same focal
    length.  Pass the TRAINING cameras only."""
    if xyz.dtype != torch.float32 or not xyz.is_cuda:
        raise TypeError("compute_filter3d needs fp32 CUDA positions")
    dev = xyz.device
    T = _stack(camera_T_worlds, (4, 4), torch.float32, dev)
    K = _stack(Ks, (3, 3), torch.float32, dev)
    W = _stack(widths, (), torch.int32, dev).reshape(-1)
    H = _stack(heights, (), torch.int32, dev).reshape(-1)
    if not (T.shape[0] == K.shape[0] == W.shape[0] == H.shape[0] >= 1):
        raise ValueError(f"need the same number (>= 1) of poses, intrinsics, widths and heights; got {T.shape[0]}, "
                         f"{K.shape[0]}, {W.shape[0]}, {H.shape[0]}")
    if not (near >= 0 and margin >= 0 and variance >= 0):
        raise ValueError("near, margin and variance must be >= 0")
    with torch.no_grad():
        return native().filter3d(xyz.detach().contiguous(), T, K, W, H, float(near), float(margin), float(variance))


def filter3d_factors(scale, filter3d):
    """(filtered log-scale, coef) of log-scales [N,3] and the filter [N] or [N,1], in torch (differentiable in scale):
    scale' = 1/2 log(exp(2 s) + f^2) per axis and coef = sqrt(prod_k t_k), t_k = exp(2 s_k) / (exp(2 s_k) + f^2)."""
    F = filter3d.reshape(-1, 1).to(scale.dtype) ** 2
    v = torch.exp(2.0 * scale)
    vp = v + F
    t = torch.where(F == 0, torch.ones_like(v), v / vp)
    return 0.5 * torch.log(vp), torch.sqrt(t.prod(dim=1, keepdim=True))


def bake_filter3d(gaussians, filter3d):
    """Gaussians with the filter folded into the parameters (Mip-Splatting's export): scale' = 1/2 log(exp(2 s) + f^2)
    and opacity logit' = logit(sigmoid(o) * coef).  They render like `gaussians` with filter3d — in any standard 3DGS
    viewer, or through rasterize() without the filter.  xyz, rgb, quaternion and sh are the same tensors; the new
    fields are differentiable functions of the old ones."""
    scale, coef = filter3d_factors(gaussians.scale, filter3d)
    opacity = torch.logit(torch.sigmoid(gaussians.opacity) * coef)
    return Gaussians(gaussians.xyz, gaussians.rgb, opacity, scale, gaussians.quaternion, gaussians.sh)
