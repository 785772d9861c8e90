"""Camera pose refinement: rigid corrections of camera_T_world that autograd can step.

rasterize(...) and rasterize_batch(...) return d loss / d camera_T_world when the pose requires grad, but a raw 4x4
gradient step leaves the rotation block non-orthonormal.  The corrections here are twists xi = (rho, omega) in se(3),
applied on the left (a perturbation in the camera frame):

    T' = se3_exp(xi) @ T

so the pose stays rigid whatever the optimiser does, and xi = 0 is the identity.  Plain torch, differentiable,
any dtype and device.
"""
from __future__ import annotations

import torch


def _hat(w):
    """[..., 3] -> [..., 3, 3], the cross-product matrix [w]x."""
    z = torch.zeros_like(w[..., 0])
    return torch.stack([torch.stack([z, -w[..., 2], w[..., 1]], -1),
                        torch.stack([w[..., 2], z, -w[..., 0]], -1),
                        torch.stack([-w[..., 1], w[..., 0], z], -1)], -2)


def se3_exp(xi):
    """The exponential of twists xi = (rho, omega) [..., 6] as rigid transforms [..., 4, 4]: the matrix exponential of
    [[ [omega]x, rho ], [0, 0]], i.e. R = exp([omega]x) (Rodrigues) and t = V rho.  Below |omega| = 1e-2 the
    coefficients sin(th)/th, (1 - cos th)/th^2 and (th - sin th)/th^3 come from their Taylor series (truncation below
    th^6 / 5040 = 2e-16), which avoids the cancellation of the closed forms in fp32 and keeps the result and its
    gradient finite at xi = 0."""
    rho, w = xi[..., :3], xi[..., 3:]
    th2 = (w * w).sum(-1)
    small = th2 < 1e-4
    th2_safe = torch.where(small, torch.ones_like(th2), th2)
    th = torch.sqrt(th2_safe)
    a = torch.where(small, 1 - th2 / 6 + th2 * th2 / 120, torch.sin(th) / th)
    b = torch.where(small, 0.5 - th2 / 24 + th2 * th2 / 720, (1 - torch.cos(th)) / th2_safe)
    c = torch.where(small, 1.0 / 6 - th2 / 120 + th2 * th2 / 5040, (th - torch.sin(th)) / (th2_safe * th))
    Wx = _hat(w)
    Wx2 = Wx @ Wx
    eye = torch.eye(3, dtype=xi.dtype, device=xi.device).expand(Wx.shape)
    R = eye + a[..., None, None] * Wx + b[..., None, None] * Wx2
    V = eye + b[..., None, None] * Wx + c[..., None, None] * Wx2
    t = (V @ rho[..., None])[..., 0]
    top = torch.cat([R, t[..., None]], -1)
    bottom = torch.zeros(xi.shape[:-1] + (1, 4), dtype=xi.dtype, device=xi.device)
    bottom[..., 0, 3] = 1
    return torch.cat([top, bottom], -2)


class PoseDelta(torch.nn.Module):
    """Zero-initialised corrections of n_cameras poses, one twist [6] per camera (self.xi [n, 6]).

    forward(T, idx) returns se3_exp(xi[idx]) @ T: T [4,4] with an int idx, or T [C,4,4] with idx [C] (a tensor or a
    sequence), for rasterize_batch.  Optimise self.xi with its own optimiser (usually a smaller learning rate than the
    gaussians', and often without weight decay)."""

    def __init__(self, n_cameras: int, dtype=torch.float32, device=None):
        super().__init__()
        self.xi = torch.nn.Parameter(torch.zeros(n_cameras, 6, dtype=dtype, device=device))

    def forward(self, T, idx):
        if not torch.is_tensor(idx):
            idx = torch.as_tensor(idx, dtype=torch.long, device=self.xi.device)
        return se3_exp(self.xi[idx]).to(T.dtype) @ T
