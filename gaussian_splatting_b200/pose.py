"""Camera pose refinement: rigid corrections of camera_T_world that autograd can step.

rasterize(...) and rasterize_batch(...) return d loss / d camera_T_world when the pose requires grad, but a raw 4x4
gradient step leaves the rotation block non-orthonormal.  The corrections here are twists xi = (rho, omega) in se(3),
applied on the left (a perturbation in the camera frame):

    T' = se3_exp(xi) @ T

so the pose stays rigid whatever the optimiser does, and xi = 0 is the identity.  se3_log inverts se3_exp, and
shutter_from_endpoints turns a rolling shutter's first-line and last-line poses into rasterize's (camera_T_world,
rolling_shutter).  Plain torch, differentiable, any dtype and device.
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


def se3_log(T):
    """The inverse of se3_exp: rigid transforms T [..., 4, 4] -> twists xi = (rho, omega) [..., 6] with |omega| < pi.
    The angle is atan2(|vee(R - R^T)| / 2, (tr R - 1) / 2), which keeps its precision near 0; below th^2 = 1e-4 the
    coefficients th / (2 sin th) and (1 - th sin th / (2 (1 - cos th))) / th^2 of omega = coef vee(R - R^T) and
    rho = V^-1 t come from their Taylor series, so the result and its gradient are finite at the identity.  Near
    |omega| = pi the rotation's axis is ill-conditioned (as for any logarithm)."""
    R, t = T[..., :3, :3], T[..., :3, 3]
    v = torch.stack([R[..., 2, 1] - R[..., 1, 2], R[..., 0, 2] - R[..., 2, 0], R[..., 1, 0] - R[..., 0, 1]], -1)
    s = 0.5 * torch.linalg.vector_norm(v, dim=-1)
    c = 0.5 * (R[..., 0, 0] + R[..., 1, 1] + R[..., 2, 2] - 1)
    th = torch.atan2(s, c)
    th2 = th * th
    small = th2 < 1e-4
    th_safe = torch.where(small, torch.ones_like(th), th)
    s_safe = torch.where(small, torch.ones_like(s), s)
    half = torch.where(small, 0.5 + th2 / 12 + 7 * th2 * th2 / 720, th_safe / (2 * s_safe))
    w = half[..., None] * v
    d = torch.where(small, 1.0 / 12 + th2 / 720 + th2 * th2 / 30240,
                    (1 - th_safe * s_safe / (2 * (1 - torch.cos(th_safe)))) / (th_safe * th_safe))
    Wx = _hat(w)
    eye = torch.eye(3, dtype=T.dtype, device=T.device).expand(Wx.shape)
    Vinv = eye - 0.5 * Wx + d[..., None, None] * (Wx @ Wx)
    rho = (Vinv @ t[..., None])[..., 0]
    return torch.cat([rho, w], -1)


def shutter_from_endpoints(T_start, T_end):
    """(camera_T_world of the middle line, xi) for rasterize(..., rolling_shutter=xi) from the poses of a rolling
    shutter's first and last lines ([..., 4, 4] each): xi = se3_log(T_end @ inverse(T_start)), the motion over the
    readout applied on the left, and T_mid = se3_exp(xi / 2) @ T_start, so that se3_exp((tau - 1/2) xi) @ T_mid is
    T_start at tau = 0 and T_end at tau = 1."""
    xi = se3_log(T_end @ torch.linalg.inv(T_start))
    return se3_exp(0.5 * xi) @ T_start, xi


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
