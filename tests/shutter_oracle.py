"""fp64 oracle of the rolling-shutter per-gaussian stage: rasterize(..., rolling_shutter=xi).  TEST INFRASTRUCTURE.

Plain torch in float64 with autograd, written from the model (DESIGN.md 3.24), not from the kernels:

    T(tau) = se3_exp((tau - 1/2) xi) @ T,  p(tau) = T(tau) x,  u(tau) = pi(p(tau)),  r(u) = r0 + e^T u
    tau* = clamp(r(u(tau*)), 0, 1)                        (solved to convergence, no fixed step count)
    f = J p',  p' = omega x p + rho,  lambda = e^T f,  A = I + f e^T / (1 - lambda)   (A = I where tau* is clamped)
    Sigma_2D = A J W(tau*) Sigma W(tau*)^T J^T A^T

tau* enters autograd through one implicit-function step, tau = tau_0 - phi(tau_0) / (1 - lambda_0) with tau_0 and
lambda_0 detached: its value is tau_0 and its derivative the implicit one, e^T du/dtheta / (1 - lambda).  J is formed
by autograd with create_graph, so its derivatives (the second-order terms of the backward) are autograd's too.

    out = forward(lens, params, T, K, k, xi, readout, H, W, antialiased=..., filter3d=...)
    g = vjp(out, rows)       # rows [N,12] in the layout of the render backward's gradient rows
"""
from __future__ import annotations

import torch

from gaussian_splatting_b200.pose import se3_exp

LAMBDA_MAX = 0.75
READOUTS = ("top_to_bottom", "bottom_to_top", "left_to_right", "right_to_left")


def readout_line(readout, H, W):
    """(r0, e [2]) of r(u) = r0 + e^T u"""
    vertical = readout in READOUTS[:2]
    n = H if vertical else W
    d = 1.0 / (n - 1)
    rev = readout in ("bottom_to_top", "right_to_left")
    e = [0.0, -d if rev else d] if vertical else [-d if rev else d, 0.0]
    return (1.0 if rev else 0.0), torch.tensor(e, dtype=torch.float64)


def project(lens, p, K, k):
    """[..., 3] camera-frame points -> [..., 2] pixel coordinates through the lens"""
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    if lens == "pinhole":
        a, b = x / z, y / z
    elif lens == "fisheye":
        rho = torch.sqrt(x * x + y * y)
        th = torch.atan2(rho, z)
        t = th * th
        thd = th * (1 + t * (k[0] + t * (k[1] + t * (k[2] + t * k[3]))))
        s = thd / rho
        a, b = s * x, s * y
    else:
        a0, b0 = x / z, y / z
        r2 = a0 * a0 + b0 * b0
        radial = 1 + r2 * (k[0] + r2 * (k[1] + r2 * k[4]))
        a = a0 * radial + 2 * k[2] * a0 * b0 + k[3] * (r2 + 2 * a0 * a0)
        b = b0 * radial + k[2] * (r2 + 2 * b0 * b0) + 2 * k[3] * a0 * b0
    return torch.stack([fx * a + cx, fy * b + cy], -1)


def jacobian(lens, p, K, k):
    """[N, 2, 3] d pi / dp with create_graph (each row of u depends on its own point only)"""
    if not p.requires_grad:
        p = p.detach().requires_grad_(True)
    u = project(lens, p, K, k)
    rows = [torch.autograd.grad(u[:, i].sum(), p, create_graph=True)[0] for i in range(2)]
    return torch.stack(rows, 1)


def _pose_at(T, xi, s):
    """T(tau) [N,4,4] for s = tau - 1/2 [N]; T [4,4] or [N,4,4] and xi [6] or [N,6] (per-gaussian copies give
    per-gaussian contributions to the camera gradients)"""
    return se3_exp(s[:, None] * xi) @ T


def _points(T, xi, s, xyz):
    Ts = _pose_at(T, xi, s)
    return (Ts[:, :3, :3] @ xyz[:, :, None])[..., 0] + Ts[:, :3, 3], Ts[:, :3, :3]


def solve_tau(lens, xyz, T, K, k, xi, r0, e, iters=60):
    """tau* per gaussian to convergence (projected Newton with the exact lambda), float64, no autograd; also the
    residual |tau - clamp(r(u(tau)))| and lambda at tau*"""
    with torch.no_grad():
        n = xyz.shape[0]
        tau = torch.full((n,), 0.5, dtype=torch.float64)
        for _ in range(iters):
            tau, lam, r = _newton(lens, xyz, T, K, k, xi, r0, e, tau)
        return tau, (tau - r.clamp(0, 1)).abs(), lam, r


def _newton(lens, xyz, T, K, k, xi, r0, e, tau):
    with torch.enable_grad():
        p, _ = _points(T, xi, tau - 0.5, xyz)
        J = jacobian(lens, p, K, k).detach()
    p = p.detach()
    u = project(lens, p, K, k)
    pd = torch.cross(xi[..., 3:].expand_as(p), p, dim=-1) + xi[..., :3]
    f = (J @ pd[:, :, None])[..., 0]
    lam = f @ e
    r = r0 + u @ e
    nt = (tau - (tau - r) / (1 - lam)).clamp(0, 1)
    return torch.where(lam < LAMBDA_MAX, nt, tau), lam, r


def forward(lens, xyz, quat, scale, opa_logit, T, K, k, xi, readout, H, W, antialiased=False, filter3d=None):
    """Per-gaussian outputs of the rolling-shutter stage (all gaussians, no culling): dict of uv [N,2], conic [N,3]
    (Sigma_2D00, Sigma_2D01 + Sigma_2D10, Sigma_2D11, before the renderer's dilation), opacity [N] (with the filter's
    coef and the antialiased rho), z [N], tau, residual, lambda and clamped [N]."""
    r0, e = readout_line(readout, H, W)
    k = None if k is None else torch.as_tensor(k, dtype=torch.float64)
    tau0, res, lam0, r_fin = solve_tau(lens, xyz.detach(), T.detach(), K, k, xi.detach(), r0, e)
    clamped = (r_fin < 0) | (r_fin > 1)
    # one implicit-function step: the value tau0, the derivative e^T du/dtheta / (1 - lambda)
    p_a, _ = _points(T, xi, tau0 - 0.5, xyz)
    u_a = project(lens, p_a, K, k)
    phi = tau0 - (r0 + u_a @ e)
    tau = torch.where(clamped, tau0, tau0 - phi / (1 - lam0))
    p, Wt = _points(T, xi, tau - 0.5, xyz)
    u = project(lens, p, K, k)
    J = jacobian(lens, p, K, k)
    pd = torch.cross(xi[..., 3:].expand_as(p), p, dim=-1) + xi[..., :3]
    f = (J @ pd[:, :, None])[..., 0]
    lam = f @ e
    A = torch.eye(2, dtype=torch.float64) + f[:, :, None] * e[None, None, :] / (1 - lam)[:, None, None]
    A = torch.where(clamped[:, None, None], torch.eye(2, dtype=torch.float64).expand_as(A), A)
    # world covariance (quaternion w, x, y, z; scale = log standard deviation), optionally 3-D filtered
    q = quat / quat.norm(dim=-1, keepdim=True)
    w, x, y, z = q.unbind(-1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1).view(-1, 3, 3)
    v = torch.exp(2 * scale)
    coef = torch.ones_like(opa_logit)
    if filter3d is not None:
        F = filter3d * filter3d
        coef = torch.sqrt(torch.prod(v / (v + F[:, None]), -1))
        v = v + F[:, None]
    Sigma = R @ torch.diag_embed(v) @ R.transpose(1, 2)
    M = A @ J @ Wt
    S2 = M @ Sigma @ M.transpose(1, 2)
    conic = torch.stack([S2[:, 0, 0], S2[:, 0, 1] + S2[:, 1, 0], S2[:, 1, 1]], -1)
    opa = torch.sigmoid(opa_logit) * coef
    if antialiased:
        c0, c1, c2 = conic.unbind(-1)
        bh = 0.5 * c1
        rho = torch.sqrt(torch.clamp(c0 * c2 - bh * bh, min=0) / ((c0 + 0.25) * (c2 + 0.25) - bh * bh))
        opa = opa * rho
    return dict(uv=u, conic=conic, opacity=opa, z=p[:, 2], tau=tau0, residual=res, lam=lam, clamped=clamped,
                cov=S2)


def loss_from_rows(out, rows, depth):
    """<rows, outputs> for rows [N,12] (rgb3 opa | uv2 conic0 conic1 | conic2 z pad): the rgb slot is not used (no SH)"""
    val = (rows[:, 3] * out["opacity"]).sum() + (rows[:, 4:6] * out["uv"]).sum()
    val = val + (rows[:, 6] * out["conic"][:, 0]).sum() + (rows[:, 7] * out["conic"][:, 1]).sum()
    val = val + (rows[:, 8] * out["conic"][:, 2]).sum()
    if depth:
        val = val + (rows[:, 9] * out["z"]).sum()
    return val
