"""fp64 reference for the bilateral-grid slice and total variation (gaussian_splatting_b200/appearance.py).

`slice_forward` / `slice_backward` are an explicit numpy trilinear slice and its gradients, written from the formulas
of include/gsr_bilagrid.h: for pixel (i, j) of a view with grid n,

    fx = (j + 0.5) / W (GX - 1),  fy = (i + 0.5) / H (GY - 1),  fz = clamp(lum, 0, 1) (L - 1),
    lum = 0.299 r + 0.587 g + 0.114 b,
    a = sum over the 8 nodes (floor(f), floor(f) + 1 clamped to the grid) of the trilinear weight times G[n, :, z, y, x],
    out = A[:, :3] rgb + A[:, 3],  A = a.reshape(3, 4).

`grid_sample_slice` is the same operation as a torch expression (F.grid_sample with border padding and
align_corners=True, then the affine), `total_variation` the regulariser as a torch expression; both run in whatever
dtype they are given and serve as the formulation a user would otherwise write.
"""
from __future__ import annotations

import numpy as np

LUMA = np.array([0.299, 0.587, 0.114])


def _axis(n, G):
    f = (np.arange(n) + 0.5) / n * (G - 1)
    i0 = np.floor(f).astype(np.int64)
    return i0, np.minimum(i0 + 1, G - 1), f - i0


def _terms(grids, rgb, ids):
    """the 8 nodes' indices and weights, a [C,H,W,12] and da/dfz [C,H,W,12]"""
    grids = np.asarray(grids, np.float64)
    rgb = np.asarray(rgb, np.float64)
    C, H, W, _ = rgb.shape
    _, _, L, GY, GX = grids.shape
    x0, x1, tx = _axis(W, GX)
    y0, y1, ty = _axis(H, GY)
    lum = rgb @ LUMA
    fz = np.clip(lum, 0.0, 1.0) * (L - 1)
    z0 = np.floor(fz).astype(np.int64)
    z1 = np.minimum(z0 + 1, L - 1)
    tz = fz - z0
    yy = lambda v: np.broadcast_to(v[None, :, None], (C, H, W))  # noqa: E731
    xx = lambda v: np.broadcast_to(v[None, None, :], (C, H, W))  # noqa: E731
    nodes = []
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                wz = tz if dz else 1.0 - tz
                wy = yy(ty if dy else 1.0 - ty)
                wx = xx(tx if dx else 1.0 - tx)
                nodes.append(((z1 if dz else z0), yy(y1 if dy else y0), xx(x1 if dx else x0), wz * wy * wx,
                              (1.0 if dz else -1.0) * wy * wx))
    a = np.zeros((C, H, W, 12))
    da = np.zeros((C, H, W, 12))
    for c in range(C):
        g = grids[ids[c]]
        for z, y, x, w, dw in nodes:
            v = np.moveaxis(g[:, z[c], y[c], x[c]], 0, -1)
            a[c] += w[c][..., None] * v
            da[c] += dw[c][..., None] * v
    return nodes, a, da, lum, L


def slice_forward(grids, rgb, ids):
    """out [C,H,W,3] in fp64 for rgb [C,H,W,3], grids [N,12,L,GY,GX] and one grid id per view."""
    rgb = np.asarray(rgb, np.float64)
    _, a, _, _, _ = _terms(grids, rgb, ids)
    A = a.reshape(*a.shape[:3], 3, 4)
    return np.einsum("chwkj,chwj->chwk", A[..., :3], rgb) + A[..., 3]


def slice_backward(grids, rgb, ids, grad_out):
    """(d rgb [C,H,W,3], d grids [N,12,L,GY,GX]) in fp64 for the upstream gradient grad_out [C,H,W,3]."""
    grids = np.asarray(grids, np.float64)
    rgb = np.asarray(rgb, np.float64)
    g = np.asarray(grad_out, np.float64)
    nodes, a, da, lum, L = _terms(grids, rgb, ids)
    C = rgb.shape[0]
    A = a.reshape(*a.shape[:3], 3, 4)
    v1 = np.concatenate([rgb, np.ones(rgb.shape[:3] + (1,))], -1)
    gA = (g[..., :, None] * v1[..., None, :]).reshape(*g.shape[:3], 12)  # d loss / d a
    d_rgb = np.einsum("chwkj,chwk->chwj", A[..., :3], g)
    inside = (lum > 0.0) & (lum < 1.0)
    d_lum = np.where(inside, (L - 1) * (gA * da).sum(-1), 0.0)
    d_rgb += d_lum[..., None] * LUMA
    d_grids = np.zeros_like(grids)
    _, _, L, GY, GX = grids.shape
    for c in range(C):
        dg = np.zeros((12, L * GY * GX))
        for z, y, x, w, _ in nodes:
            node = ((z[c] * GY + y[c]) * GX + x[c]).reshape(-1)
            contrib = (w[c][..., None] * gA[c]).reshape(-1, 12)
            for k in range(12):
                dg[k] += np.bincount(node, contrib[:, k], minlength=L * GY * GX)
        d_grids[ids[c]] += dg.reshape(grids.shape[1:])
    return d_rgb, d_grids


def grid_sample_slice(grids, rgb, ids):
    """The slice as torch's F.grid_sample expression, in the dtype of its inputs, differentiable (rgb [C,H,W,3])."""
    import torch
    import torch.nn.functional as F

    C, H, W, _ = rgb.shape
    yy, xx = torch.meshgrid((torch.arange(H, dtype=rgb.dtype, device=rgb.device) + 0.5) / H,
                            (torch.arange(W, dtype=rgb.dtype, device=rgb.device) + 0.5) / W, indexing="ij")
    xy = torch.stack([xx, yy], -1)[None].expand(C, H, W, 2) * 2 - 1
    luma = torch.tensor(LUMA.tolist(), dtype=rgb.dtype, device=rgb.device)
    z = (rgb @ luma)[..., None] * 2 - 1
    coords = torch.cat([xy, z], -1)[:, None]  # [C,1,H,W,3] as (x, y, z)
    idx = torch.as_tensor(ids, device=grids.device)
    a = F.grid_sample(grids[idx], coords, mode="bilinear", padding_mode="border", align_corners=True)
    a = a[:, :, 0].permute(0, 2, 3, 1).reshape(C, H, W, 3, 4)
    return (a[..., :3] @ rgb[..., None])[..., 0] + a[..., 3]


def total_variation(grids):
    """sum over the L, GY, GX axes of mean((G[k + 1] - G[k])^2), as a torch expression"""
    return sum((grids.diff(dim=d) ** 2).mean() for d in (2, 3, 4))
