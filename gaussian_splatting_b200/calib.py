"""Camera self-calibration: corrections of the intrinsics K that autograd can step.

rasterize(...) and rasterize_batch(...) return d loss / d K when camera.K requires grad (fx, fy, cx, cy; every other
entry 0).  The corrections here are per camera (log fx scale, log fy scale, delta cx, delta cy):

    fx' = fx exp(sx),  fy' = fy exp(sy),  cx' = cx + dcx,  cy' = cy + dcy

so the focal lengths stay positive whatever the optimiser does, a step in the scales is relative (the same learning
rate suits a 500 px and a 3000 px focal length), and zero corrections give K back bit for bit.  Lens coefficients need
no module: optimise a CPU nn.Parameter [n_cameras, n] and pass a row as fisheye= / distortion= (DESIGN.md 3.23).
Plain torch, differentiable, any dtype and device.
"""
from __future__ import annotations

import torch


class IntrinsicsDelta(torch.nn.Module):
    """Zero-initialised corrections of the intrinsics of n_cameras cameras: self.log_focal [n, 2] (log fx scale,
    log fy scale; with shared_focal=True [n, 1], one scale for fx and fy, for COLMAP's SIMPLE_* models whose fx == fy)
    and self.principal [n, 2] (delta cx, delta cy in pixels).  Two parameters, so that an optimiser can give the
    relative focal scales and the principal point in pixels learning rates of their own.

    forward(K, idx) returns the corrected K: K [3,3] with an int idx, or K [C,3,3] (or a shared [3,3]) with idx [C] (a
    tensor or a sequence), for rasterize_batch.  At zero corrections the result equals K bit for bit.  Pass K.detach()
    wherever K is read as a constant (e.g. DensificationStats.accumulate)."""

    def __init__(self, n_cameras: int, shared_focal: bool = False, dtype=torch.float32, device=None):
        super().__init__()
        self.shared_focal = bool(shared_focal)
        self.log_focal = torch.nn.Parameter(torch.zeros(n_cameras, 1 if self.shared_focal else 2, dtype=dtype,
                                                        device=device))
        self.principal = torch.nn.Parameter(torch.zeros(n_cameras, 2, dtype=dtype, device=device))

    def forward(self, K, idx):
        if not torch.is_tensor(idx) and not isinstance(idx, int):
            idx = torch.as_tensor(idx, dtype=torch.long, device=self.log_focal.device)
        lf, pp = self.log_focal[idx].to(K.dtype), self.principal[idx].to(K.dtype)
        sx, sy = lf[..., 0], lf[..., -1]
        dcx, dcy = pp[..., 0], pp[..., 1]
        one, zero = torch.ones_like(sx), torch.zeros_like(sx)
        # K * S + A: exp(0) = 1 and + 0 leave every entry's bits as they are
        S = torch.stack([torch.exp(sx), one, one, one, torch.exp(sy), one, one, one, one], -1)
        A = torch.stack([zero, zero, dcx, zero, zero, dcy, zero, zero, zero], -1)
        shape = sx.shape + (3, 3)
        return K * S.view(shape) + A.view(shape)
