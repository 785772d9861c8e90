"""CPU oracle of the camera pose gradient: rasterize(..., camera_T_world requiring grad).  TEST INFRASTRUCTURE.

The fp64 forward is the lens oracle's (fisheye_oracle / distortion_oracle; the pinhole is distortion_oracle with zero
coefficients, exactly the pinhole model).  pose_oracle.c reuses their Jacobian and its VJP and adds the pose chain:

    o = LENS.rasterize(xyz, ..., T, K, H, W, k, antialiased=..., filter3d=...)
    c = contributions(o, lens, rows)       # [N, 12], T[:3, :] row-major per gaussian
    grad = c.sum(0).reshape(3, 4)          # dL/dT[:3, :]; dL/dT[3, :] = 0

`rows` are render-stage rows over all N gaussians (g_rgb, g_opa on the opacity the renderer was fed, g_uv, g_conic,
g_z), from the oracle's own render backward or from the GPU's slab.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from pathlib import Path
from types import SimpleNamespace

import numpy as np

from tests import antialiased_oracle as aao
from tests import distortion_oracle as dto
from tests import fisheye_oracle as feo

HERE = Path(__file__).resolve().parent
ORACLE = HERE.parent / "oracle"
LENSES = ("pinhole", "fisheye", "distortion")
ZERO_K = (0.0, 0.0, 0.0, 0.0, 0.0)
_libs = {}


def _build(which: int) -> Path:
    base = "fisheye_oracle.c" if which == 1 else "distortion_oracle.c"
    srcs = [HERE / "pose_oracle.c", HERE / base, ORACLE / "gsr_oracle.c", ORACLE / "gsr_oracle_body.inc"]
    digest = hashlib.sha256(b"".join(p.read_bytes() for p in srcs)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_pose_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_pose_oracle_{which}_{digest}.so"
    if not out.exists():
        tmp = out.with_suffix(f".{os.getpid()}.tmp")
        subprocess.run(["gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-mfma", "-shared", "-fPIC", f"-I{ORACLE}",
                        f"-I{HERE}", f"-DPOSE_LENS={which}", str(srcs[0]), "-o", str(tmp), "-lm"], check=True,
                       capture_output=True)
        os.replace(tmp, out)
    return out


def lib(lens):
    which = 1 if lens == "fisheye" else 2
    if which not in _libs:
        _libs[which] = C.CDLL(str(_build(which)))
    return _libs[which]


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _d(a):
    return None if a is None else np.ascontiguousarray(a, np.float64)


def rasterize(lens, xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, k=None, **kw):
    """The lens oracle's fp64 forward; k: the lens coefficients (ignored for the pinhole)."""
    if lens == "fisheye":
        return feo.rasterize(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, k, **kw)
    return dto.rasterize(xyz, quaternion, scale, opacity, rgb, sh, T, K, H, W, ZERO_K if lens == "pinhole" else k,
                         **kw)


def contributions(o, lens, rows, visible=None):
    """Per-gaussian pose gradient [N, 12] from render-stage rows (a namespace with rgb [N,3], opacity [N], uv [N,2],
    conic [N,3], z [N] or None).  visible: the gaussians to count (default: the oracle's own)."""
    xyz, quaternion, scale, opacity, rgb, sh, T, K = o.inputs
    N = xyz.shape[0]
    vis = o.keep if visible is None else np.asarray(visible, bool)
    g_conic = np.asarray(rows.conic, np.float64).reshape(N, 3).copy()
    g_opa = np.asarray(rows.opacity, np.float64).reshape(-1)
    if o.antialiased:
        conic = o.pg.conic[vis]
        rho, _ = aao.compensate(np.ascontiguousarray(conic), o.pg.opacity[vis] * o.coef_full[vis])
        g_conic[vis] += (g_opa[vis] * o.pg.opacity[vis] * o.coef_full[vis])[:, None] * aao.rho_grad(conic, rho)
    g_z = np.zeros(N) if rows.z is None else np.asarray(rows.z, np.float64).reshape(-1)
    out = np.zeros((N, 12))
    lib(lens).pose_vjp_f64(C.c_int(N), _p(_d(xyz)), _p(_d(quaternion)), _p(_d(o.sp)), _p(_d(T)), _p(_d(K)),
                           _p(_d(o.kc)), _p(np.ascontiguousarray(vis, np.uint8)),
                           _p(_d(np.reshape(rows.uv, (N, 2)))), _p(_d(g_conic)), _p(_d(g_z)), _p(out))
    return out


def pose_grad(o, lens, rows, visible=None):
    """(dL/dT [4,4], sum_i |contribution_i| [4,4]) in fp64."""
    c = contributions(o, lens, rows, visible)
    g, a = np.zeros((4, 4)), np.zeros((4, 4))
    g[:3] = c.sum(0).reshape(3, 4)
    a[:3] = np.abs(c).sum(0).reshape(3, 4)
    return g, a


def rows_from_slab(slab, depth):
    """The render-stage rows of the fused path's interleaved slab [N*12] (numpy): rgb3 opa | uv2 conic0 conic1 |
    conic2 z (depth mode) pad."""
    r = np.asarray(slab, np.float64).reshape(-1, 12)
    return SimpleNamespace(rgb=r[:, 0:3], opacity=r[:, 3], uv=r[:, 4:6], conic=r[:, 6:9],
                           z=r[:, 9] if depth else None)
