"""CPU oracle of the intrinsics and lens-coefficient gradients: rasterize(..., camera.K or the lens coefficients
requiring grad).  TEST INFRASTRUCTURE.

The fp64 forward is pose_oracle's (the lens oracles'; the pinhole is distortion_oracle with zero coefficients).
calib_oracle.c adds, per visible gaussian, the gradients on fx fy cx cy and on the lens coefficients from render-stage
rows (the oracle's own render backward's, or the GPU's slab):

    o = pose_oracle.rasterize(lens, xyz, ..., T, K, H, W, k, antialiased=..., filter3d=...)
    c = contributions(o, lens, rows)        # [N, 4 + n]: fx fy cx cy, k_1..k_n
    g_K, g_k = c[:, :4].sum(0), c[:, 4:].sum(0)
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from pathlib import Path

import numpy as np

from tests import antialiased_oracle as aao
from tests import pose_oracle as po

HERE = Path(__file__).resolve().parent
ORACLE = HERE.parent / "oracle"
N_COEFFS = {"pinhole": 0, "fisheye": 4, "distortion": 5}
_libs = {}


def _build(which: int) -> Path:
    base = "fisheye_oracle.c" if which == 1 else "distortion_oracle.c"
    srcs = [HERE / "calib_oracle.c", HERE / "pose_oracle.c", HERE / base, ORACLE / "gsr_oracle.c",
            ORACLE / "gsr_oracle_body.inc"]
    digest = hashlib.sha256(b"".join(p.read_bytes() for p in srcs)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_calib_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_calib_oracle_{which}_{digest}.so"
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


def contributions(o, lens, rows, visible=None):
    """Per-gaussian [N, 4 + n] (fx fy cx cy, then the lens's n coefficients) from render-stage rows (a namespace with
    opacity [N], uv [N,2], conic [N,3]; pose_oracle.rows_from_slab).  visible: the gaussians to count (default: the
    oracle's own)."""
    xyz, quaternion, scale, opacity, rgb, sh, T, K = o.inputs
    N = xyz.shape[0]
    vis = o.keep if visible is None else np.asarray(visible, bool)
    g_conic = np.asarray(rows.conic, np.float64).reshape(N, 3).copy()
    g_opa = np.asarray(rows.opacity, np.float64).reshape(-1)
    if o.antialiased:
        conic = o.pg.conic[vis]
        rho, _ = aao.compensate(np.ascontiguousarray(conic), o.pg.opacity[vis] * o.coef_full[vis])
        g_conic[vis] += (g_opa[vis] * o.pg.opacity[vis] * o.coef_full[vis])[:, None] * aao.rho_grad(conic, rho)
    nk = 4 if lens == "fisheye" else 5
    out = np.zeros((N, 4 + nk))
    lib(lens).calib_vjp_f64(C.c_int(N), _p(_d(xyz)), _p(_d(quaternion)), _p(_d(o.sp)), _p(_d(T)), _p(_d(K)),
                            _p(_d(o.kc)), _p(np.ascontiguousarray(vis, np.uint8)),
                            _p(_d(np.reshape(rows.uv, (N, 2)))), _p(_d(g_conic)), _p(out))
    return out[:, :4 + N_COEFFS[lens]]


def camera_grad(o, lens, rows, visible=None):
    """(dL/d(fx, fy, cx, cy) [4], dL/dk [n], sum_i |contribution_i| [4 + n]) in fp64."""
    c = contributions(o, lens, rows, visible)
    g = c.sum(0)
    return g[:4], g[4:], np.abs(c).sum(0)


def K_grad(g4):
    """[3,3] from (fx, fy, cx, cy)."""
    out = np.zeros((3, 3))
    out[0, 0], out[1, 1], out[0, 2], out[1, 2] = g4
    return out


rasterize = po.rasterize
rows_from_slab = po.rows_from_slab
