"""fp64 oracle of rasterize_surfels(..., median_depth=True) (tests/surfels_median_oracle.c): every pixel's ray against
every visible surfel in depth order, no tiles, with the analytic backward of <G, median>.  TEST INFRASTRUCTURE.

    o = render(scene)                     # o.median [H,W], o.id [H,W] (-1: none), o.flag [H,W], o.visible, o.rays
    o = render(scene, grads=G)            # + o.rows [N,20], o.mass [N,20], o.g (xyz, quaternion, scale, opacity)

lens, kc: None (the pinhole: the lens oracle with zero OPENCV coefficients; rows are then mapped from d loss / d M' to
the pinhole kernels' d loss / d M, M = K M'), or as tests/surfels_lens_oracle.render.
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

from tests import surfels_lens_oracle as lo
from tests.surfels_oracle import _f64, _p

HERE = Path(__file__).resolve().parent
_lib = None


def build() -> Path:
    """Compile into a per-user cache directory outside the tree (keyed by the sources' digest)."""
    srcs = [HERE / "surfels_median_oracle.c", HERE / "surfels_lens_oracle.c"]
    digest = hashlib.sha256(b"".join(s.read_bytes() for s in srcs)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"gsr_surfels_median_oracle_{os.getuid()}"
    out_dir.mkdir(exist_ok=True)
    out = out_dir / f"libgsr_surfels_median_oracle_{digest}.so"
    if not out.exists():
        tmp = out.with_suffix(f".{os.getpid()}.tmp")
        subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", str(srcs[0]), "-o", str(tmp), "-lm"],
                       check=True, capture_output=True)
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.surfel_median_oracle.restype = C.c_int
    return _lib


def render(scene, grads=None, lens=None, kc=None, near=0.3, far=500.0, pad=100.0, mh=3.0, sort_z=None, limit=None):
    N, H, W = scene["xyz"].shape[0], int(scene["H"]), int(scene["W"])
    o = SimpleNamespace(median=np.zeros((H, W)), id=np.zeros((H, W), np.int32), flag=np.zeros((H, W), np.uint8),
                        visible=np.zeros(N, np.uint8), rays=np.zeros((H, W, 3)))
    G = None
    if grads is not None:
        G = _f64(np.reshape(grads, (H, W)))
        o.rows, o.mass = np.zeros((N, 20)), np.zeros((N, 20))
        o.g = dict(xyz=np.zeros((N, 3)), quaternion=np.zeros((N, 4)), scale=np.zeros((N, 3)), opacity=np.zeros(N))
    if lens is None:
        kcd = _f64(np.array([0.0, 0.0, 0.0, 0.0, 0.0, np.inf]))
        lens_id = lo.LENS_ID["distortion"]
    else:
        kcd = _f64(lo.lens_constants(lens, kc, limit))
        lens_id = lo.LENS_ID[lens]
    keep = [_f64(scene["xyz"]), _f64(scene["quaternion"]), _f64(scene["scale"]), _f64(np.reshape(scene["opacity"], -1)),
            _f64(scene["T"]), _f64(scene["K"])]
    zs = None if sort_z is None else _f64(sort_z)
    nul = (lambda a: None) if G is None else _p
    o.M = lib().surfel_median_oracle(
        C.c_int(lens_id), _p(kcd), C.c_int(N), *[_p(a) for a in keep], C.c_int(H), C.c_int(W), C.c_double(near),
        C.c_double(far), C.c_double(pad), C.c_double(mh), None if G is None else _p(G), _p(o.median), _p(o.id),
        _p(o.flag), _p(o.visible), *[nul(getattr(o, "rows", None)), nul(getattr(o, "mass", None))],
        *[nul(o.g[k]) if G is not None else None for k in ("xyz", "quaternion", "scale", "opacity")], _p(zs),
        _p(o.rays))
    if G is not None:
        o.g["opacity"] = o.g["opacity"].reshape(np.shape(scene["opacity"]))
        if lens is None:
            # the pinhole rows are d loss / d M with M = K M': column j of d loss / d M is K^-T (d loss / d M')[:, j]
            Kinv_t = np.linalg.inv(keep[5]).T
            for r in (o.rows, o.mass):
                gm = r[:, :9].reshape(N, 3, 3)
                r[:, :9] = np.einsum("ab,nbj->naj", np.abs(Kinv_t) if r is o.mass else Kinv_t, gm).reshape(N, 9)
    return o


def loss(o, grads):
    """<G, median> of a forward, for central differences."""
    return float((np.reshape(grads, o.median.shape) * o.median).sum())
