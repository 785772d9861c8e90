"""fp64 reference of rasterize_surfels(..., features=F) built from the surfel oracles (tests/surfels_oracle.c,
tests/surfels_lens_oracle.c) with no new C.  TEST INFRASTRUCTURE.

The oracles blend a colour [N,3] that is an input.  A 3-channel chunk of F passed as that colour, with a zero background
and a gradient on the image only, gives the chunk's feature map as the image, d loss / d F of the chunk as the colour
gradient, and the chunk's part of d alpha in the rows and in the geometry gradients.  The branch decisions depend only
on the geometry, so the parts summed over the chunks are the feature loss's gradient.

    o = render(scene, F)                         # o.fmap [H,W,D], o.alpha, o.near, o.visible, o.uv
    o = render(scene, F, grads=G)                # + o.g (xyz, quaternion, scale, opacity, F), o.rows (colour slots 0),
                                                 #   o.uv_grad, o.mass, o.mass_F
    lens, kc: None (the pinhole), or as tests/surfels_lens_oracle.render
"""
from __future__ import annotations

import ctypes as C
from types import SimpleNamespace

import numpy as np

from tests import surfels_lens_oracle as lo
from tests import surfels_oracle as so
from tests.surfels_oracle import _f64, _p


def _chunk(scene, colour, G_img, lens, kc, near, far, pad, mh, sort_z, limit):
    N, H, W = scene["xyz"].shape[0], int(scene["H"]), int(scene["W"])
    o = SimpleNamespace(image=np.zeros((H, W, 3)), depth=np.zeros((H, W, 1)), alpha=np.zeros((H, W, 1)),
                        normal=np.zeros((H, W, 3)), dist=np.zeros((H, W, 1)), visible=np.zeros(N, np.uint8),
                        uv=np.zeros((N, 2)), near=np.zeros((H, W), np.uint8), rays=np.zeros((H, W, 3)))
    grads = None
    if G_img is not None:
        grads = [_f64(G_img)] + [np.zeros((H, W, c)) for c in (1, 1, 3, 1)]
        o.g = dict(xyz=np.zeros((N, 3)), quaternion=np.zeros((N, 4)), scale=np.zeros((N, 3)), opacity=np.zeros(N),
                   colour=np.zeros((N, 3)))
        o.rows, o.uv_grad, o.mass = np.zeros((N, 20)), np.zeros((N, 2)), np.zeros((N, 20))
    keep = [_f64(scene["xyz"]), _f64(scene["quaternion"]), _f64(scene["scale"]), _f64(np.reshape(scene["opacity"], -1)),
            _f64(colour), _f64(scene["T"]), _f64(scene["K"])]
    gp = [None] * 5 if grads is None else [_p(g) for g in grads]
    og = [None] * 5 if grads is None else [_p(o.g[k]) for k in ("xyz", "quaternion", "scale", "opacity", "colour")]
    rest = [None, None, None] if grads is None else [_p(o.rows), _p(o.uv_grad), _p(o.mass)]
    zs = None if sort_z is None else _f64(sort_z)
    args = [C.c_int(N), *[_p(a) for a in keep[:5]], _p(keep[5]), _p(keep[6]), C.c_int(H), C.c_int(W),
            C.c_double(near), C.c_double(far), C.c_double(pad), C.c_double(mh), _p(np.zeros(3)), *gp, _p(o.image),
            _p(o.depth), _p(o.alpha), _p(o.normal), _p(o.dist), _p(o.visible), _p(o.uv), *og, *rest, _p(o.near),
            _p(zs)]
    if lens is None:
        so.lib().surfel_oracle(*args)
    else:
        kcd = _f64(lo.lens_constants(lens, kc, limit))
        lo.lib().surfel_lens_oracle(C.c_int(lo.LENS_ID[lens]), _p(kcd), *args, _p(o.rays))
    return o


def render(scene, F, grads=None, lens=None, kc=None, near=0.3, far=500.0, pad=100.0, mh=3.0, sort_z=None, limit=None):
    """F [N, D]; grads: None or G [H,W,D], the upstream gradient of the feature map."""
    F = np.asarray(F, np.float64)
    N, D = F.shape
    H, W = int(scene["H"]), int(scene["W"])
    out = SimpleNamespace(fmap=np.zeros((H, W, D)), near=np.zeros((H, W), np.uint8))
    if grads is not None:
        out.g = dict(xyz=np.zeros((N, 3)), quaternion=np.zeros((N, 4)), scale=np.zeros((N, 3)),
                     opacity=np.zeros(np.shape(scene["opacity"])), F=np.zeros((N, D)))
        out.rows, out.uv_grad, out.mass = np.zeros((N, 20)), np.zeros((N, 2)), np.zeros((N, 20))
        out.mass_F = np.zeros((N, D))
    for c0 in range(0, D, 3):
        nc = min(3, D - c0)
        colour = np.zeros((N, 3))
        colour[:, :nc] = F[:, c0:c0 + nc]
        G_img = None
        if grads is not None:
            G_img = np.zeros((H, W, 3))
            G_img[..., :nc] = grads[..., c0:c0 + nc]
        o = _chunk(scene, colour, G_img, lens, kc, near, far, pad, mh, sort_z, limit)
        out.fmap[..., c0:c0 + nc] = o.image[..., :nc]
        out.alpha, out.visible, out.uv, out.rays = o.alpha, o.visible, o.uv, o.rays
        out.near |= o.near
        if grads is not None:
            for k in ("xyz", "quaternion", "scale"):
                out.g[k] += o.g[k]
            out.g["opacity"] += o.g["opacity"].reshape(np.shape(scene["opacity"]))
            out.g["F"][:, c0:c0 + nc] = o.g["colour"][:, :nc]
            out.mass_F[:, c0:c0 + nc] = o.mass[:, 10:10 + nc]
            out.rows += o.rows
            out.mass += o.mass
            out.uv_grad += o.uv_grad
    if grads is not None:
        out.rows[:, 10:13] = 0.0  # the colour's slots: the chunk gradients are d loss / d F
        out.mass[:, 10:13] = 0.0
    return out


def loss(o, grads):
    """<G, feature map> of a forward, for central differences."""
    return float((np.asarray(grads) * o.fmap).sum())
