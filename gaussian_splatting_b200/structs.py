"""Containers on the rasterization path (mirror of the reference's splat_py/structs.py:30-138).

Only what the path touches is here: the Gaussian parameter set, the pinhole camera and the
16-pixel tile grid.  Field names and shapes are the reference's so that objects built by the
reference trainer can be passed straight in.
"""
from __future__ import annotations

import torch

TILE_EDGE_LENGTH_PX = 16  # splat_py/structs.py:4


class Camera:
    """Pinhole camera: image size in pixels and a 3x3 intrinsic matrix (splat_py/structs.py:30-43)."""

    def __init__(self, width, height, K):
        self.width = width
        self.height = height
        self.K = K


# COLMAP camera model -> its parameter names (colmap/src/colmap/sensor/models.h), for the models the fused rasterizer
# projects through
_COLMAP_PARAMS = {
    "SIMPLE_PINHOLE": ("f", "cx", "cy"),
    "PINHOLE": ("fx", "fy", "cx", "cy"),
    "SIMPLE_RADIAL": ("f", "cx", "cy", "k"),
    "RADIAL": ("f", "cx", "cy", "k1", "k2"),
    "OPENCV": ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2"),
    "FULL_OPENCV": ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3", "k4", "k5", "k6"),
    "OPENCV_FISHEYE": ("fx", "fy", "cx", "cy", "k1", "k2", "k3", "k4"),
}


def camera_from_colmap(model, width, height, params, device="cpu"):
    """(Camera, lens_kwargs) for a COLMAP camera: `model` is COLMAP's model name, `params` its parameter list in
    COLMAP's order.  K [3,3] fp32 on `device` holds fx fy cx cy; lens_kwargs is the keyword the lens needs for
    rasterize / rasterize_batch: {} for SIMPLE_PINHOLE and PINHOLE, {"distortion": (k1, k2, p1, p2, k3)} for
    SIMPLE_RADIAL, RADIAL, OPENCV and FULL_OPENCV, {"fisheye": (k1, k2, k3, k4)} for OPENCV_FISHEYE:

        cam, lens = camera_from_colmap(c.model, c.width, c.height, c.params, "cuda")
        image, mask, uv = rasterize(gaussians, T, cam, 0.3, 500.0, 100, 3.0, True, bg, **lens)

    FULL_OPENCV is accepted only with k4 = k5 = k6 = 0 (the rational terms are not modelled).  Any other model, or a
    parameter list of the wrong length, raises ValueError."""
    name = str(model).upper()
    if name not in _COLMAP_PARAMS:
        raise ValueError(f"COLMAP camera model {model!r} is not supported: use one of {', '.join(_COLMAP_PARAMS)}")
    params = [float(v) for v in params]
    if len(params) != len(_COLMAP_PARAMS[name]):
        raise ValueError(f"COLMAP {name} has {len(_COLMAP_PARAMS[name])} parameters "
                         f"({' '.join(_COLMAP_PARAMS[name])}), got {len(params)}")
    p = dict(zip(_COLMAP_PARAMS[name], params))
    if "f" in p:
        p["fx"] = p["fy"] = p["f"]
    if name == "FULL_OPENCV" and (p["k4"], p["k5"], p["k6"]) != (0.0, 0.0, 0.0):
        raise ValueError("COLMAP FULL_OPENCV with rational terms k4 k5 k6 != 0 is not supported")
    K = torch.tensor([[p["fx"], 0.0, p["cx"]], [0.0, p["fy"], p["cy"]], [0.0, 0.0, 1.0]], dtype=torch.float32,
                     device=device)
    cam = Camera(int(width), int(height), K)
    if name == "OPENCV_FISHEYE":
        return cam, {"fisheye": (p["k1"], p["k2"], p["k3"], p["k4"])}
    if name in ("SIMPLE_PINHOLE", "PINHOLE"):
        return cam, {}
    if name == "SIMPLE_RADIAL":
        p["k1"] = p["k"]
    return cam, {"distortion": tuple(p.get(k, 0.0) for k in ("k1", "k2", "p1", "p2", "k3"))}


class Image:
    """An 8-bit RGB image with its camera id and world->camera pose (splat_py/structs.py:14-27)."""

    def __init__(self, image, camera_id, camera_T_world):
        self.image = image
        self.camera_id = camera_id
        self.camera_T_world = camera_T_world


class Gaussians(torch.nn.Module):
    """Mutable Gaussian parameters (splat_py/structs.py:46-114).

    xyz [N,3] world positions, quaternion [N,4] (w,x,y,z, not normalised), scale [N,3] (log),
    opacity [N,1] (logit), rgb [N,3] (SH DC term, colour / 0.28209), sh [N,3,K] or None.
    """

    _FIELDS = ("xyz", "rgb", "opacity", "scale", "quaternion", "sh")

    def __init__(self, xyz, rgb, opacity, scale, quaternion, sh=None):
        super().__init__()
        self.xyz, self.rgb, self.opacity = xyz, rgb, opacity
        self.scale, self.quaternion, self.sh = scale, quaternion, sh
        self.verify_sizes()

    def __len__(self):
        return self.xyz.shape[0]

    def verify_sizes(self):
        n = self.xyz.shape[0]
        expect = {"xyz": 3, "rgb": 3, "opacity": 1, "scale": 3, "quaternion": 4}
        for name, cols in expect.items():
            t = getattr(self, name)
            assert t.shape[0] == n and t.shape[1] == cols, f"{name} must be [{n},{cols}], got {tuple(t.shape)}"
        if self.sh is not None:
            assert self.sh.shape[0] == n and self.sh.shape[1] == 3, "sh must be [N,3,K]"

    def filter_in_place(self, keep_mask):
        for name in self._FIELDS:
            t = getattr(self, name)
            if t is not None:
                setattr(self, name, torch.nn.Parameter(t.detach()[keep_mask]))
        self.verify_sizes()

    def append(self, xyz, rgb, opacity, scale, quaternion, sh=None):
        new = dict(xyz=xyz, rgb=rgb, opacity=opacity, scale=scale, quaternion=quaternion, sh=sh)
        for name, extra in new.items():
            if extra is None:
                continue
            cur = getattr(self, name)
            setattr(self, name, torch.nn.Parameter(torch.cat((cur.detach(), extra.detach()), dim=0)))
        self.verify_sizes()


class Tiles:
    """Tile grid covering an image, padded up to whole tiles (splat_py/structs.py:117-138)."""

    def __init__(self, image_height, image_width, device):
        e = TILE_EDGE_LENGTH_PX
        self.image_height, self.image_width, self.device = image_height, image_width, device
        self.tile_edge_size = e
        self.y_tiles_count = -(-int(image_height) // e)
        self.x_tiles_count = -(-int(image_width) // e)
        self.image_height_padded = self.y_tiles_count * e
        self.image_width_padded = self.x_tiles_count * e
        self.tile_count = self.y_tiles_count * self.x_tiles_count
