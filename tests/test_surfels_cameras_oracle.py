"""The camera cases of tests/test_surfels_cameras_gpu.py are sensitive to the faults they are chosen for (CPU only).

The fp64 surfel oracles stand in for a kernel with the fault: they render the case's scene with the parameter the fault
gets wrong (K with fx and fy or cx and cy swapped, the pose's rotation transposed, m_scale = 1 with the far cull kept,
the default mh = 3, the default near or pad, the SH truncated by one degree, the lens ignored).  Against the correct
oracle of the same lens, that render must fail the GPU test's forward criterion, compare_forward with its default
tolerances."""
import math

import numpy as np
import pytest
import torch

from tests import surfels_lens_oracle as lo
from tests import surfels_oracle as so
from tests.test_surfels_cameras_gpu import CASES, TILE, camera_scene
from tests.test_surfels_gpu import MAPS, compare_forward
from tests.test_surfels_lens_gpu import LENSES


def swap_f(sc, p, cam):
    K = sc["K"].copy()
    K[0, 0], K[1, 1] = K[1, 1], K[0, 0]
    return dict(sc, K=K), p, cam


def swap_c(sc, p, cam):
    K = sc["K"].copy()
    K[0, 2], K[1, 2] = K[1, 2], K[0, 2]
    return dict(sc, K=K), p, cam


def transpose_rotation(sc, p, cam):
    T = sc["T"].copy()
    T[:3, :3] = T[:3, :3].T
    return dict(sc, T=T), p, cam


def sh_degree(d):
    def f(sc, p, cam):
        return dict(sc, sh=None if d == 0 else np.ascontiguousarray(sc["sh"][:, :, :(d + 1) ** 2 - 1])), p, cam
    return f


def param(**kw):
    def f(sc, p, cam):
        return sc, dict(p, **kw), cam
    return f


def m_scale_ignored(sc, p, cam):
    """m_scale = 1 with the same visible set: the surfels beyond far dropped (the kernel culls them), far = inf"""
    T = sc["T"].astype(np.float64)
    keep = (sc["xyz"].astype(np.float64) @ T[:3, :3].T + T[:3, 3])[:, 2] <= p["far"]
    n = sc["xyz"].shape[0]
    return {k: (v[keep] if isinstance(v, np.ndarray) and v.shape[:1] == (n,) else v) for k, v in sc.items()}, \
        dict(p, far=math.inf), cam


def lens_ignored(sc, p, cam):
    return sc, p, "pinhole"


FAULTS = [("A", "pinhole", "fx and fy swapped", swap_f), ("A", "pinhole", "cx and cy swapped", swap_c),
          ("A", "pinhole", "rotation transposed", transpose_rotation),
          ("A", "pinhole", "SH 1 read as degree 0", sh_degree(0)),
          ("A", "fisheye", "fx and fy swapped", swap_f), ("A", "opencv", "lens ignored", lens_ignored),
          ("B", "pinhole", "m_scale = 1, far cull kept", m_scale_ignored),
          ("B", "fisheye", "m_scale = 1, far cull kept", m_scale_ignored),
          ("B", "pinhole", "mh = 3 instead of 2", param(mh=3.0)),
          ("B", "pinhole", "near = 0.3 instead of 0.8", param(near=0.3)),
          ("B", "pinhole", "pad = 100 instead of 0", param(pad=100.0)),
          ("B", "pinhole", "SH 2 read as degree 1", sh_degree(1)), ("B", "fisheye", "lens ignored", lens_ignored),
          ("C", "pinhole", "fx and fy swapped", swap_f), ("C", "pinhole", "cx and cy swapped", swap_c),
          ("C", "pinhole", "rotation transposed", transpose_rotation),
          ("C", "pinhole", "mh = 3 instead of 4", param(mh=3.0)),
          ("C", "pinhole", "SH 3 read as degree 2", sh_degree(2)), ("C", "opencv", "cx and cy swapped", swap_c)]
BG = np.array([0.2, 0.4, 0.7])
_cache = {}


def render(sc, p, cam):
    if cam == "pinhole":
        return so.render(sc, BG, **p)
    lens, k = LENSES[cam]
    return lo.render(sc, BG, lens, k, **p)


def reference(case, cam):
    if (case, cam) not in _cache:
        c = CASES[case]
        sc = camera_scene(case)
        p = dict(near=c.near, far=c.far, pad=c.pad, mh=c.mh)
        _cache[case, cam] = (sc, p, render(sc, p, cam))
    return _cache[case, cam]


@pytest.mark.parametrize("case", list(CASES))
def test_the_correct_render_passes_its_own_criteria(case):
    """The criteria are not trivially failed: the oracle against itself passes, and the case's frame has partial-tile
    pixels with contributors."""
    c = CASES[case]
    sc, p, o = reference(case, "pinhole")
    compare_forward({k: torch.from_numpy(getattr(o, k)) for k, _ in MAPS}, o)
    a = o.alpha[..., 0]
    assert (a[:, c.W // TILE * TILE:] > 0).sum() >= 10 and (a[c.H // TILE * TILE:, :] > 0).sum() >= 10


@pytest.mark.parametrize("case,cam,fault,mutate", FAULTS, ids=[f"{c} {m}: {f}" for c, m, f, _ in FAULTS])
def test_each_fault_fails_the_case_s_criteria(case, cam, fault, mutate):
    sc, p, o = reference(case, cam)
    f = render(*mutate(sc, p, cam))
    out = {k: torch.from_numpy(getattr(f, k)) for k, _ in MAPS}
    with pytest.raises(AssertionError) as e:
        compare_forward(out, o)
    print(f"case {case}, {cam}, {fault}: {e.value}")
