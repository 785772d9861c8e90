"""The tile renderers' exact recompute of flagged pixels actually runs on the scenes built for it (tests/scenes.py
FLAGGED), and those scenes are what they claim to be — needs an H100 and nvcc.

The forward walk raises a sticky flag instead of doing slow arithmetic inline, and after the walk the whole warp
recomputes each flagged pixel from scratch (gsr_render.cu render_fwd).  Every check of the exact path in the mode
tests (depth/alpha, features, weight statistics, absgrad, antialiased, filter3d, batch, gradient rows) is only worth
something if that path runs.  The renderers are compiled once more with -DGSR_STATS (the same kernels plus device
counters, into a temporary directory) and driven through the C ABI over the fused path's records and pair list:
counter 2 counts the lanes whose pixels carry the walk's `bad` flag (a blend hazard, or build_lists' |det| outside
[1e-18, 1e18] for the whole warp), counter 3 the lanes with `badbits` (a Mahalanobis numerator outside
[2^-67, 2^61), e.g. 0 at an exact centre)."""
import ctypes as C

import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import build as B
from gaussian_splatting_b200.rasterize import rasterize
from tests import scenes
from tests.test_fwd_culling_gpu import forward, np_gaussians

pytestmark = pytest.mark.gpu
TILE = 16
R_DET = 7  # record field: det of the dilated 2-D covariance


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    stats = C.CDLL(str(B.build_render_variant(tmp_path_factory.mktemp("gsr_stats"), ["-DGSR_STATS"])))
    stats.gsr_debug_stats.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    return C.CDLL(str(B.LIB)), stats


def dev():
    return torch.device("cuda:0")


def state_and_uv(sc):
    g, T, cam = np_gaussians(sc)
    with torch.no_grad():
        out = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, torch.tensor([0.3, 0.5, 0.7], device=dev()),
                        return_state=True, render_depth_alpha=True)
    return out[-1], out[2]


def live_lanes(st):
    """Lanes of the warps the forward walks: tiles with a non-empty pair list, warps (16 x 4 pixel bands) with at
    least one pixel in the image; a warp whose pixels all lie outside starts saturated and builds no lists."""
    H, W = st.H, st.W
    tiles_x = (W + TILE - 1) // TILE
    counts = (st.ranges[1:] - st.ranges[:-1]).cpu().numpy()
    lanes = 0
    for t in np.flatnonzero(counts > 0):
        by = (t // tiles_x) * TILE
        lanes += 32 * sum(1 for w in range(TILE // 4) if by + 4 * w < H)
    return lanes


def flag_counts(stats, st, depth):
    buf = (C.c_ulonglong * 16)()
    stats.gsr_debug_stats(buf, 1)
    out = forward(stats, st, True, depth)
    stats.gsr_debug_stats(buf, 1)
    return int(buf[2]), int(buf[3]), out


def huge_listed_in_every_tile(st):
    """Some record with det > 1e18 sits in the pair list of every non-empty tile."""
    det = st.records.view(-1, 12)[:, R_DET].double().cpu().numpy()
    ids = st.ids_sorted.long().cpu().numpy()
    ranges = st.ranges.cpu().numpy()
    huge = det[ids] > 1e18
    nonempty = [(a, b) for a, b in zip(ranges[:-1], ranges[1:]) if b > a]
    return len(nonempty) > 0 and all(huge[a:b].any() for a, b in nonempty)


@pytest.mark.parametrize("name", list(scenes.FLAGGED))
def test_the_scenes_are_what_they_claim(name):
    st, uv = state_and_uv(scenes.flagged_scene(name))
    u = uv.cpu().numpy()
    on_pixels = (u == np.round(u)).all(1) & (u[:, 0] >= 0) & (u[:, 0] < st.W) & (u[:, 1] >= 0) & (u[:, 1] < st.H)
    assert int(on_pixels.sum()) >= 150, int(on_pixels.sum())   # exact-centre splats survived culling
    assert huge_listed_in_every_tile(st) == ("huge" in name)


@pytest.mark.parametrize("depth", [False, True], ids=["colour", "depth"])
@pytest.mark.parametrize("name", list(scenes.FLAGGED))
def test_flags_are_raised_and_change_no_output(libs, name, depth):
    lib, stats = libs
    st, _ = state_and_uv(scenes.flagged_scene(name))
    lanes = live_lanes(st)
    bad, badbits, out = flag_counts(stats, st, depth)
    print(f"{name} {'depth' if depth else 'colour'}: {bad} lanes bad, {badbits} lanes badbits, of {lanes}")
    assert badbits > 0
    if "huge" in name:  # whole warps: those whose band some det > 1e18 record's ellipse reaches (measured on an H100:
        # 42 of the 64 warps at 64 x 64, 13 of the 40 live ones at 37 x 61; the off-axis huge splats are needles)
        assert bad % 32 == 0 and bad >= lanes // 4
    else:
        assert bad <= lanes // 100
    ref = forward(lib, st, True, depth)
    for k in ("image", "n", "w", "depth", "alpha", "masks"):
        if ref[k] is not None:
            assert torch.equal(out[k].view(torch.int32), ref[k].view(torch.int32)), k
    assert torch.equal(ref["n"], st.n_per_pixel) and torch.equal(ref["w"].view(torch.int32),
                                                                   st.w_per_pixel.view(torch.int32))
