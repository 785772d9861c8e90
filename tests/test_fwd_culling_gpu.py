"""The forward's exact ellipse-vs-block culling (gsr_record.cuh row_cull) is invisible in the results: the tile
renderers built with it and built with the bounding circle AND box it replaces (-DGSR_CULL_BOX=1, the same kernels)
give the same image, per-pixel count, final weight, contribution-mask words and depth / alpha bits on the same
inputs, and the unmasked backward (which repeats the forward's culling) the same gradients up to the atomics' order.
Needs an H100 and nvcc (the variant is compiled into a temporary directory)."""
import ctypes as C

import numpy as np
import pytest
import torch

from gaussian_splatting_b200 import build as B
from gaussian_splatting_b200 import synth
from gaussian_splatting_b200.rasterize import rasterize
from gaussian_splatting_b200.structs import Camera, Gaussians
from tests import scenes
from tests.test_gradient_rows_gpu import ragged, stack

pytestmark = pytest.mark.gpu
GRAD_ROW = 12  # floats per interleaved per-gaussian gradient row (GSR_GRAD_ROW_FLOATS)


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    box = B.build_render_variant(tmp_path_factory.mktemp("cull_box"), ["-DGSR_CULL_BOX=1"])
    return C.CDLL(str(B.LIB)), C.CDLL(str(box))


def dev():
    return torch.device("cuda:0")


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def np_gaussians(sc):
    to = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev())  # noqa: E731
    return (Gaussians(to(sc["xyz"]), to(sc["rgb"]), to(sc["opacity"]), to(sc["scale"]), to(sc["quaternion"]),
                      to(sc["sh"])), to(sc["T"]), Camera(sc["W"], sc["H"], to(sc["K"])))


def needle_scene():
    """needles: one axis 30-300x the other, at all orientations, over a 320x192 frame"""
    rng = np.random.default_rng(9)
    sc = scenes.np_scene(20_000, "small", sh_degree=0, seed=9)
    n = sc["xyz"].shape[0]
    s = np.log(rng.uniform(0.02, 0.2, n))
    sc["scale"] = np.stack([s, s - np.log(rng.uniform(30, 300, n)), s - np.log(rng.uniform(30, 300, n))],
                           1).astype(np.float32)
    q = rng.normal(size=(n, 4))
    sc["quaternion"] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    return sc


def state_of(g, T, cam, depth_alpha=False, antialiased=False):
    bg = torch.tensor([0.3, 0.5, 0.7], device=dev())
    with torch.no_grad():
        out = rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg, return_state=True, render_depth_alpha=depth_alpha,
                        antialiased=antialiased)
    st = out[-1]
    assert st.P > 0
    return st


def forward(lib, st, masks, depth):
    H, W = st.H, st.W
    n = torch.zeros(H, W, dtype=torch.int32, device=dev())
    w, img = torch.zeros(H, W, device=dev()), torch.zeros(H, W, 3, device=dev())
    d = a = m = None
    if depth:
        d, a = torch.zeros(H, W, device=dev()), torch.zeros(H, W, device=dev())
    if masks:
        lib.gsr_contribution_mask_words.restype = C.c_size_t
        lib.gsr_contribution_mask_words.argtypes = [C.c_int64, C.c_int, C.c_int]
        m = torch.zeros(lib.gsr_contribution_mask_words(st.P, H, W), dtype=torch.int32, device=dev())
    keys = st.keys_sorted if st.keys_sorted is not None else None
    ids = None if keys is not None else st._ids_sorted
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.gsr_render_forward_gather(ptr(st.records), ptr(keys), C.c_int(st.id_bits), ptr(ids),
                                       ptr(st.zkey) if depth else None, C.c_uint32(st.depth_base),
                                       C.c_int(st.depth_bits), ptr(st.ranges), ptr(st.background), C.c_int(H),
                                       C.c_int(W), ptr(n), ptr(w), ptr(img), ptr(d), ptr(a), ptr(m), stream)
    assert rc == 0
    torch.cuda.synchronize()
    return dict(image=img, n=n, w=w, depth=d, alpha=a, masks=m)


def backward_unmasked(lib, st, fw):
    H, W = st.H, st.W
    G = torch.from_numpy(np.random.default_rng(3).normal(size=(H, W, 3)).astype(np.float32) / (H * W)).to(dev())
    rows = torch.zeros(st.N * GRAD_ROW, device=dev())
    keys = st.keys_sorted if st.keys_sorted is not None else None
    ids = None if keys is not None else st._ids_sorted
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.gsr_render_backward_gather(C.c_int(0), ptr(st.records), ptr(keys), C.c_int(st.id_bits), ptr(ids), None,
                                        C.c_uint32(st.depth_base), C.c_int(st.depth_bits), ptr(st.ranges),
                                        ptr(st.background), C.c_int(H), C.c_int(W), ptr(fw["n"]), ptr(fw["w"]), ptr(G),
                                        None, None, None, None, None, None, ptr(rows), None, stream)
    assert rc == 0
    torch.cuda.synchronize()
    return rows


def same_bits(st, libs, masks=True, depth=False, grads=False):
    new, box = (forward(lib, st, masks, depth) for lib in libs)
    for k in ("image", "n", "w", "depth", "alpha", "masks"):
        if new[k] is None:
            continue
        assert torch.equal(new[k].view(torch.int32) if new[k].is_floating_point() else new[k],
                           box[k].view(torch.int32) if box[k].is_floating_point() else box[k]), k
    assert int(new["n"].max()) > 0
    if masks:
        assert bool((new["masks"] != 0).any())
    if grads:  # the unmasked backward builds the same candidate lists as the forward; only the order of the
        # per-(gaussian, tile) atomics differs between runs (4e-5 of the largest entry measured on the needle scene)
        g_new, g_box = (backward_unmasked(lib, st, new) for lib in libs)
        scale = float(g_box.abs().max())
        assert scale > 0 and float((g_new - g_box).abs().max()) <= 2e-4 * scale


@pytest.fixture(scope="module")
def bench_scene():
    return synth.make_gaussians(3_000_000, "1080p", sh_degree=3, seed=0, device=dev()), \
        synth.make_camera("1080p", device=dev())


@pytest.mark.parametrize("pose", [0, 3, 6])
def test_bench_scene_same_bits(libs, bench_scene, pose):
    g, cam = bench_scene
    same_bits(state_of(g, synth.make_pose(pose, 8, device=dev()), cam), libs, grads=pose == 0)


def test_bench_scene_depth_alpha_and_antialiased(libs, bench_scene):
    g, cam = bench_scene
    st = state_of(g, synth.make_pose(1, 8, device=dev()), cam, depth_alpha=True, antialiased=True)
    same_bits(st, libs, depth=True)
    same_bits(st, libs, masks=False, depth=True)


def test_720p_100k_same_bits(libs):
    g, T, cam = np_gaussians(scenes.np_scene(100_000, "720p", 3, seed=0))
    st = state_of(g, T, cam)
    same_bits(st, libs)
    same_bits(st, libs, masks=False, grads=True)


@pytest.mark.parametrize("H,W", [(50, 37), (17, 33)])
def test_ragged_sizes_same_bits(libs, H, W):
    g, T, cam = np_gaussians(ragged(H, W, 0))
    same_bits(state_of(g, T, cam), libs, grads=True)


@pytest.mark.parametrize("which", ["deep", "saturating"])
def test_stacks_same_bits(libs, which):
    sc = stack(3000, -5.0) if which == "deep" else stack(6000, 3.0, spread=0.05, scale=(0.03, 0.07))
    g, T, cam = np_gaussians(sc)
    st = state_of(g, T, cam)
    same_bits(st, libs, grads=True)
    same_bits(st, libs, depth=True)


@pytest.mark.parametrize("mode", ["plain", "depth_alpha", "antialiased"])
def test_needles_same_bits(libs, mode):
    g, T, cam = np_gaussians(needle_scene())
    st = state_of(g, T, cam, depth_alpha=mode == "depth_alpha", antialiased=mode == "antialiased")
    same_bits(st, libs, depth=mode == "depth_alpha", grads=mode == "plain")
    same_bits(st, libs, masks=False)
