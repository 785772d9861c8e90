"""The C ABI driven with RAW device pointers through ctypes — no torch types cross the boundary (torch is only the
allocator here, any cudaMalloc'd memory would do).  What a cgo / JNI / ctypes host binding would call: the tile
renderer forward + backward on packed per-gaussian records read through a sorted id array, and the camera-centre
kernel; checked against the torch binding of the same library (which the parity tests pin to the reference)."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

import gaussian_splatting_b200 as gsb
from gaussian_splatting_b200 import synth
from gaussian_splatting_b200.rasterize import project_and_bin
from gaussian_splatting_b200.structs import Camera
from tests import scenes

pytestmark = pytest.mark.gpu
LIB = Path(__file__).resolve().parents[1] / "gaussian_splatting_b200" / "libgsr_b200.so"


def ptr(t):
    return C.c_void_p(t.data_ptr())


def test_render_through_ctypes_matches_the_binding():
    lib = C.CDLL(str(LIB))
    dev = torch.device("cuda:0")
    sc = scenes.np_scene(3000, "tiny", sh_degree=0, seed=2, sigma_px=(2.0, 0.5, 0.5, 8.0))
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    from gaussian_splatting_b200.structs import Gaussians

    g = Gaussians(to(sc["xyz"]), to(sc["rgb"]), to(sc["opacity"]), to(sc["scale"]), to(sc["quaternion"]), None)
    cam = Camera(sc["W"], sc["H"], to(sc["K"]))
    with torch.no_grad():
        s = project_and_bin(g, to(sc["T"]), cam, 0.3, 500.0, 100, 3.0)
    M, P, H, W = s.uv.shape[0], s.sorted_idx.numel(), sc["H"], sc["W"]
    uv, opa, rgb, conic = (t.contiguous() for t in (s.uv, s.opacity.reshape(-1), s.rgb, s.conic))
    bg = torch.full((3,), 0.5, device=dev)
    G = synth.make_upstream_grad("tiny", device=dev)
    # --- the C ABI, raw pointers
    rec = torch.empty(max(M, 1), 12, device=dev)
    n_px = torch.empty(H, W, dtype=torch.int32, device=dev)
    w_px, image = torch.empty(H, W, device=dev), torch.empty(H, W, 3, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    lib.gsr_contribution_mask_words.restype = C.c_size_t
    lib.gsr_contribution_mask_words.argtypes = [C.c_int64, C.c_int, C.c_int]
    words = lib.gsr_contribution_mask_words(P, H, W)
    masks = torch.zeros(words, dtype=torch.int32, device=dev)
    assert lib.gsr_pack_gaussian_records(C.c_int(M), ptr(uv), ptr(opa), ptr(rgb), ptr(conic), ptr(rec), stream) == 0
    # pair list as a sorted id array (no keys, id_bits 0), no depth / alpha maps
    ids = (None, C.c_int(0), ptr(s.sorted_idx), None, C.c_uint32(0), C.c_int(0))
    assert lib.gsr_render_forward_gather(ptr(rec), *ids, ptr(s.tile_ranges), ptr(bg), C.c_int(H), C.c_int(W),
                                         ptr(n_px), ptr(w_px), ptr(image), None, None, ptr(masks), stream) == 0
    grads = [torch.zeros(M, 3, device=dev), torch.zeros(M, device=dev), torch.zeros(M, 2, device=dev),
             torch.zeros(M, 3, device=dev)]

    def backward(out, m):  # planar gradient arrays (grad_rows NULL)
        return lib.gsr_render_backward_gather(C.c_int(0), ptr(rec), *ids, ptr(s.tile_ranges), ptr(bg), C.c_int(H),
                                              C.c_int(W), ptr(n_px), ptr(w_px), ptr(G), None, None,
                                              *[ptr(t) for t in out], None, m, stream)

    assert backward(grads, ptr(masks)) == 0
    # the same without the forward's masks (NULL): the backward finds its candidates itself
    grads0 = [torch.zeros_like(t) for t in grads]
    assert backward(grads0, None) == 0
    # --- the torch binding (reference surface)
    ext = gsb.native()
    n2, w2, image2 = torch.zeros_like(n_px), torch.zeros_like(w_px), torch.zeros_like(image)
    rays = torch.zeros(1, 1, 1, device=dev)
    ext.render_tiles_cuda(uv, opa.view(-1, 1), rgb, conic, rays, s.tile_ranges, s.sorted_idx, bg, n2, w2, image2)
    g2 = [torch.zeros(M, 3, device=dev), torch.zeros(M, 1, device=dev), torch.zeros(M, 2, device=dev),
          torch.zeros(M, 3, device=dev)]
    ext.render_tiles_backward_cuda(uv, opa.view(-1, 1), rgb, conic, rays, s.tile_ranges, s.sorted_idx, bg, n2, w2, G, *g2)
    torch.cuda.synchronize()
    assert torch.equal(image, image2) and torch.equal(n_px, n2) and torch.equal(w_px, w2)
    for a, a0, b in zip(grads, grads0, g2):
        scale = float(b.abs().max())
        assert float((a.reshape(-1) - b.reshape(-1)).abs().max()) <= 2e-5 * scale
        assert float((a0.reshape(-1) - b.reshape(-1)).abs().max()) <= 2e-5 * scale
    # bad arguments come back as status codes, not exceptions or crashes
    assert lib.gsr_render_forward_gather(ptr(rec), *ids, ptr(s.tile_ranges), ptr(bg), C.c_int(0), C.c_int(W),
                                         ptr(n_px), ptr(w_px), ptr(image), None, None, None, stream) != 0


def test_camera_centre_through_ctypes():
    lib = C.CDLL(str(LIB))
    dev = torch.device("cuda:0")
    T = synth.make_pose(5, 8, device=dev)
    out = torch.empty(3, device=dev)
    assert lib.gsr_camera_centre(ptr(T), ptr(out), C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    torch.cuda.synchronize()
    assert torch.equal(out, torch.inverse(T)[:3, 3].contiguous())
    assert lib.gsr_camera_centre(None, ptr(out), None) != 0
