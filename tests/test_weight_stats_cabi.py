"""The C ABI entry point gsr_render_forward_gather_stats called directly (ctypes): its argument checks (no GPU
needed: they return before any launch), and on the GPU that all-NULL statistics give exactly gsr_render_forward_gather,
that the statistics equal rasterize(weight_stats=...)'s, and that the pair-count guard adds nothing."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GSR_ERR_BAD_ARG = -1
P = C.c_void_p
ARGS = [P, P, C.c_int, P, P, C.c_uint32, C.c_int, P, P, C.c_int, C.c_int, P, P, P, P, P, P]
STATS_ARGS = ARGS + [P, P, P, P, C.c_int64, P]


def lib():
    so = C.CDLL(str(ROOT / "gaussian_splatting_b200" / "libgsr_b200.so"))
    so.gsr_render_forward_gather.argtypes = ARGS + [P]
    so.gsr_render_forward_gather_stats.argtypes = STATS_ARGS
    return so


def call_stats(so, common, stats, pair_total=None, capacity=0, stream=None):
    return so.gsr_render_forward_gather_stats(*common, *stats, pair_total, capacity, stream)


def dummy_common():
    x = P(256)  # never dereferenced: every call below is refused before a launch
    return [x, x, 20, None, None, 0, 0, x, x, 16, 16, x, x, x, None, None, None]


def test_partial_statistics_and_bad_capacity_are_refused():
    so = lib()
    x = P(256)
    common = dummy_common()
    for stats in ([x, None, None], [None, x, None], [None, None, x], [x, x, None], [x, None, x], [None, x, x]):
        assert call_stats(so, common, stats) == GSR_ERR_BAD_ARG, stats
    for cap in (-1, 2**32, 2**40):
        assert call_stats(so, common, [x, x, x], pair_total=x, capacity=cap) == GSR_ERR_BAD_ARG, cap
    both = list(common)
    both[3] = x  # keys and ids both given
    assert call_stats(so, both, [x, x, x]) == GSR_ERR_BAD_ARG
    half = list(common)
    half[14] = x  # depth without alpha
    assert call_stats(so, half, [x, x, x]) == GSR_ERR_BAD_ARG


def ptr(t):
    return None if t is None else P(t.data_ptr())


@pytest.mark.gpu
def test_direct_calls_on_the_gpu():
    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.densify import WeightStats
    from gaussian_splatting_b200.rasterize import rasterize

    dev = torch.device("cuda:0")
    so = lib()
    g = synth.make_gaussians(20_000, "small", sh_degree=0, seed=4, device=dev, sigma_px=(2.5, 0.5, 0.5, 10.0))
    cam = synth.make_camera("small", device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    ws = WeightStats(20_000, dev)
    with torch.no_grad():
        image, _, _, st = rasterize(g, synth.make_pose(0, 3, device=dev), cam, 0.3, 500.0, 100, 3.0, True, bg,
                                    return_state=True, weight_stats=ws)
    H, W = st.H, st.W
    keyed = st.keys_sorted is not None and st.keys_sorted.numel() > 0
    keys, ids = (st.keys_sorted, None) if keyed else (None, st.ids_sorted)

    def outs():
        return (torch.empty(H, W, dtype=torch.int32, device=dev), torch.empty(H, W, device=dev),
                torch.empty(H, W, 3, device=dev))

    def common(o):
        return [ptr(st.records), ptr(keys), st.id_bits, ptr(ids), None, 0, 0, ptr(st.ranges), ptr(st.background), H, W,
                ptr(o[0]), ptr(o[1]), ptr(o[2]), None, None, None]

    stream = P(torch.cuda.current_stream().cuda_stream)
    ref = outs()
    assert so.gsr_render_forward_gather(*common(ref), stream) == 0
    a = outs()
    assert call_stats(so, common(a), [None, None, None], stream=stream) == 0   # all NULL: the plain call
    ws2 = WeightStats(20_000, dev)
    b = outs()
    assert call_stats(so, common(b), [ptr(ws2.weight_sum), ptr(ws2.weight_max), ptr(ws2.pixel_count)],
                      stream=stream) == 0
    # the guard: a pair total above the capacity the buffers had (a discarded speculative run) adds nothing
    ws3 = WeightStats(20_000, dev)
    total = torch.tensor([(st.M << 32) | st.P], dtype=torch.int64, device=dev)
    c = outs()
    assert call_stats(so, common(c), [ptr(ws3.weight_sum), ptr(ws3.weight_max), ptr(ws3.pixel_count)],
                      pair_total=ptr(total), capacity=st.P - 1, stream=stream) == 0
    ws4 = WeightStats(20_000, dev)
    d = outs()
    assert call_stats(so, common(d), [ptr(ws4.weight_sum), ptr(ws4.weight_max), ptr(ws4.pixel_count)],
                      pair_total=ptr(total), capacity=st.P, stream=stream) == 0
    torch.cuda.synchronize()
    for o in (a, b, c, d):
        for x, y in zip(o, ref):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    assert torch.equal(ref[2], image) and torch.equal(ref[0], st.n_per_pixel)
    assert int(ws.pixel_count.sum()) > 0
    for w in (ws2, ws4):
        assert torch.equal(w.pixel_count, ws.pixel_count) and torch.equal(w.weight_max, ws.weight_max)
        assert float((w.weight_sum - ws.weight_sum).abs().max()) <= 1e-6 * float(ws.weight_sum.abs().max())
    assert int(ws3.pixel_count.abs().sum()) == 0 and float(ws3.weight_sum.abs().sum()) == 0.0
    assert float(ws3.weight_max.abs().sum()) == 0.0
    assert np.isfinite(ws.weight_sum.cpu().numpy()).all()
