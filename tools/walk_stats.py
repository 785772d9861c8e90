"""Walk-step counts of the tile renderers on the bench scene (1080p, 3M Gaussians, SH 3, the 8 bench poses), for the
forward's exact ellipse-vs-block culling and for the bounding circle AND box it replaced (-DGSR_CULL_BOX=1, whose
kernels are the previous ones instruction for instruction).

    python tools/walk_stats.py [--out FILE]

Both variants of the renderers are compiled with -DGSR_STATS into a temporary directory and driven through the C ABI
on the pair lists rasterize() built; per variant and pose, from the GSR_STATS counters:
  fwd_steps_check / fwd_steps_plain  forward walk steps (a warp's steps per batch: its longest lane-group list) in the
                                     CHECK walk and in the plain one
  fwd_listed                         (record, lane group) pairs the forward's lists hold
  bwd_steps / bwd_listed             the same for the masked backward (which walks the contributors only)
Prints one JSON object; needs a GPU and nvcc."""
import argparse
import ctypes as C
import json
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from gaussian_splatting_b200 import build as B  # noqa: E402
from gaussian_splatting_b200 import synth  # noqa: E402
from gaussian_splatting_b200.rasterize import rasterize  # noqa: E402

GRAD_ROW = 12
NAMES = {0: "fwd_steps_check", 1: "fwd_steps_plain", 4: "fwd_listed", 7: "fwd_warp_batches", 8: "bwd_steps",
         15: "bwd_listed", 13: "bwd_warp_batches"}


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def run(lib, st, G):
    H, W, dev = st.H, st.W, st.records.device
    lib.gsr_contribution_mask_words.restype = C.c_size_t
    lib.gsr_contribution_mask_words.argtypes = [C.c_int64, C.c_int, C.c_int]
    masks = torch.zeros(lib.gsr_contribution_mask_words(st.P, H, W), dtype=torch.int32, device=dev)
    n = torch.zeros(H, W, dtype=torch.int32, device=dev)
    w, img = torch.zeros(H, W, device=dev), torch.zeros(H, W, 3, device=dev)
    rows = torch.zeros(st.N * GRAD_ROW, device=dev)
    ids = None if st.keys_sorted is not None else st._ids_sorted
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    stats = (C.c_ulonglong * 16)()
    lib.gsr_debug_stats(stats, 1)
    assert lib.gsr_render_forward_gather(ptr(st.records), ptr(st.keys_sorted), C.c_int(st.id_bits), ptr(ids), None,
                                         C.c_uint32(st.depth_base), C.c_int(st.depth_bits), ptr(st.ranges),
                                         ptr(st.background), C.c_int(H), C.c_int(W), ptr(n), ptr(w), ptr(img), None,
                                         None, ptr(masks), stream) == 0
    assert lib.gsr_render_backward_gather(C.c_int(0), ptr(st.records), ptr(st.keys_sorted), C.c_int(st.id_bits),
                                          ptr(ids), None, C.c_uint32(st.depth_base), C.c_int(st.depth_bits),
                                          ptr(st.ranges), ptr(st.background), C.c_int(H), C.c_int(W), ptr(n), ptr(w),
                                          ptr(G), None, None, None, None, None, None, ptr(rows), ptr(masks),
                                          stream) == 0
    lib.gsr_debug_stats(stats, 1)
    return {name: int(stats[i]) for i, name in NAMES.items()}, img


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    with tempfile.TemporaryDirectory() as tmp:
        variants = {"circle_and_box": ["-DGSR_CULL_BOX=1"], "exact": []}
        for name in variants:
            (Path(tmp) / name).mkdir()
        with ThreadPoolExecutor(2) as ex:
            built = ex.map(lambda kv: B.build_render_variant(Path(tmp) / kv[0], ["-DGSR_STATS", *kv[1]]),
                           variants.items())
            libs = {name: C.CDLL(str(so)) for name, so in zip(variants, built)}
        g = synth.make_gaussians(3_000_000, "1080p", sh_degree=3, seed=0, device=dev)
        cam = synth.make_camera("1080p", device=dev)
        bg = torch.full((3,), 0.5, device=dev)
        G = torch.from_numpy(np.random.default_rng(1).normal(size=(1080, 1920, 3)).astype(np.float32) / 2e6).to(dev)
        out = {"gpu": torch.cuda.get_device_name(0), "scene": "bench: 3M Gaussians, 1080p, SH 3, poses 0-7 of 8",
               "per_pose": []}
        tot = {k: {n: 0 for n in NAMES.values()} for k in libs}
        for pose in range(8):
            with torch.no_grad():
                st = rasterize(g, synth.make_pose(pose, 8, device=dev), cam, 0.3, 500.0, 100, 3.0, True, bg,
                               return_state=True)[-1]
            row, images = {"pose": pose, "P": int(st.P)}, []
            for k, lib in libs.items():
                row[k], img = run(lib, st, G)
                images.append(img)
                for n in NAMES.values():
                    tot[k][n] += row[k][n]
            row["images_equal"] = bool(torch.equal(images[0], images[1]))
            out["per_pose"].append(row)
        out["total"] = tot
        old, new = tot["circle_and_box"], tot["exact"]
        fs = lambda t: t["fwd_steps_check"] + t["fwd_steps_plain"]  # noqa: E731
        out["ratio_exact_over_circle_and_box"] = {
            "fwd_steps": fs(new) / fs(old), "fwd_steps_check": new["fwd_steps_check"] / old["fwd_steps_check"],
            "fwd_steps_plain": new["fwd_steps_plain"] / old["fwd_steps_plain"],
            "fwd_listed": new["fwd_listed"] / old["fwd_listed"], "bwd_steps": new["bwd_steps"] / old["bwd_steps"],
            "bwd_listed": new["bwd_listed"] / old["bwd_listed"]}
    line = json.dumps(out)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
