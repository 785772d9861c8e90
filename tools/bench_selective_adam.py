"""Cost of the visibility-masked Adam step against the dense one at 3 M gaussians, SH degree 3
(FlatAdam.step(grad, visible=...), csrc/gsr_adam_selective.cu, against FlatAdam.step(grad), csrc/gsr_adam.cu).

CUDA events around `--iters` launches; for every mask, `--rounds` rounds that alternate the dense and the selective
step in one process after `--warmup` launches of each; median round reported with min / max.  Masks:
  * view:        the `state.visible` of bench.py's eight 1080p views of the synthetic scene (its near / far / culling
                 padding), with the visible fraction of each;
  * random f:    each row visible with probability f, f in 0.1, 0.25, 0.5, 0.75, 1.0;
  * contiguous f: the first round(f N) rows.
Traffic model: 28 B per parameter of the rows updated (p, g, m, v read; p, m, v written) + N mask bytes for the
selective step, 28 B per parameter for the dense one.  Prints one JSON line with the card's name, power limit and
clocks, read in the same run."""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_loss import gpu_info  # noqa: E402

FRACTIONS = (0.1, 0.25, 0.5, 0.75, 1.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3_000_000)
    ap.add_argument("--sh-degree", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.flat_adam import FlatAdam
    from gaussian_splatting_b200.rasterize import rasterize

    assert torch.cuda.is_available(), "bench_selective_adam measures on a CUDA device"
    dev = torch.device("cuda:0")
    n = a.n
    g = synth.make_gaussians(n, "1080p", sh_degree=a.sh_degree, seed=0, device=dev)
    opt = FlatAdam.for_gaussians(g)
    floats_per_row = 14 + 3 * ((a.sh_degree + 1) ** 2 - 1)
    grad = torch.randn_like(opt.p) * 1e-3

    # bench.py's views: synth pose ring of 8, 1080p, synth.DEFAULTS culling
    cam = synth.make_camera("1080p", device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    d = synth.DEFAULTS
    masks = {}
    for v in range(8):
        with torch.no_grad():
            _, _, _, st = rasterize(g, synth.make_pose(v, 8, device=dev), cam, d["near_thresh"], d["far_thresh"],
                                    d["cull_mask_padding"], d["mh_dist"], True, bg, return_state=True)
        masks[f"view{v}"] = st.visible.clone()
        del st
    gen = torch.Generator(device=dev).manual_seed(0)
    for f in FRACTIONS:
        masks[f"random_{f}"] = (torch.rand(n, device=dev, generator=gen) < f).to(torch.uint8)
        cont = torch.zeros(n, dtype=torch.uint8, device=dev)
        cont[:round(f * n)] = 1
        masks[f"contiguous_{f}"] = cont
    torch.cuda.empty_cache()

    def timed(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(a.iters):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / a.iters

    def summary(v):
        return dict(median=round(statistics.median(v), 4), min=round(min(v), 4), max=round(max(v), 4))

    dense_fn = lambda: opt.step(grad)  # noqa: E731
    for _ in range(a.warmup):
        dense_fn()
        opt.step(grad, visible=masks["random_0.5"])
    torch.cuda.synchronize()

    dense_bytes = 28 * opt.p.numel()
    dense_all, results = [], {}
    for name, mask in masks.items():
        sel_fn = lambda mask=mask: opt.step(grad, visible=mask)  # noqa: E731
        dense_t, sel_t = [], []
        for _ in range(a.rounds):
            dense_t.append(timed(dense_fn))
            sel_t.append(timed(sel_fn))
        dense_all += dense_t
        rows = int((mask != 0).sum())
        sel_bytes = 28 * floats_per_row * rows + n
        med_d, med_s = statistics.median(dense_t), statistics.median(sel_t)
        results[name] = dict(
            visible_fraction=round(rows / n, 4), dense_ms=summary(dense_t), selective_ms=summary(sel_t),
            selective_over_dense=round(med_s / med_d, 4), model_bytes=sel_bytes,
            achieved_GBps=round(sel_bytes / (med_s * 1e-3) / 1e9, 1))

    line = {
        "bench": "selective_adam", "n": n, "sh_degree": a.sh_degree, "flat_floats": opt.p.numel(),
        "iters": a.iters, "rounds": a.rounds,
        "dense_ms_all_rounds": summary(dense_all), "dense_model_bytes": dense_bytes,
        "dense_achieved_GBps": round(dense_bytes / (statistics.median(dense_all) * 1e-3) / 1e9, 1),
        "masks": results,
        "device": torch.cuda.get_device_name(0),
        "power_limit_and_max_sm_clock": gpu_info(),
    }
    text = json.dumps(line)
    print(text)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
