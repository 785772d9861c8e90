"""Cost of the anti-aliased mode: rasterize() forward + backward at 1080p, 3 M gaussians, SH degree 3, in its default
form and with antialiased=True (opacity compensation for the 0.25 px^2 dilation; a loss on the image).

Timing: CUDA events around `--iters` forward+backward steps, the two arms alternated in `--rounds` rounds in one
process after `--warmup` steps of each; the median round is reported, with min / max.  Per-stage times (the
rasterizer's own CUDA-event profile: preprocess, binning, render forward / backward, per-gaussian backward) are the
median over `--profile-steps` separate profiled steps of each arm.  Also reported: the (gaussian, tile) pair count of
each arm (the compensated opacity gives tighter culling bounds).  Prints one JSON line with the card's name and power
limit."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3_000_000)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.rasterize import rasterize
    from gaussian_splatting_b200.structs import Camera

    assert torch.cuda.is_available(), "bench_antialiased.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam0 = synth.make_camera("1080p", device=dev)
    cam = Camera(1920, 1080, cam0.K)
    T = synth.make_pose(2, 8, device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    gen = torch.Generator().manual_seed(1)
    G = (torch.randn(1080, 1920, 3, generator=gen) / (3.0 * 1080 * 1920)).to(dev)
    params = [p for p in (g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh)]

    def step(antialiased, profile=None):
        for p in params:
            p.grad = None
        out = rasterize(g, T, cam, 0.3, 500.0, 100.0, 3.0, True, bg, profile=profile, return_state=True,
                        antialiased=antialiased)
        out[0].backward(G)
        return out[-1].P

    arms = {"default": lambda: step(False), "antialiased": lambda: step(True)}
    pairs = {}
    for name, fn in arms.items():
        for _ in range(a.warmup):
            pairs[name] = int(fn())
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                fn()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.iters)
    ms = {k: statistics.median(v) for k, v in times.items()}

    stages = {}
    for name, flag in (("default", False), ("antialiased", True)):
        per = {}
        for _ in range(a.profile_steps):
            prof = []
            step(flag, profile=prof)
            torch.cuda.synchronize()
            for stage, e0, e1 in prof:
                per.setdefault(stage, []).append(e0.elapsed_time(e1))
        stages[name] = {k: round(statistics.median(v), 4) for k, v in per.items()}

    line = {
        "bench": "rasterize_antialiased", "gaussians": a.n, "sh_degree": 3, "image_hw": [1080, 1920],
        "ms_fwd_bwd": {k: round(v, 4) for k, v in ms.items()},
        "ms_spread_min_max": {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
        "antialiased_overhead_ms": round(ms["antialiased"] - ms["default"], 4),
        "antialiased_overhead_rel": round(ms["antialiased"] / ms["default"] - 1.0, 4),
        "pairs": pairs,
        "ms_per_stage_median": stages,
        "timing": f"CUDA events, {a.warmup} warm-up steps per arm, {a.rounds} alternating rounds of {a.iters} steps, "
                  f"median round; stages: median of {a.profile_steps} profiled steps",
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
