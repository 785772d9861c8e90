"""Cost of the absolute screen-space gradients: rasterize() forward + backward at 1080p, 3 M gaussians, SH degree 3, in
its default form, with absgrad=True, and with absgrad=True + render_depth_alpha=True (a loss on all three maps).

Timing: CUDA events around `--iters` forward+backward steps, the three arms alternated in `--rounds` rounds in one
process after `--warmup` steps of each; the median round is reported, with min / max.  Per-stage times (the
rasterizer's own CUDA-event profile: preprocess, binning, render forward / backward, per-gaussian backward) are the
median over `--profile-steps` separate profiled steps of each arm.  Prints one JSON line with the card's name, power
limit and clocks."""
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

    assert torch.cuda.is_available(), "bench_absgrad.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam0 = synth.make_camera("1080p", device=dev)
    cam = Camera(1920, 1080, cam0.K)
    T = synth.make_pose(2, 8, device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    gen = torch.Generator().manual_seed(1)
    G = (torch.randn(1080, 1920, 3, generator=gen) / (3.0 * 1080 * 1920)).to(dev)
    Gd = (torch.randn(1080, 1920, 1, generator=gen) / (1080 * 1920)).to(dev)
    Ga = (torch.randn(1080, 1920, 1, generator=gen) / (1080 * 1920)).to(dev)
    params = [p for p in (g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh)]

    def step(absgrad, depth_alpha, profile=None):
        for p in params:
            p.grad = None
        out = rasterize(g, T, cam, 0.3, 500.0, 100.0, 3.0, True, bg, profile=profile, render_depth_alpha=depth_alpha,
                        absgrad=absgrad)
        if depth_alpha:
            torch.autograd.backward([out[0], out[3], out[4]], [G, Gd, Ga])
        else:
            out[0].backward(G)

    flags = {"default": (False, False), "absgrad": (True, False), "absgrad_depth_alpha": (True, True)}
    arms = {k: (lambda f=f: step(*f)) for k, f in flags.items()}
    for fn in arms.values():
        for _ in range(a.warmup):
            fn()
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
    for name, f in flags.items():
        per = {}
        for _ in range(a.profile_steps):
            prof = []
            step(*f, profile=prof)
            torch.cuda.synchronize()
            for stage, e0, e1 in prof:
                per.setdefault(stage, []).append(e0.elapsed_time(e1))
        stages[name] = {k: round(statistics.median(v), 4) for k, v in per.items()}

    line = {
        "bench": "rasterize_absgrad", "gaussians": a.n, "sh_degree": 3, "image_hw": [1080, 1920],
        "ms_fwd_bwd": {k: round(v, 4) for k, v in ms.items()},
        "ms_spread_min_max": {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
        "absgrad_overhead_ms": round(ms["absgrad"] - ms["default"], 4),
        "absgrad_overhead_rel": round(ms["absgrad"] / ms["default"] - 1.0, 4),
        "ms_per_stage_median": stages,
        "render_bwd_overhead_rel": round(stages["absgrad"]["render_bwd"] / stages["default"]["render_bwd"] - 1.0, 4),
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
