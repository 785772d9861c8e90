"""Cost of the blend-weight statistics: rasterize() at 1080p, 3 M gaussians, SH degree 3.

Two measurements, arms alternated in `--rounds` rounds in one process after `--warmup` steps of each, CUDA events
around `--iters` repetitions, median round reported with min / max:
  * a training step (forward + backward) in its default form against the same step with weight_stats=ws, plus the
    per-stage times (the rasterizer's CUDA-event profile) as the median of `--profile-steps` profiled steps;
  * a statistics pass: `--views` forward-only renders under torch.no_grad(), without and with weight_stats.
Prints one JSON line with the card's name, power limit and clocks."""
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
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.densify import WeightStats
    from gaussian_splatting_b200.rasterize import rasterize
    from gaussian_splatting_b200.structs import Camera

    assert torch.cuda.is_available(), "bench_weight_stats.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam0 = synth.make_camera("1080p", device=dev)
    cam = Camera(1920, 1080, cam0.K)
    T = synth.make_pose(2, 8, device=dev)
    poses = [synth.make_pose(v, a.views, device=dev) for v in range(a.views)]
    bg = torch.full((3,), 0.5, device=dev)
    gen = torch.Generator().manual_seed(1)
    G = (torch.randn(1080, 1920, 3, generator=gen) / (3.0 * 1080 * 1920)).to(dev)
    params = [g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh]
    ws = WeightStats(a.n, dev)

    def train_step(stats, profile=None):
        for p in params:
            p.grad = None
        out = rasterize(g, T, cam, 0.3, 500.0, 100.0, 3.0, True, bg, profile=profile,
                        weight_stats=ws if stats else None)
        out[0].backward(G)

    def stats_pass(stats):
        with torch.no_grad():
            for Tv in poses:
                rasterize(g, Tv, cam, 0.3, 500.0, 100.0, 3.0, True, bg, weight_stats=ws if stats else None)

    arms = {"train_default": lambda: train_step(False), "train_weight_stats": lambda: train_step(True),
            "views_no_grad_default": lambda: stats_pass(False), "views_no_grad_weight_stats": lambda: stats_pass(True)}
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
    for name, flag in (("default", False), ("weight_stats", True)):
        per = {}
        for _ in range(a.profile_steps):
            prof = []
            train_step(flag, profile=prof)
            torch.cuda.synchronize()
            for stage, e0, e1 in prof:
                per.setdefault(stage, []).append(e0.elapsed_time(e1))
        stages[name] = {k: round(statistics.median(v), 4) for k, v in per.items()}

    line = {
        "bench": "rasterize_weight_stats", "gaussians": a.n, "sh_degree": 3, "image_hw": [1080, 1920],
        "views_per_pass": a.views,
        "ms": {k: round(v, 4) for k, v in ms.items()},
        "ms_spread_min_max": {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
        "train_overhead_rel": round(ms["train_weight_stats"] / ms["train_default"] - 1.0, 4),
        "views_no_grad_overhead_rel": round(ms["views_no_grad_weight_stats"] / ms["views_no_grad_default"] - 1.0, 4),
        "ms_per_stage_median": stages,
        "render_fwd_overhead_rel": round(stages["weight_stats"]["render_fwd"] / stages["default"]["render_fwd"] - 1.0,
                                         4),
        "timing": f"CUDA events, {a.warmup} warm-up repetitions per arm, {a.rounds} alternating rounds of {a.iters} "
                  f"repetitions, median round (views arms: one repetition = {a.views} views); stages: median of "
                  f"{a.profile_steps} profiled training steps",
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
