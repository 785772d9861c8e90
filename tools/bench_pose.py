"""Cost of the camera pose gradient: forward + backward on the bench scene (synth-v1, 3 M gaussians, SH degree 3, 1080p,
bench.py's intrinsics K and pose) with the pose gradient off and on, for the pinhole, for a typical OPENCV calibration
(K_TYPICAL below) and for rasterize_batch with C = 8 views (the bench's 8 poses), loss <G, image> (per view).

Timing: CUDA events around `--iters` forward+backward steps, the six arms alternated in `--rounds` rounds in one process
after `--warmup` steps of each; the median round is reported, with min / max.  Per-stage times (the rasterizer's own
CUDA-event profile, where "preprocess_bwd" is the per-gaussian backward and, with the pose, its reduction) are the
median over `--profile-steps` separate profiled steps of each arm.  Prints one JSON line with the card's name and power
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

K_TYPICAL = (-0.12, 0.03, 5e-4, -3e-4, 0.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3_000_000)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import rasterize_batch, synth
    from gaussian_splatting_b200.rasterize import rasterize

    assert torch.cuda.is_available(), "bench_pose.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam = synth.make_camera("1080p", device=dev)
    T = synth.make_pose(2, 8, device=dev)
    Ts = torch.stack([synth.make_pose(c, a.views, device=dev) for c in range(a.views)])
    bg = torch.full((3,), 0.5, device=dev)
    gen = torch.Generator().manual_seed(1)
    G = (torch.randn(cam.height, cam.width, 3, generator=gen) / (3.0 * cam.height * cam.width)).to(dev)
    params = [g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh]
    arms = {"pinhole": (False, None, False), "pinhole_pose": (False, None, True),
            "distortion": (False, K_TYPICAL, False), "distortion_pose": (False, K_TYPICAL, True),
            f"batch{a.views}": (True, None, False), f"batch{a.views}_pose": (True, None, True)}

    def step(arm, profile=None):
        batch, k, pose = arms[arm]
        for p in params:
            p.grad = None
        if batch:
            Tp = Ts.detach().requires_grad_(pose)
            out = rasterize_batch(g, Tp, cam, 0.3, 500.0, 100.0, 3.0, True, bg, profile=profile)
            (out[0] * G).sum().backward()
        else:
            Tp = T.detach().requires_grad_(pose)
            out = rasterize(g, Tp, cam, 0.3, 500.0, 100.0, 3.0, True, bg, profile=profile, distortion=k)
            (out[0] * G).sum().backward()
        assert (Tp.grad is not None) == pose

    for arm in arms:
        for _ in range(a.warmup):
            step(arm)
    torch.cuda.synchronize()
    times = {arm: [] for arm in arms}
    for _ in range(a.rounds):
        for arm in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                step(arm)
            e1.record()
            e1.synchronize()
            times[arm].append(e0.elapsed_time(e1) / a.iters)
    ms = {arm: statistics.median(v) for arm, v in times.items()}

    stages = {}
    for arm in arms:
        per = {}
        for _ in range(a.profile_steps):
            prof = []
            step(arm, profile=prof)
            torch.cuda.synchronize()
            for stage, e0, e1 in prof:
                per.setdefault(stage, []).append(e0.elapsed_time(e1))
        stages[arm] = {s: round(statistics.median(v), 4) for s, v in per.items()}

    line = {
        "bench": "rasterize_pose_gradient", "gaussians": a.n, "sh_degree": 3, "image_hw": [cam.height, cam.width],
        "views_batch": a.views, "distortion_k": list(K_TYPICAL), "loss": "<G, image>",
        "ms_fwd_bwd": {arm: round(v, 4) for arm, v in ms.items()},
        "ms_spread_min_max": {arm: [round(min(v), 4), round(max(v), 4)] for arm, v in times.items()},
        "ms_preprocess_bwd_median": {arm: st.get("preprocess_bwd") for arm, st in stages.items()},
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
