"""Cost of 2-D Gaussian surfels: forward + backward of rasterize_surfels with all five maps in the loss, against
rasterize with the image only, on the bench scene (synth-v1, 3 M gaussians, SH degree 3, 1080p, bench.py's intrinsics
and pose).  Loss <G, image> (+ <G_d, depth> + <G_a, alpha> + <G_n, normal> + <G_x, distortion> for the surfels).

Timing: CUDA events around `--iters` forward+backward steps, the two arms alternated in `--rounds` rounds in one
process after `--warmup` steps of each; the median round is reported, with min / max.  Per-kernel times come from a
separate torch.profiler run of `--profile-steps` steps per arm (CUDA activity, summed per kernel name and divided by
the steps).  Prints one JSON line with the card's name and power limit (read in the same process) and writes it to
--out."""
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
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_surfels_h100.json"), help="write the JSON line here")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.rasterize import rasterize
    from gaussian_splatting_b200.surfels import rasterize_surfels

    assert torch.cuda.is_available(), "bench_surfels.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam = synth.make_camera("1080p", device=dev)
    T = synth.make_pose(2, 8, device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    gen = torch.Generator().manual_seed(1)
    H, W = cam.height, cam.width
    G = {k: (torch.randn(H, W, c, generator=gen) / (3.0 * H * W)).to(dev)
         for k, c in (("image", 3), ("depth", 1), ("alpha", 1), ("normal", 3), ("dist", 1))}
    params = [g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh]

    def step(arm):
        for p in params:
            p.grad = None
        if arm == "rasterize":
            out = rasterize(g, T, cam, 0.3, 500.0, 100.0, 3.0, True, bg)
            loss = (out[0] * G["image"]).sum()
        else:
            image, _, _, depth, alpha, normal, dist = rasterize_surfels(g, T, cam, 0.3, 500.0, 100.0, 3.0, bg)
            loss = ((image * G["image"]).sum() + (depth * G["depth"]).sum() + (alpha * G["alpha"]).sum()
                    + (normal * G["normal"]).sum() + (dist * G["dist"]).sum())
        loss.backward()

    arms = ("rasterize", "surfels")
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

    kernels = {}
    from torch.profiler import ProfilerActivity, profile

    for arm in arms:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_steps):
                step(arm)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            if t > 0:
                per[ev.key] = round(t / 1000.0 / a.profile_steps, 4)
        kernels[arm] = dict(sorted(per.items(), key=lambda kv: -kv[1])[:25])

    line = {
        "bench": "rasterize_surfels", "gaussians": a.n, "sh_degree": 3, "image_hw": [H, W],
        "loss": {"rasterize": "<G, image>", "surfels": "<G, image> + depth + alpha + normal + distortion terms"},
        "ms_fwd_bwd": {arm: round(statistics.median(v), 4) for arm, v in times.items()},
        "ms_spread_min_max": {arm: [round(min(v), 4), round(max(v), 4)] for arm, v in times.items()},
        "ms_per_kernel_top25": kernels,
        "timing": f"CUDA events, {a.warmup} warm-up steps per arm, {a.rounds} alternating rounds of {a.iters} steps, "
                  f"median round; kernels: torch.profiler over {a.profile_steps} steps per arm, in a separate run",
        "device": torch.cuda.get_device_name(0),
        "power_limit_and_max_sm_clock": gpu_info(),
    }
    text = json.dumps(line)
    print(text)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
