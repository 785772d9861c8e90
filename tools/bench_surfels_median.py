"""Cost of the median depth of 2-D Gaussian surfels: forward + backward of rasterize_surfels on the bench scene
(synth-v1, 3 M gaussians, SH degree 3, 1080p, bench.py's intrinsics and pose), three arms:

    pinhole          the five surfel maps in the loss, no median
    pinhole_median   the five maps plus the median depth in the loss
    fisheye_median   the same through a ScanNet++-like fisheye

Timing: CUDA events around `--iters` forward+backward steps, the arms alternated in `--rounds` rounds in one process
after `--warmup` steps of each; the median round is reported, with min / max.  Then, with the timing done, a few steps of
each arm run under torch.profiler (CUDA activity) for the per-kernel times of the surfel tile kernels and the median
kernels.  Prints one JSON line with the card's name and power limit (read in the same process) and writes it to
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

FISHEYE = (0.03, -0.01, 0.002, -0.0005)      # ScanNet++-like OPENCV_FISHEYE coefficients
ARMS = {"pinhole": (False, {}), "pinhole_median": (True, {}), "fisheye_median": (True, dict(fisheye=FISHEYE))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3_000_000)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_surfels_median_h100.json"),
                    help="write the JSON line here")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.surfels import rasterize_surfels

    assert torch.cuda.is_available(), "bench_surfels_median.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam = synth.make_camera("1080p", device=dev)
    T = synth.make_pose(2, 8, device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    gen = torch.Generator().manual_seed(1)
    H, W = cam.height, cam.width
    G = {k: (torch.randn(H, W, c, generator=gen) / (3.0 * H * W)).to(dev)
         for k, c in (("image", 3), ("depth", 1), ("alpha", 1), ("normal", 3), ("dist", 1), ("median", 1))}
    params = [g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh]
    pixels = {}

    def step(arm):
        median, kw = ARMS[arm]
        for p in params:
            p.grad = None
        out = rasterize_surfels(g, T, cam, 0.3, 500.0, 100.0, 3.0, bg, median_depth=median, **kw)
        image, _, _, depth, alpha, normal, dist = out[:7]
        loss = ((image * G["image"]).sum() + (depth * G["depth"]).sum() + (alpha * G["alpha"]).sum()
                + (normal * G["normal"]).sum() + (dist * G["dist"]).sum())
        if median:
            loss = loss + (out[7] * G["median"]).sum()
        loss.backward()
        if median and arm not in pixels:
            pixels[arm] = float((alpha > 0).float().mean())

    for arm in ARMS:
        for _ in range(a.warmup):
            step(arm)
    torch.cuda.synchronize()
    times = {arm: [] for arm in ARMS}
    for _ in range(a.rounds):
        for arm in ARMS:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                step(arm)
            e1.record()
            e1.synchronize()
            times[arm].append(e0.elapsed_time(e1) / a.iters)

    # per-kernel times, the timing above done: the surfel tile kernels' and the median kernels' mean CUDA time per step
    from torch.profiler import ProfilerActivity, profile

    kernels = {}
    for arm in ARMS:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_steps):
                step(arm)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            name = ev.key
            if "k_surfel_render" in name or "k_surfel_median" in name or "k_surfel_lens_render" in name:
                short = name.split("(")[0].split("::")[-1].split("<")[0]
                tag = "<true>" if "ILb1E" in name or "<true>" in name else ("<false>" if "ILb0E" in name or
                                                                             "<false>" in name else "")
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                per[short + tag] = round(per.get(short + tag, 0.0) + t / 1000.0 / a.profile_steps, 4)
        kernels[arm] = per

    line = {
        "bench": "rasterize_surfels with the median depth", "gaussians": a.n, "sh_degree": 3, "image_hw": [H, W],
        "arms": {arm: dict(median=m, lens="fisheye" if kw else "pinhole") for arm, (m, kw) in ARMS.items()},
        "fisheye": FISHEYE,
        "loss": "<G, image> + depth + alpha + normal + distortion terms (+ <G, median> in the median arms)",
        "covered_pixel_fraction": pixels,
        "ms_fwd_bwd": {arm: round(statistics.median(v), 4) for arm, v in times.items()},
        "ms_spread_min_max": {arm: [round(min(v), 4), round(max(v), 4)] for arm, v in times.items()},
        "ms_per_step_kernels": kernels,
        "timing": f"CUDA events, {a.warmup} warm-up steps per arm, {a.rounds} alternating rounds of {a.iters} steps, "
                  f"median round; kernels: torch.profiler over {a.profile_steps} steps per arm after the timing",
        "device": torch.cuda.get_device_name(0),
        "power_limit_and_max_sm_clock": gpu_info(),
    }
    text = json.dumps(line)
    print(text)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
