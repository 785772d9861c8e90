"""Cost of Mip-Splatting's 3-D filter (DESIGN.md 3.13).

1. rasterize() forward + backward at 1080p, 3 M gaussians, SH degree 3, a loss on the image: default, with
   filter3d=f, and with filter3d=f plus antialiased=True.  f is compute_filter3d from the 8 ring poses of the bench
   scene.  CUDA events around `--iters` steps, the arms alternated in `--rounds` rounds after `--warmup` steps of each;
   the median round is reported with min / max.  Per-stage times (the rasterizer's CUDA-event profile) are the median
   over `--profile-steps` profiled steps of each arm.
2. compute_filter3d (one native launch) at 3 M gaussians x {100, 300} cameras against a torch restatement of
   Mip-Splatting's per-camera loop (min depth and max focal length, boolean-mask scatters), same cameras (one shared
   focal length, where the two definitions agree; the largest relative difference and the fraction of gaussians
   beyond 1e-5 are reported: the loop rounds differently, which matters for points on a frustum edge).

Prints one JSON line with the card's name, power limit and SM clocks, queried in the same run."""
from __future__ import annotations

import argparse
import json
import math
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), (s.strip() for s in out[0].split(",")))) if out else "unknown"
    except Exception as e:  # query only; the numbers stand without it
        return f"unknown ({e.__class__.__name__})"


def mip_splatting_loop(xyz, Ts, Ks, widths, heights, focal_x, near=0.2, margin=0.15, variance=0.2):
    import torch

    dist = torch.full((xyz.shape[0],), 100000.0, device=xyz.device)
    valid = torch.zeros(xyz.shape[0], dtype=torch.bool, device=xyz.device)
    focal = 0.0
    for T, K, W, H, fx in zip(Ts, Ks, widths, heights, focal_x):
        p = xyz @ T[:3, :3].T + T[:3, 3]
        z = p[:, 2]
        x = p[:, 0] / z * K[0, 0] + W / 2.0
        y = p[:, 1] / z * K[1, 1] + H / 2.0
        ok = (z > near) & (x >= -margin * W) & (x <= (1 + margin) * W) & (y >= -margin * H) & (y <= (1 + margin) * H)
        dist[ok] = torch.min(dist[ok], z[ok])
        valid = valid | ok
        focal = max(focal, fx)
    dist[~valid] = dist[valid].max()
    return dist / focal * math.sqrt(variance)


def timed(fn, warmup, reps):
    import torch

    for _ in range(warmup):
        fn()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


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
    from gaussian_splatting_b200.filter3d import compute_filter3d
    from gaussian_splatting_b200.rasterize import rasterize
    from gaussian_splatting_b200.structs import Camera

    assert torch.cuda.is_available(), "bench_filter3d.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    info_before = gpu_info()
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam0 = synth.make_camera("1080p", device=dev)
    cam = Camera(1920, 1080, cam0.K)
    T = synth.make_pose(2, 8, device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    gen = torch.Generator().manual_seed(1)
    G = (torch.randn(1080, 1920, 3, generator=gen) / (3.0 * 1080 * 1920)).to(dev)
    params = [g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh]
    ring = torch.stack([synth.make_pose(v, 8, device=dev) for v in range(8)])
    filt = compute_filter3d(g.xyz, ring, cam.K[None].expand(8, 3, 3).contiguous(), [1920] * 8, [1080] * 8)
    with torch.no_grad():
        coef = torch.sqrt(torch.prod(torch.exp(2 * g.scale) / (torch.exp(2 * g.scale) + filt[:, None] ** 2), 1))

    def step(kw, profile=None):
        for p in params:
            p.grad = None
        out = rasterize(g, T, cam, 0.3, 500.0, 100.0, 3.0, True, bg, profile=profile, return_state=True, **kw)
        out[0].backward(G)
        return out[-1].P

    arm_kw = {"default": {}, "filter3d": dict(filter3d=filt), "filter3d_antialiased": dict(filter3d=filt, antialiased=True)}
    pairs = {}
    for name, kw in arm_kw.items():
        for _ in range(a.warmup):
            pairs[name] = int(step(kw))
    torch.cuda.synchronize()
    times = {k: [] for k in arm_kw}
    for _ in range(a.rounds):
        for name, kw in arm_kw.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                step(kw)
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.iters)
    ms = {k: statistics.median(v) for k, v in times.items()}
    stages = {}
    for name, kw in arm_kw.items():
        per = {}
        for _ in range(a.profile_steps):
            prof = []
            step(kw, profile=prof)
            torch.cuda.synchronize()
            for stage, e0, e1 in prof:
                per.setdefault(stage, []).append(e0.elapsed_time(e1))
        stages[name] = {k: round(statistics.median(v), 4) for k, v in per.items()}

    # the sampling pass
    sampling = {}
    xyz = g.xyz.detach()
    for C in (100, 300):
        poses = torch.stack([synth.make_pose(v, C, device=dev) for v in range(C)])
        Ks = cam.K[None].expand(C, 3, 3).contiguous()
        Ws, Hs = [1920] * C, [1080] * C
        native_ms = timed(lambda: compute_filter3d(xyz, poses, Ks, Ws, Hs), 2, 7)
        fx = [float(cam.K[0, 0])] * C
        torch_ms = timed(lambda: mip_splatting_loop(xyz, poses, Ks, Ws, Hs, fx), 1, 3)
        a_, b_ = compute_filter3d(xyz, poses, Ks, Ws, Hs), mip_splatting_loop(xyz, poses, Ks, Ws, Hs, fx)
        sampling[str(C)] = dict(native_ms=round(statistics.median(native_ms), 4),
                                native_ms_min_max=[round(min(native_ms), 4), round(max(native_ms), 4)],
                                torch_loop_ms=round(statistics.median(torch_ms), 3),
                                max_rel_diff=float(((a_ - b_).abs() / b_.abs().clamp_min(1e-30)).max()),
                                **{"frac_rel_diff_above_1e-5": float((((a_ - b_).abs() / b_.abs().clamp_min(1e-30))
                                                                       > 1e-5).float().mean())})

    line = {
        "bench": "rasterize_filter3d", "gaussians": a.n, "sh_degree": 3, "image_hw": [1080, 1920],
        "ms_fwd_bwd": {k: round(v, 4) for k, v in ms.items()},
        "ms_spread_min_max": {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
        "pairs": pairs,
        "coef_quantiles_0.1_0.5_0.9": [round(float(q), 4) for q in torch.quantile(
            coef[torch.randperm(a.n, device=dev)[:1_000_000]], torch.tensor([0.1, 0.5, 0.9], device=dev))],
        "ms_per_stage_median": stages,
        "compute_filter3d_3M": sampling,
        "timing": f"CUDA events, {a.warmup} warm-up steps per arm, {a.rounds} alternating rounds of {a.iters} steps, "
                  f"median round; stages: median of {a.profile_steps} profiled steps; sampling: median of 7 (torch "
                  "loop: 3) calls",
        "device": torch.cuda.get_device_name(0),
        "gpu_before": info_before,
        "gpu_after": gpu_info(),
    }
    text = json.dumps(line)
    print(text)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
