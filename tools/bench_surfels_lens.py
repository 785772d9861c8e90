"""Cost of 2-D Gaussian surfels through a lens: forward + backward of rasterize_surfels with all five maps in the loss,
for the pinhole, a fisheye (fisheye=FISHEYE) and an OPENCV camera (distortion=OPENCV), on the bench scene (synth-v1,
3 M gaussians, SH degree 3, 1080p, bench.py's intrinsics and pose).

Timing: CUDA events around `--iters` forward+backward steps, the three arms alternated in `--rounds` rounds in one
process after `--warmup` steps of each; the median round is reported, with min / max.  Also reported: the ray-map
kernel alone (CUDA events over `--ray-iters` launches per lens) and the (gaussian, tile) pair count of each arm, where
a loose binning bound shows first.  Prints one JSON line with the card's name and power limit (read in the same
process) and writes it to --out."""
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
OPENCV = (-0.12, 0.03, 5e-4, -3e-4, 0.01)    # a typical OPENCV calibration


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3_000_000)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ray-iters", type=int, default=50)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_surfels_lens_h100.json"),
                    help="write the JSON line here")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import native, synth
    from gaussian_splatting_b200.surfels import _surfel_lens, rasterize_surfels

    assert torch.cuda.is_available(), "bench_surfels_lens.py measures on a CUDA device"
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
    arms = {"pinhole": {}, "fisheye": dict(fisheye=FISHEYE), "opencv": dict(distortion=OPENCV)}
    pairs = {}

    def step(arm):
        for p in params:
            p.grad = None
        image, _, _, depth, alpha, normal, dist, st = rasterize_surfels(g, T, cam, 0.3, 500.0, 100.0, 3.0, bg,
                                                                        return_state=True, **arms[arm])
        loss = ((image * G["image"]).sum() + (depth * G["depth"]).sum() + (alpha * G["alpha"]).sum()
                + (normal * G["normal"]).sum() + (dist * G["dist"]).sum())
        loss.backward()
        pairs[arm] = int(st.P)

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

    ext, ray_ms = native(), {}
    K = cam.K.contiguous()
    for arm in ("fisheye", "opencv"):
        code, consts = _surfel_lens(arms[arm].get("fisheye"), arms[arm].get("distortion"), dev)
        for _ in range(3):
            ext.surfel_rays(code, consts, K, H, W)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.ray_iters):
            ext.surfel_rays(code, consts, K, H, W)
        e1.record()
        e1.synchronize()
        ray_ms[arm] = round(e0.elapsed_time(e1) / a.ray_iters, 4)

    line = {
        "bench": "rasterize_surfels through lenses", "gaussians": a.n, "sh_degree": 3, "image_hw": [H, W],
        "lenses": {"fisheye": FISHEYE, "opencv": OPENCV},
        "loss": "<G, image> + depth + alpha + normal + distortion terms",
        "ms_fwd_bwd": {arm: round(statistics.median(v), 4) for arm, v in times.items()},
        "ms_spread_min_max": {arm: [round(min(v), 4), round(max(v), 4)] for arm, v in times.items()},
        "ms_ray_map": ray_ms,
        "pairs": pairs,
        "timing": f"CUDA events, {a.warmup} warm-up steps per arm, {a.rounds} alternating rounds of {a.iters} steps, "
                  f"median round; ray map: {a.ray_iters} launches per lens",
        "device": torch.cuda.get_device_name(0),
        "power_limit_and_max_sm_clock": gpu_info(),
    }
    text = json.dumps(line)
    print(text)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
