"""Cost of the feature maps: rasterize() forward + backward at 1080p, 3 M gaussians, SH degree 3, for D feature
channels (D = 0: no features) with a loss <G, image> + |feature_map|^2 / (H W D).

Timing: CUDA events around `--iters` forward+backward steps, the arms (one per D) alternated in `--rounds` rounds in
one process after `--warmup` steps of each; the median round is reported, with min / max.  Per-stage times (the
rasterizer's own CUDA-event profile, features_fwd / features_bwd being the feature kernels) are the median over
`--profile-steps` separate profiled steps of each arm.  Also reports the feature kernels' chunk width and their
registers and CTAs per SM (cuobjdump on libgsr_features.so, when available).  Prints one JSON line with the card's
name and power limit."""
from __future__ import annotations

import argparse
import json
import re
import shutil
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_loss import gpu_info  # noqa: E402

CHUNK = 4  # channels per CTA of the feature kernels (FCH, csrc/gsr_features.cu)


def kernel_resources():
    """{kernel: {"registers", "shared_bytes", "ctas_per_sm"}} of libgsr_features.so (None without cuobjdump)."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    lib = ROOT / "gaussian_splatting_b200" / "libgsr_features.so"
    if not Path(exe).exists():
        return None
    out = subprocess.run([exe, "--dump-resource-usage", str(lib)], capture_output=True, text=True).stdout
    res = {}
    for name, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out):
        u = {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
        short = re.search(r"k_features_\w+?(?=E|I|N|$)", name).group(0) + ("<masks>" if "ILb1E" in name else
                                                                             "<no masks>" if "ILb0E" in name else "")
        regs, smem = u["REG"], u["SHARED"]
        # H100: 64 K registers (allocated per warp in units of 256), 228 KB shared memory (1 KB reserved per CTA),
        # 32 CTAs and 64 warps per SM; a CTA is 4 warps
        by_regs = 65536 // (4 * ((regs * 32 + 255) // 256 * 256))
        by_smem = (228 * 1024) // (smem + 1024)
        res[short] = {"registers": regs, "shared_bytes": smem, "ctas_per_sm": min(by_regs, by_smem, 16)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3_000_000)
    ap.add_argument("--dims", default="0,3,16,32")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.rasterize import rasterize
    from gaussian_splatting_b200.structs import Camera

    assert torch.cuda.is_available(), "bench_features.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam0 = synth.make_camera("1080p", device=dev)
    cam = Camera(1920, 1080, cam0.K)
    T = synth.make_pose(2, 8, device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    gen = torch.Generator().manual_seed(1)
    G = (torch.randn(1080, 1920, 3, generator=gen) / (3.0 * 1080 * 1920)).to(dev)
    dims = [int(d) for d in a.dims.split(",")]
    feats = {D: torch.randn(a.n, D, generator=gen).to(dev).requires_grad_(True) for D in dims if D > 0}
    params = [p for p in (g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh)] + list(feats.values())

    def step(D, profile=None):
        for p in params:
            p.grad = None
        out = rasterize(g, T, cam, 0.3, 500.0, 100.0, 3.0, True, bg, profile=profile, features=feats.get(D))
        loss = (out[0] * G).sum()
        if D:
            loss = loss + out[3].square().sum() / (1080 * 1920 * D)
        loss.backward()

    for D in dims:
        for _ in range(a.warmup):
            step(D)
    torch.cuda.synchronize()
    times = {D: [] for D in dims}
    for _ in range(a.rounds):
        for D in dims:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                step(D)
            e1.record()
            e1.synchronize()
            times[D].append(e0.elapsed_time(e1) / a.iters)
    ms = {D: statistics.median(v) for D, v in times.items()}

    stages = {}
    for D in dims:
        per = {}
        for _ in range(a.profile_steps):
            prof = []
            step(D, profile=prof)
            torch.cuda.synchronize()
            for stage, e0, e1 in prof:
                per.setdefault(stage, []).append(e0.elapsed_time(e1))
        stages[f"D={D}"] = {k: round(statistics.median(v), 4) for k, v in per.items()}

    base = ms.get(0)
    line = {
        "bench": "rasterize_features", "gaussians": a.n, "sh_degree": 3, "image_hw": [1080, 1920],
        "loss": "<G, image> + |feature_map|^2 / (H W D)",
        "ms_fwd_bwd": {f"D={D}": round(v, 4) for D, v in ms.items()},
        "ms_spread_min_max": {f"D={D}": [round(min(v), 4), round(max(v), 4)] for D, v in times.items()},
        "overhead_ms_vs_D0": {f"D={D}": round(v - base, 4) for D, v in ms.items() if D and base is not None},
        "ms_per_stage_median": stages,
        "channels_per_cta": CHUNK,
        "kernel_resources": kernel_resources(),
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
