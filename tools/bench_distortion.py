"""Cost of radial-tangential lens distortion: rasterize() forward + backward on the bench scene (synth-v1, 3 M
gaussians, SH degree 3, 1080p, bench.py's intrinsics K) with three arms: the pinhole (distortion=None), all-zero
coefficients (the distortion kernels computing the pinhole) and a typical OPENCV calibration (K_TYPICAL below), all
with the same K and pose, and the loss <G, image>.

Barrel distortion pulls the periphery in, so more gaussians fit in the frame: the visible count M and the (gaussian,
tile) pair count P are reported per arm next to the times.  The tile stages are comparable between the pinhole and the
zero arm (same M and P), the per-gaussian stages across all three (same N).

Timing: CUDA events around `--iters` forward+backward steps, the arms alternated in `--rounds` rounds in one process
after `--warmup` steps of each; the median round is reported, with min / max.  Per-stage times (the rasterizer's own
CUDA-event profile) are the median over `--profile-steps` separate profiled steps of each arm.  Also reports the
per-gaussian kernels' registers and CTAs per SM (cuobjdump), pinhole and distortion.  Prints one JSON line with the
card's name and power limit."""
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

K_TYPICAL = (-0.12, 0.03, 5e-4, -3e-4, 0.0)


def kernel_resources():
    """SH-3 per-gaussian kernels (plain mode) of libgsr_b200.so and libgsr_distortion.so: registers, CTAs per SM."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(exe).exists():
        return None
    want = {"libgsr_b200.so": {"pinhole_fwd": r"16k_preprocess_fwdILi16ELb1E",
                               "pinhole_bwd": r"16k_preprocess_bwdILi16ELb1E"},
            "libgsr_distortion.so": {"distortion_fwd": r"k_distortion_preprocess_fwdILi16ELb1ELb0ELb0E",
                                     "distortion_bwd": r"k_distortion_preprocess_bwdILi16ELb1ELb0ELb0ELb0E"}}
    res = {}
    for lib, names in want.items():
        out = subprocess.run([exe, "--dump-resource-usage", str(ROOT / "gaussian_splatting_b200" / lib)],
                             capture_output=True, text=True).stdout
        for fn, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out):
            for short, pat in names.items():
                if re.search(pat, fn):
                    u = {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
                    regs, smem = u["REG"], u["SHARED"]
                    by_regs = 65536 // (4 * ((regs * 32 + 255) // 256 * 256))
                    by_smem = (228 * 1024) // (smem + 1024)
                    res[short] = {"registers": regs, "shared_bytes": smem, "local_bytes": u["LOCAL"],
                                  "ctas_per_sm": min(by_regs, by_smem, 16)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3_000_000)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.rasterize import distortion_r2_max, rasterize

    assert torch.cuda.is_available(), "bench_distortion.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam = synth.make_camera("1080p", device=dev)
    T = synth.make_pose(2, 8, device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    gen = torch.Generator().manual_seed(1)
    G = (torch.randn(cam.height, cam.width, 3, generator=gen) / (3.0 * cam.height * cam.width)).to(dev)
    arms = {"pinhole": None, "distortion_zero": (0.0, 0.0, 0.0, 0.0, 0.0), "distortion_typical": K_TYPICAL}
    params = [g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh]

    def step(k, profile=None, state=False):
        for p in params:
            p.grad = None
        out = rasterize(g, T, cam, 0.3, 500.0, 100.0, 3.0, True, bg, profile=profile, return_state=state, distortion=k)
        (out[0] * G).sum().backward()
        return out[-1] if state else None

    counts = {}
    for name, k in arms.items():
        for _ in range(a.warmup):
            step(k)
        st = step(k, state=True)
        counts[name] = {"M": int(st.M), "P": int(st.P)}
    torch.cuda.synchronize()
    times = {name: [] for name in arms}
    for _ in range(a.rounds):
        for name, k in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                step(k)
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.iters)
    ms = {name: statistics.median(v) for name, v in times.items()}

    stages = {}
    for name, k in arms.items():
        per = {}
        for _ in range(a.profile_steps):
            prof = []
            step(k, profile=prof)
            torch.cuda.synchronize()
            for stage, e0, e1 in prof:
                per.setdefault(stage, []).append(e0.elapsed_time(e1))
        stages[name] = {s: round(statistics.median(v), 4) for s, v in per.items()}

    line = {
        "bench": "rasterize_distortion", "gaussians": a.n, "sh_degree": 3, "image_hw": [cam.height, cam.width],
        "K": [round(float(v), 4) for v in cam.K.reshape(-1).tolist()], "loss": "<G, image>",
        "arms": {name: (None if k is None else {"k": list(k), "r2_max": str(distortion_r2_max(k))})
                 for name, k in arms.items()},
        "ms_fwd_bwd": {name: round(v, 4) for name, v in ms.items()},
        "ms_spread_min_max": {name: [round(min(v), 4), round(max(v), 4)] for name, v in times.items()},
        "visible_and_pairs": counts,
        "ms_per_stage_median": stages,
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
