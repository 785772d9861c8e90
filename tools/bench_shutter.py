"""Cost of rolling-shutter cameras: forward + backward on the bench scene (synth-v1, 3 M gaussians, SH degree 3, 1080p,
bench.py's intrinsics K and pose) for each lens (the pinhole, a typical OPENCV_FISHEYE and OPENCV calibration), with a
global shutter and with a rolling shutter (a twist of about 5 % of the image over the readout, top to bottom), each with
no camera gradient and with the pose and the twist requiring grad.  Loss <G, image>.

Timing: CUDA events around `--iters` forward+backward steps, the arms alternated in `--rounds` rounds in one process
after `--warmup` steps of each; the median round is reported, with min / max.  Per-stage times (the rasterizer's own
CUDA-event profile: "preprocess_fwd" and "preprocess_bwd" are the per-gaussian stages) are the median over
`--profile-steps` separate profiled steps of each arm.  Then bench.py runs in a subprocess on the same card (its JSON
line is included).  Prints one JSON line with the card's name and power limit (read in the same process) and writes it
to --out."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_loss import gpu_info  # noqa: E402

FISHEYE_K = (0.08, -0.03, 0.01, -0.002)
OPENCV_K = (-0.12, 0.03, 5e-4, -3e-4, 0.0)
LENS_K = {"pinhole": None, "fisheye": FISHEYE_K, "distortion": OPENCV_K}
SHUTTERS = ("global", "rolling")
GRADS = ("none", "camera")  # no camera gradient; the pose (and with a rolling shutter the twist)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--bench-steps", type=int, default=20)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_shutter_h100.json"), help="write the JSON line here")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.rasterize import rasterize

    assert torch.cuda.is_available(), "bench_shutter.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam = synth.make_camera("1080p", device=dev)
    T = synth.make_pose(2, 8, device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    # about 5 % of the image over the readout: yaw and pitch of 0.05 rad-ish at bench.py's focal length, and a
    # translation
    fx = float(cam.K[0, 0])
    xi0 = torch.tensor([0.02, -0.01, 0.01, 0.05 * cam.height / fx, 0.05 * cam.width / fx, 0.01], device=dev)
    gen = torch.Generator().manual_seed(1)
    G = (torch.randn(cam.height, cam.width, 3, generator=gen) / (3.0 * cam.height * cam.width)).to(dev)
    params = [g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh]
    arms = {f"{lens}_{sh}_{grad}": (lens, sh, grad) for lens in LENS_K for sh in SHUTTERS for grad in GRADS}

    def step(arm, profile=None):
        lens, sh, grad = arms[arm]
        for p in params:
            p.grad = None
        Tp = T.detach().requires_grad_(grad != "none")
        xi = xi0.detach().requires_grad_(grad != "none") if sh == "rolling" else None
        kw = {} if lens == "pinhole" else {lens: LENS_K[lens]}
        out = rasterize(g, Tp, cam, 0.3, 500.0, 100.0, 3.0, True, bg, profile=profile, rolling_shutter=xi, **kw)
        (out[0] * G).sum().backward()
        assert (Tp.grad is not None) == (grad != "none")

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

    bench = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--gpus", "1", "--steps", str(a.bench_steps),
                            "--warmup", "5"], capture_output=True, text=True, cwd=str(ROOT))
    bench_line = None
    for ln in bench.stdout.splitlines():
        if ln.startswith("{"):
            bench_line = json.loads(ln)

    line = {
        "bench": "rasterize_rolling_shutter", "gaussians": a.n, "sh_degree": 3, "image_hw": [cam.height, cam.width],
        "fisheye_k": list(FISHEYE_K), "distortion_k": list(OPENCV_K), "twist": [round(float(v), 6) for v in xi0],
        "readout": "top_to_bottom", "loss": "<G, image>",
        "ms_fwd_bwd": {arm: round(v, 4) for arm, v in ms.items()},
        "ms_spread_min_max": {arm: [round(min(v), 4), round(max(v), 4)] for arm, v in times.items()},
        "ms_preprocess_fwd_median": {arm: st.get("preprocess_fwd") for arm, st in stages.items()},
        "ms_preprocess_bwd_median": {arm: st.get("preprocess_bwd") for arm, st in stages.items()},
        "ms_per_stage_median": stages,
        "bench_py": bench_line,
        "timing": f"CUDA events, {a.warmup} warm-up steps per arm, {a.rounds} alternating rounds of {a.iters} steps, "
                  f"median round; stages: median of {a.profile_steps} profiled steps; bench.py in a subprocess after",
        "device": torch.cuda.get_device_name(0),
        "power_limit_and_max_sm_clock": gpu_info(),
    }
    text = json.dumps(line)
    print(text)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
