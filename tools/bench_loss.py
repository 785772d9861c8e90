"""Photometric loss at 1080p: the fused kernels (gaussian_splatting_b200.loss.photometric_loss) against the SSIM
stand-in path exactly as the trainer runs it (tools/e2e/train_view_parallel.py: L1 on the [H,W,3] image, SSIM through
the permuted NCHW views, backward to the [H,W,3] image).  Both arms end in the rasterizer's `grad.contiguous()`
(an identity node stands in for the image node), so each pays for whatever gradient layout it hands back.

Timing: CUDA events around `--iters` forward+backward calls, arms alternated in `--rounds` rounds in one process
after `--warmup` calls of each; the median round is reported.  Also times the fused forward alone (the evaluation
path under no_grad).  Algorithmic bytes of the fused kernels: forward reads pred and target (2*H*W*C*4), backward
reads both and writes the gradient (3*H*W*C*4); achieved rates are those bytes over the measured time, shares are
against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools" / "e2e" / "shims"))

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # query only; the number stands without it
        return f"unknown ({e.__class__.__name__})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--ssim-frac", type=float, default=0.2)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()

    import torch
    from torchmetrics.image import StructuralSimilarityIndexMeasure  # tools/e2e/shims

    from gaussian_splatting_b200.loss import photometric_loss, ssim as fused_ssim

    assert torch.cuda.is_available(), "bench_loss.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    H, W, C = a.height, a.width, 3
    frac = a.ssim_frac
    gen = torch.Generator(device=dev).manual_seed(0)
    image = torch.rand(H, W, C, device=dev, generator=gen).requires_grad_(True)
    gt = (image.detach() + 0.1 * torch.randn(H, W, C, device=dev, generator=gen)).clamp(0, 1)
    shim = StructuralSimilarityIndexMeasure(data_range=1.0).to(dev)

    class ImageNode(torch.autograd.Function):  # the rasterizer's image node: its backward makes the gradient HWC
        @staticmethod
        def forward(ctx, x):
            return x.view_as(x)

        @staticmethod
        def backward(ctx, g):
            return g.contiguous()

    def shim_arm():
        img = ImageNode.apply(image)
        l1 = torch.nn.functional.l1_loss(img, gt)
        s = shim(img.unsqueeze(0).permute(0, 3, 1, 2), gt.unsqueeze(0).permute(0, 3, 1, 2))
        loss = (1.0 - frac) * l1 + frac * (1.0 - s)
        return loss, torch.autograd.grad(loss, image)[0]

    def fused_arm():
        loss = photometric_loss(ImageNode.apply(image), gt, frac)
        return loss, torch.autograd.grad(loss, image)[0]

    def fused_fwd():
        with torch.no_grad():
            return fused_ssim(image, gt)

    arms = dict(shim=shim_arm, fused=fused_arm, fused_forward_only=fused_fwd)
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

    loss_s, grad_s = shim_arm()
    loss_f, grad_f = fused_arm()
    torch.cuda.synchronize()
    elems = H * W * C
    fwd_bytes, bwd_bytes = 2 * elems * 4, 3 * elems * 4
    fused_s = ms["fused"] * 1e-3
    line = {
        "bench": "photometric_loss", "shape_hwc": [H, W, C], "dtype": "float32", "ssim_frac": frac,
        "ms_fwd_bwd": {"shim": round(ms["shim"], 4), "fused": round(ms["fused"], 4)},
        "ms_fused_forward_only": round(ms["fused_forward_only"], 4),
        "ms_spread_min_max": {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
        "speedup_fwd_bwd": round(ms["shim"] / ms["fused"], 2),
        "algorithmic_bytes": {"forward": fwd_bytes, "backward": bwd_bytes},
        "fused_fwd_bwd_GBps": round((fwd_bytes + bwd_bytes) / fused_s / 1e9, 1),
        "fused_fwd_bwd_share_of_3.35TBps": round((fwd_bytes + bwd_bytes) / fused_s / HBM_BYTES_PER_S, 3),
        "fused_forward_GBps": round(fwd_bytes / (ms["fused_forward_only"] * 1e-3) / 1e9, 1),
        "loss": {"shim": loss_s.item(), "fused": loss_f.item(), "abs_diff": abs(loss_s.item() - loss_f.item())},
        "grad_max_abs_diff": float((grad_s - grad_f).abs().max()),
        "grad_max_abs_diff_over_max_abs": float((grad_s - grad_f).abs().max() / grad_s.abs().max()),
        "timing": f"CUDA events, {a.warmup} warm-up calls per arm, {a.rounds} alternating rounds of {a.iters} calls, "
                  "median round",
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
