"""Bilateral-grid appearance correction on the GPU: the native kernels (gaussian_splatting_b200.appearance) against
the fp32 torch formulation a user would otherwise write (oracle/bilagrid_oracle.py: F.grid_sample with border
padding and align_corners=True, then the affine; the TV regulariser as three diff / square / mean chains).

Measured, each in one process with CUDA events, warm-up calls of every arm, `--rounds` alternating rounds of
`--iters` calls and the median round:
  - slice at 1080p, C = 1 and C = 8 views, 16 x 16 x 8 grids (N = 300 of them, as for a capture of 300 images):
    forward + backward (gradients to the grids and the image) and forward alone; the native backward also with
    only the image gradient and only the grid gradient;
  - TV forward + backward at N = 1 and N = 300 grids;
  - the added cost per training step: rasterize + slice + photometric_loss + backward against the same step without
    the slice, on bench.py's scene (3 M Gaussians, SH 3, 1080p).
Algorithmic bytes: the forward reads rgb and writes out (24 B/pixel), the backward reads rgb and the upstream
gradient and writes the rgb gradient (36 B/pixel); both read the views' grids once.  Achieved rates are those bytes
over the measured time; the floor is the bytes over the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).
Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # query only; the number stands without it
        return f"unknown ({e.__class__.__name__})"


def timed(arms, warmup, iters, rounds):
    import torch

    for fn in arms.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / iters)
    return {k: round(statistics.median(v), 4) for k, v in times.items()}, \
        {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--grids", type=int, default=300)
    ap.add_argument("--n", type=int, default=3_000_000, help="Gaussians of the training-step arms")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import native, synth
    from gaussian_splatting_b200.appearance import bilateral_slice, identity_grids, total_variation
    from gaussian_splatting_b200.loss import photometric_loss
    from gaussian_splatting_b200.rasterize import rasterize
    from oracle import bilagrid_oracle as bo

    assert torch.cuda.is_available(), "bench_bilagrid.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    H, W, N = a.height, a.width, a.grids
    gen = torch.Generator(device=dev).manual_seed(0)
    grids = (identity_grids(N, device=dev) + 0.1 * torch.randn(N, 12, 8, 16, 16, device=dev, generator=gen))
    grids.requires_grad_()
    res = {}

    # ---- slice ----------------------------------------------------------------------------------------------------
    for C in (1, 8):
        image = torch.rand(C, H, W, 3, device=dev, generator=gen).requires_grad_()
        g_out = torch.randn(C, H, W, 3, device=dev, generator=gen)
        ids = [(37 * c + 11) % N for c in range(C)]
        ids_dev = torch.tensor(ids, device=dev)
        ids_i32 = ids_dev.int()

        def nat_fb():
            return torch.autograd.grad(bilateral_slice(grids, image, ids), (grids, image), g_out)

        def ref_fb():
            return torch.autograd.grad(bo.grid_sample_slice(grids, image, ids_dev), (grids, image), g_out)

        def nat_f():
            with torch.no_grad():
                return bilateral_slice(grids, image, ids)

        def ref_f():
            with torch.no_grad():
                return bo.grid_sample_slice(grids, image, ids_dev)

        def nat_b_rgb():
            return native().bilagrid_slice_backward(image.detach(), grids.detach(), ids_i32, g_out, True, False)

        def nat_b_grids():
            return native().bilagrid_slice_backward(image.detach(), grids.detach(), ids_i32, g_out, False, True)

        arms = {"native_fwd_bwd": nat_fb, "torch_fwd_bwd": ref_fb, "native_fwd": nat_f, "torch_fwd": ref_f,
                "native_bwd_rgb_only": nat_b_rgb, "native_bwd_grids_only": nat_b_grids}
        ms, spread = timed(arms, a.warmup, a.iters, a.rounds)
        o_n, o_t = nat_f(), ref_f()
        (gg_n, gr_n), (gg_t, gr_t) = nat_fb(), ref_fb()
        px = C * H * W
        grid_bytes = C * 12 * 8 * 16 * 16 * 4
        fwd_bytes, bwd_bytes = 24 * px + grid_bytes, 36 * px + grid_bytes
        res[f"slice_C{C}"] = {
            "ms": ms, "ms_spread_min_max": spread,
            "speedup_fwd_bwd": round(ms["torch_fwd_bwd"] / ms["native_fwd_bwd"], 2),
            "speedup_fwd": round(ms["torch_fwd"] / ms["native_fwd"], 2),
            "algorithmic_bytes": {"forward": fwd_bytes, "backward": bwd_bytes},
            "hbm_floor_us": {"forward": round(fwd_bytes / HBM_BYTES_PER_S * 1e6, 1),
                             "backward": round(bwd_bytes / HBM_BYTES_PER_S * 1e6, 1)},
            "native_fwd_GBps": round(fwd_bytes / (ms["native_fwd"] * 1e-3) / 1e9, 1),
            "native_fwd_share_of_floor": round(fwd_bytes / HBM_BYTES_PER_S / (ms["native_fwd"] * 1e-3), 3),
            "native_fwd_bwd_GBps": round((fwd_bytes + bwd_bytes) / (ms["native_fwd_bwd"] * 1e-3) / 1e9, 1),
            "native_fwd_bwd_share_of_floor": round((fwd_bytes + bwd_bytes) / HBM_BYTES_PER_S
                                                   / (ms["native_fwd_bwd"] * 1e-3), 3),
            "max_abs_diff_vs_torch": {"out": float((o_n - o_t).abs().max()),
                                      "grad_rgb": float((gr_n - gr_t).abs().max()),
                                      "grad_grids_over_max": float((gg_n - gg_t).abs().max() / gg_t.abs().max())},
        }
        del image, g_out

    # ---- total variation ------------------------------------------------------------------------------------------
    for n in (1, N):
        gv = grids[:n].detach().clone().requires_grad_()
        arms = {"native_fwd_bwd": lambda: torch.autograd.grad(total_variation(gv), gv),
                "torch_fwd_bwd": lambda: torch.autograd.grad(bo.total_variation(gv), gv)}
        ms, spread = timed(arms, a.warmup, a.iters, a.rounds)
        tv_n, tv_t = float(total_variation(gv)), float(bo.total_variation(gv.double()))
        res[f"tv_N{n}"] = {"ms": ms, "ms_spread_min_max": spread,
                           "speedup": round(ms["torch_fwd_bwd"] / ms["native_fwd_bwd"], 2),
                           "rel_diff_vs_fp64": abs(tv_n - tv_t) / abs(tv_t)}

    # ---- training step ------------------------------------------------------------------------------------------
    g = synth.make_gaussians(a.n, "1080p", sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam = synth.make_camera("1080p", device=dev)
    T = synth.make_pose(2, 8, device=dev)
    bg = torch.full((3,), 0.5, device=dev)
    gt = torch.rand(cam.height, cam.width, 3, device=dev, generator=gen)
    params = [g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh]
    idx7 = torch.tensor([7], device=dev)

    def step(kind):
        def fn():
            for p in params:
                p.grad = None
            grids.grad = None
            image = rasterize(g, T, cam, 0.3, 500.0, 100.0, 3.0, True, bg)[0]
            if kind == "native":
                image = bilateral_slice(grids, image, 7)
            elif kind == "torch":
                image = bo.grid_sample_slice(grids, image[None], idx7)[0]
            photometric_loss(image, gt, 0.2).backward()
        return fn

    ms, spread = timed({k: step(k) for k in ("no_slice", "native", "torch")}, 3, 5, a.rounds)
    res["training_step"] = {"ms": ms, "ms_spread_min_max": spread,
                            "added_ms_native": round(ms["native"] - ms["no_slice"], 4),
                            "added_ms_torch": round(ms["torch"] - ms["no_slice"], 4),
                            "added_share_native": round(ms["native"] / ms["no_slice"] - 1, 4)}

    line = {
        "bench": "bilagrid", "shape_hw": [H, W], "grid": [N, 12, 8, 16, 16], "dtype": "float32", **res,
        "step_scene": f"synth {a.n} Gaussians, SH 3, 1080p, pose 2 of 8; photometric_loss ssim_frac 0.2",
        "timing": f"CUDA events, {a.warmup} warm-up calls per arm, {a.rounds} alternating rounds of {a.iters} calls "
                  "(training step: 3 warm-up, 5 calls), median round",
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
