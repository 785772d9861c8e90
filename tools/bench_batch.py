"""rasterize_batch against a loop of rasterize calls, forward + backward, on one GPU.

    python tools/bench_batch.py [--rounds 15] [--views 1,2,4,8] [--out profiles/bench_batch_h100.json]

Two scenes: the bench scene (3 M Gaussians, SH 3, 1080p, the ring of 8 poses of bench.py) and a smaller one (500 k
Gaussians, SH 3, 720p) where fixed per-call costs weigh more.  For every C the two arms alternate in rounds in one
process and the median round is reported, per view:
  batch: one rasterize_batch(C poses) forward + backward;
  loop:  C rasterize(pose c) forward + backward calls into the same parameters, autograd accumulating the gradient.
Per-stage times come from one extra profiled call of each arm, peak memory from its own call.  The same run checks
that the timed outputs agree: images bit for bit per view, gradients within the render backward's atomics noise."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from gaussian_splatting_b200 import synth  # noqa: E402
from gaussian_splatting_b200.rasterize import rasterize, rasterize_batch  # noqa: E402
from gaussian_splatting_b200.structs import Camera  # noqa: E402

ARGS = (0.3, 500.0, 100, 3.0, True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def params(g):
    return [t for t in (g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh) if t is not None]


def zero(g):
    for t in params(g):
        t.grad = None


def arm_batch(g, T, cam, bg, G, profile=None):
    imgs = rasterize_batch(g, T, cam, *ARGS, bg, profile=profile)[0]
    (imgs * G).sum().backward()
    return imgs


def arm_loop(g, T, cam, bg, G, profile=None):
    imgs = []
    for c in range(T.shape[0]):
        img = rasterize(g, T[c], cam, *ARGS, bg, profile=profile)[0]
        (img * G[c]).sum().backward()
        imgs.append(img)
    return torch.stack(imgs)


def timed(fn, *a):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn(*a)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), out


def stages(fn, *a):
    prof = []
    fn(*a, profile=prof)
    torch.cuda.synchronize()
    tot = {}
    for name, s, e in prof:
        tot[name] = tot.get(name, 0.0) + s.elapsed_time(e)
    return {k: round(v, 3) for k, v in tot.items()}


def peak(fn, *a):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn(*a)
    torch.cuda.synchronize()
    return round(torch.cuda.max_memory_allocated() / 2**20, 1)


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def grads(g):
    return [t.grad.clone() for t in params(g)]


def run_scene(name, n, res, views, rounds, dev):
    g = synth.make_gaussians(n, res, sh_degree=3, seed=0, device=dev, requires_grad=True)
    cam = synth.make_camera(res, device=dev)
    T_all = torch.stack([synth.make_pose(v, 8, device=dev) for v in range(8)])
    bg = torch.zeros(3, device=dev)
    H, W = cam.height, cam.width
    out = []
    for C in views:
        T = T_all[:C].contiguous()
        G = (torch.randn(C, H, W, 3, generator=torch.Generator().manual_seed(C)) / (3.0 * H * W)).to(dev)
        a = (g, T, cam, bg, G)
        for _ in range(3):  # warm-up (and the speculative pair sizing's history) for both arms
            zero(g); arm_batch(*a)
            zero(g); arm_loop(*a)
        tb, tl = [], []
        for _ in range(rounds):
            zero(g); t, img_b = timed(arm_batch, *a); tb.append(t); g_b = grads(g)
            zero(g); t, img_l = timed(arm_loop, *a); tl.append(t); g_l = grads(g)
        # noise bound: two runs of the loop arm
        zero(g); arm_loop(*a); g_l2 = grads(g)
        same_images = all(torch.equal(img_b[c].view(torch.int32), img_l[c].view(torch.int32)) for c in range(C))
        grad_rel = max(rel(x, y) for x, y in zip(g_b, g_l))
        noise = max(rel(x, y) for x, y in zip(g_l2, g_l))
        zero(g); st_b = stages(arm_batch, *a)
        zero(g); st_l = stages(arm_loop, *a)
        zero(g); pk_b = peak(arm_batch, *a)
        zero(g); pk_l = peak(arm_loop, *a)
        mb, ml = statistics.median(tb), statistics.median(tl)
        row = dict(scene=name, N=n, H=H, W=W, C=C, rounds=rounds,
                   batch_ms_per_view=round(mb / C, 3), loop_ms_per_view=round(ml / C, 3),
                   batch_over_loop=round(mb / ml, 4), batch_ms=round(mb, 3), loop_ms=round(ml, 3),
                   stages_batch_ms=st_b, stages_loop_ms=st_l, peak_mib_batch=pk_b, peak_mib_loop=pk_l,
                   images_bit_identical=bool(same_images), grad_max_rel_vs_loop=grad_rel,
                   grad_max_rel_loop_vs_loop=noise)
        print(json.dumps(row), flush=True)
        out.append(row)
        assert same_images, f"{name} C={C}: images differ between the arms"
        assert grad_rel <= max(1e-5, 10 * noise), f"{name} C={C}: gradients differ by {grad_rel} (noise {noise})"
    del g
    torch.cuda.empty_cache()
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--views", default="1,2,4,8")
    ap.add_argument("--out", default=None)
    ap.add_argument("--scenes", default="bench,small")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_batch.py needs a CUDA device")
    dev = torch.device("cuda:0")
    views = [int(v) for v in a.views.split(",")]
    defs = {"bench": (3_000_000, "1080p"), "small": (500_000, "720p")}
    result = dict(card=card(), torch=torch.__version__, rows=[])
    print(json.dumps(dict(card=result["card"])), flush=True)
    for s in a.scenes.split(","):
        result["rows"] += run_scene(s, *defs[s], views, a.rounds, dev)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(result, indent=1) + "\n")


if __name__ == "__main__":
    main()
