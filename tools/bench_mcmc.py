"""Cost of 3DGS-MCMC on the flat buffers at 3 M gaussians, SH degree 3 (gaussian_splatting_b200.mcmc).

CUDA events around `--iters` launches, `--rounds` rounds after `--warmup` launches, median round reported with min /
max, in one process:
  * per step: the position-noise kernel (gsr_mcmc_noise) and, in the same rounds, FlatAdam's step (gsr_adam_step)
    on the same buffer, with the bytes each must move and the rate that gives;
  * per refinement: relocation of the dead rows (plan_relocate + apply_mcmc_plan) and growth by 5 % (plan_grow +
    apply_mcmc_plan), wall clock to a device synchronise (the plans read counts back to the host), each on a fresh
    copy of the same state with a fifth of the rows dead.
Prints one JSON line with the card's name, power limit and clocks."""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_loss import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3_000_000)
    ap.add_argument("--sh-degree", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--refine-rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()

    import torch

    from gaussian_splatting_b200 import native, synth
    from gaussian_splatting_b200.flat_adam import FlatAdam
    from gaussian_splatting_b200.mcmc import MCMCConfig, MCMCDensityControl, apply_mcmc_plan, plan_grow, plan_relocate
    from gaussian_splatting_b200.structs import Gaussians

    assert torch.cuda.is_available(), "bench_mcmc measures on a CUDA device"
    dev = torch.device("cuda:0")
    n = a.n
    g = synth.make_gaussians(n, "1080p", sh_degree=a.sh_degree, seed=0, device=dev)
    with torch.no_grad():
        g.opacity[::5] = -8.0
    opt = FlatAdam.for_gaussians(g)
    n_rest = 0 if g.sh is None else int(g.sh.shape[2])
    mcmc = MCMCDensityControl(g, opt, MCMCConfig(cap_max=10 ** 9))
    grad = torch.randn_like(opt.p) * 1e-3
    xyz_lr = opt.lrs[0]

    def timed(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(a.iters):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / a.iters

    step = [0]

    def noise():
        step[0] += 1
        mcmc.inject_noise(step[0], xyz_lr, seed=1)

    arms = dict(noise=noise, adam=lambda: opt.step(grad))
    for fn in arms.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    per = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            per[k].append(timed(fn))

    def summary(v):
        return dict(median=round(statistics.median(v), 4), min=round(min(v), 4), max=round(max(v), 4))

    flat_bytes = opt.p.numel() * 4
    bytes_moved = dict(noise=n * (44 + 12), adam=flat_bytes * 7)  # adam: p, g, m, v read; p, m, v written

    # refinement on fresh copies of one state
    base = {f: getattr(g, f).detach().clone() for f in ("xyz", "rgb", "opacity", "scale", "quaternion", "sh")
            if getattr(g, f) is not None}
    cfg = MCMCConfig(cap_max=10 ** 9)
    refine = dict(relocate=[], grow=[])
    info = {}
    for r in range(a.refine_rounds + 1):
        gg = Gaussians(**{k: v.clone() for k, v in base.items()})
        o2 = FlatAdam.for_gaussians(gg)
        gen = torch.Generator(device=dev).manual_seed(r)
        for name, planner in (("relocate", plan_relocate), ("grow", plan_grow)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            plan = planner(gg, cfg, gen)
            apply_mcmc_plan(plan, gg, o2)
            torch.cuda.synchronize()
            if r > 0:  # the first round warms up
                refine[name].append((time.perf_counter() - t0) * 1e3)
            info[name] = dict(plan.info)
        del gg, o2
        torch.cuda.empty_cache()

    line = {
        "bench": "mcmc", "n": n, "sh_degree": a.sh_degree, "flat_floats": opt.p.numel(),
        "iters": a.iters, "rounds": a.rounds,
        "kernel_ms": {k: summary(v) for k, v in per.items()},
        "bytes_per_call": bytes_moved,
        "achieved_GBps_median": {k: round(bytes_moved[k] / (statistics.median(per[k]) * 1e-3) / 1e9, 1) for k in per},
        "refine_ms_wall": {k: summary(v) for k, v in refine.items()},
        "refine_info": info,
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
