"""BASELINE.json configs[4]: the reference's training loop (splat_py/trainer.py:348-460, `colmap_splat.py 7k`
schedule) with everything the rasterizer hands over kept on this library's fast path, on 1..8 GPUs of one node:

    rank r, step i : view = r-th of `world` views drawn (same draw on every rank) -> fused rasterize -> the reference's
                     loss ((1 - ssim_frac) * L1 + ssim_frac * (1 - SSIM)) -> backward (all parameter gradients of the
                     view land in ONE flat buffer)
    all            : ONE NCCL all-reduce (average) of that buffer  [world > 1]
    all            : gsr_adam_step on the flat parameter buffer (torch.optim.Adam's values, reference LR groups)
    all            : gsr_densify_accumulate (per-view statistics); on the reference's schedule the statistics are
                     summed over ranks and `adaptive_density_control` runs identically on every rank: the plan on
                     per-row scalars with the reference's torch expressions, clone / split / delete applied to the
                     flat parameter + Adam buffers by ONE native pass (gsr_densify_apply); reset_opacity, add_sh_band.

Iteration convention (SURVEY.md §8(e)): the reference takes ONE view per optimizer step.  Here an optimizer step
averages the gradients of `world` views; `--iters` counts optimizer steps and every schedule constant of the
reference (densification interval, opacity reset, SH bands, background) is kept in optimizer steps, the learning
rates are the reference's.  So `world` GPUs see `world` x the views of the reference in the same number of steps.

Launch:  python tools/e2e/train_view_parallel.py --scene DIR                                       (1 GPU)
         python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
             --master-port P tools/e2e/train_view_parallel.py --scene DIR                            (8 GPUs)
Prints one JSON line (rank 0): wall-clock of train(), steps/s, views/s, final test PSNR / SSIM (same evaluation as
the reference: every 8th image, black background, clipped), gaussian counts, replica consistency.
The COLMAP loader, the initialisation and the SSIM stand-in are the ones tools/e2e/run_trainer.py uses for the
reference arm (oracle/_ref's splat_py.dataloader, tools/e2e/shims) so both arms start from the same state."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent / "shims"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", default="gpurun_out/e2e_scene")
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=7000)
    ap.add_argument("--max-gaussians", type=int, default=4250000)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--test-eval-interval", type=int, default=500)
    ap.add_argument("--optimizer", choices=["flat", "sharded"], default="flat",
                    help="flat: one NCCL all-reduce(avg) of the flat gradient bucket + gsr_adam_step on the replicated "
                         "flat buffer; sharded: ONE kernel per rank doing reduce-scatter + Adam + all-gather over NVLink "
                         "peer memory (gsr_adam_step_sharded), Adam state sharded over the ranks (needs >= 2 ranks)")
    ap.add_argument("--loss", choices=["shim", "fused"], default="shim",
                    help="shim: L1 + the SSIM stand-in through permuted NCHW views, like run_trainer.py's reference arm; "
                         "fused: gaussian_splatting_b200.loss.photometric_loss in the step and its ssim() in evaluate() "
                         "(one forward and one backward kernel)")
    a = ap.parse_args()

    real_stdout = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)
    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    import gaussian_splatting_b200 as gsb
    from gaussian_splatting_b200.densify import AdaptiveDensityControl, DensificationStats
    from gaussian_splatting_b200.flat_adam import REFERENCE_LR_MULTIPLIERS as mult, FlatAdam
    from gaussian_splatting_b200.loss import photometric_loss, ssim as fused_ssim
    from gaussian_splatting_b200.rasterize import rasterize
    from gaussian_splatting_b200.structs import Camera
    from gaussian_splatting_b200.view_parallel import GradientBucket, all_reduce_statistics
    from oracle import ref_loader

    gsb.install_as_splat_cuda()                 # the reference's loader imports splat_py.* which imports splat_cuda
    sys.path.insert(0, str(ref_loader.REF_DIR))
    from splat_py.config import SplatConfig
    from splat_py.dataloader import ColmapData
    from torchmetrics.image import StructuralSimilarityIndexMeasure  # tools/e2e/shims

    scale = a.iters / 7000.0  # the "7k" schedule, shortened proportionally when --iters < 7000 (as run_trainer.py)
    sched = {}
    if a.iters != 7000:
        base = SplatConfig()
        for key in ("adaptive_control_start", "adaptive_control_end", "use_background_end", "reset_opacity_start",
                    "reset_opacity_end", "reset_opacity_interval", "add_sh_band_interval"):
            sched[key] = max(1, int(getattr(base, key) * scale))
    out = a.out or f"gpurun_out/e2e_vp{world}"
    config = SplatConfig(dataset_path=a.scene, downsample_factor=1, output_dir=out, num_iters=a.iters,
                         max_gaussians=a.max_gaussians, test_eval_interval=a.test_eval_interval, **sched)

    torch.manual_seed(a.seed)                   # every rank: same initial state and the same random streams
    data = ColmapData(config.dataset_path, dev, downsample_factor=1, config=config)
    g = data.create_gaussians()                 # xyz, rgb, opacity, scale, quaternion; sh = None (added by bands)
    images, cameras = data.get_images(), data.get_cameras()
    for im in images:                           # trainer.py:44-49
        im.image = im.image.to(torch.float32) / config.saturated_pixel_value
    cams = {cid: Camera(c.width, c.height, c.K) for cid, c in cameras.items()}
    n0 = g.xyz.shape[0]
    for name in ("xyz", "quaternion", "scale", "opacity", "rgb"):
        getattr(g, name).requires_grad_(True)
    sharded = a.optimizer == "sharded"
    grads_sym = None
    if sharded:
        assert world > 1, "--optimizer sharded needs torchrun with at least 2 ranks"
        import types

        import torch.distributed._symmetric_memory as symm_mem

        from gaussian_splatting_b200.flat_adam import ShardedFlatAdam, flatten_gaussians, section_ends

        def alloc_sym(n):
            return symm_mem.empty(int(n), dtype=torch.float32, device=dev)

        params_sym = alloc_sym(section_ends(n0, 0)[-1])
        flat, ends, names = flatten_gaussians(g, flat=params_sym)
        grads_sym = alloc_sym(flat.numel())
        grads_sym.zero_()
        opt = ShardedFlatAdam(params_sym, grads_sym, ends, [config.base_lr * mult[f] for f in names])
    else:
        opt = FlatAdam.for_gaussians(g, base_lr=config.base_lr, multipliers=mult)
    stats = DensificationStats(n0, dev)
    adc = AdaptiveDensityControl(g, opt, stats, config, alloc_flat=alloc_sym if sharded else None)

    def relayout(fn):
        """Run a step that may re-lay-out the parameter buffer (densification, opacity reset, a new SH band).  With
        the sharded optimizer the Adam state is first gathered to full size, the step runs on a full-state stand-in
        of the optimizer, and the state is sharded again — over new symmetric buffers if the layout changed."""
        nonlocal opt, grads_sym
        if not sharded:
            return fn()
        m_full, v_full = opt.full_state()
        shim = types.SimpleNamespace(p=opt.p, m=m_full, v=v_full, ends=list(opt.ends), lrs=list(opt.lrs))
        adc.optimizer = shim
        out = fn()
        if shim.p is not opt.p:
            grads_sym = alloc_sym(shim.p.numel())
            grads_sym.zero_()
            t = opt.t
            opt = ShardedFlatAdam(shim.p, grads_sym, shim.ends, shim.lrs)
            opt.load_full_state(shim.m, shim.v, t)
        else:
            opt.load_full_state(shim.m, shim.v, opt.t)
        adc.optimizer = opt
        return out
    ssim = StructuralSimilarityIndexMeasure(data_range=1.0).to(dev)

    # trainer.py:32-43: every `test_split_ratio`-th image is a test image, uniform sampling over the rest
    import numpy as np

    n_img = len(images)
    test_split = np.arange(0, n_img, config.test_split_ratio)
    train_split = torch.tensor(sorted(set(range(n_img)) - set(test_split.tolist())), dtype=torch.int, device=dev)
    train_prob = torch.ones(len(train_split), dtype=torch.float32, device=dev) / len(train_split)

    def evaluate():
        psnrs, ssims = [], []
        with torch.no_grad():
            for t in test_split:
                im = images[int(t)]
                pred, _, _ = rasterize(g, im.camera_T_world, cams[im.camera_id], config.near_thresh, config.far_thresh,
                                       config.cull_mask_padding, config.mh_dist, config.use_sh_precompute,
                                       torch.zeros(3, device=dev))
                l2 = torch.nn.functional.mse_loss(pred.clip(0, 1), im.image)
                psnrs.append(-10 * torch.log10(l2).item())
                if a.loss == "fused":
                    ssims.append(fused_ssim(pred.clip(0, 1), im.image).item())
                else:
                    ssims.append(ssim(pred.unsqueeze(0).permute(0, 3, 1, 2).clip(0, 1),
                                      im.image.unsqueeze(0).permute(0, 3, 1, 2)).item())
        return float(np.mean(psnrs)), float(np.mean(ssims))

    fields = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")
    curve, adc_log = [], []
    phase_ms = dict(rasterize_fwd=[], loss_and_backward=[], stats_reduce_adam=[])  # CUDA events, every 50th step
    t_adc = 0.0
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    t0 = time.time()
    for i in range(config.num_iters):
        for f in fields:
            p = getattr(g, f, None)
            if p is not None:
                p.grad = None
        if i % config.test_eval_interval == 0:
            curve.append(round(evaluate()[0], 2))
        # `world` distinct training views per step, the same draw on every rank (same generator state)
        draw = torch.multinomial(train_prob, num_samples=min(world, len(train_split)), replacement=False)
        image_idx = int(train_split[draw[rank % len(draw)]].item())
        im = images[image_idx]
        background = torch.zeros(3, device=dev)
        if config.use_background and i < config.use_background_end:
            background = torch.ones(3, device=dev) * float(i % 255) / 255.0
        timed = (i % 50 == 25)
        if timed:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
        image, mask, uv, state = rasterize(g, im.camera_T_world, cams[im.camera_id], config.near_thresh,
                                           config.far_thresh, config.cull_mask_padding, config.mh_dist,
                                           config.use_sh_precompute, background, return_state=True,
                                           grad_out=grads_sym)
        uv.retain_grad()
        if timed:
            ev[1].record()
        if a.loss == "fused":
            loss = photometric_loss(image, im.image, config.ssim_frac)
        else:
            l1 = torch.nn.functional.l1_loss(image, im.image)
            ssim_loss = 1.0 - ssim(image.unsqueeze(0).permute(0, 3, 1, 2), im.image.unsqueeze(0).permute(0, 3, 1, 2))
            loss = (1.0 - config.ssim_frac) * l1 + config.ssim_frac * ssim_loss
        loss.backward()
        if timed:
            ev[2].record()
        # per-view statistics BEFORE the collective: they are this rank's own view (trainer.py:376-385); the xyz
        # gradient they use is this view's, so they are taken from the still un-averaged buffer
        stats.accumulate(state, uv, g.xyz, cams[im.camera_id].K)
        if sharded:
            opt.step()  # barrier, reduce-scatter + Adam + all-gather in one kernel over peer memory, barrier
        else:
            bucket = GradientBucket.adopt(state.grad_flat, g)
            bucket.all_reduce(average=True)
            opt.step(bucket)
        if timed:
            ev[3].record()
            torch.cuda.synchronize()
            for k, (a0, a1) in zip(phase_ms, ((0, 1), (1, 2), (2, 3))):
                phase_ms[k].append(ev[a0].elapsed_time(ev[a1]))
        if config.adaptive_control_start < i < config.adaptive_control_end and i % config.adaptive_control_interval == 0:
            t_a = time.time()
            all_reduce_statistics([stats.uv_grad_accum, stats.xyz_grad_accum, stats.grad_accum_count])
            info = relayout(lambda: adc.adaptive_density_control(i))
            torch.cuda.synchronize()
            t_adc += time.time() - t_a
            adc_log.append(dict(iter=i, **{k: info.get(k) for k in ("deleted", "cloned", "split", "n_out")}))
        if config.reset_opacity_start < i < config.reset_opacity_end and i % config.reset_opacity_interval == 0:
            relayout(adc.reset_opacity)
        if i > 0 and i % config.add_sh_band_interval == 0:
            relayout(lambda: adc.add_sh_band(config.base_lr, config.sh_lr_multiplier))
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    seconds = time.time() - t0

    psnr, ssim_v = evaluate()
    consistent = True
    if world > 1:  # replicas must be bit-identical: compare a checksum of the flat parameter buffer
        chk = opt.p.double().sum().reshape(1)
        lo, hi = chk.clone(), chk.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        consistent = bool((lo == hi).item())
    if rank == 0:
        line = {
            "impl": f"b200-view-parallel x{world}", "iters": a.iters, "views_per_step": world, "seed": a.seed,
            "train_seconds": round(seconds, 2), "iters_per_second": round(a.iters / seconds, 2),
            "views_per_second": round(a.iters * world / seconds, 2),
            "final_test_psnr": round(psnr, 3), "final_test_ssim": round(ssim_v, 4),
            "max_test_psnr": round(max(curve + [psnr]), 3), "test_psnr_curve": curve,
            "gaussians_start": n0, "gaussians_end": int(g.xyz.shape[0]), "views": n_img,
            "image": [int(images[0].image.shape[1]), int(images[0].image.shape[0])],
            "replicas_consistent": consistent, "adc_passes": len(adc_log), "adc_last": adc_log[-3:],
            "adc_seconds_total": round(t_adc, 2),
            "phase_ms_mean_gpu": {k: round(sum(v) / max(len(v), 1), 3) for k, v in phase_ms.items()},
            "phase_ms_last_quarter": {k: round(sum(v[-len(v) // 4:]) / max(len(v[-len(v) // 4:]), 1), 3)
                                      for k, v in phase_ms.items()},
            "optimizer": ("ShardedFlatAdam: gsr_adam_step_sharded (reduce-scatter + Adam + all-gather over NVLink peer "
                          "memory in one kernel, Adam state sharded)") if sharded else
                         ("FlatAdam (gsr_adam_step) after one NCCL all-reduce(avg) of the flat gradient bucket"
                          if world > 1 else "FlatAdam (gsr_adam_step)"),
            "loss": ("fused: photometric_loss (gsr_photometric_loss_forward / _backward), ssim() in evaluation"
                     if a.loss == "fused" else "shim: l1_loss + SSIM stand-in (tools/e2e/shims) through NCHW views"),
            "device": torch.cuda.get_device_name(local),
        }
        real_stdout.write("E2E " + json.dumps(line) + "\n")
        real_stdout.flush()
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "result.json"), "w") as f:
            json.dump(line, f, indent=1)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
