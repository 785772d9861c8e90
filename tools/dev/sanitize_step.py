"""Workload for compute-sanitizer: four fwd+bwd steps of the fused path on a small scene — the first reads the pair
count eagerly, the others take the speculative path (padded pair buffers); contribution masks, in-kernel record
gather (cp.async on the stage barriers), tile-hit masks all on.

    compute-sanitizer --tool memcheck  python tools/dev/sanitize_step.py 30000 small
    compute-sanitizer --tool racecheck --racecheck-report analysis python tools/dev/sanitize_step.py 12000 small
"""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
from gaussian_splatting_b200 import rasterize as R  # noqa: E402
from gaussian_splatting_b200 import synth  # noqa: E402

dev = torch.device("cuda")
n, res = int(sys.argv[1]), sys.argv[2]
g = synth.make_gaussians(n, res, sh_degree=3, seed=0, device=dev, requires_grad=True, sigma_px=(2.5, 0.5, 0.5, 10.0))
cam = synth.make_camera(res, device=dev)
G = synth.make_upstream_grad(res, device=dev)
bg = torch.full((3,), 0.5, device=dev)
for i in range(4):
    for p in (g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh):
        p.grad = None
    T = synth.make_pose(i % 3, 3, device=dev)
    image, _, uv = R.rasterize(g, T, cam, 0.3, 500.0, 100, 3.0, True, bg)
    if i == 1:
        uv.retain_grad()
    image.backward(G)
torch.cuda.synchronize()
print("ok", float(image.mean()), float(g.xyz.grad.abs().sum()))
