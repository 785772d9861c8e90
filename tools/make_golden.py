"""Generate tests/golden/*.npz by running the UNMODIFIED reference (oracle/_ref: its CUDA extension +
its splat_py package) on the GPU:

    python tools/make_golden.py --out <dir>          # the operator / small-scene fixtures
    python tools/make_golden.py --live --out <dir>   # live_reference.npz: the larger scenes, as digests + samples
    python tools/make_golden.py --sh12 --out <dir>   # sh12_reference.npz: SH degrees 1 and 2, both SH modes

then copy the files into tests/golden/.  Scenes are regenerated from seeds by the tests
(gaussian_splatting_b200.synth / tests/scenes.py); the fixtures hold only the reference's OUTPUTS.  Nothing here
touches the product code.
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from gaussian_splatting_b200 import synth  # noqa: E402  (scene generator only)
from oracle import ref_loader  # noqa: E402
from tests import scenes  # noqa: E402

SMALL_SIGMA = (2.5, 0.5, 0.5, 10.0)


def t(a, dev, dtype=None):
    x = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return x if dtype is None else x.to(dtype)


def n(x):
    return x.detach().cpu().numpy()


def run_rasterize(ref, sc, dev, use_sh_precompute=True, bg=0.0, G=None, near=0.3, far=500.0, pad=100, mh=3.0):
    ras = sys.modules["splat_py_ref.rasterize"]
    structs = sys.modules["splat_py_ref.structs"]
    P = {k: t(sc[k], dev).requires_grad_(True) for k in ("xyz", "rgb", "opacity", "scale", "quaternion")}
    sh = None if sc["sh"] is None else t(sc["sh"], dev).requires_grad_(True)
    g = structs.Gaussians(P["xyz"], P["rgb"], P["opacity"], P["scale"], P["quaternion"], sh)
    cam = structs.Camera(sc["W"], sc["H"], t(sc["K"], dev))
    background = torch.full((3,), bg, device=dev, dtype=P["xyz"].dtype)
    image, mask, uv = ras.rasterize(g, t(sc["T"], dev), cam, near, far, pad, mh, use_sh_precompute, background)
    out = dict(image=n(image), culling_mask=n(mask), uv=n(uv))
    if G is not None:
        uv.retain_grad()
        image.backward(t(G, dev))
        out.update(g_xyz=n(P["xyz"].grad), g_rgb=n(P["rgb"].grad), g_opacity=n(P["opacity"].grad),
                   g_scale=n(P["scale"].grad), g_quaternion=n(P["quaternion"].grad), g_uv=n(uv.grad))
        if sh is not None:
            out["g_sh"] = n(sh.grad)
    return out


def stages(ref_ext, sc, dev, near=0.3, far=500.0, pad=100, mh=3.0):
    """Per-operator outputs of the reference on one scene (fp32)."""
    utils = sys.modules["splat_py_ref.utils"]
    N = sc["xyz"].shape[0]
    xyz, q, s, K, T = (t(sc[k], dev) for k in ("xyz", "quaternion", "scale", "K", "T"))
    xyz_cam = utils.transform_points_torch(xyz, T)
    uv = torch.zeros(N, 2, device=dev)
    ref_ext.camera_projection_cuda(xyz_cam, K, uv)
    S = torch.zeros(N, 3, 3, device=dev)
    ref_ext.compute_sigma_world_cuda(q, s, S)
    J = torch.zeros(N, 2, 3, device=dev)
    ref_ext.compute_projection_jacobian_cuda(xyz_cam, K, J)
    conic = torch.zeros(N, 3, device=dev)
    ref_ext.compute_conic_cuda(S, J, T, conic)
    W, H = sc["W"], sc["H"]
    mask = ((xyz_cam[:, 2] < near) | (xyz_cam[:, 2] > far) | (uv[:, 0] < -pad) | (uv[:, 0] > W + pad)
            | (uv[:, 1] < -pad) | (uv[:, 1] > H + pad))
    keep = ~mask
    uvk, xk, ck = uv[keep].contiguous(), xyz_cam[keep].contiguous(), conic[keep].contiguous()
    sorted_idx, ranges = ref_ext.get_sorted_gaussian_list(1024, uvk, xk, ck, (W + 15) // 16, (H + 15) // 16, mh)
    opa = torch.sigmoid(t(sc["opacity"], dev)[keep]).contiguous()
    rgb = t(sc["rgb"], dev)[keep].contiguous()
    if sc["sh"] is not None:
        coeffs = torch.cat((rgb.unsqueeze(2), t(sc["sh"], dev)[keep]), dim=2).contiguous()
        rgb_out = torch.zeros(uvk.shape[0], 3, device=dev)
        ref_ext.precompute_rgb_from_sh_cuda(xyz[keep].contiguous(), coeffs, torch.inverse(T).contiguous(), rgb_out)
        rgb = rgb_out
    return dict(xyz_cam=n(xyz_cam), uv_all=n(uv), sigma_world=n(S), jacobian=n(J), conic_all=n(conic),
                sorted_idx=n(sorted_idx), tile_ranges=n(ranges), opacity_act=n(opa), render_rgb=n(rgb))


def render_state(ref_ext, st, sc, dev, bg):
    """num_splats_per_pixel / final_weight_per_pixel of the reference renderer on stage outputs."""
    keep = ~((st["xyz_cam"][:, 2] < 0.3) | (st["xyz_cam"][:, 2] > 500.0) | (st["uv_all"][:, 0] < -100)
             | (st["uv_all"][:, 0] > sc["W"] + 100) | (st["uv_all"][:, 1] < -100) | (st["uv_all"][:, 1] > sc["H"] + 100))
    H, W = sc["H"], sc["W"]
    img = torch.zeros(H, W, 3, device=dev)
    npp = torch.zeros(H, W, dtype=torch.int32, device=dev)
    wl = torch.zeros(H, W, device=dev)
    ref_ext.render_tiles_cuda(t(st["uv_all"][keep], dev), t(st["opacity_act"], dev).reshape(-1, 1).contiguous(),
                              t(st["render_rgb"], dev), t(st["conic_all"][keep], dev), torch.zeros(1, 1, 1, device=dev),
                              t(st["tile_ranges"], dev), t(st["sorted_idx"], dev),
                              torch.full((3,), bg, device=dev), npp, wl, img)
    return dict(num_splats_per_pixel=n(npp).astype(np.int32), final_weight_per_pixel=n(wl), image_from_stages=n(img))


def grad_summary(key, g, k=64):
    """A gradient as a fixed row sample plus whole-array column sums (tests/test_parity_gpu.py assert_grad_close)."""
    a = n(g).astype(np.float64).reshape(g.shape[0], -1)
    return {f"{key}_rows": a[scenes.sample_rows(a.shape[0], k)].astype(np.float32), f"{key}_absmax": np.abs(a).max(),
            f"{key}_colsum": a.sum(0), f"{key}_colabs": np.abs(a).sum(0)}


def live(out, dev):
    """The reference's outputs on the scenes of the live-reference tests: forward outputs as digests (compared bit
    for bit), gradients as samples + column sums, the reference's own run-to-run noise where a test uses it."""
    ref_ext, _ = ref_loader.load_reference()
    ras = sys.modules["splat_py_ref.rasterize"]
    structs = sys.modules["splat_py_ref.structs"]
    rec = {}

    def run(prefix, sc, G, sh_precompute=True):
        P = {k: t(sc[k], dev).requires_grad_(True) for k in ("xyz", "rgb", "opacity", "scale", "quaternion")}
        sh = None if sc["sh"] is None else t(sc["sh"], dev).requires_grad_(True)
        g = structs.Gaussians(P["xyz"], P["rgb"], P["opacity"], P["scale"], P["quaternion"], sh)
        image, mask, uv = ras.rasterize(g, t(sc["T"], dev), structs.Camera(sc["W"], sc["H"], t(sc["K"], dev)), 0.3,
                                        500.0, 100, 3.0, sh_precompute, torch.full((3,), 0.5, device=dev))
        uv.retain_grad()
        image.backward(t(G, dev))
        rec.update({f"{prefix}_mask": scenes.digest(mask), f"{prefix}_uv": scenes.digest(uv),
                    f"{prefix}_image": scenes.digest(image)})
        if not sh_precompute:  # per-pixel SH: the image is compared to a tolerance, not bit for bit
            rec.update(grad_summary(f"{prefix}_image_px", image.reshape(-1, 3)))
        grads = dict(g_uv=uv.grad, **{f"g_{k}": v.grad for k, v in P.items()}, **({"g_sh": sh.grad} if sh is not None else {}))
        for k, v in grads.items():
            rec.update(grad_summary(f"{prefix}_{k}", v))

    for pose in ("yaw", "general"):
        sc = scenes.np_scene(100_000, "720p", sh_degree=3, seed=0, view=0, n_views=3)
        if pose == "general":
            sc["T"] = scenes.general_pose()
        run(f"r100k_{pose}", sc, synth.make_upstream_grad("720p").numpy())
    run("exact", scenes.exact_arithmetic_scene(), synth.make_upstream_grad("tiny").numpy())
    sc = scenes.np_scene(20_000, "small", sh_degree=3, seed=5, view=1, n_views=3, sigma_px=(2.5, 0.5, 0.5, 10.0))
    run("perpixel", sc, synth.make_upstream_grad("small").numpy(), sh_precompute=False)

    names = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")
    for H in (1080, 1088):
        g, cam, T, G = scenes.headline_inputs(H, dev)
        gr = structs.Gaussians(g.xyz, g.rgb, g.opacity, g.scale, g.quaternion, g.sh)
        runs = []
        for _ in range(2):  # twice: the reference's own nondeterminism (fp32 atomics) is the noise floor
            im, mk, uvr = ras.rasterize(gr, T, structs.Camera(1920, H, cam.K), 0.3, 500.0, 100, 3.0, True,
                                        torch.full((3,), 0.5, device=dev))
            uvr.retain_grad()
            im.backward(G)
            gd = {k: getattr(g, k).grad.clone() for k in names}
            gd["uv"] = uvr.grad.clone()
            for k in names:
                getattr(g, k).grad = None
            runs.append((im.detach(), mk, uvr.detach(), gd))
        (im_a, mask_r, uv_r, gr_a), (im_b, _, _, gr_b) = runs
        p = f"h{H}"
        body = (H // 16) * 16
        rec.update({f"{p}_mask": scenes.digest(mask_r), f"{p}_uv": scenes.digest(uv_r),
                    f"{p}_image_body": scenes.digest(im_a[:body])})
        if body < H:  # ragged bottom tile row: only the pixels where the reference reproduces itself
            stable = (im_a[body:] == im_b[body:]).all(dim=2)
            rec.update({f"{p}_stable": np.packbits(n(stable)), f"{p}_image_stable": scenes.digest(im_a[body:][stable])})
        for k, v in gr_a.items():
            rec.update(grad_summary(f"{p}_g_{k}", v))
            a, b = n(v).astype(np.float64), n(gr_b[k]).astype(np.float64)
            rec[f"{p}_g_{k}_noise"] = np.abs(b - a).max() / max(np.abs(a).max(), 1e-30)
        del g, gr, runs, gr_a, gr_b, im_a, im_b
        torch.cuda.empty_cache()
    rec.update(adc_reference(dev))
    rec["gpu"] = torch.cuda.get_device_name(0)
    np.savez_compressed(out / "live_reference.npz", **{k: np.asarray(v) for k, v in rec.items()})
    print({k: v for k, v in rec.items() if k.endswith("_noise")})


def sh12(out, dev):
    """The reference at SH degrees 1 and 2 (tests/scenes.py sh12_scene), with the SH colour precomputed per gaussian
    and per pixel: forward outputs as digests (the per-pixel image as a sample, it has no bit contract), gradients as
    samples + column sums, and the reference's own run-to-run noise of each gradient."""
    ref_loader.load_reference()
    rec = {}
    G = synth.make_upstream_grad("small").numpy()
    for deg in (1, 2):
        sc = scenes.sh12_scene(deg)
        for mode in ("precompute", "perpixel"):
            a, b = (run_rasterize(None, sc, dev, mode == "precompute", 0.5, G) for _ in range(2))
            p = f"sh{deg}_{mode}"
            rec.update({f"{p}_mask": scenes.digest(a["culling_mask"]), f"{p}_uv": scenes.digest(a["uv"])})
            if mode == "precompute":
                rec[f"{p}_image"] = scenes.digest(a["image"])
            else:
                rec.update(grad_summary(f"{p}_image_px", torch.from_numpy(a["image"].reshape(-1, 3))))
            for k in [k for k in a if k.startswith("g_")]:
                rec.update(grad_summary(f"{p}_{k}", torch.from_numpy(a[k])))
                x, y = a[k].astype(np.float64), b[k].astype(np.float64)
                rec[f"{p}_{k}_noise"] = np.abs(y - x).max() / max(np.abs(x).max(), 1e-30)
    rec["gpu"] = torch.cuda.get_device_name(0)
    np.savez_compressed(out / "sh12_reference.npz", **{k: np.asarray(v) for k, v in rec.items()})
    print({k: float(v) for k, v in rec.items() if k.endswith("_noise")})


def adc_reference(dev):
    """The reference trainer's adaptive_density_control (splat_py/trainer.py + optimizer_manager.py on
    torch.optim.Adam), two consecutive passes on the 100k-gaussian case of tests/test_densify_gpu.py: digests of
    every parameter and Adam moment after each pass."""
    from tests.test_densify_plan import make_case

    ref_loader.load_reference_trainer()
    RT = sys.modules["splat_py_trainer_ref.trainer"]
    RC = sys.modules["splat_py_trainer_ref.config"]
    RO = sys.modules["splat_py_trainer_ref.optimizer_manager"]
    RS = sys.modules["splat_py_trainer_ref.structs"]
    n_ = 100_000
    P, M, V, uv_acc, xyz_acc, cnt = make_case(n_, seed=21, device=dev, n_rest=15)
    config = RC.SplatConfig()
    gr = RS.Gaussians(*(torch.nn.Parameter(P[k].clone()) for k in ("xyz", "rgb", "opacity", "scale", "quaternion")),
                      sh=torch.nn.Parameter(P["sh"].clone()))
    trainer = object.__new__(RT.SplatTrainer)
    trainer.gaussians, trainer.config = gr, config
    trainer.optimizer_manager = RO.OptimizerManager(gr, config)
    order = ("xyz", "quaternion", "scale", "opacity", "rgb", "sh")  # optimizer_manager.py:13-44 group order
    for k, group in zip(order, trainer.optimizer_manager.optimizer.param_groups):
        trainer.optimizer_manager.optimizer.state[group["params"][0]] = dict(
            step=torch.tensor(7.0), exp_avg=M[k].clone(), exp_avg_sq=V[k].clone())
    trainer.uv_grad_accum, trainer.xyz_grad_accum, trainer.grad_accum_count = uv_acc.clone(), xyz_acc.clone(), cnt.clone()
    rec = {}
    for it in (800, 900):
        torch.manual_seed(100 + it)
        trainer.adaptive_density_control(it)
        state = trainer.optimizer_manager.optimizer.state
        for k, group in zip(order, trainer.optimizer_manager.optimizer.param_groups):
            p = group["params"][0]
            rec[f"adc{it}_{k}"] = scenes.digest(getattr(gr, k).detach())
            rec[f"adc{it}_{k}_m"] = scenes.digest(state[p]["exp_avg"])
            rec[f"adc{it}_{k}_v"] = scenes.digest(state[p]["exp_avg_sq"])
        rec[f"adc{it}_n"] = gr.xyz.shape[0]
        n_now = gr.xyz.shape[0]
        gen = torch.Generator(device=dev).manual_seed(it)
        uv2 = torch.rand(n_now, 2, device=dev, generator=gen) * 1e-3
        xyz2 = torch.rand(n_now, 3, device=dev, generator=gen) * 1e-3
        cnt2 = torch.randint(0, 4, (n_now,), device=dev, generator=gen, dtype=torch.int32)
        uv2[cnt2 == 0] = 0.0
        trainer.uv_grad_accum, trainer.xyz_grad_accum, trainer.grad_accum_count = uv2, xyz2, cnt2
    return rec


def fixture6(out, dev):
    """A. the reference's own 6-gaussian unit-test scene (test/gaussian_test_data.py)"""
    ref_ext, _ = ref_loader.load_reference()
    fx = scenes.reference_fixture()
    stA = stages(ref_ext, fx, dev, near=0.3, far=100.0, pad=10, mh=3.0)
    fx_logit = dict(fx, opacity=scenes.inverse_sigmoid(fx["opacity"]))
    rA = run_rasterize(None, fx_logit, dev, True, 0.0, None, 0.3, 100.0, 10, 3.0)
    fx_sh = dict(fx_logit, sh=np.full((6, 3, 15), 0.1, np.float32))
    rA_sh = run_rasterize(None, fx_sh, dev, True, 0.0, None, 0.3, 100.0, 10, 3.0)
    rA_pp = run_rasterize(None, fx_sh, dev, False, 0.0, None, 0.3, 100.0, 10, 3.0)
    # images as digests (compared bit for bit) and, for the per-pixel SH mode (compared to a tolerance), a pixel
    # sample + channel sums: the file stays small
    np.savez_compressed(out / "fixture6_fp32.npz", **{f"st_{k}": v for k, v in stA.items()},
                        image_nosh=scenes.digest(rA["image"]), image_sh_precompute=scenes.digest(rA_sh["image"]),
                        **grad_summary("image_sh_perpixel", torch.from_numpy(rA_pp["image"].reshape(-1, 3)), k=4096),
                        culling_mask=rA["culling_mask"], uv=rA["uv"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="golden_out")
    ap.add_argument("--live", action="store_true")
    ap.add_argument("--fixture6-only", action="store_true")
    ap.add_argument("--sh12", action="store_true")
    args = ap.parse_args()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    dev = torch.device("cuda")
    if args.live:
        return live(out, dev)
    if args.sh12:
        return sh12(out, dev)
    if args.fixture6_only:
        return fixture6(out, dev)
    ref_ext, _ = ref_loader.load_reference()
    meta = dict(gpu=torch.cuda.get_device_name(0), torch=torch.__version__)

    fixture6(out, dev)

    # B/C. synthetic scenes: tiny (SH3, 2000 gaussians, 64x64) and small (SH3, 20000 gaussians, 320x192,
    #      fat splats: > 960 splats in some tiles, saturated pixels)
    for name, nG, res, sig, sh_deg in (("synth_tiny", 2000, "tiny", (2.0, 0.5, 0.5, 8.0), 3),
                                       ("synth_small", 12000, "small", SMALL_SIGMA, 3),
                                       ("synth_deep_nosh", 60000, "small", SMALL_SIGMA, 0)):
        sc = scenes.np_scene(nG, res, sh_degree=sh_deg, seed=0, view=0, n_views=3, sigma_px=sig)
        G = synth.make_upstream_grad(res).numpy()
        st = stages(ref_ext, sc, dev)
        rs = render_state(ref_ext, st, sc, dev, 0.5)
        r = run_rasterize(None, sc, dev, True, 0.5, G)
        r2 = run_rasterize(None, sc, dev, True, 0.5, G)  # the reference's own run-to-run noise
        noise = {k: float(np.abs(r2[k] - r[k]).max() / max(np.abs(r[k]).max(), 1e-30)) for k in r if k.startswith("g_")}
        keepers = dict(r)
        if "g_sh" in keepers and nG > 4000:
            keepers["g_sh_rows8"] = keepers.pop("g_sh")[::8].copy()
        if nG > 30000:  # keep the deep fixture small: every 8th gaussian's gradients
            for k in [k for k in keepers if k.startswith("g_") and k != "g_uv"]:
                keepers[k + "_rows8"] = keepers.pop(k)[::8].copy()
            keepers["g_uv_rows8"] = keepers.pop("g_uv")[::8].copy()
        cnt = st["tile_ranges"][1:] - st["tile_ranges"][:-1]
        np.savez_compressed(out / f"{name}_fp32.npz", **keepers, **rs,
                            **({} if nG > 30000 else dict(
                                st_uv_all=st["uv_all"], st_conic_all=st["conic_all"], st_render_rgb=st["render_rgb"],
                                st_opacity_act=st["opacity_act"], st_xyz_cam=st["xyz_cam"])),
                            st_sorted_idx=st["sorted_idx"], st_tile_ranges=st["tile_ranges"],
                            ref_noise=np.array([noise[k] for k in sorted(noise)]), ref_noise_keys=np.array(sorted(noise)),
                            max_splats_per_tile=int(cnt.max()))
        meta[name] = dict(P=int(st["sorted_idx"].size), max_splats_per_tile=int(cnt.max()), M=int((~r["culling_mask"]).sum()),
                          noise=noise, image_self_equal=bool((r2["image"] == r["image"]).all()))

    # D. fp64 operator surface (the reference's gradcheck dtype): RenderImage on 128 gaussians, 64x64,
    #    N_SH = 1 and 16 (per-pixel SH)
    af = sys.modules["splat_py_ref.cuda_autograd_functions"]
    utils = sys.modules["splat_py_ref.utils"]
    structs = sys.modules["splat_py_ref.structs"]
    sc = scenes.np_scene(128, "tiny", sh_degree=3, seed=3, view=0, n_views=3, dtype=np.float64, sigma_px=(3.0, 0.4, 1.0, 6.0))
    d64 = {}
    for n_sh in (1, 16):
        P = {k: t(sc[k], dev).requires_grad_(True) for k in ("xyz", "rgb", "opacity", "scale", "quaternion", "sh")}
        T64, K64 = t(sc["T"], dev), t(sc["K"], dev)
        xyz_cam = utils.transform_points_torch(P["xyz"], T64)
        uv = af.CameraPointProjection.apply(xyz_cam, K64)
        S = af.ComputeSigmaWorld.apply(P["quaternion"], P["scale"])
        J = af.ComputeProjectionJacobian.apply(xyz_cam, K64)
        conic = af.ComputeConic.apply(S, J, T64)
        tiles = structs.Tiles(64, 64, dev)
        sidx, rng = ref_ext.get_sorted_gaussian_list(1024, uv.detach().float().contiguous(), xyz_cam.detach().float().contiguous(),
                                                     conic.detach().float().contiguous(), tiles.x_tiles_count,
                                                     tiles.y_tiles_count, 3.0)
        opa = torch.sigmoid(P["opacity"])
        cam = structs.Camera(64, 64, K64)
        if n_sh == 1:
            rgb_in, rays = P["rgb"], torch.zeros(1, 1, 1, dtype=torch.float64, device=dev)
        else:
            rgb_in = torch.cat((P["rgb"].unsqueeze(2), P["sh"]), dim=2)
            rays = utils.compute_rays_in_world_frame(cam, T64)
        image = af.RenderImage.apply(rgb_in, opa, uv, conic, rays, rng, sidx, torch.tensor([64, 64], device=dev),
                                     torch.full((3,), 0.5, dtype=torch.float64, device=dev))
        G64 = synth.make_upstream_grad("tiny", dtype=torch.float64).to(dev)
        image.backward(G64)
        d64.update({f"nsh{n_sh}_image": n(image), f"nsh{n_sh}_sorted_idx": n(sidx), f"nsh{n_sh}_ranges": n(rng),
                    **{f"nsh{n_sh}_g_{k}": n(v.grad) for k, v in P.items() if v.grad is not None}})
    np.savez_compressed(out / "synth_tiny_fp64.npz", **d64)

    import json

    (out / "golden_meta.json").write_text(json.dumps(meta, indent=1))
    print(json.dumps(meta, indent=1))


if __name__ == "__main__":
    main()
