"""rasterize_surfels(): 2-D Gaussian surfels (2DGS, Huang et al., SIGGRAPH 2024) in the fused rasterizer.

The scene is the 3DGS scene (mean, quaternion, scales, opacity logit, SH) and binning is the 3DGS binning; each gaussian
is rendered as a flat disk whose two tangent axes are scale[:, 0] and scale[:, 1] (scale[:, 2] is not used and gets an
exact 0 gradient).  Per pixel the ray meets the surfel at a point (a, b) of its plane, so depth lies on the surface and
every surfel has a normal.  The model is DESIGN.md 3.25; the kernels are libgsr_surfels.so (include/gsr_surfels.h).
Through a fisheye or OPENCV lens (DESIGN.md 3.26) each pixel intersects its own undistorted ray, from a ray map, with
the surfel; those kernels are libgsr_surfels_lens.so (include/gsr_surfels_lens.h).  Per-gaussian feature channels
blended with the colour's weights (DESIGN.md 3.27) are libgsr_surfels_features.so's (include/gsr_surfels_features.h),
the median depth (DESIGN.md 3.28) libgsr_surfels_median.so's (include/gsr_surfels_median.h).

Two autograd nodes, as in rasterize():

    _ProjectSurfels    params -> uv [M,2], carrier          (gsr_surfel_preprocess_forward, binning, tile forward)
    _CompositeSurfels  uv, carrier[, features] -> image, depth, alpha, normal, distortion[, median][, feature map]

``carrier`` only carries the tile backward's per-surfel gradient rows [N,20] to the per-gaussian backward, which writes
the flat gradient layout of rasterize() (state.grad_flat, or grad_out), so FlatAdam, DensificationStats,
AdaptiveDensityControl and MCMCDensityControl drive a surfel scene unchanged.
"""
from __future__ import annotations

import math
import weakref

import torch

from . import native
from .rasterize import (IN_KERNEL_TRANSFORM, IN_KERNEL_TRANSFORM_MIN_N, _depth_key_params, _lens_arg,
                        _lens_constants, in_kernel_transform_ok, native_centre_ok, tail_positions)
from .utils import transform_points_torch


class _SurfelState:
    """Per-view buffers shared by the two autograd nodes (return_state=True hands it out).  vis_idx / vis_idx32: the
    visible gaussians, ascending (the order of uv); grad_flat: the flat gradient of the last backward; lens: None (the
    pinhole) or (the native SURFEL_LENS_* value, its device constants); rays: the lens's ray map [H,W,3] (0 where a
    pixel has no ray); median_ids: each pixel's median surfel [H,W] int32 (-1: none), with median_depth."""

    __slots__ = ("N", "M", "P", "H", "W", "visible", "vis_idx", "vis_idx32", "scan", "surfels", "ranges", "keys_sorted",
                 "ids_sorted", "id_bits", "maps", "last", "totals", "background", "near", "m_scale", "mh", "grad_flat",
                 "grad_out", "uv_ref", "uv_grad_emitted", "uv_absgrad", "lens", "rays", "K", "median_ids")

    def __init__(self):
        self.grad_flat = self.grad_out = self.uv_ref = self.uv_absgrad = self.lens = self.rays = self.median_ids = None
        self.uv_grad_emitted = False


class _ProjectSurfels(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, quaternion, scale, opacity, rgb, sh, camera_T_world, K, state, cfg):
        ext = native()
        H, W, near, far, pad, mh = cfg
        depth_base, depth_bits = _depth_key_params(near, far)
        opacity_flat = opacity.reshape(-1)
        N = xyz.shape[0]
        # camera-frame positions and camera centre exactly as rasterize() forms them, so that uv and the culling mask
        # are bit-identical to rasterize's
        if IN_KERNEL_TRANSFORM and N >= IN_KERNEL_TRANSFORM_MIN_N and in_kernel_transform_ok(xyz.device):
            xyz_cam = tail_positions(xyz, camera_T_world)
        else:
            xyz_cam = transform_points_torch(xyz, camera_T_world)
        centre = None
        if sh is not None:
            if native_centre_ok(xyz.device):
                centre = ext.camera_centre(camera_T_world)
            else:
                centre = torch.linalg.inv_ex(camera_T_world)[0][:3, 3].contiguous()
        args = (xyz, xyz_cam, quaternion, scale, opacity_flat, rgb, sh, camera_T_world, K, centre, H, W, near, far,
                pad, mh, depth_base)
        if state.lens is None:
            surfels, bins, zkey, visible, scan, tile_mask, tile_win = ext.surfel_forward(*args)
        else:
            state.rays = ext.surfel_rays(*state.lens, K, H, W)
            surfels, bins, zkey, visible, scan, tile_mask, tile_win = ext.surfel_lens_forward(*state.lens, *args)
        total = int(scan[-1].item()) if N > 0 else 0
        M, P = total >> 32, total & 0xFFFFFFFF
        if M > N or P >= 2**31:
            raise RuntimeError(f"rasterize_surfels: {P} (gaussian, tile) pairs / {M} visible of {N} gaussians exceed "
                               "the int32 pair index of the native path (P must be < 2^31)")
        ids_sorted, ranges, vis_idx, uv, keys_sorted, id_bits = ext.fused_bin(
            bins, zkey, visible, scan, M, P, H, W, mh, depth_bits, False, tile_mask, tile_win)
        m_scale = far / (far - near) if math.isfinite(far) else 1.0
        rargs = (surfels, ranges, state.background, H, W, P, keys_sorted, ids_sorted, int(id_bits), near, m_scale, mh)
        rendered = (ext.surfel_render_forward(*rargs) if state.lens is None
                    else ext.surfel_lens_render_forward(state.rays, *rargs))
        state.N, state.M, state.P, state.H, state.W = N, M, P, H, W
        state.visible, state.vis_idx, state.vis_idx32, state.scan = visible, vis_idx, vis_idx, scan
        state.surfels, state.ranges, state.keys_sorted, state.ids_sorted, state.id_bits = (
            surfels, ranges, keys_sorted, ids_sorted, int(id_bits))
        state.maps, state.last, state.totals = rendered[:5], rendered[5], rendered[6]
        state.near, state.m_scale, state.mh, state.K = near, m_scale, mh, K
        ctx.state = state
        ctx.has_sh = sh is not None
        ctx.opacity_shape = opacity.shape
        ctx.save_for_backward(xyz, quaternion, scale, opacity_flat, sh, camera_T_world, K, centre)
        carrier = torch.empty(20 * N, dtype=xyz.dtype, device=xyz.device)
        return uv, carrier

    @staticmethod
    def backward(ctx, grad_uv, grad_carrier):
        xyz, quaternion, scale, opacity_flat, sh, camera_T_world, K, centre = ctx.saved_tensors
        st = ctx.state
        if grad_carrier is None:
            grad_carrier = torch.zeros(20 * st.N, dtype=xyz.dtype, device=xyz.device)
        guv = grad_uv.contiguous() if grad_uv is not None and st.M > 0 else None
        args = (grad_carrier.contiguous(), xyz, quaternion, scale, opacity_flat, sh, camera_T_world, K, centre,
                st.visible, st.surfels, st.grad_out, guv, st.scan if guv is not None else None, st.uv_grad_emitted)
        out = (native().surfel_backward(*args) if st.lens is None
               else native().surfel_lens_backward(*st.lens, *args))
        g_xyz, g_q, g_s, g_o, g_dc = out[:5]
        g_sh = out[5] if ctx.has_sh else None
        st.grad_flat = out[-1]
        return g_xyz, g_q, g_s, g_o.view(ctx.opacity_shape), g_dc, g_sh, None, None, None, None


class _CompositeSurfels(torch.autograd.Function):
    """uv, carrier[, features] -> (image, depth, alpha, normal, distortion[, median][, feature map]); the tile forward
    already ran in _ProjectSurfels, the median (DESIGN.md 3.28) and feature (DESIGN.md 3.27) forwards run here on its
    pair list, `last` and ray map."""

    @staticmethod
    def forward(ctx, uv, carrier, state, features=None, median_depth=False):
        ctx.state = state
        ctx.set_materialize_grads(False)  # an output without a gradient comes as None: no feature / median backward
        maps = state.maps
        state.maps = None
        outs = tuple(maps)
        ctx.median_depth = median_depth
        if median_depth:
            median, state.median_ids = native().surfel_median_forward(
                state.rays, state.surfels, state.ranges, state.H, state.W, state.P, state.keys_sorted,
                state.ids_sorted, state.id_bits, state.mh, state.last)
            outs = outs + (median,)
        fpad = None
        ctx.n_features = 0
        if features is not None:
            # the feature kernels read 4 channels per CTA with 16-byte copies: rows padded to a multiple of 4 columns
            D = features.shape[1]
            stride = (D + 3) // 4 * 4
            fpad = features
            if stride != D:
                fpad = torch.nn.functional.pad(features, (0, stride - D))
            elif features.data_ptr() % 16 != 0:
                fpad = features.clone()
            fmap = native().surfel_features_forward(state.rays, state.surfels, state.ranges, state.H, state.W, state.P,
                                                    state.keys_sorted, state.ids_sorted, state.id_bits, state.mh,
                                                    state.last, fpad, D)
            ctx.n_features = D
            outs = outs + (fmap,)
        ctx.save_for_backward(maps[2], fpad)  # alpha: the backward's total weight and final transmittance
        return outs

    @staticmethod
    def backward(ctx, g_image, g_depth, g_alpha, g_normal, g_dist, *g_rest):
        st = ctx.state
        g_median = g_rest[0] if ctx.median_depth else None
        g_features = g_rest[1:] if ctx.median_depth else g_rest
        alpha, fpad = ctx.saved_tensors

        def grad(g, k):
            return torch.zeros(st.H, st.W, k, device=alpha.device) if g is None else g.contiguous()

        args = (st.N, st.surfels, st.ranges, st.background, st.H, st.W, st.P, st.keys_sorted, st.ids_sorted,
                st.id_bits, st.near, st.m_scale, st.mh, alpha, st.last, st.totals, grad(g_image, 3), grad(g_depth, 1),
                grad(g_alpha, 1), grad(g_normal, 3), grad(g_dist, 1))
        ext = native()
        rows = (ext.surfel_render_backward(*args) if st.lens is None
                else ext.surfel_lens_render_backward(st.rays, *args))
        grad_features = None
        if ctx.n_features and g_features[0] is not None:
            # into the same rows, before uv.grad and the per-gaussian backward read them: the feature loss's part of
            # d alpha
            gpad = ext.surfel_features_backward(st.rays, st.surfels, st.ranges, st.H, st.W, st.P, st.keys_sorted,
                                                st.ids_sorted, st.id_bits, st.mh, st.last, st.totals, fpad,
                                                ctx.n_features, g_features[0].contiguous(), rows)
            if ctx.needs_input_grad[3]:
                grad_features = gpad if gpad.shape[1] == ctx.n_features else gpad[:, :ctx.n_features]
        if g_median is not None:
            # into the same rows, after the colour and feature backwards and before uv.grad and the per-gaussian backward
            # read them: the median loss through each pixel's median surfel's z
            ext.surfel_median_backward(st.rays, st.surfels, st.H, st.W, st.mh, st.median_ids, g_median.contiguous(),
                                       rows)
        # uv.grad (d loss / d footprint translation) is formed only when somebody can observe it, as in rasterize()
        uv_t = st.uv_ref() if st.uv_ref is not None else None
        watched = uv_t is None or uv_t.retains_grad or bool(uv_t._backward_hooks)
        st.uv_grad_emitted = bool(watched)
        grad_uv = None
        if watched:
            grad_uv = (ext.surfel_uv_grad(st.vis_idx, st.surfels, rows) if st.lens is None
                       else ext.surfel_lens_uv_grad(*st.lens, st.K, st.vis_idx, st.surfels, rows))
        return grad_uv, rows.view(-1), None, grad_features, None


def _surfel_lens(fisheye, distortion, device):
    """(native SURFEL_LENS_* value, [n+1] device constants) for the lens arguments, or None for the pinhole"""
    lens = _lens_arg(fisheye, distortion)
    if lens is None:
        return None
    ext = native()
    code = ext.SURFEL_LENS_FISHEYE if lens[0] == "fisheye" else ext.SURFEL_LENS_DISTORTION
    return code, _lens_constants(*lens, device).reshape(-1)


def rasterize_surfels(gaussians, camera_T_world, camera, near_thresh, far_thresh, cull_mask_padding, mh_dist,
                      background_rgb, return_state=False, grad_out=None, fisheye=None, distortion=None, features=None,
                      median_depth=False):
    """Render the gaussians as 2-D surfels.  Arguments as rasterize() with use_sh_precompute=True; mh_dist is the
    cutoff radius r in the surfel's own units (a pixel takes part where rho <= r^2) and must be > 0.

    Returns (image [H,W,3], culling_mask [N] bool, uv [M,2], depth [H,W,1], alpha [H,W,1], normal [H,W,3],
    distortion [H,W,1]), then the median [H,W,1] with median_depth, the feature map [H,W,D] with features, and the
    state with return_state.  Per pixel,
    with the blend weights w_i = T_i alpha_i of the colour: alpha = sum w_i; depth = sum w_i z_i (z_i the camera z of the ray-surfel intersection, or p_z where the
    low-pass filter decides; expected depth is depth / alpha); normal = sum w_i n_i (camera frame, each n_i facing the
    camera, not normalised); distortion = sum_i w_i sum_{j<i} w_j (m_i - m_j)^2 with m = (f / (f - n)) (1 - n / z),
    n, f = near_thresh, far_thresh (2DGS's depth-distortion term).  Every output is differentiable; gradients reach
    xyz, quaternion, scale[:, :2], opacity, rgb and sh (the colour is the SH colour at the centre's view direction,
    held constant for xyz as in rasterize).  uv.grad is d loss / d delta, delta a pixel translation of the surfel's
    whole footprint (DESIGN.md 3.25), for densification.  The backward writes rasterize()'s flat gradient layout
    (state.grad_flat, or grad_out when given).

    fisheye=k (COLMAP's OPENCV_FISHEYE, k1 k2 k3 k4) or distortion=k (COLMAP's OPENCV, k1 k2 p1 p2 k3) renders through
    that lens, with the coefficients as rasterize() takes them (host values; the two are exclusive).  Each pixel then
    meets the surfel along its own undistorted ray (state.rays; DESIGN.md 3.26), which is exact for the central lens;
    uv, the depth keys and the culling mask are rasterize()'s with the same lens, and a pixel with no ray on the lens's
    monotone branch (beyond fisheye_theta_max or distortion_r2_max) shows the background.  uv.grad is then
    J_n^-T g_n + g_c, the gradient on a translation of the footprint in the normalised plane mapped to pixels through
    the lens Jacobian at the centre; its sum is d loss / d(cx, cy) for the pinhole only.

    features: an fp32 CUDA tensor [N, D] (D >= 1, contiguous, on the gaussians' device; it may require grad) of
    per-gaussian channels (semantics, instance ids, distilled features, any attribute).  The feature map [H,W,D],
    feature_map[p, c] = sum_i w_i F[i, c] with exactly the colour's surfels, order and fp32 weights w_i and no
    background term, is then returned after the distortion (DESIGN.md 3.27).  Its gradient reaches F (returned through
    autograd, not part of the flat layout) and, through the blend weights, the geometry: the feature loss lands in the
    same gradient rows as the maps', so uv.grad, state.grad_flat / grad_out and everything that reads them see it.

    median_depth=True also returns the median depth [H,W,1] after the distortion, before the feature map (2DGS's
    median; DESIGN.md 3.28): per pixel the camera z (as depth blends it) of the last of the colour's surfels whose
    transmittance in front of it, 1 - A in fp32, is above 0.5; 0 where no surfel contributes.  state.median_ids holds
    those surfels' indices [H,W] (-1: none).  Its gradient goes to that surfel's z only (its position, orientation and
    the surfel plane; not its opacity, colour or the choice of surfel), into the same gradient rows as the maps'.
    2DGS's bounded-scene depth is (1 - r) depth / alpha + r median (INTEGRATION.md B23).

    fp32 CUDA tensors only (TypeError otherwise); a camera_T_world, K or lens-coefficient tensor that requires grad
    raises ValueError: no camera gradient is formed for surfels."""
    g = gaussians
    tensors = [g.xyz, g.quaternion, g.scale, g.opacity, g.rgb, camera_T_world, camera.K, background_rgb]
    if g.sh is not None:
        tensors.append(g.sh)
    for t in tensors:
        if not torch.is_tensor(t) or t.dtype != torch.float32:
            raise TypeError("rasterize_surfels takes fp32 tensors only, got "
                            + (str(t.dtype) if torch.is_tensor(t) else type(t).__name__))
    if camera_T_world.requires_grad or camera.K.requires_grad:
        raise ValueError("rasterize_surfels forms no camera gradient: pass camera_T_world.detach() and "
                         "camera.K.detach()")
    if any(torch.is_tensor(k) and k.requires_grad for k in (fisheye, distortion)):
        raise ValueError("rasterize_surfels forms no camera gradient: pass lens coefficients that do not require grad")
    if features is not None:
        if not torch.is_tensor(features):
            raise TypeError("features must be a torch tensor [N, D]")
        if features.dtype != torch.float32:
            raise TypeError(f"features must be float32, got {features.dtype}")
        n = g.xyz.shape[0]
        if features.dim() != 2 or features.shape[0] != n or features.shape[1] < 1:
            raise ValueError(f"features has shape {tuple(features.shape)} but must be [{n}, D] with D >= 1 (one row "
                             "per gaussian)")
        if features.device != g.xyz.device or not features.is_contiguous():
            raise ValueError("features must be contiguous and on the gaussians' device")
    lens = _lens_arg(fisheye, distortion)
    if any(t.device.type != "cuda" or t.device != g.xyz.device for t in tensors):
        raise ValueError("rasterize_surfels needs every tensor on the gaussians' CUDA device")
    if not float(mh_dist) > 0.0:
        raise ValueError(f"mh_dist must be > 0, got {mh_dist}")
    if background_rgb.numel() != 3:
        raise ValueError("background_rgb must hold 3 values")
    state = _SurfelState()
    if lens is not None:
        state.lens = _surfel_lens(fisheye, distortion, g.xyz.device)
    state.grad_out = grad_out
    state.background = background_rgb.contiguous()
    cfg = (int(camera.height), int(camera.width), float(near_thresh), float(far_thresh), float(cull_mask_padding),
           float(mh_dist))
    uv, carrier = _ProjectSurfels.apply(
        g.xyz.contiguous(), g.quaternion.contiguous(), g.scale.contiguous(), g.opacity.contiguous(), g.rgb.contiguous(),
        None if g.sh is None else g.sh.contiguous(), camera_T_world.contiguous(), camera.K.contiguous(), state, cfg)
    state.uv_ref = weakref.ref(uv)
    culling_mask = state.visible == 0
    maps = _CompositeSurfels.apply(uv, carrier, state, features, bool(median_depth))
    image, depth, alpha, normal, distortion = maps[:5]
    result = (image, culling_mask, uv, depth, alpha, normal, distortion) + tuple(maps[5:])
    return (*result, state) if return_state else result


def depth_normals(depth, alpha, camera, eps=1e-6, fisheye=None, distortion=None):
    """Normals of the rendered surface [H,W,3] for 2DGS's normal-consistency loss 1 - n . N: the expected depth
    z = depth / alpha.clamp_min(eps) is back-projected along each pixel's ray, and each interior pixel gets the
    normalised cross product of the central differences along x and y, turned towards the camera.  Border pixels are 0.
    The ray is K^-1 (x, y, 1) for the pinhole, and with fisheye=k / distortion=k the lens's ray d of rasterize_surfels
    (point = d z / d_z, CUDA tensors only); pixels next to one without a ray are 0 as well."""
    H, W = depth.shape[0], depth.shape[1]
    d = (depth / alpha.clamp_min(eps)).reshape(H, W, 1)
    valid = None
    if fisheye is None and distortion is None:
        ys, xs = torch.meshgrid(torch.arange(H, device=d.device, dtype=d.dtype),
                                torch.arange(W, device=d.device, dtype=d.dtype), indexing="ij")
        pix = torch.stack((xs, ys, torch.ones_like(xs)), -1)
        rays = pix @ torch.linalg.inv(camera.K.to(d.dtype)).T
    else:
        if d.device.type != "cuda":
            raise ValueError("depth_normals with a lens needs CUDA tensors: the rays come from the native ray kernel")
        code, consts = _surfel_lens(fisheye, distortion, d.device)
        ray = native().surfel_rays(code, consts, camera.K.to(d.device, torch.float32).contiguous(), H, W)
        ray = ray.to(d.dtype)
        valid = ray[..., 2:] > 0
        rays = torch.where(valid, ray / torch.where(valid, ray[..., 2:], torch.ones_like(ray[..., 2:])), 0.0)
    pts = rays * d
    out = torch.zeros_like(pts)
    dx = pts[1:-1, 2:] - pts[1:-1, :-2]
    dy = pts[2:, 1:-1] - pts[:-2, 1:-1]
    n = torch.nn.functional.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    facing = (n * pts[1:-1, 1:-1]).sum(-1, keepdim=True) > 0
    inner = torch.where(facing, -n, n)
    if valid is not None:
        ok = valid[1:-1, 2:] & valid[1:-1, :-2] & valid[2:, 1:-1] & valid[:-2, 1:-1] & valid[1:-1, 1:-1]
        inner = torch.where(ok, inner, 0.0)
    out[1:-1, 1:-1] = inner
    return out
