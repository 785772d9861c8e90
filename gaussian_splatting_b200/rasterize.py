"""rasterize(): drop-in for splat_py.rasterize.rasterize (splat_py/rasterize.py:18-112).

Same nine positional arguments, same return triple ``(image [H,W,3], culling_mask [N] bool,
uv [M,2])``, same values.  ``uv`` is a graph tensor whose ``.grad`` after ``backward()`` is the
render pass's gradient on the projected means, exactly what the reference trainer reads for
densification (splat_py/trainer.py:360,379-385).

Implementation: two autograd nodes around the native fused kernels

    _ProjectGaussians   params -> uv [M,2], carrier          (gsr_preprocess_forward + binning)
    _CompositeTiles     uv, carrier[, features] -> image[, depth, alpha][, feature map]
                                                          (gsr_render_forward_gather; gsr_render_features_*)

(The tile renderer's forward kernel is enqueued by the projection node, right behind the binning and BEFORE the
host reads the pair count; `_CompositeTiles` only ties its image into the graph.)

``carrier`` is an uninitialised [12N] tensor that only carries gradient: the render backward returns its
per-Gaussian sums as the carrier's gradient — interleaved rows ``rgb3 opacity | uv2 conic0 conic1 | conic2 pad3`` —
and the per-Gaussian backward consumes them.  One host read per forward (the pair count, which sizes the pair
buffers) and it is taken off the critical path: the buffers are sized from the previous views' counts and the
count is only checked afterwards (DESIGN.md 3.5); the reference path has ~25 syncs.

``use_sh_precompute=False`` (per-pixel view directions) is routed through the operator-by-operator
path `rasterize_unfused`, which mirrors the reference's structure on this library's operators.
"""
from __future__ import annotations

import weakref

import torch

from . import native
from .cuda_autograd_functions import (
    CameraPointProjection,
    ComputeConic,
    ComputeProjectionJacobian,
    ComputeSigmaWorld,
    PrecomputeRGBFromSH,
    RenderImage,
)
from .structs import Tiles
from .tile_culling import get_splats
from .utils import compute_rays_in_world_frame, transform_points_torch


import os

# world->camera inside the fused kernel (saves a torch.matmul over all points).  The kernel reproduces the rounding
# order of the cuBLAS kernel torch dispatches to for full 65535-matrix chunks; a last chunk whose size cuBLAS sends
# through another kernel (on H100 / cuBLAS 12.8: sizes of roughly 16 K to 35 K matrices, and small ones) is formed by
# torch.matmul, found out per device and chunk size (chunk_matches_kernel).  Below IN_KERNEL_TRANSFORM_MIN_N, or
# with GSR_TORCH_TRANSFORM=1, positions are formed by torch.matmul exactly as the reference does
# (splat_py/utils.py:60-72).
IN_KERNEL_TRANSFORM = os.environ.get("GSR_TORCH_TRANSFORM", "0") != "1"
# the forward records which (8x4 pixel block, splat) pairs contributed; the backward then visits exactly those
# (GSR_NO_MASKS=1: the backward redoes the forward's conservative footprint test instead)
USE_CONTRIBUTION_MASKS = os.environ.get("GSR_NO_MASKS", "0") != "1"
# pair emission expands the tile-hit masks of the per-gaussian stage (GSR_RETEST_TILES=1: repeats the OBB tests)
USE_TILE_MASKS = os.environ.get("GSR_RETEST_TILES", "0") != "1"
IN_KERNEL_TRANSFORM_MIN_N = 16384
CUBLAS_BATCH_CHUNK = 65535   # gridDim limit cuBLAS batches against
SMALL_BATCH = 1024           # chunks below ~300 use another kernel (measured: 100 differs, 300 matches)


_TRANSFORM_OK = {}  # (device index, n) -> bool: did the in-kernel transform reproduce torch.matmul on n points?


def tail_positions(xyz, camera_T_world):
    """Camera-frame positions of the last cuBLAS chunk when the in-kernel transform would not reproduce
    torch.matmul's bits for a chunk of that size (None when it does); all of them for a single such chunk."""
    N = xyz.shape[0]
    tail = N % CUBLAS_BATCH_CHUNK
    if tail == 0 or (tail >= SMALL_BATCH and chunk_matches_kernel(xyz.device, tail)):
        return None
    return transform_points_torch(xyz[N - tail:], camera_T_world)


def chunk_matches_kernel(device, n: int) -> bool:
    """Does cuBLAS round a single chunk of `n` matrices the way the fused kernel does?  (cached per device and n)"""
    return in_kernel_transform_ok(device, n=n, warn=False)


def in_kernel_transform_ok(device, n: int = 70_000, seed: int = 1234, warn: bool = True) -> bool:
    """One-time self-check per device (a cuBLAS / torch upgrade could change the rounding order the fused
    kernel mimics): `n` random points (more than one 65535-matrix cuBLAS chunk) under a random rigid pose, camera
    z and uv from the in-kernel transform compared BIT FOR BIT with the reference's op
    (splat_py/utils.py:60-72, torch.matmul).  On a mismatch the fused path forms positions with torch.matmul
    itself from then on (the reference's own op on the GPU, +2.3 ms at 3M points) and says so once."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    ok = _TRANSFORM_OK.get((idx, n))
    if ok is not None:
        return ok
    import math
    import warnings

    ext = native()
    gen = torch.Generator().manual_seed(seed)
    xyz = (torch.rand(n, 3, generator=gen) * torch.tensor([8.0, 6.0, 10.0]) + torch.tensor([-4.0, -3.0, 1.0])).to(device)
    q = torch.randn(4, generator=gen)
    w, x, y, z = (q / q.norm()).tolist()
    T = torch.eye(4)
    T[:3, :3] = torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                              [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                              [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    T[:3, 3] = torch.randn(3, generator=gen)
    T = T.to(device)
    K = torch.tensor([[1200.0, 0.0, 960.0], [0.0, 1200.0, 540.0], [0.0, 0.0, 1.0]], device=device)
    quat = torch.zeros(n, 4, device=device)
    quat[:, 0] = 1.0
    zeros3, zeros1 = torch.zeros(n, 3, device=device), torch.zeros(n, device=device)
    big = 1e30
    with torch.no_grad():
        rec, zkey, _, _ = ext.fused_preprocess_forward(xyz, None, quat, zeros3, zeros1, zeros3, None, T, K, None, 1080,
                                                       1920, -big, big, big, 3.0, 0)
        ref = transform_points_torch(xyz, T)
        zref = ref[:, 2].contiguous().view(torch.int32)
        zref = torch.where(zref < 0, ~zref, zref | -2**31)
        uv = torch.zeros(n, 2, device=device)
        ext.camera_projection_cuda(ref, K, uv)
        fin = torch.isfinite(uv).all(dim=1) & torch.isfinite(rec[:, :2]).all(dim=1)
        same = bool((zkey == zref).all()) and bool((rec[:, 0:2][fin].contiguous().view(torch.int32)
                                                    == uv[fin].contiguous().view(torch.int32)).all())
    _TRANSFORM_OK[(idx, n)] = same
    if not same and warn:
        warnings.warn("gaussian_splatting_b200: the in-kernel world->camera transform no longer reproduces "
                      "torch.matmul bit for bit on this device (cuBLAS changed its rounding order?); "
                      "falling back to torch.matmul for camera-frame positions", RuntimeWarning)
    return same


# ---- speculative sizing of the pair buffers (see _ProjectGaussians.forward) -----------------------------------------
SPECULATIVE_BINNING = os.environ.get("GSR_EAGER_COUNTS", "0") != "1"
_PAIR_HISTORY = {}   # (device index, N, H, W) -> pair counts of the most recent views
_PINNED = {}         # device index -> [pinned int64 ring, next slot]
PAIR_HEADROOM = 1.04  # capacity = max(recent P) * headroom + 64 Ki pairs


def _pair_capacity(key):
    hist = _PAIR_HISTORY.get(key)
    if not hist:
        return None
    cap = int(max(hist) * PAIR_HEADROOM) + 65536
    return min((cap + 127) // 128 * 128, 2**31 - 128)


def _fit_masks(ext, rendered, P, H, W):
    """The renderer's outputs of a speculative run that fitted its capacity, with the contribution masks cut to the
    words of the P pairs actually binned (the buffer was sized for the capacity; the words past them stay zero), so that
    the state does not depend on the pair counts of earlier views."""
    rendered = tuple(rendered)
    masks = rendered[3]
    if masks.numel() == 0:
        return rendered
    return rendered[:3] + (masks.narrow(0, 0, ext.contribution_mask_words(P, H, W)),) + rendered[4:]


def _note_pairs(key, P):
    hist = _PAIR_HISTORY.setdefault(key, [])
    hist.append(int(P))
    del hist[:-8]
    if len(_PAIR_HISTORY) > 64:  # scenes come and go (densification changes N): keep the table small
        for k in list(_PAIR_HISTORY)[:-32]:
            del _PAIR_HISTORY[k]


_SIDE = {}           # device index -> side stream for the count read-back


def _side_stream(device):
    idx = device.index if device.index is not None else torch.cuda.current_device()
    st = _SIDE.get(idx)
    if st is None:
        st = _SIDE[idx] = torch.cuda.Stream(device=device)
    return st


def _pinned_slot(device):
    idx = device.index if device.index is not None else torch.cuda.current_device()
    ring = _PINNED.get(idx)
    if ring is None:
        ring = _PINNED[idx] = [torch.empty(16, dtype=torch.int64).pin_memory(), 0]
    ring[1] = (ring[1] + 1) % 16
    return ring[0][ring[1]:ring[1] + 1]


_CENTRE_OK = {}  # device index -> bool: does gsr_camera_centre reproduce torch's inverse on this device?


def native_centre_ok(device, n: int = 8, seed: int = 4321) -> bool:
    """One-time self-check per device: the camera centre from the library's single kernel (the arithmetic of
    cuSOLVER getrf + cuBLAS trsm as pinned by tools/dev/inverse_probe2.py, csrc/gsr_preprocess.cu `camera_centre`) against
    torch.linalg.inv_ex, BIT FOR BIT, on `n` random rigid poses and a few general matrices.  A cuSOLVER / cuBLAS
    upgrade that changes the rounding order makes rasterize() use torch's own inverse again (15 micro-kernels)."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    ok = _CENTRE_OK.get(idx)
    if ok is not None:
        return ok
    import warnings

    ext = native()
    gen = torch.Generator().manual_seed(seed)
    same = True
    with torch.no_grad():
        for k in range(n):
            if k % 4 == 3:
                T = torch.eye(4)
                T[:3, :] = torch.randn(3, 4, generator=gen)
            else:
                q = torch.randn(4, generator=gen)
                w, x, y, z = (q / q.norm()).tolist()
                T = torch.eye(4)
                T[:3, :3] = torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                                          [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                                          [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
                T[:3, 3] = torch.randn(3, generator=gen) * 3.0
            T = T.to(device)
            a = ext.camera_centre(T)
            b = torch.linalg.inv_ex(T)[0][:3, 3].contiguous()
            same = same and bool((a.view(torch.int32) == b.view(torch.int32)).all())
    _CENTRE_OK[idx] = same
    if not same:
        warnings.warn("gaussian_splatting_b200: gsr_camera_centre no longer reproduces torch.linalg.inv_ex bit for "
                      "bit on this device; using torch's inverse for the camera centre", RuntimeWarning)
    return same


import functools


@functools.lru_cache(maxsize=64)
def _depth_key_params(near, far):
    """(base, bits): depth keys are float bits of z minus `base`; `bits` low bits are significant."""
    import math
    import struct

    def fbits(v):
        return struct.unpack("<I", struct.pack("<f", v))[0]

    FLT_MAX = 3.4028234663852886e38
    if near > 0.0 and math.isfinite(far) and near < far <= FLT_MAX:
        b0, b1 = fbits(near), fbits(far)  # struct.pack rounds to nearest: a tiny `near` can round to 0.0f
        if b0 > 0 and b1 > b0:
            return b0, max(1, (b1 - b0).bit_length())
    # no usable positive range (near <= 0 or rounding to 0.0f, far infinite / beyond FLT_MAX / NaN): full 32-bit
    # order-preserving keys (depth_key() sets bit 31, so depth_bits MUST be 32 whenever the base is 0)
    return 0, 32


class _ViewState:
    """Non-differentiable per-view buffers shared by the two autograd nodes."""

    __slots__ = ("N", "M", "P", "H", "W", "visible", "vis_idx", "_ids_sorted", "ranges",
                 "records", "keys_sorted", "id_bits",
                 "n_per_pixel", "w_per_pixel", "background", "profile", "grad_flat", "grad_out", "vis_idx32", "scan", "masks", "uv_ref", "uv_grad_emitted", "image", "speculation_overflowed",
                 "mode", "zkey", "depth_base", "depth_bits", "depth", "alpha", "uv_absgrad", "filter3d",
                 "weight_stats", "lens", "shutter")

    @property
    def ids_sorted(self):
        """int32 [P]: gaussian id of every sorted (gaussian, tile) pair (the reference's
        `sorted_gaussian_idx_by_splat_idx`).  When the id rides in the sort key the tile kernels read it from the
        keys and nobody writes this array: it is extracted on demand."""
        if self._ids_sorted is not None and self._ids_sorted.numel() == 0 and self.P > 0 and self.keys_sorted is not None:
            mask = (1 << self.id_bits) - 1
            self._ids_sorted = (self.keys_sorted[:self.P] & mask).to(torch.int32)
        return self._ids_sorted

    @property
    def gather(self):
        """Always True: the tile kernels read every record through the sorted pair list (there is no other record
        source any more; kept readable for callers of return_state that check it)."""
        return True

    def __init__(self, profile=None):
        self.profile = profile  # optional list: (stage name, start event, end event) per native call
        self.grad_flat = None   # set by the backward pass: flat buffer holding all parameter gradients
        self.grad_out = None    # optional caller-owned buffer (same layout) the backward writes them into
        self.uv_ref = None      # weak reference to the uv tensor handed to the caller
        self.uv_grad_emitted = False
        self.background = None  # set by rasterize() before the projection node runs (it pre-launches the renderer)
        self.image = None
        self.speculation_overflowed = False
        # MODE_* bits of the native fused path: MODE_DEPTH_ALPHA (render_depth_alpha: the tile kernels also produce
        # depth / alpha [H,W,1]), MODE_ANTIALIASED (opacity compensation for the 0.25 px^2 dilation), MODE_ABSGRAD
        # (the render backward also sums |d loss_p / d uv| per pixel), MODE_FILTER3D (Mip-Splatting's 3-D filter in the
        # per-gaussian stages: filter3d [N], a constant)
        self.mode = 0
        self.filter3d = None
        self.lens = None        # a lens model: (its LENS_* value, its constants on the device) (_lens_state)
        self.shutter = None     # a rolling shutter: (its twist [6] on the device, its READOUT_* value)
        self.depth = self.alpha = None
        self.uv_absgrad = None  # MODE_ABSGRAD: [M,2], set by every render backward
        self.weight_stats = None  # optional densify.WeightStats the render forward accumulates into


class _stage:
    """CUDA-event bracket around one native stage (only when the caller asked for a profile)."""

    def __init__(self, state, name):
        self.rec = state.profile
        self.name = name

    def __enter__(self):
        if self.rec is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *exc):
        if self.rec is not None:
            self.e1.record()
            self.rec.append((self.name, self.e0, self.e1))


# ---- lens models: fisheye and radial-tangential distortion -------------------------------------------------------------
# name -> (coefficient names, the native cull limit of one row of coefficients, the native LENS_* value)
_LENSES = {"fisheye": ("k1 k2 k3 k4", "fisheye_theta_max", "LENS_FISHEYE"),
           "distortion": ("k1 k2 p1 p2 k3", "distortion_r2_max", "LENS_DISTORTION")}


def fisheye_theta_max(k) -> float:
    """The cull limit of COLMAP's OPENCV_FISHEYE model with coefficients k = (k1, k2, k3, k4): the first theta in
    (0, pi/2) where d theta_d / d theta = 1 + 3 k1 theta^2 + 5 k2 theta^4 + 7 k3 theta^6 + 9 k4 theta^8 reaches 0 (beyond
    it the model folds points back into the image), else pi/2; found in fp64 for the fp32 coefficients and rounded down
    to fp32 (gsr_fisheye_theta_max, the value the kernels cull with)."""
    return native().fisheye_theta_max([float(v) for v in _lens_coefficients("fisheye", k)])


def distortion_r2_max(k) -> float:
    """The cull limit of COLMAP's OPENCV (radial-tangential) model with coefficients k = (k1, k2, p1, p2, k3): the
    smallest positive s = r^2 where d (r radial(r^2)) / dr = 1 + 3 k1 s + 5 k2 s^2 + 7 k3 s^3 reaches 0 (beyond it
    barrel distortion folds points back into the image), else +inf; found in fp64 for the fp32 coefficients and
    rounded down to fp32 (gsr_distortion_r2_max, the value the kernels cull with).  The tangential p1 p2 do not enter
    it: COLMAP's are of order 1e-3."""
    return native().distortion_r2_max([float(v) for v in _lens_coefficients("distortion", k)])


def _lens_coefficients(lens, k, C=None):
    """A lens's host coefficients as float32 numpy [n] (C None) or [C,n]; ValueError for a CUDA tensor, a wrong shape
    or non-finite values.  Batches take [n] (shared) or [C,n]."""
    import numpy as np

    names = _LENSES[lens][0]
    n = len(names.split())
    if torch.is_tensor(k):
        if k.device.type != "cpu":
            raise ValueError(f"{lens} coefficients are camera constants read on the host: pass a CPU tensor or a "
                             "sequence, not a tensor on " + str(k.device))
        k = k.detach().to(torch.float64).numpy()
    else:
        try:
            k = np.asarray(k, dtype=np.float64)
        except (TypeError, ValueError) as e:
            raise ValueError(f"{lens} must be {n} numbers {names}: {e}") from None
    shapes = ((n,),) if C is None else ((n,), (C, n))
    if k.shape not in shapes:
        want = f"[{n}]" if C is None else f"[{n}] or [{C},{n}]"
        raise ValueError(f"{lens} has shape {list(k.shape)} but must be {want} ({names})")
    with np.errstate(over="ignore"):
        k32 = k.astype(np.float32)
    if not np.isfinite(k32).all():
        raise ValueError(f"{lens} coefficients must be finite (in fp32)")
    return k32 if C is None or k.ndim == 2 else np.broadcast_to(k32, (C, n))


def _lens_arg(fisheye, distortion, C=None):
    """None (the pinhole) or (lens name, coefficients as _lens_coefficients returns them)."""
    if fisheye is not None and distortion is not None:
        raise ValueError("pass either fisheye or distortion: a camera has one lens model")
    if fisheye is not None:
        return "fisheye", _lens_coefficients("fisheye", fisheye, C)
    if distortion is not None:
        return "distortion", _lens_coefficients("distortion", distortion, C)
    return None


_LENS_CONSTS = {}  # (lens, device, coefficient bytes) -> [C, n+1] device constants


def _lens_constants(lens, k, device):
    """[C, n+1] fp32 on the device: each row the n coefficients and the lens's cull limit.  Copied from pinned memory
    without blocking the host and kept per (lens, device, coefficients), so a camera's constants are uploaded once."""
    import numpy as np

    limit = getattr(native(), _LENSES[lens][1])
    k = np.ascontiguousarray(np.reshape(k, (-1, np.shape(k)[-1])), np.float32)
    key = (lens, str(device), k.tobytes())
    t = _LENS_CONSTS.get(key)
    if t is None:
        lim = [limit([float(v) for v in row]) for row in k]
        host = torch.from_numpy(np.concatenate([k, np.asarray(lim, np.float32)[:, None]], 1)).pin_memory()
        t = host.to(device, non_blocking=True)
        if len(_LENS_CONSTS) >= 64:
            _LENS_CONSTS.clear()
        _LENS_CONSTS[key] = t
    return t


def _lens_state(lens, device):
    """state.lens for _lens_arg's result: None (the pinhole), or (the native LENS_* value, its device constants)"""
    if lens is None:
        return None
    return getattr(native(), _LENSES[lens[0]][2]), _lens_constants(*lens, device)


def _lens_kwargs(lens):
    """The lens arguments of the per-gaussian bindings for a state's lens"""
    lens, consts = lens or (native().LENS_PINHOLE, None)
    return dict(lens=lens, lens_consts=consts)


def _lens_input(fisheye, distortion):
    """The lens coefficient tensor that takes a gradient: a CPU tensor that requires grad, else None (a sequence of
    numbers and a tensor that does not require grad stay host constants)."""
    k = fisheye if fisheye is not None else distortion
    return k if torch.is_tensor(k) and k.requires_grad else None


def _intrinsics_grad(g):
    """d loss / d K [..., 3, 3] from the kernels' [..., 4] (fx, fy, cx, cy); every other entry (the skew, the last
    row) is exactly 0: the projection never reads it."""
    out = g.new_zeros(*g.shape[:-1], 9)
    out[..., 0], out[..., 4], out[..., 2], out[..., 5] = g[..., 0], g[..., 1], g[..., 2], g[..., 3]
    return out.view(*g.shape[:-1], 3, 3)


def _lens_grad(g, k):
    """The lens-coefficient gradient [n] / [C,n] on the device, brought to the host in k's shape and dtype: one blocking
    device->host copy (the coefficients are host constants, DESIGN.md 3.23).  A [C,n] gradient for a shared [n] k is
    summed over the views in fp64."""
    g = g.to("cpu").to(torch.float64)
    if g.dim() == 2 and k.dim() == 1:
        g = g.sum(0)
    return g.to(k.dtype)


READOUTS = ("top_to_bottom", "bottom_to_top", "left_to_right", "right_to_left")


def _shutter_arg(xi, readout, K, lens_k, device, H, W, C=None):
    """Checks rasterize's / rasterize_batch's rolling_shutter and readout (before any launch); returns
    (twists [6] or [C,6] for the kernels, the native READOUT_* value), or None for a global shutter."""
    if readout not in READOUTS:
        raise ValueError(f"readout must be one of {READOUTS}, got {readout!r}")
    if xi is None:
        return None
    if not torch.is_tensor(xi):
        raise TypeError("rolling_shutter must be a torch tensor [6] (a twist (rho, omega), pose.se3_exp's convention)")
    if xi.dtype != torch.float32:
        raise TypeError(f"rolling_shutter must be float32, got {xi.dtype}")
    shapes = ((6,),) if C is None else ((6,), (C, 6))
    if tuple(xi.shape) not in shapes:
        raise ValueError(f"rolling_shutter has shape {tuple(xi.shape)} but must be "
                         + (" or ".join(str(list(t)) for t in shapes)))
    if xi.device != device:
        raise ValueError("rolling_shutter must be on the gaussians' device")
    if (H if readout in READOUTS[:2] else W) < 2:
        raise ValueError(f"a {readout} readout needs at least 2 lines")
    if K.requires_grad or lens_k is not None:
        raise ValueError("intrinsics and lens-coefficient gradients are not available with rolling_shutter: pass "
                         "camera.K.detach() and constant lens coefficients")
    xi = xi.detach()
    if C is not None and xi.dim() == 1:
        xi = xi.expand(C, 6)
    return xi.contiguous(), getattr(native(), "READOUT_" + readout.upper())


def _shutter_kwargs(shutter):
    """The rolling-shutter arguments of the per-gaussian forward bindings for a state's shutter"""
    return {} if shutter is None else dict(rolling_shutter=shutter[0], readout=shutter[1])


def _preprocess_backward(ctx, native_fn, args):
    """The per-gaussian backward: (gaussian grads..., flat), g_pose, g_K, g_k, g_xi (None where no gradient is
    wanted).  The intrinsics or the lens coefficients require grad: the camera-gradient kernels (libgsr_calib.so); only
    the pose: the pose kernels (libgsr_pose.so); neither: the plain kernels.  With a rolling shutter the shutter
    kernels (libgsr_shutter.so), with the camera row when the pose or the twists require grad."""
    need = ctx.needs_input_grad
    st = ctx.state
    if st.shutter is not None:
        camera_grads = 1 if need[6] or need[11] else 0
        out = native_fn(*args, **_lens_kwargs(st.lens), camera_grads=camera_grads, **_shutter_kwargs(st.shutter),
                        height=st.H, width=st.W)
        n = 6 + ctx.has_sh
        grads, cam = out[:n], out[n:]
        g_xi = None
        if need[11]:
            g_xi = cam[1] if ctx.xi_shape == tuple(cam[1].shape) else cam[1].sum(0)
        return grads, cam[0] if need[6] else None, None, None, g_xi
    camera_grads = 2 if need[7] or need[10] else 1 if need[6] else 0
    out = native_fn(*args, **_lens_kwargs(st.lens), camera_grads=camera_grads)
    n = 6 + ctx.has_sh  # the gaussian gradients and the flat allocation, then the camera gradients
    grads, cam = out[:n], out[n:]
    g_pose = cam[0] if need[6] else None
    g_K = _intrinsics_grad(cam[1]) if need[7] else None
    g_k = _lens_grad(cam[2], ctx.lens_k) if ctx.lens_k is not None and need[10] else None
    return grads, g_pose, g_K, g_k, None


class _ProjectGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, quaternion, scale, opacity, rgb, sh, camera_T_world, K, state, cfg, lens_k=None, xi=None):
        # lens_k: the lens coefficient tensor when it requires grad (an input for its gradient only: the forward reads
        # the constants uploaded to state.lens); xi likewise the rolling-shutter twist (state.shutter)
        ext = native()
        # torch.matmul takes another path (other rounding) for an operand that requires grad: the forward's bits must
        # not depend on whether the pose does
        camera_T_world = camera_T_world.detach()
        H, W, near, far, pad, mh = cfg
        depth_base, depth_bits = _depth_key_params(near, far)
        opacity_flat = opacity.reshape(-1)
        # camera-frame positions: by default formed exactly like the reference does (torch.matmul,
        # splat_py/utils.py:60-72), because their bits decide tile membership and the 1/255 skip and the
        # rounding order inside cuBLAS is not ours to pin; IN_KERNEL_TRANSFORM folds it into the kernel.
        N = xyz.shape[0]
        if IN_KERNEL_TRANSFORM and N >= IN_KERNEL_TRANSFORM_MIN_N and in_kernel_transform_ok(xyz.device):
            # cuBLAS runs the batched product in chunks of 65535 matrices; a last chunk it sends through another
            # kernel (different rounding order) is formed by torch itself
            xyz_cam = tail_positions(xyz, camera_T_world)
        else:
            xyz_cam = transform_points_torch(xyz, camera_T_world)
        # camera centre for the SH view direction = inverse(camera_T_world)[:3, 3] with the bits of the reference's
        # torch.inverse (splat_py/rasterize.py:91-93): ONE native kernel that reproduces torch's LU arithmetic
        # (verified per device, native_centre_ok), else torch's own inverse (inv_ex: no host sync)
        centre = None
        if sh is not None:
            if native_centre_ok(xyz.device):
                centre = ext.camera_centre(camera_T_world)
            else:
                centre = torch.linalg.inv_ex(camera_T_world)[0][:3, 3].contiguous()
        with _stage(state, "preprocess_fwd"):
            # tile_mask / tile_win: the tiles each gaussian hits, tested once here and only expanded by the pair emission
            records, zkey, visible, scan, tile_mask, tile_win = ext.fused_preprocess_forward(
                xyz, xyz_cam, quaternion, scale, opacity_flat, rgb, sh, camera_T_world, K, centre, H, W, near, far, pad,
                mh, depth_base, True, state.mode, state.filter3d, **_lens_kwargs(state.lens),
                **_shutter_kwargs(state.shutter))
        # a backward pass can follow (the camera counts: a pose-, intrinsics- or shutter-only refinement needs the
        # masks too)
        record_masks = USE_CONTRIBUTION_MASKS and (any(ctx.needs_input_grad[:8]) or any(ctx.needs_input_grad[10:]))
        background = state.background

        def counts(total):
            M_, P_ = total >> 32, total & 0xFFFFFFFF
            # M and P share one u64 scan (M<<32 | P) and the native entry points index pairs with int32: a scene
            # with >= 2^31 (gaussian, tile) pairs must fail loudly, not wrap into an empty render
            if M_ > N or P_ >= 2**31:
                raise RuntimeError(f"rasterize: {P_} (gaussian, tile) pairs / {M_} visible of {N} gaussians exceed "
                                   "the int32 pair index of the native path (P must be < 2^31)")
            return M_, P_

        depth_keys = zkey if state.mode & ext.MODE_DEPTH_ALPHA else None

        ws = state.weight_stats
        stats = () if ws is None else (ws.weight_sum, ws.weight_max, ws.pixel_count)

        def bin_and_render(M_, P_, speculative):
            with _stage(state, "bin_sort_gather"):
                binned = ext.fused_bin(records, zkey, visible, scan, M_, P_, H, W, mh, depth_bits, speculative,
                                       tile_mask if USE_TILE_MASKS else None, tile_win if USE_TILE_MASKS else None)
            # weight statistics of a speculative run: the kernel compares the scan's pair count with the capacity and
            # adds nothing when the run is discarded for overflowing it
            guard = (scan, P_) if (stats and speculative) else ()
            with _stage(state, "render_fwd"):
                rendered = ext.fused_render_forward(records, binned[1], background, H, W, P_, record_masks, binned[4],
                                                    binned[0], binned[5], depth_keys, depth_base, depth_bits, *stats,
                                                    *guard)
            return binned, rendered

        # The host needs M and P (the shape of the returned uv; the size of the pair buffers).  Reading them right
        # here stalls the GPU for a launch round trip (35 us resident, ~100 us when the step's host->device copies
        # share the queue).  Instead the pair buffers are sized from the pair counts of the recent views of this
        # (N, H, W) plus headroom, binning AND the tile renderer are enqueued, and only then the counts — copied to
        # pinned memory right behind the scan — are read: by then they are long there.  Padding behind the real
        # pairs sorts to the end and is ignored (gsr_emit_*'s capacity).  If a view overflows the guess, the two
        # stages run again with the exact sizes (and the guess grows); the first view of a kind reads eagerly.
        key = (xyz.device.index, N, H, W)
        cap = _pair_capacity(key) if (SPECULATIVE_BINNING and N > 0) else None
        if cap is None:
            total = int(scan[-1].item()) if N > 0 else 0
            M, P = counts(total)
            binned, rendered = bin_and_render(M, P, False)
        else:
            # the 8-byte copy goes on a side stream: on the main stream the binning kernels would queue behind it,
            # and it is slow when the step's own host<->device traffic shares the copy engines (25 us, measured)
            slot = _pinned_slot(xyz.device)
            side = _side_stream(xyz.device)
            scanned = torch.cuda.Event()
            scanned.record()
            with torch.cuda.stream(side):
                side.wait_event(scanned)
                slot.copy_(scan[-1:], non_blocking=True)
                ready = torch.cuda.Event()
                ready.record(side)
            binned, rendered = bin_and_render(N, cap, True)
            ready.synchronize()
            M, P = counts(int(slot.item()))
            if P > cap:  # the guess was too small: nothing usable was produced, run the two stages again
                binned, rendered = bin_and_render(M, P, False)
                state.speculation_overflowed = True
            else:
                ids_c, ranges_c, vis_c, uv_c, keys_c, idb = binned
                binned = (ids_c.narrow(0, 0, P) if ids_c.numel() else ids_c, ranges_c, vis_c.narrow(0, 0, M),
                          uv_c.narrow(0, 0, M), keys_c, idb)
                rendered = _fit_masks(ext, rendered, P, H, W)
        _note_pairs(key, P)
        ids_sorted, ranges, vis_idx, uv, keys_sorted, id_bits = binned
        state.records, state.keys_sorted, state.id_bits = records, keys_sorted, int(id_bits)
        state.image, state.n_per_pixel, state.w_per_pixel, state.masks, state.depth, state.alpha = rendered
        state.zkey, state.depth_base, state.depth_bits = depth_keys, depth_base, depth_bits
        state.N, state.M, state.P, state.H, state.W = xyz.shape[0], M, P, H, W
        state.visible = visible
        state.vis_idx = state.vis_idx32 = vis_idx                # int32 [M]: visible gaussians, ascending
        state._ids_sorted, state.ranges = ids_sorted, ranges
        state.scan = scan
        # gradient slab: one interleaved row of 12 floats per gaussian
        carrier = torch.empty(12 * xyz.shape[0], dtype=xyz.dtype, device=xyz.device)
        ctx.state = state
        ctx.has_sh = sh is not None
        ctx.lens_k = lens_k
        ctx.xi_shape = None if xi is None else tuple(xi.shape)
        ctx.save_for_backward(xyz, quaternion, scale, opacity_flat, sh, camera_T_world, K, centre)
        return uv, carrier

    @staticmethod
    def backward(ctx, grad_uv, grad_carrier):
        xyz, quaternion, scale, opacity_flat, sh, camera_T_world, K, centre = ctx.saved_tensors
        st = ctx.state
        N = st.N
        if grad_carrier is None:
            grad_carrier = torch.zeros(12 * N, dtype=xyz.dtype, device=xyz.device)
        slab = grad_carrier.contiguous()
        # Gradient on the projected means: the render backward's sums sit in the slab's uv section (by gaussian).
        # What autograd hands us for the COMPACT uv is either nothing / only what the caller added upstream of uv
        # (the render node did not emit its part: added to the slab's section in the kernel, row = rank among the
        # visible gaussians from the forward's scan), or the TOTAL (the render node did emit it because somebody
        # watches uv.grad: it then replaces the slab's section).  Incoming gradients are never edited.
        guv = None
        if grad_uv is not None and st.M > 0:
            guv = grad_uv.contiguous()
        with _stage(st, "preprocess_bwd"):
            args = (slab, xyz, quaternion, scale, opacity_flat, sh, camera_T_world, K, centre, st.visible, st.grad_out,
                    guv, st.scan if guv is not None else None, not st.uv_grad_emitted, st.mode, st.filter3d)
            grads, g_pose, g_K, g_k, g_xi = _preprocess_backward(ctx, native().fused_preprocess_backward, args)
        g_xyz, g_q, g_s, g_o, g_dc = grads[:5]
        g_sh = grads[5] if ctx.has_sh else None
        st.grad_flat = grads[-1]  # the one allocation all parameter gradients of this view are views of
        return g_xyz, g_q, g_s, g_o.view(-1, 1), g_dc, g_sh, g_pose, g_K, None, None, g_k, g_xi


class _CompositeTiles(torch.autograd.Function):
    """uv, carrier[, features] -> image, or (image, depth, alpha) with the depth/alpha maps, then the feature map."""

    @staticmethod
    def forward(ctx, uv, carrier, background_rgb, state, features=None):
        # the tile renderer was already enqueued by the projection node (right behind the binning, before the host
        # learned the pair count): this node only ties its outputs to uv and to the gradient carrier
        outs = (state.image,) if state.depth is None else (state.image, state.depth, state.alpha)
        state.image = state.depth = state.alpha = None
        ctx.state = state
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
            # P is final here: the projection node reran binning and the renderer if the speculative guess overflowed
            with _stage(state, "features_fwd"):
                fmap = native().fused_render_features_forward(state.records, state.ranges, state.H, state.W, state.P,
                                                              state.keys_sorted, state._ids_sorted, state.id_bits,
                                                              fpad, D)
            ctx.n_features = D
            ctx.save_for_backward(fpad)
            outs = outs + (fmap,)
        return outs if len(outs) > 1 else outs[0]

    @staticmethod
    def backward(ctx, grad_image, *grad_maps):
        st = ctx.state
        grad_depth = grad_alpha = None
        if st.mode & native().MODE_DEPTH_ALPHA:
            grad_depth, grad_alpha = grad_maps[:2]
        with _stage(st, "render_bwd"):
            slab = native().fused_render_backward(
                grad_image.contiguous(), st.N, st.P, st.records, st._ids_sorted, st.ranges, st.background,
                st.n_per_pixel, st.w_per_pixel, st.masks, st.keys_sorted, st.id_bits,
                None if grad_depth is None else grad_depth.contiguous(),
                None if grad_alpha is None else grad_alpha.contiguous(), st.zkey, st.depth_base, st.depth_bits,
                st.mode)
        grad_features = None
        if ctx.n_features:
            # into the same slab, before the per-gaussian backward reads it: the feature loss's part of d alpha
            (fpad,) = ctx.saved_tensors
            with _stage(st, "features_bwd"):
                gpad = native().fused_render_features_backward(
                    grad_maps[-1].contiguous(), slab, st.P, st.records, st._ids_sorted, st.ranges, st.n_per_pixel,
                    st.w_per_pixel, st.masks, st.keys_sorted, st.id_bits, fpad)
            if ctx.needs_input_grad[4]:
                grad_features = gpad if gpad.shape[1] == ctx.n_features else gpad[:, :ctx.n_features]
        uv_t = st.uv_ref() if st.uv_ref is not None else None
        if st.mode & native().MODE_ABSGRAD:
            # sum over pixels of |d loss_p / d uv| (rows' slots 10-11), in the compact order of uv; replaced, not
            # accumulated, by every backward.  Also set as uv.absgrad (gsplat's convention) while uv is alive.  The two
            # columns are selected before the rows: gathering whole 48-byte rows first costs 1.5 ms at 3M (H100)
            st.uv_absgrad = slab.view(st.N, 12)[:, 10:12].index_select(0, st.vis_idx)
            if uv_t is not None:
                uv_t.absgrad = st.uv_absgrad
        # The render pass's gradient on the compact uv is a gather of the slab's uv section (28 us at 3M).  It
        # reaches the per-gaussian backward through the slab anyway, so it is only materialised when it can be
        # OBSERVED: the caller retained uv's gradient (the reference trainer does, splat_py/trainer.py:360) or
        # hooked the tensor.
        watched = uv_t is None or uv_t.retains_grad or bool(uv_t._backward_hooks)
        st.uv_grad_emitted = bool(watched)
        if not watched:
            return None, slab, None, None, grad_features
        # interleaved rows: rgb3 opa | uv2 conic0 conic1 | conic2 pad3 (depth mode: z pad2)
        grad_uv = slab.view(st.N, 12).index_select(0, st.vis_idx)[:, 4:6].contiguous()
        return grad_uv, slab, None, None, grad_features


def rasterize(gaussians, camera_T_world, camera, near_thresh, far_thresh, cull_mask_padding, mh_dist,
              use_sh_precompute, background_rgb, return_state=False, profile=None, grad_out=None,
              render_depth_alpha=False, antialiased=False, absgrad=False, filter3d=None, weight_stats=None,
              features=None, fisheye=None, distortion=None, rolling_shutter=None, readout="top_to_bottom"):
    """render_depth_alpha=True: also the per-pixel depth and alpha maps, differentiable, from the same tile walk —
    returns (image, culling_mask, uv, depth [H,W,1], alpha [H,W,1]) (+ state with return_state).  alpha is the
    accumulated blend weight before the background; depth = sum of w_i * z_i over the same splats and weights as the
    colour, z_i the camera-frame z, with no background term (expected depth: depth / alpha.clamp_min(eps)).  fp32
    and precomputed SH colours only.

    antialiased=True: every splat's opacity is multiplied by rho = sqrt(max(det S, 0) / det(S + 0.25 I)), S its 2-D
    covariance, so that the 0.25 px^2 dilation the renderer applies no longer adds mass to splats smaller than a pixel
    (the "antialiased" mode of Mip-Splatting's 2-D filter).  Gradients flow through rho to the covariance.  Return
    values are unchanged; combines with render_depth_alpha.  fp32 and precomputed SH colours only.

    absgrad=True: the render backward also sums, per visible gaussian, the ABSOLUTE value of every pixel's gradient on
    its projected mean, sum_p |d <G_p, out_p> / d uv| (AbsGS; gsplat's absgrad), where uv.grad sums the signed values
    and lets opposite pulls of the pixels under a large splat cancel.  After each backward it is uv.absgrad [M,2] (set
    on the returned uv while that tensor is alive; no retain_grad() needed) and state.uv_absgrad, replaced, not
    accumulated.  Pixels in units, like uv.grad; only the render stage's part (not a gradient the caller adds on uv);
    G_p includes the depth / alpha maps' upstream gradients with render_depth_alpha.  For densification:
    DensificationStats.accumulate(..., absgrad=True).  Return values, uv.grad and all gradients are unchanged;
    combines with render_depth_alpha and antialiased.  fp32 and precomputed SH colours only.

    filter3d: Mip-Splatting's 3-D smoothing filter, an fp32 CUDA tensor [N] or [N,1] of standard deviations f in world
    units (gaussian_splatting_b200.filter3d.compute_filter3d, from the training cameras).  Every gaussian is rendered
    with the world covariance R diag(exp(2 scale) + f^2) R^T and the opacity sigmoid(o) * coef, coef =
    sqrt(prod_k exp(2 scale_k) / (exp(2 scale_k) + f^2)), which keeps its 3-D mass (DESIGN.md 3.13); f is only used
    squared, and f = 0 renders exactly as without the filter.  The filter is a constant: it gets no gradient, and the
    parameter gradients (state.grad_flat as usual) are those of the raw parameters.  Return values and uv.grad keep
    their meaning; combines with antialiased (coef comes before rho), render_depth_alpha, absgrad, return_state and
    grad_out.  After densification changes N the filter must be recomputed: a filter of another length raises
    ValueError.  fp32 and precomputed SH colours only; the values are not checked (no host synchronisation).

    weight_stats: a densify.WeightStats of N Gaussians the render forward accumulates blend-weight importance into:
    per Gaussian, over the pixels where it takes part in the colour blend, the sum and the max of its blend weight
    w = T * alpha (the float the image uses; with antialiased / filter3d alpha carries the compensated opacity) and
    the number of such pixels (DESIGN.md 3.14).  Added to, never zeroed, by every call, with or without gradients, for
    importance pruning (AdaptiveDensityControl.prune).  Return values, uv.grad, uv.absgrad and all gradients are
    unchanged and the statistics are not differentiable; combines with render_depth_alpha, antialiased, filter3d,
    absgrad, return_state and grad_out.  A WeightStats of another length raises ValueError (make a new one after
    densification changes N).  fp32 and precomputed SH colours only.

    features: an fp32 CUDA tensor [N, D] (D >= 1, contiguous, on the gaussians' device; it may require grad) of
    per-gaussian feature vectors to blend with the colour's weights, for feature or semantic distillation,
    instance channels or rendered normals.  The return tuple gains feature_map [H,W,D] after depth/alpha and before
    state: (image, culling_mask, uv[, depth, alpha][, feature_map][, state]).  Per pixel feature_map[p, c] =
    sum_i w_i * F[i, c] over exactly the splats, in exactly the order and with exactly the blend weights w_i = T * alpha
    (the same floats) as the colour, with no background term (composite with alpha, render_depth_alpha=True, for one).
    The gradient reaches F (sum_p w_ip * G[p, c], zero for culled gaussians) and, through alpha, opacity and the
    geometry: uv.grad is the total loss's gradient on the projected means (DESIGN.md 3.17).  Separate tile kernels
    process the channels in chunks of 4, each chunk walking the tile's pairs again.  The image, mask, uv, depth /
    alpha, weight statistics and all other gradients are unchanged; combines with render_depth_alpha, antialiased,
    filter3d, weight_stats, return_state and grad_out, not with absgrad (ValueError).  fp32 and precomputed SH colours
    only.

    fisheye: COLMAP's OPENCV_FISHEYE (Kannala-Brandt) camera instead of the pinhole, k = (k1, k2, k3, k4) =
    params[4:8] of the COLMAP camera as 4 host numbers (a sequence or a CPU tensor [4]; fx fy cx cy stay in camera.K).
    A camera-frame point (x, y, z) projects to u = fx (theta_d / rho) x + cx, v = fy (theta_d / rho) y + cy with
    rho = |(x, y)|, theta = atan2(rho, z), theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8);
    k = 0 is the equidistant fisheye, not the pinhole.  The 2-D covariance uses the Jacobian of that projection at the
    mean (EWA), and a gaussian at theta >= fisheye_theta_max(k), where the model folds back, is culled on top of the
    near / far / padding rules.  Depth keys, the depth map and the SH view direction keep camera-frame z and the
    position; uv and uv.grad are the fisheye pixel coordinates and their gradient (DESIGN.md 3.19); for K and k
    requiring grad see camera.K below.  The coefficients are constants of the camera, uploaded once per camera without synchronising
    with the device.  Combines with every other option.  None (the default) is the pinhole.  A CUDA tensor, a wrong
    shape or non-finite coefficients raise ValueError; fp32 and precomputed SH colours only.

    distortion: COLMAP's OPENCV radial-tangential camera (OpenCV's 5-coefficient model) instead of the pinhole,
    k = (k1, k2, p1, p2, k3) in OpenCV's distCoeffs order as 5 host numbers; structs.camera_from_colmap builds it from
    a COLMAP camera (OPENCV, FULL_OPENCV without rational terms, RADIAL, SIMPLE_RADIAL).  With a = x / z, b = y / z,
    s = a^2 + b^2 and radial = 1 + k1 s + k2 s^2 + k3 s^3 a camera-frame point projects to u = fx a_d + cx,
    v = fy b_d + cy, a_d = a radial + 2 p1 a b + p2 (s + 2 a^2), b_d = b radial + p1 (s + 2 b^2) + 2 p2 a b.  The 2-D
    covariance uses the exact Jacobian of that projection at the mean, and a gaussian at s >= distortion_r2_max(k),
    where barrel distortion folds back, is culled on top of the other rules.  Everything else is as for fisheye
    (DESIGN.md 3.20); k = 0 runs the distortion kernels and gives the pinhole up to fp32 rounding.  Passing both
    fisheye and distortion raises ValueError.

    camera_T_world: when it requires grad (a leaf, or e.g. pose.PoseDelta's se3_exp(xi) @ T0), the backward also gives
    d loss / d camera_T_world [4,4], for pose refinement, with every lens and option above.  With W = T[:3,:3] and
    p_i = W x_i + t: dL/dT[:3,:3] = sum_i (g_p,i x_i^T + J_i^T (2 G_i M_i Sigma_i)), dL/dT[:3,3] = sum_i g_p,i,
    dL/dT[3,:] = 0, over the visible gaussians, g_p the gradient on the camera-frame mean (projection, lens, depth and
    any gradient on uv), G the gradient on the 2-D covariance M Sigma M^T, M = J W.  The camera centre of the SH view
    direction is held constant, as it is for xyz (exact with SH degree 0).  Reduced natively in a fixed order, so the
    same render-stage rows give the same bits (DESIGN.md 3.21).  Everything else is unchanged.  A pose that does not
    require grad runs exactly the kernels without it.  rasterize_unfused (and fp64 / per-pixel SH) gives the pose only
    what autograd gets through its torch transform of the means.

    camera.K: when it requires grad (e.g. calib.IntrinsicsDelta's output), the backward also gives d loss / d K [3,3]
    for self-calibration: dL/dfx = sum_i (g_u a_d + sum_j gJ[0,j] J[0,j] / fx), dL/dcx = sum_i g_u (fy, cy with row 1),
    u = fx a_d + cx the lens's projection, g_u the complete gradient on u, gJ the gradient on the Jacobian; every other
    entry (the skew, the last row) is exactly 0.  Lens coefficients: a CPU tensor that requires grad passed as fisheye=
    or distortion= gets d loss / d k in its shape and dtype, through one blocking device -> host copy of n floats at the
    end of the backward (only then; a sequence of numbers gets none).  Cull limits get no gradient.  Every lens and
    option combine with it; outputs, gaussian gradients and the pose gradient are bit-identical to a run without it
    (DESIGN.md 3.23).

    rolling_shutter: a rolling-shutter camera whose lines are read out one after another while it moves.
    camera_T_world is then the pose of the image's middle line, and rolling_shutter an fp32 tensor xi = (rho, omega)
    [6] on the gaussians' device (pose.se3_exp's convention, e.g. a row of an nn.Parameter of zeros [n_images, 6]): the
    camera's motion over the whole readout, applied on the left, T(tau) = se3_exp((tau - 1/2) xi) @ camera_T_world for
    the line read at time tau in [0, 1].  readout gives the line time of a pixel: "top_to_bottom" (the default,
    tau = v / (H - 1)), "bottom_to_top", "left_to_right" (u / (W - 1)) or "right_to_left"; pose.shutter_from_endpoints
    turns first-line / last-line poses into (camera_T_world, xi).  Each gaussian is projected at its own line's time
    tau* = clamp(r(u(tau*)), 0, 1) (a fixed number of Newton steps), with the pose, depth and lens Jacobian of that
    time; its 2-D covariance includes the time's dependence on image position, A J W Sigma W^T J^T A^T with
    A = I + f e^T / (1 - lambda), f = du/dtau and lambda the point's speed along the readout (a shear for a pan across
    the lines, a stretch for motion along them).  A gaussian with lambda >= 3/4 or an unconverged time is culled.  The
    SH view direction keeps the centre of camera_T_world.  xi = 0 renders bit-identically to the call without it.
    Gradients are exact derivatives of this model (tau* an implicit function of the inputs): to the gaussians, to
    camera_T_world when it requires grad, and to xi when it requires grad (DESIGN.md 3.24).  The values of xi are read
    by the kernels without a host synchronisation and are not checked.  Combines with every lens and option above
    except K or lens-coefficient gradients (ValueError).  A wrong shape, device (ValueError) or dtype (TypeError) of
    xi, an unknown readout or a 1-line image raise before any launch; None (the default) runs exactly the kernels
    without it.  fp32 and precomputed SH colours only."""
    lens = _lens_arg(fisheye, distortion)
    if rolling_shutter is not None:
        if gaussians.xyz.dtype != torch.float32:
            raise TypeError("rolling_shutter needs fp32 inputs (the fused rasterizer's per-gaussian stages apply it)")
        if gaussians.sh is not None and not use_sh_precompute:
            raise ValueError("rolling_shutter needs use_sh_precompute=True (per-pixel SH colours are not supported)")
    shutter = _shutter_arg(rolling_shutter, readout, camera.K, _lens_input(fisheye, distortion), gaussians.xyz.device,
                           int(camera.height), int(camera.width))
    if lens is not None:
        if gaussians.xyz.dtype != torch.float32:
            raise TypeError(f"{lens[0]} needs fp32 inputs (the fused rasterizer's per-gaussian stages project through "
                            "it)")
        if gaussians.sh is not None and not use_sh_precompute:
            raise ValueError(f"{lens[0]} needs use_sh_precompute=True (per-pixel SH colours are not supported)")
    if features is not None:
        if not torch.is_tensor(features):
            raise TypeError("features must be a torch tensor [N, D]")
        if gaussians.xyz.dtype != torch.float32:
            raise TypeError("features needs fp32 inputs (the fused rasterizer's tile kernels blend them)")
        if gaussians.sh is not None and not use_sh_precompute:
            raise ValueError("features needs use_sh_precompute=True (per-pixel SH colours are not supported)")
        if features.dtype != torch.float32:
            raise TypeError(f"features must be float32, got {features.dtype}")
        n = gaussians.xyz.shape[0]
        if features.dim() != 2 or features.shape[0] != n or features.shape[1] < 1:
            raise ValueError(f"features has shape {tuple(features.shape)} but must be [{n}, D] with D >= 1 (one row "
                             "per gaussian)")
        if features.device != gaussians.xyz.device or not features.is_contiguous():
            raise ValueError("features must be contiguous and on the gaussians' device")
        if absgrad:
            raise ValueError("absgrad with features is not supported: the per-pixel |d loss / d uv| cannot be "
                             "split across the colour and the feature kernels")
    if weight_stats is not None:
        if gaussians.xyz.dtype != torch.float32:
            raise TypeError("weight_stats needs fp32 inputs (the fused rasterizer's render forward accumulates them)")
        if gaussians.sh is not None and not use_sh_precompute:
            raise ValueError("weight_stats needs use_sh_precompute=True (per-pixel SH colours are not supported)")
        n = gaussians.xyz.shape[0]
        fields = (weight_stats.weight_sum, weight_stats.weight_max, weight_stats.pixel_count)
        if any(tuple(f.shape) != (n,) for f in fields):
            raise ValueError(f"weight_stats holds {tuple(fields[0].shape)} rows but there are {n} gaussians: make a new "
                             "WeightStats after densification changes the gaussians")
        for f, dt in zip(fields, (torch.float32, torch.float32, torch.int32)):
            if f.dtype != dt:
                raise TypeError(f"weight_stats fields must be float32, float32, int32; got {f.dtype}")
            if f.device != gaussians.xyz.device or not f.is_contiguous():
                raise ValueError("weight_stats fields must be contiguous and on the gaussians' device")
    if filter3d is not None:
        if gaussians.xyz.dtype != torch.float32:
            raise TypeError("filter3d needs fp32 inputs (the fused rasterizer's per-gaussian stages apply it)")
        if gaussians.sh is not None and not use_sh_precompute:
            raise ValueError("filter3d needs use_sh_precompute=True (per-pixel SH colours are not supported)")
        if filter3d.requires_grad:
            raise ValueError("filter3d is a constant of the scene (no gradient flows to it): pass filter3d.detach()")
        if filter3d.dtype != torch.float32:
            raise TypeError(f"filter3d must be float32, got {filter3d.dtype}")
        n = gaussians.xyz.shape[0]
        if not (tuple(filter3d.shape) in ((n,), (n, 1))):
            raise ValueError(f"filter3d has shape {tuple(filter3d.shape)} but there are {n} gaussians: recompute it "
                             "(compute_filter3d) after densification changes the gaussians")
    if absgrad and gaussians.xyz.dtype != torch.float32:
        raise TypeError("absgrad needs fp32 inputs (the fused rasterizer's render backward forms it)")
    if absgrad and gaussians.sh is not None and not use_sh_precompute:
        raise ValueError("absgrad needs use_sh_precompute=True (per-pixel SH colours are not supported)")
    if antialiased and gaussians.xyz.dtype != torch.float32:
        raise TypeError("antialiased needs fp32 inputs (the fp64 renderer applies no dilation to compensate)")
    if antialiased and gaussians.sh is not None and not use_sh_precompute:
        raise ValueError("antialiased needs use_sh_precompute=True (per-pixel SH colours are not supported)")
    if render_depth_alpha and gaussians.sh is not None and not use_sh_precompute:
        raise ValueError("render_depth_alpha needs use_sh_precompute=True (per-pixel SH colours are not supported)")
    if gaussians.sh is not None and not use_sh_precompute:
        return rasterize_unfused(gaussians, camera_T_world, camera, near_thresh, far_thresh,
                                 cull_mask_padding, mh_dist, use_sh_precompute, background_rgb)
    if gaussians.xyz.dtype != torch.float32:
        raise TypeError("the fused rasterizer is fp32; use rasterize_unfused for float64 inputs")
    ext = native()
    state = _ViewState(profile)
    state.grad_out = grad_out
    state.mode = ((ext.MODE_DEPTH_ALPHA if render_depth_alpha else 0) | (ext.MODE_ANTIALIASED if antialiased else 0)
                  | (ext.MODE_ABSGRAD if absgrad else 0) | (ext.MODE_FILTER3D if filter3d is not None else 0))
    state.filter3d = None if filter3d is None else filter3d.reshape(-1).contiguous()
    state.lens = _lens_state(lens, gaussians.xyz.device)
    state.shutter = shutter
    state.weight_stats = weight_stats
    state.background = background_rgb.contiguous()
    cfg = (int(camera.height), int(camera.width), float(near_thresh), float(far_thresh),
           float(cull_mask_padding), float(mh_dist))
    uv, carrier = _ProjectGaussians.apply(
        gaussians.xyz.contiguous(), gaussians.quaternion.contiguous(), gaussians.scale.contiguous(),
        gaussians.opacity.contiguous(), gaussians.rgb.contiguous(),
        None if gaussians.sh is None else gaussians.sh.contiguous(),
        camera_T_world.contiguous(), camera.K.contiguous(), state, cfg, _lens_input(fisheye, distortion),
        rolling_shutter if shutter is not None and rolling_shutter.requires_grad else None)
    state.uv_ref = weakref.ref(uv)
    culling_mask = state.visible == 0
    outs = _CompositeTiles.apply(uv, carrier, state.background, state, features)
    image, maps = (outs[0], outs[1:]) if isinstance(outs, tuple) else (outs, ())
    result = (image, culling_mask, uv, *maps)
    return (*result, state) if return_state else result


def project_and_bin(gaussians, camera_T_world, camera, near_thresh, far_thresh, cull_mask_padding, mh_dist):
    """The per-gaussian part of the reference chain, one native op per reference op (any dtype):
    transform -> pinhole -> frustum cull -> Sigma_world / J / conic -> tile binning.  Returns a namespace with
    culling_mask [N] and, for the survivors, uv, xyz_cam, xyz, opacity (post-sigmoid), rgb, sh, conic,
    sorted_idx, tile_ranges."""
    from types import SimpleNamespace

    xyz_cam = transform_points_torch(gaussians.xyz, camera_T_world)
    uv = CameraPointProjection.apply(xyz_cam, camera.K)
    z, pad = xyz_cam[:, 2], cull_mask_padding
    culling_mask = (
        (z < near_thresh) | (z > far_thresh)
        | (uv[:, 0] < -1 * pad) | (uv[:, 0] > camera.width + pad)
        | (uv[:, 1] < -1 * pad) | (uv[:, 1] > camera.height + pad)
    )
    keep = ~culling_mask
    s = SimpleNamespace(culling_mask=culling_mask, uv=uv[keep, :], xyz_cam=xyz_cam[keep, :], xyz=gaussians.xyz[keep, :],
                        opacity=torch.sigmoid(gaussians.opacity[keep]), rgb=gaussians.rgb[keep, :],
                        sh=None if gaussians.sh is None else gaussians.sh[keep, :])
    sigma_world = ComputeSigmaWorld.apply(gaussians.quaternion[keep, :], gaussians.scale[keep, :])
    J = ComputeProjectionJacobian.apply(s.xyz_cam, camera.K)
    s.conic = ComputeConic.apply(sigma_world, J, camera_T_world)
    tiles = Tiles(camera.height, camera.width, uv.device)
    s.sorted_idx, s.tile_ranges = get_splats(s.uv.detach(), tiles, s.conic.detach(), s.xyz_cam.detach(), mh_dist)
    return s


def rasterize_unfused(gaussians, camera_T_world, camera, near_thresh, far_thresh, cull_mask_padding, mh_dist,
                      use_sh_precompute, background_rgb):
    """Operator-by-operator evaluation (any dtype, either SH mode); same return triple as rasterize()."""
    s = project_and_bin(gaussians, camera_T_world, camera, near_thresh, far_thresh, cull_mask_padding, mh_dist)
    rays = torch.zeros(1, 1, 1, dtype=gaussians.xyz.dtype, device=gaussians.xyz.device)  # unused unless per-pixel SH
    if s.sh is None:
        render_rgb = s.rgb
    else:
        coeffs = torch.cat((s.rgb.unsqueeze(dim=2), s.sh), dim=2)
        if use_sh_precompute:
            render_rgb = PrecomputeRGBFromSH.apply(coeffs, s.xyz, torch.inverse(camera_T_world).contiguous())
        else:
            render_rgb, rays = coeffs, compute_rays_in_world_frame(camera, camera_T_world)
    image = RenderImage.apply(render_rgb, s.opacity, s.uv, s.conic, rays, s.tile_ranges, s.sorted_idx,
                              (camera.height, camera.width), background_rgb)
    return image, s.culling_mask, s.uv


# ---- multi-view: C cameras of one scene in one call ------------------------------------------------------------------
class _BatchView:
    """What one view of a rasterize_batch call exposes (state.views[c]): the fields DensificationStats.accumulate
    reads (vis_idx32, uv_absgrad, N, M) and the view's pair list."""

    __slots__ = ("N", "M", "P", "vis_idx", "vis_idx32", "uv_absgrad", "ranges", "keys_sorted", "_ids_sorted", "id_bits",
                 "n_per_pixel", "w_per_pixel", "masks")

    ids_sorted = _ViewState.ids_sorted

    def __init__(self):
        self.uv_absgrad = None


class _BatchState:
    """Non-differentiable buffers of a rasterize_batch call shared by its two autograd nodes; per-view arrays are
    stacked view-major ([C, N, ...])."""

    def __init__(self, profile=None):
        self.profile = profile
        self.grad_flat = None    # set by the backward pass: the gradient summed over the views (flat layout)
        self.grad_out = None
        self.uv_refs = None      # weak references to the C uv tensors handed to the caller
        self.uv_grad_emitted = False
        self.speculation_overflowed = False
        self.mode = 0
        self.filter3d = None
        self.lens = None         # a lens model: (its LENS_* value, [C, n+1] constants on the device) (_lens_state)
        self.shutter = None      # a rolling shutter: (the views' twists [C,6] on the device, a READOUT_* value)
        self.views = []
        self.images = self.depth = self.alpha = None


class _ProjectBatch(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, quaternion, scale, opacity, rgb, sh, camera_T_world, K, state, cfg, lens_k=None, xi=None):
        camera_T_world = camera_T_world.detach()  # as in _ProjectGaussians.forward
        ext = native()
        H, W, near, far, pad, mh = cfg
        C, N = camera_T_world.shape[0], xyz.shape[0]
        depth_base, depth_bits = _depth_key_params(near, far)
        opacity_flat = opacity.reshape(-1)
        # per view exactly the camera-frame positions and camera centre rasterize() forms (DESIGN.md 4)
        if IN_KERNEL_TRANSFORM and N >= IN_KERNEL_TRANSFORM_MIN_N and in_kernel_transform_ok(xyz.device):
            tails = [tail_positions(xyz, camera_T_world[c]) for c in range(C)]
            xyz_cam = None if tails[0] is None else torch.stack(tails)
        else:
            xyz_cam = torch.stack([transform_points_torch(xyz, camera_T_world[c]) for c in range(C)])
        centre = None
        if sh is not None:
            if native_centre_ok(xyz.device):
                centre = torch.stack([ext.camera_centre(camera_T_world[c]) for c in range(C)])
            else:
                centre = torch.stack([torch.linalg.inv_ex(camera_T_world[c])[0][:3, 3] for c in range(C)])
        with _stage(state, "preprocess_fwd"):
            records, zkey, visible, scan, tile_mask, tile_win = ext.batch_preprocess_forward(
                xyz, xyz_cam, quaternion, scale, opacity_flat, rgb, sh, camera_T_world, K, centre, H, W, near, far, pad,
                mh, depth_base, state.mode, state.filter3d, **_lens_kwargs(state.lens), **_shutter_kwargs(state.shutter))
        record_masks = USE_CONTRIBUTION_MASKS and (any(ctx.needs_input_grad[:8]) or any(ctx.needs_input_grad[10:]))
        background = state.background
        depth_mode = bool(state.mode & ext.MODE_DEPTH_ALPHA)

        def counts(totals):
            Ms, Ps = [t >> 32 for t in totals], [t & 0xFFFFFFFF for t in totals]
            # the native entry points index pairs with int32: the batch's pairs, over all views, must stay below 2^31
            if any(m > N for m in Ms) or sum(Ps) >= 2**31:
                raise RuntimeError(f"rasterize_batch: {sum(Ps)} (gaussian, tile) pairs over {C} views exceed the int32 "
                                   "pair index of the native path (the batch's P must be < 2^31)")
            return Ms, Ps

        def bin_and_render(c, M_, P_, speculative):
            with _stage(state, "bin_sort_gather"):
                binned = ext.fused_bin(records[c], zkey[c], visible[c], scan[c], M_, P_, H, W, mh, depth_bits,
                                       speculative, tile_mask[c] if USE_TILE_MASKS else None,
                                       tile_win[c] if USE_TILE_MASKS else None)
            with _stage(state, "render_fwd"):
                rendered = ext.fused_render_forward(records[c], binned[1], background[c], H, W, P_, record_masks,
                                                    binned[4], binned[0], binned[5], zkey[c] if depth_mode else None,
                                                    depth_base, depth_bits)
            return binned, rendered

        # One host read for the whole batch: every view's pair buffers are sized from the recent views of this
        # (N, H, W, C) and enqueued, and only then the C (M, P) totals, copied together to pinned memory on a side
        # stream right behind the scans, are read (DESIGN.md 3.5 and 3.18).  Views that overflowed their guess run
        # again with exact sizes.
        key = (xyz.device.index, N, H, W, C)
        cap = _pair_capacity(key) if (SPECULATIVE_BINNING and N > 0) else None
        out = [None] * C
        if N == 0:
            Ms, Ps = [0] * C, [0] * C
            out = [bin_and_render(c, 0, 0, False) for c in range(C)]
        elif cap is None:
            Ms, Ps = counts(scan[:, -1].tolist())
            out = [bin_and_render(c, Ms[c], Ps[c], False) for c in range(C)]
        else:
            totals = scan[:, -1].contiguous()
            slot = torch.empty(C, dtype=torch.int64, pin_memory=True)
            side = _side_stream(xyz.device)
            scanned = torch.cuda.Event()
            scanned.record()
            with torch.cuda.stream(side):
                side.wait_event(scanned)
                slot.copy_(totals, non_blocking=True)
                ready = torch.cuda.Event()
                ready.record(side)
            totals.record_stream(side)
            out = [bin_and_render(c, N, cap, True) for c in range(C)]
            ready.synchronize()
            Ms, Ps = counts(slot.tolist())
            for c in range(C):
                if Ps[c] > cap:
                    out[c] = bin_and_render(c, Ms[c], Ps[c], False)
                    state.speculation_overflowed = True
                else:
                    (ids_c, ranges_c, vis_c, uv_c, keys_c, idb), rendered = out[c]
                    out[c] = ((ids_c.narrow(0, 0, Ps[c]) if ids_c.numel() else ids_c, ranges_c,
                               vis_c.narrow(0, 0, Ms[c]), uv_c.narrow(0, 0, Ms[c]), keys_c, idb),
                              _fit_masks(ext, rendered, Ps[c], H, W))
        for P_ in Ps:
            _note_pairs(key, P_)
        views, uvs = [], []
        for c in range(C):
            (ids_sorted, ranges, vis_idx, uv, keys_sorted, id_bits), rendered = out[c]
            v = _BatchView()
            v.N, v.M, v.P = N, Ms[c], Ps[c]
            v.vis_idx = v.vis_idx32 = vis_idx
            v._ids_sorted, v.ranges, v.keys_sorted, v.id_bits = ids_sorted, ranges, keys_sorted, int(id_bits)
            _, v.n_per_pixel, v.w_per_pixel, v.masks, _, _ = rendered
            views.append(v)
            uvs.append(uv)
        state.images = torch.stack([o[1][0] for o in out])
        if depth_mode:
            state.depth = torch.stack([o[1][4] for o in out])
            state.alpha = torch.stack([o[1][5] for o in out])
        state.views, state.C, state.N, state.H, state.W = views, C, N, H, W
        state.records, state.zkey, state.visible, state.scan = records, zkey, visible, scan
        state.depth_base, state.depth_bits = depth_base, depth_bits
        uv_all = torch.cat(uvs) if C > 1 else uvs[0].contiguous()
        carrier = torch.empty(C * 12 * N, dtype=xyz.dtype, device=xyz.device)
        ctx.state = state
        ctx.has_sh = sh is not None
        ctx.lens_k = lens_k
        ctx.xi_shape = None if xi is None else tuple(xi.shape)
        ctx.save_for_backward(xyz, quaternion, scale, opacity_flat, sh, camera_T_world, K, centre)
        return uv_all, carrier

    @staticmethod
    def backward(ctx, grad_uv, grad_carrier):
        xyz, quaternion, scale, opacity_flat, sh, camera_T_world, K, centre = ctx.saved_tensors
        st = ctx.state
        C, N = st.C, st.N
        if grad_carrier is None:
            grad_carrier = torch.zeros(C * 12 * N, dtype=xyz.dtype, device=xyz.device)
        slab = grad_carrier.contiguous()
        # as in _ProjectGaussians.backward: the uv gradient is either only what the caller added on the uvs (added to
        # the rows' uv sums) or the total (it replaces them); view c's rows of the compact uv follow views 0..c-1
        guv = None
        if grad_uv is not None and grad_uv.shape[0] > 0:
            guv = grad_uv.contiguous()
        with _stage(st, "preprocess_bwd"):
            args = (slab, xyz, quaternion, scale, opacity_flat, sh, camera_T_world, K, centre, st.visible, st.grad_out,
                    guv, st.scan if guv is not None else None, not st.uv_grad_emitted, st.mode, st.filter3d)
            grads, g_pose, g_K, g_k, g_xi = _preprocess_backward(ctx, native().batch_preprocess_backward, args)
        g_xyz, g_q, g_s, g_o, g_dc = grads[:5]
        g_sh = grads[5] if ctx.has_sh else None
        st.grad_flat = grads[-1]
        return g_xyz, g_q, g_s, g_o.view(-1, 1), g_dc, g_sh, g_pose, g_K, None, None, g_k, g_xi


class _CompositeBatch(torch.autograd.Function):
    """carrier, uv_0 .. uv_{C-1} -> images [C,H,W,3], or (images, depth, alpha) [C,H,W,1] each.  The per-view uvs
    (views of the projection node's compact uv) are the inputs, so that their .grad is the render pass's gradient."""

    @staticmethod
    def forward(ctx, carrier, background_rgb, state, *uvs):
        outs = (state.images,) if state.depth is None else (state.images, state.depth, state.alpha)
        state.images = state.depth = state.alpha = None
        ctx.state = state
        return outs if len(outs) > 1 else outs[0]

    @staticmethod
    def backward(ctx, grad_images, *grad_maps):
        ext = native()
        st = ctx.state
        grad_depth = grad_alpha = None
        if st.mode & ext.MODE_DEPTH_ALPHA:
            grad_depth, grad_alpha = grad_maps[:2]
        vs = st.views
        empty = torch.empty(0, dtype=torch.int64, device=grad_images.device)
        with _stage(st, "render_bwd"):
            slab = ext.batch_render_backward(
                grad_images.contiguous(), st.N, [v.P for v in vs], st.records,
                [v._ids_sorted for v in vs], [v.keys_sorted if v.keys_sorted is not None else empty for v in vs],
                [v.id_bits for v in vs], [v.ranges for v in vs], st.background, [v.n_per_pixel for v in vs],
                [v.w_per_pixel for v in vs], [v.masks for v in vs],
                None if grad_depth is None else grad_depth.contiguous(),
                None if grad_alpha is None else grad_alpha.contiguous(), st.zkey, st.depth_base, st.depth_bits,
                st.mode)
        rows = slab.view(st.C, st.N, 12)
        uvs = [r() for r in st.uv_refs] if st.uv_refs is not None else [None] * st.C
        if st.mode & ext.MODE_ABSGRAD:
            for c, v in enumerate(vs):
                v.uv_absgrad = rows[c][:, 10:12].index_select(0, v.vis_idx)
                if uvs[c] is not None:
                    uvs[c].absgrad = v.uv_absgrad
        watched = any(u is None or u.retains_grad or bool(u._backward_hooks) for u in uvs)
        st.uv_grad_emitted = bool(watched)
        if not watched:
            return (slab.view(-1), None, None) + (None,) * st.C
        return (slab.view(-1), None, None) + tuple(rows[c].index_select(0, v.vis_idx)[:, 4:6].contiguous()
                                                   for c, v in enumerate(vs))


def _check_batch_args(gaussians, camera_T_world, camera, use_sh_precompute, background_rgb, filter3d, weight_stats,
                      features):
    xyz = gaussians.xyz
    if weight_stats is not None:
        raise ValueError("weight_stats is not supported by rasterize_batch: use rasterize per view")
    if features is not None:
        raise ValueError("features is not supported by rasterize_batch: use rasterize per view")
    if gaussians.sh is not None and not use_sh_precompute:
        raise ValueError("rasterize_batch needs use_sh_precompute=True (per-pixel SH colours are not supported)")
    if xyz.dtype != torch.float32:
        raise TypeError("rasterize_batch is fp32 (the fused rasterizer); use rasterize_unfused per view for float64")
    if not torch.is_tensor(camera_T_world) or camera_T_world.dim() != 3 or tuple(camera_T_world.shape[1:]) != (4, 4) \
            or camera_T_world.shape[0] < 1:
        raise ValueError("camera_T_world must be a [C,4,4] tensor with C >= 1")
    C = camera_T_world.shape[0]
    K = camera.K
    if not torch.is_tensor(K) or tuple(K.shape) not in ((3, 3), (C, 3, 3)):
        raise ValueError(f"camera.K must be [3,3] or [{C},3,3]")
    if not torch.is_tensor(background_rgb) or tuple(background_rgb.shape) not in ((3,), (C, 3)):
        raise ValueError(f"background_rgb must be [3] or [{C},3]")
    for name, t in (("camera_T_world", camera_T_world), ("camera.K", K), ("background_rgb", background_rgb)):
        if t.dtype != torch.float32:
            raise TypeError(f"{name} must be float32, got {t.dtype}")
        if t.device != xyz.device:
            raise ValueError(f"{name} must be on the gaussians' device")
    if filter3d is not None:
        if filter3d.requires_grad:
            raise ValueError("filter3d is a constant of the scene (no gradient flows to it): pass filter3d.detach()")
        if filter3d.dtype != torch.float32:
            raise TypeError(f"filter3d must be float32, got {filter3d.dtype}")
        n = xyz.shape[0]
        if not (tuple(filter3d.shape) in ((n,), (n, 1))):
            raise ValueError(f"filter3d has shape {tuple(filter3d.shape)} but there are {n} gaussians: recompute it "
                             "(compute_filter3d) after densification changes the gaussians")
    return C


def rasterize_batch(gaussians, camera_T_world, camera, near_thresh, far_thresh, cull_mask_padding, mh_dist,
                    use_sh_precompute, background_rgb, return_state=False, profile=None, grad_out=None,
                    render_depth_alpha=False, antialiased=False, absgrad=False, filter3d=None, weight_stats=None,
                    features=None, fisheye=None, distortion=None, rolling_shutter=None, readout="top_to_bottom"):
    """C cameras of one scene in one call: rasterize()'s nine positional arguments with camera_T_world [C,4,4]
    (C >= 1), camera.K [3,3] (shared) or [C,3,3], camera.height / width shared, background_rgb [3] or [C,3].

    Returns (images [C,H,W,3], culling_mask [C,N] bool, uvs[, depth [C,H,W,1], alpha [C,H,W,1]][, state]).  uvs is a
    tuple of C tensors [M_c,2], views of one compact tensor in view order; uvs[c].retain_grad() gives uvs[c].grad
    after backward, and with absgrad=True uvs[c].absgrad is set, as rasterize() does for its uv.

    Forward: view c is bit-identical to rasterize(gaussians, camera_T_world[c], K_c, ..., background_c) with the same
    flags (image, mask, uv, depth / alpha): every view gets exactly the single-view camera-frame positions, camera
    centre, depth keys, pair list and tile kernels.  Backward: one gradient for the batch, the sum over the views of
    each view's parameter gradient, added per gaussian in view order in fp32 (g = g_0; g += g_1; ...), which is what
    autograd's accumulation over C rasterize() calls gives for the same render-stage rows.  The per-gaussian backward
    reads the parameters once and writes the gradient once for all views (libgsr_batch.so, DESIGN.md 3.18).  filter3d
    gets no gradient.  A camera_T_world that requires grad gets one gradient per view [C,4,4], as rasterize() defines
    it; view c's is bit-identical to the single-view kernel's on view c's rows (DESIGN.md 3.21).

    state (return_state=True): state.views[c] has vis_idx32, uv_absgrad, N and M, so that
    DensificationStats.accumulate(state.views[c], uvs[c], xyz, K_c) works per view; state.grad_flat (or grad_out, a
    caller-owned buffer of the flat layout) holds the batch's one gradient.

    Supports render_depth_alpha, antialiased, absgrad, filter3d ([N], one filter for all views), return_state,
    profile and grad_out.  weight_stats and features raise ValueError (use rasterize per view), fp64 inputs
    TypeError, per-pixel SH (use_sh_precompute=False) ValueError, and so do poses, K or backgrounds of the wrong
    shape (ValueError), dtype (TypeError) or device (ValueError).

    fisheye: OPENCV_FISHEYE cameras as in rasterize(), k [4] shared by every view or [C,4] one row per view (host
    values: a sequence or a CPU tensor); view c is then bit-identical to rasterize(..., fisheye=k_c).  distortion:
    radial-tangential cameras likewise, k [5] or [C,5] (rasterize(..., distortion=k_c)).

    A camera.K that requires grad gets d loss / d K as rasterize() defines it, [C,3,3] per view (a shared [3,3]: the sum
    over the views), and a CPU coefficient tensor that requires grad its gradient in its shape ([n]: summed over the
    views); view c's values are bit-identical to the single-view kernel's on view c's rows (DESIGN.md 3.23).

    rolling_shutter: rolling-shutter cameras as in rasterize(), xi [6] shared by every view or [C,6] one row per view,
    with one readout for all views; view c is bit-identical to rasterize(..., rolling_shutter=xi_c).  A shared [6] that
    requires grad gets the views' summed gradient, a [C,6] one row per view (DESIGN.md 3.24)."""
    C = _check_batch_args(gaussians, camera_T_world, camera, use_sh_precompute, background_rgb, filter3d, weight_stats,
                          features)
    lens = _lens_arg(fisheye, distortion, C)
    shutter = _shutter_arg(rolling_shutter, readout, camera.K, _lens_input(fisheye, distortion), gaussians.xyz.device,
                           int(camera.height), int(camera.width), C)
    ext = native()
    K = camera.K if camera.K.dim() == 3 else camera.K.expand(C, 3, 3)
    state = _BatchState(profile)
    state.grad_out = grad_out
    state.mode = ((ext.MODE_DEPTH_ALPHA if render_depth_alpha else 0) | (ext.MODE_ANTIALIASED if antialiased else 0)
                  | (ext.MODE_ABSGRAD if absgrad else 0) | (ext.MODE_FILTER3D if filter3d is not None else 0))
    state.filter3d = None if filter3d is None else filter3d.reshape(-1).contiguous()
    state.lens = _lens_state(lens, gaussians.xyz.device)
    state.shutter = shutter
    state.background = (background_rgb if background_rgb.dim() == 2 else background_rgb.expand(C, 3)).contiguous()
    cfg = (int(camera.height), int(camera.width), float(near_thresh), float(far_thresh),
           float(cull_mask_padding), float(mh_dist))
    uv_all, carrier = _ProjectBatch.apply(
        gaussians.xyz.contiguous(), gaussians.quaternion.contiguous(), gaussians.scale.contiguous(),
        gaussians.opacity.contiguous(), gaussians.rgb.contiguous(),
        None if gaussians.sh is None else gaussians.sh.contiguous(),
        camera_T_world.contiguous(), K.contiguous(), state, cfg, _lens_input(fisheye, distortion),
        rolling_shutter if shutter is not None and rolling_shutter.requires_grad else None)
    uvs = torch.split(uv_all, [v.M for v in state.views])
    state.uv_refs = [weakref.ref(u) for u in uvs]
    culling_mask = state.visible == 0
    outs = _CompositeBatch.apply(carrier, state.background, state, *uvs)
    images, maps = (outs[0], outs[1:]) if isinstance(outs, tuple) else (outs, ())
    result = (images, culling_mask, uvs, *maps)
    return (*result, state) if return_state else result
