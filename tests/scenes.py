"""Shared scene builders for the tests (numpy views of gaussian_splatting_b200.synth scenes and the
reference's 6-gaussian fixture, test/gaussian_test_data.py:7-79, restated), and the digest / row sample that
stored reference outputs are compared through (tools/make_golden.py writes them, tests/test_parity_gpu.py reads)."""
import hashlib

import numpy as np
import torch

from gaussian_splatting_b200 import synth

SH0 = 0.28209479177387814


def np_scene(n, res, sh_degree=3, seed=0, view=0, n_views=3, dtype=np.float32, sigma_px=(1.2, 0.6, 0.3, 12.0)):
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    g = synth.make_gaussians(n, res, sh_degree=sh_degree, seed=seed, dtype=tdt, sigma_px=sigma_px)
    cam = synth.make_camera(res, dtype=tdt)
    T = synth.make_pose(view, n_views, dtype=tdt)
    a = lambda t: None if t is None else t.detach().numpy()  # noqa: E731
    return dict(xyz=a(g.xyz), quaternion=a(g.quaternion), scale=a(g.scale), opacity=a(g.opacity), rgb=a(g.rgb),
                sh=a(g.sh), T=a(T), K=a(cam.K), H=cam.height, W=cam.width)


def sh12_scene(sh_degree):
    """20 000 gaussians at SH degree 1 or 2, 320x192: the scenes of tests/golden/sh12_reference.npz."""
    return np_scene(20_000, "small", sh_degree=sh_degree, seed=20 + sh_degree, view=1, n_views=3,
                    sigma_px=(2.5, 0.5, 0.5, 10.0))


def reference_fixture(dtype=np.float32):
    """The reference's own unit-test scene: 6 gaussians, 640x480 camera, tilted pose."""
    xyz = np.array([[1, 2, -4], [4, 5, 6], [7, 8, -9], [1, 2, 15], [2.5, -1, 4], [-1, -2, 10]], dtype)
    rgb = np.full((6, 3), 0.5, dtype)
    rgb[3], rgb[4], rgb[5] = [0.5, 0, 0], [0, 0.5, 0], [0, 0, 0.5]
    rgb = (rgb / dtype(SH0)).astype(dtype)
    opacity = np.ones((6, 1), dtype)
    scale = np.log(np.array([[0.02, 0.03, 0.04], [0.01, 0.05, 0.02], [0.09, 0.03, 0.01], [1, 3, 0.1], [2, 0.2, 0.1],
                             [2, 1, 0.1]], dtype))
    quaternion = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [1, 0, 0, 0], [0.714, -0.002, -0.664, 0.221],
                           [1, 0, 0, 0]], dtype)
    K = np.array([[430, 0, 320], [0, 410, 240], [0, 0, 1]], dtype)
    T = np.array([[0.9999, 0.0089, 0.0073, -0.3283], [-0.0106, 0.9568, 0.2905, -1.9260],
                  [-0.0044, -0.2906, 0.9568, 2.9581], [0, 0, 0, 1]], dtype)
    return dict(xyz=xyz, quaternion=quaternion, scale=scale, opacity=opacity, rgb=rgb, sh=None, T=T, K=K, H=480, W=640)


def inverse_sigmoid(x):
    p = np.clip(x, 1e-4, 1 - 1e-4)
    return np.log(p / (1 - p)).astype(x.dtype)


def digest(a):
    """sha256 of an array's dtype, shape and bytes: a bit-for-bit comparison against a stored reference output."""
    a = np.ascontiguousarray(a.detach().cpu().numpy() if torch.is_tensor(a) else a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def sample_rows(n, k=64, seed=0):
    """Fixed, seeded row sample of an [n, ...] output (sorted indices)."""
    return np.sort(np.random.default_rng(seed).choice(n, size=min(k, n), replace=False))


def general_pose():
    """A pose with roll, pitch and translation (the bench's ring only yaws)."""
    c, s = np.cos(0.3), np.sin(0.3)
    R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], np.float64) @ np.array([[1, 0, 0], [0, 0.995, -0.0998], [0, 0.0998, 0.995]])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, [0.13, -0.21, 0.37]
    return T.astype(np.float32)


def exact_arithmetic_scene(n_exact=300, n_huge=12, H=64, W=64):
    """Splats whose centre falls EXACTLY on a pixel centre and splats whose 2-D covariance determinant exceeds 1e18.

    The tile renderers recompute a flagged pixel with the exact arithmetic (gsr_render.cu render_fwd): a listed
    record with |det| outside [1e-18, 1e18] flags its whole warp, an exact centre (Mahalanobis numerator 0) the
    pixels of its lane.  The n_huge splats are ~1800 world units wide at z = 2 with opacity sigmoid(-3) ~ 0.047:
    those near the axis reach det ~ 1e19 px^4 and every pixel, those off the axis project to needles; together they
    flag about two thirds of the 64 x 64 frame's warps and contribute to every pixel.  H x W other than 64 x 64: the
    principal point stays an integer (W // 2, H // 2), so the exact centres still land on pixel centres."""
    rng = np.random.default_rng(7)
    sc = np_scene(3000, "tiny", sh_degree=0, seed=3, sigma_px=(2.0, 0.5, 0.5, 8.0))
    cx, cy = W // 2, H // 2
    # powers of two: u = 64*x/z + cx is exact
    sc["K"] = np.array([[64, 0, cx], [0, 64, cy], [0, 0, 1]], np.float32)
    sc["T"] = np.eye(4, dtype=np.float32)
    sc["H"], sc["W"] = H, W
    z = np.full(n_exact, 2.0, np.float32)
    px, py = rng.integers(0, W, n_exact), rng.integers(0, H, n_exact)
    sc["xyz"][:n_exact] = np.stack([(px - cx) / 64.0 * z, (py - cy) / 64.0 * z, z], 1).astype(np.float32)
    sc["xyz"][n_exact:n_exact + n_huge, 2] = 2.0
    sc["scale"][n_exact:n_exact + n_huge] = 7.5       # exp(7.5) = 1808 world units -> det(Sigma_2D) ~ 1e19
    sc["opacity"][n_exact:n_exact + n_huge] = -3.0
    return sc


# Scenes whose pixels the tile renderers recompute with the exact arithmetic: "huge" flags whole warps (huge splats)
# plus exact centres, "scattered" only the pixels at exact centres (n_huge = 0), in the same warps as pixels the walk
# computes; the 37 x 61 variants add an odd width (a lane's second pixel outside the image) and partial edge tiles.
FLAGGED = {"exact huge": dict(), "exact scattered": dict(n_huge=0),
           "exact huge 37x61": dict(H=37, W=61), "exact scattered 37x61": dict(n_huge=0, H=37, W=61)}


def flagged_scene(name):
    return exact_arithmetic_scene(**FLAGGED[name])


def headline_inputs(H, device):
    """3M gaussians, SH 3, 1920 x H, pose 2 of 8, and a seeded upstream gradient."""
    from gaussian_splatting_b200.structs import Camera

    g = synth.make_gaussians(3_000_000, "1080p", sh_degree=3, seed=0, device=device, requires_grad=True)
    cam0 = synth.make_camera("1080p", device=device)
    T = synth.make_pose(2, 8, device=device)
    gen = torch.Generator().manual_seed(1)
    G = (torch.randn(H, 1920, 3, generator=gen, dtype=torch.float64) / (3.0 * H * 1920)).float().to(device)
    return g, Camera(1920, H, cam0.K), T, G
