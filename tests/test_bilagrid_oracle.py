"""The bilateral-grid slice without a GPU: the fp64 oracle against torch's grid_sample, the host validation of
appearance.py, and the built library (symbols, sm_90a, no local memory, the other libraries' SASS unchanged)."""
import ctypes as C
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import bilagrid_oracle as bo

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "gaussian_splatting_b200"
LIB = PKG / "libgsr_bilagrid.so"

# (N, L, GY, GX, C, H, W): the default grid, and odd sizes with an odd image
SIZES = [(2, 8, 16, 16, 1, 24, 40), (3, 3, 4, 6, 2, 37, 53), (2, 2, 2, 2, 2, 5, 7)]


def _inputs(N, L, GY, GX, C, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    grids = torch.randn(N, 12, L, GY, GX, generator=g, dtype=torch.float64)
    # luminances inside and outside [0, 1]
    rgb = torch.rand(C, H, W, 3, generator=g, dtype=torch.float64) * 1.4 - 0.2
    ids = [(2 * c + 1) % N for c in range(C)]
    return grids, rgb, ids


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "x".join(map(str, s)))
def test_oracle_forward_matches_grid_sample(size):
    grids, rgb, ids = _inputs(*size)
    lum = rgb.numpy() @ bo.LUMA
    assert (lum < 0).any() and (lum > 1).any() and ((lum > 0) & (lum < 1)).any()
    ref = bo.grid_sample_slice(grids, rgb, ids).numpy()
    out = bo.slice_forward(grids.numpy(), rgb.numpy(), ids)
    assert np.abs(out - ref).max() < 1e-12


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "x".join(map(str, s)))
def test_oracle_gradients_match_grid_sample_autograd(size):
    grids, rgb, ids = _inputs(*size, seed=1)
    g_out = torch.randn(rgb.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
    gr, rr = grids.clone().requires_grad_(), rgb.clone().requires_grad_()
    bo.grid_sample_slice(gr, rr, ids).backward(g_out)
    d_rgb, d_grids = bo.slice_backward(grids.numpy(), rgb.numpy(), ids, g_out.numpy())
    assert np.abs(d_rgb - rr.grad.numpy()).max() < 1e-12
    assert np.abs(d_grids - gr.grad.numpy()).max() < 1e-12


class _OracleSlice(torch.autograd.Function):
    """the numpy oracle as an autograd function, so gradcheck compares its analytic gradients to finite differences"""

    @staticmethod
    def forward(ctx, grids, rgb, ids):
        ctx.save_for_backward(grids, rgb)
        ctx.ids = ids
        return torch.from_numpy(bo.slice_forward(grids.numpy(), rgb.numpy(), ids))

    @staticmethod
    def backward(ctx, g):
        grids, rgb = ctx.saved_tensors
        d_rgb, d_grids = bo.slice_backward(grids.numpy(), rgb.numpy(), ctx.ids, g.numpy())
        return torch.from_numpy(d_grids), torch.from_numpy(d_rgb), None


def test_oracle_passes_gradcheck():
    grids, rgb, ids = _inputs(3, 3, 4, 6, 2, 37, 53, seed=2)
    ids = [2, 2]  # a shared grid: its gradient is the sum over both views
    gr, rr = grids.requires_grad_(), rgb.requires_grad_()
    assert torch.autograd.gradcheck(lambda a, b: _OracleSlice.apply(a, b, ids), (gr, rr), eps=1e-6, atol=1e-6,
                                    rtol=1e-5, fast_mode=True)


def test_oracle_identity_grid_returns_the_input():
    from gaussian_splatting_b200.appearance import identity_grids

    rgb = np.random.default_rng(0).uniform(-0.2, 1.2, (2, 9, 11, 3))
    out = bo.slice_forward(identity_grids(2, 5, 4, 3).double().numpy(), rgb, [1, 0])
    assert np.abs(out - rgb).max() < 1e-15


def test_total_variation_expression():
    g = torch.randn(2, 12, 3, 4, 5, dtype=torch.float64)
    tv = sum(float(((g.narrow(d, 1, g.shape[d] - 1) - g.narrow(d, 0, g.shape[d] - 1)) ** 2).mean()) for d in (2, 3, 4))
    assert abs(float(bo.total_variation(g)) - tv) < 1e-12


# ---- host validation: every error is raised before any launch, without a GPU --------------------------------------
def _cuda_like(t):
    """a stand-in the checks see as a CUDA tensor; the validation must raise before anything touches it"""

    class Fake(torch.Tensor):
        @property
        def is_cuda(self):
            return True

        @property
        def device(self):
            return torch.device("cuda:0")

    return t.as_subclass(Fake)


def _good():
    from gaussian_splatting_b200.appearance import identity_grids

    return _cuda_like(identity_grids(4, 4, 4, 3)), _cuda_like(torch.rand(2, 6, 8, 3))


@pytest.mark.parametrize("case", ["cuda_ids", "out_of_range", "negative", "count", "float_ids", "bool_ids"])
def test_bad_ids_raise_value_error(case):
    from gaussian_splatting_b200.appearance import bilateral_slice

    grids, image = _good()
    ids = {"cuda_ids": _cuda_like(torch.tensor([0, 1])), "out_of_range": [0, 4], "negative": [-1, 0],
           "count": [0, 1, 2], "float_ids": [0.0, 1.0], "bool_ids": torch.tensor([True, False])}[case]
    with pytest.raises(ValueError):
        bilateral_slice(grids, image, ids)


def test_single_image_takes_an_int_and_counts_one_id():
    from gaussian_splatting_b200.appearance import bilateral_slice

    grids, image = _good()
    with pytest.raises(ValueError, match="expected 1"):
        bilateral_slice(grids, image[0], [0, 1])
    with pytest.raises(ValueError, match="out of range"):
        bilateral_slice(grids, image[0], 7)


@pytest.mark.parametrize("case", ["fp64_image", "fp16_grids", "int_image"])
def test_non_fp32_inputs_raise_type_error(case):
    from gaussian_splatting_b200.appearance import bilateral_slice

    grids, image = _good()
    if case == "fp64_image":
        image = _cuda_like(torch.rand(2, 6, 8, 3, dtype=torch.float64))
    elif case == "fp16_grids":
        grids = _cuda_like(grids.half())
    else:
        image = _cuda_like(torch.zeros(2, 6, 8, 3, dtype=torch.int32))
    with pytest.raises(TypeError):
        bilateral_slice(grids, image, [0, 1])


@pytest.mark.parametrize("which", ["image", "grids"])
def test_cpu_tensors_raise_value_error(which):
    from gaussian_splatting_b200.appearance import bilateral_slice, identity_grids, total_variation

    grids, image = _good()
    if which == "image":
        image = torch.rand(2, 6, 8, 3)
    else:
        grids = identity_grids(4, 4, 4, 3)
        with pytest.raises(ValueError):
            total_variation(grids)
    with pytest.raises(ValueError):
        bilateral_slice(grids, image, [0, 1])


@pytest.mark.parametrize("shape", [(2, 6, 8, 4), (6, 8, 1), (6, 8), (1, 2, 6, 8, 3)])
def test_bad_image_shapes_raise_value_error(shape):
    from gaussian_splatting_b200.appearance import bilateral_slice

    grids, _ = _good()
    with pytest.raises(ValueError):
        bilateral_slice(grids, _cuda_like(torch.rand(shape)), [0, 1])


@pytest.mark.parametrize("shape", [(4, 12, 1, 4, 4), (4, 12, 3, 1, 4), (4, 12, 3, 4, 1), (4, 11, 3, 4, 4),
                                   (0, 12, 3, 4, 4), (12, 3, 4, 4), (1, 12, 257, 2, 2)])
def test_bad_grid_shapes_raise_value_error(shape):
    from gaussian_splatting_b200.appearance import BilateralGrid, bilateral_slice, total_variation

    _, image = _good()
    grids = _cuda_like(torch.zeros(shape))
    with pytest.raises(ValueError):
        bilateral_slice(grids, image, [0, 0])
    with pytest.raises(ValueError):
        total_variation(grids)
    with pytest.raises(ValueError):
        BilateralGrid(3, grid_x=1)


def test_bilateral_grid_module_is_identity_initialised():
    from gaussian_splatting_b200.appearance import BilateralGrid

    m = BilateralGrid(3, grid_x=5, grid_y=4, grid_guidance=6)
    assert isinstance(m.grids, torch.nn.Parameter) and m.grids.shape == (3, 12, 6, 4, 5)
    A = m.grids.detach().permute(0, 2, 3, 4, 1).reshape(-1, 3, 4)
    assert torch.equal(A, torch.cat([torch.eye(3), torch.zeros(3, 1)], 1).expand_as(A))
    torch.optim.Adam([{"params": m.parameters(), "lr": 2e-3}])


# ---- the library -----------------------------------------------------------------------------------------------------
def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists():
        pytest.skip(f"{name} is not available")
    return exe


def _cuobjdump(*args, lib=LIB):
    if not lib.exists():
        pytest.skip("the built library is missing")
    return subprocess.run([_tool("cuobjdump"), *args, str(lib)], check=True, capture_output=True, text=True).stdout


def test_header_symbols_are_all_exported():
    header = (ROOT / "include" / "gsr_bilagrid.h").read_text()
    declared = set(re.findall(r"^\w[\w\s\*]*?\b(gsr_\w+)\s*\(", header, re.M))
    assert declared == {"gsr_bilagrid_slice_forward", "gsr_bilagrid_slice_backward_temp_bytes",
                        "gsr_bilagrid_slice_backward", "gsr_bilagrid_tv_temp_bytes", "gsr_bilagrid_tv_forward",
                        "gsr_bilagrid_tv_backward"}, declared
    if not LIB.exists():
        pytest.skip("libgsr_bilagrid.so is not built")
    lib = C.CDLL(str(LIB))
    for name in declared:
        assert hasattr(lib, name), name
    nm = subprocess.run(["nm", "-D", "--defined-only", str(LIB)], capture_output=True, text=True).stdout
    assert set(re.findall(r"\bT (gsr_\w+)", nm)) == declared
    # argument errors are reported without touching the device
    lib.gsr_bilagrid_slice_forward.argtypes = [C.c_int] * 3 + [C.c_void_p] * 3 + [C.c_int] * 4 + [C.c_void_p] * 3
    strides = (C.c_int64 * 4)(0, 0, 0, 0)
    assert lib.gsr_bilagrid_slice_forward(1, 4, 4, 8, strides, 8, 1, 1, 2, 2, 8, 8, None) == -1  # L < 2
    assert lib.gsr_bilagrid_slice_forward(1, 4, 4, None, strides, 8, 1, 2, 2, 2, 8, 8, None) == -1  # no rgb
    lib.gsr_bilagrid_slice_backward_temp_bytes.restype = C.c_size_t
    assert lib.gsr_bilagrid_slice_backward_temp_bytes(1, 0, 8, 16, 16) == 0


def test_kernels_are_sm90a_and_use_no_local_memory():
    elfs = _cuobjdump("--list-elf")
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage")))
    kinds = ["k_bilagrid_sliceILb0", "k_bilagrid_sliceILb1", "k_bilagrid_grid_grad", "k_bilagrid_grid_grad_finish",
             "k_bilagrid_tv_fwd", "k_bilagrid_tv_bwd"]
    assert len(usage) == len(kinds), sorted(usage)
    for kind in kinds:
        names = [k for k in usage if re.search(rf"\d{kind}(?!_)", k)]
        assert len(names) == 1, (kind, names)
        u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[names[0]])}
        assert u["LOCAL"] == 0 and u["STACK"] == 0, (kind, u)


def test_existing_kernels_keep_their_sass():
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_bilagrid.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    libs = ("libgsr_b200.so", "libgsr_selective_adam.so", "libgsr_features.so", "libgsr_batch.so",
            "libgsr_fisheye.so", "libgsr_distortion.so", "libgsr_pose.so")
    assert set(rec) - {"nvcc"} == set(libs)
    for lib in libs:
        if not (PKG / lib).exists():
            pytest.skip(f"{lib} is not built")
        now = {k: d for k, (d, n) in sass_digest.per_kernel(PKG / lib).items()}
        assert set(now) == set(rec[lib]), lib
        changed = sorted(k for k, d in rec[lib].items() if now[k] != d)
        assert not changed, (lib, changed)
        assert "bilagrid" not in "".join(now)
