"""The drop-in boundary without a GPU: the C-ABI library loads and exports every symbol declared in
include/gsr_b200.h; the torch binding exports the reference's 14 callables
(src/bindings.cpp:118-159); argument errors surface as RuntimeError like the reference's TORCH_CHECKs;
the product package never touches the oracle."""
import ctypes
import re
from pathlib import Path

import pytest
import torch

import gaussian_splatting_b200 as g

ROOT = Path(__file__).resolve().parent.parent

REFERENCE_SURFACE = [
    "render_tiles_cuda", "render_tiles_backward_cuda", "camera_projection_cuda",
    "camera_projection_backward_cuda", "compute_sigma_world_cuda", "compute_sigma_world_backward_cuda",
    "compute_projection_jacobian_cuda", "compute_projection_jacobian_backward_cuda", "compute_conic_cuda",
    "compute_conic_backward_cuda", "get_sorted_gaussian_list", "precompute_rgb_from_sh_cuda",
    "precompute_rgb_from_sh_backward_cuda", "render_depth_cuda",
]


def declared_symbols():
    text = (ROOT / "include" / "gsr_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(gsr_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_the_path():
    syms = declared_symbols()
    assert len(syms) >= 25
    for must in ("gsr_preprocess_forward", "gsr_sort_pairs", "gsr_render_forward_gather", "gsr_render_backward_gather",
                 "gsr_preprocess_backward", "gsr_binning_emit_sort"):
        assert must in syms


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(str(ROOT / "gaussian_splatting_b200" / "libgsr_b200.so"))
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"declared in gsr_b200.h but not exported: {missing}"
    lib.gsr_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.gsr_version()


def test_library_is_sm90a_only_and_has_tma():
    import subprocess

    so = ROOT / "gaussian_splatting_b200" / "libgsr_b200.so"
    elfs = subprocess.run(["cuobjdump", "-lelf", str(so)], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", elfs))
    assert archs == {"90a"}, archs
    names = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True).stdout
    fwd = re.findall(r"Function : (\S*16k_preprocess_fwdILi16ELb1\S*)", names)  # SH degree 3
    assert fwd, "k_preprocess_fwd<16, true> not in the library"
    sass = subprocess.run(["cuobjdump", "-sass", "-fun", fwd[0], str(so)], capture_output=True, text=True).stdout
    assert "UBLKCP" in sass, "per-gaussian forward kernel should stage through TMA bulk copies (UBLKCP)"


def test_binding_exports_reference_surface():
    ext = g.native()
    for name in REFERENCE_SURFACE:
        assert callable(getattr(ext, name)), name
    assert g.install_as_splat_cuda() is ext
    import splat_cuda  # noqa: F401  (resolves to this library now)

    assert splat_cuda is ext


def test_argument_errors_are_runtime_errors():
    ext = g.native()
    xyz, K, uv = torch.zeros(4, 3), torch.eye(3), torch.zeros(4, 2)
    with pytest.raises(RuntimeError, match="not a CUDA tensor"):  # src/checks.cuh:5
        ext.camera_projection_cuda(xyz, K, uv)
    with pytest.raises(RuntimeError):
        ext.get_sorted_gaussian_list(1024, uv, xyz, torch.zeros(4, 3), 4, 4, 3.0)


def test_product_does_not_import_the_oracle():
    pkg = ROOT / "gaussian_splatting_b200"
    for p in list(pkg.glob("*.py")) + list((pkg / "csrc").glob("*")):
        text = p.read_text(errors="ignore")
        assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), p
        assert "gsr_oracle" not in text and "oracle/" not in text.replace("oracle/_ref", ""), p


def test_no_cpu_fallback():
    """CPU tensors are rejected, never silently computed on the host."""
    from gaussian_splatting_b200 import synth
    from gaussian_splatting_b200.rasterize import rasterize

    gs = synth.make_gaussians(16, "tiny", sh_degree=0)
    cam = synth.make_camera("tiny")
    with pytest.raises(RuntimeError):
        rasterize(gs, synth.make_pose(), cam, 0.3, 500.0, 100, 3.0, True, torch.zeros(3))
