"""H100-native (sm_90a) differentiable Gaussian-splat rasterizer.

Drop-in for the rasterization path of joeyan/gaussian_splatting:

  * ``gaussian_splatting_b200.splat_cuda``  — native module exporting the 14 callables of the
    reference's ``splat_cuda`` extension (src/bindings.cpp:118-159) on top of the C ABI in
    ``include/gsr_b200.h``; ``install_as_splat_cuda()`` registers it under that name so the
    reference's own ``splat_py`` package runs on it unmodified.
  * ``gaussian_splatting_b200.rasterize.rasterize`` — same signature and return values as
    ``splat_py.rasterize.rasterize`` (splat_py/rasterize.py:18-112), fused implementation.
  * ``gaussian_splatting_b200.rasterize_batch`` — C cameras of one scene in one fused forward and backward.
  * ``gaussian_splatting_b200.appearance`` — per-image bilateral grids (appearance correction) on native kernels.
  * ``gaussian_splatting_b200.calib`` — ``IntrinsicsDelta``, camera self-calibration with the fused path's K gradient.
  * ``cuda_autograd_functions`` / ``tile_culling`` / ``structs`` / ``utils`` / ``depth`` — host-side
    mirror of the reference modules of the same names.

There is no CPU fallback: importing the native module fails loudly when it has not been built
(``python -m gaussian_splatting_b200.build``), and every operator requires CUDA tensors.
"""
from __future__ import annotations

import importlib.util
import sys
from pathlib import Path

_PKG = Path(__file__).resolve().parent
_native = None


def native():
    """The compiled `splat_cuda` module (loads libgsr_b200.so through its rpath)."""
    global _native
    if _native is None:
        import torch  # noqa: F401  (libtorch must be loaded before the extension)
        from .build import ext_path

        path = ext_path()
        if not path.exists() or not all((_PKG / lib).exists() for lib in ("libgsr_b200.so", "libgsr_selective_adam.so",
                                                                    "libgsr_features.so", "libgsr_batch.so")):
            raise ImportError(
                f"gaussian_splatting_b200 native code is not built ({path} missing); "
                "run `python -m gaussian_splatting_b200.build` (needs nvcc, sm_90a)"
            )
        spec = importlib.util.spec_from_file_location("splat_cuda", str(path))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _native = mod
    return _native


def install_as_splat_cuda():
    """Make `import splat_cuda` resolve to this library (the reference's module name)."""
    sys.modules["splat_cuda"] = native()
    return sys.modules["splat_cuda"]


def __getattr__(name):
    if name == "splat_cuda":
        return native()
    if name == "rasterize_batch":
        from .rasterize import rasterize_batch

        return rasterize_batch
    raise AttributeError(name)


__version__ = "0.1.0"
