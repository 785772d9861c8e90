"""In-tree build of the native code (no JIT cache: the .so files ship with the tree).

  libgsr_b200.so            CUDA kernels + C ABI (include/gsr_b200.h), nvcc, sm_90a only, no torch
  libgsr_selective_adam.so  the visibility-masked Adam step (include/gsr_selective_adam.h), same flags
  libgsr_features.so        the feature-channel tile kernels (include/gsr_features.h), same flags
  libgsr_batch.so           the multi-view per-gaussian kernels of rasterize_batch (include/gsr_batch.h), same flags
  libgsr_fisheye.so         the per-gaussian kernels for fisheye cameras (include/gsr_fisheye.h), same flags
  libgsr_distortion.so      the per-gaussian kernels for radial-tangential lens distortion (include/gsr_distortion.h);
                            both built from gsr_lens.cu, once per lens
  libgsr_pose.so            the per-gaussian backward with the camera pose gradient, every lens (include/gsr_pose.h)
  libgsr_calib.so           the same sources compiled with the pose, intrinsics and lens-coefficient gradients
                            (include/gsr_calib.h)
  libgsr_shutter.so         the per-gaussian stages for rolling-shutter cameras, every lens, with the pose and
                            readout-motion gradients (include/gsr_shutter.h)
  libgsr_bilagrid.so        bilateral-grid appearance correction: slice forward / backward, total variation
                            (include/gsr_bilagrid.h)
  libgsr_surfels.so         2-D Gaussian surfels: per-gaussian and tile kernels of rasterize_surfels
                            (include/gsr_surfels.h)
  libgsr_surfels_lens.so    the same through fisheye and radial-tangential lenses, with the ray-map kernel
                            (include/gsr_surfels_lens.h)
  libgsr_surfels_features.so  per-gaussian feature channels blended with the surfel colour's weights, every lens
                            (include/gsr_surfels_features.h)
  libgsr_surfels_median.so  the median depth of the surfel blend, every lens (include/gsr_surfels_median.h)
  _ext/splat_cuda.*.so      torch binding exporting the reference's `splat_cuda` surface

`python -m gaussian_splatting_b200.build` builds all fifteen (the CUDA libraries from the LIBS table);
`build(force=False)` is incremental.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / "csrc"
OBJ = PKG / "_build"
EXT_DIR = PKG / "_ext"
LIB = PKG / "libgsr_b200.so"

CU_SOURCES = [
    "gsr_pergaussian.cu",
    "gsr_preprocess.cu",
    "gsr_filter3d.cu",
    "gsr_binning.cu",
    "gsr_render.cu",
    "gsr_render_generic.cu",
    "gsr_adam.cu",
    "gsr_densify.cu",
    "gsr_mcmc.cu",
    "gsr_loss.cu",
]
HEADERS = [
    CSRC / "gsr_common.cuh",
    CSRC / "gsr_math.cuh",
    CSRC / "gsr_math_bwd.cuh",
    CSRC / "gsr_record.cuh",
    CSRC / "gsr_f32x2.cuh",
    CSRC / "gsr_tile_walk.cuh",
    CSRC / "gsr_preprocess.cuh",
    ROOT / "include" / "gsr_b200.h",
]
CUH = [h for h in HEADERS if h.suffix == ".cuh"]
# The sources of a library are file names, or (file name, object stem, extra nvcc flags) for a file compiled more
# than once.  gsr_lens.cu is compiled once per lens model (GSR_LENS: 1 fisheye, 2 distortion), gsr_pose.cu once per
# camera model (GSR_POSE_LENS: 0 pinhole, 1 fisheye, 2 distortion), and again with GSR_POSE_CAMERA for libgsr_calib.so
# (the camera-gradient kernels); gsr_shutter.cu once per camera model (GSR_SHUTTER_LENS).
LENS_HEADERS = CUH + [CSRC / "gsr_fisheye.cuh", CSRC / "gsr_distortion.cuh", CSRC / "gsr_poly_roots.h",
                      ROOT / "include" / "gsr_b200.h", ROOT / "include" / "gsr_fisheye.h",
                      ROOT / "include" / "gsr_distortion.h"]
POSE_HEADERS = CUH + [CSRC / "gsr_pose.cuh", CSRC / "gsr_calib.cuh", CSRC / "gsr_fisheye.cuh",
                      CSRC / "gsr_distortion.cuh", ROOT / "include" / "gsr_b200.h", ROOT / "include" / "gsr_fisheye.h",
                      ROOT / "include" / "gsr_distortion.h", ROOT / "include" / "gsr_pose.h",
                      ROOT / "include" / "gsr_calib.h"]
# the surfel kernels' bodies (gsr_surfels.cuh) are shared by the pinhole and the lens library
SURFEL_HEADERS = CUH + [CSRC / "gsr_surfels.cuh", CSRC / "gsr_surfels_lens.cuh", CSRC / "gsr_fisheye.cuh",
                        CSRC / "gsr_distortion.cuh", ROOT / "include" / "gsr_b200.h", ROOT / "include" / "gsr_surfels.h",
                        ROOT / "include" / "gsr_surfels_lens.h"]
# (library, sources, headers, stamp): each library apart, so that every library keeps exactly its kernels (and their
# SASS) when another one changes
LIBS = [
    (LIB, CU_SOURCES, HEADERS, "lib.sha256"),
    (PKG / "libgsr_selective_adam.so", ["gsr_adam_selective.cu"],
     [CSRC / "gsr_common.cuh", ROOT / "include" / "gsr_b200.h", ROOT / "include" / "gsr_selective_adam.h"],
     "selective_lib.sha256"),
    (PKG / "libgsr_features.so", ["gsr_features.cu"],
     CUH + [ROOT / "include" / "gsr_b200.h", ROOT / "include" / "gsr_features.h"], "features_lib.sha256"),
    (PKG / "libgsr_batch.so", ["gsr_batch.cu"],
     CUH + [ROOT / "include" / "gsr_b200.h", ROOT / "include" / "gsr_batch.h"], "batch_lib.sha256"),
    (PKG / "libgsr_fisheye.so", [("gsr_lens.cu", "gsr_fisheye", ["-DGSR_LENS=1"])], LENS_HEADERS,
     "fisheye_lib.sha256"),
    (PKG / "libgsr_distortion.so", [("gsr_lens.cu", "gsr_distortion", ["-DGSR_LENS=2"])], LENS_HEADERS,
     "distortion_lib.sha256"),
    (PKG / "libgsr_pose.so", [("gsr_pose.cu", f"gsr_pose_{i}", [f"-DGSR_POSE_LENS={i}"]) for i in range(3)],
     POSE_HEADERS, "pose_lib.sha256"),
    (PKG / "libgsr_calib.so",
     [("gsr_pose.cu", f"gsr_camera_{i}", [f"-DGSR_POSE_LENS={i}", "-DGSR_POSE_CAMERA"]) for i in range(3)],
     POSE_HEADERS, "calib_lib.sha256"),
    (PKG / "libgsr_shutter.so", [("gsr_shutter.cu", f"gsr_shutter_{i}", [f"-DGSR_SHUTTER_LENS={i}"]) for i in range(3)],
     POSE_HEADERS + [CSRC / "gsr_shutter.cuh", ROOT / "include" / "gsr_shutter.h"], "shutter_lib.sha256"),
    (PKG / "libgsr_bilagrid.so", ["gsr_bilagrid.cu"],
     [CSRC / "gsr_common.cuh", ROOT / "include" / "gsr_b200.h", ROOT / "include" / "gsr_bilagrid.h"],
     "bilagrid_lib.sha256"),
    (PKG / "libgsr_surfels.so", ["gsr_surfels.cu"], SURFEL_HEADERS, "surfels_lib.sha256"),
    (PKG / "libgsr_surfels_lens.so", ["gsr_surfels_lens.cu"],
     SURFEL_HEADERS + [ROOT / "include" / "gsr_fisheye.h", ROOT / "include" / "gsr_distortion.h"],
     "surfels_lens_lib.sha256"),
    (PKG / "libgsr_surfels_features.so", ["gsr_surfels_features.cu"],
     SURFEL_HEADERS + [ROOT / "include" / "gsr_surfels_features.h"], "surfels_features_lib.sha256"),
    (PKG / "libgsr_surfels_median.so", ["gsr_surfels_median.cu"],
     SURFEL_HEADERS + [ROOT / "include" / "gsr_surfels_median.h"], "surfels_median_lib.sha256"),
]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    cand = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else "nvcc"


def _digest(paths, extra="") -> str:
    h = hashlib.sha256(extra.encode())
    for p in paths:
        h.update(Path(p).read_bytes())
    return h.hexdigest()


def _run(cmd):
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        sys.stderr.write(" ".join(map(str, cmd)) + "\n" + proc.stdout + proc.stderr)
        raise RuntimeError(f"build step failed: {cmd[0]}")
    return proc.stdout + proc.stderr


def ext_path() -> Path:
    suffix = sysconfig.get_config_var("EXT_SUFFIX")
    return EXT_DIR / f"splat_cuda{suffix}"


def _build_cuda_lib(lib: Path, sources, headers, stamp_name: str, force: bool, verbose: bool) -> Path:
    """sources: file names, or (file name, object stem, extra nvcc flags) for a file compiled more than once."""
    OBJ.mkdir(exist_ok=True)
    stamp = OBJ / stamp_name
    units = [s if isinstance(s, tuple) else (s, Path(s).stem, []) for s in sources]
    want = _digest(sorted({CSRC / s for s, _, _ in units}) + headers,
                   " ".join(NVCC_FLAGS + [f for _, _, fl in units for f in fl]))
    if not force and lib.exists() and stamp.exists() and stamp.read_text() == want:
        return lib

    def compile_one(unit):
        src, stem, flags = unit
        obj = OBJ / (stem + ".o")
        cmd = [_nvcc(), *NVCC_FLAGS, *flags, "-c", str(CSRC / src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        out = _run(cmd)
        if verbose:
            print(out)
        return obj

    with ThreadPoolExecutor(max_workers=min(len(sources), os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, units))
    _run([_nvcc(), "-shared", "-o", str(lib), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a",
          "-cudart", "shared"])
    stamp.write_text(want)
    return lib


def build_ext(force: bool = False) -> Path:
    import torch  # noqa: F401  (needed for include/library paths)
    from torch.utils import cpp_extension as ce

    OBJ.mkdir(exist_ok=True)
    EXT_DIR.mkdir(exist_ok=True)
    out = ext_path()
    src = CSRC / "splat_cuda_module.cpp"
    stamp = OBJ / "ext.sha256"
    want = _digest([src, ROOT / "include" / "gsr_b200.h", ROOT / "include" / "gsr_selective_adam.h",
                    ROOT / "include" / "gsr_features.h", ROOT / "include" / "gsr_batch.h",
                    ROOT / "include" / "gsr_fisheye.h", ROOT / "include" / "gsr_distortion.h",
                    ROOT / "include" / "gsr_pose.h", ROOT / "include" / "gsr_bilagrid.h",
                    ROOT / "include" / "gsr_calib.h", ROOT / "include" / "gsr_shutter.h",
                    ROOT / "include" / "gsr_surfels.h", ROOT / "include" / "gsr_surfels_lens.h",
                    ROOT / "include" / "gsr_surfels_features.h", ROOT / "include" / "gsr_surfels_median.h"],
                   torch.__version__)
    if not force and out.exists() and stamp.exists() and stamp.read_text() == want:
        return out
    incs = [f"-I{p}" for p in ce.include_paths("cuda")] + [f"-I{sysconfig.get_paths()['include']}"]
    torch_lib = Path(torch.__file__).parent / "lib"
    cuda_lib = Path(ce.CUDA_HOME or "/usr/local/cuda") / "lib64"
    cmd = [
        "g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden",
        "-DTORCH_EXTENSION_NAME=splat_cuda", "-DTORCH_API_INCLUDE_EXTENSION_H",
        f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}",
        *incs, str(src), "-o", str(out),
        f"-L{PKG}", "-lgsr_b200", "-lgsr_selective_adam", "-lgsr_features", "-lgsr_batch", "-lgsr_fisheye",
        "-lgsr_distortion", "-lgsr_pose", "-lgsr_bilagrid", "-lgsr_calib", "-lgsr_shutter", "-lgsr_surfels",
        "-lgsr_surfels_lens", "-lgsr_surfels_features", "-lgsr_surfels_median",
        f"-L{torch_lib}", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10",
        "-lc10_cuda", "-ltorch_python", f"-L{cuda_lib}", "-lcudart",
        "-Wl,-rpath,$ORIGIN/..", f"-Wl,-rpath,{torch_lib}", f"-Wl,-rpath,{cuda_lib}",
    ]
    _run(cmd)
    stamp.write_text(want)
    return out


def build_render_variant(out_dir, flags) -> Path:
    """The tile renderers alone (gsr_render.cu: the gsr_render_* entry points of the C ABI) compiled with extra -D
    flags into out_dir/libgsr_render_variant.so, for A/B checks of compile-time alternatives (not used by the
    package; out_dir should lie outside the tree)."""
    out = Path(out_dir) / "libgsr_render_variant.so"
    _run([_nvcc(), *NVCC_FLAGS, *flags, "-shared", "-cudart", "shared", str(CSRC / "gsr_render.cu"), "-o", str(out)])
    return out


def build(force: bool = False, verbose: bool = False):
    for lib, sources, headers, stamp in LIBS:
        _build_cuda_lib(lib, sources, headers, stamp, force, verbose)
    ext = build_ext(force=force)
    return LIB, ext


if __name__ == "__main__":
    lib, ext = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(lib)
    print(ext)
