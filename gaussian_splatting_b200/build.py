"""In-tree build of the native code (no JIT cache: the .so files ship with the tree).

  libgsr_b200.so            CUDA kernels + C ABI (include/gsr_b200.h), nvcc, sm_90a only, no torch
  _ext/splat_cuda.*.so      torch binding exporting the reference's `splat_cuda` surface

`python -m gaussian_splatting_b200.build` builds both; `build(force=False)` is incremental.
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
    "gsr_binning.cu",
    "gsr_render.cu",
    "gsr_render_generic.cu",
    "gsr_adam.cu",
    "gsr_densify.cu",
    "gsr_loss.cu",
]
HEADERS = [
    CSRC / "gsr_common.cuh",
    CSRC / "gsr_math.cuh",
    CSRC / "gsr_math_bwd.cuh",
    CSRC / "gsr_record.cuh",
    CSRC / "gsr_f32x2.cuh",
    ROOT / "include" / "gsr_b200.h",
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


def build_lib(force: bool = False, verbose: bool = False) -> Path:
    OBJ.mkdir(exist_ok=True)
    stamp = OBJ / "lib.sha256"
    want = _digest([CSRC / s for s in CU_SOURCES] + HEADERS, " ".join(NVCC_FLAGS))
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == want:
        return LIB

    def compile_one(src):
        obj = OBJ / (Path(src).stem + ".o")
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", str(CSRC / src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        out = _run(cmd)
        if verbose:
            print(out)
        return obj

    with ThreadPoolExecutor(max_workers=min(len(CU_SOURCES), os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, CU_SOURCES))
    _run([_nvcc(), "-shared", "-o", str(LIB), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a",
          "-cudart", "shared"])
    stamp.write_text(want)
    return LIB


def build_ext(force: bool = False) -> Path:
    import torch  # noqa: F401  (needed for include/library paths)
    from torch.utils import cpp_extension as ce

    OBJ.mkdir(exist_ok=True)
    EXT_DIR.mkdir(exist_ok=True)
    out = ext_path()
    src = CSRC / "splat_cuda_module.cpp"
    stamp = OBJ / "ext.sha256"
    want = _digest([src, ROOT / "include" / "gsr_b200.h"], torch.__version__)
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
        f"-L{PKG}", "-lgsr_b200", f"-L{torch_lib}", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10",
        "-lc10_cuda", "-ltorch_python", f"-L{cuda_lib}", "-lcudart",
        "-Wl,-rpath,$ORIGIN/..", f"-Wl,-rpath,{torch_lib}", f"-Wl,-rpath,{cuda_lib}",
    ]
    _run(cmd)
    stamp.write_text(want)
    return out


def build(force: bool = False, verbose: bool = False):
    lib = build_lib(force=force, verbose=verbose)
    ext = build_ext(force=force)
    return lib, ext


if __name__ == "__main__":
    lib, ext = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(lib)
    print(ext)
