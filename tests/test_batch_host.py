"""rasterize_batch without a GPU: argument errors of the Python entry point and of the C entry point through ctypes,
the kernels of libgsr_batch.so, and the single-view kernels of libgsr_b200.so left as they were."""
import ctypes as C
import json
import re
import shutil
import subprocess
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
BATCH_LIB = ROOT / "gaussian_splatting_b200" / "libgsr_batch.so"
MAIN_LIB = ROOT / "gaussian_splatting_b200" / "libgsr_b200.so"
BAD_ARG = -1


# ---- rasterize_batch argument errors ----------------------------------------------------------------------------------
def _gaussians(n=4, dtype=torch.float32, sh=None):
    from gaussian_splatting_b200.structs import Gaussians

    return Gaussians(torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 1, dtype=dtype),
                     torch.zeros(n, 3, dtype=dtype), torch.zeros(n, 4, dtype=dtype), sh)


def _call(g=None, T=None, K=None, bg=None, **kw):
    from gaussian_splatting_b200 import rasterize_batch
    from gaussian_splatting_b200.structs import Camera

    g = _gaussians() if g is None else g
    dt = g.xyz.dtype
    T = torch.eye(4, dtype=dt).expand(2, 4, 4) if T is None else T
    K = torch.eye(3, dtype=dt) if K is None else K
    bg = torch.zeros(3, dtype=dt) if bg is None else bg
    return rasterize_batch(g, T, Camera(64, 64, K), 0.3, 500.0, 100, 3.0, kw.pop("use_sh_precompute", True), bg, **kw)


def test_rasterize_batch_argument_errors():
    with pytest.raises(ValueError):
        _call(T=torch.zeros(0, 4, 4))                          # C < 1
    with pytest.raises(ValueError):
        _call(T=torch.eye(4))                                  # not [C,4,4]
    with pytest.raises(ValueError):
        _call(T=torch.zeros(2, 3, 4))
    with pytest.raises(TypeError):
        _call(T=torch.zeros(2, 4, 4, dtype=torch.float64))     # pose dtype
    with pytest.raises(ValueError):
        _call(T=torch.zeros(2, 4, 4, device="meta"))           # pose device
    with pytest.raises(ValueError):
        _call(K=torch.eye(3).expand(3, 3, 3))                  # K of another C
    with pytest.raises(ValueError):
        _call(K=torch.eye(4))
    with pytest.raises(TypeError):
        _call(K=torch.eye(3, dtype=torch.float64))
    with pytest.raises(ValueError):
        _call(bg=torch.zeros(3, 3))                            # background of another C
    with pytest.raises(ValueError):
        _call(bg=torch.zeros(4))
    with pytest.raises(TypeError):
        _call(bg=torch.zeros(2, 3, dtype=torch.float64))
    with pytest.raises(ValueError):
        _call(bg=torch.zeros(2, 3, device="meta"))
    with pytest.raises(ValueError):
        _call(weight_stats=object())                           # out of scope in a batch
    with pytest.raises(ValueError):
        _call(features=torch.zeros(4, 3))
    with pytest.raises(TypeError):
        _call(_gaussians(dtype=torch.float64))                 # fp64
    with pytest.raises(ValueError):
        _call(_gaussians(sh=torch.zeros(4, 3, 3)), use_sh_precompute=False)
    with pytest.raises(ValueError):
        _call(filter3d=torch.zeros(5))                         # filter of another N
    with pytest.raises(ValueError):
        _call(filter3d=torch.zeros(4, requires_grad=True))
    with pytest.raises(TypeError):
        _call(filter3d=torch.zeros(4, dtype=torch.float64))


# ---- the C entry point ------------------------------------------------------------------------------------------------
def _batch_lib():
    if not BATCH_LIB.exists():
        pytest.skip("libgsr_batch.so is not built")
    return C.CDLL(str(BATCH_LIB))


def test_c_entry_point_rejects_bad_arguments_before_any_launch():
    """Pointers are never dereferenced on the host: every call below fails its checks before a launch, so fake
    (16-byte aligned) device addresses are enough."""
    fn = _batch_lib().gsr_batch_preprocess_backward
    fn.restype = C.c_int
    P = C.c_void_p
    dev, mis = P(0x10000), P(0x10004)

    def call(mode=0, Cv=2, N=100, n_rest=3, xyz=dev, quat=dev, scale=dev, opa=dev, f3d=None, T=dev, K=dev, cam=None,
             vis=dev, rows=dev, rows_uv=1, guv=None, scan=None, o_xyz=dev, o_q=dev, o_s=dev, o_o=dev, o_dc=dev,
             o_sh=dev):
        return fn(C.c_int(mode), C.c_int(Cv), C.c_int(N), C.c_int(n_rest), xyz, quat, scale, opa, f3d, T, K, cam, vis,
                  rows, C.c_int(rows_uv), guv, scan, o_xyz, o_q, o_s, o_o, o_dc, o_sh, None)

    for kw in (dict(Cv=0), dict(Cv=-1), dict(N=-1), dict(mode=16), dict(mode=8), dict(f3d=dev), dict(xyz=None),
               dict(quat=None), dict(scale=None), dict(opa=None), dict(T=None), dict(K=None), dict(vis=None),
               dict(rows=None), dict(rows=mis), dict(guv=dev), dict(o_xyz=None), dict(o_q=None), dict(o_s=None),
               dict(o_o=None), dict(o_dc=None), dict(o_sh=None), dict(n_rest=0)):
        assert call(**kw) == BAD_ARG, kw
    assert call(N=0) == 0                    # nothing to do, nothing launched
    assert call(N=0, Cv=0) == BAD_ARG


# ---- the libraries ----------------------------------------------------------------------------------------------------
def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists():
        pytest.skip(f"{name} is missing")
    return exe


def _cuobjdump(*args, lib=BATCH_LIB):
    if not lib.exists():
        pytest.skip("the built library is missing")
    return subprocess.run([_tool("cuobjdump"), *args, str(lib)], check=True, capture_output=True, text=True).stdout


def test_batch_kernels_are_sm90a_and_keep_nothing_in_local_memory():
    elfs = _cuobjdump("--list-elf")
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    text = _cuobjdump("-sass")
    bodies = {n.strip(): b for n, b in (f.split("\n", 1) for f in re.split(r"\n\s+Function : ", text)[1:])}
    assert len(bodies) == 32 and all("k_batch_preprocess_bwd" in n for n in bodies), sorted(bodies)
    for name, body in bodies.items():
        assert not re.search(r"\b(?:STL|LDL)\b", body), name
        assert re.search(r"\bUBLKCP\b", body), name   # the bulk stores of the single-view kernel
    usage = re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage"))
    assert len(usage) == 32
    for name, line in usage:
        u = {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
        assert u["STACK"] == 0 and u["LOCAL"] == 0 and u["REG"] <= 128, (name, u)


def test_batch_library_exports_every_symbol_its_header_declares():
    header = (ROOT / "include" / "gsr_batch.h").read_text()
    declared = set(re.findall(r"^\w[\w\s\*]*?\b(gsr_\w+)\s*\(", header, re.M))
    assert declared == {"gsr_batch_preprocess_backward"}, declared
    lib = _batch_lib()
    for name in declared:
        assert hasattr(lib, name), name


def test_main_library_keeps_the_sass_of_every_kernel_recorded_before_the_batch():
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    if not MAIN_LIB.exists():
        pytest.skip("libgsr_b200.so is not built")
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_batch.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    now = {k: d for k, (d, n) in sass_digest.per_kernel(MAIN_LIB).items()}
    assert set(now) == set(rec["kernels"])
    changed = sorted(k for k, d in rec["kernels"].items() if now[k] != d)
    assert not changed, changed
    assert "k_batch" not in _cuobjdump("-sass", lib=MAIN_LIB)
