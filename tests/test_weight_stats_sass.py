"""The blend-weight statistics kernels in the built library: every kernel that existed before them compiles to the same
SASS, and the new ones keep no more in local memory than their default counterparts.  Needs nvcc's cuobjdump and the
built library, no GPU."""
import importlib.util
import json
import re
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
LIB = ROOT / "gaussian_splatting_b200" / "libgsr_b200.so"
# new kernel (mangled-name fragment) -> its default counterpart
STATS_KERNELS = {"18k_render_fwd_statsILb0E": "12k_render_fwdILb0E", "18k_render_fwd_statsILb1E": "12k_render_fwdILb1E",
                 "24k_render_fwd_depth_statsILb0E": "18k_render_fwd_depthILb0E",
                 "24k_render_fwd_depth_statsILb1E": "18k_render_fwd_depthILb1E"}


def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists() or not LIB.exists():
        pytest.skip(f"{name} or the built library is missing")
    return exe


def _usage():
    out = subprocess.run([_tool("cuobjdump"), "--dump-resource-usage", str(LIB)], check=True, capture_output=True,
                         text=True).stdout
    return {name: {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
            for name, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out)}


def _local_ops():
    out = subprocess.run([_tool("cuobjdump"), "-sass", str(LIB)], check=True, capture_output=True, text=True).stdout
    ops = {}
    for f in re.split(r"\n\s+Function : ", out)[1:]:
        name, body = f.split("\n", 1)
        ops[name.strip()] = len(re.findall(r"\b(?:STL|LDL)\b", body))
    return ops


def test_stats_kernels_use_no_more_local_memory_than_the_defaults():
    usage, local = _usage(), _local_ops()
    for new, old in STATS_KERNELS.items():
        u_new = next(v for k, v in usage.items() if new in k)
        u_old = next(v for k, v in usage.items() if old in k and "stats" not in k)
        l_new = next(v for k, v in local.items() if new in k)
        l_old = next(v for k, v in local.items() if old in k and "stats" not in k)
        print(new, u_new, "local ops", l_new, "| default", u_old, "local ops", l_old)
        assert u_new["LOCAL"] <= u_old["LOCAL"] and u_new["STACK"] <= u_old["STACK"], (new, u_new, u_old)
        assert l_new <= l_old, (new, l_new, l_old)


def test_kernels_that_existed_before_the_weight_statistics_compile_to_the_same_sass():
    """Per-kernel digests of the SASS instruction listing (tools/dev/sass_digest.py) of every kernel of the library
    before the statistics kernels were added.  Only meaningful with the nvcc release that recorded them."""
    rec = json.loads((Path(__file__).parent / "golden" / "sass_digests_before_weight_stats.json").read_text())
    ver = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if ver != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {ver}")
    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    now = mod.per_kernel(LIB)
    missing = [k for k in rec["kernels"] if k not in now]
    changed = [k for k, d in rec["kernels"].items() if k in now and now[k][0] != d]
    assert not missing and not changed, (missing, changed)
    assert sum(1 for k in now if "stats" in k) == 4
