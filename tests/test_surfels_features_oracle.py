"""Feature channels for surfels without a GPU: the chunk composition of the fp64 surfel oracles
(tests/surfels_features_oracle.py) against central differences, argument errors, and libgsr_surfels_features.so
(symbols, resources, launch bounds, untouched SASS of every other library)."""
import json
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import surfels_features_oracle as fo
from tests.test_surfels_oracle import _cuobjdump, _stack, _tool, _torch_scene

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "gaussian_splatting_b200"
FEATURES_LIB = PKG / "libgsr_surfels_features.so"


# ---- the fp64 reference ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lens,kc", [(None, None), ("fisheye", (0.03, -0.01, 0.002, -0.0005))])
def test_chunk_composition_matches_central_differences(lens, kc):
    """D = 5: a full 3-channel chunk and a padded one; the summed parts are the gradient of sum G . feature_map."""
    sc = _stack(n=4, seed=1)
    rng = np.random.default_rng(11)
    D = 5
    F = rng.normal(size=(4, D))
    G = rng.normal(size=(sc["H"], sc["W"], D))
    o = fo.render(sc, F, grads=G, lens=lens, kc=kc)
    assert (o.alpha > 0).sum() > 50
    # the feature map is the blend of F with the alpha map's weights: F = 1 gives alpha in every channel
    ones = fo.render(sc, np.ones((4, D)), lens=lens, kc=kc)
    np.testing.assert_allclose(ones.fmap, np.repeat(o.alpha, D, 2), rtol=1e-12, atol=1e-15)
    h = 1e-6
    params = dict(sc, F=F)
    for name in ("F", "xyz", "quaternion", "scale", "opacity"):
        num = np.zeros_like(params[name], dtype=float)
        for idx in np.ndindex(params[name].shape):
            vals = []
            for sgn in (1, -1):
                p2 = dict(params)
                p2[name] = params[name].astype(float).copy()
                p2[name][idx] += sgn * h
                vals.append(fo.loss(fo.render(p2, p2["F"], lens=lens, kc=kc), G))
            num[idx] = (vals[0] - vals[1]) / (2 * h)
        scale = np.abs(num).max()
        assert scale > 0, name
        np.testing.assert_allclose(o.g[name], num, rtol=0, atol=2e-6 * scale + 1e-9, err_msg=name)
    # the colour slots of the rows are cleared; the feature loss reaches no normal or p_z slot
    assert (o.rows[:, 10:16] == 0).all() and (o.rows[:, 18:] == 0).all()


# ---- arguments -------------------------------------------------------------------------------------------------------
def test_feature_arguments_are_checked_before_any_launch():
    from gaussian_splatting_b200.surfels import rasterize_surfels

    g, cam, T, bg = _torch_scene()
    n = g.xyz.shape[0]

    def call(features):
        rasterize_surfels(g, T, cam, 0.3, 100.0, 10.0, 3.0, bg, features=features)

    with pytest.raises(TypeError, match="tensor"):
        call(np.zeros((n, 3), np.float32))
    with pytest.raises(TypeError, match="float32"):
        call(torch.zeros(n, 3, dtype=torch.float64))
    with pytest.raises(ValueError, match="shape"):
        call(torch.zeros(n, 0))
    with pytest.raises(ValueError, match="shape"):
        call(torch.zeros(n + 1, 3))
    with pytest.raises(ValueError, match="shape"):
        call(torch.zeros(n * 3))
    with pytest.raises(ValueError, match="contiguous"):
        call(torch.zeros(3, n).t())
    with pytest.raises(ValueError, match="device"):
        call(torch.zeros(n, 3, device="meta"))


# ---- the library -----------------------------------------------------------------------------------------------------
def test_c_abi_exports_exactly_the_declared_symbols():
    header = (ROOT / "include" / "gsr_surfels_features.h").read_text()
    declared = set(re.findall(r"^(?:int|size_t) (gsr_\w+)\(", header, re.M))
    assert declared == {"gsr_surfel_render_features_forward", "gsr_surfel_render_features_backward"}
    if not FEATURES_LIB.exists():
        pytest.skip("libgsr_surfels_features.so is not built")
    nm = subprocess.run(["nm", "-D", "--defined-only", str(FEATURES_LIB)], capture_output=True, text=True).stdout
    assert set(re.findall(r"\bT (gsr_\w+)", nm)) == declared


def test_feature_kernels_are_sm90a_use_no_local_memory_and_declare_their_launch_bounds():
    elfs = _cuobjdump("--list-elf", lib=FEATURES_LIB)
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage", lib=FEATURES_LIB)))
    names = [k for k in usage if "k_surfel_features" in k]
    assert len(names) == 4, names  # forward and backward, pinhole and ray map
    assert set(usage) == set(names), sorted(usage)
    for name in names:
        u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[name])}
        assert u["LOCAL"] == 0 and u["STACK"] == 0, (name, u)
        assert u["REG"] <= 64, (name, u)  # 256 threads: the launch bound's register budget
    # __launch_bounds__(256): the ELF records the maximum block size of every kernel
    elf = _cuobjdump("--dump-elf", lib=FEATURES_LIB)
    bounds = re.findall(r"\.nv\.info\.(\S+)[\s\S]*?EIATTR_MAX_THREADS[\s\S]*?Value:\s*(0x[0-9a-f]+)\s+(0x[0-9a-f]+)\s+"
                        r"(0x[0-9a-f]+)", elf)
    got = {k: tuple(int(v, 16) for v in vals) for k, *vals in bounds}
    assert set(got) == set(names), sorted(got)
    assert all(v == (256, 1, 1) for v in got.values()), got


def test_existing_kernels_keep_their_sass():
    """Every kernel of the twelve libraries that existed before the surfel feature channels keeps its instructions,
    and no library gains a kernel: the feature kernels are libgsr_surfels_features.so's."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_surfels_features.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    libs = ("libgsr_b200.so", "libgsr_selective_adam.so", "libgsr_features.so", "libgsr_batch.so",
            "libgsr_fisheye.so", "libgsr_distortion.so", "libgsr_pose.so", "libgsr_calib.so", "libgsr_shutter.so",
            "libgsr_bilagrid.so", "libgsr_surfels.so", "libgsr_surfels_lens.so")
    assert set(rec) - {"nvcc"} == set(libs)
    for lib in libs:
        if not (PKG / lib).exists():
            pytest.skip(f"{lib} is not built")
        now = {k: d for k, (d, n) in sass_digest.per_kernel(PKG / lib).items()}
        assert set(now) == set(rec[lib]), (lib, sorted(set(now) ^ set(rec[lib]))[:4])
        changed = sorted(k for k, d in rec[lib].items() if now[k] != d)
        assert not changed, (lib, changed)
