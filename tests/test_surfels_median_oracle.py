"""Median depth for surfels without a GPU: the fp64 oracle (tests/surfels_median_oracle.c) on known answers and against
central differences, argument errors, and libgsr_surfels_median.so (symbols, resources, launch bounds, untouched SASS of
every other library)."""
import json
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import surfels_median_oracle as mo
from tests import surfels_oracle as so
from tests.test_surfels_oracle import _cuobjdump, _single, _stack, _tool, _torch_scene

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "gaussian_splatting_b200"
MEDIAN_LIB = PKG / "libgsr_surfels_median.so"
LENSES = {None: None, "fisheye": (0.03, -0.01, 0.002, -0.0005), "distortion": (-0.12, 0.03, 5e-4, -3e-4, 0.01)}


# ---- known answers ---------------------------------------------------------------------------------------------------
def test_fronto_parallel_stack_crosses_on_the_known_layer():
    """Identity rotations, so every hit's z is its layer's p_z.  At the pixel next to the centre the layers' alphas are
    about their opacities, 0.3, 0.2, 0.25, 0.6: the transmittance in front of them is 1, 0.7, 0.56, 0.42, so the median is the
    third layer, the last one with more than half the light still in front of it."""
    K = np.array([[50.0, 0, 10.3], [0, 50.0, 8.2], [0, 0, 1]])  # the centre off the pixel: no rho3 = rho2 tie there
    z = np.array([2.0, 2.5, 3.0, 3.5])
    opa = np.array([0.3, 0.2, 0.25, 0.6])
    n = len(z)
    sc = dict(xyz=np.column_stack([np.zeros((n, 2)), z]), quaternion=np.tile([1.0, 0, 0, 0], (n, 1)),
              scale=np.column_stack([np.log(0.4 * z[:, None]) * np.ones((n, 2)), np.zeros(n)]),
              opacity=np.log(opa / (1 - opa))[:, None], rgb=np.ones((n, 3)), sh=None, T=np.eye(4), K=K, H=17, W=21)
    o = mo.render(sc)
    assert o.id[8, 10] == 2 and o.median[8, 10] == 3.0 and not o.flag[8, 10]
    # every covered pixel takes one of the layers' depths exactly
    hit = o.id >= 0
    assert hit.sum() > 100
    np.testing.assert_array_equal(o.median[hit], z[o.id[hit]])
    assert (o.median[~hit] == 0).all()
    # with the first layer at 0.6 (0.4 of the light behind it) it is the median alone
    sc1 = dict(sc, opacity=np.log(np.array([0.6, 0.2, 0.25, 0.6]) / np.array([0.4, 0.8, 0.75, 0.4]))[:, None])
    assert mo.render(sc1).id[8, 10] == 0


@pytest.mark.parametrize("lens", list(LENSES))
def test_single_surfel_median_is_depth_over_alpha(lens):
    sc = _single((1.0, 0.1, 0.05, 0.0), (np.log(0.08), np.log(0.05), 0.3))
    o = mo.render(sc, lens=lens, kc=LENSES[lens])
    if lens is None:
        r = so.render(sc, np.zeros(3))
    else:
        from tests import surfels_lens_oracle as lo

        r = lo.render(sc, np.zeros(3), lens, LENSES[lens])
    a = r.alpha[..., 0]
    hit = a > 0
    assert hit.sum() > 20
    assert ((o.id == 0) == hit).all() and (o.id[~hit] == -1).all()
    np.testing.assert_allclose(o.median[hit], r.depth[..., 0][hit] / a[hit], rtol=1e-13)
    assert (o.median[~hit] == 0).all()


# ---- gradients against central differences ---------------------------------------------------------------------------
@pytest.mark.parametrize("lens", list(LENSES))
def test_gradients_match_central_differences(lens):
    sc = _stack(n=5, seed=1)
    kc = LENSES[lens]
    G = np.random.default_rng(5).normal(size=(sc["H"], sc["W"]))
    # a central difference across a flagged pixel's decision would not be a derivative: those pixels get no gradient
    flag = mo.render(sc, lens=lens, kc=kc).flag > 0
    assert flag.sum() <= 3
    G[flag] = 0.0
    o = mo.render(sc, grads=G, lens=lens, kc=kc)
    assert len(np.unique(o.id[o.id >= 0])) >= 3
    h = 1e-6
    for name in ("xyz", "quaternion", "scale"):
        num = np.zeros_like(sc[name], dtype=float)
        for idx in np.ndindex(sc[name].shape):
            vals = []
            for sgn in (1, -1):
                s2 = dict(sc)
                s2[name] = sc[name].astype(float).copy()
                s2[name][idx] += sgn * h
                vals.append(mo.loss(mo.render(s2, lens=lens, kc=kc), G))
            num[idx] = (vals[0] - vals[1]) / (2 * h)
        ref = max(np.abs(num).max(), np.abs(o.g["xyz"]).max())
        np.testing.assert_allclose(o.g[name], num, rtol=0, atol=2e-6 * ref + 1e-9, err_msg=f"{lens}: {name}")
    assert np.abs(o.g["xyz"]).max() > 0 and np.abs(o.g["quaternion"]).max() > 0
    # the intersection's z does not depend on the scales: d median / d scale vanishes, though dM's scale columns do not
    assert np.abs(o.rows[:, 0:2]).max() > 0
    # nothing reaches opacity, colour, normal or the low-pass centre
    assert (o.g["opacity"] == 0).all()
    assert (o.rows[:, 9:18] == 0).all() and (o.rows[:, 19] == 0).all()


@pytest.mark.parametrize("k", [(0, 2), (1, 2)])
def test_pinhole_rows_are_d_loss_d_k_m(k):
    """The pinhole rows are d loss / d M with M = K M'.  The principal point enters M only (M_r += c_r M'_2), so
    d loss / d c_r = sum_i sum_j rows_i[r, j] M'_2j: the rows' mapping from M' to M against a step in cx or cy."""
    sc = _stack(n=4, seed=2)
    G = np.random.default_rng(6).normal(size=(sc["H"], sc["W"]))
    o = mo.render(sc, grads=G)
    h = 1e-6
    vals = []
    for sgn in (1, -1):
        s2 = dict(sc, K=sc["K"].copy())
        s2["K"][k] += sgn * h
        vals.append(mo.loss(mo.render(s2), G))
    num = (vals[0] - vals[1]) / (2 * h)
    r = k[0]
    ana = 0.0
    for i in range(sc["xyz"].shape[0]):
        Rc = sc["T"][:3, :3] @ _rot(sc["quaternion"][i])
        p = sc["T"][:3, :3] @ sc["xyz"][i] + sc["T"][:3, 3]
        su, sv = np.exp(sc["scale"][i, :2])
        M2 = np.array([su * Rc[2, 0], sv * Rc[2, 1], p[2]])
        ana += (o.rows[i, 3 * r:3 * r + 3] * M2).sum()
    assert abs(num) > 1e-3
    np.testing.assert_allclose(ana, num, rtol=1e-5)


def _rot(q):
    w, x, y, z = np.asarray(q, float) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


# ---- arguments -------------------------------------------------------------------------------------------------------
def test_median_depth_argument_keeps_every_other_argument_check():
    from gaussian_splatting_b200.surfels import rasterize_surfels

    g, cam, T, bg = _torch_scene(torch.float64)
    with pytest.raises(TypeError):
        rasterize_surfels(g, T, cam, 0.3, 100.0, 10.0, 3.0, bg, median_depth=True)
    g, cam, T, bg = _torch_scene()
    with pytest.raises(ValueError, match="CUDA"):
        rasterize_surfels(g, T, cam, 0.3, 100.0, 10.0, 3.0, bg, median_depth=True)


# ---- the library -----------------------------------------------------------------------------------------------------
def test_c_abi_exports_exactly_the_declared_symbols():
    header = (ROOT / "include" / "gsr_surfels_median.h").read_text()
    declared = set(re.findall(r"^(?:int|size_t) (gsr_\w+)\(", header, re.M))
    assert declared == {"gsr_surfel_render_median_forward", "gsr_surfel_render_median_backward"}
    if not MEDIAN_LIB.exists():
        pytest.skip("libgsr_surfels_median.so is not built")
    nm = subprocess.run(["nm", "-D", "--defined-only", str(MEDIAN_LIB)], capture_output=True, text=True).stdout
    assert set(re.findall(r"\bT (gsr_\w+)", nm)) == declared


def test_median_kernels_are_sm90a_use_no_local_memory_and_declare_their_launch_bounds():
    elfs = _cuobjdump("--list-elf", lib=MEDIAN_LIB)
    assert "sm_90a" in elfs and not re.search(r"sm_(?!90a)\d+", elfs), elfs
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", _cuobjdump("--dump-resource-usage", lib=MEDIAN_LIB)))
    names = [k for k in usage if "k_surfel_median" in k]
    assert len(names) == 4, names  # forward and backward, pinhole and ray map
    assert set(usage) == set(names), sorted(usage)
    for name in names:
        u = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", usage[name])}
        assert u["LOCAL"] == 0 and u["STACK"] == 0, (name, u)
        assert u["REG"] <= 64, (name, u)  # 256 threads: the launch bound's register budget
    elf = _cuobjdump("--dump-elf", lib=MEDIAN_LIB)
    bounds = re.findall(r"\.nv\.info\.(\S+)[\s\S]*?EIATTR_MAX_THREADS[\s\S]*?Value:\s*(0x[0-9a-f]+)\s+(0x[0-9a-f]+)\s+"
                        r"(0x[0-9a-f]+)", elf)
    got = {k: tuple(int(v, 16) for v in vals) for k, *vals in bounds}
    assert set(got) == set(names), sorted(got)
    assert all(v == (256, 1, 1) for v in got.values()), got


def test_existing_kernels_keep_their_sass():
    """Every kernel of the thirteen libraries that existed before the surfel median depth keeps its instructions, and
    no library gains or loses a kernel: the median kernels are libgsr_surfels_median.so's."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_digest", ROOT / "tools" / "dev" / "sass_digest.py")
    sass_digest = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass_digest)
    _tool("cuobjdump")
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_surfels_median.json").read_text())
    nvcc = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if nvcc != rec["nvcc"]:
        pytest.skip(f"digests were recorded with {rec['nvcc']}, this is {nvcc}")
    libs = ("libgsr_b200.so", "libgsr_selective_adam.so", "libgsr_features.so", "libgsr_batch.so",
            "libgsr_fisheye.so", "libgsr_distortion.so", "libgsr_pose.so", "libgsr_calib.so", "libgsr_shutter.so",
            "libgsr_bilagrid.so", "libgsr_surfels.so", "libgsr_surfels_lens.so", "libgsr_surfels_features.so")
    assert set(rec) - {"nvcc"} == set(libs)
    for lib in libs:
        if not (PKG / lib).exists():
            pytest.skip(f"{lib} is not built")
        now = {k: d for k, (d, n) in sass_digest.per_kernel(PKG / lib).items()}
        assert set(now) == set(rec[lib]), (lib, sorted(set(now) ^ set(rec[lib]))[:4])
        changed = sorted(k for k, d in rec[lib].items() if now[k] != d)
        assert not changed, (lib, changed)
