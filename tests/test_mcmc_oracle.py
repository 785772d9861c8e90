"""3DGS-MCMC without a GPU: the relocation formula (fp64 oracle against mpmath, its identities, and why fp32 is not
enough), the plans' semantics on CPU tensors, the noise oracle, the regulariser gradients, the C ABI's argument checks
and the new kernels in the built library."""
import ctypes as C
import importlib.util
import json
import math
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from gaussian_splatting_b200.flat_adam import flatten_gaussians, section_ends
from gaussian_splatting_b200.mcmc import MCMCConfig, add_regularizer_grads, grow_count, plan_grow, plan_relocate
from gaussian_splatting_b200.structs import Gaussians
from tests import mcmc_oracle as mo

ROOT = Path(__file__).resolve().parents[1]
LIB = ROOT / "gaussian_splatting_b200" / "libgsr_b200.so"
GRID_O = [1e-3, 0.005, 0.5, 0.99, 1 - 2.0 ** -23]
GSR_ERR_BAD_ARG = -1


# relocation --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("o", GRID_O)
def test_fp64_relocation_matches_mpmath(o):
    """The fp64 double sum against 50-digit mpmath for N = 1..51, and N > 51 clamped to 51: o_hat to 1e-14 and the
    scale coefficient to 1e-11 relative; the clamped opacity equals the rounded exact o_hat, clamped."""
    o32 = np.float32(o)
    ratios = np.array(list(range(1, 52)) + [52, 60, 1000])
    oh, new_o, new_s = mo.relocation_f64(np.full(len(ratios), o32), np.ones((len(ratios), 3)), ratios)
    for r, a, b, c in zip(ratios, oh, new_o, new_s[:, 0]):
        oh_mp, coeff_mp = mo.relocation_mp(o32, r)
        assert abs(a / float(oh_mp) - 1) < 1e-14, (o, r)
        assert abs(c / float(coeff_mp) - 1) < 1e-11, (o, r, c, float(coeff_mp))
        want = min(max(np.float32(float(oh_mp)), np.float32(0.005)), np.float32(1 - 2.0 ** -23))
        assert abs(int(np.float32(b).view(np.int32)) - int(np.float32(want).view(np.int32))) <= 1, (o, r)
    assert np.array_equal(new_s[-4:], np.repeat(new_s[50:51], 4, 0))  # clamped to n_max


@pytest.mark.parametrize("o", GRID_O)
def test_relocation_identities(o):
    """N = 1 keeps opacity and scale; N copies of o_hat stack to the source's opacity, 1 - (1 - o_hat)^N = o."""
    import mpmath

    o32 = np.float32(o)
    oh, coeff = mo.relocation_mp(o32, 1)
    assert abs(oh - float(o32)) < 1e-45 and abs(coeff - 1) < 1e-45
    _, _, s = mo.relocation_f64([o32], [[0.3, 1.0, 2.0]], [1])
    np.testing.assert_allclose(s[0], np.float32([0.3, 1.0, 2.0]), rtol=1e-15)
    with mpmath.workdps(50):
        for n in (2, 7, 51):
            oh, _ = mo.relocation_mp(o32, n)
            assert abs(1 - (1 - oh) ** n - float(o32)) < 1e-45, (o, n)


def test_fp32_sum_visibly_fails_near_opaque():
    """At o = 1 - 2^-23 and N = 51 the terms' magnitudes add up to 2.9e4 times the sum: accumulated in fp32 the scale
    coefficient is off by more than 1e-5 (about 2e-4), in fp64 by less than 1e-11.  Where the sum does not cancel
    (o = 0.5) both are fine."""
    o = np.float32(1 - 2.0 ** -23)
    _, exact = mo.relocation_mp(o, 51)
    oh = -math.expm1(math.log1p(-float(o)) / 51)
    mags = sum(math.comb(51, j) * oh ** j / math.sqrt(j) for j in range(1, 52))
    assert mags * float(exact) / float(o) > 1e4
    err32 = abs(float(mo.relocation_f32([o], [51])[0]) / float(exact) - 1)
    err64 = abs(float(mo.relocation_f64([o], [[1, 1, 1]], [51])[2][0, 0]) / float(exact) - 1)
    print("fp32", err32, "fp64", err64)
    assert err32 > 1e-5 and err64 < 1e-11
    _, half = mo.relocation_mp(np.float32(0.5), 51)
    assert abs(float(mo.relocation_f32([np.float32(0.5)], [51])[0]) / float(half) - 1) < 2e-6


# plans on CPU tensors ----------------------------------------------------------------------------------------------
def _gaussians(opacity_sigmoid=None, n=400, seed=0, logits=None):
    g = torch.Generator().manual_seed(seed)
    if logits is None:
        o = torch.as_tensor(opacity_sigmoid, dtype=torch.float32) if opacity_sigmoid is not None else \
            torch.rand(n, generator=g)
        logits = torch.logit(o.clamp(1e-7, 1 - 1e-7))
    n = logits.numel()
    return Gaussians(torch.randn(n, 3, generator=g), torch.rand(n, 3, generator=g), logits.reshape(n, 1).clone(),
                     torch.randn(n, 3, generator=g) - 3, torch.randn(n, 4, generator=g))


def _threshold_logits(thr=0.005):
    """Logits whose sigmoids lie at and on both sides of the threshold: l0 the largest float with sigmoid(l0) <= thr."""
    lo = torch.tensor(math.log(thr / (1 - thr)), dtype=torch.float32)
    while torch.sigmoid(lo) > thr:
        lo = torch.nextafter(lo, torch.tensor(-1e9))
    while torch.sigmoid(torch.nextafter(lo, torch.tensor(1e9))) <= thr:
        lo = torch.nextafter(lo, torch.tensor(1e9))
    hi = torch.nextafter(lo, torch.tensor(1e9))
    assert torch.sigmoid(lo) <= thr < torch.sigmoid(hi)
    return lo, hi


def test_relocate_plan_semantics():
    cfg = MCMCConfig()
    lo, hi = _threshold_logits(cfg.min_opacity)
    base = torch.logit(torch.rand(300, generator=torch.Generator().manual_seed(1)) * 0.9 + 0.05)
    logits = base.clone()
    logits[5::11] = -12.0                            # dead
    logits[::7] = lo                                 # dead: the largest logit at or below the threshold
    logits[3::7] = hi                                # alive by one ulp
    g = _gaussians(logits=logits)
    plan = plan_relocate(g, cfg, torch.Generator().manual_seed(0))
    dead = torch.sigmoid(logits) <= cfg.min_opacity
    dead_idx = torch.nonzero(dead).squeeze(1)
    n = 300
    assert plan.n_out == n and plan.info["relocated"] == int(dead.sum()) and not dead[3::7].any()
    src, set_row = plan.src.long(), plan.set_row.long()
    assert torch.equal(src[~dead], torch.arange(n)[~dead])          # live rows stay where they are
    assert not dead[src[dead_idx]].any()                            # sources are never dead rows
    assert torch.equal(src[dead_idx], plan.sources)                 # dead row j copies draw j
    counts = torch.bincount(plan.sources, minlength=n)
    assert torch.equal(plan.ratio.long(), counts[plan.sources] + 1)  # ratio = multiplicity + 1
    # every drawn source and every dead row take a copy's values; nothing else changes
    changed = torch.zeros(n, dtype=torch.bool)
    changed[dead_idx] = True
    changed[plan.sources] = True
    assert torch.equal(set_row >= 0, changed)
    assert torch.equal(set_row[dead_idx], torch.arange(len(dead_idx)))
    assert torch.equal(plan.sources[set_row[plan.sources]], plan.sources)  # a source points at one of its own draws
    assert plan.src.dtype == plan.set_row.dtype == plan.ratio.dtype == torch.int32


def test_relocate_draws_in_proportion_to_opacity():
    """Two live rows with opacities 0.2 and 0.6 and 20 000 dead rows: the 0.6 row takes about 3/4 of the copies."""
    o = torch.full((20_002,), 0.001)
    o[0], o[1] = 0.2, 0.6
    plan = plan_relocate(_gaussians(o), MCMCConfig(), torch.Generator().manual_seed(3))
    share = float((plan.sources == 1).float().mean())
    assert set(plan.sources.tolist()) == {0, 1} and abs(share - 0.75) < 0.015


def test_relocate_identity_and_all_dead():
    cfg = MCMCConfig()
    plan = plan_relocate(_gaussians(torch.full((50,), 0.3)), cfg)
    assert plan.is_identity() and plan.info["relocated"] == 0 and "skipped" not in plan.info
    plan = plan_relocate(_gaussians(torch.full((50,), 0.001)), cfg)
    assert plan.is_identity() and plan.info["relocated"] == 0 and plan.info["skipped"] == "every gaussian is dead"


def test_grow_count_at_and_near_cap():
    cfg = MCMCConfig(cap_max=1000, growth=0.05)
    assert grow_count(100, cfg) == 5 and grow_count(19, cfg) == 0 and grow_count(20, cfg) == 1
    assert grow_count(950, cfg) == 47 and grow_count(952, cfg) == 47 and grow_count(953, cfg) == 47
    assert grow_count(960, cfg) == 40 and grow_count(999, cfg) == 1 and grow_count(1000, cfg) == 0
    assert grow_count(1200, cfg) == 0 and grow_count(0, cfg) == 0
    assert grow_count(10_000, MCMCConfig(cap_max=10**9, growth=0.5)) == 5000


def test_grow_plan_semantics():
    cfg = MCMCConfig(cap_max=1000)
    g = _gaussians(n=400)
    plan = plan_grow(g, cfg, torch.Generator().manual_seed(2))
    n, n_add = 400, 20
    assert plan.n_out == n + n_add and plan.info["added"] == n_add
    src, set_row = plan.src.long(), plan.set_row.long()
    assert torch.equal(src[:n], torch.arange(n))                    # old rows first, in order
    assert torch.equal(src[n:], plan.sources)                       # appended copies in draw order
    assert torch.equal(set_row[n:], torch.arange(n_add))
    changed = torch.zeros(n, dtype=torch.bool)
    changed[plan.sources] = True
    assert torch.equal(set_row[:n] >= 0, changed)
    assert torch.equal(plan.sources[set_row[plan.sources]], plan.sources)
    assert torch.equal(plan.ratio.long(), torch.bincount(plan.sources, minlength=n)[plan.sources] + 1)
    # at the cap: nothing to add
    full = plan_grow(_gaussians(n=1000), cfg, torch.Generator().manual_seed(2))
    assert full.is_identity() and full.info["added"] == 0


def test_plans_are_reproducible_with_a_fixed_generator():
    o = torch.rand(5000, generator=torch.Generator().manual_seed(9))
    o[::3] = 0.001
    g = _gaussians(o)
    cfg = MCMCConfig(cap_max=10**6)
    for planner in (plan_relocate, plan_grow):
        a = planner(g, cfg, torch.Generator().manual_seed(5))
        b = planner(g, cfg, torch.Generator().manual_seed(5))
        c = planner(g, cfg, torch.Generator().manual_seed(6))
        for k in ("src", "set_row", "sources", "ratio"):
            assert torch.equal(getattr(a, k), getattr(b, k)), k
        assert not torch.equal(a.sources, c.sources)


# noise oracle ------------------------------------------------------------------------------------------------------
def test_noise_weight_values():
    w = mo.noise_weight([0.0, 0.005, 0.5, 1.0])
    np.testing.assert_allclose(w[:2], [1 / (1 + math.exp(-0.5)), 0.5], rtol=1e-15)
    assert 3.0e-22 < w[2] < 3.5e-22 and 0 < w[3] < 1e-43


def test_noise_oracle_covariance():
    """The oracle's Sigma eps equals scipy's rotation matrix R diag(exp(2 s)) R^T applied to eps (quaternions in
    (w, x, y, z), not normalised), and an isotropic scale moves by exp(2 s) eps whatever the rotation."""
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(0)
    n = 64
    q = rng.standard_normal((n, 4)) * 3
    s = rng.uniform(-3, 0.5, (n, 3))
    eps = rng.standard_normal((n, 3))
    opl = np.full(n, -20.0)                       # sigmoid ~ 2e-9: w = 1 / (1 + exp(-0.5))
    out, _ = mo.noise_f64(np.zeros((n, 3)), q, s, opl, eps, scaler=2.0)
    R = Rotation.from_quat(q[:, [1, 2, 3, 0]]).as_matrix()
    sig = R @ (np.exp(2 * s)[:, :, None] * np.transpose(R, (0, 2, 1)))
    want = 2.0 * mo.noise_weight(1 / (1 + np.exp(20.0)))[None] * np.einsum("nij,nj->ni", sig, eps)
    np.testing.assert_allclose(out, want, rtol=1e-12, atol=1e-15)
    iso = np.repeat(s[:, :1], 3, 1)
    out, _ = mo.noise_f64(np.zeros((n, 3)), q, iso, opl, eps, scaler=1.0)
    np.testing.assert_allclose(out, mo.noise_weight(1 / (1 + np.exp(20.0))) * np.exp(2 * iso) * eps, rtol=1e-12)


# regulariser gradients ---------------------------------------------------------------------------------------------
def _flat_gaussians(n=257, sh=3, seed=4):
    g = torch.Generator().manual_seed(seed)
    gs = Gaussians(torch.randn(n, 3, generator=g), torch.rand(n, 3, generator=g), torch.randn(n, 1, generator=g),
                   torch.randn(n, 3, generator=g) - 2, torch.randn(n, 4, generator=g),
                   torch.randn(n, 3, sh, generator=g) if sh else None)
    flat, ends, names = flatten_gaussians(gs)
    return gs, flat, ends


@pytest.mark.parametrize("sh", [0, 3])
def test_regularizer_grads_match_autograd(sh):
    gs, flat, ends = _flat_gaussians(sh=sh)
    cfg = MCMCConfig(opacity_reg=0.03, scale_reg=0.07)
    grad_flat = torch.zeros(flat.numel())
    add_regularizer_grads(grad_flat, gs, cfg)
    loss = cfg.opacity_reg * torch.sigmoid(gs.opacity).mean() + cfg.scale_reg * torch.exp(gs.scale).mean()
    loss.backward()
    n = gs.xyz.shape[0]
    torch.testing.assert_close(grad_flat[ends[1]:ends[1] + 3 * n].view(n, 3), gs.scale.grad, rtol=1e-6, atol=0)
    torch.testing.assert_close(grad_flat[ends[2]:ends[2] + n].view(n, 1), gs.opacity.grad, rtol=1e-6, atol=0)
    other = torch.ones(flat.numel(), dtype=torch.bool)
    other[ends[1]:ends[1] + 3 * n] = False
    other[ends[2]:ends[2] + n] = False
    assert not grad_flat[other].any()                             # no other section (nor padding) is touched
    # it adds to what the buffer holds (the rasterizer's gradients)
    held = torch.randn(flat.numel(), generator=torch.Generator().manual_seed(1))
    acc = held.clone()
    add_regularizer_grads(acc, gs, cfg)
    torch.testing.assert_close(acc, held + grad_flat, rtol=1e-6, atol=1e-7)
    assert torch.equal(acc[other], held[other])


def test_regularizer_in_the_loss_would_miss_the_flat_gradient_buffer():
    """Adding the terms to the loss makes autograd write NEW .grad tensors for scale and opacity: they share no memory
    with the flat gradient buffer an optimizer step reads, which therefore stays without the regulariser."""
    gs, flat, ends = _flat_gaussians()
    grad_flat = torch.zeros(flat.numel())
    (0.01 * torch.sigmoid(gs.opacity).mean() + 0.01 * torch.exp(gs.scale).mean()).backward()
    lo, hi = grad_flat.data_ptr(), grad_flat.data_ptr() + 4 * grad_flat.numel()
    for t in (gs.opacity.grad, gs.scale.grad):
        assert t is not None and t.abs().sum() > 0
        assert not (lo <= t.data_ptr() < hi)
    assert not grad_flat.any()
    add_regularizer_grads(grad_flat, gs, MCMCConfig())
    assert grad_flat.any()


# C ABI argument checks (they return before any launch) -------------------------------------------------------------
P = C.c_void_p


def _lib():
    so = C.CDLL(str(LIB))
    so.gsr_mcmc_relocation.argtypes = [C.c_int, P, P, P, C.c_int, C.c_float, P, P, P]
    so.gsr_mcmc_apply.argtypes = [C.c_int, C.c_int, C.c_int] + [P] * 11
    so.gsr_mcmc_noise.argtypes = [C.c_int, C.c_int, P, C.c_double, C.c_double, C.c_double, C.c_uint64, C.c_uint64,
                                  P, P, P]
    return so


def test_header_declares_and_library_exports_the_mcmc_entry_points():
    from tests.test_cabi import declared_symbols

    so = C.CDLL(str(LIB))
    for name in ("gsr_mcmc_relocation", "gsr_mcmc_apply", "gsr_mcmc_noise"):
        assert name in declared_symbols() and hasattr(so, name), name


def test_relocation_argument_errors():
    so = _lib()
    a, b, c, d, e = (P(0x10000 * k) for k in range(1, 6))   # disjoint fake device ranges, never dereferenced
    assert so.gsr_mcmc_relocation(-1, a, b, c, 51, 0.005, d, e, None) == GSR_ERR_BAD_ARG
    assert so.gsr_mcmc_relocation(8, a, b, c, 0, 0.005, d, e, None) == GSR_ERR_BAD_ARG        # n_max < 1
    assert so.gsr_mcmc_relocation(8, a, b, c, 51, 0.005, None, e, None) == GSR_ERR_BAD_ARG    # missing output
    assert so.gsr_mcmc_relocation(8, a, b, c, 51, 0.005, d, d, None) == GSR_ERR_BAD_ARG       # outputs alias
    assert so.gsr_mcmc_relocation(8, a, b, c, 51, 0.005, a, e, None) == GSR_ERR_BAD_ARG       # output aliases input
    assert so.gsr_mcmc_relocation(8, a, b, c, 51, 0.005, d, P(0x10000 * 2 + 16), None) == GSR_ERR_BAD_ARG  # overlap
    assert so.gsr_mcmc_relocation(0, None, None, None, 51, 0.005, None, None, None) == 0       # empty: ok


def test_apply_argument_errors():
    so = _lib()
    x = [P(0x1000000 * k) for k in range(1, 11)]
    p_in, m_in, v_in, src, srow, nop, nsc, p_out, m_out, v_out = x

    def call(n_in=10, n_out=12, sh=0, **over):
        args = dict(p_in=p_in, m_in=m_in, v_in=v_in, src=src, srow=srow, nop=nop, nsc=nsc, p_out=p_out, m_out=m_out,
                    v_out=v_out)
        args.update(over)
        return so.gsr_mcmc_apply(n_in, n_out, sh, *args.values(), None)

    assert call(n_in=-1) == GSR_ERR_BAD_ARG
    assert call(n_out=9) == GSR_ERR_BAD_ARG                                   # n_out < n_in
    assert call(sh=-1) == GSR_ERR_BAD_ARG
    assert call(v_in=None) == GSR_ERR_BAD_ARG                                 # m without v
    assert call(m_out=None, v_out=None) == GSR_ERR_BAD_ARG                    # moments in without moments out
    assert call(nop=None) == GSR_ERR_BAD_ARG                                  # set_row without its tables
    assert call(srow=None) == GSR_ERR_BAD_ARG                                 # tables without set_row
    assert call(p_out=p_in) == GSR_ERR_BAD_ARG                                # output aliases an input
    assert call(m_out=v_in) == GSR_ERR_BAD_ARG
    assert call(v_out=m_out) == GSR_ERR_BAD_ARG                               # outputs alias
    assert call(p_in=None) == GSR_ERR_BAD_ARG
    assert call(n_in=0, n_out=0) == 0                                         # empty: ok


def test_noise_argument_errors():
    so = _lib()
    p, e_in, e_out = P(0x1000000), P(0x3000000), P(0x5000000)
    assert so.gsr_mcmc_noise(-1, 0, p, 1.0, 100.0, 0.995, 0, 0, None, None, None) == GSR_ERR_BAD_ARG
    assert so.gsr_mcmc_noise(10, -1, p, 1.0, 100.0, 0.995, 0, 0, None, None, None) == GSR_ERR_BAD_ARG
    assert so.gsr_mcmc_noise(10, 0, None, 1.0, 100.0, 0.995, 0, 0, None, None, None) == GSR_ERR_BAD_ARG
    assert so.gsr_mcmc_noise(10, 0, p, 1.0, 100.0, 0.995, 0, 0, None, P(0x1000000 + 64), None) == GSR_ERR_BAD_ARG
    assert so.gsr_mcmc_noise(10, 0, p, 1.0, 100.0, 0.995, 0, 0, e_in, e_in, None) == GSR_ERR_BAD_ARG
    assert so.gsr_mcmc_noise(10, 0, p, 1.0, 100.0, 0.995, 0, 0, P(0x1000000 + 64), e_out, None) == GSR_ERR_BAD_ARG
    assert so.gsr_mcmc_noise(0, 0, None, 1.0, 100.0, 0.995, 0, 0, None, None, None) == 0


def test_binding_rejects_cpu_tensors():
    from gaussian_splatting_b200 import native

    o, s, r = torch.rand(4), torch.rand(4, 3), torch.ones(4, dtype=torch.int32)
    with pytest.raises(RuntimeError):
        native().mcmc_relocation(o, s, r, 51, 0.005)
    p = torch.zeros(section_ends(4, 0)[-1])
    with pytest.raises(RuntimeError):
        native().mcmc_noise(p, 4, 0, 1.0, 100.0, 0.995, 0, 0)
    with pytest.raises(RuntimeError):
        native().mcmc_apply(p, None, None, 4, 0, torch.arange(4, dtype=torch.int32), None, None, None)


# the kernels in the built library ---------------------------------------------------------------------------------
MCMC_KERNELS = ("17k_mcmc_relocation", "12k_mcmc_apply", "12k_mcmc_noise")


def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists() or not LIB.exists():
        pytest.skip(f"{name} or the built library is missing")
    return exe


def test_mcmc_kernels_use_no_local_memory_and_relocation_runs_in_fp64():
    out = subprocess.run([_tool("cuobjdump"), "--dump-resource-usage", str(LIB)], check=True, capture_output=True,
                         text=True).stdout
    usage = {name: {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
             for name, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out)}
    sass = subprocess.run([_tool("cuobjdump"), "-sass", str(LIB)], check=True, capture_output=True, text=True).stdout
    bodies = {}
    for f in re.split(r"\n\s+Function : ", sass)[1:]:
        name, body = f.split("\n", 1)
        bodies[name.strip()] = body
    for k in MCMC_KERNELS:
        u = next(v for n, v in usage.items() if k in n)
        body = next(b for n, b in bodies.items() if k in n)
        assert u["LOCAL"] == 0 and u["STACK"] == 0, (k, u)
        assert not re.search(r"\b(?:STL|LDL)\b", body), k
        assert ("DFMA" in body) == (k == "17k_mcmc_relocation"), k


def test_kernels_that_existed_before_mcmc_compile_to_the_same_sass():
    """Per-kernel digests of the SASS instruction listing (tools/dev/sass_digest.py) of every kernel of the library
    before the MCMC kernels were added (gsr_densify_apply's and gsr_adam_step's included).  Only meaningful with the
    nvcc release that recorded them."""
    rec = json.loads((Path(__file__).parent / "golden" / "sass_digests_before_mcmc.json").read_text())
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
    assert sorted(k for k in now if k not in rec["kernels"]) == sorted(
        next(n for n in now if k in n) for k in MCMC_KERNELS)
