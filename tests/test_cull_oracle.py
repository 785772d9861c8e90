"""The forward's exact ellipse-vs-block culling test (gsr_record.cuh row_cull) against the kernel-order per-pixel alpha,
on more than a million random and adversarial (record, 4x4 block) cases, restated in tests/cull_oracle.c:

* every block the new test culls has no pixel whose alpha passes the walk's 1/255 test (conservative);
* the new test never lists a block the previous bounding circle AND box (footprint_bounds) culls (a refinement);
* it culls a real share of what the old test listed (the point of the change).
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = HERE / "cull_oracle.c"
        digest = hashlib.sha256(src.read_bytes()).hexdigest()[:16]
        out_dir = Path(tempfile.gettempdir()) / f"gsr_cull_oracle_{os.getuid()}"
        out_dir.mkdir(exist_ok=True)
        out = out_dir / f"libgsr_cull_oracle_{digest}.so"
        if not out.exists():
            tmp = out.with_suffix(f".{os.getpid()}.tmp")
            subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", str(src), "-o", str(tmp), "-lm"],
                           check=True, capture_output=True)
            os.replace(tmp, out)
        _lib = C.CDLL(str(out))
    return _lib


def check(cases, w=3.0):
    """flags per case (bit 0 new lists, bit 1 old lists, bit 2 some pixel contributes) and the rule-break count"""
    f32 = {k: np.ascontiguousarray(cases[k], np.float32) for k in ("u", "v", "a", "b2", "c", "opa", "tau", "x0", "y0")}
    n = f32["u"].size
    flags = np.zeros(n, np.uint8)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    bad = lib().cull_check(C.c_int(n), *(p(f32[k]) for k in ("u", "v", "a", "b2", "c", "opa", "tau", "x0", "y0")),
                           C.c_float(w), p(flags))
    return flags, bad


def covariance(rng, n, log_sigma_mean, log_sigma_sd, max_ratio=None):
    """[n] dilated 2-D covariances (a, 2b, c) of rotated ellipses, as make_record forms them from the conic"""
    s1 = np.exp(rng.normal(log_sigma_mean, log_sigma_sd, n))
    s2 = np.exp(rng.normal(log_sigma_mean, log_sigma_sd, n))
    if max_ratio is not None:  # needles: minor axis = major / ratio, ratio log-uniform up to max_ratio
        s2 = s1 / np.exp(rng.uniform(0.0, np.log(max_ratio), n))
    th = rng.uniform(0, np.pi, n)
    ct, st = np.cos(th), np.sin(th)
    c0 = ct * ct * s1 * s1 + st * st * s2 * s2
    c2 = st * st * s1 * s1 + ct * ct * s2 * s2
    c1 = 2 * ct * st * (s1 * s1 - s2 * s2)
    f = np.float32
    return (c0.astype(f) + f(0.25)).astype(f), c1.astype(f), (c2.astype(f) + f(0.25)).astype(f)


def block_and_centre(rng, n, a, c, spread=3.0):
    """blocks on the 4-pixel grid of a 1080p frame; centres around them out to a few footprint radii"""
    x0 = (rng.integers(0, 480, n) * 4).astype(np.float32)
    y0 = (rng.integers(0, 270, n) * 4).astype(np.float32)
    r = spread * np.sqrt(np.maximum(a, c) * 11.0) + 4.0
    u = (x0 + 1.5 + rng.uniform(-1, 1, n) * r).astype(np.float32)
    v = (y0 + 1.5 + rng.uniform(-1, 1, n) * r).astype(np.float32)
    return x0, y0, u, v


def opacity(rng, n):
    """mostly uniform, a quarter at the 1/255 edge (tau' near 0)"""
    o = rng.uniform(0.0, 1.0, n)
    edge = rng.random(n) < 0.25
    o[edge] = rng.uniform(0.0038, 0.0045, edge.sum())
    return o.astype(np.float32)


def make_cases(kind, n, seed):
    rng = np.random.default_rng(seed)
    tau = np.full(n, np.nan, np.float32)
    if kind == "bench":      # the bench scene's splats: per-axis sigma LogNormal(ln 1.2, 0.6) px
        a, b2, c = covariance(rng, n, np.log(1.2), 0.6)
    elif kind == "large":    # big splats (tens to hundreds of pixels)
        a, b2, c = covariance(rng, n, np.log(40.0), 1.2)
    elif kind == "needle":   # needles at all angles, condition numbers up to 1e6
        a, b2, c = covariance(rng, n, np.log(8.0), 1.0, max_ratio=1e3)
    elif kind == "det_small":  # record-space covariances with det near 1e-18 (no dilation floor)
        a = np.exp(rng.uniform(np.log(1e-10), np.log(1e-8), n)).astype(np.float32)
        c = (1e-18 / a * np.exp(rng.uniform(0.0, 3.0, n))).astype(np.float32)
        b2 = (2 * np.sqrt(a.astype(np.float64) * c) * rng.uniform(-0.9, 0.9, n)).astype(np.float32)
    elif kind == "det_large":  # det near 1e18
        a = np.exp(rng.uniform(np.log(1e8), np.log(1e10), n)).astype(np.float32)
        c = (1e18 / a * np.exp(rng.uniform(-1.0, 1.0, n))).astype(np.float32)
        b2 = (2 * np.sqrt(a.astype(np.float64) * c) * rng.uniform(-0.99, 0.99, n)).astype(np.float32)
    else:
        raise ValueError(kind)
    x0, y0, u, v = block_and_centre(rng, n, a, c, spread=1.5 if kind.startswith("det") else 3.0)
    if kind == "det_small":  # sub-pixel splats: centres within a few sigma of a pixel of a block near the origin
        x0 = (rng.integers(0, 3, n) * 4).astype(np.float32)
        y0 = (rng.integers(0, 3, n) * 4).astype(np.float32)
        u = (x0 + rng.integers(-1, 5, n) + np.sqrt(a) * rng.normal(0, 1.5, n)).astype(np.float32)
        v = (y0 + rng.integers(-1, 5, n) + np.sqrt(c) * rng.normal(0, 1.5, n)).astype(np.float32)
    elif kind == "det_large":
        u = (x0 + rng.uniform(-4, 8, n)).astype(np.float32)
        v = (y0 + rng.uniform(-4, 8, n)).astype(np.float32)
    return dict(u=u, v=v, a=a, b2=b2, c=c, opa=opacity(rng, n), tau=tau, x0=x0, y0=y0)


def edges_and_sentinels(n, seed):
    """centres exactly on block edges and corners (and one float step off them), and tau' = +-inf / -1 / 0"""
    rng = np.random.default_rng(seed)
    a, b2, c = covariance(rng, n, np.log(1.5), 0.8)
    x0 = (rng.integers(0, 480, n) * 4).astype(np.float32)
    y0 = (rng.integers(0, 270, n) * 4).astype(np.float32)
    off = np.array([-1.0, -0.5, 0.0, 1.5, 3.0, 3.5, 4.0, 5.0], np.float32)
    u = (x0 + rng.choice(off, n)).astype(np.float32)
    v = (y0 + rng.choice(off, n)).astype(np.float32)
    step = rng.integers(-1, 2, (2, n))
    u = np.where(step[0] == 0, u, np.nextafter(u, u + step[0])).astype(np.float32)
    v = np.where(step[1] == 0, v, np.nextafter(v, v + step[1])).astype(np.float32)
    tau = np.full(n, np.nan, np.float32)
    opa = opacity(rng, n)
    pick = rng.integers(0, 6, n)
    tau[pick == 0] = np.inf  # nothing proven: any opacity
    tau[pick == 1] = -np.inf  # never reaches 1/255: opacity below cull_tau's cut
    tau[pick == 2] = -1.0
    opa[(pick == 1) | (pick == 2)] = rng.uniform(0.0, 0.0039137, ((pick == 1) | (pick == 2)).sum())
    tau[pick == 3] = 0.0  # only the centre itself: opacity below the cut as well
    opa[pick == 3] = rng.uniform(0.0, 0.0039137, (pick == 3).sum())
    return dict(u=u, v=v, a=a, b2=b2, c=c, opa=opa, tau=tau, x0=x0, y0=y0)


CASES = [("bench", 400_000), ("large", 150_000), ("needle", 300_000), ("det_small", 50_000), ("det_large", 50_000)]


@pytest.mark.parametrize("kind,n", CASES)
def test_exact_block_culling_is_conservative_and_never_looser(kind, n):
    cases = make_cases(kind, n, seed=[k for k, _ in CASES].index(kind) + 1)
    flags, bad = check(cases)
    new, old, contrib = flags & 1, (flags >> 1) & 1, (flags >> 2) & 1
    assert int((contrib & (1 - new)).sum()) == 0, f"{kind}: a culled block has a contributing pixel"
    assert int((new & (1 - old)).sum()) == 0, f"{kind}: the new test lists a block the old one culls"
    assert bad == 0
    assert contrib.sum() > n // 50, f"{kind}: too few contributing blocks to say anything"


def test_edges_corners_and_sentinels():
    cases = edges_and_sentinels(200_000, seed=5)
    flags, bad = check(cases)
    assert bad == 0
    tau, new = cases["tau"], flags & 1
    assert (new[tau == np.inf] == 1).all(), "tau' = +inf must always list"
    assert (new[(tau == -np.inf) | (tau == -1.0)] == 0).all(), "tau' < 0 must never list"


def test_new_test_culls_what_the_old_one_listed_needlessly():
    """on the bench scene's splat shapes the old test lists blocks no pixel of which is reached; the exact test drops
    a clear share of them, and still lists every contributing block"""
    flags, bad = check(make_cases("bench", 200_000, seed=11))
    new, old, contrib = flags & 1, (flags >> 1) & 1, (flags >> 2) & 1
    assert bad == 0
    wasted_old = int((old & (1 - contrib)).sum())
    dropped = int((old & (1 - new)).sum())
    assert wasted_old > 0 and dropped > 0.3 * wasted_old, (wasted_old, dropped)


def test_the_c_restatement_is_the_kernels_arithmetic():
    """guard against the restatement drifting from gsr_record.cuh: the constants and operations it names"""
    src = (HERE.parent / "gaussian_splatting_b200" / "csrc" / "gsr_record.cuh").read_text()
    body = src[src.index("RowCull row_cull("):src.index("bool row_block_hits(")]
    for s in ("1.0f + 0x1p-18f", "EREL = 0x1p-18f", "MABS = 0x1p-12f", "1.0f - 0x1p-19f",
              "fminf(tc, fmaf(tau, c, 1.0f))", "fmaf(-lo1, lo1, tc)", "fmaf(-hi1, hi1, tc)", "fminf(R + m, B)",
              "fmaxf(L - m, -B) - w", "fmaf(X, EREL, MABS)"):
        assert s in body, s
