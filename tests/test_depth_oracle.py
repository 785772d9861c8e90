"""The depth-walk oracle (tests/depth_oracle.py) on the CPU: its roundings, the strict threshold, the -1 of pixels
that never reach it, the range (not z), and that the reference order and the fp32-FMA order really disagree on the
kind of input tests/test_splat_cuda_surface_gpu.py feeds the GPU."""
from fractions import Fraction

import numpy as np

from tests import depth_oracle as dor

F32 = np.float32


def round_to_f32(x: Fraction) -> np.float32:
    """Exact round-to-nearest-even of a rational to float32 (normal range)."""
    f = F32(float(x))
    cands = [np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(np.array(c).view(np.uint32)) & 1))
    return F32(best)


def test_fma32_rounds_once():
    rng = np.random.default_rng(0)
    a = rng.uniform(-2, 2, 3000).astype(F32)
    b = rng.uniform(-2, 2, 3000).astype(F32) * F32(2.0) ** rng.integers(-30, 0, 3000).astype(F32)
    c = rng.uniform(-2, 2, 3000).astype(F32)
    got = dor.fma32(a, b, c)
    want = [round_to_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)]
    assert (got.view(np.uint32) == np.array(want, F32).view(np.uint32)).all()
    # a product that puts the float64 sum exactly on a float32 midpoint: rounding the double twice would tie to even
    a1, b1, c1 = F32(1 + 2.0 ** -18), F32(2.0 ** -24 * (1 - 2.0 ** -18)), F32(1 + 2.0 ** -23)
    exact = Fraction(float(a1)) * Fraction(float(b1)) + Fraction(float(c1))
    assert float(a1) * float(b1) + float(c1) == 1 + 3 * 2.0 ** -24          # the double sum is the midpoint
    assert dor.fma32(a1, b1, c1) == round_to_f32(exact) == F32(1 + 2.0 ** -23)


def test_threshold_is_strict():
    xyz = np.array([[[0, 0, 5]]], F32)
    half = np.array([[0.5]], F32)
    assert dor.first_surface(half, xyz, 0.5)[0] == -1.0          # A == threshold does not count
    assert dor.first_surface(half, xyz, np.nextafter(F32(0.5), F32(0)))[0] == 5.0


def test_never_reached_gives_minus_one():
    alphas = np.full((3, 4), 0.1, F32)
    xyz = np.tile(np.array([1, 2, 2], F32), (3, 4, 1))
    A = dor.accumulate(alphas)
    assert A[0, -1] < 0.5
    assert (dor.first_surface(alphas, xyz, 0.5) == -1.0).all()
    assert (dor.first_surface(alphas, xyz, 0.2) == 3.0).all()
    assert (dor.first_surface(np.zeros((2, 0), F32), np.zeros((2, 0, 3), F32), 0.0) == -1.0).all()


def test_output_is_the_range_not_z():
    alphas = np.array([[0.3, 0.6]], F32)
    xyz = np.array([[[2, 3, 6], [3, 4, 12]]], F32)
    assert dor.first_surface(alphas, xyz, 0.2)[0] == 7.0       # sqrt(4 + 9 + 36), z = 6
    assert dor.first_surface(alphas, xyz, 0.5)[0] == 13.0      # second splat: A = 0.3 + 0.7 * 0.6 = 0.72
    # non-integer positions follow the kernel's FMUL / FFMA / FFMA order
    p = np.random.default_rng(1).normal(size=(1000, 3)).astype(F32)
    r = dor.splat_range(p)
    assert np.abs(r.astype(np.float64) - np.linalg.norm(p.astype(np.float64), axis=1)).max() < 1e-6 * 10


def test_reference_order_accumulates_in_double_then_float():
    a = np.array([[0.3, 0.7, 0.01]], F32)
    A = 0.0
    for x in a[0]:
        A = F32(A + F32((1.0 - float(A)) * float(x)))
    assert dor.accumulate(a)[0, -1] == A


def test_the_two_orders_disagree_on_gpu_like_inputs():
    """Seeded alphas in [1/255, 0.6): the orders differ in some steps, and at every separating threshold the
    first-surface answer differs for the pixel it came from — the GPU test built the same way can fail."""
    rng = np.random.default_rng(2)
    alphas = rng.uniform(1 / 255, 0.6, (1536, 8)).astype(F32)
    ref, fma = dor.accumulate(alphas, "reference"), dor.accumulate(alphas, "fma")
    frac = float((ref != fma).mean())
    assert 0.005 < frac < 0.5, frac
    xyz = np.broadcast_to(np.array([[1, 2, 2], [2, 3, 6], [1, 4, 8], [2, 6, 9], [3, 4, 12], [2, 10, 11],
                                    [1, 12, 12], [4, 13, 16]], F32), (1536, 8, 3))
    ts = dor.separating_thresholds(alphas)
    assert len(ts) == 8
    for t, p, k in ts:
        a = dor.first_surface(alphas[p:p + 1], xyz[p:p + 1], t, "reference")[0]
        b = dor.first_surface(alphas[p:p + 1], xyz[p:p + 1], t, "fma")[0]
        assert a != b, (t, p, k)
