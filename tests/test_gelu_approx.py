"""The GELU the GEMM epilogues evaluate (csrc/tp_ptx.cuh: gelu_erf / gelu_erf_pk, erf by Abramowitz & Stegun 7.1.28) emulated
operation by operation in float32 on the CPU, against the exact erf form nn.GELU() computes (builder.py:63,69,81).  The
coefficients are parsed out of the CUDA source, so the claim in DESIGN.md §3.1 (|error| < 1e-6 absolute, three orders below the
bf16 rounding of the stored result) is checked against the code that ships."""
import os
import re

import numpy as np

from oracle import tokenpacker_oracle as tpo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _fma(a, b, c):
    """Single-rounding a*b+c in float32 (the product of two float32 is exact in float64)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def _coefficients():
    text = open(os.path.join(ROOT, "tokenpacker_b200", "csrc", "tp_ptx.cuh")).read()
    body = text[text.index("__device__ __forceinline__ float gelu_erf(float x)"):]
    body = body[:body.index("}")]
    first = re.search(r"float p = ([0-9.]+)f;", body).group(1)
    rest = re.findall(r"p = fmaf\(p, t, ([0-9.]+)f\);", body)
    assert len(rest) == 6 and rest[-1] == "1.0", rest
    return [f32(first)] + [f32(v) for v in rest]


def gelu_device(x):
    """The instruction sequence of gelu_erf: h = x/2; t = |h| sqrt2; Horner (6 fma); 4 squarings; one reciprocal; e = 1 - r;
    fma(|h|, e, h)."""
    x = x.astype(f32)
    h = (f32(0.5) * x).astype(f32)
    ah = np.abs(h)
    t = (ah * f32(1.41421356237309504880)).astype(f32)
    c = _coefficients()
    p = np.full_like(x, c[0])
    for coef in c[1:]:
        p = _fma(p, t, np.full_like(x, coef))
    with np.errstate(over="ignore"):
        for _ in range(4):
            p = (p * p).astype(f32)                      # +inf for |x| > ~24 -> r = 0 -> erf = 1
        r = (f32(1.0) / p).astype(f32)                   # MUFU.RCP: within 1 ulp of this
    e = (f32(1.0) - r).astype(f32)
    return _fma(ah, e, h)


def test_coefficients_are_abramowitz_stegun_7_1_28():
    want = [0.0000430638, 0.0002765672, 0.0001520143, 0.0092705272, 0.0422820123, 0.0705230784, 1.0]
    np.testing.assert_allclose(np.array(_coefficients(), dtype=np.float64), want, rtol=1e-7)


def test_absolute_error_below_one_millionth():
    x = np.concatenate([np.linspace(-30, 30, 600001), np.linspace(-1e-3, 1e-3, 2001), [0.0, -0.0, 1e-30, -1e-30, 50.0, -50.0]])
    exact = tpo.gelu_erf(x.astype(np.float64))
    got = gelu_device(x.astype(f32)).astype(np.float64)
    assert np.isfinite(got).all()
    err = np.abs(got - exact)
    assert err.max() < 1e-6, (err.max(), x[err.argmax()])
    # an extra ulp of reciprocal error (MUFU.RCP is approximate) moves the result by at most |x| * 2^-24
    assert err.max() + 30 * 2.0 ** -24 < 3e-6


def test_error_is_far_below_bf16_rounding_of_the_result():
    """Where it matters: |y| >= 1e-3.  bf16 keeps 8 significant bits: half an ulp is 2^-9 |y| = 2e-3 |y|."""
    x = np.linspace(-4.0, 8.0, 240001)
    exact = tpo.gelu_erf(x)
    got = gelu_device(x.astype(f32)).astype(np.float64)
    rel = np.abs(got - exact) / np.maximum(np.abs(exact), 1e-30)
    assert rel[np.abs(exact) >= 1e-3].max() < 2e-3 / 4       # negative tail, |y| ~ 1e-3: 3e-7 absolute is 3e-4 relative
    assert rel[np.abs(exact) >= 1e-2].max() < 2e-3 / 40
    assert np.median(rel[np.abs(exact) >= 1e-3]) < 2e-7


def test_limits():
    x = np.array([40.0, -40.0, 0.0], dtype=f32)
    y = gelu_device(x)
    assert y[0] == f32(40.0) and y[1] == 0.0 and y[2] == 0.0


def test_no_overflow_at_the_top_of_the_range():
    """GELU(x) = x for large x: 0.5 * (x + |x| e) evaluated as written reaches 2x = +inf for x >= 2^127."""
    big = np.finfo(f32).max
    x = np.array([2.0 ** 127, big, -(2.0 ** 127), -big], dtype=f32)
    with np.errstate(over="ignore"):
        y = gelu_device(x)
    assert y[0] == x[0] and y[1] == x[1] and y[2] == 0.0 and y[3] == 0.0


def test_halving_first_keeps_the_bits_of_the_unhalved_form():
    """h = x/2 is exact for |x| >= 2^-125, and then fma(|h|, e, h) = 0.5 * fma(|x|, e, x) and |h| sqrt2 = |x| / sqrt2 bit for bit."""
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(200000) * 4, np.linspace(-30, 30, 60001)]).astype(f32)
    h = (f32(0.5) * x).astype(f32)
    assert np.array_equal((np.abs(h) * f32(1.41421356237309504880)).astype(f32), (np.abs(x) * f32(0.70710678118654752440)).astype(f32))
    e = rng.random(x.shape).astype(f32)
    assert np.array_equal(_fma(np.abs(h), e, h), (f32(0.5) * _fma(np.abs(x), e, x)).astype(f32))
