"""CPU emulation of the f16x3 GEMM arithmetic (csrc/gemm.cu): per (outer index, 128-k chunk) a power-of-two scale that
brings the chunk maximum to [2^13, 2^14), hi = fp16(x s), lo = fp16(x s - hi), products hi.hi + hi.lo + lo.hi per
chunk, folded with the inverse scales.  The emulation keeps the row-scaled error of every output row within the bound
of tests/test_gpu_gemm_f16.py (3e-6) on rows and chunks 2^+-30 apart, zero chunks and fp32-subnormal rows; the same
arithmetic with one scale per tensor does not."""
import numpy as np
import pytest

CK = 128
BOUND = 3e-6


def _exp(amax):
    """the kernel's scale exponent: 13 - floor(log2 amax), clamped to [-126, 126]; 0 for an all-zero chunk"""
    e = np.zeros(amax.shape, np.int64)
    nz = amax > 0
    e[nz] = np.clip(13 - np.floor(np.log2(amax[nz])).astype(np.int64), -126, 126)
    return e


def _split(x, per_tensor=False):
    """x[outer, K] (fp32 values) -> hi, lo (fp16 values as float64, [outer, chunks, CK]) and exponents [outer, chunks]"""
    outer, K = x.shape
    Kp = -(-K // CK) * CK
    xp = np.zeros((outer, Kp), np.float64)
    xp[:, :K] = x
    xc = xp.reshape(outer, Kp // CK, CK)
    amax = np.abs(xc).max(2)
    e = _exp(np.full_like(amax, np.abs(xc).max())) if per_tensor else _exp(amax)
    xs = xc * np.exp2(e)[:, :, None]                       # exact: power of two, in range
    hi = xs.astype(np.float16).astype(np.float64)
    lo = (xs - hi).astype(np.float16).astype(np.float64)
    return hi, lo, e


def _gemm(a, b, per_tensor=False):
    ah, al, ea = _split(a, per_tensor)
    bh, bl, eb = _split(b, per_tensor)
    d = (np.einsum("mck,nck->mnc", ah, bh) + np.einsum("mck,nck->mnc", ah, bl) + np.einsum("mck,nck->mnc", al, bh))
    return (d * np.exp2(-ea)[:, None, :] * np.exp2(-eb)[None, :, :]).sum(2)


def _row_err(c, a, b):
    ref = a.astype(np.float64) @ b.astype(np.float64).T
    scale = np.abs(ref).max(1)
    live = scale > 0
    assert np.all(c[~live] == 0)
    return float((np.abs(c - ref).max(1)[live] / scale[live]).max())


def _operands(case, rng):
    M, N, K = 48, 40, 3 * CK + 40                                  # a K tail inside the last chunk
    a = rng.standard_normal((M, K))
    b = rng.standard_normal((N, K)) * 0.05
    if case == "rows":                                              # rows 2^-30 ... 2^+30 apart
        a *= np.exp2(rng.integers(-30, 31, (M, 1)))
    elif case == "chunks":                                          # chunks 2^+-30 apart, B's chunks inverse: all count
        s = np.exp2(np.array([30, -30, 0, -30]))
        a *= np.repeat(s, CK)[:K]
        b /= np.repeat(s, CK)[:K]
    elif case == "zero":                                            # zero chunks and zero rows
        a[:, CK:2 * CK] = 0
        a[::5] = 0
    elif case == "subnormal":                                       # fp32-subnormal rows next to rows of order 1
        a[::2] *= 2.0 ** -135
    return a.astype(np.float32), b.astype(np.float32)


@pytest.mark.parametrize("case", ["rows", "chunks", "zero", "subnormal"])
def test_chunk_scales_keep_fp32_class(case):
    a, b = _operands(case, np.random.default_rng(len(case)))
    assert _row_err(_gemm(a, b), a, b) < BOUND


@pytest.mark.parametrize("case", ["rows", "chunks", "subnormal"])
def test_one_scale_per_tensor_fails(case):
    a, b = _operands(case, np.random.default_rng(len(case)))
    assert _row_err(_gemm(a, b, per_tensor=True), a, b) > 100 * BOUND


def test_scale_exponent_edges():
    amax = np.array([2.0 ** 13, 2.0 ** 14 - 1, 1.0, 2.0 ** -149, 3.0e38])
    e = _exp(amax)
    assert list(e) == [0, 0, 13, 126, -114]
    assert np.all(amax[:3] * np.exp2(e[:3]) >= 2.0 ** 13) and np.all(amax[:3] * np.exp2(e[:3]) < 2.0 ** 14)


def _element_bound(a, b):
    """The product terms of tests/test_gpu_gemm_parity.py's f16x3 bound: 3 * 2^-22 |a| |b| per product and
    2^-37 * 128 cmax_a cmax_b per chunk (the emulation sums exactly, so the accumulation terms are left out)."""
    a, b = a.astype(np.float64), b.astype(np.float64)
    K = a.shape[1]
    Kp = -(-K // CK) * CK
    ap, bp = np.zeros((a.shape[0], Kp)), np.zeros((b.shape[0], Kp))
    ap[:, :K], bp[:, :K] = np.abs(a), np.abs(b)
    ca, cb = ap.reshape(len(a), -1, CK).max(2), bp.reshape(len(b), -1, CK).max(2)
    return 3 * 2.0 ** -22 * (ap @ bp.T) + 2.0 ** -37 * CK * (ca @ cb.T)


@pytest.mark.parametrize("case", ["rows", "chunks", "zero", "subnormal"])
def test_per_element_bound(case):
    """Every element of the emulated f16x3 product within half its own bound; one scale per tensor far outside it."""
    a, b = _operands(case, np.random.default_rng(len(case)))
    ref = a.astype(np.float64) @ b.astype(np.float64).T
    bnd = _element_bound(a, b)
    live = bnd > 0

    def ratio(c):
        assert np.all(c[~live] == 0)                 # zero rows: exactly zero
        return float((np.abs(c - ref)[live] / bnd[live]).max())
    assert ratio(_gemm(a, b)) <= 0.5
    if case != "zero":
        assert ratio(_gemm(a, b, per_tensor=True)) >= 4
