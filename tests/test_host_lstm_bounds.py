"""CPU checks for tests/test_gpu_lstm_variants.py: the variant table of the BiLSTM dispatcher, and that the parity bound
used there has teeth.

The bound  err(row) <= K * max(err_fp32(row), FLOOR)  is applied here to numpy emulations of the step products at
the GPU tests' input distribution: the correct "2 x 2 block" fp16 hi/lo split (hi = fp16(x), lo = fp16((x - hi) *
2048), product hi.hi + (hi.lo + lo.hi) / 2048, dG rows scaled by their own power of two), and five defects a kernel
could plausibly have.  The correct emulation must pass; every defect must fail by a wide margin.
"""
import numpy as np
import pytest

import test_gpu_lstm_variants as V
from oracle import lstm_ref


# ------------------------------------------------------------------------------------------- variant table
def test_gpu_cases_reach_the_variants_they_name(pkg):
    """Every parity case of the GPU file reaches the variant it names, and together they cover the sweep."""
    lib = pkg.load_library()
    for B, H, ndir, mode, _, fwd, bwd in V.CASES:
        assert V._labels(lib, B, H, ndir, mode) == (fwd, bwd), (B, H, ndir, mode)
    for B, H, ndir, mode, fwd, bwd in V.EDGE_SHAPES:
        assert V._labels(lib, B, H, ndir, mode) == (fwd, bwd), (B, H, ndir, mode)
    covered = set()
    for B, H, ndir, mode, *_ in V.CASES:
        covered |= lstm_ref.case_features(lib, B, H, ndir, mode)
    assert covered == lstm_ref.sweep_features(lib)


@pytest.mark.parametrize("B,H,ndir,mode,fwd,bwd", [
    (64, 512, 2, 0, "wgmma16/flag/vec", "wgmma16/poll"),
    (64, 512, 2, 256, "wgmma16/flag+strict/vec", "wgmma16/poll"),      # strict acquire: flag protocol only
    (64, 512, 2, 3, "mma.sync/v2", "mma.sync"),
    (64, 512, 2, 1, "fma2x8", "fma2x8/vec"),
    (64, 256, 2, 256, "wgmma8/flag+strict/vec", "wgmma8/poll"),
    (32, 640, 2, 0, "wgmma12/flag/scalar", "wgmma16/poll"),           # cfg D: the backward keeps no inbox in smem
    (32, 640, 2, 256, "wgmma12/flag+strict/scalar", "wgmma16/poll"),
    (32, 640, 2, 3, "mma.sync/v2", "mma.sync"),
    (32, 640, 2, 1, "fma2x8", "fma2x8/scalar"),
    (64, 768, 2, 0, "fma2x8 x4", "wgmma16/poll x2"),                  # no wgmma forward plan above H = 640 at B 64
    (64, 768, 2, 3, "fma2x8 x4", "fma2x8/vec x4"),                    # ... and no mma.sync plan: mode 3 runs FMA
    (32, 768, 2, 0, "fma2x8 x2", "wgmma16/poll"),
    (64, 448, 2, 0, "wgmma16/flag/scalar", "mma.sync"),               # H % 128 != 0: no wgmma backward
    (3, 16, 2, 0, "fma1x4", "fma1x4/scalar"),
    (32, 1024, 1, 0, "fma2x8 x2", "fma2x8/vec x2"),
])
def test_lstm_variant_table(pkg, B, H, ndir, mode, fwd, bwd):
    assert V._labels(pkg.load_library(), B, H, ndir, mode) == (fwd, bwd)


def test_lstm_variant_query_without_a_plan(pkg):
    lib = pkg.load_library()
    assert lstm_ref.variant(lib, 8, 20, 2, False) is None        # H % 16 != 0
    assert lstm_ref.variant(lib, 8, 16, 3, False) is None        # bad ndir


# ------------------------------------------------------------------------------------------- emulated products
def _f16_split(x):
    x = x.astype(np.float32)
    hi = x.astype(np.float16).astype(np.float32)
    lo = ((x - hi) * np.float32(2048)).astype(np.float16).astype(np.float32)
    return hi, lo


def _tf32(x):
    return (x.astype(np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _split_product(a, w, drop_w_lo=False, drop_a_lo=False):
    ah, al = _f16_split(a)
    wh, wl = _f16_split(w)
    cross = (0 if drop_w_lo else ah @ wl) + (0 if drop_a_lo else al @ wh)
    return ah @ wh + cross / np.float32(2048)         # fp32 products and accumulation


def _row_scaled(prod, per_cta=False):
    """dG . W with every row (or, as a defect, the whole 32-row CTA) brought to [2^13, 2^14) before the split."""
    def f(a, w):
        m = np.abs(a).max(axis=1, keepdims=True)
        if per_cta:
            m = np.broadcast_to(m.max(), m.shape)
        e = np.clip(np.floor(np.log2(np.where(m > 0, m, 1.0))), -113, 127)
        return prod((a * 2.0 ** (13 - e)).astype(np.float32), w) * (2.0 ** (e - 13)).astype(np.float32)
    return f


PRODUCTS = {
    "correct 2 x 2 split": (_split_product, _row_scaled(_split_product), 1),
    "W in fp16 hi only": (lambda a, w: _split_product(a, w, drop_w_lo=True),
                          _row_scaled(lambda a, w: _split_product(a, w, drop_w_lo=True)), 1),
    "single-pass TF32": (lambda a, w: (_tf32(a) @ _tf32(w)).astype(np.float32),
                         lambda a, w: (_tf32(a) @ _tf32(w)).astype(np.float32), 1),
    "lo . hi cross term dropped": (lambda a, w: _split_product(a, w, drop_a_lo=True),
                                   _row_scaled(lambda a, w: _split_product(a, w, drop_a_lo=True)), 1),
    "per-CTA dG scale": (_split_product, _row_scaled(_split_product, per_cta=True), 1),
    "h read one step late": (_split_product, _row_scaled(_split_product), 2),
}


def _sig(x):
    return 1 / (1 + np.exp(-x))


def _emulate(pre, whh, dout, dt, fprod, bprod, lag=1):
    """One direction of the recurrence and its BPTT in dtype `dt`, with the step products done by fprod / bprod,
    in the order of the kernels (pointwise backward as in csrc/lstm.cu).  pre [B, T, H, 4], whh [4H, H]."""
    B, T, H, _ = pre.shape
    pre, w, dout = pre.astype(dt), whh.astype(dt), dout.astype(dt)
    wt = np.ascontiguousarray(w.T)                             # [H, 4H]
    hs = [np.zeros((B, H), dt)] * (lag + 1)
    c = np.zeros((B, H), dt)
    out, cst, gts = np.zeros((B, T, H), dt), np.zeros((B, T, H), dt), np.zeros((B, T, H, 4), dt)
    for t in range(T):
        z = pre[:, t] + fprod(hs[-lag], wt).astype(dt).reshape(B, 4, H).transpose(0, 2, 1)
        i, f, g, o = _sig(z[..., 0]), _sig(z[..., 1]), np.tanh(z[..., 2]), _sig(z[..., 3])
        c = f * c + i * g
        h = o * np.tanh(c)
        hs = hs[1:] + [h]
        out[:, t], cst[:, t], gts[:, t] = h, c, np.stack([i, f, g, o], -1)
    dG = np.zeros_like(gts)
    dc_next = np.zeros((B, H), dt)
    part = np.zeros((B, H), dt)
    for t in range(T - 1, -1, -1):
        i, f, g, o = (gts[:, t, :, q] for q in range(4))
        cp = cst[:, t - 1] if t > 0 else np.zeros((B, H), dt)
        dh = dout[:, t] + part
        tc = np.tanh(cst[:, t])
        dc = dc_next + dh * o * (1 - tc * tc)
        d = np.stack([dc * g * i * (1 - i), dc * cp * f * (1 - f), dc * i * (1 - g * g), dh * tc * o * (1 - o)], -1)
        dG[:, t] = d
        dc_next = dc * f
        part = bprod(d.transpose(0, 2, 1).reshape(B, 4 * H), w).astype(dt)
    return out, cst, gts, dG


def _exact(a, w):
    return a.astype(np.float64) @ w.astype(np.float64)


def _plain32(a, w):
    return a.astype(np.float32) @ w.astype(np.float32)


def _worst_ratio(got, r64, r32):
    """max over tensors and rows of err / bound (the GPU test's bound, rows by batch)."""
    worst = 0.0
    for k, r, f in zip(got, r64, r32):
        k, r, f = (x.reshape(x.shape[0], -1).astype(np.float64) for x in (k, r, f))
        for b in range(r.shape[0]):
            s = np.abs(r[b]).max()
            if s == 0:
                continue
            ek = np.abs(k[b] - r[b]).max() / s
            ef = np.abs(f[b] - r[b]).max() / s
            worst = max(worst, ek / (V.K * max(ef, V.FLOOR)))
    return worst


@pytest.mark.parametrize("H,T,wscale", [(128, 9, 1.0), (256, 17, 1.0), (128, 9, 3.0)])
def test_bound_accepts_the_split_product_and_rejects_defects(H, T, wscale):
    B = 32
    pre, whh, dout = (x.numpy().astype(np.float64) for x in V._inputs(B, T, H, 1, seed=H + T, wscale=wscale))
    pre, whh = pre[0], whh[0]
    r64 = _emulate(pre, whh, dout, np.float64, _exact, _exact)
    r32 = _emulate(pre, whh, dout, np.float32, _plain32, _plain32)
    ratios = {}
    for name, (fp, bp, lag) in PRODUCTS.items():
        ratios[name] = _worst_ratio(_emulate(pre, whh, dout, np.float32, fp, bp, lag), r64, r32)
    print(ratios)
    assert ratios.pop("correct 2 x 2 split") <= 0.25, ratios
    for name, r in ratios.items():
        assert r >= 8.0, (name, r)
