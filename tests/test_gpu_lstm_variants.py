"""Every step-kernel variant of the persistent (Bi)LSTM recurrence, through the C ABI, against a float64 recurrence.

The dispatcher (bilstm_run in csrc/lstm.cu) picks a kernel generation - wgmma with fp16 hi/lo operands, 3xTF32
mma.sync, packed fp32 FMA - and within it a template instance, loop form and number of launches.
It makes that choice through b200asr_debug_lstm_variant, so every case below asserts the variant it reaches, and one
test checks that the cases together reach every code path a broad (B, H, ndir, mode) sweep of the query reaches.

b200asr_bilstm_fwd / _bwd are called directly, and all four outputs are compared: the layer output, the cell-state
stash, the activated-gate stash and dG (written in place into `gates`).  Errors are taken PER BATCH ROW, relative to
that row's own largest float64 value, so that a row far below the batch maximum cannot hide behind the others.

Bounds (EPS = 2^-24), fixed here and independent of any run:
    err_kernel(row) <= K * max(err_fp32(row), FLOOR),   K = 8,   FLOOR = 16 * EPS
  * err_fp32 is the error of the same recurrence run in float32 on the CPU (oracle/lstm_ref.recurrence) against the
    same float64 result, computed in the test.  It carries the conditioning of the recurrence at these inputs: how
    much the steps amplify one rounding (saturated gates, W_hh scale, T).
  * The kernels differ from that float32 loop only in the step products h . W_hh^T and dG . W_hh: their operands
    hold about 22 significant bits (fp16 hi + lo / 2048, or TF32 hi + lo with the lo . lo term dropped; DESIGN.md
    section 4) instead of 24, a product rounding at most 4x that of fp32, accumulated in fp32 in another order.
    K = 8 is that 4x with a factor 2 for the summation order.
  * FLOOR covers rows the float32 loop happens to get almost exactly (T = 1 has no product at all): per step the
    pointwise cell is five expf / tanhf (within 2 ulp each) and four multiply-adds, about 12 ulp; 16 ulp of the row
    scale.
tests/test_host_lstm_bounds.py shows on the CPU that this bound accepts an emulation of the correct split product
and rejects the defects a kernel could plausibly have (W in fp16 hi only, a single-pass TF32 product, a dropped
hi . lo term, a per-CTA instead of per-row dG scale, h read one step late) by a wide margin.
"""
import pytest
import torch

from oracle import lstm_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24
K = 8.0
FLOOR = 16 * EPS
DOUT_EXPONENTS = (0, -60, -20, 20, 60)   # dout row b is scaled by 2^DOUT_EXPONENTS[b % 5]

# (B, H, ndir, mode, T, expected forward variant, expected backward variant)
CASES = [
    (64, 512, 2, 0, 9, "wgmma16/flag/vec", "wgmma16/poll"),               # cfg B / C
    (40, 512, 1, 0, 9, "wgmma8/flag/vec", "wgmma8/poll"),                 # second batch group mostly padding
    (1, 512, 2, 0, 9, "wgmma8/flag/vec", "wgmma8/poll"),
    (33, 512, 2, 0, 9, "wgmma16/flag/vec", "wgmma16/poll"),
    (130, 512, 2, 0, 5, "wgmma16/flag/vec x3", "wgmma16/poll x3"),
    (64, 256, 2, 0, 9, "wgmma8/flag/vec", "wgmma8/poll"),
    (64, 384, 2, 0, 9, "wgmma12/flag/vec", "wgmma16/poll"),               # last n-block of the backward 128 wide
    (64, 192, 2, 0, 9, "wgmma8/flag/scalar", "mma.sync"),                 # UB = 6 in the UBP = 8 instance
    (32, 640, 2, 0, 9, "wgmma12/flag/scalar", "wgmma16/poll"),            # cfg D
    (64, 640, 2, 0, 5, "wgmma12/flag/scalar x2", "wgmma16/poll x2"),
    (64, 768, 2, 0, 5, "fma2x8 x4", "wgmma16/poll x2"),
    (32, 1024, 1, 0, 5, "fma2x8 x2", "fma2x8/vec x2"),                    # the RNN-LM layer
    (64, 512, 2, 256, 9, "wgmma16/flag+strict/vec", "wgmma16/poll"),
    (64, 256, 2, 256, 9, "wgmma8/flag+strict/vec", "wgmma8/poll"),        # strict acquire in every UBP instance,
    (64, 384, 2, 256, 9, "wgmma12/flag+strict/vec", "wgmma16/poll"),      # with the scalar publish and over
    (32, 640, 2, 256, 9, "wgmma12/flag+strict/scalar", "wgmma16/poll"),   # several launches
    (130, 512, 2, 256, 5, "wgmma16/flag+strict/vec x3", "wgmma16/poll x3"),
    (64, 448, 2, 0, 9, "wgmma16/flag/scalar", "mma.sync"),                # UB = 14 in the UBP = 16 instance
    (64, 704, 2, 0, 5, "wgmma12/flag/scalar x2", "fma2x8/scalar x2"),
    (64, 512, 2, 3, 9, "mma.sync/v2", "mma.sync"),
    (64, 640, 2, 3, 5, "mma.sync/v2 x2", "mma.sync x2"),
    (64, 192, 2, 3, 9, "mma.sync<2>", "mma.sync"),
    (64, 96, 2, 0, 9, "mma.sync<1>", "mma.sync"),
    (64, 480, 2, 3, 9, "mma.sync<1>", "mma.sync"),
    (130, 512, 2, 3, 5, "mma.sync/v2 x3", "mma.sync x3"),
    (64, 160, 2, 0, 9, "fma2x4", "fma2x4/vec"),
    (64, 512, 2, 1, 9, "fma2x8", "fma2x8/vec"),
    (8, 320, 2, 0, 9, "wgmma8/flag/scalar", "fma1x4/scalar"),
    (5, 800, 2, 0, 5, "fma1x4 x2", "fma1x4/vec x2"),
    (130, 512, 2, 1, 5, "fma2x8 x3", "fma2x8/vec x3"),
]


def _ids(cases):
    return ["B%d-H%d-d%d-m%d-T%d" % c[:5] for c in cases]


def _labels(lib, B, H, ndir, mode):
    return tuple(lstm_ref.label(lstm_ref.variant(lib, B, H, ndir, bwd, mode), bwd) for bwd in (False, True))


def test_cases_cover_every_dispatched_variant(pkg):
    """The variant query over the parity cases reaches every code path that the sweep reaches (same set)."""
    lib = pkg.load_library()
    swept = lstm_ref.sweep_features(lib)
    covered = set()
    for B, H, ndir, mode, *_ in CASES:
        covered |= lstm_ref.case_features(lib, B, H, ndir, mode)
    assert covered == swept, (sorted(swept - covered, key=str), sorted(covered - swept, key=str))


# ------------------------------------------------------------------------------------------- inputs and the C ABI
def _inputs(B, T, H, ndir, seed, wscale=1.0, saturate=0.03):
    """Pre-activations with a fraction driven to +-30 and an all-zero row 0 (a padded utterance), W_hh at `wscale`
    times the nn.LSTM init scale, dout rows scaled by 2^k and an all-zero dout row 1."""
    g = torch.Generator().manual_seed(seed)
    pre = torch.randn(ndir, B, T, H, 4, generator=g)
    sat = torch.rand(pre.shape, generator=g) < saturate
    pre = torch.where(sat, 30.0 * torch.sign(torch.randn(pre.shape, generator=g)), pre)
    if B > 1:
        pre[:, 0] = 0.0
    k = 1.0 / H ** 0.5
    whh = (torch.rand(ndir, 4 * H, H, generator=g) * 2 - 1) * (k * wscale)
    dout = torch.randn(B, T, ndir * H, generator=g)
    for b in range(B):
        dout[b] *= 2.0 ** DOUT_EXPONENTS[b % len(DOUT_EXPONENTS)]
    if B > 2:
        dout[1] = 0.0
    return pre, whh, dout


def _run(pkg, pre, whh, dout, mode):
    """b200asr_bilstm_fwd then _bwd under debug `mode`: (out, cstate, activated-gate stash, dG) on the CPU."""
    L = pkg.lib
    lib = pkg.load_library()
    ndir, B, T, H, _ = pre.shape
    gates = pre.to(DEV).contiguous()
    w = whh.to(DEV).contiguous()
    cst = torch.empty((ndir, B, T, H), device=DEV)
    out = torch.empty((B, T, ndir * H), device=DEV)
    lib.b200asr_debug_set_lstm_mode(mode)
    try:
        nbytes = lib.b200asr_bilstm_workspace_bytes(B, T, H, ndir)     # the plan (and its size) follows the mode
        ws = torch.empty(nbytes, device=DEV, dtype=torch.uint8)
        L.check(lib.b200asr_bilstm_fwd(L.ptr(gates), L.ptr(w), L.ptr(cst), L.ptr(out), B, T, H, ndir, L.ptr(ws),
                                       nbytes, L.stream()), "bilstm_fwd")
        stash = gates.clone()
        dd = dout.to(DEV).contiguous()
        L.check(lib.b200asr_bilstm_bwd(L.ptr(gates), L.ptr(w), L.ptr(cst), L.ptr(dd), B, T, H, ndir, L.ptr(ws),
                                       nbytes, L.stream()), "bilstm_bwd")
    finally:
        lib.b200asr_debug_set_lstm_mode(0)
    return out.cpu(), cst.cpu(), stash.cpu(), gates.cpu()


def _by_row(t, axis):
    t = t.double().movedim(axis, 0)
    return t.reshape(t.shape[0], -1)


NAMES = ("out", "cstate", "gates", "dG")
ROW_AXIS = (0, 1, 1, 1)


def _check_rows(got, r64, r32, what):
    """Per batch row: NaN exactly where float64 has NaN; rows without NaN within K * max(err_fp32, FLOOR) of their own
    scale; a row whose float64 values are all zero is exactly zero.  Returns the worst error / bound and error."""
    worst_ratio, worst_err = 0.0, 0.0
    for name, ax, k, r, f in zip(NAMES, ROW_AXIS, got, r64, r32):
        k, r, f = _by_row(k, ax), _by_row(r, ax), _by_row(f, ax)
        nan = torch.isnan(r)
        assert torch.equal(torch.isnan(k), nan), (what, name, "NaN pattern",
                                                  torch.nonzero(torch.isnan(k) != nan)[:5].tolist())
        for b in range(r.shape[0]):
            if bool(nan[b].any()):
                continue
            scale = float(r[b].abs().max())
            if scale == 0.0:
                assert float(k[b].abs().max()) == 0.0, (what, name, b, "zero row")
                continue
            ek = float((k[b] - r[b]).abs().max()) / scale
            ef = float((f[b] - r[b]).abs().max()) / scale
            bound = K * max(ef, FLOOR)
            assert ek <= bound, (what, name, "row", b, ek, ef, bound)
            worst_ratio = max(worst_ratio, ek / bound)
            worst_err = max(worst_err, ek)
    return worst_ratio, worst_err


def _bits(t):
    return t.contiguous().view(torch.int32)


def _parity(pkg, B, H, ndir, mode, T, seed, wscale=1.0, pre_nan=None, dout_nan=None, twice=True):
    pre, whh, dout = _inputs(B, T, H, ndir, seed, wscale)
    if pre_nan is not None:
        b, t = pre_nan
        pre[0, b, t, H // 3, 1] = float("nan")
    if dout_nan is not None:
        b, t = dout_nan
        dout[b, t, H // 2] = float("nan")
    got = _run(pkg, pre, whh, dout, mode)
    r64 = lstm_ref.recurrence(pre, whh, dout, torch.float64)
    r32 = lstm_ref.recurrence(pre, whh, dout, torch.float32)
    res = _check_rows(got, r64, r32, (B, H, ndir, mode, T))
    if twice:
        # the same inputs again (gates is overwritten in place, so it is filled afresh): bit-identical results
        again = _run(pkg, pre, whh, dout, mode)
        for name, a, b in zip(NAMES, got, again):
            assert torch.equal(_bits(a), _bits(b)), (name, "differs between two runs")
    return res


# ------------------------------------------------------------------------------------------- parity per variant
@pytest.mark.parametrize("B,H,ndir,mode,T,fwd,bwd", CASES, ids=_ids(CASES))
def test_recurrence_vs_fp64_per_row(pkg, B, H, ndir, mode, T, fwd, bwd):
    assert _labels(pkg.load_library(), B, H, ndir, mode) == (fwd, bwd)
    ratio, err = _parity(pkg, B, H, ndir, mode, T, seed=B * 7 + H + mode)
    print("variant %s | %s: worst row error %.3g (%.3g of the bound)" % (fwd, bwd, err, ratio))


# (B, H, ndir, mode) of the time-edge, long-sequence, NaN and W_hh-scale cases: one per generation, and strict acquire
EDGE_SHAPES = [
    (32, 256, 2, 0, "wgmma8/flag/vec", "wgmma8/poll"),
    (32, 256, 2, 256, "wgmma8/flag+strict/vec", "wgmma8/poll"),
    (32, 256, 2, 3, "mma.sync/v2", "mma.sync"),
    (32, 256, 2, 1, "fma1x4", "fma1x4/vec"),
]


@pytest.mark.parametrize("T", [1, 2, 5, 9, 17])
@pytest.mark.parametrize("B,H,ndir,mode,fwd,bwd", EDGE_SHAPES, ids=[str(s[3]) for s in EDGE_SHAPES])
def test_time_edges(pkg, B, H, ndir, mode, fwd, bwd, T):
    """T across the two-image exchange of the flag protocol and the 4-step tag period of the polling backward."""
    assert _labels(pkg.load_library(), B, H, ndir, mode) == (fwd, bwd)
    _parity(pkg, B, H, ndir, mode, T, seed=100 + T, twice=False)


@pytest.mark.parametrize("B,H,ndir,mode,fwd,bwd", EDGE_SHAPES, ids=[str(s[3]) for s in EDGE_SHAPES])
def test_long_sequence(pkg, B, H, ndir, mode, fwd, bwd):
    assert _labels(pkg.load_library(), B, H, ndir, mode) == (fwd, bwd)
    ratio, err = _parity(pkg, B, H, ndir, mode, 300, seed=7, twice=False)
    print("T = 300 %s | %s: worst row error %.3g (%.3g of the bound)" % (fwd, bwd, err, ratio))


@pytest.mark.parametrize("wscale", [0.01, 3.0])
@pytest.mark.parametrize("B,H,ndir,mode,fwd,bwd", EDGE_SHAPES, ids=[str(s[3]) for s in EDGE_SHAPES])
def test_whh_scale(pkg, B, H, ndir, mode, fwd, bwd, wscale):
    """W_hh at 0.01x and 3x the nn.LSTM init scale (1x is every other case)."""
    _parity(pkg, B, H, ndir, mode, 17, seed=11, wscale=wscale, twice=False)


@pytest.mark.parametrize("B,H,ndir,mode,fwd,bwd", EDGE_SHAPES, ids=[str(s[3]) for s in EDGE_SHAPES])
def test_nan_stays_in_its_row(pkg, B, H, ndir, mode, fwd, bwd):
    """A NaN pre-activation in row 3 at frame 4 and a NaN dout in row 6 at frame 2: NaN exactly where float64 has it,
    every other row within the bound."""
    assert _labels(pkg.load_library(), B, H, ndir, mode) == (fwd, bwd)
    _parity(pkg, B, H, ndir, mode, 9, seed=13, pre_nan=(3, 4), dout_nan=(6, 2), twice=False)


@pytest.mark.parametrize("mode,bwd", [(0, "wgmma8/poll"), (3, "mma.sync"), (1, "fma1x4/vec")])
def test_huge_dout_row(pkg, mode, bwd):
    """A dout row at 2^105 (dG near 2^103): each generation keeps it finite and within the bound, like ATen.  The
    wgmma backward scales a row by 2^(13 - e) before its fp16 split; e must not be clamped below the row's exponent."""
    B, H, ndir, T = 32, 256, 2, 9
    assert _labels(pkg.load_library(), B, H, ndir, mode)[1] == bwd
    pre, whh, dout = _inputs(B, T, H, ndir, 17)
    dout[5] = torch.randn(T, ndir * H, generator=torch.Generator().manual_seed(3)) * 2.0 ** 105
    got = _run(pkg, pre, whh, dout, mode)
    assert bool(torch.isfinite(got[3]).all())
    _check_rows(got, lstm_ref.recurrence(pre, whh, dout, torch.float64),
                lstm_ref.recurrence(pre, whh, dout, torch.float32), ("2^105", mode))


# ------------------------------------------------------------------------------------------- through ops.bilstm
@pytest.mark.parametrize("mode,fwd", [(0, "wgmma8/flag/vec"), (3, "mma.sync/v2"), (1, "fma1x4")])
def test_ops_bilstm_vs_fp64_nn_lstm(pkg, mode, fwd):
    """The autograd layer once per generation: output, dx, dW_ih, dW_hh, db_ih, db_hh against torch.nn.LSTM in
    float64, per tensor, with the same bound against nn.LSTM in float32."""
    B, T, I, H = 32, 12, 40, 256
    lib = pkg.load_library()
    assert lstm_ref.label(lstm_ref.variant(lib, B, H, 2, False, mode), False) == fwd
    torch.manual_seed(21)
    ref32 = torch.nn.LSTM(I, H, bidirectional=True, batch_first=True)
    ref64 = torch.nn.LSTM(I, H, bidirectional=True, batch_first=True).double()
    ref64.load_state_dict({k: v.double() for k, v in ref32.state_dict().items()})
    x = torch.randn(B, T, I)
    gy = torch.randn(B, T, 2 * H)
    res = []
    for m, dt in ((ref64, torch.float64), (ref32, torch.float32)):
        xr = x.clone().to(dt).requires_grad_(True)
        y, _ = m(xr)
        y.backward(gy.to(dt))
        res.append([y.detach(), xr.grad] + [p.grad for p in m.parameters()])
    params = [p.detach().clone().to(DEV).requires_grad_(True) for p in ref32.parameters()]
    xg = x.to(DEV).requires_grad_(True)
    lib.b200asr_debug_set_lstm_mode(mode)
    try:
        y = pkg.ops.bilstm(xg, params, 2)
        y.backward(gy.to(DEV))
    finally:
        lib.b200asr_debug_set_lstm_mode(0)
    got = [y.detach().cpu(), xg.grad.cpu()] + [p.grad.cpu() for p in params]
    names = ["out", "dx"] + [n for n, _ in ref32.named_parameters()]
    for name, k, r, f in zip(names, got, *res):
        scale = float(r.abs().max())
        ek = float((k.double() - r).abs().max()) / scale
        ef = float((f.double() - r).abs().max()) / scale
        assert ek <= K * max(ef, FLOOR), (name, ek, ef)
