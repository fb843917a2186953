"""CPU checks for tests/test_gpu_step_kernels.py: oracle/step_ref.py against float64 autograd of the reference's
expressions (nn.LSTMCell, F.cross_entropy(ignore_index=0), F.conv1d(stride=2, padding=1)) and against a float64
restatement of the reference's numpy CTCPrefixScore.cheap_compute; an fp32 emulation of each kernel's arithmetic
stays within half of every bound, and planted defects exceed it at least 10x; the GPU file's case table has no
redundant case.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_gpu_gemm_parity as GP
import test_gpu_step_kernels as G
import test_host_gemm_bounds as HG
from oracle import step_ref as sr

F32 = np.float32


def ratio(got, want, bnd):
    """max err / bound over the elements where float64 is finite (0 where the error is 0)."""
    got, want, bnd = (np.asarray(a, np.float64) for a in (got, want, bnd))
    fin = np.isfinite(want)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    err = np.abs(got[fin] - want[fin])
    return float(np.where(err > 0, err / np.where(err > 0, bnd[fin], 1.0), 0.0).max()) if err.size else 0.0


# ------------------------------------------------------------------------------------------------ oracle vs autograd
def test_lstm_oracle_matches_lstmcell_autograd():
    torch.manual_seed(0)
    B, I, H = 5, 7, 6
    cell = torch.nn.LSTMCell(I, H).double()
    x = torch.randn(B, I, dtype=torch.float64)
    h0 = torch.randn(B, H, dtype=torch.float64)
    c0 = (3 * torch.randn(B, H, dtype=torch.float64)).requires_grad_(True)
    h1, c1 = cell(x, (h0, c0))
    dh, dc = torch.randn(B, H, dtype=torch.float64), torch.randn(B, H, dtype=torch.float64)
    torch.autograd.backward([h1, c1], [dh, dc])
    with torch.no_grad():
        pre = (x @ cell.weight_ih.t() + cell.bias_ih + h0 @ cell.weight_hh.t() + cell.bias_hh).numpy()
    h, c, gates = sr.lstm_cell_fwd(pre, c0.detach().numpy())
    assert np.abs(h - h1.detach().numpy()).max() < 1e-14 and np.abs(c - c1.detach().numpy()).max() < 1e-14
    dpre, dcp = sr.lstm_cell_bwd(gates, c0.detach().numpy(), c, dh.numpy(), dc.numpy())
    assert np.abs(dcp - c0.grad.numpy()).max() < 1e-13
    assert np.abs(dpre.T @ x.numpy() - cell.weight_ih.grad.numpy()).max() < 1e-13
    assert np.abs(dpre.sum(0) - cell.bias_hh.grad.numpy()).max() < 1e-13
    # without dc_next the same as a zero dc_next
    a, b = sr.lstm_cell_bwd(gates, c0.detach().numpy(), c, dh.numpy())
    a0, b0 = sr.lstm_cell_bwd(gates, c0.detach().numpy(), c, dh.numpy(), np.zeros((B, H)))
    assert np.array_equal(a, a0) and np.array_equal(b, b0)


@pytest.mark.parametrize("V", [1, 12, 33, 5000])
def test_ce_oracle_matches_aten(V):
    """Every row of the GPU file's inputs (non-finite rows included): loss, gradient and their NaN pattern."""
    x, tgt, ign = G.ce_inputs(V, seed=V)
    xa = x.double().requires_grad_(True)
    rows = F.cross_entropy(xa, tgt, ignore_index=ign, reduction="none")
    (0.37 * rows.sum()).backward()
    loss, grad = sr.ce_fwd_bwd(x.double().numpy(), tgt.numpy(), 0.37, ign)
    want_l, want_g = rows.detach().numpy(), xa.grad.numpy()
    ignored = tgt.numpy() == ign                                  # ATen: NaN gradient in an ignored row holding a NaN
    assert np.isnan(want_g[31]).all() and (grad[ignored] == 0).all()
    want_g = np.where(ignored[:, None], 0.0, want_g)
    assert np.array_equal(np.isnan(loss), np.isnan(want_l)) and np.array_equal(np.isnan(grad), np.isnan(want_g))
    fin = ~np.isnan(want_l)
    assert np.array_equal(np.isinf(loss[fin]), np.isinf(want_l[fin]))
    ok = np.isfinite(want_l)
    assert np.abs(loss[ok] - want_l[ok]).max() < 1e-12
    ok = np.isfinite(want_g)
    assert np.abs(grad[ok] - want_g[ok]).max() < 1e-12
    if V > 1:                                                     # the project's ignore_index = 0 on finite rows
        xf = torch.randn(8, V, dtype=torch.float64, requires_grad=True)
        t = torch.tensor([0, 1, V - 1, 0, 2 % V, 1, 1, 0])
        F.cross_entropy(xf, t, ignore_index=0).backward()
        n = int((t != 0).sum())
        l, g = sr.ce_fwd_bwd(xf.detach().numpy(), t.numpy(), 1.0 / n)
        assert abs(l.sum() / n - F.cross_entropy(xf, t, ignore_index=0).item()) < 1e-13
        assert np.abs(g - xf.grad.numpy()).max() < 1e-13


@pytest.mark.parametrize("B,T,C,O", [(3, 2, 4, 5), (2, 3, 6, 3), (3, 5, 4, 2), (2, 41, 8, 5)])
def test_conv_oracle_matches_conv1d_autograd(B, T, C, O):
    torch.manual_seed(T)
    x = torch.randn(B, T, C, dtype=torch.float64, requires_grad=True)
    w = torch.randn(O, C, 4, dtype=torch.float64, requires_grad=True)
    b = torch.randn(O, dtype=torch.float64, requires_grad=True)
    y = F.conv1d(x.transpose(1, 2), w, b, stride=2, padding=1).transpose(1, 2)
    dy = torch.randn_like(y)
    y.backward(dy)
    ref = sr.conv_k4s2(x.detach(), w.detach(), b.detach(), dy)
    for k, want in (("y", y.detach()), ("dx", x.grad), ("dw", w.grad), ("db", b.grad)):
        assert ref[k].shape == want.shape and float((ref[k] - want).abs().max()) < 1e-12, k


def reference_cheap_compute(x, g, r_prev, candidates, blank=0, eos=1, logzero=sr.LOGZERO):
    """The reference's CTCPrefixScore.cheap_compute (src/ctc.py:81-116) statement by statement in float64, numpy view
    semantics and first-occurrence `index` included."""
    x, r_prev = np.asarray(x, np.float64), np.asarray(r_prev, np.float64)
    T = x.shape[0]
    odim = len(candidates)
    r = np.full((T, 2, odim), logzero)
    start = max(1, len(g))
    if len(g) == 0:
        r[0, 0, :] = x[0, candidates]
    psi = r[start - 1, 0, :]                                   # a view (raises IndexError for len(g) > T)
    sum_prev = np.logaddexp(r_prev[:, 0], r_prev[:, 1])
    phi = np.repeat(sum_prev[..., None], odim, axis=-1)
    if len(g) > 0 and g[-1] in candidates:
        phi[:, candidates.index(g[-1])] = r_prev[:, 1]
    for t in range(start, T):
        r[t, 0, :] = np.logaddexp(r[t - 1, 0, :], phi[t - 1]) + x[t, candidates]
        r[t, 1, :] = np.logaddexp(r[t - 1, 1, :], r[t - 1, 0, :]) + x[t, blank]
        psi = np.logaddexp(psi, phi[t - 1] + x[t, candidates])
    if eos in candidates:
        psi[candidates.index(eos)] = sum_prev[-1]
    return psi, np.rollaxis(r, 2)


@pytest.mark.parametrize("name", ["t1_v12", "t2_v31", "t37_v12"])
def test_prefix_oracle_matches_reference_scorer(name):
    """Equal to the reference's scorer except where the module docstring says: every occurrence of a duplicated last
    token (and eos) is special, r[T-1, 0, eos] is not written at max(|g|, 1) = T, and |g| > T scores log-zero where the
    reference raises."""
    T, V, N, C = G.PREFIX_CASES[name]
    x, r_prev, prefixes, cands = G.prefix_inputs(T, V, N, C, seed=T + V)
    psi, r, _, _ = sr.prefix_score(x, r_prev, prefixes, cands)
    checked = 0
    for n, g in enumerate(prefixes):
        cl = [int(v) for v in cands[n]]
        if len(g) > T:
            with pytest.raises(IndexError):
                reference_cheap_compute(x, g, r_prev[n], cl)
            assert (r[n] == sr.LOGZERO).all() and (psi[n][np.array(cl) != 1] == sr.LOGZERO).all()
            continue
        rpsi, rr = reference_cheap_compute(x, g, r_prev[n], cl)
        rpsi = rpsi.copy()                                                      # may be a view of r
        keep = np.ones(C, bool)
        for c in set(cl):
            if (g and c == g[-1]) or c == 1:
                keep[[i for i, v in enumerate(cl) if v == c][1:]] = False      # later duplicates
        if max(len(g), 1) == T and 1 in cl:
            rr[cl.index(1), T - 1, 0] = r[n, cl.index(1), T - 1, 0]            # the reference's view write
        with np.errstate(invalid="ignore"):
            assert np.allclose(psi[n][keep], rpsi[keep], rtol=0, atol=1e-9, equal_nan=True)
            assert np.allclose(r[n][keep], rr[keep], rtol=0, atol=1e-9, equal_nan=True)
        checked += 1
    assert checked >= 2


# ------------------------------------------------------------------------------------------------ fp32 emulations
def fma(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def emu_lstm(pre, c_prev, dh, dcn, defect=None):
    """csrc/lstm.cu lstm_cell_fwd / _bwd in fp32 (numpy float32 exp / tanh)."""
    pre, c_prev, dh = (np.asarray(a, F32) for a in (pre, c_prev, dh))
    H = c_prev.shape[1]
    with np.errstate(over="ignore"):
        sig = lambda a: (F32(1) / (F32(1) + np.exp(-a))).astype(F32)          # noqa: E731
        i, f, o = sig(pre[:, :H]), sig(pre[:, H:2 * H]), sig(pre[:, 3 * H:])
    g = np.tanh(pre[:, 2 * H:3 * H])
    c = fma(f, c_prev, i * g)
    h = o * np.tanh(c)
    tc = np.tanh(c)
    dc = dh * o * (F32(1) - tc * tc)
    if dcn is not None and defect != "dc_next ignored":
        dc = dc + np.asarray(dcn, F32)
    a, b = (f, i) if defect == "f and i swapped in d pre" else (i, f)
    dpre = np.concatenate([dc * g * a * (F32(1) - a), dc * c_prev * b * (F32(1) - b), dc * i * (F32(1) - g * g),
                           dh * tc * o * (F32(1) - o)], 1)
    return h, c, np.concatenate([i, f, g, o], 1), dpre, dc * f


def lstm_ratios(defect=None):
    worst = {}
    for B, H in ((5, 1000), (3, 31)):
        pre, c_prev, dh, dcn, _ = G.lstm_inputs(B, H, seed=B * 7 + H)
        p, cp, d, dn = (a.numpy() for a in (pre, c_prev, dh, dcn))
        h, c, gates, dpre, dcp = emu_lstm(p, cp, d, dn, defect)
        wh, wc, wg = sr.lstm_cell_fwd(p.astype(np.float64), cp.astype(np.float64))
        bh, bc, bg = sr.lstm_cell_fwd_bound(p.astype(np.float64), cp.astype(np.float64))
        rdpre, rdcp = sr.lstm_cell_bwd(gates, cp, c, d, dn)
        bdpre, bdcp = sr.lstm_cell_bwd_bound(gates, cp, c, d, dn)
        for k, r in (("h", ratio(h, wh, bh)), ("c", ratio(c, wc, bc)), ("gates", ratio(gates, wg, bg)),
                     ("dpre", ratio(dpre, rdpre, bdpre)), ("dc_prev", ratio(dcp, rdcp, bdcp))):
            worst[k] = max(worst.get(k, 0.0), r)
    return worst


def emu_ce(x, tgt, ign, scale, defect=None):
    """csrc/ce.cu in fp32: one warp per row, lane l holds logits l, l + 32, ... with an online (m, s), the xor tree."""
    x = np.asarray(x, F32)
    N, V = x.shape
    n = -(-V // 32)
    xl = np.full((N, n * 32), -np.inf, F32)
    xl[:, :V] = x
    if defect == "lse over V-1 classes":
        xl[:, V - 1] = -np.inf
    xl = xl.reshape(N, n, 32)
    m = np.full((N, 32), -np.inf, F32)
    s = np.zeros((N, 32), F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(n):
            v = xl[:, k]
            up = v > m
            s_up = fma(s, np.exp(m - v), F32(1))
            s_add = np.where(v != -np.inf, s + np.exp(v - m), s).astype(F32)
            s = np.where(up, s_up, s_add).astype(F32)
            m = np.where(up, v, m)
        M = np.fmax.reduce(m, axis=1)[:, None]
        t = (s * np.where(m == -np.inf, F32(0), np.exp(m - M))).astype(F32)
        for o in (16, 8, 4, 2, 1):
            t = (t + t[:, np.arange(32) ^ o]).astype(F32)
        lse = (M[:, 0] + np.log(t[:, 0])).astype(F32)
        rows = np.arange(N)
        keep = (tgt != ign) & (tgt >= 0) & (tgt < V)
        tt = np.where(keep, tgt, 0)
        loss = np.where(keep, lse - x[rows, tt], F32(0))
        p = np.exp(x - lse[:, None]).astype(F32)
    oh = tt + 1 if defect == "onehot at t + 1" else tt
    p[rows, np.minimum(oh, V - 1)] -= np.where(oh < V, F32(1), F32(0))
    dx = np.where(keep[:, None], p * F32(scale), F32(0))
    return loss, dx


def ce_ratios(defect=None):
    worst = {}
    for V in (12, 33, 5000):
        x, tgt, ign = G.ce_inputs(V, seed=V)
        x64, t = x.double().numpy(), tgt.numpy()
        loss, dx = emu_ce(x.numpy(), t, ign, 0.375, defect)
        wl, wg = sr.ce_fwd_bwd(x64, t, 0.375, ign)
        bl, bg = sr.ce_bounds(x64, t, 0.375, ign)
        for k, r in (("loss", ratio(loss, wl, bl)), ("dx", ratio(dx, wg, bg))):
            worst[k] = max(worst.get(k, 0.0), r)
    return worst


def emu_gemm_bound(form, A, B, babs):
    """The 3xTF32 bound at the plan the emulation runs (one slice, chunks of 4 K blocks)."""
    M, K = A.shape
    plan = dict(nsplit=1, KB=-(-K // 32), chunk=4)
    return GP.bound(type("Call", (), dict(form=form, A=A, B=B)), plan, A.abs() @ B.abs(), 0 if babs is None else babs, 0)


def emu_conv(x, w, b, dy, defect=None):
    """Conv1dK4S2Fn's three GEMMs with test_host_gemm_bounds.emulate's 3xTF32 arithmetic, the overlap-add and the
    bias sum in fp32."""
    B, T, C = x.shape
    O = w.shape[0]
    Tout, half, Tp, M = sr.conv_geometry(B, T)
    A = sr.conv_view(x.double())
    if defect == "taps shifted one frame":
        A = torch.cat([A[:, C:], A.new_zeros(A.shape[0], C)], 1)
    A = A.numpy()
    wm = sr.conv_weight_matrix(w.double()).numpy()
    y = np.zeros((B * half, O))
    y[:M] = HG.emulate(A[:M], wm.T, b.double().numpy(), np.zeros((M, O)))
    dyf = np.zeros((B, half, O))
    dyf[:, :Tout] = dy.double().numpy()
    dy2 = dyf.reshape(B * half, O)
    dcols = HG.emulate(dy2, wm, np.zeros(4 * C), np.zeros((B * half, 4 * C))).reshape(B, half, 2, 2 * C)
    dxp = np.zeros((B, half + 1, 2 * C), F32)
    dxp[:, :half] += dcols[:, :, 0].astype(F32)
    if defect != "overlap-add seam dropped":
        dxp[:, 1:] += dcols[:, :, 1].astype(F32)
    dx = dxp.reshape(B, Tp + 2, C)[:, 1:T + 1]
    dwm = HG.emulate(dy2[:M].T, A[:M], np.zeros(4 * C), np.zeros((O, 4 * C)))
    dw = dwm.reshape(O, 4, C).transpose(0, 2, 1)
    db = dy.numpy().astype(F32).reshape(-1, O).sum(0, dtype=F32)
    return dict(y=y.reshape(B, half, O)[:, :Tout], dx=dx, dw=dw, db=db)


def conv_ratios(defect=None):
    worst = {}
    for B, T, C, O in ((3, 5, 8, 6), (2, 2, 4, 5), (3, 8, 40, 16)):
        g = torch.Generator().manual_seed(T)
        x = torch.randn(B, T, C, generator=g)
        x[1:, 0] = 1e6 * (1 + torch.rand(B - 1, C, generator=g))
        dy = torch.randn(B, T // 2, O, generator=g)
        dy[1:, 0] = 1e6 * (1 + torch.rand(B - 1, O, generator=g))
        w, b = torch.randn(O, C, 4, generator=g), torch.randn(O, generator=g)
        got = emu_conv(x, w, b, dy, defect)
        ref = sr.conv_k4s2(x, w, b, dy)
        bnd = sr.conv_k4s2_bounds(x, w, b, dy, emu_gemm_bound)
        for k in ("y", "dx", "dw", "db"):
            worst[k] = max(worst.get(k, 0.0), ratio(got[k], ref[k].numpy(), bnd[k].numpy()))
    return worst


def emu_prefix(x, r_prev, prefixes, cands, blank=0, eos=1, defect=None):
    """csrc/prefix.cu in fp32 (numpy's float32 logaddexp is the kernel's formula with the a == b branch)."""
    x, r_prev = np.asarray(x, F32), np.asarray(r_prev, F32)
    cands = np.asarray(cands)
    N, C = cands.shape
    T = x.shape[0]
    lae = np.logaddexp
    plen = np.array([len(g) for g in prefixes])
    last = np.array([g[-1] if g else -1 for g in prefixes])
    same = (plen[:, None] > 0) & (cands == last[:, None]) & (defect != "phi not switched for the last token")
    start = np.maximum(plen, 1)
    lz = F32(sr.LOGZERO)
    r = np.full((N, C, T, 2), lz, F32)
    r0 = np.where(plen[:, None] == 0, x[0][cands], lz).astype(F32)
    r[:, :, 0, 0] = r0
    q0 = np.where((start == 1)[:, None], r0, lz).astype(F32)
    q1 = np.full((N, C), lz, F32)
    psi = q0.copy()
    with np.errstate(invalid="ignore"):
        for t in range(1, T):
            live = (t >= start)[:, None]
            p0, p1 = r_prev[:, t - 1, 0][:, None], r_prev[:, t - 1, 1][:, None]
            phi = np.where(same, p1, lae(p0, p1)).astype(F32)
            xc, xb = x[t][cands], x[t, blank]
            n0, n1 = lae(q0, phi) + xc, lae(q1, q0) + xb
            npsi = lae(psi, phi + xc)
            q0, q1, psi = np.where(live, n0, q0), np.where(live, n1, q1), np.where(live, npsi, psi)
            r[:, :, t, 0] = np.where(live, q0, r[:, :, t, 0])
            r[:, :, t, 1] = np.where(live, q1, r[:, :, t, 1])
    if defect != "psi not reset for eos":
        psi = np.where(cands == eos, lae(r_prev[:, T - 1, 0], r_prev[:, T - 1, 1])[:, None], psi)
    return psi, r


def prefix_ratios(defect=None):
    worst = {}
    for name in ("t37_v12", "t299_v5000"):
        T, V, N, C = G.PREFIX_CASES[name]
        x, r_prev, prefixes, cands = G.prefix_inputs(T, V, N, C, seed=T + V)
        psi, r = emu_prefix(x, r_prev, prefixes, cands, defect=defect)
        wpsi, wr, bpsi, br = sr.prefix_score(x, r_prev, prefixes, cands)
        for k, rt in (("psi", ratio(psi, wpsi, bpsi)), ("r", ratio(r, wr, br))):
            worst[k] = max(worst.get(k, 0.0), rt)
    return worst


RATIOS = {"lstm": lstm_ratios, "ce": ce_ratios, "conv": conv_ratios, "prefix": prefix_ratios}
DEFECTS = [("lstm", "f and i swapped in d pre", "dpre"), ("lstm", "dc_next ignored", "dpre"),
           ("lstm", "dc_next ignored", "dc_prev"),
           ("ce", "onehot at t + 1", "dx"), ("ce", "lse over V-1 classes", "loss"), ("ce", "lse over V-1 classes", "dx"),
           ("conv", "taps shifted one frame", "y"), ("conv", "taps shifted one frame", "dw"),
           ("conv", "overlap-add seam dropped", "dx"),
           ("prefix", "phi not switched for the last token", "r"), ("prefix", "phi not switched for the last token",
                                                                     "psi"),
           ("prefix", "psi not reset for eos", "psi")]


@pytest.mark.parametrize("kernel", list(RATIOS))
def test_fp32_emulation_sits_inside_the_bounds(kernel):
    worst = RATIOS[kernel]()
    print(kernel, worst)
    assert max(worst.values()) <= 0.5, worst


@pytest.mark.parametrize("kernel,defect,output", DEFECTS)
def test_bounds_reject_planted_defects(kernel, defect, output):
    try:
        worst = RATIOS[kernel](defect)
    except AssertionError:                  # a defect that moves a NaN is caught by the NaN pattern already
        return
    assert worst[output] >= 10, worst


def test_prefix_fix_matches_numpy_logaddexp():
    """numpy's float32 logaddexp returns a + ln 2 for a == b (so -inf for two -inf); the kernel's formula without that
    branch gives NaN there, which this case table's inputs reach."""
    with np.errstate(invalid="ignore"):
        a = F32(-np.inf)
        assert np.logaddexp(a, a) == -np.inf
        assert np.isnan(a + np.log1p(np.exp(-np.abs(a - a))))
    x, r_prev, prefixes, cands = G.prefix_inputs(37, 12, 6, 8, seed=49)
    _, r, _, _ = sr.prefix_score(x, r_prev, prefixes, cands)
    assert (r == -np.inf).any() and not np.isnan(r).any()


# ------------------------------------------------------------------------------------------------ case table
def test_gpu_cases_reach_every_class():
    """Each GPU case reaches a class no other case of its kernel reaches, and together they reach every listed one."""
    tables = {"lstm": {n: G.lstm_classes(*c) for n, c in G.LSTM_CASES.items()},
              "ce": {n: G.ce_classes(c) for n, c in G.CE_CASES.items()},
              "conv": {n: G.conv_classes(*c) for n, c in G.CONV_CASES.items()},
              "prefix": {n: G.prefix_classes(*c) for n, c in G.PREFIX_CASES.items()}}
    required = {"lstm one element", "lstm rows off the warp grid", "lstm tail block", "lstm B=64 H=512",
                "lstm B=32 H=1024", "ce idle lanes", "ce V=32k", "ce V=32k+1", "ce ceil(V/32)=1, V mod 32=1",
                "ce ceil(V/32)=1, V mod 32=12", "ce ceil(V/32)=3, V mod 32=1", "ce ceil(V/32)=500, V mod 32=0",
                "conv T odd", "conv T even", "conv C=120", "conv C=640", "prefix several blocks", "prefix V=5000"}
    required |= {"conv T=%d" % t for t in (2, 3, 4, 5, 41, 1198)} | {"prefix T=%d" % t for t in (1, 2, 37, 299)} | {"prefix V=%d" % v for v in (12, 31)}
    reached = set()
    for kernel, tab in tables.items():
        for name, r in tab.items():
            others = set().union(*(x for n, x in tab.items() if n != name))
            assert r - others, (kernel, name)
            reached |= r
    assert not required - reached, required - reached
