"""Per-element float64 parity of four step kernels (bounds derived in oracle/step_ref.py, fixed before any run): the
LSTM cell (`b200asr_lstm_cell_fwd / _bwd`, `ops.lstm_cell`), cross-entropy (`b200asr_ce_fwd_bwd`,
`ops.cross_entropy`), the CNN prenet's Conv1d(k 4, s 2, p 1) (`ops.conv1d_k4s2p1`) and CTC prefix scoring
(`b200asr_ctc_prefix_score`, `ctc.CTCPrefixScore`).  Outputs a call must write start as NaN, two runs of every case
are bit-identical, and non-finite outputs appear exactly where float64 has them.  Each case reaches a class no other
case reaches (tests/test_host_step_kernels.py checks the table).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_gpu_gemm_parity as GP
from oracle import oracle_np as onp
from oracle import step_ref as sr

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
INF = float("inf")

# (B, H)
LSTM_CASES = {"b1_h1": (1, 1), "b3_h31": (3, 31), "b5_h1000": (5, 1000), "decoder": (64, 512), "lm": (32, 1024)}
# V; ignore_index is 0 (the project's) except at V = 1, where class 0 is the only target
CE_CASES = {"v%d" % v: v for v in (1, 2, 12, 31, 32, 33, 64, 65, 5000, 16000)}
# (B, T, C, O)
CONV_CASES = {"t2": (3, 2, 120, 640), "t3": (5, 3, 640, 640), "t4": (2, 4, 120, 640), "t5": (3, 5, 640, 640),
              "t41": (3, 41, 120, 640), "t1198": (2, 1198, 120, 640)}
# (T, V, N, C)
PREFIX_CASES = {"t1_v12": (1, 12, 3, 5), "t2_v31": (2, 31, 6, 6), "t37_v12": (37, 12, 6, 8),
                "t299_v5000": (299, 5000, 10, 40)}


def lstm_classes(B, H):
    n = B * H
    out = {"lstm B=%d H=%d" % (B, H)}
    out |= {"lstm one element"} if n == 1 else set()
    out |= {"lstm rows off the warp grid"} if H % 32 and B > 1 else set()
    out |= {"lstm tail block"} if n > 256 and n % 256 else set()
    return out


def ce_classes(V):
    out = {"ce ceil(V/32)=%d, V mod 32=%d" % (-(-V // 32), V % 32)}
    out |= {"ce idle lanes"} if V < 32 else set()
    out |= {"ce V=32k"} if V % 32 == 0 else set()
    out |= {"ce V=32k+1"} if V % 32 == 1 and V > 1 else set()
    return out


def conv_classes(B, T, C, O):
    return {"conv T=%d" % T, "conv T odd" if T % 2 else "conv T even", "conv C=%d" % C}


def prefix_classes(T, V, N, C):
    out = {"prefix T=%d V=%d" % (T, V), "prefix T=%d" % T, "prefix V=%d" % V}
    out |= {"prefix several blocks"} if N * C > 128 else set()
    return out


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _np(t):
    return t.detach().cpu().double().numpy()


WORST = {}


def check(key, got, want, bnd):
    """NaN exactly where float64 has it, +-inf equal, finite elements within the bound; records the worst ratio."""
    got, want, bnd = (np.asarray(a, np.float64) for a in (got, want, bnd))
    assert np.array_equal(np.isnan(got), np.isnan(want)), (key, int(np.isnan(got).sum()), int(np.isnan(want).sum()))
    inf = np.isinf(want)
    assert np.array_equal(got[inf], want[inf]), key
    fin = np.isfinite(want)
    assert np.isfinite(got[fin]).all(), key
    err = np.abs(got[fin] - want[fin])
    ratio = float(np.where(err > 0, err / np.where(err > 0, bnd[fin], 1.0), 0.0).max()) if err.size else 0.0
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    print("worst err/bound %-28s %.3g" % (key, ratio))
    assert ratio <= 1.0, (key, ratio)


# --------------------------------------------------------------------------------------------- LSTM cell
def lstm_inputs(B, H, seed):
    g = torch.Generator().manual_seed(seed)
    pre = 60 * torch.rand(B, 4 * H, generator=g) - 30                           # gates saturate at +-30
    far = torch.rand(B, 4 * H, generator=g) < 0.1
    pre[far] = torch.where(torch.rand(int(far.sum()), generator=g) < 0.5, -100.0, 100.0)   # and at +-100
    c = 1e3 * (2 * torch.rand(B, H, generator=g) - 1)
    c[:, ::3] *= 1e-3                                                            # small c_prev (d pre_f scale)
    dh, dcn = torch.randn(B, H, generator=g), torch.randn(B, H, generator=g)
    rows = {}
    if B >= 3:
        rows = dict(zero_dh=B // 2, nan_pre=B - 1, nan_c=0)
        dh[B // 2] = 0
        pre[B - 1, H // 3] = NAN
        c[0, H // 2] = NAN
    return pre, c, dh, dcn, rows


def lstm_capi(pkg, pre, c_prev, dh, dcn):
    L = pkg.lib
    lib = L.load()
    B, H = c_prev.shape
    pre, c_prev, dh = pre.to(DEV), c_prev.to(DEV), dh.to(DEV)
    gates, c, h = torch.full_like(pre, NAN), torch.full_like(c_prev, NAN), torch.full_like(c_prev, NAN)
    L.check(lib.b200asr_lstm_cell_fwd(L.ptr(pre), L.ptr(c_prev), L.ptr(gates), L.ptr(c), L.ptr(h), B, H, L.stream()))
    out = dict(h=h, c=c, gates=gates)
    for tag, d in (("", None), ("_dcn", dcn.to(DEV))):
        dpre, dcp = torch.full_like(pre, NAN), torch.full_like(c_prev, NAN)
        L.check(lib.b200asr_lstm_cell_bwd(L.ptr(gates), L.ptr(c_prev), L.ptr(c), L.ptr(dh), L.ptr(d), L.ptr(dpre),
                                          L.ptr(dcp), B, H, L.stream()))
        out["dpre" + tag], out["dc_prev" + tag] = dpre, dcp
    return out


@pytest.mark.parametrize("name", list(LSTM_CASES))
def test_lstm_cell_matches_float64(pkg, name):
    B, H = LSTM_CASES[name]
    pre, c_prev, dh, dcn, rows = lstm_inputs(B, H, seed=B * 7 + H)
    out = lstm_capi(pkg, pre, c_prev, dh, dcn)
    out2 = lstm_capi(pkg, pre, c_prev, dh, dcn)
    for k in out:                                                               # run to run: bit identical
        assert torch.equal(_bits(out[k]), _bits(out2[k])), k
    got = {k: _np(v) for k, v in out.items()}
    p64, c64, dh64, dcn64 = (a.double().numpy() for a in (pre, c_prev, dh, dcn))
    h, c, gates = sr.lstm_cell_fwd(p64, c64)
    bh, bc, bg = sr.lstm_cell_fwd_bound(p64, c64)
    check("lstm h", got["h"], h, bh)
    check("lstm c", got["c"], c, bc)
    check("lstm gates", got["gates"], gates, bg)
    # the backward on the kernel's own stash, dc_next NULL and given
    kg, kc = got["gates"], got["c"]
    for tag, d in (("", None), ("_dcn", dcn64)):
        dpre, dcp = sr.lstm_cell_bwd(kg, c64, kc, dh64, d)
        bdpre, bdcp = sr.lstm_cell_bwd_bound(kg, c64, kc, dh64, d)
        check("lstm dpre" + tag, got["dpre" + tag], dpre, bdpre)
        check("lstm dc_prev" + tag, got["dc_prev" + tag], dcp, bdcp)
    # a NaN stays in its own elements: gates column j of the NaN pre row, element j of the NaN c_prev row
    if rows:
        j, jc = H // 3, H // 2
        nan_h = np.isnan(got["h"])
        assert set(zip(*np.nonzero(nan_h))) == {(rows["nan_pre"], j), (rows["nan_c"], jc)}
        assert set(zip(*np.nonzero(np.isnan(got["gates"])))) == {(rows["nan_pre"], j)}
        want = {(rows["nan_pre"], j + k * H) for k in range(4)} | {(rows["nan_c"], jc + k * H) for k in range(4)}
        assert set(zip(*np.nonzero(np.isnan(got["dpre_dcn"])))) == want
    ok = np.ones(B, bool)
    if rows:
        ok[[rows["nan_pre"], rows["nan_c"]]] = False
        z = rows["zero_dh"]
        assert (got["dpre"][z] == 0).all() and (got["dc_prev"][z] == 0).all()       # zero dh, no dc_next: exactly 0
        assert (got["dpre_dcn"][z, 3 * H:] == 0).all()
    sat = (np.abs(p64) >= 100) & ok[:, None]                                     # saturated gates: exactly 0, not NaN
    for tag in ("", "_dcn"):
        assert (got["dpre" + tag][sat] == 0).all()
    # ops.lstm_cell: the same kernels through autograd, both output gradients given
    p = pre.to(DEV).requires_grad_(True)
    cp = c_prev.to(DEV).requires_grad_(True)
    ho, co = pkg.ops.lstm_cell(p, cp)
    assert torch.equal(_bits(ho), _bits(out["h"])) and torch.equal(_bits(co), _bits(out["c"]))
    torch.autograd.backward([ho, co], [dh.to(DEV), dcn.to(DEV)])
    assert torch.equal(_bits(p.grad), _bits(out["dpre_dcn"])) and torch.equal(_bits(cp.grad), _bits(out["dc_prev_dcn"]))


# --------------------------------------------------------------------------------------------- cross-entropy
def ce_inputs(V, seed):
    """40 rows: 30 ordinary (a few with a dominant or a large-magnitude logit, the last class hot in some), 4 ignored
    (one of them holding a NaN), then a NaN logit, +inf on the target, +inf elsewhere, all -inf, -inf on the target
    only and a row with -inf classes around a finite target."""
    ign = 0 if V > 1 else -1
    g = torch.Generator().manual_seed(seed)
    N = 40
    x = 3 * torch.randn(N, V, generator=g)
    x[5:8] *= 30
    tgt = torch.randint(1, V, (N,), generator=g) if V > 1 else torch.zeros(N, dtype=torch.long)
    x[torch.arange(10, 15), tgt[10:15]] += 20
    x[15:18, V - 1] += 15
    tgt[30:34] = ign
    x[31, 0] = NAN
    other = (tgt + 1) % V
    x[34, other[34]] = NAN
    x[35, tgt[35]] = INF
    if V > 1:
        x[36, other[36]] = INF
    x[37] = -INF
    if V > 1:
        x[38, tgt[38]] = -INF
    keep = x[39, tgt[39]].clone()
    x[39, torch.rand(V, generator=g) < 0.3] = -INF
    x[39, tgt[39]] = keep
    return x, tgt, ign


def ce_capi(pkg, x, tgt, ign, scale):
    L = pkg.lib
    lib = L.load()
    N, V = x.shape
    xd, td = x.to(DEV), tgt.to(DEV)
    sc = torch.tensor([scale], device=DEV)
    row, dx = torch.full((N,), NAN, device=DEV), torch.full_like(xd, NAN)
    L.check(lib.b200asr_ce_fwd_bwd(L.ptr(xd), L.ptr(td), ign, N, V, L.ptr(sc), L.ptr(row), L.ptr(dx), L.stream()))
    return row, dx


@pytest.mark.parametrize("name", list(CE_CASES))
def test_cross_entropy_matches_float64(pkg, name):
    V = CE_CASES[name]
    x, tgt, ign = ce_inputs(V, seed=V)
    scale = float(np.float32(0.37))
    row, dx = ce_capi(pkg, x, tgt, ign, scale)
    row2, dx2 = ce_capi(pkg, x, tgt, ign, scale)
    assert torch.equal(_bits(row), _bits(row2)) and torch.equal(_bits(dx), _bits(dx2))
    x64, t64 = x.double().numpy(), tgt.numpy()
    loss, grad = sr.ce_fwd_bwd(x64, t64, scale, ign)
    bl, bg = sr.ce_bounds(x64, t64, scale, ign)
    check("ce row loss", _np(row), loss, bl)
    check("ce dlogits", _np(dx), grad, bg)
    ignored = t64 == ign
    assert (_np(row)[ignored] == 0).all() and (_np(dx)[ignored] == 0).all()
    # NaN rows are float64 ATen's
    xa = x.double().requires_grad_(True)
    rows_a = F.cross_entropy(xa, tgt, ignore_index=ign, reduction="none")
    rows_a.sum().backward()
    assert np.array_equal(np.isnan(_np(row)), np.isnan(rows_a.detach().numpy()))
    valid = ~ignored                                    # ATen's ignored row 31 holds a NaN: its gradient is NaN there
    assert np.array_equal(np.isnan(_np(dx)[valid]), np.isnan(xa.grad.numpy()[valid]))
    # ops.cross_entropy, both reductions and an upstream scale: the whole batch (NaN where ATen is NaN), then the
    # finite rows under the reduced-loss bound
    up = 0.75
    fin = np.isfinite(loss)
    for reduction in ("mean", "sum"):
        xd = x.to(DEV).requires_grad_(True)
        out = pkg.ops.cross_entropy(xd, tgt.to(DEV), ignore_index=ign, reduction=reduction)
        (out * up).backward()
        xa = x.double().requires_grad_(True)
        ref = F.cross_entropy(xa, tgt, ignore_index=ign, reduction=reduction)
        (ref * up).backward()
        assert np.isnan(out.item()) == np.isnan(ref.item())
        n_valid = int((tgt != ign).sum())
        sc = up / n_valid if reduction == "mean" else up
        _, g_or = sr.ce_fwd_bwd(x64, t64, sc, ign)
        _, b_or = sr.ce_bounds(x64, t64, sc, ign)
        assert np.array_equal(np.isnan(g_or[valid]), np.isnan(xa.grad.numpy()[valid]))
        check("ce ops dlogits", _np(xd.grad), g_or, b_or)
        sub = torch.from_numpy(np.nonzero(fin)[0])
        xd = x[sub].to(DEV)
        out = pkg.ops.cross_entropy(xd, tgt[sub].to(DEV), ignore_index=ign, reduction=reduction)
        l64, _ = sr.ce_fwd_bwd(x64[fin], t64[fin], 1.0, ign)
        bl64, _ = sr.ce_bounds(x64[fin], t64[fin], 1.0, ign)
        n = max(int((tgt[sub] != ign).sum()), 1) if reduction == "mean" else 1
        want = l64.sum() / n
        bnd = (bl64.sum() + (len(l64) + 2) * sr.U * np.abs(l64).sum()) / n + 2 * sr.U * abs(want)
        check("ce ops loss", [out.item()], [want], [bnd])


def test_cross_entropy_all_ignored_batch(pkg):
    """Every row ignored: the mean is 0/0 = NaN and the gradient is zero, as in ATen; the sum is 0."""
    x = torch.randn(6, 33)
    tgt = torch.zeros(6, dtype=torch.long)
    for reduction in ("mean", "sum"):
        xd = x.to(DEV).requires_grad_(True)
        out = pkg.ops.cross_entropy(xd, tgt.to(DEV), ignore_index=0, reduction=reduction)
        out.backward()
        xa = x.double().requires_grad_(True)
        ref = F.cross_entropy(xa, tgt, ignore_index=0, reduction=reduction)
        ref.backward()
        assert np.isnan(out.item()) == np.isnan(ref.item()) == (reduction == "mean")
        if reduction == "sum":
            assert out.item() == 0
        assert (xd.grad == 0).all() and (xa.grad == 0).all()


# --------------------------------------------------------------------------------------------- Conv1d k4 s2 p1
def gemm_bound_on_device(lib):
    """step_ref's GEMM-bound callable: the 3xTF32 bound for the plan ops' call of that form makes."""
    def gb(form, A, B, babs):
        M, K = A.shape
        N = B.shape[1]
        if form == "tn":                                   # ops.gemm_tn_ld passes no workspace
            plan = GP.gemm_plan(lib, "tn", M, N, K, 1, 0)
        elif form == "nn":                                 # ops.gemm_nn: split-K only for M <= 256
            plan = GP.gemm_plan(lib, "nn", M, N, K, 1, None if M <= 256 else 0)
        else:
            plan = GP.gemm_plan(lib, "nt", M, N, K, 1)
        S = A.abs() @ B.abs()
        return GP.bound(type("Call", (), dict(form=form, A=A, B=B)), plan, S, 0 if babs is None else babs, 0)
    return gb


def conv_run(pkg, x, conv, dy):
    xd = x.to(DEV).requires_grad_(True)
    conv.weight.grad = conv.bias.grad = None
    y = pkg.ops.conv1d_k4s2p1(xd, conv)
    y.backward(dy.to(DEV))
    return y.detach(), xd.grad, conv.weight.grad.clone(), conv.bias.grad.clone()


def conv_check(pkg, tag, x, conv, dy, exact=False):
    got = conv_run(pkg, x, conv, dy)
    got2 = conv_run(pkg, x, conv, dy)
    for a, b in zip(got, got2):
        assert torch.equal(_bits(a), _bits(b))
    w, b = conv.weight.detach(), conv.bias.detach()
    ref = sr.conv_k4s2(x.to(DEV), w, b, dy.to(DEV))
    bnd = sr.conv_k4s2_bounds(x.to(DEV), w, b, dy.to(DEV), gemm_bound_on_device(pkg.load_library()))
    for k, g in zip(("y", "dx", "dw", "db"), got):
        if exact:
            assert torch.equal(g.double(), ref[k]), k
        check("conv %s %s" % (tag, k), _np(g), ref[k].cpu().numpy(), bnd[k].cpu().numpy())


@pytest.mark.parametrize("name", list(CONV_CASES))
def test_conv1d_k4s2_matches_float64(pkg, name):
    """Each utterance after the first starts with distinct values near 1e6, so a window that reads across the seam
    (the view's last row of an utterance reads the next one) or an overlap-add that lands in the wrong utterance
    shows far above the bound."""
    B, T, C, O = CONV_CASES[name]
    g = torch.Generator().manual_seed(T * 13 + C)
    x = torch.randn(B, T, C, generator=g)
    x[1:, 0] = 1e6 * (1 + torch.rand(B - 1, C, generator=g))
    dy = torch.randn(B, T // 2, O, generator=g)
    dy[1:, 0] = 1e6 * (1 + torch.rand(B - 1, O, generator=g))
    torch.manual_seed(T)
    conv = torch.nn.Conv1d(C, O, 4, stride=2, padding=1).to(DEV)
    conv_check(pkg, "random", x, conv, dy)


def test_conv1d_k4s2_exact_on_the_integer_grid(pkg):
    """Integer operands |x|, |w|, |dy| <= 7 and an integer bias: every partial sum is an fp32 integer far below 2^24, so
    the output and all three gradients equal float64 bit for bit."""
    for B, T, C, O in ((3, 41, 120, 640), (2, 5, 640, 640)):
        g = torch.Generator(device=DEV).manual_seed(T)
        x = GP.grid_operand("int", B * T, C, g).view(B, T, C).cpu()
        dy = GP.grid_operand("int", B * (T // 2), O, g).view(B, T // 2, O).cpu()
        conv = torch.nn.Conv1d(C, O, 4, stride=2, padding=1).to(DEV)
        with torch.no_grad():
            conv.weight.copy_(GP.grid_operand("int", O, 4 * C, g).view(O, C, 4))
            conv.bias.copy_(GP.grid_extra("int", (O,), g))
        conv_check(pkg, "exact", x, conv, dy, exact=True)


def test_cnn_extractor_at_cfg_d_shape(pkg):
    """Both layers of CNNExtractor at cfg D's shape (B = 32, T = 1198, 120 -> 640 -> 640), each against float64 on the
    input it was given (the second layer on the first layer's fp32 output)."""
    from importlib import import_module
    module = import_module("end-to-end-asr-pytorch_b200.module")
    torch.manual_seed(0)
    cnn = module.CNNExtractor(120, 640).to(DEV)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(32, 1198, 120, generator=g)
    c1, c2 = cnn.extractor
    y1 = pkg.ops.conv1d_k4s2p1(x.to(DEV), c1).detach()
    dy2 = torch.randn(32, 299, 640, generator=g)
    feat, flen = cnn(x.to(DEV), torch.full((32,), 1198, device=DEV))
    assert feat.shape == (32, 299, 640) and int(flen[0]) == 299
    y2 = pkg.ops.conv1d_k4s2p1(y1, c2).detach()
    assert torch.equal(_bits(feat), _bits(y2))
    conv_check(pkg, "cfgD layer2", y1.cpu(), c2, dy2)
    conv_check(pkg, "cfgD layer1", x, c1, torch.randn(32, 599, 640, generator=g))


def test_conv1d_library_fallback_for_odd_c_and_t1(pkg):
    """Odd C (a 2C row pitch that is not 16-byte aligned) and T = 1 (no full window) take the library convolution:
    odd C computes it, T = 1 raises the library's error, and neither launches a kernel of this library."""
    from test_gpu_kernels import _kernel_names
    conv = torch.nn.Conv1d(7, 16, 4, stride=2, padding=1).to(DEV)
    x = torch.randn(2, 9, 7, device=DEV)
    names = _kernel_names(pkg, lambda: pkg.ops.conv1d_k4s2p1(x, conv))
    assert not names & {"gemm3x_tn", "gemm3x_nn", "gemm3x_nt"}, names
    y = pkg.ops.conv1d_k4s2p1(x, conv)
    ref = F.conv1d(x.double().transpose(1, 2), conv.weight.double(), conv.bias.double(), stride=2,
                   padding=1).transpose(1, 2)
    assert y.shape == ref.shape == (2, 4, 16)
    conv = torch.nn.Conv1d(120, 16, 4, stride=2, padding=1).to(DEV)
    before = pkg.lib.launch_count()
    with pytest.raises(RuntimeError):
        pkg.ops.conv1d_k4s2p1(torch.randn(3, 1, 120, device=DEV), conv)
    assert pkg.lib.launch_count() == before


# --------------------------------------------------------------------------------------------- CTC prefix scoring
def prefix_inputs(T, V, N, C, seed):
    """Log-probs with -inf entries (and frames where a candidate and blank are both -inf), prefixes of length 0, 1, 2,
    T-1, T and T+2, candidates that include the last token, blank and eos (and once the last token twice)."""
    rng = np.random.default_rng(seed)
    x = torch.log_softmax(torch.from_numpy(rng.standard_normal((T, V)) * 3), -1).float().numpy()
    x[rng.random((T, V)) < 0.05] = -np.inf
    both = rng.random(T) < 0.2
    x[both, 0] = -np.inf
    x[both, 2] = -np.inf
    lens = [0, 1, 2, T - 1, T, T + 2]
    prefixes, cands = [], []
    for n in range(N):
        plen = max(lens[n % len(lens)], 0)
        g = list(rng.integers(2, V, plen)) if V > 2 else [2] * plen
        prefixes.append([int(v) for v in g])
        c = [0, 1, 2] + [int(v) for v in rng.permutation(np.arange(3, V))[:C - 3]] if V > 3 else [0, 1, 2]
        c = (c + [int(v) for v in rng.integers(0, V, C)])[:C]
        if g:
            c[3 % C] = g[-1]
            if n == 3:
                c[4 % C] = g[-1]
        cands.append(c)
    r_prev = rng.uniform(-60, 0, (N, T, 2)).astype(np.float32)
    r_prev[rng.random((N, T, 2)) < 0.1] = sr.LOGZERO
    r_prev[rng.random((N, T, 2)) < 0.05] = -np.inf
    return x, r_prev, prefixes, np.asarray(cands, np.int32)


def prefix_capi(pkg, x, r_prev, prefixes, cands, eos):
    L = pkg.lib
    lib = L.load()
    T, V = x.shape
    N, C = cands.shape
    xd, rp = torch.from_numpy(x).to(DEV), torch.from_numpy(r_prev).to(DEV)
    last = torch.tensor([g[-1] if g else 0 for g in prefixes], dtype=torch.int32, device=DEV)
    plen = torch.tensor([len(g) for g in prefixes], dtype=torch.int32, device=DEV)
    cd = torch.from_numpy(cands).to(DEV)
    psi, r = torch.full((N, C), NAN, device=DEV), torch.full((N, C, T, 2), NAN, device=DEV)
    L.check(lib.b200asr_ctc_prefix_score(L.ptr(xd), T, V, L.ptr(rp), L.ptr(last), L.ptr(plen), L.ptr(cd), N, C, 0,
                                         eos, L.ptr(psi), L.ptr(r), L.stream()))
    return psi, r


@pytest.mark.parametrize("name", list(PREFIX_CASES))
def test_prefix_score_matches_float64(pkg, name):
    T, V, N, C = PREFIX_CASES[name]
    x, r_prev, prefixes, cands = prefix_inputs(T, V, N, C, seed=T + V)
    for eos in (1, -1):
        psi, r = prefix_capi(pkg, x, r_prev, prefixes, cands, eos)
        psi2, r2 = prefix_capi(pkg, x, r_prev, prefixes, cands, eos)
        assert torch.equal(_bits(psi), _bits(psi2)) and torch.equal(_bits(r), _bits(r2))
        wpsi, wr, bpsi, br = sr.prefix_score(x, r_prev, prefixes, cands, 0, eos)
        check("prefix psi", _np(psi), wpsi, bpsi)
        check("prefix r", _np(r), wr, br)
    # the same through CTCPrefixScore.cheap_compute_batch (blank 0, eos 1)
    sc = pkg.ctc.CTCPrefixScore(torch.from_numpy(x)[None].to(DEV))
    psi_b, r_b = sc.cheap_compute_batch(prefixes, torch.from_numpy(r_prev).to(DEV), cands.tolist())
    psi, r = prefix_capi(pkg, x, r_prev, prefixes, cands, 1)
    assert torch.equal(_bits(psi_b), _bits(psi)) and torch.equal(_bits(r_b), _bits(r))


def test_prefix_score_chain_matches_reference_scorer(pkg):
    """Five steps driven like the reference's decoder (init_state, then extend the best non-eos candidate), each step
    against oracle_np's float32 restatement of the reference's scorer within twice the propagated bound (both are
    within it of float64) on the kernel's own r_prev.  No duplicate candidates and |g| < T: the reference's
    first-occurrence rule and its psi view at |g| = T (oracle/step_ref.py) do not arise here."""
    T, V = 37, 12
    rng = np.random.default_rng(5)
    x = torch.log_softmax(torch.from_numpy(rng.standard_normal((T, V)) * 2), -1).float().numpy()
    x[rng.random((T, V)) < 0.05] = -np.inf
    sc = pkg.ctc.CTCPrefixScore(torch.from_numpy(x)[None].to(DEV))
    r_prev = sc.init_state().cpu().numpy()
    assert np.array_equal(r_prev, onp.ctc_prefix_init(x))
    prefix = []
    for step in range(5):
        cands = [1, 0] + [int(v) for v in rng.permutation(np.arange(2, V))[:4]]
        if prefix and prefix[-1] not in cands:
            cands[2] = prefix[-1]
        psi, r = sc.cheap_compute(prefix, r_prev, cands)
        rpsi, rr = onp.ctc_prefix_cheap(x, prefix, r_prev, cands)
        _, _, bpsi, br = sr.prefix_score(x, r_prev[None], [prefix], [cands])
        check("prefix chain psi", psi, rpsi, 2 * bpsi[0])
        check("prefix chain r", r, rr, 2 * br[0])
        order = [i for i in np.argsort(-psi) if cands[i] != 1]
        best = order[0]
        prefix = prefix + [cands[best]]
        r_prev = r[best]


def test_prefix_score_refuses_ids_outside_the_vocabulary(pkg):
    """Candidate ids and prefix tokens outside [0, V) raise on the host before any launch (the kernel would gather
    log-probs outside x)."""
    T, V = 7, 12
    x = torch.log_softmax(torch.randn(1, T, V), -1).to(DEV)
    sc = pkg.ctc.CTCPrefixScore(x)
    r0 = sc.init_state()
    before = pkg.lib.launch_count()
    for prefixes, cands in (([[]], [[2, V]]), ([[]], [[-1, 3]]), ([[3, V + 4]], [[2, 3]]), ([[-2]], [[2, 3]])):
        with pytest.raises(ValueError):
            sc.cheap_compute_batch(prefixes, r0[None], cands)
    assert pkg.lib.launch_count() == before
