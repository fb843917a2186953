"""Every kernel variant the host dispatchers choose among, at the sizes the train step runs, against float64 references.

The CTC lattice dispatcher picks a kernel by the padded target width, the location-attention backward by batch size and
dimensions, and the log-softmax kernels by alignment; each test here pins which variant it reaches (through the debug
queries of include/b200asr_debug.h) so that moving a threshold cannot silently drop a variant from the suite.

Bounds come from fp32 rounding (EPS = 2^-24, the unit roundoff) of the computation under test and are fixed here,
independent of what any run measured:
  * CTC: a T-step fp32 lattice carries at most about T roundings of the log-domain values, each <= EPS * |lattice|, and
    |lattice| <= |nll|.  So nll is within T * EPS relative, and each gradient element (an exp of alpha + beta + nll - lp,
    times the row weight) within T * EPS * |nll| of the row weight.
  * log-softmax / cross-entropy: per-lane sums of V / 32 exponentials, a 5-level shuffle tree, exp / log within 2 ulp.
  * attention: contractions of at most n = max(T, D, E, K * (2R + 1)) fp32 terms, n * EPS of the tensor's scale.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden, scaled_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24


def _bits(t):
    """Bit pattern of an fp32 tensor (NaN-aware equality)."""
    return t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------- CTC
CTC_WIDTHS = [15, 16, 47, 48, 63, 64, 141, 511, 512, 600]


def test_ctc_widths_cover_every_lattice_variant(pkg):
    """1-4: warp kernel with R positions per lane; 5: block kernel, one position per thread; 6: strided block kernel.
    (L_max = 600 also needs more than 48 KB of shared memory in the gradient kernel: S = 1201 positions.)"""
    lib = pkg.load_library()
    got = {L: lib.b200asr_debug_ctc_variant(L) for L in CTC_WIDTHS}
    assert set(got.values()) == {1, 2, 3, 4, 5, 6}, got
    assert got[63] == 4 and got[64] == 5 and got[511] == 5 and got[512] == 6, got


def _no_repeat(n, hi, g):
    """n labels in [1, hi) without adjacent repeats."""
    out = []
    for _ in range(n):
        c = int(torch.randint(1, hi, (1,), generator=g))
        if out and c == out[-1]:
            c = c % (hi - 1) + 1
        out.append(c)
    return out


def _frames_needed(t):
    return len(t) + sum(1 for i in range(1, len(t)) if t[i] == t[i - 1])


def _ctc_batch(B, T, V, Lmax, seed):
    """Logits and a batch that mixes the edge rows: 0 empty target; 1 exactly feasible with adjacent repeats;
    2 long occurrence chains (3 classes); 3 the target of row 1 one frame short (infeasible); 4 input_length 0 with a
    non-empty target; the rest random targets and input lengths (mostly < T)."""
    assert B >= 5
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, T, V, generator=g)
    txt = torch.zeros(B, Lmax, dtype=torch.long)
    tl = torch.zeros(B, dtype=torch.long)
    il = torch.full((B,), T, dtype=torch.long)
    rep = _no_repeat(Lmax, V, g)
    for j in range(max(1, min(Lmax // 8, T - Lmax))):
        rep[2 * j + 1] = rep[2 * j]
    need = _frames_needed(rep)
    assert need <= T
    rows = {1: (rep, need), 2: (_no_repeat(Lmax, 4, g), T), 3: (rep, need - 1),
            4: (_no_repeat(Lmax // 2 + 1, V, g), 0)}
    for b in range(5, B):
        n = int(torch.randint(1, Lmax + 1, (1,), generator=g))
        t = _no_repeat(n, V, g)
        for i in range(1, n, 5):
            if _frames_needed(t) < T - 1:
                t[i] = t[i - 1]
        lo = _frames_needed(t)
        assert lo <= T
        rows[b] = (t, int(torch.randint(lo, T + 1, (1,), generator=g)))
    for b, (t, n) in rows.items():
        txt[b, :len(t)] = torch.tensor(t)
        tl[b] = len(t)
        il[b] = n
    return logits, txt, il, tl


def _ctc_reference(logits, txt, il, tl, up):
    """float64 ATen: per-utterance nll and the logit gradient of up * sum_b nll_b / (max(tl_b, 1) * B)."""
    B = logits.shape[0]
    xr = logits.double().requires_grad_(True)
    nll = F.ctc_loss(F.log_softmax(xr, -1).transpose(0, 1), txt, il, tl, blank=0, reduction="none",
                     zero_infinity=False)
    w = 1.0 / (tl.clamp_min(1).double() * B)
    ((nll * w).sum() * up).backward()
    return nll.detach(), xr.grad, w


def _ctc_run(pkg, logits, txt, il, tl, fused, up):
    x = logits.to(DEV).requires_grad_(True)
    if fused:
        head = pkg.ops.ctc_head(x)                                   # row lse + arg-max, logits straight into the loss
    else:
        head, _ = pkg.ops.log_softmax(x, ctc_head=True)              # log-probs; the CTC gradient reaches x unchanged
    crit = pkg.CTCLoss(blank=0)
    loss = crit(head.transpose(0, 1), txt.to(DEV), il.to(DEV), tl.to(DEV))
    (loss * up).backward()
    return loss.item(), crit.last_nll.cpu(), x.grad.cpu()


def _check_ctc_batch(pkg, B, T, V, Lmax, seed):
    lib = pkg.load_library()
    assert lib.b200asr_debug_ctc_variant(Lmax) >= 1
    logits, txt, il, tl = _ctc_batch(B, T, V, Lmax, seed)
    up = 0.3
    torch.set_num_threads(16)
    ref_nll, ref_g, w = _ctc_reference(logits, txt, il, tl, up)
    assert math.isinf(ref_nll[3]) and math.isinf(ref_nll[4]) and torch.isnan(ref_g[3, :int(il[3])]).all()
    padded = logits.clone()
    for b in range(B):
        padded[b, int(il[b]):] = float("nan")                        # frames t >= input_length: never read
    fin = torch.isfinite(ref_nll)
    for fused in (False, True):
        loss, nll, grad = _ctc_run(pkg, logits, txt, il, tl, fused, up)
        assert math.isinf(loss) and loss > 0
        # per-utterance nll: +inf exactly where ATen has it, T * EPS relative elsewhere
        assert torch.equal(torch.isinf(nll), torch.isinf(ref_nll)) and bool((nll[~fin] > 0).all())
        err = ((nll[fin].double() - ref_nll[fin]).abs() / ref_nll[fin].abs()).max().item()
        assert err <= T * EPS, (fused, err)
        # gradient: identical NaN pattern, padded frames exactly 0, finite rows within T * EPS * |nll| of their weight
        assert torch.equal(torch.isnan(grad), torch.isnan(ref_g)), fused
        for b in range(B):
            assert bool((grad[b, int(il[b]):] == 0).all()), (fused, b)
            if fin[b]:
                e = (grad[b].double() - ref_g[b]).abs().max().item() / (float(w[b]) * up)
                assert e <= T * EPS * float(ref_nll[b]), (fused, b, e, T * EPS * float(ref_nll[b]))
        # deterministic, and blind to whatever the padded frames hold
        _, nll2, grad2 = _ctc_run(pkg, logits, txt, il, tl, fused, up)
        _, nll3, grad3 = _ctc_run(pkg, padded, txt, il, tl, fused, up)
        for n_, g_ in ((nll2, grad2), (nll3, grad3)):
            assert torch.equal(_bits(n_), _bits(nll)) and torch.equal(_bits(g_), _bits(grad)), fused


@pytest.mark.parametrize("Lmax", [15, 16, 47, 48, 63, 64, 141])
def test_ctc_cfg_b_batch(pkg, Lmax):
    """cfg B: batch 64, T = 299 encoder frames, 31 characters."""
    _check_ctc_batch(pkg, 64, 299, 31, Lmax, seed=Lmax)


@pytest.mark.parametrize("Lmax", [15, 16, 47, 48, 63, 64, 141])
def test_ctc_cfg_c_batch(pkg, Lmax):
    """cfg C: batch 64, T = 149 encoder frames, 5000 subwords."""
    _check_ctc_batch(pkg, 64, 149, 5000, Lmax, seed=1000 + Lmax)


@pytest.mark.parametrize("Lmax", [511, 512, 600])
def test_ctc_wide_targets(pkg, Lmax):
    """Widths beyond the one-position-per-thread block kernel: small batch, T >= 2 L_max + 1."""
    _check_ctc_batch(pkg, 6, 2 * Lmax + 21, 31, Lmax, seed=2000 + Lmax)


def test_ctc_infeasible_golden_case_gradient_is_nan(pkg):
    """ctc_cases.npz case 3 (4 repeated labels in 6 frames) was made by the reference: +inf nll, NaN gradient."""
    g = load_golden("ctc_cases.npz")
    assert np.isinf(g["c3_nll"][0]) and np.isnan(g["c3_grad"]).all()
    for fused in (False, True):
        lp = torch.from_numpy(g["c3_lp"])[None]                      # [1, T, V] log-probs (their lse is 0)
        x = lp.to(DEV).requires_grad_(True)
        head = pkg.ops.ctc_head(x) if fused else pkg.ops.log_softmax(x, ctc_head=True)[0]
        loss = pkg.CTCLoss(blank=0, reduction="sum")(head.transpose(0, 1), torch.from_numpy(g["c3_tgt"])[None].to(DEV),
                                                     torch.from_numpy(g["c3_il"]).to(DEV),
                                                     torch.from_numpy(g["c3_tl"]).to(DEV))
        assert math.isinf(loss.item()) and loss.item() > 0
        loss.backward()
        assert torch.equal(torch.isnan(x.grad[0].cpu()), torch.from_numpy(np.isnan(g["c3_grad"])))


# ------------------------------------------------------------------------------------------- train step
def _skip_batch(lens, long_text):
    g = torch.Generator().manual_seed(9)
    waves = [torch.clamp(0.05 * torch.randn(1, n, generator=g), -1, 1) for n in lens]
    texts = [[3, 4, 4, 5, 1], [6, 7, 1], long_text]
    batch = torch.zeros(3, max(lens))
    txt = torch.zeros(3, max(len(t) for t in texts), dtype=torch.long)
    for i in range(3):
        batch[i, :lens[i]] = waves[i][0]
        txt[i, :len(texts[i])] = torch.tensor(texts[i])
    return waves, texts, batch, txt


# 25 tokens without adjacent repeats: they need 25 encoder frames; 6400 samples give 38 fbank frames, 19 after the
# tiny encoder's 2x downsampling (infeasible), 9000 samples give 27 (feasible)
LONG_TEXT = [3 + i % 9 for i in range(24)] + [1]


@pytest.mark.parametrize("kind", ["ctc", "hybrid"])
def test_infeasible_utterance_skips_the_step_like_the_cpu_path(pkg, kind):
    from oracle import ref_port
    from test_gpu_model import _tiny_config
    cfg = _tiny_config(kind)
    step = pkg.TrainStep(cfg, 12, device=DEV, seed=3)
    P = {k: v.detach().cpu().clone() for k, v in step.model.state_dict().items()}
    cpu = ref_port.CpuTrainer(P, cfg["model"], cfg["data"]["audio"])
    opt = step.optimizer
    before = [t.clone() for t in (opt.buf.flat, opt.state1, opt.state2)]
    cpu_before = {k: v.detach().clone() for k, v in cpu.P.items()}
    waves, texts, batch, txt = _skip_batch([9000, 7700, 6400], LONG_TEXT)
    loss = step(batch.to(DEV), torch.tensor([9000, 7700, 6400]), txt.to(DEV))
    ref_loss, ref_norm = cpu.step(waves, texts)
    assert math.isinf(ref_loss) and ref_loss > 0 and math.isnan(ref_norm)
    assert math.isinf(loss.item()) and loss.item() > 0
    assert math.isnan(step.last["grad_norm"].item())
    for a, b in zip(before, (opt.buf.flat, opt.state1, opt.state2)):      # parameters, square_avg, acc_delta
        assert torch.equal(_bits(a), _bits(b))
    assert all(torch.equal(cpu_before[k], cpu.P[k].detach()) for k in cpu_before)
    # the next, feasible batch: as test_two_train_steps_match_cpu_reference_path
    waves, texts, batch, txt = _skip_batch([9000, 7700, 6400], [8, 9, 10, 1])
    loss = step(batch.to(DEV), torch.tensor([9000, 7700, 6400]), txt.to(DEV))
    ref_loss, ref_norm = cpu.step(waves, texts)
    assert abs(loss.item() - ref_loss) < 1e-4 * abs(ref_loss), (loss.item(), ref_loss)
    assert abs(step.last["grad_norm"].item() - ref_norm) < 2e-4 * ref_norm
    for k, v in step.model.state_dict().items():
        ref = cpu.P[k].detach()
        assert float((v.cpu() - ref).abs().max()) < 2e-4 * max(float(ref.abs().max()), 1e-2), k


def test_infeasible_utterance_skips_the_replayed_step(pkg):
    """Captured on a feasible batch; a replay whose third wave is cut to 6400 samples has no CTC alignment."""
    from test_gpu_model import _tiny_config
    _, _, batch, txt = _skip_batch([9000, 9000, 9000], LONG_TEXT)
    wave, txt = batch.to(DEV), txt.to(DEV)
    step = pkg.TrainStep(_tiny_config("hybrid"), 12, device=DEV, seed=5)
    assert step.capture(wave, torch.tensor([9000, 9000, 9000]), txt, warmup=3), step.graph_error
    opt = step.optimizer
    loss = step(wave, torch.tensor([9000, 9000, 9000]), txt)
    assert math.isfinite(loss.item()) and math.isfinite(opt.grad_norm.item())
    before = [t.clone() for t in (opt.buf.flat, opt.state1, opt.state2)]
    loss = step(wave, torch.tensor([9000, 9000, 6400]), txt)
    torch.cuda.synchronize()
    assert step.graph is not None
    assert math.isinf(loss.item()) and loss.item() > 0 and math.isnan(opt.grad_norm.item())
    for a, b in zip(before, (opt.buf.flat, opt.state1, opt.state2)):
        assert torch.equal(_bits(a), _bits(b))
    loss = step(wave, torch.tensor([9000, 9000, 9000]), txt)                 # and training goes on
    assert math.isfinite(loss.item()) and not torch.equal(before[0], opt.buf.flat)


# ------------------------------------------------------------------------------------------- log-softmax
def _lsm_values(kind, N, V, g):
    if kind == "normal":
        x = 3 * torch.randn(N, V, generator=g)
    elif kind == "ties":                                             # integer logits: many tied maxima
        x = torch.randint(-3, 4, (N, V), generator=g).float()
    elif kind == "neginf":
        x = 3 * torch.randn(N, V, generator=g)
        x[torch.rand(N, V, generator=g) < 0.3] = float("-inf")
        x[0, :] = float("-inf")
        x[0, V // 2] = 1.0                                           # one finite class
        x[1, : V - 1] = float("-inf")                                # the finite class is the last one
        x[1, V - 1] = 2.0
    else:                                                            # "large": |logit| around 50
        x = 50 + 2 * torch.randn(N, V, generator=g)
        x[::2] *= -1
    return x


def _lsm_fwd(lib, L, x, y, lse, am):
    N, V = x.shape
    L.check(lib.b200asr_log_softmax_fwd(L.ptr(x), L.ptr(y), L.ptr(lse), L.ptr(am), N, V, L.stream()))


def _offset_copy(src, off):
    """Copy of `src` as a contiguous view that starts `off` floats into a fresh buffer."""
    return torch.empty(src.numel() + 4, device=DEV)[off:off + src.numel()].view(src.shape).copy_(src)


def _check_lsm_fwd(x64, y, lse, am, x_cpu):
    V = x64.shape[1]
    ref = torch.log_softmax(x64, -1)
    L = torch.logsumexp(x64, -1, keepdim=True)
    y = y.cpu().double()
    inf = torch.isinf(ref)
    assert torch.equal(inf, torch.isinf(y)) and bool((y[inf] == ref[inf]).all())
    tol = EPS * (4 * (x64.abs() + L.abs()) + V / 8 + 64)
    assert bool(((y - ref).abs() <= tol)[~inf].all()), float(((y - ref).abs() - tol)[~inf].max())
    if lse is not None:
        assert bool(((lse.cpu().double() - L[:, 0]).abs() <= EPS * (4 * L[:, 0].abs() + V / 8 + 64)).all())
    assert torch.equal(am.cpu(), torch.argmax(x_cpu, -1))           # first index of the maximum, like torch


def _check_lsm_bwd(lp, g, dx):
    lp, g, dx = lp.cpu().double(), g.cpu().double(), dx.cpu().double()
    V = lp.shape[1]
    p = lp.exp()
    s = g.sum(-1, keepdim=True)
    ref = g - p * s
    tol = 2 * EPS * (g.abs() + p * (2 * s.abs() + (V / 32 + 8) * g.abs().sum(-1, keepdim=True)))
    assert bool(((dx - ref).abs() <= tol).all()), float(((dx - ref).abs() - tol).max())


@pytest.mark.parametrize("kind", ["normal", "ties", "neginf", "large"])
@pytest.mark.parametrize("V", [64, 200, 1000, 31, 4999])
def test_log_softmax_edges_vs_fp64(pkg, V, kind):
    """V = 64 / 200 / 1000: 16 / 50 / 250 float4 vectors per row (<32, 32-64, >64 per warp); 31 and 4999 scalar."""
    L = pkg.lib
    lib = L.load()
    N = 37
    g = torch.Generator().manual_seed(V + len(kind))
    x_cpu = _lsm_values(kind, N, V, g)
    x64 = x_cpu.double()
    x = x_cpu.to(DEV)
    y = torch.empty_like(x)
    lse = torch.empty(N, device=DEV)
    am = torch.empty(N, device=DEV, dtype=torch.int64)
    _lsm_fwd(lib, L, x, y, None, am)
    _check_lsm_fwd(x64, y, None, am, x_cpu)
    am2 = torch.empty_like(am)
    _lsm_fwd(lib, L, x, None, lse, am2)                              # statistics only (the fused CTC head)
    _check_lsm_fwd(x64, y, lse, am2, x_cpu)
    gr = torch.randn(N, V, generator=g).to(DEV)
    dx = torch.empty_like(x)
    L.check(lib.b200asr_log_softmax_bwd(L.ptr(y), L.ptr(gr), L.ptr(dx), N, V, L.stream()))
    _check_lsm_bwd(y, gr, dx)


@pytest.mark.parametrize("V", [64, 200, 1000, 5000])
def test_log_softmax_misaligned_views(pkg, V):
    """Contiguous views that start 1-3 floats into their buffer take the scalar path: same bounds as aligned rows."""
    L = pkg.lib
    lib = L.load()
    N = 29
    g = torch.Generator().manual_seed(V)
    x_cpu = 3 * torch.randn(N, V, generator=g)
    x64 = x_cpu.double()
    gr_cpu = torch.randn(N, V, generator=g)
    for ox, oy in [(0, 0), (1, 0), (0, 2), (3, 3), (2, 1)]:
        x = _offset_copy(x_cpu.to(DEV), ox)
        y = _offset_copy(torch.zeros_like(x), oy)
        lse = torch.empty(N + 1, device=DEV)[1:]
        am = torch.empty(N, device=DEV, dtype=torch.int64)
        _lsm_fwd(lib, L, x, y, None, am)
        _check_lsm_fwd(x64, y, None, am, x_cpu)
        _lsm_fwd(lib, L, x, None, lse, am)
        _check_lsm_fwd(x64, y, lse, am, x_cpu)
        for olp, og, odx in [(0, 0, 0), (ox, 0, 0), (0, 2, 0), (0, 0, 3), (oy, 1, 3)]:
            lp = _offset_copy(y, olp)
            gr = _offset_copy(gr_cpu.to(DEV), og)
            dx = _offset_copy(torch.zeros_like(y), odx)
            L.check(lib.b200asr_log_softmax_bwd(L.ptr(lp), L.ptr(gr), L.ptr(dx), N, V, L.stream()))
            _check_lsm_bwd(lp, gr, dx)
    # through autograd: ops.log_softmax keeps a contiguous view as it is
    x = _offset_copy(x_cpu.to(DEV), 1).requires_grad_(True)
    y, am = pkg.ops.log_softmax(x)
    gr = _offset_copy(gr_cpu.to(DEV), 3)
    y.backward(gr)
    _check_lsm_fwd(x64, y.detach(), None, am, x_cpu)
    _check_lsm_bwd(y.detach(), gr, x.grad)


# ------------------------------------------------------------------------------------------- cross-entropy
@pytest.mark.parametrize("reduction", ["mean", "sum"])
@pytest.mark.parametrize("mag", [3.0, 50.0])
def test_cross_entropy_decoder_size_vs_fp64(pkg, reduction, mag):
    """cfg C's decoder output: 64 utterances x 46 steps over 5000 subwords, a quarter of the rows ignored (index 0)."""
    L = pkg.lib
    lib = L.load()
    N, V = 64 * 46, 5000
    g = torch.Generator().manual_seed(int(mag) + len(reduction))
    x_cpu = mag * torch.randn(N, V, generator=g)
    tgt = torch.randint(1, V, (N,), generator=g)
    tgt[torch.randperm(N, generator=g)[: N // 4]] = 0
    if mag == 3.0:                                                   # masked classes: -inf logits, targets finite
        keep = x_cpu[torch.arange(N), tgt].clone()
        x_cpu[torch.rand(N, V, generator=g) < 0.05] = float("-inf")
        x_cpu[torch.arange(N), tgt] = keep
    up = 0.7
    x64 = x_cpu.double().requires_grad_(True)
    rows = F.cross_entropy(x64, tgt, ignore_index=0, reduction="none")
    ref = F.cross_entropy(x64, tgt, ignore_index=0, reduction=reduction)
    (ref * up).backward()
    lse = torch.logsumexp(x64.detach(), -1)
    row_tol = EPS * (4 * (x64.detach().nan_to_num(neginf=0.0).abs().max(-1).values + lse.abs()) + V / 8 + 64)
    # per-row loss straight from the kernel
    x = x_cpu.to(DEV)
    row = torch.empty(N, device=DEV)
    one = torch.ones(1, device=DEV)
    L.check(lib.b200asr_ce_fwd_bwd(L.ptr(x), L.ptr(tgt.to(DEV)), 0, N, V, L.ptr(one), L.ptr(row), None, L.stream()))
    assert bool(((row.cpu().double() - rows.detach()).abs() <= row_tol).all())
    assert bool((row.cpu()[tgt == 0] == 0).all())
    # reduced loss and logit gradient through ops.cross_entropy, with an upstream scale
    xd = x_cpu.to(DEV).requires_grad_(True)
    loss = pkg.ops.cross_entropy(xd, tgt.to(DEV), ignore_index=0, reduction=reduction)
    (loss * up).backward()
    n_valid = int((tgt != 0).sum())
    sc = 1.0 / n_valid if reduction == "mean" else 1.0
    assert abs(loss.item() - ref.item()) <= sc * float(row_tol.sum()) + 64 * EPS * abs(ref.item())
    grad = xd.grad.cpu().double()
    p = (x64.detach() - lse[:, None]).exp()
    gtol = up * sc * (p * row_tol[:, None] + 4 * EPS)
    assert bool(((grad - x64.grad).abs() <= gtol).all()), float(((grad - x64.grad).abs() - gtol).max())
    assert bool((grad[tgt == 0] == 0).all())


# ------------------------------------------------------------------------------------------- attention
def _loc_attention_torch(q, key, value, prev, lens, cw, pw, ew, eb, temp):
    T = key.shape[1]
    R = (cw.shape[2] - 1) // 2
    conv = F.conv1d(prev.unsqueeze(1), cw, padding=R)
    loc = torch.tanh(F.linear(conv.transpose(1, 2), pw))
    e = F.linear(torch.tanh(key + q.unsqueeze(1) + loc), ew, eb).squeeze(2) / temp
    mask = torch.arange(T)[None, :] >= lens[:, None]
    a = torch.softmax(e.masked_fill(mask, float("-inf")), -1)
    return torch.bmm(a.unsqueeze(1), value).squeeze(1), a


def _attn_inputs(B, T, D, E, K, R, L, seed):
    g = torch.Generator().manual_seed(seed)
    mk = lambda *s, sc=1.0: torch.randn(*s, generator=g) * sc
    lens = torch.linspace(T, T // 4, B).round().long()
    qs, key, value = mk(L, B, D), mk(B, T, D), mk(B, T, E)
    pad = torch.arange(T)[None] >= lens[:, None]
    key[pad] = 1e6 * torch.sign(mk(int(pad.sum()), D))                # finite garbage the kernels must never use
    value[pad] = 1e6 * torch.sign(mk(int(pad.sum()), E))
    prev = torch.rand(B, T, generator=g) * ~pad
    prev = prev / prev.sum(1, keepdim=True)
    cw, pw, ew, eb = mk(K, 1, 2 * R + 1, sc=0.3), mk(D, K, sc=0.5), mk(1, D, sc=0.3), mk(1)
    return lens, qs, key, value, prev, (cw, pw, ew, eb), mk(L, B, E), mk(L, B, T)


def _check_attn_grads(names, dev_in, ref_in, bound):
    for n, x, r in zip(names, dev_in, ref_in):
        if n == "eb":        # softmax is shift invariant: d/d(b_energy) = sum of d(energy) = 0 up to rounding.  Its scale:
            # sum |d(key)| = sum over frames of |d(energy)| * sum_d |w_e| (1 - s^2), larger than sum |d(energy)| here
            assert float(x.grad.abs().max()) <= bound * float(ref_in[names.index("key")].grad.abs().sum()), n
        else:
            assert scaled_err(x.grad.cpu().numpy(), r.grad.numpy()) <= bound, n


@pytest.mark.parametrize("case", ["minb2", "d512_e4096"])
def test_loc_attention_step_production_sizes(pkg, case):
    """minb2: sm_count // 4 + 1 utterances of cfg C (T = 149, D = 300, E = 2048; 4-CTA clusters) - more CTAs than SMs,
    so the two-CTAs-per-SM backward instance.  d512_e4096: the kernels' limits D = 512 and E / CS = 1024."""
    lib = pkg.load_library()
    sms = lib.b200asr_device_sm_count()
    B, T, D, E = (sms // 4 + 1, 149, 300, 2048) if case == "minb2" else (3, 149, 512, 4096)
    K, R = 10, 100
    assert lib.b200asr_locattn_cluster_size(T, E) == 4
    assert lib.b200asr_debug_locattn_bwd_minb(B, T, D, E) == (2 if case == "minb2" else 1)
    if case == "minb2":
        assert lib.b200asr_debug_locattn_bwd_minb(sms // 4, T, D, E) == 1
    lens, qs, key, value, prev, w, gc, ga = _attn_inputs(B, T, D, E, K, R, 1, seed=B + D)
    bound = max(T, D, E, K * (2 * R + 1)) * EPS
    names = ["q", "key", "value", "prev", "cw", "pw", "ew", "eb"]
    torch.set_num_threads(16)
    ref_in = [t.double().requires_grad_(True) for t in (qs[0], key, value, prev) + w]
    cr, ar = _loc_attention_torch(ref_in[0], ref_in[1], ref_in[2], ref_in[3], lens, *ref_in[4:], 0.5)
    ((cr * gc[0].double()).sum() + (ar * ga[0].double()).sum()).backward()
    dev_in = [t.to(DEV).requires_grad_(True) for t in (qs[0], key, value, prev) + w]
    c, a = pkg.ops.loc_attention_step(dev_in[0], dev_in[1], dev_in[2], dev_in[3], lens.to(DEV), *dev_in[4:], 0.5)
    assert scaled_err(a.detach().cpu().numpy(), ar.detach().numpy()) <= bound
    assert scaled_err(c.detach().cpu().numpy(), cr.detach().numpy()) <= bound
    ((c * gc[0].to(DEV)).sum() + (a * ga[0].to(DEV)).sum()).backward()
    _check_attn_grads(names, dev_in, ref_in, bound)
    pad = torch.arange(T)[None] >= lens[:, None]
    assert float(dev_in[1].grad.cpu()[pad].abs().max()) == 0 and float(dev_in[2].grad.cpu()[pad].abs().max()) == 0


@pytest.mark.parametrize("case", ["minb2", "d512_e4096"])
def test_loc_attention_decode_loop_production_sizes(pkg, case):
    """The decode loop's form (b200asr_locattn_bwd_acc per step, b200asr_attn_dvalue once) over cfg C's 46 steps."""
    lib = pkg.load_library()
    sms = lib.b200asr_device_sm_count()
    B, T, D, E, Ls = (sms // 4 + 1, 149, 300, 2048, 46) if case == "minb2" else (3, 149, 512, 4096, 8)
    K, R = 10, 100
    assert lib.b200asr_debug_locattn_bwd_minb(B, T, D, E) == (2 if case == "minb2" else 1)
    lens, qs, key, value, prev, w, gc, ga = _attn_inputs(B, T, D, E, K, R, Ls, seed=7 * B + D)
    # one more level of accumulation (over the Ls steps) on top of a single step's contractions
    bound = (2 * max(T, D, E, K * (2 * R + 1)) + Ls) * EPS
    names = ["q", "key", "value", "cw", "pw", "ew", "eb"]
    torch.set_num_threads(16)
    ref_in = [t.double().requires_grad_(True) for t in (qs, key, value) + w]
    p_ref, tot = prev.double(), 0
    for l in range(Ls):
        c, a = _loc_attention_torch(ref_in[0][l], ref_in[1], ref_in[2], p_ref, lens, *ref_in[3:], 0.5)
        tot = tot + (c * gc[l].double()).sum() + (a * ga[l].double()).sum()
        p_ref = a
    tot.backward()
    dev_in = [t.to(DEV).requires_grad_(True) for t in (qs, key, value) + w]
    mem, mkey, mval, mcw, mpw, mew, meb, token = pkg.ops.attention_memory(*dev_in[1:])
    p_dev, tot = prev.to(DEV), 0
    for l in range(Ls):
        c, a = pkg.ops.loc_attention_mem_step(mem, token, dev_in[0][l], mkey, mval, p_dev, lens.to(DEV), mcw, mpw, mew,
                                              meb, 0.5)
        tot = tot + (c * gc[l].to(DEV)).sum() + (a * ga[l].to(DEV)).sum()
        p_dev = a
    tot.backward()
    _check_attn_grads(names, dev_in, ref_in, bound)
    pad = torch.arange(T)[None] >= lens[:, None]
    assert float(dev_in[1].grad.cpu()[pad].abs().max()) == 0 and float(dev_in[2].grad.cpu()[pad].abs().max()) == 0


# ------------------------------------------------------------------------------------------- small kernels, real size
@pytest.mark.parametrize("with_dc", [False, True])
def test_lstm_cell_decoder_size(pkg, with_dc):
    """The decoder cell at B = 64, H = 512, pre-activations up to +-30 (saturated gates); dc_next NULL or given.
    Each output is a product of at most three sigmoid / tanh values and c: 16 EPS of the tensor's scale."""
    torch.manual_seed(5)
    B, H = 64, 512
    pre = 60 * torch.rand(B, 4 * H) - 30
    c0 = 3 * torch.randn(B, H)
    a = pre.to(DEV).requires_grad_(True)
    c = c0.to(DEV).requires_grad_(True)
    h1, c1 = pkg.ops.lstm_cell(a, c)
    ar = pre.double().requires_grad_(True)
    c0r = c0.double().requires_grad_(True)
    i, f, g_, o = ar[:, :H].sigmoid(), ar[:, H:2 * H].sigmoid(), ar[:, 2 * H:3 * H].tanh(), ar[:, 3 * H:].sigmoid()
    cn = f * c0r + i * g_
    hn = o * cn.tanh()
    assert scaled_err(h1.detach().cpu().numpy(), hn.detach().numpy()) <= 16 * EPS
    assert scaled_err(c1.detach().cpu().numpy(), cn.detach().numpy()) <= 16 * EPS
    gh, gc = torch.randn(B, H), torch.randn(B, H)
    if with_dc:
        (h1 * gh.to(DEV)).sum().add((c1 * gc.to(DEV)).sum()).backward()
        ((hn * gh.double()).sum() + (cn * gc.double()).sum()).backward()
    else:
        (h1 * gh.to(DEV)).sum().backward()                           # c1 unused: the backward gets dc_next = NULL
        (hn * gh.double()).sum().backward()
    assert scaled_err(a.grad.cpu().numpy(), ar.grad.numpy()) <= 16 * EPS
    assert scaled_err(c.grad.cpu().numpy(), c0r.grad.numpy()) <= 16 * EPS


def test_grad_norm_full_parameter_buffer(pkg):
    """73 M + 3 gradients (cfg D's parameter count class): ~135 grid-stride passes and a 3-element tail that is not a
    multiple of 4 (and large, so that dropping it shows).  fp64 accumulation, one fp32 rounding of the result."""
    L = pkg.lib
    lib = L.load()
    n = 73_000_003
    g = torch.Generator(device=DEV).manual_seed(4)
    grad = torch.randn(n, device=DEV, generator=g)
    grad[-3:] = torch.tensor([3000.0, -2000.0, 1000.0], device=DEV)
    norm = torch.zeros(1, device=DEV)
    scratch = torch.empty(lib.b200asr_grad_norm_scratch_bytes(), dtype=torch.uint8, device=DEV)
    L.check(lib.b200asr_grad_norm(L.ptr(grad), n, L.ptr(norm), L.ptr(scratch), L.stream()))
    ref = math.sqrt(float((grad.double() ** 2).sum()))
    assert abs(norm.item() - ref) <= 2 * EPS * ref, (norm.item(), ref)
    L.check(lib.b200asr_grad_norm(L.ptr(grad), n - 3, L.ptr(norm), L.ptr(scratch), L.stream()))
    ref = math.sqrt(float((grad[:-3].double() ** 2).sum()))
    assert abs(norm.item() - ref) <= 2 * EPS * ref, (norm.item(), ref)
