"""Parity of every CUDA kernel (through the C ABI) against the CPU oracle / committed golden vectors.
Run with: python -m pytest tests -m gpu."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden, rel_err, scaled_err
from oracle import oracle_np as onp
from oracle import ref_port
from oracle.make_golden import AUDIO_CFG

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ------------------------------------------------------------------------------------------- front end
def _frontend(pkg, **over):
    cfg = dict(AUDIO_CFG)
    cfg.update(over)
    tr, dim = pkg.create_transform(cfg, device=DEV)
    return tr, dim


def test_fbank_sample_wav_vs_reference_golden(pkg):
    g = load_golden("frontend.npz")
    wave = torch.from_numpy(g["sample_pcm"].astype(np.float32) / 32768.0)[None].to(DEV)
    tr, _ = _frontend(pkg, delta_order=0, apply_cmvn=False)
    fb, n = tr.batch(wave, [wave.shape[1]])
    assert int(n[0]) == 392 and fb.shape == (1, 392, 40)
    assert rel_err(fb[0].cpu().numpy(), g["sample_fbank_raw"], floor=1.0) < 1e-4
    for order in (0, 1, 2):
        tr, dim = _frontend(pkg, delta_order=order)
        y, n = tr.batch(wave, [wave.shape[1]])
        assert dim == 40 * (order + 1) and y.shape == (1, 392, dim)
        assert float(np.max(np.abs(y[0].cpu().numpy() - g["sample_feat_d%d" % order]))) < 1e-3


def test_fbank_pcm16_ingest_equals_fp32_path(pkg):
    """16-bit PCM fed straight to the kernel (sample / 32768 on the fly) is bit-identical to the fp32 path, ragged batch."""
    g = load_golden("frontend.npz")
    pcm = torch.from_numpy(g["sample_pcm"])
    batch = torch.zeros(2, pcm.numel(), dtype=torch.int16)
    batch[0] = pcm
    batch[1, :30000] = pcm[5000:35000]
    lens = [pcm.numel(), 30000]
    tr, _ = _frontend(pkg)
    y16, n16 = tr.batch(batch.to(DEV), lens)
    y32, n32 = tr.batch((batch.float() / 32768.0).to(DEV), lens)
    assert torch.equal(n16, n32) and torch.equal(y16, y32)
    assert float(np.max(np.abs(y16[0].cpu().numpy() - g["sample_feat_d2"]))) < 1e-3


def test_fbank_ragged_batch_vs_reference_golden(pkg):
    g = load_golden("frontend.npz")
    waves = [g["syn%d_wave" % i] for i in (3, 2, 1, 0)]           # 16000, 7013, 4000, 400 samples
    lens = [len(w) for w in waves]
    batch = torch.zeros(len(waves), max(lens))
    for i, w in enumerate(waves):
        batch[i, :len(w)] = torch.from_numpy(w)
    tr, _ = _frontend(pkg)
    raw, _ = _frontend(pkg, delta_order=0, apply_cmvn=False)
    fb, n = raw.batch(batch.to(DEV), lens)
    feat, n2 = tr.batch(batch.to(DEV), lens)
    assert n.tolist() == [98, 42, 23, 1] == n2.tolist()
    for row, i in enumerate((3, 2, 1, 0)):
        m = int(n[row])
        assert rel_err(fb[row, :m].cpu().numpy(), g["syn%d_raw" % i], floor=1.0) < 1e-4
        assert float(fb[row, m:].abs().max() if m < fb.shape[1] else 0) == 0
        if i > 0:
            assert float(np.max(np.abs(feat[row, :m].cpu().numpy() - g["syn%d_feat" % i]))) < 2e-3
            assert float(feat[row, m:].abs().max() if m < feat.shape[1] else 0) == 0   # pad_sequence zeros
    # a single-frame utterance has an undefined unbiased std: NaN like torch.std
    assert torch.isnan(feat[3, 0]).all()


def test_fbank_filepath_transform_contract(pkg, tmp_path):
    from scipy.io import wavfile
    g = load_golden("frontend.npz")
    p = str(tmp_path / "s.wav")
    wavfile.write(p, 16000, g["sample_pcm"])
    tr, dim = _frontend(pkg)
    y = tr(p)
    assert y.shape == (392, 120) and dim == 120 and y.device.type == "cpu"
    assert float(np.max(np.abs(y.numpy() - g["sample_feat_d2"]))) < 1e-3
    # properties the reference's own tests pin (tests/test_audio.py:87,103)
    assert torch.allclose(y.mean(0), torch.zeros(120), atol=5e-5)
    assert torch.allclose(y.std(0), torch.ones(120), atol=1e-5)


def test_fbank_long_batch_linearity_property(pkg):
    """Full-size property (12 s utterances): log-mel of a*x equals log-mel of x + 2*log(a) wherever the floor is
    inactive, so the CMVN-normalised STATIC channel is invariant to the gain.  (The delta channels are not: their
    edge frames see the reference's ZERO padding, src/audio.py:51-54, which does not shift with the gain, and that
    moves the per-utterance mean/std of the whole channel.)"""
    torch.manual_seed(0)
    B, N = 8, 192000
    x = torch.clamp(0.05 * torch.randn(B, N), -1, 1).to(DEV)
    raw, _ = _frontend(pkg, delta_order=0, apply_cmvn=False)
    full, _ = _frontend(pkg)
    fb1, n = raw.batch(x, [N] * B)
    fb2, _ = raw.batch(0.5 * x, [N] * B)
    assert n.tolist() == [1198] * B
    assert float((fb2 - fb1 - 2 * np.log(0.5)).abs().max()) < 1e-4
    f1, _ = full.batch(x, [N] * B)
    f2, _ = full.batch(0.5 * x, [N] * B)
    assert float((f1 - f2)[:, :, :40].abs().max()) < 1e-3
    assert float(f1[:, :, :40].mean(1).abs().max()) < 1e-4           # CMVN: zero mean over time
    assert float((f1[:, :, :].std(1) - 1).abs().max()) < 1e-4         # unit (unbiased) std, all 120 columns


# ------------------------------------------------------------------------------------------- log-softmax / CTC
@pytest.mark.parametrize("shape", [(7, 31), (3, 5, 1000), (2, 4, 5000)])
def test_log_softmax_fwd_bwd(pkg, shape):
    torch.manual_seed(1)
    x = (3 * torch.randn(*shape)).to(DEV).requires_grad_(True)
    y, am = pkg.ops.log_softmax(x)
    xr = x.detach().cpu().double().requires_grad_(True)
    yr = F.log_softmax(xr, -1)
    assert rel_err(y.detach().cpu().numpy(), yr.detach().numpy()) < 1e-5
    assert torch.equal(am.cpu(), yr.argmax(-1))
    g = torch.randn(*shape)
    y.backward(g.to(DEV))
    yr.backward(g.double())
    assert scaled_err(x.grad.cpu().numpy(), xr.grad.numpy()) < 1e-5


def test_ctc_golden_cases(pkg):
    g = load_golden("ctc_cases.npz")
    for i in range(int(g["n_cases"])):
        lp = torch.from_numpy(g["c%d_lp" % i])[:, None, :].to(DEV).requires_grad_(True)     # [T,1,V]
        tgt = torch.from_numpy(g["c%d_tgt" % i])[None].to(DEV)
        tl = torch.from_numpy(g["c%d_tl" % i])
        il = torch.from_numpy(g["c%d_il" % i])
        crit = pkg.CTCLoss(blank=0, reduction="sum")
        loss = crit(lp, tgt, il, tl)
        ref = float(g["c%d_nll" % i][0])
        if np.isinf(ref):
            assert torch.isinf(loss).item() and loss.item() > 0        # infeasible -> +inf (zero_infinity=False)
            continue
        assert abs(loss.item() - ref) < 1e-4 * max(1.0, abs(ref))
        loss.backward()
        assert np.max(np.abs(lp.grad[:, 0].cpu().numpy() - g["c%d_grad" % i])) < 1e-5


@pytest.mark.parametrize("head", [False, True])
@pytest.mark.parametrize("B,T,V,Lmax", [(4, 50, 31, 20), (3, 37, 500, 9), (6, 149, 5000, 40), (2, 300, 31, 141)])
def test_ctc_random_vs_aten_cpu(pkg, B, T, V, Lmax, head):
    """head=True: the CTC-head contract of ops.log_softmax (its backward is the identity because the CTC gradient in
    ATen's convention already is the logit gradient, SURVEY.md F9) must give the same logit gradient."""
    gen = torch.Generator().manual_seed(B * 1000 + T)
    logits = torch.randn(B, T, V, generator=gen)
    tl = torch.randint(1, Lmax, (B,), generator=gen)
    tl[0] = Lmax - 1
    il = torch.randint(T // 2 + Lmax, T + 1, (B,), generator=gen).clamp(max=T)
    il[0] = T
    txt = torch.zeros(B, Lmax, dtype=torch.long)
    for b in range(B):
        txt[b, :tl[b]] = torch.randint(1, V, (int(tl[b]),), generator=gen)
        if tl[b] > 2:
            txt[b, 1] = txt[b, 0]
    x = logits.to(DEV).requires_grad_(True)
    lp, _ = pkg.ops.log_softmax(x, ctc_head=head)
    loss = pkg.CTCLoss(blank=0)(lp.transpose(0, 1), txt.to(DEV), il.to(DEV), tl.to(DEV)) * 0.3   # upstream scale
    loss.backward()
    loss = loss / 0.3
    x.grad /= 0.3
    xr = logits.clone().requires_grad_(True)
    lpr = F.log_softmax(xr, -1)
    ref = F.ctc_loss(lpr.transpose(0, 1), txt, il, tl, blank=0, reduction="mean", zero_infinity=False)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-4 * abs(ref.item())
    # fp32 budget: the occupancy term exp(log sum(alpha*beta) + nll - lp) cancels two numbers of magnitude
    # ~T*log(V) (1e3 at V=5000), so ATen's own fp32 result carries ~1e-4 relative noise there
    assert scaled_err(x.grad.cpu().numpy(), xr.grad.numpy()) < (1e-4 if V < 1000 else 1e-3)
    # greedy path ids are bit exact
    assert torch.equal(lp.argmax(-1).cpu(), lpr.argmax(-1))


@pytest.mark.parametrize("B,T,V,Lmax", [(4, 50, 31, 20), (3, 37, 500, 9), (6, 149, 5000, 40), (2, 300, 31, 141), (5, 64, 30, 1)])
def test_ctc_fused_head_vs_aten_cpu(pkg, B, T, V, Lmax):
    """The train step's CTC path: ops.ctc_head (row lse + arg-max, no V-wide log-prob tensor) -> CTCLoss on logits - lse
    -> the gradient kernel writes the LOGIT gradient.  Same loss / per-utterance nll / logit gradient / ids as
    log_softmax + F.ctc_loss on the CPU, and bit-identical nll to the unfused kernels."""
    gen = torch.Generator().manual_seed(B * 1000 + T + 7)
    logits = torch.randn(B, T, V, generator=gen)
    tl = torch.randint(1, max(Lmax, 2), (B,), generator=gen)
    tl[0] = max(Lmax - 1, 1)
    il = torch.randint(T // 2 + Lmax, T + 1, (B,), generator=gen).clamp(max=T)
    il[0] = T
    txt = torch.zeros(B, max(Lmax, 2), dtype=torch.long)
    for b in range(B):
        txt[b, :tl[b]] = torch.randint(1, V, (int(tl[b]),), generator=gen)
        if tl[b] > 2:
            txt[b, 1] = txt[b, 0]
    x = logits.to(DEV).requires_grad_(True)
    head = pkg.ops.ctc_head(x)
    assert isinstance(head, pkg.ops.CTCHeadOutput) and tuple(head.shape) == (B, T, V)
    crit = pkg.CTCLoss(blank=0)
    loss = crit(head.transpose(0, 1), txt.to(DEV), il.to(DEV), tl.to(DEV)) * 0.3                # upstream scale
    nll_fused = crit.last_nll.clone()
    loss.backward()
    xr = logits.clone().requires_grad_(True)
    lpr = F.log_softmax(xr, -1)
    ref = F.ctc_loss(lpr.transpose(0, 1), txt, il, tl, blank=0, reduction="mean", zero_infinity=False) * 0.3
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-4 * abs(ref.item())
    # (T = 300 with 140 labels: ATen's own fp32 lattice carries ~1e-4 of noise there, see the unfused test above)
    assert scaled_err(x.grad.cpu().numpy(), xr.grad.numpy()) < (2e-4 if V < 1000 else 1e-3)
    assert torch.equal(head.argmax(-1).cpu(), lpr.argmax(-1))                                   # greedy ids bit exact
    assert rel_err(head.materialize().cpu().numpy(), lpr.detach().numpy()) < 1e-5
    # unfused kernels on materialised log-probs: same lattice arithmetic up to the rounding of x - lse
    x2 = logits.to(DEV).requires_grad_(True)
    lp, _ = pkg.ops.log_softmax(x2, ctc_head=True)
    crit(lp.transpose(0, 1), txt.to(DEV), il.to(DEV), tl.to(DEV))
    assert rel_err(nll_fused.cpu().numpy(), crit.last_nll.cpu().numpy()) < 1e-6
    # padded frames get a zero gradient, rows beyond the batch's lengths are never touched by NaNs
    for b in range(B):
        assert float(x.grad[b, int(il[b]):].abs().max()) == 0.0 if int(il[b]) < T else True


# ------------------------------------------------------------------------------------------- LSTM
def _torch_lstm(I, H, bidir, seed):
    torch.manual_seed(seed)
    return torch.nn.LSTM(I, H, bidirectional=bidir, num_layers=1, batch_first=True)


def _check_bilstm(pkg, B, T, I, H, bidir, wtol=1e-4):
    ref = _torch_lstm(I, H, bidir, 3)
    torch.manual_seed(4)
    x = torch.randn(B, T, I)
    xr = x.clone().requires_grad_(True)
    yr, _ = ref(xr)
    gy = torch.randn_like(yr)
    yr.backward(gy)
    ndir = 2 if bidir else 1
    params = [p.detach().clone().to(DEV).requires_grad_(True) for p in ref.parameters()]
    xg = x.to(DEV).requires_grad_(True)
    y = pkg.ops.bilstm(xg, params, ndir)
    assert y.shape == yr.shape
    assert scaled_err(y.detach().cpu().numpy(), yr.detach().numpy()) < 2e-5
    y.backward(gy.to(DEV))
    assert scaled_err(xg.grad.cpu().numpy(), xr.grad.numpy()) < 1e-4
    for p, q, (name, _) in zip(params, ref.parameters(), ref.named_parameters()):
        scale = float(q.grad.abs().max())
        assert float((p.grad.cpu() - q.grad).abs().max()) < wtol * max(scale, 1e-3), name


@pytest.mark.parametrize("B,T,I,H,bidir", [
    (3, 7, 8, 16, True),        # UB=1 scalar scatter path, partial batch block
    (5, 9, 12, 32, False),      # unidirectional
    (4, 1, 8, 32, True),        # single step
    (9, 6, 10, 48, True),       # two batch groups, tail rows
    (8, 13, 40, 320, True),     # UB % 4 == 0 path with several unit blocks
    (32, 11, 24, 640, True),    # cfg-D shape: UB = 10 (tensor-core step kernels, 3 unit pairs, one padded)
    (64, 10, 120, 512, True),   # cfg-B/C shape: UB = 16, Bc = 32, 128 CTAs (tensor-core step kernels)
    (40, 9, 16, 512, False),    # unidirectional tensor-core plan (UB = 8), second batch group mostly padding rows
    (130, 5, 16, 512, True),    # more CTAs than SMs: three consecutive launches over 44-row blocks
    (64, 4, 24, 640, True),     # cfg D at batch 64: two launches of 32 rows
    (64, 300, 64, 512, True),   # T = 300: 75 periods of the wgmma backward's 4-step generation tag
    (64, 11, 24, 256, True),    # wgmma UB = 8: forward UBP 8, backward UB 8
    (64, 11, 24, 384, True),    # wgmma forward UBP 12, backward UB 16 with a last n-block 128 wide
    (64, 9, 16, 192, True),     # wgmma forward with UB = 6 (scalar publish), mma.sync backward
    (64, 5, 16, 768, True),     # FMA forward over four launches, wgmma backward over two
    (1, 9, 16, 512, True),      # a single batch row
    (96, 5, 16, 512, True),     # wgmma forward and backward over two launches
])
def test_bilstm_fwd_bwd_vs_aten_cpu(pkg, B, T, I, H, bidir):
    _check_bilstm(pkg, B, T, I, H, bidir, wtol=2e-4 if T > 100 else 1e-4)


@pytest.mark.parametrize("B,T,I,H,bidir", [(32, 11, 24, 640, True), (64, 10, 120, 512, True), (130, 5, 16, 512, True)])
def test_bilstm_fp32_fma_kernels_on_the_large_shapes(pkg, B, T, I, H, bidir):
    """The packed-FMA step kernels stay the fallback for shapes without a 16-row-tile plan; keep them covered at
    the BASELINE shapes too by forcing them."""
    lib = pkg.load_library()
    lib.b200asr_debug_set_lstm_mode(1)
    try:
        _check_bilstm(pkg, B, T, I, H, bidir)
    finally:
        lib.b200asr_debug_set_lstm_mode(0)


@pytest.mark.parametrize("B,T,I,H,bidir", [(32, 11, 24, 640, True), (64, 10, 120, 512, True), (40, 9, 16, 512, False),
                                           (64, 300, 64, 512, True), (130, 5, 16, 512, True), (64, 11, 24, 384, True)])
def test_bilstm_mma_sync_generation_on_the_large_shapes(pkg, B, T, I, H, bidir):
    """The warp-level mma.sync 3xTF32 kernels (round 1) remain the path for shapes the wgmma kernels do not take
    (H % 64 != 0 ...); keep them covered at the BASELINE shapes by forcing them (mode 3)."""
    lib = pkg.load_library()
    lib.b200asr_debug_set_lstm_mode(3)
    try:
        assert lib.b200asr_bilstm_uses_tcgen05(B, H, 2 if bidir else 1) == 0
        _check_bilstm(pkg, B, T, I, H, bidir, wtol=2e-4 if T > 100 else 1e-4)
    finally:
        lib.b200asr_debug_set_lstm_mode(0)


def test_bilstm_baseline_shapes_run_on_tcgen05(pkg):
    lib = pkg.load_library()
    assert lib.b200asr_bilstm_uses_tcgen05(64, 512, 2) == 1      # cfg B / C
    assert lib.b200asr_bilstm_uses_tcgen05(32, 640, 2) == 1      # cfg D (per GPU)
    assert lib.b200asr_bilstm_uses_tcgen05(3, 16, 2) == 0        # tiny shapes: fp32 FMA kernels


@pytest.mark.parametrize("B,T,I,H", [(64, 1198, 120, 512), (64, 599, 2048, 512), (32, 299, 640, 640)])
def test_bilstm_full_size_vs_aten_cpu(pkg, B, T, I, H):
    """BASELINE sizes (cfg B/C layer 0 and layer 1, cfg D): the recurrence over the full 1198 / 599 / 299 sequential
    steps against ATen's CPU LSTM - forward outputs, input gradient and every weight gradient."""
    torch.set_num_threads(16)
    # weight gradients are fp32 sums over B*T = 19k..77k rows of N(0,1) test gradients: the two fp32 summation orders
    # (ATen's blocked CPU GEMM vs fp32-accumulating tensor cores) differ at the 1e-4-of-max level there
    _check_bilstm(pkg, B, T, I, H, True, wtol=5e-4)


def test_bilstm_pad_through_semantics(pkg):
    """The recurrence runs over padded frames (SURVEY F5): appending zero frames changes the reverse direction."""
    ref = _torch_lstm(8, 16, True, 5)
    torch.manual_seed(6)
    x = torch.randn(2, 6, 8)
    xp = torch.cat([x, torch.zeros(2, 3, 8)], 1)
    params = [p.detach().to(DEV) for p in ref.parameters()]
    y = pkg.ops.bilstm(xp.to(DEV), params, 2).cpu()
    yr, _ = ref(xp)
    assert rel_err(y.numpy(), yr.detach().numpy()) < 1e-4
    y_short = pkg.ops.bilstm(x.to(DEV), params, 2).cpu()
    assert float((y[:, :6, :16] - y_short[:, :, :16]).abs().max()) < 1e-6      # forward direction unchanged
    assert float((y[:, :6, 16:] - y_short[:, :, 16:]).abs().max()) > 1e-4      # reverse direction saw the padding


def test_bilstm_rejects_bad_hidden_size(pkg):
    ref = _torch_lstm(8, 20, True, 1)
    params = [p.detach().to(DEV) for p in ref.parameters()]
    with pytest.raises(pkg.B200AsrError):
        pkg.ops.bilstm(torch.randn(2, 3, 8, device=DEV), params, 2)


def test_no_cpu_fallback(pkg):
    with pytest.raises(pkg.B200AsrError):
        pkg.ops.log_softmax(torch.randn(2, 5))


def test_lstm_cell(pkg):
    torch.manual_seed(0)
    B, H = 6, 32
    pre = torch.randn(B, 4 * H)
    c0 = torch.randn(B, H)
    a = pre.to(DEV).requires_grad_(True)
    c = c0.to(DEV).requires_grad_(True)
    h1, c1 = pkg.ops.lstm_cell(a, c)
    hr, cr = onp.lstm_cell(pre.double().numpy(), c0.double().numpy())
    assert scaled_err(h1.detach().cpu().numpy(), hr) < 1e-6 and scaled_err(c1.detach().cpu().numpy(), cr) < 1e-6
    gh, gc = torch.randn(B, H), torch.randn(B, H)
    (h1 * gh.to(DEV)).sum().add((c1 * gc.to(DEV)).sum()).backward()
    ar = pre.double().requires_grad_(True)
    c0r = c0.double().requires_grad_(True)
    i, f, g_, o = ar[:, :H].sigmoid(), ar[:, H:2 * H].sigmoid(), ar[:, 2 * H:3 * H].tanh(), ar[:, 3 * H:].sigmoid()
    cn = f * c0r + i * g_
    hn = o * cn.tanh()
    ((hn * gh.double()).sum() + (cn * gc.double()).sum()).backward()
    assert scaled_err(a.grad.cpu().numpy(), ar.grad.numpy()) < 1e-6
    assert scaled_err(c.grad.cpu().numpy(), c0r.grad.numpy()) < 1e-6


def _loc_attention_torch(q, key, value, prev, lens, cw, pw, ew, eb, temp):
    T = key.shape[1]
    R = (cw.shape[2] - 1) // 2
    conv = F.conv1d(prev.unsqueeze(1), cw, padding=R)
    loc = torch.tanh(F.linear(conv.transpose(1, 2), pw))
    e = F.linear(torch.tanh(key + q.unsqueeze(1) + loc), ew, eb).squeeze(2) / temp
    mask = torch.arange(T)[None, :] >= lens[:, None]
    a = torch.softmax(e.masked_fill(mask, float("-inf")), -1)
    return torch.bmm(a.unsqueeze(1), value).squeeze(1), a


@pytest.mark.parametrize("B,T,D,E,K,R,lens", [
    (3, 12, 16, 64, 4, 5, [12, 9, 5]),                 # single-CTA path (cluster size 1)
    (4, 40, 300, 256, 10, 100, [40, 33, 17, 8]),       # cluster of 4, reference-sized location conv
    (2, 149, 300, 2048, 10, 100, [149, 120]),          # cfg-C shape
    (2, 70, 48, 72, 3, 2, [70, 1]),                    # cluster of 2, a single valid frame
])
def test_loc_attention_step_fwd_bwd(pkg, B, T, D, E, K, R, lens):
    g = torch.Generator().manual_seed(B * 100 + T)
    mk = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc)
    q, key, value = mk(B, D), mk(B, T, D), mk(B, T, E)
    lens = torch.tensor(lens)
    prev = torch.rand(B, T, generator=g)
    prev = prev * (torch.arange(T)[None] < lens[:, None])
    prev = prev / prev.sum(1, keepdim=True)
    cw, pw, ew, eb = mk(K, 1, 2 * R + 1, sc=0.3), mk(D, K, sc=0.5), mk(1, D, sc=0.3), mk(1)
    gc, ga = mk(B, E), mk(B, T)
    names = ["q", "key", "value", "prev", "cw", "pw", "ew", "eb"]
    ref_in = [t.double().requires_grad_(True) for t in (q, key, value, prev, cw, pw, ew, eb)]
    cr, ar = _loc_attention_torch(ref_in[0], ref_in[1], ref_in[2], ref_in[3], lens, *ref_in[4:], 0.5)
    ((cr * gc.double()).sum() + (ar * ga.double()).sum()).backward()
    dev_in = [t.to(DEV).requires_grad_(True) for t in (q, key, value, prev, cw, pw, ew, eb)]
    c, a = pkg.ops.loc_attention_step(dev_in[0], dev_in[1], dev_in[2], dev_in[3], lens.to(DEV), *dev_in[4:], 0.5)
    assert scaled_err(a.detach().cpu().numpy(), ar.detach().numpy()) < 1e-5
    assert scaled_err(c.detach().cpu().numpy(), cr.detach().numpy()) < 1e-5
    assert float(a.detach().cpu()[torch.arange(T)[None] >= lens[:, None]].abs().max()) == 0      # masked frames
    ((c * gc.to(DEV)).sum() + (a * ga.to(DEV)).sum()).backward()
    for n, x, r in zip(names, dev_in, ref_in):
        if n == "eb":    # softmax is shift invariant: d/d(b_energy) is exactly 0 up to rounding
            assert float(x.grad.abs().max()) < 1e-5 and float(r.grad.abs().max()) < 1e-12
        else:
            assert scaled_err(x.grad.cpu().numpy(), r.grad.numpy()) < 2e-5, n


@pytest.mark.parametrize("B,T,D,E,K,R,lens,L", [
    (3, 12, 16, 64, 4, 5, [12, 9, 5], 3),
    (4, 40, 300, 256, 10, 100, [40, 33, 17, 8], 5),
    (2, 149, 300, 2048, 10, 100, [149, 120], 4),          # cfg-C shape
])
def test_loc_attention_memory_decode_loop(pkg, B, T, D, E, K, R, lens, L):
    """The decode loop's form: L chained steps (the alignment of step l feeds step l+1) on ONE attention memory -
    d(key) / weight partials accumulated in place, d(value) formed once after the loop - against the fp64 torch loop."""
    g = torch.Generator().manual_seed(B * 100 + T + L)
    mk = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc)
    qs, key, value = mk(L, B, D), mk(B, T, D), mk(B, T, E)
    lens = torch.tensor(lens)
    prev = (torch.arange(T)[None] < lens[:, None]).float()
    prev = prev / prev.sum(1, keepdim=True)
    cw, pw, ew, eb = mk(K, 1, 2 * R + 1, sc=0.3), mk(D, K, sc=0.5), mk(1, D, sc=0.3), mk(1)
    gc, ga = mk(L, B, E), mk(L, B, T)
    extra_gv = mk(B, T, E)                                 # value also feeds something else (the CTC head in the model)
    names = ["q", "key", "value", "cw", "pw", "ew", "eb"]
    ref_in = [t.double().requires_grad_(True) for t in (qs, key, value, cw, pw, ew, eb)]
    p_ref, tot = prev.double(), 0
    for l in range(L):
        c, a = _loc_attention_torch(ref_in[0][l], ref_in[1], ref_in[2], p_ref, lens, *ref_in[3:], 0.5)
        tot = tot + (c * gc[l].double()).sum() + (a * ga[l].double()).sum()
        p_ref = a
    (tot + (ref_in[2] * extra_gv.double()).sum()).backward()
    dev_in = [t.to(DEV).requires_grad_(True) for t in (qs, key, value, cw, pw, ew, eb)]
    mem, mkey, mval, mcw, mpw, mew, meb, token = pkg.ops.attention_memory(*dev_in[1:])
    p_dev, tot = prev.to(DEV), 0
    for l in range(L):
        c, a = pkg.ops.loc_attention_mem_step(mem, token, dev_in[0][l], mkey, mval, p_dev, lens.to(DEV), mcw, mpw, mew, meb, 0.5)
        tot = tot + (c * gc[l].to(DEV)).sum() + (a * ga[l].to(DEV)).sum()
        p_dev = a
    (tot + (dev_in[2] * extra_gv.to(DEV)).sum()).backward()
    for n, x, r in zip(names, dev_in, ref_in):
        if n == "eb":
            assert float(x.grad.abs().max()) < 1e-4 and float(r.grad.abs().max()) < 1e-10
        else:
            assert scaled_err(x.grad.cpu().numpy(), r.grad.numpy()) < 5e-5, n
    assert mem.dkey is None and not mem.attn                # the memory released its accumulators


@pytest.mark.parametrize("B,I,H,L", [(3, 96, 32, 4), (64, 2560, 512, 3), (32, 1792, 512, 2)])
def test_decoder_step_gemm_loop(pkg, B, I, H, L):
    """The speller's LSTM step on the own GEMM (one skinny split-K product on [x | h] . [W_ih | W_hh]^T per step, the
    weight gradients of all steps as ONE contraction at the end of the loop) against fp64 F.linear + autograd."""
    torch.manual_seed(B + I)
    w_ih, w_hh = torch.randn(4 * H, I) * 0.05, torch.randn(4 * H, H) * 0.05
    b_ih, b_hh = torch.randn(4 * H) * 0.1, torch.randn(4 * H) * 0.1
    xs, gs = torch.randn(L, B, I), torch.randn(L, B, 4 * H)
    h0 = torch.randn(B, H) * 0.5
    ref_in = [t.double().requires_grad_(True) for t in (w_ih, w_hh, b_ih, b_hh, xs, h0)]
    h, tot = ref_in[5], 0
    for l in range(L):
        pre = F.linear(ref_in[4][l], ref_in[0], ref_in[2]) + F.linear(h, ref_in[1], ref_in[3])
        tot = tot + (pre * gs[l].double()).sum()
        h = torch.tanh(pre[:, :H])                          # feed a function of the step back, like the cell does
    tot.backward()
    dev_in = [t.to(DEV).requires_grad_(True) for t in (w_ih, w_hh, b_ih, b_hh, xs, h0)]
    dw = pkg.ops.decoder_weights(*dev_in[:4])
    h, tot = dev_in[5], 0
    for l in range(L):
        pre = pkg.ops.decoder_step(dw, dev_in[4][l], h)
        tot = tot + (pre * gs[l].to(DEV)).sum()
        h = torch.tanh(pre[:, :H])
    tot.backward()
    for n, x, r in zip(["w_ih", "w_hh", "b_ih", "b_hh", "xs", "h0"], dev_in, ref_in):
        assert scaled_err(x.grad.cpu().numpy(), r.grad.numpy()) < 1e-5, n
    assert not dw[0].dpre                                   # the accumulator released its step records


def test_gemm_tf32x3_is_fp32_class(pkg):
    """The error-compensated tensor-core GEMM must be as accurate as an fp32 SGEMM (vs an fp64 product)."""
    torch.manual_seed(0)
    a = torch.randn(3000, 1024, device=DEV)
    b = torch.randn(2048, 1024, device=DEV) * 0.03
    bias = torch.randn(2048, device=DEV)
    ref = (a.double() @ b.double().t() + bias.double()).cpu().numpy()
    out = pkg.ops.mm3(pkg.ops.Split(a), pkg.ops.Split(b).t(), bias=bias,
                      out=torch.empty(3000, 2048, device=DEV)).cpu().numpy()
    sg = torch.addmm(bias, a, b.t()).cpu().numpy()          # cuBLAS SGEMM (TF32 off)
    e3, e1 = scaled_err(out, ref), scaled_err(sg, ref)
    assert e3 < 3e-6 and e3 < 20 * max(e1, 1e-7), (e3, e1)
    s = pkg.ops.Split(a)
    assert torch.equal(s.hi + s.lo, a) and int((s.hi.view(torch.int32) & 0x1fff).abs().max()) == 0


def test_linear3x_matches_fp64_linear(pkg):
    """CTC head / vocabulary projection through the 3xTF32 path: forward and all three gradients."""
    torch.manual_seed(3)
    lin = torch.nn.Linear(256, 1000)
    x = torch.randn(4, 70, 256)
    xr = x.double().requires_grad_(True)
    ref = torch.nn.functional.linear(xr, lin.weight.detach().double(), lin.bias.detach().double())
    g = torch.randn(4, 70, 1000)
    ref.backward(g.double())
    lin_d = torch.nn.Linear(256, 1000).to(DEV)
    lin_d.load_state_dict(lin.state_dict())
    xd = x.to(DEV).requires_grad_(True)
    y = pkg.ops.linear3x(xd, lin_d)
    assert y.shape == (4, 70, 1000) and scaled_err(y.detach().cpu().numpy(), ref.detach().numpy()) < 1e-5
    y.backward(g.to(DEV))
    w64 = lin.weight.detach().double().requires_grad_(True)
    b64 = lin.bias.detach().double().requires_grad_(True)
    torch.nn.functional.linear(x.double(), w64, b64).backward(g.double())
    assert scaled_err(xd.grad.cpu().numpy(), xr.grad.numpy()) < 1e-5
    assert scaled_err(lin_d.weight.grad.cpu().numpy(), w64.grad.numpy()) < 1e-5
    assert scaled_err(lin_d.bias.grad.cpu().numpy(), b64.grad.numpy()) < 1e-5
    # tiny problems stay on the plain library path
    small = torch.nn.Linear(8, 4).to(DEV)
    assert pkg.ops.linear3x(torch.randn(3, 8, device=DEV), small).shape == (3, 4)


# ------------------------------------------------------------------------------------------- optimizer
def test_grad_norm_adadelta_and_step_count_vs_torch(pkg):
    """The fused clip + Adadelta update (csrc/optim.cu) against torch.optim.Adadelta after clip_grad_norm_, 3 steps,
    then the NaN-skip rule of src/solver.py:86-89; the device step count is torch's state["step"] throughout."""
    L = pkg.lib
    lib = L.load()
    torch.manual_seed(2)
    n = 100003
    p0 = torch.randn(n)
    g0 = torch.randn(n) * 3
    p = p0.clone().to(DEV)
    g = g0.clone().to(DEV)
    sq = torch.zeros(n, device=DEV)
    acc = torch.zeros(n, device=DEV)
    norm = torch.zeros(1, device=DEV)
    count = torch.zeros(1, dtype=torch.int64, device=DEV)
    scratch = torch.empty(lib.b200asr_grad_norm_scratch_bytes(), dtype=torch.uint8, device=DEV)
    pr = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adadelta([pr], lr=1.0, eps=1e-8)
    for it in range(3):
        L.check(lib.b200asr_grad_norm(L.ptr(g), n, L.ptr(norm), L.ptr(scratch), L.stream()))
        L.check(lib.b200asr_adadelta_step(L.ptr(p), L.ptr(g), L.ptr(sq), L.ptr(acc), n, 1.0, 0.9, 1e-8, 0.0,
                                          L.ptr(norm), 5.0, L.ptr(count), L.stream()))
        pr.grad = g0.clone()
        tn = torch.nn.utils.clip_grad_norm_([pr], 5.0)
        opt.step()
        assert abs(norm.item() - tn.item()) < 1e-5 * tn.item()
        assert rel_err(p.cpu().numpy(), pr.detach().numpy(), floor=1e-3) < 1e-5
    # NaN norm -> the update is skipped (src/solver.py:86-89)
    before = p.clone()
    g[5] = float("nan")
    L.check(lib.b200asr_grad_norm(L.ptr(g), n, L.ptr(norm), L.ptr(scratch), L.stream()))
    L.check(lib.b200asr_adadelta_step(L.ptr(p), L.ptr(g), L.ptr(sq), L.ptr(acc), n, 1.0, 0.9, 1e-8, 0.0,
                                      L.ptr(norm), 5.0, L.ptr(count), L.stream()))
    assert torch.isnan(norm).item() and torch.equal(p, before)
    assert count.item() == 3 == int(opt.state_dict()["state"][0]["step"])


def test_grad_norm_adam_and_step_count_vs_torch(pkg):
    """The fused clip + Adam update (csrc/optim.cu) against torch.optim.Adam after clip_grad_norm_, 3 steps with bias
    correction, then the NaN-skip rule of src/solver.py:86-89 (the device step count does not advance)."""
    L = pkg.lib
    lib = L.load()
    torch.manual_seed(3)
    n = 70001
    p0 = torch.randn(n)
    p = p0.clone().to(DEV)
    m = torch.zeros(n, device=DEV)
    v = torch.zeros(n, device=DEV)
    norm = torch.zeros(1, device=DEV)
    count = torch.zeros(1, dtype=torch.int64, device=DEV)
    scratch = torch.empty(lib.b200asr_grad_norm_scratch_bytes(), dtype=torch.uint8, device=DEV)
    pr = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([pr], lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
    for it in range(3):
        g0 = torch.randn(n) * (0.01 if it == 1 else 3.0)         # step 1 is below the clip threshold
        g = g0.clone().to(DEV)
        L.check(lib.b200asr_grad_norm(L.ptr(g), n, L.ptr(norm), L.ptr(scratch), L.stream()))
        L.check(lib.b200asr_adam_step(L.ptr(p), L.ptr(g), L.ptr(m), L.ptr(v), n, 1e-3, 0.9, 0.999, 1e-8, 0.0,
                                      L.ptr(norm), 5.0, L.ptr(count), L.stream()))
        pr.grad = g0.clone()
        tn = torch.nn.utils.clip_grad_norm_([pr], 5.0)
        opt.step()
        assert abs(norm.item() - tn.item()) < 1e-5 * tn.item()
        assert rel_err(p.cpu().numpy(), pr.detach().numpy(), floor=1e-3) < 1e-5
    before = p.clone()
    g[7] = float("nan")
    L.check(lib.b200asr_grad_norm(L.ptr(g), n, L.ptr(norm), L.ptr(scratch), L.stream()))
    L.check(lib.b200asr_adam_step(L.ptr(p), L.ptr(g), L.ptr(m), L.ptr(v), n, 1e-3, 0.9, 0.999, 1e-8, 0.0,
                                  L.ptr(norm), 5.0, L.ptr(count), L.stream()))
    assert torch.isnan(norm).item() and torch.equal(p, before)
    assert count.item() == 3 == int(opt.state_dict()["state"][0]["step"])


def test_ctc_prefix_score_vs_reference_scorer(pkg):
    """GPU CTCPrefixScore (one launch for all hypotheses x candidates) against the reference's numpy scorer."""
    g = load_golden("ctc_prefix.npz")
    x = torch.from_numpy(g["x"]).to(DEV)
    sc = pkg.ctc.CTCPrefixScore(x)
    assert rel_err(sc.init_state().cpu().numpy(), g["r_init"]) < 1e-6
    n = int(g["n_steps"])
    for s in range(n):                                        # the reference's one-hypothesis call
        psi, r = sc.cheap_compute(list(g["s%d_prefix" % s]), g["s%d_rprev" % s], list(g["s%d_cands" % s]))
        assert rel_err(psi, g["s%d_psi" % s]) < 1e-5
        assert rel_err(r, g["s%d_r" % s]) < 1e-5
    # batched: steps 0 and 2 have 4 candidates each -> two hypotheses in one launch
    psi, r = sc.cheap_compute_batch([list(g["s0_prefix"]), list(g["s2_prefix"])],
                                    [g["s0_rprev"], g["s2_rprev"]], [list(g["s0_cands"]), list(g["s2_cands"])])
    assert rel_err(psi[0].cpu().numpy(), g["s0_psi"]) < 1e-5 and rel_err(psi[1].cpu().numpy(), g["s2_psi"]) < 1e-5
    assert rel_err(r[1].cpu().numpy(), g["s2_r"]) < 1e-5


@pytest.mark.parametrize("M,N,K,acc", [(3000, 2048, 1024, False), (300, 31, 120, False), (129, 257, 64, True),
                                      (1000, 5000, 2048, False), (77, 300, 2048, True), (5, 8, 4, False)])
def test_gemm3x_tn_is_fp32_class(pkg, M, N, K, acc):
    """csrc/gemm.cu (wgmma tf32, raw tiles as hi + on-the-fly residual tiles, register accumulator) must be as
    accurate as an fp32 SGEMM against an fp64 product - incl. M / N / K tails, bias, accumulate and ldc > N."""
    torch.manual_seed(M + N)
    a = torch.randn(M, K, device=DEV)
    b = torch.randn(N, K, device=DEV) * 0.05
    bias = torch.randn(N, device=DEV)
    ldc = N + (4 if acc else 0)
    buf = torch.randn(M, ldc, device=DEV)
    out = buf[:, :N]
    c0 = out.clone()
    ref = a.double() @ b.double().t() + bias.double() + (c0.double() if acc else 0)
    pkg.ops.gemm_tn(a, b, bias=bias, out=out, accumulate=acc)
    sg = torch.addmm(bias, a, b.t()) + (c0 if acc else 0)                       # cuBLAS SGEMM (TF32 off)
    e3 = scaled_err(out.cpu().numpy(), ref.cpu().numpy())
    e1 = scaled_err(sg.cpu().numpy(), ref.cpu().numpy())
    assert e3 < 3e-6 and e3 < 20 * max(e1, 1e-7), (e3, e1)
    # pre-split form: the residual of B computed once (b200asr_tf32_residual) and loaded by TMA
    blo = pkg.ops.tf32_residual(b)
    assert torch.equal((b.view(torch.int32) & -8192).view(torch.float32) + blo, b)
    out.copy_(c0)
    pkg.ops.gemm_tn(a, b, bias=bias, out=out, accumulate=acc, w_lo=blo)
    e3 = scaled_err(out.cpu().numpy(), ref.cpu().numpy())
    assert e3 < 3e-6 and e3 < 20 * max(e1, 1e-7), (e3, e1)
    if acc:
        assert torch.equal(buf[:, N:], buf[:, N:])                              # padding columns untouched (no NaN)


@pytest.mark.parametrize("n", [1, 5, 4096, 4099, 3 * 4096 + 1027, 1 << 20])
def test_tf32_residual_pass(pkg, n):
    """lo = x - trunc_tf32(x) elementwise (unrolled 128-bit body + scalar tail; unaligned views take the scalar path)."""
    torch.manual_seed(n)
    x = torch.randn(n + 1, device=DEV)
    for v in (x[:n], x[1:]):
        lo = pkg.ops.tf32_residual(v)
        assert torch.equal((v.contiguous().view(torch.int32) & -8192).view(torch.float32) + lo, v)
        assert float(lo.abs().max()) <= float(v.abs().max()) * 2.0 ** -10


def _kernel_names(pkg, fn):
    """Run fn() with the kernel timer on: the names of the timed launches it made."""
    timer = pkg.lib.TIMER
    timer.reset()
    timer.enabled = True
    try:
        fn()
    finally:
        timer.enabled = False
    names = {r[0] for r in timer.records}
    timer.reset()
    return names


@pytest.mark.parametrize("B,T,C,O", [(3, 41, 120, 640), (2, 10, 640, 640)])
def test_conv1d_k4s2_selects_the_gemm_kernel(pkg, B, T, C, O):
    """CNNExtractor's Conv1d(k=4, s=2, p=1) runs as one wgmma GEMM over the in-place im2col view (overlapping rows,
    lda = 2C < K = 4C), checked against the library convolution in fp64: output, input gradient, weight / bias
    gradients; its forward and both gradients go through the tn / nn / nt forms of csrc/gemm.cu."""
    torch.manual_seed(C + T)
    conv = torch.nn.Conv1d(C, O, 4, stride=2, padding=1)
    x = torch.randn(B, T, C)
    xr = x.double().requires_grad_(True)
    ref = torch.nn.functional.conv1d(xr.transpose(1, 2), conv.weight.detach().double(), conv.bias.detach().double(),
                                     stride=2, padding=1).transpose(1, 2)
    gy = torch.randn(B, T // 2, O)
    ref.backward(gy.double())
    cd = torch.nn.Conv1d(C, O, 4, stride=2, padding=1).to(DEV)
    cd.load_state_dict(conv.state_dict())
    xd = x.to(DEV).requires_grad_(True)

    def step():
        y = pkg.ops.conv1d_k4s2p1(xd, cd)
        assert y.shape == ref.shape and scaled_err(y.detach().cpu().numpy(), ref.detach().numpy()) < 1e-5
        y.backward(gy.to(DEV))

    names = _kernel_names(pkg, step)
    assert {"gemm3x_tn", "gemm3x_nn", "gemm3x_nt"} <= names, names
    assert scaled_err(xd.grad.cpu().numpy(), xr.grad.numpy()) < 1e-5
    wref = torch.autograd.grad(torch.nn.functional.conv1d(x.double().transpose(1, 2), conv.weight.double(),
                                                          conv.bias.double(), stride=2, padding=1).transpose(1, 2),
                               [conv.weight, conv.bias], gy.double())
    assert scaled_err(cd.weight.grad.cpu().numpy(), wref[0].numpy()) < 1e-5
    assert scaled_err(cd.bias.grad.cpu().numpy(), wref[1].numpy()) < 1e-5


def test_bilstm_gemm_path_follows_the_input_width(pkg):
    """The BiLSTM layer's GEMMs follow the input width alone: I % 4 != 0 runs three cuBLAS TF32 GEMMs on
    b200asr_split_tf32 operands (Split + mm3), I % 4 == 0 the f16x3 products and never the 3xTF32 kernel."""
    for B, T, I, H in [(8, 13, 42, 320), (64, 10, 122, 512)]:
        names = _kernel_names(pkg, lambda: _check_bilstm(pkg, B, T, I, H, True))
        assert "split_tf32" in names and "f16_split" not in names, names
    for B, T, I, H in [(8, 13, 40, 320), (64, 10, 120, 512)]:
        names = _kernel_names(pkg, lambda: _check_bilstm(pkg, B, T, I, H, True))
        assert "f16_split" in names and not any(n.startswith("gemm3x_") for n in names), names


def test_linear3x_fn_selects_the_gemm_kernel(pkg):
    """Linear3xFn forward and input gradient against fp64; forward and both gradients go through the tn / nn / nt forms
    of csrc/gemm.cu."""
    torch.manual_seed(3)
    lin = torch.nn.Linear(256, 1000)
    x = torch.randn(4, 70, 256)
    xr = x.double().requires_grad_(True)
    ref = torch.nn.functional.linear(xr, lin.weight.detach().double(), lin.bias.detach().double())
    g = torch.randn(4, 70, 1000)
    ref.backward(g.double())
    lin_d = torch.nn.Linear(256, 1000).to(DEV)
    lin_d.load_state_dict(lin.state_dict())
    xd = x.to(DEV).requires_grad_(True)

    def step():
        y = pkg.ops.Linear3xFn.apply(xd, lin_d.weight, lin_d.bias)
        assert scaled_err(y.detach().cpu().numpy(), ref.detach().numpy()) < 1e-5
        y.backward(g.to(DEV))

    names = _kernel_names(pkg, step)
    assert {"gemm3x_tn", "gemm3x_nn", "gemm3x_nt"} <= names, names
    assert scaled_err(xd.grad.cpu().numpy(), xr.grad.numpy()) < 1e-5


@pytest.mark.parametrize("M,N,K,acc", [(3000, 2048, 1024, False), (300, 120, 2048, False), (129, 260, 64, True),
                                      (77, 300, 2048, True), (5, 8, 4, False)])
def test_gemm3x_nn_is_fp32_class(pkg, M, N, K, acc):
    """Input-gradient form C (+)= A[M,K] . B[K,N]: B read in place as an MN-major tensor-core operand."""
    torch.manual_seed(M + N + 1)
    a = torch.randn(M, K, device=DEV)
    b = torch.randn(K, N, device=DEV) * 0.05
    out = torch.randn(M, N, device=DEV)
    c0 = out.clone()
    ref = a.double() @ b.double() + (c0.double() if acc else 0)
    pkg.ops.gemm_nn(a, b, out=out, accumulate=acc)
    sg = a @ b + (c0 if acc else 0)
    e3 = scaled_err(out.cpu().numpy(), ref.cpu().numpy())
    e1 = scaled_err(sg.cpu().numpy(), ref.cpu().numpy())
    assert e3 < 3e-6 and e3 < 20 * max(e1, 1e-7), (e3, e1)


@pytest.mark.parametrize("M,N,T,batches,shift,perm", [
    (2048, 120, 5000, 1, 0, True),        # dW_ih of layer 0: long contraction, one narrow column tile -> split-K
    (2048, 512, 37, 8, -1, True),         # dW_hh, forward direction: h_prev = output shifted by one step, per utterance
    (2048, 512, 37, 8, 1, True),          # dW_hh, reverse direction
    (300, 31, 700, 1, 0, False),          # CTC head (V = 31): M / N tails
    (100, 260, 64, 3, 0, False),          # two column tiles, the second almost empty
    (2560, 640, 20000, 1, 0, True),       # cfg D size class: 20 x 3 tiles, long K, no split
])
def test_gemm3x_nt_is_fp32_class(pkg, M, N, T, batches, shift, perm):
    """Weight-gradient form C = sum_(b,t) A[b,t,:]^T B[b,t+shift,:] (both operands MN-major, TMA zero fill outside
    [0,T), row permutation in the epilogue, deterministic split-K) against fp64."""
    torch.manual_seed(M + N + T)
    ldb = (N + 3) // 4 * 4 + 4                     # padded pitch: the operand is a column slice of a wider buffer
    a = torch.randn(batches, T, M, device=DEV)
    bfull = torch.randn(batches, T, ldb, device=DEV)
    b = bfull[:, :, :N]
    bs = torch.zeros(batches, T, N, device=DEV, dtype=torch.float64)
    if shift == 0:
        bs[:] = b.double()
    elif shift < 0:
        bs[:, 1:] = b[:, :-1].double()
    else:
        bs[:, :-1] = b[:, 1:].double()
    ref = torch.einsum("btm,btn->mn", a.double(), bs)
    sg = torch.einsum("btm,btn->mn", a, bs.float())
    if perm:
        idx = torch.arange(M, device=DEV)
        dst = (idx % 4) * (M // 4) + idx // 4
        r2 = torch.empty_like(ref); r2[dst] = ref; ref = r2
        s2 = torch.empty_like(sg); s2[dst] = sg; sg = s2
    out = pkg.ops.gemm_nt(a, bfull, M, N, T, batches=batches, a_bstride=T * M, ldb=ldb, b_bstride=T * ldb,
                          b_shift=shift, permute_rows=perm)
    out2 = pkg.ops.gemm_nt(a, bfull, M, N, T, batches=batches, a_bstride=T * M, ldb=ldb, b_bstride=T * ldb,
                           b_shift=shift, permute_rows=perm)
    assert torch.equal(out, out2)                                               # deterministic (split-K in fixed order)
    e3 = scaled_err(out.cpu().numpy(), ref.cpu().numpy())
    e1 = scaled_err(sg.cpu().numpy(), ref.cpu().numpy())
    assert e3 < 3e-6 and e3 < 20 * max(e1, 1e-7), (e3, e1)
