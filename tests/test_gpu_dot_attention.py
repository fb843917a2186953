"""Scaled dot-product attention (attention.mode: dot, one or more heads) on the GPU: b200asr_dotattn_fwd /
b200asr_dotattn_bwd_acc + b200asr_attn_dvalue through ops.attention_memory / ops.dot_attention_mem_step against a
float64 restatement of the reference's ScaleDotAttention, the golden dot models through ASR, and CUDA-graph replay.

Bounds (EPS = 2^-24, the fp32 unit roundoff), fixed here, independent of any run: every output and gradient is a
contraction of at most n = max(T, D, E) fp32 terms followed by a softmax (expf within 2 ulp), so n * EPS of the
tensor's scale for one step; the decode loop adds one more level of accumulation over its L steps.
"""
import numpy as np
import pytest
import torch

import test_gpu_model as gm
from conftest import load_golden, rel_err, scaled_err
from oracle.make_golden import tiny_model_cfg
from oracle.make_golden_dotattn import dotattn_model_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24
MAX_T = 8192                    # B200ASR_DOTATTN_MAX_T


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _dot_attention_torch(q, key, value, lens, N, temp):
    """The reference's ScaleDotAttention.forward + _attend (src/module.py:189-212) on R = B * N rows; row r is masked
    by lens[r // N] (BaseAttention.compute_mask's [B, N, T] mask viewed as [B*N, T])."""
    T = key.shape[1]
    e = torch.bmm(q.unsqueeze(1), key.transpose(1, 2)).squeeze(1) / temp
    mask = (torch.arange(T)[None, :] >= lens[:, None]).repeat_interleave(N, 0)
    a = torch.softmax(e.masked_fill(mask, float("-inf")), -1)
    return torch.bmm(a.unsqueeze(1), value).squeeze(1), a


def _inputs(B, N, T, D, E, L, seed, repeat=False):
    """Ragged lengths from T down to 1; +-1e6 garbage in every padded key and value frame.  repeat: value is the
    [B, T, E] encoder output repeated N times (Attention.forward without a value projection), so row r reads
    utterance r mod B up to the length of utterance r // N."""
    g = torch.Generator().manual_seed(seed)
    mk = lambda *s: torch.randn(*s, generator=g)
    R = B * N
    lens = torch.linspace(T, 1, B).round().long()
    qs, key = mk(L, R, D), mk(R, T, D)
    value = mk(B, T, E).repeat(N, 1, 1) if repeat else mk(R, T, E)
    pad = (torch.arange(T)[None] >= lens[:, None]).repeat_interleave(N, 0)
    key[pad] = 1e6 * torch.sign(mk(int(pad.sum()), D))                # finite garbage the kernels must never read
    value[pad] = 1e6 * torch.sign(mk(int(pad.sum()), E))
    return lens, qs, key, value, pad, mk(L, R, E), mk(L, R, T)


def _run_device(ops, lens, qs, key, value, gc, ga, N, temp, L):
    dev_in = [t.to(DEV).requires_grad_(True) for t in (qs, key, value)]
    mem, mkey, mval, token = ops.attention_memory(dev_in[1], dev_in[2])
    tot, outs = 0, []
    for l in range(L):
        c, a = ops.dot_attention_mem_step(mem, token, dev_in[0][l], mkey, mval, lens.to(DEV), N, temp)
        tot = tot + (c * gc[l].to(DEV)).sum() + (a * ga[l].to(DEV)).sum()
        outs.append((c.detach(), a.detach()))
    tot.backward()
    return dev_in, outs


def _run_reference(lens, qs, key, value, gc, ga, N, temp, L):
    torch.set_num_threads(16)
    ref_in = [t.double().requires_grad_(True) for t in (qs, key, value)]
    tot, outs = 0, []
    for l in range(L):
        c, a = _dot_attention_torch(ref_in[0][l], ref_in[1], ref_in[2], lens, N, temp)
        tot = tot + (c * gc[l].double()).sum() + (a * ga[l].double()).sum()
        outs.append((c.detach(), a.detach()))
    tot.backward()
    return ref_in, outs


# (B, N, T, D, E, repeat); "n1_cfgc" takes B = sm_count + 5 rows at run time
CASES = {
    "n1_cfgc": (None, 1, 149, 300, 2048, False),        # cfg C's decode shape, more rows than SMs
    "n4_vproj": (6, 4, 149, 300, 2048, False),          # four heads, value projection: distinct value rows
    "n4_repeat": (5, 4, 149, 300, 2048, True),          # four heads, value.repeat(4, 1, 1)
    "d512_e4096": (3, 1, 149, 512, 4096, False),        # the limits D = 512 and E / CS = 1024
    "max_t": (2, 1, MAX_T, 64, 128, False),             # the longest memory the kernels take
}


@pytest.mark.parametrize("case", list(CASES))
def test_single_step_matches_float64(pkg, case):
    lib = pkg.load_library()
    sms = lib.b200asr_device_sm_count()
    B, N, T, D, E, repeat = CASES[case]
    B = sms + 5 if B is None else B
    R = B * N
    assert pkg.ops.dot_attention_supported(T, D, E) and lib.b200asr_dotattn_supported(T, D, E) == 1
    if case == "n1_cfgc":                    # more CTAs than SMs: the two-CTAs-per-SM backward instance
        assert R > sms and lib.b200asr_debug_dotattn_bwd_minb(R, T, E) == 2
    if case == "d512_e4096":
        assert lib.b200asr_locattn_cluster_size(T, E) == 4 and lib.b200asr_debug_dotattn_bwd_minb(R, T, E) == 1
    lens, qs, key, value, pad, gc, ga = _inputs(B, N, T, D, E, 1, seed=R + D + T, repeat=repeat)
    assert int(lens.max()) == T and int(lens.min()) == 1
    bound = max(T, D, E) * EPS
    ref_in, ref_out = _run_reference(lens, qs, key, value, gc, ga, N, 0.5, 1)
    dev_in, dev_out = _run_device(pkg.ops, lens, qs, key, value, gc, ga, N, 0.5, 1)
    (c, a), (cr, ar) = dev_out[0], ref_out[0]
    assert scaled_err(a.cpu().numpy(), ar.numpy()) <= bound
    assert scaled_err(c.cpu().numpy(), cr.numpy()) <= bound
    for n, x, r in zip(("q", "key", "value"), dev_in, ref_in):
        assert scaled_err(x.grad.cpu().numpy(), r.grad.numpy()) <= bound, n
    # padded frames: attention and both memory gradients exactly 0
    assert float(a.cpu()[pad].abs().max()) == 0
    assert float(dev_in[1].grad.cpu()[pad].abs().max()) == 0 and float(dev_in[2].grad.cpu()[pad].abs().max()) == 0


def test_decode_loop_matches_float64(pkg):
    """cfg C's 46 decode steps on one memory: four heads in the repeat form (d(key) accumulated in place per step,
    d(value) formed once after the loop)."""
    B, N, T, D, E, L = 4, 4, 149, 300, 2048, 46
    lens, qs, key, value, pad, gc, ga = _inputs(B, N, T, D, E, L, seed=11, repeat=True)
    bound = (2 * max(T, D, E) + L) * EPS
    ref_in, ref_out = _run_reference(lens, qs, key, value, gc, ga, N, 0.5, L)
    dev_in, dev_out = _run_device(pkg.ops, lens, qs, key, value, gc, ga, N, 0.5, L)
    for (c, a), (cr, ar) in zip(dev_out, ref_out):
        assert scaled_err(a.cpu().numpy(), ar.numpy()) <= bound
        assert scaled_err(c.cpu().numpy(), cr.numpy()) <= bound
    for n, x, r in zip(("q", "key", "value"), dev_in, ref_in):
        assert scaled_err(x.grad.cpu().numpy(), r.grad.numpy()) <= bound, n
    assert float(dev_in[1].grad.cpu()[pad].abs().max()) == 0 and float(dev_in[2].grad.cpu()[pad].abs().max()) == 0


def test_backward_is_deterministic(pkg):
    """No float atomics: two decode loops on the same inputs give bit-identical outputs and gradients."""
    B, N, T, D, E, L = 20, 4, 149, 300, 2048, 6
    lens, qs, key, value, pad, gc, ga = _inputs(B, N, T, D, E, L, seed=5, repeat=True)
    runs = [_run_device(pkg.ops, lens, qs, key, value, gc, ga, N, 0.5, L) for _ in range(2)]
    (i0, o0), (i1, o1) = runs
    for x, y in zip(i0, i1):
        assert torch.equal(_bits(x.grad), _bits(y.grad))
    for (c0, a0), (c1, a1) in zip(o0, o1):
        assert torch.equal(_bits(c0), _bits(c1)) and torch.equal(_bits(a0), _bits(a1))


# --------------------------------------------------------------------------------------------- golden models
def _model_cfg(kind):
    return tiny_model_cfg(kind) if kind == "dot" else dotattn_model_cfg(kind)


def _golden_model(pkg, kind):
    g = load_golden("model_%s.npz" % kind)
    cfg = _model_cfg(kind)
    model = pkg.ASR(g["feat"].shape[-1], g["sd.pre_embed.weight"].shape[0], True, **cfg)
    sd = {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")}
    assert set(sd.keys()) == set(model.state_dict().keys())
    model.load_state_dict(sd)
    return g, model.to(DEV)


@pytest.mark.parametrize("kind", ["dot1", "dotrep"])
def test_train_step_matches_reference(pkg, kind):
    """Outputs, att_seq, losses, every gradient and the grad-norm of the reference's dot-attention models, to the
    tolerances of test_gpu_model.test_train_step_matches_reference."""
    g, model = _golden_model(pkg, kind)
    model.train()
    feat, flen, txt = (torch.from_numpy(g[k]).to(DEV) for k in ("feat", "feat_len", "txt"))
    txt_len = (txt != 0).sum(-1)
    ctc_out, enc_len, att_out, att_seq, _ = model(feat, flen, int(txt_len.max()), tf_rate=1.0, teacher=txt)
    assert np.array_equal(enc_len.cpu().numpy(), g["encode_len"])
    total = 0
    if ctc_out is not None:
        assert rel_err(ctc_out.detach().cpu().numpy(), g["ctc_output"]) < 1e-4
        assert np.array_equal(ctc_out.argmax(-1).cpu().numpy(), g["ctc_argmax"])
        ctc = pkg.CTCLoss(blank=0)(ctc_out.transpose(0, 1), txt, enc_len, txt_len)
        assert abs(ctc.item() - float(g["ctc_loss"])) < 1e-4 * abs(float(g["ctc_loss"]))
        total = total + ctc * model.ctc_weight
    assert rel_err(att_out.detach().cpu().numpy(), g["att_output"],
                   floor=max(1e-3, 0.05 * float(np.abs(g["att_output"]).max()))) < 1e-4
    assert att_seq.shape == g["att_seq"].shape                          # [B, N, L, T]
    assert rel_err(att_seq.detach().cpu().numpy(), g["att_seq"], floor=1e-4) < 1e-4
    assert np.array_equal(att_out.argmax(-1).cpu().numpy(), g["att_argmax"])
    b, t, _ = att_out.shape
    ce = pkg.ops.cross_entropy(att_out.view(b * t, -1), txt[:, :t].reshape(-1), ignore_index=0)
    assert abs(ce.item() - float(g["att_loss"])) < 1e-4 * abs(float(g["att_loss"]))
    total = total + ce * (1 - model.ctc_weight)
    assert abs(total.item() - float(g["total_loss"])) < 1e-4 * abs(float(g["total_loss"]))
    total.backward()
    sq, n = 0.0, 0
    for k, p in model.named_parameters():
        if "grad." + k in g:
            ref = g["grad." + k]
            assert float(np.abs(p.grad.cpu().numpy() - ref).max()) < 2e-4 * max(float(np.abs(ref).max()), 1e-4), k
            sq += float((p.grad.double() ** 2).sum())
            n += 1
    assert n == sum(1 for k in g if k.startswith("grad.")) and n > 0
    assert abs(np.sqrt(sq) - float(g["grad_norm"])) < 1e-4 * float(g["grad_norm"])


@pytest.mark.parametrize("kind", ["dot1", "dotrep"])
def test_greedy_ids_bit_exact(pkg, kind):
    g, model = _golden_model(pkg, kind)
    model.eval()
    feat, flen = torch.from_numpy(g["feat"]).to(DEV), torch.from_numpy(g["feat_len"]).to(DEV)
    with torch.no_grad():
        _, _, out, _, _ = model(feat, flen, g["greedy_argmax"].shape[1])
    assert np.array_equal(out.argmax(-1).cpu().numpy(), g["greedy_argmax"])
    assert rel_err(out.cpu().numpy(), g["greedy_output"],
                   floor=max(1e-3, 0.05 * float(np.abs(g["greedy_output"]).max()))) < 1e-4


@pytest.mark.parametrize("kind", ["dot", "dot1", "dotrep"])
def test_golden_models_run_the_dot_kernels(pkg, kind):
    """A train step of every dot-attention golden model launches dotattn_fwd once per decode step, dotattn_bwd_acc
    once per step and attn_dvalue once per batch: a silent library fallback fails here."""
    g, model = _golden_model(pkg, kind)
    model.train()
    feat, flen, txt = (torch.from_numpy(g[k]).to(DEV) for k in ("feat", "feat_len", "txt"))
    L = int((txt != 0).sum(-1).max())
    T = pkg.lib.TIMER
    T.reset()
    T.enabled = True
    try:
        _, _, att_out, _, _ = model(feat, flen, L, tf_rate=1.0, teacher=txt)
        att_out.sum().backward()
        torch.cuda.synchronize()
        s = T.summary()
    finally:
        T.enabled = False
        T.reset()
    assert s["dotattn_fwd"]["launches"] == L and s["dotattn_bwd_acc"]["launches"] == L, s
    assert s["attn_dvalue"]["launches"] == 1 and "locattn_fwd" not in s


def test_cuda_graph_replay_equals_eager_steps(pkg):
    """Whole-step CUDA graph of a four-head dot-attention model (repeat form) against the eager steps."""
    cfg = dict(gm._tiny_config("hybrid"), model=dotattn_model_cfg("dotrep"))
    g = torch.Generator().manual_seed(11)
    wave = torch.clamp(0.05 * torch.randn(3, 9000, generator=g), -1, 1).to(DEV)
    lens = torch.tensor([9000, 9000, 9000], device=DEV)
    txt = torch.tensor([[3, 4, 4, 5, 1], [6, 7, 1, 0, 0], [8, 9, 10, 1, 0]], device=DEV)
    eager = pkg.TrainStep(cfg, 12, device=DEV, seed=5)
    graph = pkg.TrainStep(cfg, 12, device=DEV, seed=5)
    assert graph.model.attention.mode == "dot" and graph.model.attention.num_head == 4
    for _ in range(3):
        eager(wave, lens, txt, max_len=5)
    assert graph.capture(wave, lens, txt, warmup=3), graph.graph_error
    for it in range(3):
        le = eager(wave * (1.0 - 0.1 * it), lens, txt, max_len=5)
        lg = graph(wave * (1.0 - 0.1 * it), lens, txt)
        assert abs(le.item() - lg.item()) <= 1e-6 * abs(le.item()), (it, le.item(), lg.item())
    for (k, a), (_, b) in zip(eager.model.state_dict().items(), graph.model.state_dict().items()):
        assert float((a - b).abs().max()) <= 1e-6 * max(float(a.abs().max()), 1e-3), k
