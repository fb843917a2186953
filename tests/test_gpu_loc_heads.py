"""Multi-head location-aware attention (attention.mode: loc, num_head > 1) on the GPU: b200asr_locattn_heads_fwd /
b200asr_locattn_heads_bwd_acc + b200asr_attn_dvalue through ops.attention_memory / ops.loc_attention_heads_mem_step
per element against the float64 closed form of oracle/attn_heads_ref.py, the golden multi-head models through ASR
against the reference, and CUDA-graph replay.

Inputs: +-1e6 garbage in every padded key and value frame (the kernels must never read them; the oracle zeroes them).
Per element, |kernel - float64| <= the bound derived in oracle/attn_heads_ref.py at the GPU's own inputs (its previous
alignment, its saved attention and the d(attn) autograd hands each step); a zero bound demands exact equality.
"""
import numpy as np
import pytest
import torch

import test_gpu_model as gm
from conftest import load_golden, rel_err
from oracle import attn_heads_ref as hr
from oracle import attn_ref as ar
from oracle.make_golden_locheads import locheads_model_cfg
from test_host_loc_heads import loc_heads_torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
TINY = 2.0 ** -126               # expf of an energy far below the maximum underflows: absolute error of an attention


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _inputs(B, N, T, D, E, K, R, L, seed, repeat):
    """Ragged lengths from T down to 1; prev [B,N,T] a normalised alignment per head; repeat: value is a [B,T,E]
    tensor repeated N times (Attention.forward without a value projection: row r reads utterance r mod B up to the
    length of utterance r // N)."""
    g = torch.Generator().manual_seed(seed)
    mk = lambda *s, sc=1.0: torch.randn(*s, generator=g) * sc
    rows = B * N
    lens = torch.linspace(T, 1, B).round().long()
    upad = torch.arange(T)[None] >= lens[:, None]                             # [B, T]
    pad = upad.repeat_interleave(N, 0)                                        # [R, T]
    value = mk(B, T, E).repeat(N, 1, 1) if repeat else mk(rows, T, E)
    key = mk(rows, T, D)
    key[pad] = 1e6 * torch.sign(mk(int(pad.sum()), D))                       # finite garbage never to be read
    value[pad] = 1e6 * torch.sign(mk(int(pad.sum()), E))
    prev = torch.softmax(mk(B, N, T), -1).masked_fill(upad[:, None, :], 0.0)
    prev = prev / prev.sum(-1, keepdim=True)
    return dict(lens=lens, pad=pad, qs=mk(L, rows, D), key=key, value=value, prev=prev,
                w_conv=mk(K, N, 2 * R + 1, sc=0.3), w_proj=mk(D, K, sc=0.5), w_e=mk(D, sc=0.3), b_e=mk(1),
                gc=mk(L, rows, E), ga=mk(L, rows, T))


def _decode_loop(pkg, inp, N, L, temp):
    """L steps on one attention memory, each step's alignment the next one's prev_att; every step's d(attn) (the
    loss's plus the next step's d(prev)) captured."""
    lens = inp["lens"].to(DEV)
    leaves = {k: inp[k].to(DEV).requires_grad_(True)
              for k in ("qs", "key", "value", "w_conv", "w_proj", "w_e", "b_e")}
    mem, mk, mv, cw, pw, ew, eb, tok = pkg.ops.attention_memory(leaves["key"], leaves["value"], leaves["w_conv"],
                                                                leaves["w_proj"], leaves["w_e"].unsqueeze(0),
                                                                leaves["b_e"])
    B, T = inp["prev"].shape[0], inp["prev"].shape[2]
    prev, tot, steps, dattn = inp["prev"].to(DEV), 0, [], {}
    for l in range(L):
        c, a = pkg.ops.loc_attention_heads_mem_step(mem, tok, leaves["qs"][l], mk, mv, prev, lens, N, cw, pw, ew, eb,
                                                    temp)
        a.register_hook(lambda gr, l=l: dattn.__setitem__(l, gr.detach().cpu()))
        steps.append((prev.detach().cpu(), a.detach().cpu(), c.detach().cpu()))
        tot = tot + (c * inp["gc"][l].to(DEV)).sum() + (a * inp["ga"][l].to(DEV)).sum()
        prev = a.view(B, N, T)
    tot.backward()
    return leaves, steps, dattn


def _check(tag, got, ref, bound):
    r = ar.worst_ratio(got, ref, bound)
    assert r <= 1.0, (tag, r)


def _check_loop(lib, inp, N, temp, leaves, steps, dattn):
    n = lambda t: t.double().numpy()
    B, _, T = inp["prev"].shape
    E = inp["value"].shape[2]
    cs = lib.b200asr_locattn_cluster_size(T, E)
    lens = inp["lens"].numpy()
    acc = {k: [] for k in ("dkey", "dwp", "dwc", "dwe", "dbe")}
    for l, (prev, a, c) in enumerate(steps):
        st = hr.loc_heads_step(n(inp["qs"][l]), n(inp["key"]), n(inp["value"]), n(prev), lens,
                               *(n(inp[k]) for k in ("w_conv", "w_proj", "w_e", "b_e")), temp, N,
                               dctx=n(inp["gc"][l]), dattn=n(dattn[l]), attn=n(a))
        _check("step %d attn" % l, n(a), st.attn, np.where(st.valid, st.attn_b + TINY, 0.0))
        _check("step %d ctx" % l, n(c), st.ctx, st.ctx_b)
        _check("step %d dq" % l, n(leaves["qs"].grad[l].cpu()), st.dq, st.dq_b + (cs + 1) * ar.U * st.dq_abs)
        if l > 0:                      # d(attn of step l-1) = the loss's + this step's d(prev), all N channels
            ga = n(inp["ga"][l - 1])
            _check("step %d dprev" % l, n(dattn[l - 1]), ga + st.dprev.reshape(ga.shape),
                   st.dprev_b.reshape(ga.shape) + 2 * ar.U * (np.abs(ga) + st.dprev_abs.reshape(ga.shape)))
        for k in acc:
            acc[k].append((getattr(st, k), getattr(st, k + "_b"), getattr(st, k + "_abs")))
    v3 = ~inp["pad"].numpy()[:, :, None]
    val, bnd = ar.accumulate(0.0, *zip(*acc["dkey"]))
    _check("dkey", n(leaves["key"].grad.cpu()), val, np.where(v3, bnd, 0.0))
    dv, dvb = ar.dvalue(np.stack([n(a) for _, a, _ in steps], 1), n(inp["gc"].transpose(0, 1)))
    _check("dvalue", n(leaves["value"].grad.cpu()), np.where(v3, dv, 0.0), np.where(v3, dvb, 0.0))
    for k, leaf in (("dwp", "w_proj"), ("dwc", "w_conv"), ("dwe", "w_e"), ("dbe", "b_e")):
        vals, bnds, abss = zip(*acc[k])
        val, bnd = ar.accumulate(0.0, [v.sum(0) for v in vals], [b.sum(0) for b in bnds], [a.sum(0) for a in abss])
        bnd = bnd + B * cs * ar.U * sum(a.sum(0) for a in abss)
        got = n(leaves[leaf].grad.cpu())
        _check(k, got, val.reshape(got.shape), bnd.reshape(got.shape))
    # padded frames: attention and both memory gradients exactly 0
    pad = inp["pad"]
    assert all(float(a[pad].abs().max()) == 0 for _, a, _ in steps)
    assert float(leaves["key"].grad.cpu()[pad].abs().max()) == 0
    assert float(leaves["value"].grad.cpu()[pad].abs().max()) == 0


# name -> (B, N, T, D, E, K, R, repeat, MINB); B None: enough utterances that the clusters outnumber the SMs
CASES = {
    "n2_vproj_cfgc": (3, 2, 149, 300, 2048, 10, 100, False, 1),
    "n4_repeat_minb2": (None, 4, 149, 300, 512, 10, 100, True, 2),
    "n4_vproj_cfgc": (2, 4, 149, 300, 2048, 10, 100, False, 1),
    "n8_repeat": (2, 8, 61, 128, 256, 6, 20, True, 1),
    "n8_d512_e4096": (2, 8, 40, 512, 4096, 16, 5, False, 1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_single_step_matches_float64(pkg, case):
    lib = pkg.load_library()
    B, N, T, D, E, K, R, repeat, minb = CASES[case]
    cs = lib.b200asr_locattn_cluster_size(T, E)
    B = lib.b200asr_device_sm_count() // cs + 1 if B is None else B
    assert pkg.ops.loc_attention_heads_supported(N, T, D, E, K, R)
    assert lib.b200asr_locattn_heads_supported(N, T, D, E, K, R) == 1
    assert lib.b200asr_debug_locattn_heads_bwd_minb(B, N, T, D, E) == minb
    inp = _inputs(B, N, T, D, E, K, R, 1, seed=B * N + T + D, repeat=repeat)
    _check_loop(lib, inp, N, 0.5, *_decode_loop(pkg, inp, N, 1, 0.5))


@pytest.mark.parametrize("N", [2, 4, 8])
@pytest.mark.parametrize("repeat", [False, True])
def test_decode_loop_matches_float64(pkg, N, repeat):
    """46 decode steps on one memory (cfg C's L): d(key) and the weight partials accumulated in place per step,
    d(value) formed once after the loop, each step's d(prev) reaching the previous step's d(attn)."""
    lib = pkg.load_library()
    B, T, D, E, K, R, L = 3, 64, 96, 256, 6, 15, 46
    inp = _inputs(B, N, T, D, E, K, R, L, seed=N * 7 + repeat, repeat=repeat)
    _check_loop(lib, inp, N, 0.7, *_decode_loop(pkg, inp, N, L, 0.7))


def test_backward_is_deterministic(pkg):
    """No float atomics: two decode loops on the same inputs give bit-identical outputs and gradients."""
    B, N, T, D, E, K, R, L = 20, 4, 149, 300, 2048, 10, 100, 6
    inp = _inputs(B, N, T, D, E, K, R, L, seed=5, repeat=True)
    runs = [_decode_loop(pkg, inp, N, L, 0.5) for _ in range(2)]
    (l0, s0, _), (l1, s1, _) = runs
    for k in l0:
        assert torch.equal(_bits(l0[k].grad), _bits(l1[k].grad)), k
    for (_, a0, c0), (_, a1, c1) in zip(s0, s1):
        assert torch.equal(_bits(c0), _bits(c1)) and torch.equal(_bits(a0), _bits(a1))


def test_empty_utterance_gives_the_reference_nan(pkg):
    """enc_len 0: the reference's softmax of an all -inf row is NaN for every head of that utterance, and so are its
    contexts and d(value); d(key) and d(q) stay 0 (masked_fill's backward)."""
    B, N, T, D, E, K, R, temp = 2, 3, 40, 16, 64, 3, 4, 0.5
    inp = _inputs(B, N, T, D, E, K, R, 1, seed=3, repeat=False)
    inp["lens"] = torch.tensor([T, 0])
    inp["prev"][1] = 0.0
    leaves, steps, _ = _decode_loop(pkg, inp, N, 1, temp)
    _, a, c = steps[0]
    got = [torch.isnan(t) for t in (c, a, leaves["qs"].grad[0].cpu(), leaves["key"].grad.cpu(),
                                    leaves["value"].grad.cpu())]
    x = [inp[k].double().clone().requires_grad_(True) for k in ("qs", "key", "value")]
    cr, ar_ = loc_heads_torch(x[0][0], x[1], x[2], inp["prev"].double(), inp["lens"], inp["w_conv"].double(),
                              inp["w_proj"].double(), inp["w_e"].double(), inp["b_e"].double(), temp, N)
    ((cr * inp["gc"][0].double()).sum() + (ar_ * inp["ga"][0].double()).sum()).backward()
    ref = [torch.isnan(t) for t in (cr.detach(), ar_.detach(), x[0].grad[0], x[1].grad, x[2].grad)]
    for name, g, r in zip(("ctx", "attn", "d(q)", "d(key)", "d(value)"), got, ref):
        assert torch.equal(g, r), name
    assert bool(got[1][N:].all()) and not bool(got[1][:N].any())
    assert float(leaves["key"].grad[N:].abs().max()) == 0


# --------------------------------------------------------------------------------------------- golden models
def _golden_model(pkg, kind):
    g = load_golden("model_%s.npz" % kind)
    model = pkg.ASR(g["feat"].shape[-1], g["sd.pre_embed.weight"].shape[0], True, **locheads_model_cfg(kind))
    sd = {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")}
    assert set(sd.keys()) == set(model.state_dict().keys())
    model.load_state_dict(sd)
    return g, model.to(DEV)


@pytest.mark.parametrize("kind", ["loc2", "locrep"])
def test_train_step_matches_reference(pkg, kind):
    """Outputs, att_seq [B,N,L,T], losses, every gradient and the grad-norm of the reference's multi-head
    location-aware models, to the tolerances of test_gpu_dot_attention.test_train_step_matches_reference."""
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


@pytest.mark.parametrize("kind", ["loc2", "locrep"])
def test_greedy_ids_bit_exact(pkg, kind):
    g, model = _golden_model(pkg, kind)
    model.eval()
    feat, flen = torch.from_numpy(g["feat"]).to(DEV), torch.from_numpy(g["feat_len"]).to(DEV)
    with torch.no_grad():
        _, _, out, _, _ = model(feat, flen, g["greedy_argmax"].shape[1])
    assert np.array_equal(out.argmax(-1).cpu().numpy(), g["greedy_argmax"])
    assert rel_err(out.cpu().numpy(), g["greedy_output"],
                   floor=max(1e-3, 0.05 * float(np.abs(g["greedy_output"]).max()))) < 1e-4


@pytest.mark.parametrize("kind", ["loc2", "locrep"])
def test_golden_models_run_the_loc_heads_kernels(pkg, kind):
    """A train step of every multi-head location-aware golden model launches locattn_heads_fwd and
    locattn_heads_bwd_acc once per decode step and attn_dvalue once per batch, and never the single-head kernels: a
    step on the library ops would leave the forward count short."""
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
    assert s["locattn_heads_fwd"]["launches"] == L and s["locattn_heads_bwd_acc"]["launches"] == L, s
    assert s["attn_dvalue"]["launches"] == 1
    assert "locattn_fwd" not in s and "locattn_bwd" not in s


def test_cuda_graph_replay_equals_eager_steps(pkg):
    """Whole-step CUDA graph of the four-head location-aware model (repeat form) against the eager steps."""
    cfg = dict(gm._tiny_config("hybrid"), model=locheads_model_cfg("locrep"))
    g = torch.Generator().manual_seed(11)
    wave = torch.clamp(0.05 * torch.randn(3, 9000, generator=g), -1, 1).to(DEV)
    lens = torch.tensor([9000, 9000, 9000], device=DEV)
    txt = torch.tensor([[3, 4, 4, 5, 1], [6, 7, 1, 0, 0], [8, 9, 10, 1, 0]], device=DEV)
    eager = pkg.TrainStep(cfg, 12, device=DEV, seed=5)
    graph = pkg.TrainStep(cfg, 12, device=DEV, seed=5)
    assert graph.model.attention.mode == "loc" and graph.model.attention.num_head == 4
    for _ in range(3):
        eager(wave, lens, txt, max_len=5)
    assert graph.capture(wave, lens, txt, warmup=3), graph.graph_error
    for it in range(3):
        le = eager(wave * (1.0 - 0.1 * it), lens, txt, max_len=5)
        lg = graph(wave * (1.0 - 0.1 * it), lens, txt)
        assert abs(le.item() - lg.item()) <= 1e-6 * abs(le.item()), (it, le.item(), lg.item())
    for (k, a), (_, b) in zip(eager.model.state_dict().items(), graph.model.state_dict().items()):
        assert float((a - b).abs().max()) <= 1e-6 * max(float(a.abs().max()), 1e-3), k
