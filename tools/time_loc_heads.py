"""Teacher-forced decode loop with multi-head location-aware attention at the cfg-C shape (B 64, T' 149, encoder width
2048, LSTM speller dim 512, 1 layer, V 5000, L 46, attention dim 300, K 10 location kernels of width 2R+1 = 201) with
four heads, in both value forms:
  * loc4-vproj - the value projection (Linear 2048 -> 4 x 2048),
  * loc4-rep   - without it (Attention.forward's value.repeat(4, 1, 1)).
For each: ms per decode step of forward + cross-entropy + backward on our path (b200asr_locattn_heads_fwd / _bwd_acc on
one attention memory, d(value) once by b200asr_attn_dvalue) against the library LocationAwareAttention sequence patched
in (conv1d, linear, tanh, repeat, add, tanh, linear, masked_fill, softmax, bmm at every step), interleaved repetitions
after warm-up; the per-kernel times of locattn_heads_fwd, locattn_heads_bwd_acc and attn_dvalue from the KernelTimer
with achieved GB/s against their algorithmic bytes; the two paths' logits, loss and attention-side gradients against
each other on the same weights.  Prints the card and its power limit.
    python tools/time_loc_heads.py            (env: REPS 7, STEPS 5, CONFIGS loc4-vproj,loc4-rep)
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import time_attention as ta                                           # noqa: E402  (shape, inputs, step, timers)

pkg, ops, L_ = ta.pkg, ta.ops, ta.L_
B, T, E, D, V, L, ADIM = ta.B, ta.T, ta.E, ta.D, ta.V, ta.L, ta.ADIM
REPS, STEPS = ta.REPS, ta.STEPS
CONFIGS = {"loc4-vproj": (4, True), "loc4-rep": (4, False)}
SELECTED = os.environ.get("CONFIGS", ",".join(CONFIGS)).split(",")
DEV = ta.DEV


def model(num_head, v_proj, seed=0):
    torch.manual_seed(seed)
    enc = dict(prenet="", module="LSTM", bidirection=True, dim=[E // 2], dropout=[0], layer_norm=[False], proj=[False],
               sample_rate=[1], sample_style="drop")
    att = dict(mode="loc", dim=ADIM, num_head=num_head, v_proj=v_proj, temperature=0.5, loc_kernel_size=100,
               loc_kernel_num=10)
    m = pkg.ASR(40, V, True, 0.0, enc, att, dict(module="LSTM", dim=D, layer=1, dropout=0))
    m.encoder = ta.Fixed()
    return m.to(DEV).train()



def library_attention(m):
    """Replace the attention step by the library sequence LocationAwareAttention runs on CPU tensors
    (src/module.py:234-258)."""
    layer = m.attention.att_layer

    def forward(q, k, v):
        bs_nh, ts, _ = k.shape
        bs = bs_nh // layer.num_head
        if layer.prev_att is None:
            layer.prev_att = layer.init_prev_att(bs, ts, k.device)
        loc = torch.tanh(layer.loc_proj(layer.loc_conv(layer.prev_att).transpose(1, 2)))
        loc = loc.unsqueeze(1).repeat(1, layer.num_head, 1, 1).view(-1, ts, layer.dim)
        energy = layer.gen_energy(torch.tanh(k + q.unsqueeze(1) + loc)).squeeze(2)
        output, attn = layer._attend(energy, v)
        attn = attn.view(bs, layer.num_head, ts)
        layer.prev_att = attn
        return output, attn
    layer.forward = forward
    return m


def compare(cfg, enc, lens, txt):
    N, vp = CONFIGS[cfg]
    ms = {"own": model(N, vp), "library": library_attention(model(N, vp))}
    res = {k: [] for k in ms}
    for m in ms.values():                                              # warm-up: every shape, every library choice
        for _ in range(2):
            ta.step(m, enc, lens, txt)
    torch.cuda.synchronize()
    for _ in range(REPS):
        for k, m in ms.items():
            res[k].append(ta.time_ms(lambda: ta.step(m, enc, lens, txt), STEPS) / L)
    med = {}
    for k in ms:
        r = sorted(res[k])
        med[k] = r[len(r) // 2]
        print("%-10s %-8s ms per decode step (fwd + CE + bwd): median %.3f  min %.3f  max %.3f" % (
            cfg, k, med[k], r[0], r[-1]), flush=True)
    print("%-10s own / library: %.3f" % (cfg, med["own"] / med["library"]), flush=True)
    return ms


def kernels(cfg, m, enc, lens, txt):
    L_.TIMER.reset()
    L_.TIMER.enabled = True
    try:
        for _ in range(3):
            ta.step(m, enc, lens, txt)
        torch.cuda.synchronize()
        s = L_.TIMER.summary()
    finally:
        L_.TIMER.enabled = False
        L_.TIMER.reset()
    for k in ("locattn_heads_fwd", "locattn_heads_bwd_acc", "attn_dvalue"):
        d = s[k]
        print("%-10s   %-22s %5d launches  %.4f ms / launch  %.0f GB/s (algorithmic bytes)" % (
            cfg, k, d["launches"], d["ms"] / d["launches"], d["bytes"] / (d["ms"] * 1e-3) / 1e9), flush=True)


def parity(cfg, paths, enc, lens, txt):
    """Our path against the library sequence on the same weights (both fp32)."""
    out = {}
    for name, m in paths.items():
        enc.grad = None
        loss, att = ta.step(m, enc, lens, txt)
        grads = {k: p.grad.detach().double() for k, p in m.named_parameters()
                 if p.grad is not None and k.startswith("attention.")}
        grads["encoder output"] = enc.grad.detach().double()
        out[name] = (float(loss.detach()), att.detach().double(), grads)
    (lo, ao, go), (ll, al, gl) = out["own"], out["library"]
    print("%-10s own vs library: logits max|d|/max|lib| %.2e   loss rel %.2e" % (
        cfg, float((ao - al).abs().max() / al.abs().max()), abs(lo - ll) / abs(ll)), flush=True)
    for k in sorted(gl):
        print("%-10s   d %-38s max|d|/max|lib| %.2e" % (cfg, k, float((go[k] - gl[k]).abs().max() /
                                                                     gl[k].abs().max())), flush=True)


if __name__ == "__main__":
    print("card:", ta.card(), flush=True)
    enc, lens, txt = ta.inputs()
    for cfg in SELECTED:
        paths = compare(cfg, enc, lens, txt)
        kernels(cfg, paths["own"], enc, lens, txt)
        parity(cfg, paths, enc, lens, txt)
        del paths
        torch.cuda.empty_cache()
