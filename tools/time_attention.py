"""Teacher-forced decode loop with scaled dot-product attention at the cfg-C shape (B 64, T' 149, encoder width 2048,
LSTM speller dim 512, 1 layer, V 5000, L 46, attention dim 300) for three attention configurations:
  * n1       - one head, no value projection,
  * n4-vproj - four heads with the value projection (Linear 2048 -> 4 x 2048),
  * n4-rep   - four heads without it (Attention.forward's value.repeat(4, 1, 1)).
For each: ms per decode step of forward + cross-entropy + backward on our path (b200asr_dotattn_fwd / _bwd_acc on one
attention memory, d(value) once by b200asr_attn_dvalue) against the library ScaleDotAttention sequence patched in (bmm,
/ temperature, masked_fill, softmax, bmm at every step), interleaved repetitions after warm-up; the per-kernel times of
dotattn_fwd, dotattn_bwd_acc and attn_dvalue from the KernelTimer with achieved GB/s against their algorithmic bytes;
float64 parity of logits, loss and the attention-side gradients (a float64 restatement of the reference's decode loop
on the same weights).  Prints the card and its power limit.
    python tools/time_attention.py            (env: REPS 7, STEPS 5, CONFIGS n1,n4-vproj,n4-rep)
"""
import importlib
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("end-to-end-asr-pytorch_b200")

ops, L_ = pkg.ops, pkg.lib
DEV = "cuda"
B, T, E, D, V, L, ADIM = 64, 149, 2048, 512, 5000, 46, 300
REPS, STEPS = int(os.environ.get("REPS", 7)), int(os.environ.get("STEPS", 5))
CONFIGS = {"n1": (1, False), "n4-vproj": (4, True), "n4-rep": (4, False)}
SELECTED = os.environ.get("CONFIGS", ",".join(CONFIGS)).split(",")


class Fixed(torch.nn.Module):
    """Stands in for the listener: the decode loop gets the encoder output as the model input."""
    out_dim, sample_rate, vgg, cnn = E, 8, False, False

    def forward(self, x, x_len):
        return x, x_len


def model(num_head, v_proj, seed=0):
    torch.manual_seed(seed)
    enc = dict(prenet="", module="LSTM", bidirection=True, dim=[E // 2], dropout=[0], layer_norm=[False], proj=[False],
               sample_rate=[1], sample_style="drop")
    att = dict(mode="dot", dim=ADIM, num_head=num_head, v_proj=v_proj, temperature=0.5, loc_kernel_size=100,
               loc_kernel_num=10)
    m = pkg.ASR(40, V, True, 0.0, enc, att, dict(module="LSTM", dim=D, layer=1, dropout=0))
    m.encoder = Fixed()
    return m.to(DEV).train()


def library_attention(m):
    """Replace the attention step by the library sequence ScaleDotAttention ran before (src/module.py:189-212)."""
    layer = m.attention.att_layer

    def forward(q, k, v):
        ts = k.shape[1]
        energy = torch.bmm(q.unsqueeze(1), k.transpose(1, 2)).squeeze(1)
        output, attn = layer._attend(energy, v)
        return output, attn.view(-1, layer.num_head, ts)
    layer.forward = forward
    return m


def inputs(seed=1):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(B, T, E, generator=g).to(DEV)
    lens = torch.sort(torch.randint(T // 2, T + 1, (B,), generator=g), descending=True)[0]
    lens[0] = T
    txt = torch.randint(3, V, (B, L), generator=g)
    for b in range(B):
        txt[b, int(torch.randint(L // 2, L, (1,), generator=g)):] = 0
    txt[0, -1] = 1
    return enc.requires_grad_(True), lens.to(DEV), txt.to(DEV)


def step(m, enc, lens, txt):
    for p in m.parameters():
        p.grad = None
    enc.grad = None
    _, _, att, _, _ = m(enc, lens, L, tf_rate=1.0, teacher=txt)
    loss = ops.cross_entropy(att.reshape(B * L, -1), txt.reshape(-1), ignore_index=0)
    loss.backward()
    m.attention.reset_mem()
    m.decoder.hidden_state = None
    m.decoder._dw = None
    return loss, att


def time_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                             "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    except OSError:
        pl = "power limit not readable"
    return "%s (%s)" % (name, pl)


def compare(cfg, enc, lens, txt):
    N, vp = CONFIGS[cfg]
    ms = {"own": model(N, vp), "library": library_attention(model(N, vp))}
    res = {k: [] for k in ms}
    for m in ms.values():                                              # warm-up: every shape, every library choice
        for _ in range(2):
            step(m, enc, lens, txt)
    torch.cuda.synchronize()
    for _ in range(REPS):
        for k, m in ms.items():
            res[k].append(time_ms(lambda: step(m, enc, lens, txt), STEPS) / L)
    med = {}
    for k in ms:
        r = sorted(res[k])
        med[k] = r[len(r) // 2]
        print("%-9s %-8s ms per decode step (fwd + CE + bwd): median %.3f  min %.3f  max %.3f" % (
            cfg, k, med[k], r[0], r[-1]), flush=True)
    print("%-9s own / library: %.3f" % (cfg, med["own"] / med["library"]), flush=True)
    return ms


def kernels(cfg, m, enc, lens, txt):
    L_.TIMER.reset()
    L_.TIMER.enabled = True
    try:
        for _ in range(3):
            step(m, enc, lens, txt)
        torch.cuda.synchronize()
        s = L_.TIMER.summary()
    finally:
        L_.TIMER.enabled = False
        L_.TIMER.reset()
    for k in ("dotattn_fwd", "dotattn_bwd_acc", "attn_dvalue"):
        d = s[k]
        print("%-9s   %-16s %5d launches  %.4f ms / launch  %.0f GB/s (algorithmic bytes)" % (
            cfg, k, d["launches"], d["ms"] / d["launches"], d["bytes"] / (d["ms"] * 1e-3) / 1e9), flush=True)


def decode64(m, enc, lens, txt):
    """The reference's teacher-forced decode loop (src/asr.py:72-155, Attention / ScaleDotAttention / Decoder) in
    float64 on the model's weights: -> logits [B, L, V]."""
    P = {k: v.detach().double().requires_grad_(True) for k, v in m.named_parameters()}
    att = m.attention
    N, ad = att.num_head, att.dim
    x = enc.detach().double().requires_grad_(True)
    key = torch.tanh(F.linear(x, P["attention.proj_k.weight"], P["attention.proj_k.bias"]))
    key = key.view(B, T, N, ad).permute(0, 2, 1, 3).reshape(B * N, T, ad)
    if att.v_proj:
        val = torch.tanh(F.linear(x, P["attention.proj_v.weight"], P["attention.proj_v.bias"]))
        val = val.view(B, T, N, E).permute(0, 2, 1, 3).reshape(B * N, T, E)
    else:
        val = x.repeat(N, 1, 1)
    pad = (torch.arange(T, device=DEV)[None] >= lens[:, None]).repeat_interleave(N, 0)
    h = x.new_zeros(B, D)
    c = x.new_zeros(B, D)
    emb = P["pre_embed.weight"]
    last = emb[torch.zeros(B, dtype=torch.long, device=DEV)]
    teach = emb[txt]
    outs = []
    for t in range(L):
        q = torch.tanh(F.linear(h, P["attention.proj_q.weight"], P["attention.proj_q.bias"])).view(B * N, ad)
        e = torch.bmm(q.unsqueeze(1), key.transpose(1, 2)).squeeze(1) / att.att_layer.temperature
        a = torch.softmax(e.masked_fill(pad, float("-inf")), -1)
        ctx = torch.bmm(a.unsqueeze(1), val).squeeze(1)
        if N > 1:
            ctx = F.linear(ctx.view(B, N * E), P["attention.merge_head.weight"], P["attention.merge_head.bias"])
        h, c = torch.lstm_cell(torch.cat([last, ctx], -1), (h, c), P["decoder.layers.weight_ih_l0"],
                               P["decoder.layers.weight_hh_l0"], P["decoder.layers.bias_ih_l0"],
                               P["decoder.layers.bias_hh_l0"])
        outs.append(F.linear(h, P["decoder.char_trans.weight"], P["decoder.char_trans.bias"]))
        last = teach[:, t]
    return torch.stack(outs, 1), P, x


def parity(cfg, paths, enc, lens, txt):
    """Both paths (fp32, same weights) against the float64 decode loop: the library sequence's own distance from
    float64 is the scale against which our path's is read (46 recurrent steps amplify fp32 rounding)."""
    att64, P, x = decode64(paths["own"], enc, lens, txt)
    loss64 = F.cross_entropy(att64.reshape(B * L, -1), txt.reshape(-1), ignore_index=0)
    loss64.backward()
    for name, m in paths.items():
        loss, att = step(m, enc, lens, txt)
        grads = {k: p.grad.detach().double() for k, p in m.named_parameters() if p.grad is not None}
        lrel = float((att.detach().double() - att64.detach()).abs().max() / att64.detach().abs().max())
        print("%-9s %-8s vs float64: logits max|d|/max|ref| %.2e   loss rel %.2e" % (
            cfg, name, lrel, abs(float(loss.detach()) - float(loss64.detach())) / abs(float(loss64.detach()))),
            flush=True)
        rows = [(k, grads[k], P[k].grad) for k in sorted(grads) if k.startswith("attention.")]
        rows.append(("encoder output (key / value memory)", enc.grad.detach().double(), x.grad))
        for k, g, r in rows:
            print("%-9s %-8s   d %-38s max|d|/max|ref| %.2e" % (cfg, name, k, float((g - r).abs().max() /
                                                                                     r.abs().max())), flush=True)


if __name__ == "__main__":
    print("card:", card(), flush=True)
    enc, lens, txt = inputs()
    for cfg in SELECTED:
        paths = compare(cfg, enc, lens, txt)
        kernels(cfg, paths["own"], enc, lens, txt)
        parity(cfg, paths, enc, lens, txt)
        del paths
        torch.cuda.empty_cache()
