"""Teacher-forced decode loop of the attention speller at the cfg-C shape (B 64, T' 149, encoder width 2048, dim 512,
1 layer, V 5000, L 46, location-aware attention): ms per decode step of forward + cross-entropy + backward for
  * lstm     - our LSTM speller (step GEMM + lstm_cell),
  * gru      - our GRU speller (packed step GEMM + gru_cell),
  * gru-lib  - the library nn.GRU speller (the reference's Decoder.forward; cuDNN on the GPU),
with interleaved repetitions after warm-up.  Then the step-GEMM layout choice of the GRU speller: the packed [4H, I+H]
product against two products gi / gh ([3H, I] and [3H, H]), forward + input gradient per step plus the weight-gradient
contraction per batch / L.  Last, the GRU speller's logits, loss and decoder gradients against float64 (the CPU port of
the reference, oracle/gru_ref, in float64 on the CPU) from the same weights.  Prints the card and its power limit.
    python tools/time_decoder.py            (env: REPS 9, STEPS 10)
"""
import importlib
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("end-to-end-asr-pytorch_b200")
from oracle import gru_ref                                                     # noqa: E402

ops = pkg.ops
DEV = "cuda"
B, T, E, D, V, L = 64, 149, 2048, 512, 5000, 46
REPS, STEPS = int(os.environ.get("REPS", 9)), int(os.environ.get("STEPS", 10))
ATT = dict(mode="loc", dim=300, num_head=1, v_proj=False, temperature=0.5, loc_kernel_size=100, loc_kernel_num=10)


class Fixed(torch.nn.Module):
    """Stands in for the listener: the decode loop gets the encoder output as the model input."""
    out_dim, sample_rate, vgg, cnn = E, 8, False, False

    def forward(self, x, x_len):
        return x, x_len


def model(module, seed=0):
    torch.manual_seed(seed)
    enc = dict(prenet="", module="LSTM", bidirection=True, dim=[E // 2], dropout=[0], layer_norm=[False], proj=[False],
               sample_rate=[1], sample_style="drop")
    m = pkg.ASR(40, V, True, 0.0, enc, ATT, dict(module=module, dim=D, layer=1, dropout=0))
    m.encoder = Fixed()
    return m.to(DEV).train()


def library_speller(m):
    """Replace the step by the reference's Decoder.forward (src/asr.py:214-221): nn.GRU on the library."""
    dec = m.decoder

    def forward(x, project=True):
        y, dec.hidden_state = dec.layers(x.unsqueeze(1), dec.hidden_state)
        y = y.squeeze(1)
        return (dec.project(y) if project else None), y
    dec.forward = forward
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
    return enc, lens.to(DEV), txt.to(DEV)


def step(m, enc, lens, txt):
    for p in m.parameters():
        p.grad = None
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


def spellers():
    enc, lens, txt = inputs()
    ms = {"lstm": model("LSTM"), "gru": model("GRU"), "gru-lib": library_speller(model("GRU"))}
    res = {k: [] for k in ms}
    for k, m in ms.items():                                            # warm-up: every shape, every library choice
        for _ in range(3):
            step(m, enc, lens, txt)
    torch.cuda.synchronize()
    for _ in range(REPS):
        for k, m in ms.items():
            res[k].append(time_ms(lambda: step(m, enc, lens, txt), STEPS) / L)
    for k in ms:
        r = sorted(res[k])
        print("%-8s ms per decode step (fwd + CE + bwd): median %.3f  min %.3f  max %.3f   [%s]" % (
            k, r[len(r) // 2], r[0], r[-1], " ".join("%.3f" % v for v in res[k])), flush=True)
    return ms["gru"], enc, lens, txt


def gemm_layouts():
    """Per decode step: packed product vs two products (forward, input gradient, weight gradient / L)."""
    I, H = D + E, D
    torch.manual_seed(3)
    w_ih, w_hh = 0.02 * torch.randn(3 * H, I, device=DEV), 0.02 * torch.randn(3 * H, H, device=DEV)
    b_ih, b_hh = torch.zeros(3 * H, device=DEV), torch.zeros(3 * H, device=DEV)
    x, h = torch.randn(B, I, device=DEV), torch.randn(B, H, device=DEV)
    wcat, bias = ops.pack_decoder_weights("GRU", w_ih, w_hh, b_ih, b_hh)
    wlo, lo_ih, lo_hh = ops.tf32_residual(wcat), ops.tf32_residual(w_ih), ops.tf32_residual(w_hh)
    xcat = torch.cat([x, h], 1)
    dpre = torch.randn(B, 4 * H, device=DEV)
    dgi, dgh = torch.randn(B, 3 * H, device=DEV), torch.randn(B, 3 * H, device=DEV)
    dpre_all, x_all = dpre.repeat(L, 1), xcat.repeat(L, 1)
    dgi_all, dgh_all, xi_all, h_all = dgi.repeat(L, 1), dgh.repeat(L, 1), x.repeat(L, 1), h.repeat(L, 1)

    def packed():
        ops.gemm_tn(torch.cat([x, h], 1), wcat, bias=bias, w_lo=wlo)
        ops.gemm_nn(dpre, wcat)

    def two():
        ops.gemm_tn(x, w_ih, bias=b_ih, w_lo=lo_ih)
        ops.gemm_tn(h, w_hh, bias=b_hh, w_lo=lo_hh)
        ops.gemm_nn(dgi, w_ih)
        ops.gemm_nn(dgh, w_hh)

    def packed_dw():
        ops.gemm_nt(dpre_all, x_all, 4 * H, I + H, B * L)

    def two_dw():
        ops.gemm_nt(dgi_all, xi_all, 3 * H, I, B * L)
        ops.gemm_nt(dgh_all, h_all, 3 * H, H, B * L)

    fns = {"packed": (packed, packed_dw), "two": (two, two_dw)}
    for f, g in fns.values():
        for _ in range(5):
            f()
            g()
    torch.cuda.synchronize()
    res = {k: [] for k in fns}
    for _ in range(REPS):
        for k, (f, g) in fns.items():
            res[k].append(time_ms(f, 200) + time_ms(g, 10) / L)
    for k in fns:
        r = sorted(res[k])
        print("step GEMMs %-6s ms per decode step (fwd + dX + dW/L): median %.4f  min %.4f  max %.4f" % (
            k, r[len(r) // 2], r[0], r[-1]), flush=True)


def parity(m, enc, lens, txt):
    """Our GRU speller (fp32) against the reference's decode loop in float64 on the same weights."""
    loss, att = step(m, enc, lens, txt)
    grads = {k: p.grad.detach().double() for k, p in m.named_parameters() if p.grad is not None}
    P = {k: v.detach().cpu().double().requires_grad_(True) for k, v in m.state_dict().items()}
    cfg = dict(module="GRU", dim=D, layer=1, dropout=0)
    torch.set_num_threads(min(16, os.cpu_count()))
    txt = txt.cpu()
    att64, _ = gru_ref.loc_attention_decode(P, ATT, cfg, enc.cpu().double(), lens.cpu(), txt, L)
    loss64 = torch.nn.functional.cross_entropy(att64.reshape(B * L, -1), txt.reshape(-1), ignore_index=0)
    loss64.backward()
    grads = {k: g.cpu() for k, g in grads.items()}
    lrel = float((att.detach().cpu().double() - att64.detach()).abs().max() / att64.detach().abs().max())
    print("GRU speller vs float64: logits max|d|/max|ref| %.2e   loss %.9f vs %.9f (rel %.2e)" % (
        lrel, float(loss), float(loss64.detach()), abs(float(loss) - float(loss64.detach())) / abs(float(loss64.detach()))))
    # a gradient that is zero in exact arithmetic (the energy bias: the softmax ignores a constant shift) is compared
    # against the largest gradient element of the model instead of its own rounding noise
    scale = max(float(P[k].grad.abs().max()) for k in grads)
    rel, zero = [], []
    for k, g in grads.items():
        ref, err = P[k].grad, float((g - P[k].grad).abs().max())
        if float(ref.abs().max()) > 1e-6 * scale:
            rel.append((err / float(ref.abs().max()), k))
        else:
            zero.append((err / scale, k))
    worst = max(rel)
    print("   gradients: worst max|d|/max|ref| %.2e (%s) over %d tensors; %s" % (
        worst[0], worst[1], len(rel), ", ".join("%s (zero in exact arithmetic) max|d| %.1e of the largest gradient" % (
            k, e) for e, k in zero) or "no zero gradients"))
    dec = max(v for v in rel if v[1].startswith("decoder.layers."))
    print("   GRU layer gradients: worst max|d|/max|ref| %.2e (%s)" % dec)


if __name__ == "__main__":
    print("card:", card(), flush=True)
    m, enc, lens, txt = spellers()
    gemm_layouts()
    parity(m, enc, lens, txt)
