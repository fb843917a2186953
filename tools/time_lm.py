"""One RNN-LM train step at lm_example size (config/b200/lm_libri.yaml: V = 16000, E = H = 1024, 2 LSTM layers, dropout
0.5, Adam, B = 32) at T = 40 and T = 150 (the halving threshold): ms/step and tokens/s from CUDA events, the per-kernel
split, the recurrence plan, the card and its power limit.  Also checks the step against the functional oracle
(oracle/ref_port_lm.lm_forward_loss, ATen nn.LSTM with packing) in fp32 and fp64, and times the same step through the
library modules (cuDNN nn.LSTM + nn.Linear + cross_entropy + clip + torch.optim.Adam, TF32 off) alternated with ours.
   env: STEPS (10), WARMUP (3), ROUNDS (3), TS ("40,150")"""
import ctypes
import importlib
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("end-to-end-asr-pytorch_b200")
from oracle import ref_port_lm  # noqa: E402

L = pkg.lib
V, E, NL, B = 16000, 1024, 2, 32
STEPS, WARMUP, ROUNDS = (int(os.environ.get(k, d)) for k, d in (("STEPS", 10), ("WARMUP", 3), ("ROUNDS", 3)))
TS = [int(t) for t in os.environ.get("TS", "40,150").split(",")]
DEV = "cuda"
assert torch.cuda.is_available(), "time_lm.py measures on the GPU; there is no CPU figure to give"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def batch(T, seed=1):
    g = torch.Generator().manual_seed(seed)
    seq = torch.randint(3, V, (B, T + 1), generator=g)
    seq[:, 0] = 0
    return seq[:, :-1].to(DEV), torch.full((B,), T, dtype=torch.long), seq[:, 1:].to(DEV)


def ours(dropout=0.5):
    torch.manual_seed(0)
    model = pkg.RNNLM(V, False, E, "LSTM", E, NL, dropout).to(DEV).train()
    opt = pkg.Optimizer(model.parameters(), "Adam", 1e-4, 1e-8, "fixed")
    opt.grad_clip = 5.0

    def step(x, lens, y, parts=None):
        opt.pre_step(0)
        pred, _ = model(x, lens)
        loss = pkg.ops.cross_entropy(pred.reshape(-1, V), y.reshape(-1), ignore_index=0)
        loss.backward()
        if parts is not None:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
        opt.step()
        if parts is not None:
            b.record()
            parts.append((a, b))
        return loss
    return model, step


def library(dropout=0.5):
    torch.manual_seed(0)
    emb = torch.nn.Embedding(V, E).to(DEV)
    rnn = torch.nn.LSTM(E, E, num_layers=NL, dropout=dropout, batch_first=True).to(DEV)
    trans = torch.nn.Linear(E, V).to(DEV)
    params = list(emb.parameters()) + list(rnn.parameters()) + list(trans.parameters())
    opt = torch.optim.Adam(params, lr=1e-4, eps=1e-8)
    dp = torch.nn.Dropout(dropout)

    def step(x, lens, y):
        opt.zero_grad()
        packed = torch.nn.utils.rnn.pack_padded_sequence(dp(emb(x)), lens, batch_first=True, enforce_sorted=False)
        out, _ = rnn(packed)
        out, _ = torch.nn.utils.rnn.pad_packed_sequence(out, batch_first=True)
        loss = F.cross_entropy(trans(dp(out)).reshape(-1, V), y.reshape(-1), ignore_index=0)
        loss.backward()
        gn = torch.nn.utils.clip_grad_norm_(params, 5.0)
        if not torch.isnan(gn):
            opt.step()
        return loss
    return step


def timed(step, args, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        step(*args)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def parity(T):
    """dropout-0 step on the kernels against the oracle in fp32 and fp64 (same weights, lengths ragged up to T)."""
    model, _ = ours(dropout=0.0)
    x, lens, y = batch(T, seed=2)
    g = torch.Generator().manual_seed(3)
    lens = torch.randint(1, T + 1, (B,), generator=g)
    lens[0] = T
    for b in range(B):
        y[b, lens[b]:] = 0
    P0 = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.zero_grad(set_to_none=True)
    pred, _ = model(x, lens)
    loss = pkg.ops.cross_entropy(pred.reshape(-1, V), y.reshape(-1), ignore_index=0)
    loss.backward()
    out = []
    for dt in (torch.float32, torch.float64):
        P = {k: v.to(dt).clone().requires_grad_(True) for k, v in P0.items()}
        rl, rp = ref_port_lm.lm_forward_loss(P, NL, x, lens, y)
        rl.backward()
        gerr = max(float((p.grad.double() - P[k].grad.double()).abs().max()) /
                   max(float(P[k].grad.double().abs().max()), 1e-30) for k, p in model.named_parameters())
        out.append("%s: loss rel %.2e  output %.2e of scale  worst gradient %.2e of scale" % (
            str(dt).replace("torch.", ""), abs(loss.item() - rl.item()) / abs(rl.item()),
            float((pred.detach().double() - rp.detach().double()).abs().max()) / float(rp.detach().double().abs().max()),
            gerr))
    return out


def main():
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    name, pl = card()
    lib = L.load()
    ub, bb, nc = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    rc = lib.b200asr_bilstm_plan(B, E, 1, ctypes.byref(ub), ctypes.byref(bb), ctypes.byref(nc))
    print("card: %s, power limit %s" % (name, pl))
    print("recurrence (B=%d, H=%d, ndir=1): plan rc=%d unit_block=%d batch_block=%d ctas=%d; tensor-core step GEMMs=%d; "
          "wgmma forward=%d" % (B, E, rc, ub.value, bb.value, nc.value, lib.b200asr_bilstm_uses_tensor_cores(B, E, 1),
                                lib.b200asr_bilstm_uses_tcgen05(B, E, 1)), flush=True)
    for line in parity(60):
        print("parity vs oracle (T<=60, dropout 0) " + line, flush=True)
    _, step = ours()
    ref_step = library()
    for T in TS:
        x, lens, y = batch(T)
        for s in (step, ref_step):
            timed(s, (x, lens, y), WARMUP)
        ms_o, ms_l = [], []
        for r in range(ROUNDS):
            ms_o.append(timed(step, (x, lens, y), STEPS))
            ms_l.append(timed(ref_step, (x, lens, y), STEPS))
        # kernel split of one step, in a separate pass
        L.TIMER.enabled = True
        L.TIMER.reset()
        parts = []
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step(x, lens, y, parts)
        b.record()
        torch.cuda.synchronize()
        L.TIMER.enabled = False
        summ = L.TIMER.summary()
        total = a.elapsed_time(b)
        groups = {"recurrence": ("bilstm_fwd", "bilstm_bwd"), "GEMMs": ("gemm3x_tn", "gemm3x_nn", "gemm3x_nt",
                                                                         "tf32_residual"),
                  "CE": ("ce_fwd_bwd",), "embedding": ("embedding_bwd",)}
        split = {g: sum(summ[k]["ms"] for k in ks if k in summ) for g, ks in groups.items()}
        split["norm+clip+Adam"] = parts[0][0].elapsed_time(parts[0][1])
        split["other"] = total - sum(split.values())
        best_o, best_l = min(ms_o), min(ms_l)
        print("T=%d B=%d: ours %.2f ms/step (%s) = %.0f tokens/s | library %.2f ms/step (%s) = %.0f tokens/s" % (
            T, B, best_o, " ".join("%.2f" % v for v in ms_o), B * T / best_o * 1e3, best_l,
            " ".join("%.2f" % v for v in ms_l), B * T / best_l * 1e3))
        print("  split of one step (%.2f ms, events around every kernel call): %s" % (total, "  ".join(
            "%s %.2f ms (%.0f%%)" % (k, v, 100 * v / total) for k, v in split.items())), flush=True)


if __name__ == "__main__":
    main()
