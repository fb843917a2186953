"""Float64 restatement of the persistent (Bi)LSTM recurrence at the C ABI of b200asr_bilstm_fwd / _bwd, and helpers
around the variant query b200asr_debug_lstm_variant (test infrastructure, NOT a product path).

ABI layout: pre-activations and the activated-gate stash `gates [ndir, B, T, H, 4]` (gate-interleaved i, f, g, o),
W_hh `[ndir, 4H, H]` (PyTorch's gate-major rows g*H + j), cell-state stash `cstate [ndir, B, T, H]`, output
`out [B, T, ndir*H]`; direction 1 runs in reverse time; zero initial state.  The backward overwrites `gates` with
dG = d(loss)/d(pre-activation) for loss = sum(out * dout).
"""
import ctypes

import torch

VARIANT_FIELDS = ("gen", "UB", "UBP", "poll", "strict", "nsplit", "form", "R", "vec")
GEN = {1: "wgmma", 2: "mma.sync", 3: "fma"}
# debug modes the dispatcher knows (include/b200asr_debug.h): 0 default, 1 FMA only, 3 no wgmma, 256 strict acquire
SWEEP_MODES = (0, 1, 3, 256)
SWEEP_B = (1, 2, 3, 4, 5, 8, 9, 16, 24, 32, 33, 40, 48, 64, 96, 128, 130, 192, 256)
SWEEP_H = tuple(range(16, 1025, 16))


def variant(lib, B, H, ndir, bwd, mode=0):
    """The step-kernel variant b200asr_bilstm_fwd (bwd=False) / _bwd runs under `mode`, as a dict; None: no plan."""
    d = (ctypes.c_int * len(VARIANT_FIELDS))()
    lib.b200asr_debug_set_lstm_mode(mode)
    try:
        rc = lib.b200asr_debug_lstm_variant(B, H, ndir, 1 if bwd else 0, d)
    finally:
        lib.b200asr_debug_set_lstm_mode(0)
    return dict(zip(VARIANT_FIELDS, d)) if rc == 0 else None


def label(v, bwd):
    """Short name of a variant, e.g. 'wgmma12/flag+strict', 'mma.sync<2>', 'fma2x8/vec x2' (x2: two launches)."""
    if v["gen"] == 1:
        s = "wgmma%d/%s%s" % (v["UBP"], "poll" if v["poll"] else "flag", "+strict" if v["strict"] else "")
        if not bwd:
            s += "/vec" if v["vec"] else "/scalar"
    elif v["gen"] == 2:
        s = "mma.sync" if bwd else ("mma.sync/v2", "mma.sync<1>", "mma.sync<2>")[v["form"]]
    else:
        s = "fma%dx%d" % (v["form"], v["R"]) + (("/vec" if v["vec"] else "/scalar") if bwd else "")
    return s + (" x%d" % v["nsplit"] if v["nsplit"] > 1 else "")


def features(v, bwd):
    """The code paths a variant selects, one tuple each: the kernel instance (wgmma template x protocol, mma.sync loop
    form, FMA halves x tile rows), the runtime branches inside it (strict acquire, vectorised stores) and whether the
    batch runs as several launches."""
    side = "bwd" if bwd else "fwd"
    gen = GEN[v["gen"]]
    f = {(side, gen, "split", v["nsplit"] > 1)}
    if v["gen"] == 1:
        f.add((side, gen, "instance", v["UBP"], v["poll"]))
        if not v["poll"]:
            f.add((side, gen, "strict", v["strict"]))
        if not bwd:
            f.add((side, gen, "vec", v["vec"]))
    elif v["gen"] == 2:
        f.add((side, gen, "form", v["form"]))
    else:
        f.add((side, gen, "NH,R", v["form"], v["R"]))
        if bwd:
            f.add((side, gen, "vec", v["vec"]))
    return f


def case_features(lib, B, H, ndir, mode):
    out = set()
    for bwd in (False, True):
        v = variant(lib, B, H, ndir, bwd, mode)
        assert v is not None, (B, H, ndir, mode)
        out |= features(v, bwd)
    return out


def sweep_features(lib):
    """Every code path the dispatcher reaches over a broad (B, H, ndir, mode) sweep."""
    out = set()
    for mode in SWEEP_MODES:
        for H in SWEEP_H:
            for B in SWEEP_B:
                for ndir in (1, 2):
                    for bwd in (False, True):
                        v = variant(lib, B, H, ndir, bwd, mode)
                        if v is not None:
                            out |= features(v, bwd)
    return out


def recurrence(pre, whh, dout=None, dtype=torch.float64):
    """The recurrence in `dtype` on the CPU: (out, cstate, gates, dG); dG is None without `dout`.
    pre [ndir, B, T, H, 4], whh [ndir, 4H, H], dout [B, T, ndir*H]."""
    ndir, B, T, H, _ = pre.shape
    p = pre.detach().to("cpu", dtype).clone().requires_grad_(dout is not None)
    w = whh.detach().to("cpu", dtype)
    outs, csts, gts = [], [], []
    for d in range(ndir):
        frames = p[d].unbind(1)             # one backward node for all T frames, not a full-size slice gradient each
        h = torch.zeros(B, H, dtype=dtype)
        c = torch.zeros(B, H, dtype=dtype)
        o_t, c_t, g_t = [None] * T, [None] * T, [None] * T
        for step in range(T):
            t = step if d == 0 else T - 1 - step
            z = frames[t] + (h @ w[d].t()).view(B, 4, H).transpose(1, 2)
            i, f, g, o = torch.sigmoid(z[..., 0]), torch.sigmoid(z[..., 1]), torch.tanh(z[..., 2]), torch.sigmoid(z[..., 3])
            c = f * c + i * g
            h = o * torch.tanh(c)
            o_t[t], c_t[t], g_t[t] = h, c, torch.stack([i, f, g, o], -1)
        outs.append(torch.stack(o_t, 1))
        csts.append(torch.stack(c_t, 1))
        gts.append(torch.stack(g_t, 1))
    out = torch.cat(outs, -1)
    dG = None
    if dout is not None:
        (out * dout.detach().to("cpu", dtype)).sum().backward()
        dG = p.grad.detach()
    return out.detach(), torch.stack(csts).detach(), torch.stack(gts).detach(), dG
