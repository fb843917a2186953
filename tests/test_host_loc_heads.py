"""Multi-head location-aware attention, CPU side: the float64 oracle (oracle/attn_heads_ref.py) against float64
autograd of the reference's expressions, its bound against three planted defects, argument refusal before any CUDA
call, the Python limits against the library's, the golden models' parameter contract, and no local memory in the
shipped kernels."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, load_golden
from oracle import attn_heads_ref as hr
from oracle.attn_ref import worst_ratio
from oracle.make_golden_locheads import locheads_model_cfg

SO = os.path.join(ROOT, "end-to-end-asr-pytorch_b200", "libb200asr.so")
FAKE = ctypes.c_void_p(256)          # never dereferenced: every call below is refused by the argument checks


def loc_heads_torch(q, key, value, prev, lens, wc, wp, we, be, temp, N, defect=None):
    """The reference's LocationAwareAttention.forward + _attend (src/module.py:189-195, 234-258) with N heads, rows
    r = b*N + n masked by lens[r // N].  defect: 'dloc_head0' (d(loc) from head 0 only), 'mask_mod' (row r masked by
    lens[r mod B]), 'conv_order' (the [K, N, W] conv weight read as [N, K, W])."""
    B, _, T = prev.shape
    K, _, W = wc.shape
    D = wp.shape[0]
    if defect == "conv_order":
        wc = wc.reshape(-1).view(N, K, W).transpose(0, 1)
    loc = torch.tanh(F.linear(F.conv1d(prev, wc, padding=(W - 1) // 2).transpose(1, 2), wp))    # [B, T, D]
    if defect == "dloc_head0":
        loc = torch.cat([loc.unsqueeze(1), loc.detach().unsqueeze(1).expand(B, N - 1, T, D)], 1)
    else:
        loc = loc.unsqueeze(1).repeat(1, N, 1, 1)
    loc = loc.reshape(-1, T, D)
    energy = F.linear(torch.tanh(key + q.unsqueeze(1) + loc), we.view(1, -1), be.view(1)).squeeze(2)
    rows = torch.arange(B * N)
    rlens = lens[rows % B] if defect == "mask_mod" else lens[rows // N]
    mask = torch.arange(T)[None, :] >= rlens[:, None]
    a = torch.softmax((energy / temp).masked_fill(mask, float("-inf")), -1)
    return torch.bmm(a.unsqueeze(1), value).squeeze(1), a


def _case(B, N, T, D, E, K, R, repeat, seed):
    g = torch.Generator().manual_seed(seed)
    mk = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc).double()
    lens = torch.linspace(T, 2, B).round().long()
    value = mk(B, T, E).repeat(N, 1, 1) if repeat else mk(B * N, T, E)
    prev = torch.softmax(mk(B, N, T), -1) * (torch.arange(T)[None, None] < lens[:, None, None])
    return dict(q=mk(B * N, D), key=mk(B * N, T, D), value=value, prev=prev, lens=lens,
                wc=mk(K, N, 2 * R + 1, sc=0.5), wp=mk(D, K, sc=0.5), we=mk(D, sc=0.5), be=mk(1), dctx=mk(B * N, E),
                dattn=mk(B * N, T))


def _autograd(c, N, temp, defect=None):
    leaves = {k: c[k].clone().requires_grad_(True) for k in ("q", "key", "value", "prev", "wc", "wp", "we", "be")}
    ctx, a = loc_heads_torch(leaves["q"], leaves["key"], leaves["value"], leaves["prev"], c["lens"], leaves["wc"],
                             leaves["wp"], leaves["we"], leaves["be"], temp, N, defect)
    ((ctx * c["dctx"]).sum() + (a * c["dattn"]).sum()).backward()
    out = {"ctx": ctx.detach(), "attn": a.detach()}
    out.update({"d" + k: v.grad for k, v in leaves.items()})
    return {k: v.numpy() for k, v in out.items()}


def _oracle(c, N, temp):
    n = lambda k: c[k].numpy()
    return hr.loc_heads_step(n("q"), n("key"), n("value"), n("prev"), c["lens"].numpy(), n("wc"), n("wp"), n("we"),
                             n("be"), temp, N, dctx=n("dctx"), dattn=n("dattn"))


PAIRS = [("ctx", "ctx", None), ("attn", "attn", None), ("dq", "dq", None), ("dkey", "dkey", None),
         ("dvalue", "dvalue", None), ("dprev", "dprev", None), ("dwc", "dwc", 0), ("dwp", "dwp", 0),
         ("dwe", "dwe", 0), ("dbe", "dbe", 0)]


def _oracle_value(st, name, reduce_axis):
    v = getattr(st, name)
    return v.sum(reduce_axis) if reduce_axis is not None else v


@pytest.mark.parametrize("N,repeat", [(2, False), (3, False), (2, True), (3, True)])
def test_oracle_equals_float64_autograd(N, repeat):
    B, T, D, E, K, R, temp = 3, 23, 12, 8, 4, 3, 0.5
    c = _case(B, N, T, D, E, K, R, repeat, seed=N * 10 + repeat)
    ref = _autograd(c, N, temp)
    st = _oracle(c, N, temp)
    for mine, theirs, ax in PAIRS:
        got = _oracle_value(st, mine, ax)
        exp = ref[theirs].reshape(got.shape)
        valid = st.valid[:, :, None] if mine in ("dkey", "dvalue") else True
        exp = np.where(valid, exp, 0.0)             # the reference's padded-frame gradients are exact zeros too
        comp = _oracle_value(st, mine + "_abs", ax) if hasattr(st, mine + "_abs") else exp
        scale = max(float(np.abs(exp).max()), float(np.abs(comp).max()))    # d(b_e) is 0 up to cancellation
        assert float(np.abs(got - exp).max()) <= 1e-12 * scale, mine


@pytest.mark.parametrize("defect,outputs", [("dloc_head0", ("dprev", "dwp", "dwc")), ("mask_mod", ("attn", "ctx")),
                                            ("conv_order", ("attn", "dwc"))])
def test_bound_catches_planted_defects(defect, outputs):
    """Each defect, computed in float64, is outside the fp32 bound of an output it corrupts by a wide margin."""
    N, B, T, D, E, K, R, temp = 2, 3, 23, 12, 8, 4, 3, 0.5
    c = _case(B, N, T, D, E, K, R, False, seed=5)
    st = _oracle(c, N, temp)
    bad = _autograd(c, N, temp, defect)
    for name in outputs:
        ax = 0 if name in ("dwp", "dwc", "dwe", "dbe") else None
        exact = _oracle_value(st, name, ax)
        bound = _oracle_value(st, name + "_b", ax)
        assert worst_ratio(bad[name].reshape(exact.shape), exact, bound) > 10, (defect, name)


def _fwd(lib, ptrs, B, N, T, D, E, K, R):
    q, k, v, pv, ln, wc, wp, we, be, a, c = ptrs
    return lib.b200asr_locattn_heads_fwd(q, k, v, pv, ln, wc, wp, we, be, 0.5, B, N, T, D, E, K, R, a, c, None)


def _bwd(lib, ptrs, B, N, T, D, E, K, R):
    q, k, v, pv, ln, wc, wp, we, a, dc, dq, dk, dp, wpart = ptrs
    return lib.b200asr_locattn_heads_bwd_acc(q, k, v, pv, ln, wc, wp, we, 0.5, a, dc, None, B, N, T, D, E, K, R, dq, dk,
                                             dp, wpart, None)


@pytest.mark.parametrize("which", ["fwd", "bwd"])
def test_null_pointers_and_bad_sizes_are_refused(pkg, which):
    lib = pkg.load_library()
    call, n = (_fwd, 11) if which == "fwd" else (_bwd, 14)
    name = "locattn_heads_fwd" if which == "fwd" else "locattn_heads_bwd_acc"
    n0 = pkg.lib.launch_count()
    for i in range(n):
        ptrs = [FAKE] * n
        ptrs[i] = None
        assert call(lib, ptrs, 2, 2, 16, 8, 8, 4, 3) == -1
        assert pkg.lib.last_error() == "%s: null pointer" % name
    ptrs = [FAKE] * n
    for args, msg in [((0, 2, 16, 8, 8, 4, 3), "bad sizes"), ((2, 0, 16, 8, 8, 4, 3), "bad sizes"),
                      ((2, 2, 0, 8, 8, 4, 3), "bad sizes"), ((2, 2, 16, 0, 8, 4, 3), "bad sizes"),
                      ((2, 2, 16, 8, 0, 4, 3), "bad sizes"), ((2, 2, 16, 8, 8, 0, 3), "bad sizes"),
                      ((2, 2, 16, 8, 8, 4, -1), "bad sizes"), ((2, 17, 16, 8, 8, 4, 3), "at most 16 heads"),
                      ((2, 2, 16, 8, 8, 17, 3), "at most 16 location kernels"),
                      ((2, 2, 16, 513, 8, 4, 3), "attention dim 513 > 512"), ((2, 2, 16, 8, 6, 4, 3), "multiple of 4"),
                      ((2, 2, 149, 8, 4104, 4, 3), "too large"), ((2, 4, 20000, 300, 2048, 10, 100), "shared memory")]:
        assert call(lib, ptrs, *args) == -1, args
        err = pkg.lib.last_error()
        assert err.startswith(name + ":") and msg in err, (args, err)
    assert pkg.lib.launch_count() == n0


def _longest_t(supported, N, D, E, K, R):
    lo, hi = 1, 1 << 20
    assert supported(N, lo, D, E, K, R) and not supported(N, hi, D, E, K, R)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if supported(N, mid, D, E, K, R) else (lo, mid)
    return lo


def test_python_limits_follow_the_library(pkg):
    """ops.loc_attention_heads_supported equals b200asr_locattn_heads_supported over a grid of shapes and at the
    longest memory each head count takes; the first memory refused is refused by both entry points."""
    lib = pkg.load_library()
    py = pkg.ops.loc_attention_heads_supported
    for N in (0, 1, 2, 4, 8, 16, 17):
        for T in (1, 7, 16, 149, 1000):
            for D in (1, 300, 512, 513):
                for E in (4, 6, 2048, 4100):
                    for K, R in ((1, 0), (10, 100), (16, 5), (17, 5)):
                        assert py(N, T, D, E, K, R) == bool(lib.b200asr_locattn_heads_supported(N, T, D, E, K, R)), \
                            (N, T, D, E, K, R)
    D, E, K, R = 300, 2048, 10, 100                 # cfg C's attention
    assert not py(16, 1, D, E, K, R)                # 16 heads' K N (2R+1) conv taps alone take 126 KB
    for N in (2, 4, 8):
        T = _longest_t(py, N, D, E, K, R)
        assert lib.b200asr_locattn_heads_supported(N, T, D, E, K, R) == 1
        assert lib.b200asr_locattn_heads_supported(N, T + 1, D, E, K, R) == 0
        assert _fwd(lib, [FAKE] * 11, 2, N, T + 1, D, E, K, R) == -1
        assert _bwd(lib, [FAKE] * 14, 2, N, T + 1, D, E, K, R) == -1
        assert "shared memory" in pkg.lib.last_error()
    assert py(4, 149, D, E, K, R) and py(8, 149, D, E, K, R)


@pytest.mark.parametrize("kind", ["loc2", "locrep"])
def test_golden_models_have_the_model_state_dict(pkg, kind):
    g = load_golden("model_%s.npz" % kind)
    model = pkg.ASR(g["feat"].shape[-1], g["sd.pre_embed.weight"].shape[0], True, **locheads_model_cfg(kind))
    ref = {k[3:]: tuple(v.shape) for k, v in g.items() if k.startswith("sd.")}
    assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == ref
    att = model.attention
    assert att.mode == "loc" and att.num_head == (2 if kind == "loc2" else 4)
    assert att.v_proj == (kind == "loc2")
    assert ref["attention.att_layer.loc_conv.weight"][1] == att.num_head       # [K, N, 2R+1]
    assert g["att_seq"].shape[1] == att.num_head                               # [B, N, L, T]
    if kind == "locrep":           # the repeat reaches another utterance only with more than one utterance per batch
        assert g["feat"].shape[0] >= 3 and len(set(g["encode_len"].tolist())) == g["feat"].shape[0]


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="needs cuobjdump")
@pytest.mark.skipif(not os.path.exists(SO), reason="library not built (run __graft_entry__.build())")
def test_loc_heads_kernels_are_shipped_without_local_memory():
    out = subprocess.run(["cuobjdump", "-res-usage", SO], capture_output=True, text=True, check=True).stdout
    found = {}
    for m in re.finditer(r"Function (\S*locattn_heads_\w*kernel\S*):\s*\n\s*(REG:.*)", out):
        found[m.group(1)] = dict(kv.split(":") for kv in m.group(2).split())
    names = sorted(found)
    assert len(names) == 3 and sum("locattn_heads_fwd_kernel" in n for n in names) == 1, names   # fwd, bwd<1>, bwd<2>
    for n, r in found.items():
        assert r["STACK"] == "0" and r["LOCAL"] == "0", (n, r)
